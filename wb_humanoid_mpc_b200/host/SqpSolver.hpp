// Host layer: the reference's solver interface (ocs2::SqpSolver, lib/ocs2_ros2/ocs2_sqp/ocs2_sqp/include/ocs2_sqp/SqpSolver.h:60-103 and
// SolverBase.h:78-140) for a BATCH of independent humanoid whole-body MPC instances, implemented over the C ABI of libb200sqp.so.
//
//   SqpSolver(settings, optimalControlProblem, initializer)   ->  SqpSolver(model, settings, batch, device)
//   reset()                                                   ->  reset()                 drops every instance's primal solution
//   run(initTime, initState, finalTime)                       ->  run(initTime, initStates[B], finalTime)
//   getReferenceManager()                                     ->  getReferenceManager(b)  per-instance gait / target trajectories
//   getPrimalSolution(finalTime, PrimalSolution*)             ->  primalSolution(b)
//   getPerformanceIndeces() / getIterationsLog()              ->  getIterationsLog(b)
//   getNumIterations()                                        ->  getNumIterations(b)
//   getBenchmarks()                                           ->  getBenchmarks()
//   getValueFunction(t, x)                                    ->  getValueFunction(b, t, x)   (settings.create_value_function)
//   getHamiltonian / getStateInputEqualityConstraintLagrangian / getIntermediateDualSolution throw, as in the reference (SqpSolver.h:82-92)
// Errors are C++ exceptions as in the reference: std::runtime_error on a failed QP or a failing library call (SqpSolver.cpp:166,306-308).
//
// Instances whose time grids have different numbers of shooting nodes (different gait phases put different numbers of event nodes inside
// the horizon) are grouped by node count; each group owns one library handle and is solved with one b200sqp_solve.
// The per-instance host work (reference manager, time grid, warm start) runs on a pool of std::threads.
#pragma once
#include <chrono>
#include <map>
#include <mutex>
#include <memory>
#include <thread>

#include "references.hpp"

namespace b200sqp::host {

struct PerformanceIndex {  // ocs2_oc/include/ocs2_oc/oc_data/PerformanceIndex.h:42-98 (the fields the SQP path fills)
  double merit = 0, cost = 0, dynamicsViolationSSE = 0, equalityConstraintsSSE = 0;
};
struct StepInfo {  // sqp::StepInfo (SqpSolverStatus.h:42-57)
  double stepSize = 0;
  int stepType = 0;  // FilterLinesearch::StepType: 0 UNKNOWN 1 CONSTRAINT 2 DUAL 3 COST 4 ZERO
  double dx_norm = 0, du_norm = 0, armijoDescentMetric = 0;
  PerformanceIndex baseline, performanceAfterStep;
  int convergence = 0;  // sqp::Convergence: 0 FALSE 1 ITERATIONS 2 STEPSIZE 3 METRICS 4 PRIMAL
};
struct Benchmarks {  // SqpSolver::getBenchmarks (ms of the last run, summed over node-count groups)
  double linearQuadraticApproximation = 0, solveQp = 0, linesearch = 0, projectionShareOfLq = 0;
  // host wall-clock split of the last run(): preRun (reference managers, time grids, warm start), packing into the staging arrays,
  // b200sqp_upload_instances, b200sqp_solve, b200sqp_download, unpacking into PrimalSolution / iteration logs
  double hostPreRun = 0, hostPack = 0, upload = 0, solve = 0, download = 0, hostUnpack = 0;
};
struct ValueFunction {  // ScalarFunctionQuadraticApproximation of getValueFunction: dfdxx (nx*nx, column-major), dfdx
  vector_t dfdxx, dfdx;
};

class SqpSolver {
 public:
  SqpSolver(const HostModel& model, const b200sqp_settings& settings, int batch, int device = 0, int hostThreads = 0)
      : model_(model), settings_(settings), device_(device), batch_(batch) {
    if (batch < 1) throw std::invalid_argument("[b200sqp::host::SqpSolver] batch must be >= 1");
    for (int b = 0; b < batch; ++b) rm_.emplace_back(model_);
    motion_.resize(batch);
    motionStarted_.assign(batch, 0);
    primal_.resize(batch);
    log_.resize(batch);
    groupOf_.assign(batch, -1);
    slotOf_.assign(batch, -1);
    const unsigned hw = std::thread::hardware_concurrency();
    threads_ = hostThreads > 0 ? hostThreads : static_cast<int>(std::max(1u, std::min(hw ? hw : 1u, 16u)));   // per-instance host work is light: more threads only add spawn cost
  }
  ~SqpSolver() {
    for (auto& g : groups_) {
      g.second.st.release();
      if (g.second.h) b200sqp_destroy(g.second.h);
    }
  }
  SqpSolver(const SqpSolver&) = delete;
  SqpSolver& operator=(const SqpSolver&) = delete;

  int batch() const { return batch_; }
  // the reference always spreads the previous solution over the new mode schedule (SqpSolver.cpp:211-213); see trajectorySpread's note on the
  // time-stamp convention clash it inherits -- switching it off keeps the previous solution's time stamps untouched
  void setTrajectorySpread(bool on) { trajectorySpread_ = on; }
  SwitchedModelReferenceManager& getReferenceManager(int b) { return rm_.at(b); }
  // per-instance gait command (the synchronized gait module): a command set before run() of cycle c shows in the schedule of cycle c + 1
  void setGaitCommand(int b, const std::string& gait) { rm_.at(b).setGaitCommand(gait); }
  // automatic gait selection: instance b runs ProceduralMpcMotionManager as its synchronized module from the next run() on (its first run takes
  // the targets of its own filtered command and evaluates no transition); the state starts at initialGait's row.  The gait schedule itself
  // is set with getReferenceManager(b).setGait as usual.
  void enableMotionManager(int b, double filterOrigin, const std::string& initialGait = "stance") {
    motion_.at(b) = std::make_unique<ProceduralMpcMotionManager>(model_, filterOrigin, initialGait);
    motionStarted_.at(b) = 0;
  }
  void disableMotionManager(int b) { motion_.at(b).reset(); }
  // the raw WalkingVelocityCommand message (v_x, v_y, pelvis height, yaw rate) of instance b's motion manager
  void setVelocityCommand(int b, const std::array<double, 4>& cmd) {
    if (!motion_.at(b)) throw std::invalid_argument("[b200sqp::host::SqpSolver] setVelocityCommand: enableMotionManager first");
    motion_[b]->setVelocityCommand(cmd);
  }
  const ProceduralMpcMotionManager* motionManager(int b) const { return motion_.at(b).get(); }

  void reset() {  // SqpSolver::reset (SqpSolver.cpp:96-106): forget the previous solutions -> the next run is a cold start
    for (auto& p : primal_) p.clear();
    for (auto& l : log_) l.clear();
  }

  // SolverBase::run(initTime, initState, finalTime) for all instances: preRun (reference managers), runImpl on the GPU, postRun bookkeeping
  void run(double initTime, const std::vector<vector_t>& initStates, double finalTime) {
    if (static_cast<int>(initStates.size()) != batch_) throw std::invalid_argument("[b200sqp::host::SqpSolver] run: one initial state per instance");
    std::vector<Instance> inst(batch_);
    bench_ = Benchmarks();
    failedInstances_.clear();
    const auto tPre = now();
    // centroidal motion managers: Ab^-1 hbar of the measured states for their target rule (device calls, made here from one thread)
    std::vector<std::array<double, 6>> baseVel(batch_);
    if (model_.centroidal)
      for (int b = 0; b < batch_; ++b)
        if (motion_[b]) baseVel[b] = centroidalBaseVelocity(model_, initStates[b], device_);
    parallelFor(batch_, [&](int b) {
      if (motion_[b] && motionStarted_[b]) rm_[b].setTargetTrajectories(motion_[b]->buffer());   // ReferenceManager::preSolverRun takes the buffer
      rm_[b].preSolverRun(initTime, finalTime);
      // synchronized modules after the reference manager (SolverBase.cpp:95-101)
      const std::array<double, 6>* bv = model_.centroidal ? &baseVel[b] : nullptr;
      if (motion_[b] && !motionStarted_[b]) {
        rm_[b].setTargetTrajectories(motion_[b]->start(initTime, finalTime, initStates[b], bv));
        motionStarted_[b] = 1;
      } else if (motion_[b]) {
        motion_[b]->preSolverRun(initTime, finalTime, initStates[b], bv);
        if (motion_[b]->gaitCommandChanged()) rm_[b].setGaitCommand(motion_[b]->gaitCommand());
      }
      rm_[b].applyGaitCommand(initTime, finalTime);
      // Trajectory spread of primalSolution_ (SqpSolver.cpp:211-213)
      if (trajectorySpread_ && !primal_[b].timeTrajectory_.empty()) trajectorySpread(primal_[b].modeSchedule_, rm_[b].getModeSchedule(), primal_[b]);
      const PrimalSolution* prev = primal_[b].timeTrajectory_.empty() ? nullptr : &primal_[b];
      inst[b] = buildInstance(model_, rm_[b], initTime, initStates[b], finalTime, model_.dt, prev);
    });
    // group by node count
    std::map<int, std::vector<int>> members;
    for (int b = 0; b < batch_; ++b) members[inst[b].n_nodes()].push_back(b);
    bench_.hostPreRun = since(tPre);
    // A receding horizon walks through a handful of node counts (115..117 for `walk`); random schedules could visit many more. Every group
    // owns device buffers sized for its batch, so groups this solve does not use are dropped once more than kMaxGroups are held.
    if (groups_.size() + members.size() > static_cast<size_t>(kMaxGroups))
      for (auto it = groups_.begin(); it != groups_.end();) {
        if (members.count(it->first) == 0 && groups_.size() > members.size()) {
          it->second.st.release();
          if (it->second.h) b200sqp_destroy(it->second.h);
          it = groups_.erase(it);
        } else {
          ++it;
        }
      }
    if (members.size() == 1 || exclusiveSolve_) {
      for (auto& kv : members) solveGroup(kv.first, kv.second, inst);
      return;
    }
    // several node-count groups (mixed contact schedules): every group has its own handle and CUDA stream, so the groups are driven by one
    // host thread each and their kernels overlap on the device -- small groups alone would leave most SMs idle
    for (auto& kv : members) groups_[kv.first];   // create the map nodes up front: the threads only look them up
    std::vector<std::thread> pool;
    std::vector<std::exception_ptr> err(members.size());
    size_t gi = 0;
    for (auto& kv : members) {
      pool.emplace_back([this, &kv, &inst, &err, gi] {
        try {
          solveGroup(kv.first, kv.second, inst);
        } catch (...) {
          err[gi] = std::current_exception();
        }
      });
      ++gi;
    }
    for (auto& th : pool) th.join();
    for (auto& e : err)
      if (e) std::rethrow_exception(e);
  }

  // see solveGroup: serialise the device phase of this object with every other SqpSolver of the process that also opted in
  void setExclusiveSolve(bool on) { exclusiveSolve_ = on; }

  // problemPtr_->costPtr->add("jointTorqueCost", getJointTorqueCost(taskFile)) (WBMpcInterface.cpp): the joint-torque cost on every intermediate
  // node of every instance, weights [nj] in MPC joint order (loadJointTorqueWeights); empty or all zeros: off.  Whole-body models only.
  void setJointTorqueCost(const std::vector<double>& weights) {
    if (!weights.empty() && static_cast<int>(weights.size()) != model_.nj)
      throw std::invalid_argument("[SqpSolver] setJointTorqueCost: " + std::to_string(weights.size()) + " weights for " + std::to_string(model_.nj) + " joints");
    for (auto& kv : groups_)
      if (kv.second.h) check(b200sqp_set_joint_torque_cost(kv.second.h, weights.empty() ? nullptr : weights.data()));
    jointTorqueWeights_ = weights;
  }

  const PrimalSolution& primalSolution(int b) const { return primal_.at(b); }
  const std::vector<StepInfo>& getIterationsLog(int b) const {
    if (log_.at(b).empty()) throw std::runtime_error("[SqpSolver]: No performance log yet, no problem solved yet?");  // SqpSolver.cpp:174
    return log_[b];
  }
  size_t getNumIterations(int b) const { return log_.at(b).size(); }
  Benchmarks getBenchmarks() const { return bench_; }

  // getValueFunction(time, state) (SqpSolver.cpp:172-191): P, p interpolated in time, then re-centred at `state`
  ValueFunction getValueFunction(int b, double time, const vector_t& state) const {
    if (!settings_.create_value_function) throw std::runtime_error("[SqpSolver] createValueFunction is false");
    const int g = groupOf_.at(b);
    if (g < 0) throw std::runtime_error("[SqpSolver] getValueFunction: no problem solved yet");
    const auto git = groups_.find(g);
    if (git == groups_.end()) throw std::runtime_error("[SqpSolver] getValueFunction: the handle of this instance's last successful solve was released");
    const Group& G = git->second;
    const int nx = model_.nx, n = G.nNodes, s = slotOf_[b];
    const vector_t& tt = primal_[b].timeTrajectory_;
    // LinearInterpolation over the node times
    const int index = static_cast<int>(lowerBoundIndex(tt, time)) - 1, last = n - 1;
    int idx = 0;
    double alpha = 1.0;
    if (index >= 0 && index < last) {
      const double len = tt[index + 1] - tt[index], till = tt[index + 1] - time;
      idx = index;
      alpha = len > 2.0 * kWeakEps ? till / len : (till < 0.5 * len ? 0.0 : 1.0);
    } else if (index >= last) {
      idx = std::max(last - 1, 0);
      alpha = 0.0;
    }
    ValueFunction v;
    v.dfdxx.resize(static_cast<size_t>(nx) * nx);
    v.dfdx.resize(nx);
    const double* P0 = G.P.data() + (static_cast<size_t>(s) * n + idx) * nx * nx;
    const double* p0 = G.p.data() + (static_cast<size_t>(s) * n + idx) * nx;
    for (int i = 0; i < nx * nx; ++i) v.dfdxx[i] = alpha * P0[i] + (1 - alpha) * P0[i + nx * nx];
    for (int i = 0; i < nx; ++i) v.dfdx[i] = alpha * p0[i] + (1 - alpha) * p0[i + nx];
    for (int i = 0; i < nx; ++i)
      for (int j = 0; j < nx; ++j) v.dfdx[i] += v.dfdxx[i + nx * j] * state[j];   // dfdx += dfdxx * x
    return v;
  }
  [[noreturn]] void getHamiltonian() const { throw std::runtime_error("[SqpSolver] getHamiltonian() not available yet."); }
  [[noreturn]] void getStateInputEqualityConstraintLagrangian() const {
    throw std::runtime_error("[SqpSolver] getStateInputEqualityConstraintLagrangian() not available yet.");
  }
  [[noreturn]] void getIntermediateDualSolution() const { throw std::runtime_error("[SqpSolver] getIntermediateDualSolution() not available yet."); }

 private:
  // page-locked staging arrays of one node-count group, allocated once per (batch, node count) and reused by every run
  struct Staging {
    double *x0 = nullptr, *xi = nullptr, *ui = nullptr, *tn = nullptr, *sw = nullptr, *imp = nullptr, *arm = nullptr, *xr = nullptr, *x = nullptr, *u = nullptr;
    uint8_t *ev = nullptr, *cf = nullptr;
    void release() {
      for (void* p : {static_cast<void*>(x0), static_cast<void*>(xi), static_cast<void*>(ui), static_cast<void*>(tn), static_cast<void*>(sw),
                      static_cast<void*>(imp), static_cast<void*>(arm), static_cast<void*>(xr), static_cast<void*>(x), static_cast<void*>(u),
                      static_cast<void*>(ev), static_cast<void*>(cf)})
        b200sqp_host_free(p);
      *this = Staging();
    }
  };
  struct Group {
    b200sqp_handle h = nullptr;
    int nNodes = 0, capacity = 0;
    Staging st;
    vector_t P, p;
  };
  template <class T>
  static T* pinned(size_t count) {
    T* p = static_cast<T*>(b200sqp_host_alloc(count * sizeof(T)));
    if (!p) throw std::runtime_error(std::string("[SqpSolver] ") + b200sqp_last_error());
    return p;
  }
  using clock_t_ = std::chrono::steady_clock;
  static clock_t_::time_point now() { return clock_t_::now(); }
  static double since(clock_t_::time_point t) { return std::chrono::duration<double, std::milli>(now() - t).count(); }
  static void check(int rc) {
    if (rc != 0) throw std::runtime_error(std::string("[SqpSolver] ") + b200sqp_last_error());
  }
  template <class F>
  void parallelFor(int n, F f) {
    const int nt = std::min(threads_, n);
    if (nt <= 1) {
      for (int i = 0; i < n; ++i) f(i);
      return;
    }
    std::vector<std::thread> pool;
    std::vector<std::exception_ptr> err(nt);
    for (int t = 0; t < nt; ++t)
      pool.emplace_back([&, t] {
        try {
          for (int i = t; i < n; i += nt) f(i);
        } catch (...) {
          err[t] = std::current_exception();
        }
      });
    for (auto& th : pool) th.join();
    for (auto& e : err)
      if (e) std::rethrow_exception(e);
  }

  void solveGroup(int nNodes, const std::vector<int>& members, const std::vector<Instance>& inst) {
    Group& G = groups_[nNodes];
    const int Bg = static_cast<int>(members.size()), nx = model_.nx, nu = model_.nu, n = nNodes;
    if (!G.h)
      check(model_.centroidal ? b200sqp_cen_create(&model_.desc, &model_.cen, &settings_, device_, &G.h)
                              : b200sqp_create(&model_.desc, &settings_, device_, &G.h));
    if (G.h && !jointTorqueWeights_.empty()) check(b200sqp_set_joint_torque_cost(G.h, jointTorqueWeights_.data()));
    const size_t B_ = static_cast<size_t>(Bg), n_ = static_cast<size_t>(n);
    if (G.capacity != Bg || G.nNodes != n) {
      // Invalidate first: if set_batch or a pinned allocation throws, the next call re-enters this branch
      // instead of reusing released (null) staging.
      G.capacity = 0;
      G.nNodes = 0;
      G.st.release();
      check(b200sqp_set_batch(G.h, Bg, n));
      Staging& S = G.st;
      S.x0 = pinned<double>(B_ * nx);
      S.xi = pinned<double>(B_ * n_ * nx);
      S.ui = pinned<double>(B_ * (n_ - 1) * nu);
      S.tn = pinned<double>(B_ * n_);
      S.sw = pinned<double>(B_ * n_ * 6);
      S.imp = pinned<double>(B_ * n_ * 2);
      S.arm = pinned<double>(B_ * n_);
      S.xr = pinned<double>(B_ * n_ * nx);
      S.x = pinned<double>(B_ * n_ * nx);
      S.u = pinned<double>(B_ * (n_ - 1) * nu);
      S.ev = pinned<uint8_t>(B_ * n_);
      S.cf = pinned<uint8_t>(B_ * n_ * 2);
      G.capacity = Bg;
      G.nNodes = n;
    }
    double *x0 = G.st.x0, *xi = G.st.xi, *ui = G.st.ui, *tn = G.st.tn, *sw = G.st.sw, *imp = G.st.imp, *arm = G.st.arm, *xr = G.st.xr;
    uint8_t *ev = G.st.ev, *cf = G.st.cf;
    auto tm = now();
    parallelFor(Bg, [&](int s) {
      const Instance& I = inst[members[s]];
      std::copy(I.x0.begin(), I.x0.end(), x0 + static_cast<size_t>(s) * nx);
      std::copy(I.x_init.begin(), I.x_init.end(), xi + static_cast<size_t>(s) * n * nx);
      std::copy(I.u_init.begin(), I.u_init.end(), ui + static_cast<size_t>(s) * (n - 1) * nu);
      std::copy(I.t_nodes.begin(), I.t_nodes.end(), tn + static_cast<size_t>(s) * n);
      std::copy(I.node_event.begin(), I.node_event.end(), ev + static_cast<size_t>(s) * n);
      std::copy(I.contact_flags.begin(), I.contact_flags.end(), cf + static_cast<size_t>(s) * n * 2);
      std::copy(I.swing_ref.begin(), I.swing_ref.end(), sw + static_cast<size_t>(s) * n * 6);
      std::copy(I.impact_factor.begin(), I.impact_factor.end(), imp + static_cast<size_t>(s) * n * 2);
      std::copy(I.arm_phase.begin(), I.arm_phase.end(), arm + static_cast<size_t>(s) * n);
      std::copy(I.x_ref.begin(), I.x_ref.end(), xr + static_cast<size_t>(s) * n * nx);
    });
    Benchmarks local;
    local.hostPack = since(tm);
    tm = now();
    check(b200sqp_upload_instances(G.h, x0, xi, ui, tn, ev, cf, sw, imp, arm, xr));
    local.upload = since(tm);
    tm = now();
    void* stream = nullptr;   // the handle's own non-blocking stream: several SqpSolver objects overlap on the device
    check(b200sqp_own_stream(G.h, &stream));
    if (exclusiveSolve_) {
      // double buffering with several SqpSolver objects: one solve on the GPU at a time, the others build / unpack their batches meanwhile.
      // Without the token concurrent solves share the GPU evenly, finish together and keep the objects in lock-step (host phases aligned,
      // GPU idle during them).
      std::lock_guard<std::mutex> token(deviceToken(device_));
      check(b200sqp_solve(G.h, stream));
      check(b200sqp_wait(G.h));   // the solve only enqueues (asynchronous): the token is kept until the device has finished it
    } else {
      check(b200sqp_solve(G.h, stream));
    }
    local.solve = since(tm);
    tm = now();
    double *x = G.st.x, *u = G.st.u;
    const int iters = settings_.sqp_iteration;
    std::vector<b200sqp_iter_log> log(static_cast<size_t>(Bg) * iters);
    std::vector<int32_t> nIter(Bg), status(Bg);
    // a failed QP of some instances (B200SQP_EQP) is a partial success: the arrays of every instance have been downloaded; the good ones are
    // unpacked below (their warm starts stay valid), the failed ones keep their previous primal solution, and the call throws afterwards
    const int rcDownload = b200sqp_download(G.h, x, u, nullptr, log.data(), nIter.data(), status.data());
    if (rcDownload != 0 && rcDownload != B200SQP_EQP) check(rcDownload);
    if (settings_.create_value_function) {
      G.P.resize(static_cast<size_t>(Bg) * n * nx * nx);
      G.p.resize(static_cast<size_t>(Bg) * n * nx);
      check(b200sqp_download_value_function(G.h, G.P.data(), G.p.data()));
    }
    local.download = since(tm);
    tm = now();
    float ms[4];
    check(b200sqp_get_stage_times(G.h, ms));
    local.linearQuadraticApproximation = ms[0];
    local.solveQp = ms[1];
    local.linesearch = ms[2];
    local.projectionShareOfLq = ms[3];
    int nFailed = 0;
    for (int s = 0; s < Bg; ++s) nFailed += status[s] != 0;
    const int gid = nNodes;
    parallelFor(Bg, [&](int s) {
      const int b = members[s];
      if (status[s] != 0) return;   // keeps primal_[b] / log_[b] of its last successful solve
      groupOf_[b] = gid;
      slotOf_[b] = s;
      primal_[b] = toPrimalSolution(inst[b], x + static_cast<size_t>(s) * n * nx, u + static_cast<size_t>(s) * (n - 1) * nu, nx, nu);
      log_[b].clear();
      for (int it = 0; it < nIter[s]; ++it) {
        const b200sqp_iter_log& L = log[static_cast<size_t>(s) * iters + it];
        StepInfo si;
        si.stepSize = L.step_size;
        si.stepType = static_cast<int>(L.step_type);
        si.dx_norm = L.dx_norm;
        si.du_norm = L.du_norm;
        si.armijoDescentMetric = L.armijo;
        si.baseline = PerformanceIndex{L.base_merit, L.base_cost, L.base_dyn_sse, L.base_eq_sse};
        si.performanceAfterStep = PerformanceIndex{L.merit, L.cost, L.dyn_sse, L.eq_sse};
        si.convergence = static_cast<int>(L.convergence);
        log_[b].push_back(si);
      }
    });
    local.hostUnpack = since(tm);
    std::lock_guard<std::mutex> lk(benchMutex_);   // groups may run on concurrent host threads
    bench_.hostPack += local.hostPack;
    bench_.upload += local.upload;
    bench_.solve += local.solve;
    bench_.download += local.download;
    bench_.hostUnpack += local.hostUnpack;
    bench_.linearQuadraticApproximation += local.linearQuadraticApproximation;
    bench_.solveQp += local.solveQp;
    bench_.linesearch += local.linesearch;
    bench_.projectionShareOfLq += local.projectionShareOfLq;
    if (nFailed > 0) {   // SqpSolver.cpp:306-308 throws per solver; here after the other instances of the batch have been kept
      {
        std::lock_guard<std::mutex> lf(benchMutex_);
        for (int s = 0; s < Bg; ++s)
          if (status[s] != 0) failedInstances_.push_back(members[s]);
      }
      throw std::runtime_error("[SqpSolver] Failed to solve QP for " + std::to_string(nFailed) + " of " + std::to_string(Bg) + " instances");
    }
  }

 public:
  /** instances whose QP failed in the last run() (their primal solution is the one of their last successful solve) */
  const std::vector<int>& failedInstances() const { return failedInstances_; }

 private:
  std::vector<int> failedInstances_;

  static std::mutex& deviceToken(int device) {
    static std::mutex tokens[16];
    return tokens[(device % 16 + 16) % 16];
  }
  static constexpr int kMaxGroups = 6;
  bool exclusiveSolve_ = false;
  std::vector<double> jointTorqueWeights_;   // setJointTorqueCost (empty: off)
  std::mutex benchMutex_;
  HostModel model_;
  b200sqp_settings settings_;
  int device_, batch_, threads_ = 1;
  std::vector<SwitchedModelReferenceManager> rm_;
  std::vector<std::unique_ptr<ProceduralMpcMotionManager>> motion_;   // null: no motion manager
  std::vector<char> motionStarted_;   // (not vector<bool>: run()'s per-instance threads write neighbouring elements)
  std::vector<PrimalSolution> primal_;
  std::vector<std::vector<StepInfo>> log_;
  std::map<int, Group> groups_;
  std::vector<int> groupOf_, slotOf_;
  Benchmarks bench_;
  bool trajectorySpread_ = true;
};

}  // namespace b200sqp::host
