// Closed-loop simulation on the device: the policy roll-out of the reference's dummy simulation, batched over instances.
//
// Reference path (MRT_ROS_Dummy_Loop::forwardSimulation -> MRT_BASE::rolloutPolicy, ocs2_mpc/src/MRT_BASE.cpp:124-151):
//   TimeTriggeredRollout::run                 ocs2_oc/src/rollout/TimeTriggeredRollout.cpp:46-116 (identity jump map, reconstructInputTrajectory)
//   RolloutBase::findActiveModesTimeInterval  ocs2_oc/src/rollout/RolloutBase.cpp:44-68
//   RungeKuttaDormandPrince5 (ODE45_OCS2)      ocs2_core/src/integration/RungeKuttaDormandPrince5.cpp:84-227, 263-289 (runIntegrateAdaptive)
//   IntegratorBase::systemFunction            ocs2_core/src/integration/IntegratorBase.cpp:47-58 (function-call budget)
//   LinearController / FeedforwardController::computeInput over LinearInterpolation::timeSegment
//   ModeSchedule::modeAtTime                  ocs2_core/src/reference/ModeSchedule.cpp:50-53
// The controller is the primal solution's policy as the shim builds it (include/ocs2_sqp/B200SqpSolver.h toPrimalSolution): node k of the plan
// carries u_src and K_src with src = k, the terminal node and PreEvent nodes repeating the stage before them, and bias_k = u_k - K_k x_k.
// The event times are the plan's PreEvent node times.  One integrator serves two systems: the value-only whole-body dynamics of K3
// (wb_dynamics.cuh, policy_rollout_kernel) and the value part of the centroidal flow map (cen_ocp.cuh, cen_policy_rollout_kernel).
//
// One 32-thread CTA per instance (K3's finding: one warp per work item keeps an SM busy).  Every scalar the integrator decides on (time, step
// size, error norm, accept / reject, retries, function calls) is computed by every thread from shared memory after a barrier, so the control
// flow is warp-uniform and the CPU harnesses (tests/emu/sim_emu.cu, tests/emu/cen_sim_emu.cu) run the same function with their own phase runners.  The error norm is a max-reduction:
// its value does not depend on how the work items are split.
#pragma once
#include <cfloat>

#include "cen_solver.cuh"
#include "wb_dynamics.cuh"
#include "wb_solver.cuh"

namespace b200sqp {

enum SimStatus { SIM_OK = 0, SIM_RETRIES = 1, SIM_BUDGET = 2, SIM_NONFINITE = 3 };

// one instance's plan (primal solution of the last solve), read through L1
struct SimPlan {
  int n;                 // nodes (N + 1)
  const double* t;       // [n]
  const uint8_t* event;  // [n]
  const uint8_t* contact;// [n][2]
  const double* x;       // [n][NX]
  const double* u;       // [n - 1][NU]
  const double* K;       // [n - 1][NU * NX] column-major remapped gains, or null (feed-forward policy)
};

// shared-memory vectors of the stepper (after the value-only DynWs prefix)
struct SimVec {
  double x[NX], dxdt[NX];              // current state and its derivative (= k1 of the next step)
  double k[5][NX];                     // k2 .. k6
  double xs[NX];                       // stage point
  double xout[NX], dout[NX];           // candidate state and its derivative
  double u[NU];                        // input of the last flow-map evaluation
  double biasA[NU], biasB[NU];         // bias of the two bracketing nodes (cached per segment)
  double part[64];                     // per-thread partial maxima
};
constexpr int SIM_SMEM_DOUBLES = DYN_VALUE_DOUBLES + static_cast<int>(sizeof(SimVec) / sizeof(double));

struct SimResult {
  double tEnd;
  int status, accepted, rejected, calls, mode;
};

// LinearInterpolation::timeSegment over the node times (ocs2_core/misc/implementation/LinearInterpolation.h:69-105)
HD void simTimeSegment(const double* T, int n, double t, int& idx, double& alpha) {
  if (n <= 1) {
    idx = 0;
    alpha = 1.0;
    return;
  }
  int lo = 0, hi = n;   // std::lower_bound
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (T[mid] < t) lo = mid + 1;
    else hi = mid;
  }
  const int index = lo - 1, last = n - 1;
  if (index < 0) {
    idx = 0;
    alpha = 1.0;
  } else if (index < last) {
    const double length = T[index + 1] - T[index], tillNext = T[index + 1] - t;
    idx = index;
    alpha = (length > 2.0 * kWeakEps) ? tillNext / length : (tillNext < 0.5 * length ? 0.0 : 1.0);
  } else {
    idx = last - 1 > 0 ? last - 1 : 0;
    alpha = 0.0;
  }
}

// stage of the plan whose input / gain node k carries (toPrimalSolution)
HD int simSource(const SimPlan& p, int k) {
  int src = (k + 1 < p.n) ? k : p.n - 2;
  if (p.event[k] == 1 && k > 0) src = k - 1;
  return src;
}

// ModeSchedule::modeAtTime with the PreEvent node times as event times: the mode of the segment that starts after the last event < t
// (lower_bound), read from the contact flags of the segment's first node (0 FLY, 1 RF, 2 LF, 3 STANCE)
HD int simModeAt(const SimPlan& p, double t) {
  int first = 0;
  for (int k = 0; k + 1 < p.n; ++k)
    if (p.event[k] == 1 && p.t[k] < t) first = k + 1;
  return 2 * p.contact[2 * first] + p.contact[2 * first + 1];
}

// bias_k = u_k - K_k x_k for the nodes idx (into a) and idx + 1 (into b); fixed order: s = u_r, then s -= K_rc x_c for c = 0 .. SX-1 (the
// system's state width; the rows of x and K keep the stride NX)
template <int SX>
HD void simPhaseBias(Par P, const SimPlan& p, int idx, SimVec& v) {
  for (int it = P.tid; it < 2 * NU; it += P.nt) {
    const int h = it / NU, r = it % NU, k = idx + h;
    const int src = simSource(p, k);
    const double* K = p.K + static_cast<size_t>(src) * NU * NX;
    const double* xk = p.x + static_cast<size_t>(k) * NX;
    double s = p.u[static_cast<size_t>(src) * NU + r];
    for (int c = 0; c < SX; ++c) s -= K[r + NU * c] * xk[c];
    (h == 0 ? v.biasA : v.biasB)[r] = s;
  }
}

// policy phase: u = computeInput(t, x).  Linear: uff = alpha bias_a + (1 - alpha) bias_b, k = alpha K_a + (1 - alpha) K_b (entry-wise), then
// u_r = uff_r + sum_c k_rc x_c in increasing c < SX.  Feed-forward: u = alpha u_a + (1 - alpha) u_b.
template <int SX>
HD void simPhasePolicy(Par P, const SimPlan& p, int idx, double alpha, const double* x, SimVec& v) {
  const int sa = simSource(p, idx), sb = simSource(p, idx + 1);
  for (int r = P.tid; r < NU; r += P.nt) {
    if (!p.K) {
      v.u[r] = alpha * p.u[static_cast<size_t>(sa) * NU + r] + (1.0 - alpha) * p.u[static_cast<size_t>(sb) * NU + r];
      continue;
    }
    const double* Ka = p.K + static_cast<size_t>(sa) * NU * NX;
    const double* Kb = p.K + static_cast<size_t>(sb) * NU * NX;
    double s = alpha * v.biasA[r] + (1.0 - alpha) * v.biasB[r];
    for (int c = 0; c < SX; ++c) s += (alpha * Ka[r + NU * c] + (1.0 - alpha) * Kb[r + NU * c]) * x[c];
    v.u[r] = s;
  }
}

// The systems the integrator runs.  A system supplies the state and input widths SX / SU that the stage combinations, the policy and the error
// norm run over (the vectors keep the stride NX / NU), and flow(phase, x, u, xdot): the value-only flow map at (x, u) as a sequence of phases.
//
// Whole-body: K3's value-only dynamics phases (wb_dynamics.cuh) in the DynWs prefix of the shared memory.
struct SimWbSystem {
  static constexpr int SX = NX, SU = NU;
  const WbDeviceModel& m;
  DynWs& W;
  template <class PH>
  HD void flow(const PH& phase, const double* x, const double* u, double* xdot) const {
    phase([&](Par P) { dynPhaseJoints<false>(P, m, x, W); });
    phase([&](Par P) { dynPhaseBodies<false>(P, m, x, u, W); });
    phase([&](Par P) { dynPhaseComposite<false>(P, m, W); });
    phase([&](Par P) { dynPhaseFinal<false>(P, m, u, W); });
    phase([&](Par P) { dynWriteFlow(P, x, u, W, xdot); });
  }
};

// Centroidal: the value part of the handle's own cenKinematics + cenFlowFromKin (cen_ocp.cuh) on x[0..35), both model types (full centroidal
// dynamics, SRBD) through its CenModel -- the OCP's CentroidalDynamicsAD, which the reference's centroidal roll-out integrates
// (CentroidalMpcInterface.cpp:107,231).  The kinematics is a serial tree walk: thread slice 0 evaluates the whole flow map, k is its scratch.
struct SimCenSystem {
  static constexpr int SX = CNX, SU = CNU;
  const CenModel& m;
  CenKin& k;
  template <class PH>
  HD void flow(const PH& phase, const double* x, const double* u, double* xdot) const {
    phase([&](Par P) {
      if (P.tid != 0) return;
      D1 xd[CNX], ud[CNU], fd[CNX];
      for (int i = 0; i < CNX; ++i) xd[i] = dmk(x[i]);
      for (int i = 0; i < CNU; ++i) ud[i] = dmk(u[i]);
      cenKinematics(m, xd + 6, k);
      cenFlowFromKin(m, k, xd, ud, fd);
      for (int i = 0; i < CNX; ++i) xdot[i] = fd[i].v;
    });
  }
};

// Runs one instance: x (in v.x) from t0 to tf under the plan's policy through system S.  PH is the phase runner: PH(f) calls f(Par) on every
// thread slice and then separates the phases (a CTA barrier on the GPU; the CPU harnesses visit the slices one after another).  Only the
// first S::SX entries of the state vectors and S::SU of the input are read or written.
template <class PH, class S>
HD SimResult simRollout(const PH& phase, const S& sys, const SimPlan& p, const b200sqp_rollout_settings& rs, double t0, double tf, SimVec& v) {
  static_assert(PH::slots >= 1 && PH::slots <= 64, "the error norm reduces over at most 64 thread slices");
  constexpr int SX = S::SX, SU = S::SU;
  static_assert(SX <= NX && SU == NU, "the policy fills every input row");
  SimResult res{t0, SIM_OK, 0, 0, 0, 0};
  const long long maxCalls = static_cast<long long>(rs.max_steps_per_second * (tf - t0 > 1.0 ? tf - t0 : 1.0));
  int cachedIdx = -1;
  // system(x, dxdt, t): policy + value-only flow map; false when the function-call budget is exceeded
  auto flow = [&](double t, const double* x, double* xdot) -> bool {
    int idx;
    double alpha;
    simTimeSegment(p.t, p.n, t, idx, alpha);
    if (p.K && idx != cachedIdx) {
      phase([&](Par P) { simPhaseBias<SX>(P, p, idx, v); });
      cachedIdx = idx;
    }
    phase([&](Par P) { simPhasePolicy<SX>(P, p, idx, alpha, x, v); });
    sys.flow(phase, x, v.u, xdot);
    return ++res.calls <= maxCalls;
  };
  // RungeKuttaDormandPrince5::runIntegrateAdaptive on [a, b]; returns the time of its last observation
  auto integrate = [&](double a, double b) -> double {
    constexpr double a2 = 1.0 / 5, a3 = 3.0 / 10, a4 = 4.0 / 5, a5 = 8.0 / 9;
    constexpr double b21 = 1.0 / 5, b31 = 3.0 / 40, b32 = 9.0 / 40, b41 = 44.0 / 45, b42 = -56.0 / 15, b43 = 32.0 / 9;
    constexpr double b51 = 19372.0 / 6561, b52 = -25360.0 / 2187, b53 = 64448.0 / 6561, b54 = -212.0 / 729;
    constexpr double b61 = 9017.0 / 3168, b62 = -355.0 / 33, b63 = 46732.0 / 5247, b64 = 49.0 / 176, b65 = -5103.0 / 18656;
    constexpr double c1 = 35.0 / 384, c3 = 500.0 / 1113, c4 = 125.0 / 192, c5 = -2187.0 / 6784, c6 = 11.0 / 84;
    constexpr double dc1 = c1 - 5179.0 / 57600, dc3 = c3 - 7571.0 / 16695, dc4 = c4 - 393.0 / 640, dc5 = c5 - -92097.0 / 339200,
                     dc6 = c6 - 187.0 / 2100, dc7 = -1.0 / 40;
    double t = a, dt = rs.time_step;
    if (!flow(t, v.x, v.dxdt)) {
      res.status = SIM_BUDGET;
      return t;
    }
    while (b - t > DBL_EPSILON) {                 // lessWithSign(t, finalTime, dt), dt > 0
      if ((t + dt) - b > DBL_EPSILON) dt = b - t;   // clip the last step to finalTime
      int tries = 0;
      for (;;) {
        // doStep: k1 = dxdt of the previous step
        const double* k1 = v.dxdt;
        double* const k2 = v.k[0];
        double* const k3 = v.k[1];
        double* const k4 = v.k[2];
        double* const k5 = v.k[3];
        double* const k6 = v.k[4];
        const double h21 = dt * b21, h31 = dt * b31, h32 = dt * b32;
        phase([&](Par P) { for (int i = P.tid; i < SX; i += P.nt) v.xs[i] = v.x[i] + h21 * k1[i]; });
        bool ok = flow(t + dt * a2, v.xs, k2);
        if (ok) {
          phase([&](Par P) { for (int i = P.tid; i < SX; i += P.nt) v.xs[i] = (v.x[i] + h31 * k1[i]) + h32 * k2[i]; });
          ok = flow(t + dt * a3, v.xs, k3);
        }
        if (ok) {
          phase([&](Par P) { for (int i = P.tid; i < SX; i += P.nt) v.xs[i] = v.x[i] + dt * ((b41 * k1[i] + b42 * k2[i]) + b43 * k3[i]); });
          ok = flow(t + dt * a4, v.xs, k4);
        }
        if (ok) {
          phase([&](Par P) {
            for (int i = P.tid; i < SX; i += P.nt) v.xs[i] = v.x[i] + dt * (((b51 * k1[i] + b52 * k2[i]) + b53 * k3[i]) + b54 * k4[i]);
          });
          ok = flow(t + dt * a5, v.xs, k5);
        }
        if (ok) {
          phase([&](Par P) {
            for (int i = P.tid; i < SX; i += P.nt)
              v.xs[i] = v.x[i] + dt * ((((b61 * k1[i] + b62 * k2[i]) + b63 * k3[i]) + b64 * k4[i]) + b65 * k5[i]);
          });
          ok = flow(t + dt, v.xs, k6);
        }
        if (ok) {
          phase([&](Par P) {
            for (int i = P.tid; i < SX; i += P.nt) v.xout[i] = v.x[i] + dt * ((((c1 * k1[i] + c3 * k3[i]) + c4 * k4[i]) + c5 * k5[i]) + c6 * k6[i]);
          });
          ok = flow(t + dt, v.xout, v.dout);
        }
        if (!ok) {
          res.status = SIM_BUDGET;
          return t;
        }
        // maxError: || x_err / (absTol + relTol (|x| + |dt| |dxdt|)) ||_inf, NaN-propagating max over fixed per-element values
        phase([&](Par P) {
          double mx = 0.0;
          for (int i = P.tid; i < SX; i += P.nt) {
            const double xe = dt * (((((dc1 * k1[i] + dc3 * k3[i]) + dc4 * k4[i]) + dc5 * k5[i]) + dc6 * k6[i]) + dc7 * v.dout[i]);
            const double e = fabs(xe / (rs.abs_tol + rs.rel_tol * (fabs(v.x[i]) + fabs(dt) * fabs(v.dxdt[i]))));
            mx = (e != e || mx != mx) ? NAN : (e > mx ? e : mx);
          }
          v.part[P.tid] = mx;
        });
        double error = 0.0;
        for (int l = 0; l < PH::slots; ++l) error = (v.part[l] != v.part[l] || error != error) ? NAN : (v.part[l] > error ? v.part[l] : error);
        if (error > 1.0) {   // reject: decreaseStep
          ++res.rejected;
          dt *= fmax(0.9 * pow(error, -1.0 / 3), 0.2);
          if (++tries > 100) {   // maxNumStepsRetries_
            res.status = SIM_RETRIES;
            return t;
          }
          continue;
        }
        // accept: t += dt, x = x_out, dxdt = dxdt_out, increaseStep
        ++res.accepted;
        t += dt;
        phase([&](Par P) {
          for (int i = P.tid; i < SX; i += P.nt) {
            v.x[i] = v.xout[i];
            v.dxdt[i] = v.dout[i];
          }
        });
        if (error < 0.5) {
          const double e = fmax(pow(5.0, -5.0), error);
          dt *= 0.9 * pow(e, -1.0 / 5);
        }
        break;
      }
    }
    return t;
  };
  // findActiveModesTimeInterval: switching times t0, the events in (t0, tf], tf; every interval starts weakEpsilon after its switching time
  auto nextEvent = [&](int from) {
    for (int k = from; k < p.n; ++k)
      if (p.event[k] == 1 && p.t[k] > t0 && p.t[k] <= tf) return k;
    return -1;
  };
  double s0 = t0;
  int je = nextEvent(0);
  for (;;) {
    const double s1 = je >= 0 ? p.t[je] : tf;
    const double a = fmin(s0 + kWeakEps, s1);
    if (a < s1) {
      res.tEnd = integrate(a, s1);
      if (res.status) return res;
    } else {
      res.tEnd = s1;   // a degenerate interval contributes one sample: (its end time, the state it starts from)
    }
    if (je < 0) break;   // (the jump map is the identity)
    s0 = s1;
    je = nextEvent(je + 1);
  }
  // the input of the last sample (reconstructInputTrajectory) and the mode at the final time
  {
    int idx;
    double alpha;
    simTimeSegment(p.t, p.n, res.tEnd, idx, alpha);
    if (p.K && idx != cachedIdx) phase([&](Par P) { simPhaseBias<SX>(P, p, idx, v); });
    phase([&](Par P) { simPhasePolicy<SX>(P, p, idx, alpha, v.x, v); });
  }
  res.mode = simModeAt(p, tf);
  bool finite = true;   // (v - v == 0 is false for infinities and NaN)
  for (int i = 0; i < SX; ++i) finite = finite && v.x[i] - v.x[i] == 0.0;
  for (int i = 0; i < SU; ++i) finite = finite && v.u[i] - v.u[i] == 0.0;
  if (!finite) res.status = SIM_NONFINITE;
  return res;
}

// the whole-body roll-out
template <class PH>
HD SimResult simRollout(const PH& phase, const WbDeviceModel& m, const SimPlan& p, const b200sqp_rollout_settings& rs, double t0, double tf,
                        DynWs& W, SimVec& v) {
  return simRollout(phase, SimWbSystem{m, W}, p, rs, t0, tf, v);
}

// centroidal handles: the state rows keep the stride NX, and their 23 dummy slots stay exactly zero.  The load reads x[0..35) only, the
// store writes the padding as zeros.
HD void simCenLoad(Par P, const double* x, SimVec& v) {
  for (int i = P.tid; i < NX; i += P.nt) v.x[i] = i < CNX ? x[i] : 0.0;
}
HD void simCenStore(Par P, const SimVec& v, double* x) {
  for (int i = P.tid; i < NX; i += P.nt) x[i] = i < CNX ? v.x[i] : 0.0;
}

HD SimPlan simPlanOf(const WbDev& d, int b) {
  const size_t n = static_cast<size_t>(d.N) + 1;
  return SimPlan{d.N + 1, d.t + b * n, d.event + b * n, d.contact + 2 * b * n, d.x + b * n * NX, d.u + b * (n - 1) * NU,
                 d.Kre ? d.Kre + b * (n - 1) * NU * NX : nullptr};
}

#ifdef __CUDACC__
struct SimCtaPhase {   // the CTA's phase runner: every thread takes its slice, then a barrier
  static constexpr int slots = 32;
  template <class F>
  __device__ void operator()(F&& f) const {
    f(Par{static_cast<int>(threadIdx.x), static_cast<int>(blockDim.x)});
    __syncthreads();
  }
};

// one CTA (32 threads) per instance: x_in [B][NX] -> x_out [B][NX] (may alias), u_out [B][NU], info [B][5] = (status, accepted, rejected,
// flow-map calls, mode)
__global__ void __launch_bounds__(32) policy_rollout_kernel(WbDev d, b200sqp_rollout_settings rs, double t0, double tf, const double* x_in,
                                                            double* x_out, double* u_out, int* info) {
  extern __shared__ double smem[];
  DynWs& W = *reinterpret_cast<DynWs*>(smem);
  SimVec& v = *reinterpret_cast<SimVec*>(smem + DYN_VALUE_DOUBLES);
  const int b = blockIdx.x;
  for (int i = threadIdx.x; i < NX; i += blockDim.x) v.x[i] = x_in[static_cast<size_t>(b) * NX + i];
  __syncthreads();
  const SimResult r = simRollout(SimCtaPhase{}, *d.model, simPlanOf(d, b), rs, t0, tf, W, v);
  for (int i = threadIdx.x; i < NX; i += blockDim.x) x_out[static_cast<size_t>(b) * NX + i] = v.x[i];
  for (int i = threadIdx.x; i < NU; i += blockDim.x) u_out[static_cast<size_t>(b) * NU + i] = v.u[i];
  if (threadIdx.x == 0) {
    int* o = info + 5 * b;
    o[0] = r.status;
    o[1] = r.accepted;
    o[2] = r.rejected;
    o[3] = r.calls;
    o[4] = r.mode;
  }
}

// the same on a centroidal handle: x_in / x_out [B][NX] padded rows, of which only the first 35 entries are read; the kernel writes zeros into
// the padding of x_out.  Thread 0 evaluates the flow map and keeps its CenKin scratch in local memory.
__global__ void __launch_bounds__(32) cen_policy_rollout_kernel(WbDev d, const CenDevModel* cm, b200sqp_rollout_settings rs, double t0, double tf,
                                                                const double* x_in, double* x_out, double* u_out, int* info) {
  extern __shared__ double smem[];
  SimVec& v = *reinterpret_cast<SimVec*>(smem);
  const int b = blockIdx.x;
  const Par P{static_cast<int>(threadIdx.x), static_cast<int>(blockDim.x)};
  simCenLoad(P, x_in + static_cast<size_t>(b) * NX, v);
  __syncthreads();
  CenKin k;
  const SimResult r = simRollout(SimCtaPhase{}, SimCenSystem{cm->ocp.kin, k}, simPlanOf(d, b), rs, t0, tf, v);
  simCenStore(P, v, x_out + static_cast<size_t>(b) * NX);
  for (int i = threadIdx.x; i < NU; i += blockDim.x) u_out[static_cast<size_t>(b) * NU + i] = v.u[i];
  if (threadIdx.x == 0) {
    int* o = info + 5 * b;
    o[0] = r.status;
    o[1] = r.accepted;
    o[2] = r.rejected;
    o[3] = r.calls;
    o[4] = r.mode;
  }
}
#endif

}  // namespace b200sqp
