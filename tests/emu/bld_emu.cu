// DEVELOPMENT HARNESS (tests only, never linked into libb200sqp.so): the device builder (wb_builder.cuh), the fleet's partition and slot helper
// (wb_fleet.cuh), the batch layout (wb_batch.cuh) and the shared-memory layouts of the Riccati kernels (riccati.cuh, riccati_cluster.cuh) executed
// on the CPU.  One context holds B instances' builder state the way the handle's batch
// allocation does, and emu_bld_build runs the work items in the order b200sqp_build_instances launches its kernels, every loop in reverse so that
// an order dependence shows as a mismatch.
// Built into tests/emu/libbldemu.so by tests/bld_emu_lib.py.  The product has no CPU path.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <type_traits>
#include <vector>

#include "../../wb_humanoid_mpc_b200/csrc/cen_host.cuh"
#include "../../wb_humanoid_mpc_b200/csrc/riccati_cluster.cuh"
#include "../../wb_humanoid_mpc_b200/csrc/wb_fleet.cuh"

using namespace b200sqp;

namespace {
struct Ctx {
  int B = 0, cap = 0;
  b200sqp_builder_desc desc{};
  int stateful = 0;
  bool motionOn = false, poseOn = false, resetOn = false;
  b200sqp_motion_desc mdesc{};
  b200sqp_pose_desc pdesc{};
  BldResetRule rule{};
  CenDevModel cen;
  bool isCen = false;
  std::vector<double> x0;   // [B][NX] the measured states of the build
  std::vector<BldScratch> scratch;
  std::vector<double> gridT;
  std::vector<uint8_t> gridE;
  std::vector<BldGaitState> gstate;
  std::vector<BldSpread> spread;
  std::vector<double> sprT, sprX, sprU;
  std::vector<int> sprLen;
  std::vector<BldMotionState> motion;
  std::vector<BldPoseState> pose;
  // reset rows and episode books (b200sqp_set_reset_states)
  std::vector<double> rsX0, rsOffset, epStart, epLast;
  std::vector<int> rsGait, epEpisode, epReason;
  std::vector<uint8_t> rst;
  // the previous solution: strides prevN + 1 / prevN without prevLen, else the capacity stride with per-instance lengths
  std::vector<double> prevT, prevX, prevU;
  std::vector<uint8_t> prevE;
  std::vector<int> prevLen;
  int prevN = 0;
  bool perInstance = true;
  // the node pass's outputs (the handle's x, u, t, ... arrays) and the node count of every instance
  std::vector<double> x, u, t, swing, impact, arm, xref;
  std::vector<uint8_t> event, contact;
  std::vector<int> nNodes;
};

template <class T>
void put(std::vector<T>& v, const T* src, size_t n) {
  v.assign(src, src + n);
}
}  // namespace

extern "C" {

// ---- one context of B instances ----------------------------------------------------------------------------------------------------------------
// md / pd NULL: no motion manager / no pose commands.  reset_on NULL: no resets, else {on, on_solve, on_rollout} with reset_max_dev [3].
// model / cen NULL: the whole-body target rule, else the centroidal one on makeCenDeviceModel's model.  NULL for a model it refuses.
void* emu_bld_create(const b200sqp_builder_desc* desc, int B, int cap, int stateful, const b200sqp_motion_desc* md, const b200sqp_pose_desc* pd,
                     const int* reset_on, const double* reset_max_dev, const b200sqp_model_desc* model, const b200sqp_cen_desc* cen) {
  Ctx* c = new Ctx();
  if (model && cen) {
    if (const char* e = makeCenDeviceModel(*model, *cen, c->cen)) {
      std::fprintf(stderr, "emu: %s\n", e);
      delete c;
      return nullptr;
    }
    c->isCen = true;
  }
  const size_t n = static_cast<size_t>(B) * cap;
  c->B = B;
  c->cap = cap;
  c->desc = *desc;
  c->stateful = stateful;
  if (md) c->motionOn = true, c->mdesc = *md;
  if (pd) c->poseOn = true, c->pdesc = *pd;
  if (reset_on) c->resetOn = true, c->rule = {reset_on[0], reset_on[1], reset_on[2], {reset_max_dev[0], reset_max_dev[1], reset_max_dev[2]}};
  c->x0.assign(B * NX, 0.0);
  c->scratch.resize(B);
  c->gridT.assign(n, 0.0);
  c->gridE.assign(n, 0);
  c->gstate.resize(B);
  c->spread.resize(B);
  c->sprT.assign(n, 0.0);
  c->sprX.assign(n * NX, 0.0);
  c->sprU.assign(n * NU, 0.0);
  c->sprLen.assign(B, 0);
  c->motion.resize(B);
  c->pose.assign(B, BldPoseState{});
  c->rsX0.assign(B * NX, 0.0);
  c->rsOffset.assign(B, 0.0);
  c->rsGait.assign(B, 0);
  c->epStart.assign(B, 0.0);
  c->epLast.assign(B, 0.0);
  c->epEpisode.assign(B, 0);
  c->epReason.assign(B, 0);
  c->rst.assign(B, 0);
  c->prevT.assign(n, 0.0);
  c->prevE.assign(n, 0);
  c->prevX.assign(n * NX, 0.0);
  c->prevU.assign(n * NU, 0.0);
  c->prevLen.assign(B, 0);
  c->x.assign(n * NX, NAN);   // (an entry the node pass leaves alone shows, the padding of centroidal rows included)
  c->u.assign(n * NU, 0.0);
  c->t.assign(n, 0.0);
  c->event.assign(n, 0);
  c->contact.assign(2 * n, 0);
  c->swing.assign(6 * n, 0.0);
  c->impact.assign(2 * n, 0.0);
  c->arm.assign(n, 0.0);
  c->xref.assign(n * NX, NAN);
  c->nNodes.assign(B, 0);
  return c;
}
void emu_bld_destroy(void* c) { delete static_cast<Ctx*>(c); }

// the reset rows [B][NX], their gait ids [B] and gait offsets [B] (b200sqp_set_reset_states)
void emu_bld_set_reset_states(void* cp, const double* rows, const int* gait, const double* offset) {
  Ctx& c = *static_cast<Ctx*>(cp);
  put(c.rsX0, rows, c.rsX0.size());
  put(c.rsGait, gait, c.B);
  put(c.rsOffset, offset, c.B);
}

// the previous solution of the next warm build, in place of the one the last build carried: prev_len NULL: every instance has prev_n + 1
// nodes (t, event [B][prev_n + 1], x [B][prev_n + 1][NX], u [B][prev_n][NU]); else instance i has prev_len[i] nodes at the capacity stride
void emu_bld_set_previous(void* cp, const int* prev_len, int prev_n, const double* t, const uint8_t* event, const double* x, const double* u) {
  Ctx& c = *static_cast<Ctx*>(cp);
  c.perInstance = prev_len != nullptr;
  const size_t rows = c.perInstance ? static_cast<size_t>(c.B) * c.cap : static_cast<size_t>(c.B) * (prev_n + 1);
  const size_t urows = c.perInstance ? rows : static_cast<size_t>(c.B) * prev_n;
  if (c.perInstance) put(c.prevLen, prev_len, c.B);
  c.prevN = c.perInstance ? 0 : prev_n;
  std::memcpy(c.prevT.data(), t, rows * sizeof(double));
  std::memcpy(c.prevE.data(), event, rows);
  std::memcpy(c.prevX.data(), x, rows * NX * sizeof(double));
  std::memcpy(c.prevU.data(), u, urows * NU * sizeof(double));
}

// One build, in the kernel order of b200sqp_build_instances:
//   1. the measured states: x0 [B][NX], or (x0 = NULL) bldX0FromPrevious;
//   2. bldResetDecide / bldResetApply with the requests reset_req [B] (NULL: none), when the context has resets;
//   3. bldCenBaseVelocity on a centroidal context;  4. bldGridInstance;  5. bldSpreadApply on a stateful warm build;
//   6. nodes = 1: bldNode into one view of the batch (rows at the stride of the common node count); nodes = 2: into one single-instance view
//      per instance through a slot map (rows at the capacity stride); nodes = 0: no node pass.
// pose_cmd [B] NULL: no pose command pending; else 1 latches pose_delta[i], 2 clears.  The previous solution of the next build is then this
// build's grid and, after a node pass, its states and inputs (the ones it had otherwise).
// Returns 0, -1 on overflow, -2 when nodes = 1 and the instances disagree on the node count.
int emu_bld_build(void* cp, int warm, double t0, double horizon, const double* x0, const int* gait, const double* gait_start, const double* cmd,
                  const uint8_t* reset_req, const uint8_t* pose_cmd, const double* pose_delta, int nodes) {
  Ctx& c = *static_cast<Ctx*>(cp);
  const int B = c.B, cap = c.cap;
  WbDev d{};
  d.B = B;
  d.x0 = c.x0.data();
  BldDev b{};
  b.scratch = c.scratch.data();
  b.gridT = c.gridT.data();
  b.gridE = c.gridE.data();
  b.cmd = cmd;
  b.gait = gait;
  b.gaitStart = gait_start;
  b.cap = cap;
  b.warm = warm;
  b.prevN = c.prevN;
  b.prevLen = c.perInstance ? c.prevLen.data() : nullptr;
  b.prevT = c.prevT.data();
  b.prevE = c.prevE.data();
  b.prevX = c.prevX.data();
  b.prevU = c.prevU.data();
  b.t0 = t0;
  b.tf = t0 + horizon;
  b.dt = c.desc.dt;
  b.desc = c.desc;
  b.cen = c.isCen ? &c.cen : nullptr;
  b.stateful = c.stateful;
  b.gstate = c.gstate.data();
  b.spread = c.spread.data();
  b.sprT = c.sprT.data();
  b.sprX = c.sprX.data();
  b.sprU = c.sprU.data();
  b.sprLen = c.sprLen.data();
  if (c.motionOn) {
    b.motion = c.motion.data();
    b.mdesc = c.mdesc;
  }
  if (c.poseOn) {
    b.pose = c.pose.data();
    b.poseCmd = pose_cmd;
    b.poseDelta = pose_delta;
    b.pdesc = c.pdesc;
  }
  if (x0) put(c.x0, x0, c.x0.size());
  else
    for (int i = B - 1; i >= 0; --i)
      for (int tid = 63; tid >= 0; --tid) bldX0FromPrevious(d, b, i, tid, 64);
  if (c.resetOn) {
    const std::vector<uint8_t> none(B, 0);
    BldResetDev r{};
    r.rule = c.rule;
    r.x0 = c.rsX0.data();
    r.req = reset_req ? reset_req : none.data();
    r.episode = c.epEpisode.data();
    r.start = c.epStart.data();
    r.lastLength = c.epLast.data();
    r.reason = c.epReason.data();
    r.rst = c.rst.data();
    r.warm = warm;
    r.B = B;
    r.cen = c.isCen;
    for (int s = B - 1; s >= 0; --s) {   // (every lane decides before any lane writes, as after the kernel's __syncwarp)
      const int why = bldResetDecide(d, r, s);
      for (int lane = 31; lane >= 0; --lane) bldResetApply(d, r, t0, s, why, lane, 32);
    }
    b.rst = c.rst.data();
    b.rsGait = c.rsGait.data();
    b.rsOffset = c.rsOffset.data();
  }
  if (c.isCen) {
    static CenKin k;
    for (int i = B - 1; i >= 0; --i) bldCenBaseVelocity(c.cen.ocp.kin, c.x0.data() + static_cast<size_t>(i) * NX, c.desc.total_mass, k, c.scratch[i].baseVel);
  }
  for (int i = B - 1; i >= 0; --i) bldGridInstance(d, b, i);
  if (c.stateful && warm)
    for (int i = B - 1; i >= 0; --i)
      for (int k = cap - 1; k >= 0; --k)
        for (int tid = 63; tid >= 0; --tid) bldSpreadApply(b, k, i, tid, 64);
  for (int i = 0; i < B; ++i) {
    if (c.scratch[i].overflow) return -1;
    c.nNodes[i] = c.scratch[i].nNodes;
  }
  d.x = c.x.data();
  d.u = c.u.data();
  d.t = c.t.data();
  d.event = c.event.data();
  d.contact = c.contact.data();
  d.swing = c.swing.data();
  d.impact = c.impact.data();
  d.arm = c.arm.data();
  d.xref = c.xref.data();
  if (nodes == 1) {
    const int n = c.nNodes[0];
    for (int i = 0; i < B; ++i)
      if (c.nNodes[i] != n) return -2;
    d.N = n - 1;
    for (int i = B - 1; i >= 0; --i)
      for (int k = n - 1; k >= 0; --k)
        for (int tid = 63; tid >= 0; --tid) bldNode(d, b, k, i, tid, 64);
  } else if (nodes == 2) {
    for (int i = B - 1; i >= 0; --i) {   // instance i as position 0 of a fleet group of size 1 at slot i
      const WbDev v = groupView(d, cap, c.nNodes[i], i, 1, nullptr);
      BldDev bi = b;
      bi.slot = &i;
      for (int k = v.N; k >= 0; --k)
        for (int tid = 63; tid >= 0; --tid) bldNode(v, bi, k, 0, tid, 64);
    }
  }
  // carry this build as the previous solution of the next, at the capacity stride
  for (int i = 0; i < B; ++i) {
    const int n = c.nNodes[i];
    const size_t node = static_cast<size_t>(i) * cap;
    const size_t src = nodes == 1 ? static_cast<size_t>(i) * n : node, srcU = nodes == 1 ? static_cast<size_t>(i) * (n - 1) : static_cast<size_t>(i) * (cap - 1);
    c.prevLen[i] = n;
    std::memcpy(&c.prevT[node], &c.gridT[node], n * sizeof(double));
    std::memcpy(&c.prevE[node], &c.gridE[node], n);
    if (nodes) {
      std::memmove(&c.prevX[node * NX], &c.x[src * NX], n * NX * sizeof(double));
      std::memmove(&c.prevU[node * NU], &c.u[srcU * NU], (n - 1) * NU * sizeof(double));
    }
  }
  c.perInstance = true;
  c.prevN = 0;
  return 0;
}

// the builder state of every instance after a build: n_nodes [B], grid_t [B][cap] (zero behind the nodes), base velocity bv [B][6], target
// knots tt_time [B][3] and tt_state [B][3][NX], spr_len [B], the window schedule n_events [B], events [B][BLD_MAX_EVENTS], modes [B][BLD_MAX_EVENTS + 1]
void emu_bld_instances(void* cp, int* n_nodes, double* grid_t, double* bv, double* tt_time, double* tt_state, int* spr_len, int* n_events, double* events,
                       int* modes) {
  Ctx& c = *static_cast<Ctx*>(cp);
  for (int i = 0; i < c.B; ++i) {
    const BldScratch& s = c.scratch[i];
    const size_t node = static_cast<size_t>(i) * c.cap;
    n_nodes[i] = s.nNodes;
    for (int k = 0; k < s.nNodes && k < c.cap; ++k) grid_t[node + k] = c.gridT[node + k];
    for (int j = 0; j < 6; ++j) bv[6 * i + j] = s.baseVel[j];
    for (int k = 0; k < 3; ++k) {
      tt_time[3 * i + k] = s.ttTime[k];
      for (int j = 0; j < NX; ++j) tt_state[(static_cast<size_t>(i) * 3 + k) * NX + j] = s.ttState[k][j];
    }
    spr_len[i] = c.sprLen[i];
    n_events[i] = s.sched.n;
    for (int k = 0; k < s.sched.n; ++k) events[static_cast<size_t>(i) * BLD_MAX_EVENTS + k] = s.sched.ev[k];
    for (int k = 0; k <= s.sched.n; ++k) modes[static_cast<size_t>(i) * (BLD_MAX_EVENTS + 1) + k] = s.sched.mode[k];
  }
}

// the motion-manager states: state [B], last_change [B], origin [B], filtered [B][4]
void emu_bld_motion(void* cp, int* state, double* last_change, double* origin, double* filtered) {
  Ctx& c = *static_cast<Ctx*>(cp);
  for (int i = 0; i < c.B; ++i) {
    const BldMotionState& m = c.motion[i];
    state[i] = m.state;
    last_change[i] = m.lastChange;
    origin[i] = m.origin;
    for (int j = 0; j < 4; ++j) filtered[4 * i + j] = m.filtered[j];
  }
}

// the pose states: active [B], t_start [B], t_reach [B], target [B][6], error [B][2]
void emu_bld_pose(void* cp, int* active, double* t_start, double* t_reach, double* target, double* error) {
  Ctx& c = *static_cast<Ctx*>(cp);
  for (int i = 0; i < c.B; ++i) {
    const BldPoseState& p = c.pose[i];
    active[i] = p.active;
    t_start[i] = p.tStart;
    t_reach[i] = p.tReach;
    for (int j = 0; j < 6; ++j) target[6 * i + j] = p.target[j];
    for (int j = 0; j < 2; ++j) error[2 * i + j] = p.error[j];
  }
}

// the node pass's output arrays as the build left them ([B * cap] rows; u: [B * cap] stage rows)
void emu_bld_nodes(void* cp, double* x, double* u, double* t, uint8_t* event, uint8_t* contact, double* swing, double* impact, double* arm, double* xref) {
  Ctx& c = *static_cast<Ctx*>(cp);
  std::memcpy(x, c.x.data(), c.x.size() * sizeof(double));
  std::memcpy(u, c.u.data(), c.u.size() * sizeof(double));
  std::memcpy(t, c.t.data(), c.t.size() * sizeof(double));
  std::memcpy(event, c.event.data(), c.event.size());
  std::memcpy(contact, c.contact.data(), c.contact.size());
  std::memcpy(swing, c.swing.data(), c.swing.size() * sizeof(double));
  std::memcpy(impact, c.impact.data(), c.impact.size() * sizeof(double));
  std::memcpy(arm, c.arm.data(), c.arm.size() * sizeof(double));
  std::memcpy(xref, c.xref.data(), c.xref.size() * sizeof(double));
}

// ---- unit entry points ---------------------------------------------------------------------------------------------------------------------------
void* emu_gait_create() { return new BldGaitState(); }
void emu_gait_destroy(void* g) { delete static_cast<BldGaitState*>(g); }

// the cold build's seed: the closed-form window [t0 - T, tf + T] of (gait, start); 0, or -1 on overflow
int emu_gait_seed(void* g, const b200sqp_builder_desc* d, int gait, double start, double t0, double tf) {
  auto& s = *static_cast<BldGaitState*>(g);
  const double T = tf - t0;
  s.tmpl = s.lastCmd = gait;
  return bldModeSchedule(*d, gait, start, t0 - T, tf + T, s.s) ? 0 : -1;
}
// the reference manager's getModeSchedule(lb, ub) with the active template
int emu_gait_get(void* g, const b200sqp_builder_desc* d, double lb, double ub) {
  auto& s = *static_cast<BldGaitState*>(g);
  return bldGetModeSchedule(*d, s.tmpl, lb, ub, s.s) ? 0 : -1;
}
// updateGaitSchedule: 0, 1 (overflow), 2 (LF phase before the first event)
int emu_gait_update(void* g, const b200sqp_builder_desc* d, int gait, double t0, double tf, double ptst) {
  auto& s = *static_cast<BldGaitState*>(g);
  s.lastCmd = gait;
  return bldUpdateGait(*d, s, gait, t0, tf, ptst);
}
int emu_gait_state(void* g, double* ev, int* modes, int cap) {
  const BldSched& s = static_cast<BldGaitState*>(g)->s;
  if (s.n > cap) return -1;
  for (int k = 0; k < s.n; ++k) ev[k] = s.ev[k];
  for (int k = 0; k <= s.n; ++k) modes[k] = s.mode[k];
  return s.n;
}

// trajectorySpread of one previous primal solution: old / new window schedules, its time grid t [n], node events [n], states x [n][NX] and
// node inputs u [n-1][NU] (as the solve leaves them).  Outputs: the spread times, states and toPrimalSolution inputs (first *len rows),
// flags = (willTruncate, willSpread), the post-event indices (*n_post), and the strategy's begin / end / value triples (*n_spread).
int emu_spread(int n_old, const double* old_ev, const int* old_modes, int n_new, const double* new_ev, const int* new_modes, int n, const double* t,
               const uint8_t* event, const double* x, const double* u, double* t_out, double* x_out, double* u_out, int* len, int* flags, int* post,
               int* n_post, int* triples, int* n_spread) {
  if (n_old > BLD_MAX_EVENTS || n_new > BLD_MAX_EVENTS || n < 2) return -1;
  BldSched o{}, w{};
  o.n = n_old;
  w.n = n_new;
  for (int k = 0; k < n_old; ++k) o.ev[k] = old_ev[k];
  for (int k = 0; k <= n_old; ++k) o.mode[k] = static_cast<signed char>(old_modes[k]);
  for (int k = 0; k < n_new; ++k) w.ev[k] = new_ev[k];
  for (int k = 0; k <= n_new; ++k) w.mode[k] = static_cast<signed char>(new_modes[k]);
  static BldSpread sp;
  std::vector<double> px(x, x + static_cast<size_t>(n) * NX), pu(u, u + static_cast<size_t>(n - 1) * NU), pt(t, t + n);
  std::vector<uint8_t> pe(event, event + n);
  std::vector<double> sT(n), sX(static_cast<size_t>(n) * NX), sU(static_cast<size_t>(n) * NU);
  int sLen = 0;
  BldDev b{};
  b.prevX = px.data();
  b.prevU = pu.data();
  b.prevT = pt.data();
  b.prevE = pe.data();
  b.prevN = n - 1;
  b.cap = n;
  b.spread = &sp;
  b.sprT = sT.data();
  b.sprX = sX.data();
  b.sprU = sU.data();
  b.sprLen = &sLen;
  bldSpreadStrategy(o, w, b.prevT, n, sp, b.sprT);
  sLen = sp.eraseFrom;
  for (int k = n - 1; k >= 0; --k) bldSpreadApply(b, k, 0, 0, 1);   // samples in reverse: no order dependence
  *len = sLen;
  for (int k = 0; k < sLen; ++k) t_out[k] = sT[k];
  for (size_t k = 0; k < static_cast<size_t>(sLen) * NX; ++k) x_out[k] = sX[k];
  for (size_t k = 0; k < static_cast<size_t>(sLen) * NU; ++k) u_out[k] = sU[k];
  flags[0] = sp.eraseFrom < n;
  flags[1] = sp.nSpread > 0;
  *n_post = sp.nPost;
  for (int k = 0; k < sp.nPost; ++k) post[k] = sp.post[k];
  *n_spread = sp.nSpread;
  for (int k = 0; k < sp.nSpread; ++k) {
    triples[3 * k] = sp.begin[k];
    triples[3 * k + 1] = sp.end[k];
    triples[3 * k + 2] = sp.value[k];
  }
  return 0;
}

// bldMotionFilter alone: raw [4] at t0 -> f [4]
void emu_motion_filter(const b200sqp_motion_desc* md, const double* raw, double t0, double* f) { bldMotionFilter(*md, raw, t0, f); }

// bldMotionTransition alone on (state, last change): filtered command f [4], base velocity bv [6] at t0
void emu_motion_transition(int* state, double* last_change, const double* f, const double* bv, double t0) {
  BldMotionState m{};
  m.state = *state;
  m.lastChange = *last_change;
  bldMotionTransition(m, f, bv, t0);
  *state = m.state;
  *last_change = m.lastChange;
}

// bldResetReason alone
int emu_reset_reason(int on, int on_solve, int on_rollout, const double* max_dev, int requested, const double* x, const double* ref, int n, int cen,
                     int solve, int rollout) {
  BldResetRule r{on, on_solve, on_rollout, {max_dev[0], max_dev[1], max_dev[2]}};
  return bldResetReason(r, requested != 0, x, ref, n, cen != 0, solve, rollout);
}

// bldResetDecide + bldResetApply over B instances in slot order (slot_inst may be NULL), with the lanes of a warp run one after the other.  x0 [B][NX] is
// replaced in place, sim_x [B][NX] (may be NULL) too; the books episode / start / last_length / reason / rst [B] are updated in place.
void emu_reset_instances(int B, int warm, int cen, double t0, int on, int on_solve, int on_rollout, const double* max_dev, double* x0, const double* rows,
                         const uint8_t* req, const int* flags, const int* slot_inst, const int* sim_info, double* sim_x, int* episode, double* start,
                         double* last_length, int* reason, uint8_t* rst) {
  WbDev d{};
  d.B = B;
  d.x0 = x0;
  BldResetDev r{};
  r.rule = {on, on_solve, on_rollout, {max_dev[0], max_dev[1], max_dev[2]}};
  r.x0 = rows;
  r.req = req;
  r.flags = flags;
  r.slotInst = slot_inst;
  r.simInfo = sim_info;
  r.simX = sim_x;
  r.episode = episode;
  r.start = start;
  r.lastLength = last_length;
  r.reason = reason;
  r.rst = rst;
  r.warm = warm;
  r.B = B;
  r.cen = cen;
  for (int s = 0; s < B; ++s) {   // (every lane decides before any lane writes, as after the kernel's __syncwarp)
    const int why = bldResetDecide(d, r, s);
    for (int lane = 31; lane >= 0; --lane) bldResetApply(d, r, t0, s, why, lane, 32);
  }
}

// fleet_partition_kernel with nt threads, phase by phase: node counts [B] -> slotInst [B], gtab [1 + 3 nBins]
void emu_fleet_partition(const int* nodes, int B, int nBins, int nt, int* slotInst, int* gtab) {
  std::vector<int> key(B), cnt(nBins, 0);
  for (int i = 0; i < B; ++i) key[i] = nodes[i] < 0 ? 0 : (nodes[i] > nBins - 1 ? nBins - 1 : nodes[i]);
  for (int t = 0; t < nt; ++t) fleetHistogram(key.data(), B, cnt.data(), t, nt);
  fleetOffsets(cnt.data(), nBins, gtab);
  for (int tile = 0; tile < B; tile += nt) {
    for (int t = nt - 1; t >= 0; --t) fleetPlace(key.data(), B, cnt.data(), slotInst, tile, t);
    for (int t = 0; t < nt; ++t) fleetAdvance(key.data(), B, cnt.data(), tile, t);
  }
}

// ---- the batch layout (wb_batch.cuh) ---------------------------------------------------------------------------------------------------------------
namespace {
#define WB_M(f) {#f, offsetof(WbDev, f)}
#define WB_Q(f) {"qp." #f, offsetof(WbDev, qp) + offsetof(QpDeviceView, f)}
// the array members of WbDev by name
const struct {
  const char* name;
  size_t off;
} kMembers[] = {WB_M(x0),   WB_M(x),       WB_M(u),        WB_M(t),     WB_M(swing), WB_M(impact),  WB_M(arm),    WB_M(xref),   WB_M(xInit),
                WB_M(uInit), WB_M(event),  WB_M(contact),  WB_Q(A),     WB_Q(Bm),    WB_Q(b),       WB_Q(Q),      WB_Q(S),      WB_Q(R),
                WB_Q(q),     WB_Q(r),      WB_Q(dx0),      WB_Q(nu),    WB_Q(K),     WB_Q(kff),     WB_Q(P),      WB_Q(p),      WB_Q(dx),
                WB_Q(du),    WB_Q(status), WB_M(Pu),       WB_M(Px),    WB_M(u0p),   WB_M(du),      WB_M(Kre),    WB_M(perfNode), WB_M(lsNode),
                WB_M(inst),  WB_M(flags),  WB_M(pending),  WB_M(mid),   WB_M(luRec), WB_M(luPerm),  WB_M(gstats), WB_M(raw),    WB_M(log)};
#undef WB_M
#undef WB_Q

// a handle's device state as set_batch walks the table: the settings and the widths the table reads
WbDev layoutBase(int valueFunction, int feedback, int maxIter, long long rawPer) {
  WbDev d{};
  d.st.create_value_function = valueFunction;
  d.st.use_feedback_policy = feedback;
  d.maxIter = maxIter;
  d.rawPer = rawPer;
  d.qp.nx = NX;
  d.qp.numax = NUT_MAX;
  return d;
}
}  // namespace

const char* emu_batch_member(int i) { return kMembers[i].name; }

// forEachBatchArray of a handle with these settings: for entry e, member[e] (emu_batch_member; -1 for a field that is no array member), its
// row kind kind[e] (0 instance, 1 node, 2 stage, 3 handle), its elements per row width[e] and its zero fill zero[e].  Returns the entries.
int emu_batch_layout(int cen, int value_function, int feedback, int raw, int max_iter, long long raw_per, int* member, int* kind, long long* width,
                     int* zero) {
  WbDev d = layoutBase(value_function, feedback, max_iter, raw_per);
  int e = 0;
  forEachBatchArray(d, cen, raw, [&](auto*& p, RowKind k, size_t w, bool z) {
    const size_t off = reinterpret_cast<const char*>(&p) - reinterpret_cast<const char*>(&d);
    member[e] = -1;
    for (size_t i = 0; i < sizeof(kMembers) / sizeof(kMembers[0]); ++i)
      if (kMembers[i].off == off) member[e] = static_cast<int>(i);
    kind[e] = k;
    width[e] = static_cast<long long>(w);
    zero[e] = z;
    ++e;
  });
  return e;
}

// The allocation of B instances at cap nodes per instance by walking the table (as set_batch does), then groupView of every group of gtab
// {G, (n, first, count) * G} with a null line-search counter: bytes[e] allocated for entry e, and off[g * E + e] the byte offset of group g's
// pointer into that allocation (-1: null).  Returns the number of entries E.
int emu_group_views(int cen, int value_function, int feedback, int raw, int max_iter, long long raw_per, int B, int cap, const int* gtab,
                    long long* bytes, long long* off) {
  WbDev d = layoutBase(value_function, feedback, max_iter, raw_per);
  std::vector<const char*> base;
  forEachBatchArray(d, cen, raw, [&](auto*& p, RowKind k, size_t w, bool) {
    const size_t n = batchRows(k, B, cap) * w * sizeof(*p);
    p = static_cast<std::remove_reference_t<decltype(p)>>(std::malloc(n));
    bytes[base.size()] = static_cast<long long>(n);
    base.push_back(reinterpret_cast<const char*>(p));
  });
  const int E = static_cast<int>(base.size());
  for (int g = 0; g < gtab[0]; ++g) {
    WbDev v = groupView(d, cap, gtab[1 + 3 * g], gtab[2 + 3 * g], gtab[3 + 3 * g], nullptr);
    int e = 0;
    forEachBatchArray(v, cen, raw, [&](auto*& p, RowKind, size_t, bool) {
      off[g * E + e] = p ? reinterpret_cast<const char*>(p) - base[e] : -1;
      ++e;
    });
  }
  for (const char* p : base) std::free(const_cast<char*>(p));
  return E;
}

// fleetSlot of every slot s < B of a batch at cap nodes per instance (gtab NULL: a plain handle): its group's n, first, count [B] and its first
// node and stage rows [B]
void emu_fleet_slots(const int* gtab, int B, int cap, int* n, int* first, int* count, long long* node, long long* stage) {
  for (int s = 0; s < B; ++s) {
    const FleetSlot r = fleetSlot(gtab, B, cap, s);
    n[s] = r.n;
    first[s] = r.first;
    count[s] = r.count;
    node[s] = static_cast<long long>(r.node);
    stage[s] = static_cast<long long>(r.stage);
  }
}

// Ab^-1 hbar of n centroidal states: x [n][NX] (padded rows) -> bv [n][6]; -1 for a model the device conversion refuses
int emu_cen_base_velocity(const b200sqp_model_desc* d, const b200sqp_cen_desc* c, double total_mass, int n, const double* x, double* bv) {
  static CenDevModel m;
  if (const char* e = makeCenDeviceModel(*d, *c, m)) {
    std::fprintf(stderr, "emu: %s\n", e);
    return -1;
  }
  static CenKin k;
  for (int i = n - 1; i >= 0; --i) bldCenBaseVelocity(m.ocp.kin, x + static_cast<size_t>(i) * NX, total_mass, k, bv + 6 * i);
  return 0;
}

// The shared-memory layouts of the generic Riccati kernels at (nx, nm), in doubles: out[0..9) riccati_layout_padded (the one-CTA kernel) and
// out[9..18) riccati_layout (the cluster kernel), each as {pq, ab, w, y, rs, linv, vec, total, kout}; out[18] riccati_smem_doubles and
// out[19] riccati_cluster_smem_doubles; out[20], out[21] the one-CTA kernel's leading dimensions ric_pad(nx), ric_pad(nm); out[22] whether
// b200sqp_qp_create accepts the size (riccati_sizes_supported); out[23] the byte limit it applies.
void emu_riccati_layout(int nx, int nm, long long* out) {
  const RicLayout ls[2] = {riccati_layout_padded(nx, nm), riccati_layout(nx, nm)};
  for (int i = 0; i < 2; ++i) {
    const RicLayout& L = ls[i];
    const int f[9] = {L.pq, L.ab, L.w, L.y, L.rs, L.linv, L.vec, L.total, L.kout};
    for (int j = 0; j < 9; ++j) out[9 * i + j] = f[j];
  }
  out[18] = static_cast<long long>(riccati_smem_doubles(nx, nm));
  out[19] = static_cast<long long>(riccati_cluster_smem_doubles(nx, nm));
  out[20] = ric_pad(nx);
  out[21] = ric_pad(nm);
  out[22] = riccati_sizes_supported(nx, nm);
  out[23] = static_cast<long long>(RIC_SMEM_BYTES_MAX);
}

}  // extern "C"
