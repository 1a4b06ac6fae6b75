// DEVELOPMENT HARNESS (tests only, never linked into libb200sqp.so): the policy roll-out of wb_sim.cuh (simRollout and its phase functions)
// executed on the CPU, with a phase runner that visits the thread slices one after another, in reverse.  Built into tests/emu/libsimemu.so by
// tests/sim_emu_lib.py.  The product has no CPU path.
#include <cstdio>

#include "../../wb_humanoid_mpc_b200/csrc/wb_host.cuh"
#include "../../wb_humanoid_mpc_b200/csrc/wb_sim.cuh"

using namespace b200sqp;

namespace {
struct EmuSimPhase {   // 48 slices: a width other than the kernel's 32, so that a result that depends on the split shows up
  static constexpr int slots = 48;
  template <class F>
  void operator()(F&& f) const {
    for (int t = slots - 1; t >= 0; --t) f(Par{t, slots});
  }
};
}  // namespace

extern "C" {

// one instance: plan t [n], event [n], contact [n][2], x [n][58], u [n-1][35], K [n-1][35*58] column-major or NULL; info = (status, accepted,
// rejected, flow-map calls, mode)
int emu_rollout_policy(const b200sqp_model_desc* d, int n, const double* t, const uint8_t* event, const uint8_t* contact, const double* x,
                       const double* u, const double* K, const b200sqp_rollout_settings* rs, double t0, double tf, const double* x_start, double* x_end,
                       double* u_end, int* info) {
  static WbDeviceModel m;
  if (const char* e = makeDeviceModel(*d, m)) {
    std::fprintf(stderr, "emu: %s\n", e);
    return -1;
  }
  static DynWs w;
  static SimVec v;
  for (int i = 0; i < NX; ++i) v.x[i] = x_start[i];
  const SimPlan p{n, t, event, contact, x, u, K};
  const SimResult r = simRollout(EmuSimPhase{}, m, p, *rs, t0, tf, w, v);
  for (int i = 0; i < NX; ++i) x_end[i] = v.x[i];
  for (int i = 0; i < NU; ++i) u_end[i] = v.u[i];
  info[0] = r.status;
  info[1] = r.accepted;
  info[2] = r.rejected;
  info[3] = r.calls;
  info[4] = r.mode;
  return 0;
}

}  // extern "C"
