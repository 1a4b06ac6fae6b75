// DEVELOPMENT HARNESS (tests only, never linked into libb200sqp.so): the policy roll-out of a centroidal handle (wb_sim.cuh: simRollout with
// SimCenSystem, simCenLoad / simCenStore) executed on the CPU, with a phase runner of 40 slices visited one after another, in reverse.  Built
// into tests/emu/libcensimemu.so by tests/cen_sim_emu_lib.py.  The product has no CPU path.
#include <cstdio>
#include <memory>

#include "../../wb_humanoid_mpc_b200/csrc/cen_host.cuh"
#include "../../wb_humanoid_mpc_b200/csrc/wb_sim.cuh"

using namespace b200sqp;

namespace {
struct EmuCenSimPhase {   // 40 slices: a width other than the kernel's 32, so that a result that depends on the split shows up
  static constexpr int slots = 40;
  template <class F>
  void operator()(F&& f) const {
    for (int t = slots - 1; t >= 0; --t) f(Par{t, slots});
  }
};
}  // namespace

extern "C" {

// one instance on padded rows (stride NX): plan t [n], event [n], contact [n][2], x [n][NX], u [n-1][NU], K [n-1][NU*NX] column-major or NULL;
// x_start [NX] -> x_end [NX] (padding written as zeros), u_end [NU]; info = (status, accepted, rejected, flow-map calls, mode)
int emu_cen_rollout_policy(const b200sqp_model_desc* md, const b200sqp_cen_desc* cd, int n, const double* t, const uint8_t* event, const uint8_t* contact,
                           const double* x, const double* u, const double* K, const b200sqp_rollout_settings* rs, double t0, double tf,
                           const double* x_start, double* x_end, double* u_end, int* info) {
  static std::unique_ptr<CenDevModel> m(new CenDevModel);
  if (const char* e = makeCenDeviceModel(*md, *cd, *m)) {
    std::fprintf(stderr, "emu: %s\n", e);
    return -1;
  }
  static CenKin k;
  static SimVec v;
  const EmuCenSimPhase phase;
  phase([&](Par P) { simCenLoad(P, x_start, v); });
  const SimPlan p{n, t, event, contact, x, u, K};
  const SimResult r = simRollout(phase, SimCenSystem{m->ocp.kin, k}, p, *rs, t0, tf, v);
  phase([&](Par P) { simCenStore(P, v, x_end); });
  for (int i = 0; i < NU; ++i) u_end[i] = v.u[i];
  info[0] = r.status;
  info[1] = r.accepted;
  info[2] = r.rejected;
  info[3] = r.calls;
  info[4] = r.mode;
  return 0;
}

}  // extern "C"
