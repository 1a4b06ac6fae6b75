// DEVELOPMENT HARNESS (tests only, never linked into libb200sqp.so): the phases of the joint-torque cost kernel (wb_torque_cost.cuh) executed
// on the CPU, every phase's work items visited in reverse order with a width other than the kernel's.  Built into tests/emu/libjtemu.so by
// tests/jt_oracle_lib.py.  The product has no CPU path.
#include <cmath>
#include <cstdio>
#include <memory>
#include <vector>

#include "../../wb_humanoid_mpc_b200/csrc/wb_torque_cost.cuh"
#include "../../wb_humanoid_mpc_b200/csrc/wb_host.cuh"

using namespace b200sqp;

namespace {
template <class F>
void reversed(F&& f) {
  constexpr int slots = 40;
  for (int t = slots - 1; t >= 0; --t) f(Par{t, slots});
}
}  // namespace

extern "C" {

// one intermediate node: w [NJ] weights; J [NZ][NJ] (column-major NJ x NZ), r [NJ]; raw: the term's raw blocks added to raw (oracle layout).
// nut >= 0: with the projection Pu (NU x NUT_MAX, column-major), Px (NU x NX), u0 (NU): Q (NX x NX), St / Rt (ld NUT_MAX), q, rt, perf [4]
// accumulated from zero.
int emu_jt_node(const b200sqp_model_desc* md, const double* weights, const double* x, const double* u, double dt, int nut, const double* Pu,
                const double* Px, const double* u0, double* J, double* r, double* raw, double* Q, double* St, double* Rt, double* q, double* rt,
                double* perf) {
  static std::unique_ptr<WbDeviceModel> wm(new WbDeviceModel);
  b200sqp_model_desc base = *md;
  if (base.n_frames > NFRAMES) base.n_frames = NFRAMES;
  if (const char* e = makeDeviceModel(base, *wm)) {
    std::fprintf(stderr, "emu: %s\n", e);
    return -1;
  }
  JtWeights w{};
  for (int j = 0; j < NJ; ++j) w.sw[j] = std::sqrt(weights[j]);
  reversed([&](Par P) { jtPhaseJacobian(P, *wm, w, x, u, J, r); });
  reversed([&](Par P) { jtPhaseRaw(P, dt, J, r, raw); });
  if (nut >= 0) {
    std::vector<double> A(NJ * (NX + NUT_MAX)), v(NJ);
    reversed([&](Par P) { jtPhaseProject(P, nut, J, Pu, Px, u0, A.data(), v.data()); });
    reversed([&](Par P) { jtPhaseAccumulate(P, nut, dt, A.data(), r, v.data(), Q, St, Rt, q, rt, perf); });
  }
  return 0;
}

}  // extern "C"
