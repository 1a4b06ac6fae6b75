// DEVELOPMENT HARNESS (tests only, never linked into libb200sqp.so): runs the __host__ __device__ phase functions of the CUDA
// kernels on the CPU, one phase at a time, with the work items of every phase visited in REVERSE order so that an
// intra-phase dependency (a missing barrier on the GPU) shows up as a mismatch against the oracle.
// It exists so that the device math can be checked where no GPU is available; the product has no CPU path.
#include <cstdio>
#include <vector>

#include "../../wb_humanoid_mpc_b200/csrc/wb_host.cuh"
#include "../../wb_humanoid_mpc_b200/csrc/wb_dynamics.cuh"
#include "../../wb_humanoid_mpc_b200/csrc/wb_torque.cuh"
#ifdef EMU_WITH_LQ
#include "../../wb_humanoid_mpc_b200/csrc/wb_lq.cuh"
#include "../../wb_humanoid_mpc_b200/csrc/cen_host.cuh"
#endif

using namespace b200sqp;

#define RUN_PHASE(NT, CALL)                          \
  for (int tid_ = (NT)-1; tid_ >= 0; --tid_) {       \
    Par P{tid_, (NT)};                               \
    CALL;                                            \
  }

extern "C" {

int emu_dyn(const b200sqp_model_desc* d, const double* x, const double* u, double* xdot, double* G, int deriv) {
  static WbDeviceModel m;
  if (const char* e = makeDeviceModel(*d, m)) {
    std::fprintf(stderr, "emu: %s\n", e);
    return -1;
  }
  static DynWs w;
  const int NT = 128;
  if (deriv) {
    RUN_PHASE(NT, dynPhaseJoints<true>(P, m, x, w));
    RUN_PHASE(NT, dynPhaseBodies(P, m, x, u, w));
    RUN_PHASE(NT, dynPhaseBmat(P, w));
    RUN_PHASE(NT, dynPhaseComposite<true>(P, m, w));
    RUN_PHASE(NT, dynPhaseFinal(P, m, u, w));
    RUN_PHASE(NT, dynWriteFlow(P, x, u, w, xdot));
    RUN_PHASE(NT, dynPhaseJacobian(P, m, w, G));
  } else {
    RUN_PHASE(NT, dynPhaseJoints<false>(P, m, x, w));
    RUN_PHASE(NT, dynPhaseBodies<false>(P, m, x, u, w));
    RUN_PHASE(NT, dynPhaseComposite<false>(P, m, w));
    RUN_PHASE(NT, dynPhaseFinal<false>(P, m, u, w));
    RUN_PHASE(NT, dynWriteFlow(P, x, u, w, xdot));
  }
  return 0;
}

int emu_joint_torques(const b200sqp_model_desc* d, const double* x, const double* u, double* tau, double* qddb) {
  static WbDeviceModel m;
  if (const char* e = makeDeviceModel(*d, m)) {
    std::fprintf(stderr, "emu: %s\n", e);
    return -1;
  }
  wbJointTorques(m, x, u, tau, qddb);
  return 0;
}

#ifdef EMU_WITH_LQ
#include "wb_emu_lq.inc"
#include "cen_emu.inc"
#endif
}
