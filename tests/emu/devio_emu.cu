// DEVELOPMENT HARNESS (tests only, never linked into libb200sqp.so): the per-row robot-state check of the device-pointer joint actions
// (wb_devio.cuh: mrtRobotStateStatus) executed on the CPU.  Built into tests/emu/libdevioemu.so by tests/devio_emu_lib.py.  The product has no
// CPU path.
#include "../../wb_humanoid_mpc_b200/csrc/wb_devio.cuh"

using namespace b200sqp;

extern "C" {

// rows [n][MRT_RS] -> status [n] (0 accepted, 1 a non-finite entry, 2 the quaternion norm is off)
int emu_robot_state_status(const double* rows, int n, int* status) {
  for (int b = 0; b < n; ++b) status[b] = mrtRobotStateStatus(rows + static_cast<size_t>(b) * MRT_RS);
  return MRT_RS;
}

}  // extern "C"
