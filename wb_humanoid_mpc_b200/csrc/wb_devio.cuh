// Device-pointer I/O of the closed loop (the b200sqp_*_dev entry points): the robot-state check of b200sqp_joint_actions moved onto the device,
// the joint actions written straight into the caller's device arrays in caller order (rejected rows NaN), and the plan gathered from the group
// views into the caller's padded arrays in one launch.  The MRT kernels themselves are those of the host path (wb_mrt.cuh).
#pragma once
#include "wb_fleet.cuh"
#include "wb_mrt.cuh"

namespace b200sqp {

// The check b200sqp_joint_actions applies to one RobotState row on the host: 0 accepted, 1 an entry is not finite, 2 the quaternion's norm
// is off 1 by more than 1e-6.  The squares are summed with explicit round-to-nearest operations on the device, so that no FMA contraction
// makes a row near the bound pass on one side and fail on the other.
HD int mrtRobotStateStatus(const double* r) {
  for (int i = 0; i < MRT_RS; ++i)
    if (!(r[i] - r[i] == 0.0)) return 1;
#ifdef __CUDA_ARCH__
  const double s = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(r[3], r[3]), __dmul_rn(r[4], r[4])), __dmul_rn(r[5], r[5])), __dmul_rn(r[6], r[6]));
#else
  const double s = r[3] * r[3] + r[4] * r[4] + r[5] * r[5] + r[6] * r[6];
#endif
  const double n = sqrt(s);
  return !(fabs(n - 1.0) <= 1e-6) ? 2 : 0;
}

// the caller's output arrays of a joint-action call, each may be null: q_des, qd_des, tau [B][NJ], x [B][nxAbi], u [B][NU], mode, status [B]
struct MrtDevOut {
  double *qDes, *qdDes, *tau, *x, *u;
  int *mode, *status;
};

#ifdef __CUDACC__
// status[b] of every caller row (robot [B][MRT_RS])
__global__ void __launch_bounds__(128) mrt_check_kernel(const double* robot, int B, int* status) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) status[b] = mrtRobotStateStatus(robot + static_cast<size_t>(b) * MRT_RS);
}

// One CTA per slot s: the MRT kernels' slot-order outputs (jout [3][count][NJ] of each group from 3 * first * NJ on, xout [B][NX], uout [B][NU],
// modeIn [B]) -> row slotInst[s] of the caller's arrays.  gtab / slotInst null: a plain handle (one group, slot = instance).  st [B] in caller
// order (null: every row accepted); a rejected row gets NaN in every double output and mode -1.
__global__ void __launch_bounds__(64) mrt_dev_out_kernel(const double* jout, const double* xout, const double* uout, const int* modeIn, const int* gtab,
                                                         const int* slotInst, const int* st, int B, int nxAbi, MrtDevOut o) {
  const int s = blockIdx.x;
  const FleetSlot sl = fleetSlot(gtab, B, 1, s);   // (one row per slot: no node rows)
  const int first = sl.first, count = sl.count;
  const size_t i = slotInst ? slotInst[s] : s, k = s - first;
  const int code = st ? st[i] : 0;
  const double nan = __longlong_as_double(0x7ff8000000000000LL);
  const double* q = jout + (3 * static_cast<size_t>(first) + k) * NJ;   // q_des; qd_des and tau follow at count and 2 count rows
  for (int j = threadIdx.x; j < NJ; j += blockDim.x) {
    if (o.qDes) o.qDes[i * NJ + j] = code ? nan : q[j];
    if (o.qdDes) o.qdDes[i * NJ + j] = code ? nan : q[count * NJ + j];
    if (o.tau) o.tau[i * NJ + j] = code ? nan : q[2 * static_cast<size_t>(count) * NJ + j];
  }
  if (o.x)
    for (int j = threadIdx.x; j < nxAbi; j += blockDim.x) o.x[i * nxAbi + j] = code ? nan : xout[static_cast<size_t>(s) * NX + j];
  if (o.u)
    for (int j = threadIdx.x; j < NU; j += blockDim.x) o.u[i * NU + j] = code ? nan : uout[static_cast<size_t>(s) * NU + j];
  if (threadIdx.x == 0) {
    if (o.mode) o.mode[i] = code ? -1 : modeIn[s];
    if (o.status) o.status[i] = code;
  }
}

// The plan of slot s (grid.y) at node row r (grid.x < maxNodes) -> caller row slotInst[s] of x [B][maxNodes][nxAbi], u [B][maxNodes-1][NU],
// K [B][maxNodes-1][NU*nxAbi] (column-major NU x nxAbi per stage: the leading nxAbi columns of the device's NU x NX) and status [B]; each may be
// null, rows past the instance's node count are zero.  gtab / slotInst null: a plain handle, capNodes = its node count.
__global__ void __launch_bounds__(128) plan_gather_kernel(WbDev base, int capNodes, const int* gtab, const int* slotInst, int maxNodes, int nxAbi,
                                                          double* x, double* u, double* K, int* status) {
  const int s = blockIdx.y, r = blockIdx.x;
  const FleetSlot sl = fleetSlot(gtab, gridDim.y, capNodes, s);
  const int n = sl.n;
  const size_t i = slotInst ? slotInst[s] : s;
  const size_t node = sl.node + r, stage = sl.stage + r;
  if (x) {
    double* o = x + (i * maxNodes + r) * nxAbi;
    for (int j = threadIdx.x; j < nxAbi; j += blockDim.x) o[j] = r < n ? base.x[node * NX + j] : 0.0;
  }
  if (r < maxNodes - 1) {
    const size_t row = i * (maxNodes - 1) + r;
    if (u)
      for (int j = threadIdx.x; j < NU; j += blockDim.x) u[row * NU + j] = r < n - 1 ? base.u[stage * NU + j] : 0.0;
    if (K)
      for (int j = threadIdx.x; j < NU * nxAbi; j += blockDim.x) K[row * NU * nxAbi + j] = r < n - 1 ? base.Kre[stage * NU * NX + j] : 0.0;
  }
  if (status && r == 0 && threadIdx.x == 0) status[i] = base.flags[static_cast<size_t>(s) * F_NF + F_STATUS];
}
#endif

}  // namespace b200sqp
