// MRT-side queries of the last solve on the device: the value function and the linear feedback gain at one time t, batched.
//
// Reference (ocs2_mpc/src/MPC_MRT_Interface.cpp):
//   getLinearFeedbackGain(time)      lines 167-178: LinearController::getFeedbackGain, the gains interpolated at time (a throw for a
//                                    feed-forward policy)
//   getValueFunction(time, state)    lines 180-183 -> SqpSolver::getValueFunction (ocs2_sqp/src/SqpSolver.cpp:172-191): the Riccati cost-to-go
//                                    (P, p) linearly interpolated over the node times, then re-centred, dfdx += dfdxx * state; f = 0
// The time segment is the policy's (wb_sim.cuh: simTimeSegment = LinearInterpolation::timeSegment, kWeakEps rule for zero-length segments
// included), the gain of node k is the stage simSource(k) (toPrimalSolution: PreEvent nodes and the terminal node repeat the stage before
// them), and the arithmetic is the host layer's getValueFunction (host/SqpSolver.hpp): every entry alpha * a + (1 - alpha) * b, then
// dfdx_r += dfdxx_rc * x_c for c = 0, 1, ... in that order.  Products and sums are rounded one by one (no FMA contraction on the device), so
// the device gives the host formula's result bit for bit.
//
// The query only reads: two P blocks, two p rows and two gain blocks per instance.  One CTA per instance (slot), plain handles and fleets.
#pragma once
#include "wb_fleet.cuh"
#include "wb_sim.cuh"

namespace b200sqp {

HD double qryMul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
HD double qryAdd(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
// alpha a + (1 - alpha) b, each operation rounded on its own
HD double qryLerp(double alpha, double a, double b) { return qryAdd(qryMul(alpha, a), qryMul(1.0 - alpha, b)); }

// One instance's query at time t.  p: its plan (node times and events; p.K the remapped gains [n-1][NU*NX], read when K is wanted).  P [n][NX*NX]
// and pv [n][NX]: its cost-to-go rows (read when dfdxx or dfdx is wanted).  sx: the state width at the ABI (NX; CNX on centroidal handles: the
// leading sx rows and columns of the padded blocks).  x [sx]: the state dfdx is re-centred at (read when dfdx is wanted).  Outputs, each may
// be null, column-major at width sx: dfdxx [sx*sx], dfdx [sx], K [NU*sx].  One phase: no output depends on another.
template <class PH>
HD void mrtQuery(const PH& phase, const SimPlan& p, const double* P, const double* pv, int sx, double t, const double* x, double* dfdxx,
                 double* dfdx, double* K) {
  int idx;
  double alpha;
  simTimeSegment(p.t, p.n, t, idx, alpha);
  phase([&](Par Q) {
    const double* Pa = P ? P + static_cast<size_t>(idx) * NX * NX : nullptr;
    const double* Pb = Pa ? Pa + NX * NX : nullptr;
    if (dfdxx)
      for (int e = Q.tid; e < sx * sx; e += Q.nt) {
        const int r = e % sx, c = e / sx;
        dfdxx[e] = qryLerp(alpha, Pa[r + NX * c], Pb[r + NX * c]);
      }
    if (dfdx) {
      const double* pa = pv + static_cast<size_t>(idx) * NX;
      for (int r = Q.tid; r < sx; r += Q.nt) {
        double s = qryLerp(alpha, pa[r], pa[NX + r]);
        for (int c = 0; c < sx; ++c) s = qryAdd(s, qryMul(qryLerp(alpha, Pa[r + NX * c], Pb[r + NX * c]), x[c]));
        dfdx[r] = s;
      }
    }
    if (K) {   // (the leading sx columns of a column-major NU x NX block are its first NU * sx entries)
      const double* Ka = p.K + static_cast<size_t>(simSource(p, idx)) * NU * NX;
      const double* Kb = p.K + static_cast<size_t>(simSource(p, idx + 1)) * NU * NX;
      for (int e = Q.tid; e < NU * sx; e += Q.nt) K[e] = qryLerp(alpha, Ka[e], Kb[e]);
    }
  });
}

// the plan of slot sl in the batch arrays of base (fleetSlot's node and stage rows)
HD SimPlan simPlanAt(const WbDev& base, const FleetSlot& sl) {
  return SimPlan{sl.n, base.t + sl.node, base.event + sl.node, base.contact + 2 * sl.node, base.x + sl.node * NX, base.u + sl.stage * NU,
                 base.Kre ? base.Kre + sl.stage * NU * NX : nullptr};
}

#ifdef __CUDACC__
// One CTA per slot s (grid = B): the query of the instance in slot s into caller row i = slotInst[s] of dfdxx [B][sx*sx], dfdx [B][sx],
// K [B][NU*sx] (each may be null), with x [B][xStride] in caller order.  gtab / slotInst null: a plain handle, capNodes = its node count.
__global__ void __launch_bounds__(256) mrt_query_kernel(WbDev base, int capNodes, const int* gtab, const int* slotInst, int sx, double t,
                                                        const double* x, int xStride, double* dfdxx, double* dfdx, double* K) {
  const int s = blockIdx.x;
  const FleetSlot sl = fleetSlot(gtab, gridDim.x, capNodes, s);
  const size_t i = slotInst ? slotInst[s] : s;
  const double* P = base.qp.P ? base.qp.P + sl.node * NX * NX : nullptr;
  const double* pv = base.qp.p + sl.node * NX;
  mrtQuery(SimCtaPhase{}, simPlanAt(base, sl), P, pv, sx, t, x ? x + i * xStride : nullptr, dfdxx ? dfdxx + i * sx * sx : nullptr,
           dfdx ? dfdx + i * sx : nullptr, K ? K + i * NU * sx : nullptr);
}

// The cost-to-go of slots [s0, s0 + gridDim.y) at node row r (grid.x < maxNodes) -> row (s - s0) of P [..][maxNodes][sx*sx] and p [..][maxNodes][sx]
// (column-major, the leading sx rows and columns of the padded blocks); rows past the slot's node count are zero.
__global__ void __launch_bounds__(128) value_gather_kernel(WbDev base, int capNodes, const int* gtab, int B, int s0, int maxNodes, int sx, double* P,
                                                           double* p) {
  const int s = s0 + blockIdx.y, r = blockIdx.x;
  const FleetSlot sl = fleetSlot(gtab, B, capNodes, s);
  const size_t row = static_cast<size_t>(blockIdx.y) * maxNodes + r, node = sl.node + r;
  const bool live = r < sl.n;
  for (int e = threadIdx.x; e < sx * sx; e += blockDim.x) P[row * sx * sx + e] = live ? base.qp.P[node * NX * NX + (e % sx) + NX * (e / sx)] : 0.0;
  for (int e = threadIdx.x; e < sx; e += blockDim.x) p[row * sx + e] = live ? base.qp.p[node * NX + e] : 0.0;
}
#endif

}  // namespace b200sqp
