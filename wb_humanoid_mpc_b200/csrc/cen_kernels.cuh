// __global__ entry points of the centroidal path (phase functions: cen_ocp.cuh, cen_solver.cuh; device state: WbDev, wb_solver.cuh).
#pragma once
#include "cen_solver.cuh"
#include "wb_solver.cuh"

namespace b200sqp {

#define PHASE(...)                                                            \
  {                                                                           \
    const Par P{static_cast<int>(threadIdx.x), static_cast<int>(blockDim.x)}; \
    __VA_ARGS__                                                               \
  }                                                                           \
  __syncthreads();

// LQ approximation of one node -> raw block (intermediate nodes) or the finished QP record (terminal / event nodes)
__global__ void __launch_bounds__(CEN_THREADS) cen_lq_kernel(WbDev d, const CenDevModel* cm) {
  extern __shared__ double smem[];
  const int k = blockIdx.x, b = blockIdx.y;
  if (d.flags[b * F_NF + F_CONVERGED]) return;
  const int N = d.N;
  const size_t node = static_cast<size_t>(b) * (N + 1) + k, stage = static_cast<size_t>(b) * N + k;
  NodeIn n;
  loadNode(d, b, k, n);
  n.x = d.x + node * NX;
  if (k < N) {
    n.u = d.u + stage * NU;
    n.xnext = d.x + (node + 1) * NX;
  }
  const CenDevModel& mb = cm[static_cast<size_t>(b) * d.modelStride];   // the instance's gains (stride 0: the handle's model)
  if (lqTerminalOrEventNode(d, n, k, node, stage, mb.QfdPad, CNX, CNU, smem)) return;
  const CenOcpModel& m = mb.ocp;
  CenLqWs s;
  cenLqWsMap(smem, s);
  double* const raw = d.raw + stage * d.rawPer;
  double* const perf = d.perfNode + node * 4;
  CenKin kin;
#include "cen_node_lq.inc"
}

__global__ void __launch_bounds__(CEN_PROJ_THREADS) cen_proj_kernel(WbDev d) {
  extern __shared__ double smem[];
  const int k = blockIdx.x, b = blockIdx.y;
  if (d.flags[b * F_NF + F_CONVERGED]) return;
  const size_t node = static_cast<size_t>(b) * (d.N + 1) + k, stage = static_cast<size_t>(b) * d.N + k;
  if (d.event[node] == 1) return;
  const double* const raw = d.raw + stage * d.rawPer;
  CenPjWs s;
  cenPjWsMap(smem, s);
  NodeOut out = nodeOut(d, node, stage);
#include "cen_node_proj.inc"
}

// value-only trial evaluation of one node at x + alpha dx (computePerformance, SqpSolver.cpp:433-482): thread 0 walks the node
__global__ void __launch_bounds__(32) cen_rollout_kernel(WbDev d, const CenDevModel* cm) {
  const int k = blockIdx.x, b = blockIdx.y;
  if (d.flags[b * F_NF + F_CONVERGED] || d.flags[b * F_NF + F_LSDONE]) return;
  __shared__ double xa[NX], xna[NX], ua[NU], tref[13];
  const int N = d.N;
  const size_t node = static_cast<size_t>(b) * (N + 1) + k, stage = static_cast<size_t>(b) * N + k;
  const double alpha = d.inst[b * I_ND + I_ALPHA];
  NodeIn n;
  loadNode(d, b, k, n);
  double* perfOut = d.lsNode + node * 4;
  for (int i = threadIdx.x; i < NX; i += blockDim.x) {
    xa[i] = fma(alpha, d.qp.dx[node * NX + i], d.x[node * NX + i]);
    if (k < N) xna[i] = fma(alpha, d.qp.dx[(node + 1) * NX + i], d.x[(node + 1) * NX + i]);
  }
  if (k < N)
    for (int i = threadIdx.x; i < NU; i += blockDim.x) ua[i] = fma(alpha, d.du[stage * NU + i], d.u[stage * NU + i]);
  __syncthreads();
  if (threadIdx.x != 0) return;
  n.x = xa;
  n.u = ua;
  n.xnext = xna;
  const CenDevModel& mb = cm[static_cast<size_t>(b) * d.modelStride];
  if (k == N || n.event == 1) {
    double c = 0.0;
    for (int i = 0; i < NX; ++i) {
      if (k == N) {
        const double dx = xa[i] - n.xref[i];
        c += 0.5 * mb.QfdPad[i] * dx * dx;
      } else {
        const double df = xa[i] - xna[i];
        c += df * df;
      }
    }
    perfOut[0] = (k == N) ? c : 0.0;
    perfOut[1] = (k == N) ? 0.0 : c;
    perfOut[2] = 0.0;
    return;
  }
  const CenOcpModel& m = mb.ocp;
  CenKin kin;
  cenTorsoReference(m, n.xref, kin, tref);
  CenDirOut o;
  cenNodeDual(m, n, tref, -1, kin, o);
  double val[CEN_ROWS];
  const int nres = cenResidualRows(n), nc = cenConstraintRows(n);
  for (int r = 0; r < CEN_MAX_RES; ++r) val[r] = (r < nres) ? o.res[r].v : 0.0;
  for (int r = 0; r < CEN_PEN_ROWS; ++r) val[CEN_MAX_RES + r] = o.pen[r].v;
  const double cost = cenRowScalars(m, n, val, nullptr, nullptr, nullptr);
  double dsse = 0.0, esse = 0.0;
  for (int i = 0; i < CNX; ++i) {
    const double df = o.xplus[i].v - xna[i];
    dsse = fma(df, df, dsse);
  }
  for (int r = 0; r < nc; ++r) esse = fma(o.g[r].v, o.g[r].v, esse);
  perfOut[0] = n.dt * cost;
  perfOut[1] = n.dt * dsse;
  perfOut[2] = n.dt * esse;
}

#undef PHASE

}  // namespace b200sqp
