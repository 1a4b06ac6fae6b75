// Device kernels of the whole-body SQP iteration and the per-handle device state.
//   K1a lq_dyn_kernel   one CTA per (instance, shooting node): dynamics/cost/constraint linearisation  (SqpSolver::setupQuadraticSubproblem)
//   K1b lq_proj_kernel  one CTA per (instance, stage): constraint projection + change of input variables (projectTranscription)
//   K2 riccati_kernel   riccati.cuh                                                            (HpipmInterface::solve)
//   K4a remap_kernel    du = Pu dut + Px dx + u0, K = Pu Kt + Px, Armijo / norm partial sums    (remapProjectedInput/Gain, armijoDescentMetric)
//   K3 rollout_kernel   one CTA per (instance, node): value-only RK4 defect, cost, constraints at x + alpha dx   (computePerformance)
//   K4b reduce kernels  PerformanceIndex sums, FilterLinesearch::acceptStep, step application, checkConvergence
#pragma once
#include <cstdint>

#include "riccati.cuh"
#include "wb_host.cuh"
#include "wb_lq.cuh"

namespace b200sqp {

// CTA widths: compile-time, overridable for the occupancy sweeps of tools/dev/variant_sweep.py (every phase loops `for (i = tid; i < n; i += nt)`,
// so any multiple of 32 gives the same results).
#ifndef B200SQP_LQA_THREADS
#define B200SQP_LQA_THREADS 96
#endif
#ifndef B200SQP_LQA_GLOBAL_MODEL
#define B200SQP_LQA_GLOBAL_MODEL 1
#endif
#ifndef B200SQP_LQA_CTAS
#define B200SQP_LQA_CTAS 4
#endif
#ifndef B200SQP_LQB_THREADS
#define B200SQP_LQB_THREADS 256
#endif
#ifndef B200SQP_RO_THREADS
#define B200SQP_RO_THREADS 32
#endif
#ifndef B200SQP_RO_GLOBAL_MODEL
#define B200SQP_RO_GLOBAL_MODEL 1
#endif
#ifndef B200SQP_RO_CTAS
#define B200SQP_RO_CTAS 12
#endif
#ifndef B200SQP_LQB1_THREADS
#define B200SQP_LQB1_THREADS 128
#endif
#ifndef B200SQP_LQB1_CTAS
#define B200SQP_LQB1_CTAS 6
#endif
#ifndef B200SQP_LQB_CTAS
#define B200SQP_LQB_CTAS 3
#endif
constexpr int LQA_THREADS = B200SQP_LQA_THREADS;
constexpr int LQB_THREADS = B200SQP_LQB_THREADS;
constexpr int LQB1_THREADS = B200SQP_LQB1_THREADS;
// K3 runs ONE WARP PER NODE (RO_THREADS = 32).  Its phases are narrow (24 bodies, 23 joints, 2 feet, a few 58-93 item loops), so in a wider
// CTA one warp works while the others wait at the barrier, and what keeps an SM busy is the number of NODES resident on it, not the threads
// per node.  The narrower the CTA, the more nodes are resident (128 threads x 3 nodes/SM, 64 x 6, 32 x 11) -- with the value-only workspace
// cut to 17.6 KB (DYN_VALUE_DOUBLES) and the model read through L1 instead of copied into every CTA's shared memory, so that shared memory
// allows 11 nodes per SM and the register cap (RO_CTAS) 12.  tools/dev/variant_sweep.py times the alternatives.
// The older RO_PACK option (several nodes per CTA in lock-step on rotated thread slices) went the wrong way for the same reason: it made the
// CTAs bigger, and fewer of them fit.
#ifndef B200SQP_RO_PACK
#define B200SQP_RO_PACK 1
#endif
constexpr int RO_PACK = B200SQP_RO_PACK;
constexpr int RO_THREADS = RO_PACK == 1 ? B200SQP_RO_THREADS : 64 * RO_PACK;
constexpr double kWeakEps = 1e-9;  // numeric_traits::weakEpsilon (ocs2_core/include/ocs2_core/NumericTraits.h:51)

enum InstD { I_BASE_MERIT = 0, I_BASE_COST, I_BASE_DYN, I_BASE_EQ, I_ARMIJO, I_DXN, I_DUN, I_ALPHA, I_STEP, I_STEPTYPE, I_NEW_MERIT, I_NEW_COST,
             I_NEW_DYN, I_NEW_EQ, I_ND = 16 };
enum InstF { F_CONVERGED = 0, F_LSDONE, F_ITER, F_STATUS, F_CONVCODE, F_RANKDEF, F_NF = 8 };

struct CenDevModel;

struct WbDev {
  int B, N;  // N intervals, N+1 nodes
  const WbDeviceModel* model;   // the handle's model (roll-outs, joint actions, builder)
  // the OCP's model of instance b (cost and penalty kernels): instModel[b * modelStride] (whole-body), instCen[b * modelStride] (centroidal);
  // the handle's model with stride 0 until per-instance gains are set (wb_gains.cuh)
  const WbDeviceModel* instModel;
  const CenDevModel* instCen;
  int modelStride;
  // instance inputs
  double *x0, *x, *u, *t, *swing, *impact, *arm, *xref;
  double *xInit, *uInit;  // uploaded initial guess (restored by b200sqp_reset)
  uint8_t *event, *contact;
  // QP (nx = 58, nu_max = 23)
  QpDeviceView qp;
  double *Pu, *Px, *u0p;
  double* du;     // remapped input step [B][N][35]
  double* Kre;    // remapped gains [B][N][35*58] or null
  double* perfNode;  // [B][N+1][4] baseline
  double* lsNode;    // [B][N+1][4] trial / partial sums
  double* inst;      // [B][I_ND]
  int* flags;        // [B][F_NF]
  int* pending;      // number of instances whose line search is still running
  double* mid;       // K1a -> K1b records [B][N][Mid::SIZE]
  double* luRec;     // lu_kernel -> K1b part 1: LU factors of D in position order; part 1 -> part 2: [X | x0], K   [B][N][LU_REC]
  int* luPerm;       // ... and the row / column permutations [B][N][52] (rowOf[16], colOf[36])
  double* gstats;    // global-step mode: per-candidate statistics [32][4]
  double* raw;       // optional [B][N][rawPer]
  long long rawPer;
  b200sqp_iter_log* log;  // [B][maxIter]
  int maxIter;
  b200sqp_settings st;
};

__device__ __forceinline__ void loadNode(const WbDev& d, int b, int k, NodeIn& n) {
  const size_t node = static_cast<size_t>(b) * (d.N + 1) + k;
  n.xref = d.xref + node * NX;
  n.event = d.event[node];
  n.terminal = (k == d.N);
  n.contact[0] = d.contact[2 * node];
  n.contact[1] = d.contact[2 * node + 1];
  for (int c = 0; c < 2; ++c) {
    for (int j = 0; j < 3; ++j) n.swing[c][j] = d.swing[(2 * node + c) * 3 + j];
    n.impact[c] = d.impact[2 * node + c];
  }
  n.armPhase = d.arm[node];
  n.dt = 0.0;
  if (k < d.N) {
    const double ts = d.t[node] + (d.event[node] == 2 ? kWeakEps : 0.0);
    const double te = d.t[node + 1] - (d.event[node + 1] == 1 ? kWeakEps : 0.0);
    n.dt = te - ts;
  }
}

// Development aid (never in the shipped build): with -DB200SQP_PHASE_CLOCK thread 0 of one CTA records (source line, clock64) after every
// phase barrier; tools/phase_clock.py turns that into a per-phase cycle table.
#ifdef B200SQP_PHASE_CLOCK
__device__ long long g_phaseClk[5][512][2];
__device__ int g_phaseCnt[5];
__device__ int g_phaseNode = 20;
#define PHASE_CLOCK_BEGIN(id)                                                                  \
  const int clkId_ = (id);                                                                     \
  int clkN_ = 0;                                                                               \
  const bool clkOn_ = (threadIdx.x == 0 && blockIdx.y == 0 && static_cast<int>(blockIdx.x) == g_phaseNode); \
  if (clkOn_) {                                                                                \
    g_phaseClk[clkId_][0][0] = 0;                                                              \
    g_phaseClk[clkId_][0][1] = clock64();                                                      \
    clkN_ = 1;                                                                                 \
  }
#define PHASE_TICK()                                   \
  if (clkOn_ && clkN_ < 512) {                         \
    g_phaseClk[clkId_][clkN_][0] = __LINE__;           \
    g_phaseClk[clkId_][clkN_][1] = clock64();          \
    g_phaseCnt[clkId_] = ++clkN_;                      \
  }
#else
#define PHASE_CLOCK_BEGIN(id)
#define PHASE_TICK()
#endif

#define PHASE(...)                                   \
  {                                                  \
    const Par P{static_cast<int>(threadIdx.x), static_cast<int>(blockDim.x)}; \
    __VA_ARGS__                                      \
  }                                                  \
  __syncthreads();                                   \
  PHASE_TICK()

__device__ __forceinline__ NodeOut nodeOut(const WbDev& d, size_t node, size_t stage) {
  NodeOut out;
  out.A = const_cast<double*>(d.qp.A) + stage * NX * NX;
  out.Bt = const_cast<double*>(d.qp.Bm) + stage * NX * NUT_MAX;
  out.b = const_cast<double*>(d.qp.b) + stage * NX;
  out.Q = const_cast<double*>(d.qp.Q) + node * NX * NX;
  out.St = const_cast<double*>(d.qp.S) + stage * NUT_MAX * NX;
  out.Rt = const_cast<double*>(d.qp.R) + stage * NUT_MAX * NUT_MAX;
  out.q = const_cast<double*>(d.qp.q) + node * NX;
  out.rt = const_cast<double*>(d.qp.r) + stage * NUT_MAX;
  out.Pu = d.Pu + stage * NU * NUT_MAX;
  out.Px = d.Px + stage * NU * NX;
  out.u0 = d.u0p + stage * NU;
  out.nut = const_cast<int*>(d.qp.nu) + stage;
  out.perf = d.perfNode + node * 4;
  out.raw = d.raw ? d.raw + stage * d.rawPer : nullptr;
  return out;
}

// Terminal and event nodes are the same for every OCP family that runs in this device state (whole-body; centroidal, cen_kernels.cuh):
// returns true when node k was one of them and has been written.  Qfd: NX diagonal final-cost weights; rawNx / rawNu: dimensions of the
// optional raw block dump.
__device__ __forceinline__ bool lqTerminalOrEventNode(const WbDev& d, const NodeIn& n, int k, size_t node, size_t stage, const double* Qfd,
                                                      int rawNx, int rawNu, double* smem) {
  const int N = d.N;
  double* perf = d.perfNode + node * 4;
  if (k == N) {
    // setupTerminalNode: final cost 1/2 (x - xref)' Qf (x - xref)   (Transcription.cpp:125-154, HumanoidCostConstraintFactory.cpp:218-228)
    double* Q = const_cast<double*>(d.qp.Q) + node * NX * NX;
    double* q = const_cast<double*>(d.qp.q) + node * NX;
    for (int i = threadIdx.x; i < NX * NX; i += blockDim.x) Q[i] = (i % NX == i / NX) ? Qfd[i % NX] : 0.0;
    double part = 0.0;
    for (int i = threadIdx.x; i < NX; i += blockDim.x) {
      const double dx = n.x[i] - n.xref[i];
      q[i] = Qfd[i] * dx;
      part += 0.5 * Qfd[i] * dx * dx;
    }
    smem[threadIdx.x] = part;
    __syncthreads();
    if (threadIdx.x == 0) {
      double c = 0.0;
      for (int i = 0; i < blockDim.x; ++i) c += smem[i];
      perf[0] = c;
      perf[1] = perf[2] = perf[3] = 0.0;
    }
    return true;
  }
  if (n.event == 1) {
    // setupEventNode: identity jump map, no cost, no input (Transcription.cpp:156-192)
    NodeOut out = nodeOut(d, node, stage);
    double part = 0.0;
    for (int i = threadIdx.x; i < NX * NX; i += blockDim.x) {
      out.A[i] = (i % NX == i / NX) ? 1.0 : 0.0;
      out.Q[i] = 0.0;
    }
    for (int i = threadIdx.x; i < NX; i += blockDim.x) {
      const double df = n.x[i] - n.xnext[i];
      out.b[i] = df;
      out.q[i] = 0.0;
      part += df * df;
    }
    smem[threadIdx.x] = part;
    __syncthreads();
    if (threadIdx.x == 0) {
      double c = 0.0;
      for (int i = 0; i < blockDim.x; ++i) c += smem[i];
      perf[0] = 0.0;
      perf[1] = c;
      perf[2] = perf[3] = 0.0;
      *out.nut = 0;
    }
    if (out.raw) {
      for (long long i = threadIdx.x; i < d.rawPer; i += blockDim.x) out.raw[i] = 0.0;
      __syncthreads();
      for (int i = threadIdx.x; i < rawNx; i += blockDim.x) {
        out.raw[i + rawNx * i] = 1.0;
        out.raw[rawNx * rawNx + rawNx * rawNu + i] = n.x[i] - n.xnext[i];
      }
    }
    return true;
  }
  return false;
}

// K1a: node physics.  Intermediate nodes write their Mid record; terminal and event nodes are finished here.
__global__ void __launch_bounds__(LQA_THREADS, B200SQP_LQA_CTAS) lq_dyn_kernel(WbDev d) {
  extern __shared__ double smem[];
  const int k = blockIdx.x, b = blockIdx.y;
  if (d.flags[b * F_NF + F_CONVERGED]) return;
  const int N = d.N;
  const size_t node = static_cast<size_t>(b) * (N + 1) + k, stage = static_cast<size_t>(b) * N + k;
  NodeIn n;
  loadNode(d, b, k, n);
  n.x = d.x + node * NX;
  double* perf = d.perfNode + node * 4;
  if (k < N) {
    n.u = d.u + stage * NU;
    n.xnext = d.x + (node + 1) * NX;
  }
  const WbDeviceModel* const mb = d.instModel + static_cast<size_t>(b) * d.modelStride;
  if (lqTerminalOrEventNode(d, n, k, node, stage, mb->Qfd, NX, NU, smem)) return;
#if B200SQP_LQA_GLOBAL_MODEL
  const WbDeviceModel& m = *mb;   // read through L1 (8.7 KB, shared by every CTA of the SM): the shared memory buys a fourth node
#else
  __shared__ WbDeviceModel msh;  // model constants staged once per CTA: the kinematic phases read them in dependent sequences
  for (int i = threadIdx.x; i < static_cast<int>(sizeof(WbDeviceModel) / 8); i += blockDim.x)
    reinterpret_cast<double*>(&msh)[i] = reinterpret_cast<const double*>(mb)[i];
  __syncthreads();
  const WbDeviceModel& m = msh;
#endif
  LqWs s;
  lqWsMap(smem, s);
  double* const mid = d.mid + stage * Mid::SIZE;
  PHASE_CLOCK_BEGIN(0)
#include "wb_node_a.inc"
}

// Complete-pivoting LU of the constraint Jacobian D of every intermediate node (Eigen::FullPivLU semantics, luPhaseFactor), one warp per node.
// The factorisation is a chain of 12-14 dependent pivot steps (inside K1b it kept the seven other warps of the CTA waiting);
// as its own kernel 32 nodes are resident per SM and hide each other's latency.
constexpr int LU_PERM = 52;
constexpr int LU_XK = NC_MAX * (NX + 1) + NC_MAX * NUT_MAX;   // [X | x0] and K in pivot order (K1b part 1 -> part 2)
constexpr int LU_REC = LU_LD * NU + LU_XK;                   // per-stage record: LU factors | [X | x0], K
__global__ void __launch_bounds__(32) lu_kernel(WbDev d) {
  const int k = blockIdx.x, b = blockIdx.y;
  if (d.flags[b * F_NF + F_CONVERGED]) return;
  const size_t node = static_cast<size_t>(b) * (d.N + 1) + k, stage = static_cast<size_t>(b) * d.N + k;
  if (d.event[node] == 1) return;
  __shared__ double LU[LU_LD * NU];
  __shared__ int perm[LU_PERM];
  const double* __restrict__ const mid = d.mid + stage * Mid::SIZE;
  const int nc = static_cast<int>(mid[Mid::META + 0]);
  const int lane = threadIdx.x;
  for (int i = lane; i < NC_MAX * NU; i += 32) LU[(i % NC_MAX) + LU_LD * (i / NC_MAX)] = mid[Mid::CD + NC_MAX * NX + i];
  for (int i = lane; i < NC_MAX; i += 32) perm[i] = i;
  for (int i = lane; i < NU; i += 32) perm[16 + i] = i;
  __syncwarp();
  luPhaseFactor(Par{lane, 32}, nc, LU, perm, perm + 16);
  __syncwarp();
  // Eigen::FullPivLU's rank test (threshold eps * min(rows, cols) * |largest pivot|; the largest pivot of a complete-pivoting LU is the first).
  // luConstraintProjection would carry on with a larger null space; this path assumes full row rank (nut = NU - nc), so a rank-deficient D
  // (singular leg configuration, redundant rows) is reported as status 2 of the instance instead of dividing by a vanishing pivot silently.
  if (lane < nc && !(fabs(LU[lane + LU_LD * lane]) > 2.220446049250313e-16 * nc * fabs(LU[0]))) d.flags[b * F_NF + F_RANKDEF] = 1;
  double* out = d.luRec + stage * LU_REC;
  for (int i = lane; i < LU_LD * NU; i += 32) out[i] = LU[i];
  int* po = d.luPerm + stage * LU_PERM;
  for (int i = lane; i < LU_PERM; i += 32) po[i] = perm[i];
}

// K1b part 1: constraint projection (from the LU factors) and the dynamics in the projected inputs; 34 KB per node, six nodes per SM.
__global__ void __launch_bounds__(LQB1_THREADS, B200SQP_LQB1_CTAS) lq_projdyn_kernel(WbDev d) {
  extern __shared__ double smem[];
  const int k = blockIdx.x, b = blockIdx.y;
  if (d.flags[b * F_NF + F_CONVERGED]) return;
  const size_t node = static_cast<size_t>(b) * (d.N + 1) + k, stage = static_cast<size_t>(b) * d.N + k;
  if (d.event[node] == 1) return;
  const double* __restrict__ const mid = d.mid + stage * Mid::SIZE;
  const double* __restrict__ const luRec = d.luRec + stage * LU_REC;
  const int* __restrict__ const luPerm = d.luPerm + stage * LU_PERM;
  double* __restrict__ const xk = d.luRec + stage * LU_REC + LU_LD * NU;
  const double dt = mid[Mid::META + 3];
  PjWs s;
  pjDynWsMap(smem, s);
  NodeOut out = nodeOut(d, node, stage);
  PHASE_CLOCK_BEGIN(4)
#include "wb_node_b1.inc"
}

// K1b part 2: the node's Hessian and its change of input variables (the cost side of projectTranscription).
__global__ void __launch_bounds__(LQB_THREADS, B200SQP_LQB_CTAS) lq_proj_kernel(WbDev d) {
  extern __shared__ double smem[];
  const int k = blockIdx.x, b = blockIdx.y;
  if (d.flags[b * F_NF + F_CONVERGED]) return;
  const size_t node = static_cast<size_t>(b) * (d.N + 1) + k, stage = static_cast<size_t>(b) * d.N + k;
  if (d.event[node] == 1) return;
  const double* __restrict__ const mid = d.mid + stage * Mid::SIZE;
  const double* __restrict__ const xk = d.luRec + stage * LU_REC + LU_LD * NU;
  const int* __restrict__ const luPerm = d.luPerm + stage * LU_PERM;
  const double dt = mid[Mid::META + 3];
  PjWs s;
  NodeOut out = nodeOut(d, node, stage);
  pjCostWsMap(smem, out.Q, s);
  PHASE_CLOCK_BEGIN(1)
#include "wb_node_b2.inc"
}

// ---- K4a: remap the projected QP solution, Armijo metric and norms (one CTA per (instance, stage)) --------------------------------------------
__global__ void __launch_bounds__(128) remap_kernel(WbDev d) {
  const int k = blockIdx.x, b = blockIdx.y;
  if (d.flags[b * F_NF + F_CONVERGED]) return;
  const int N = d.N;
  const size_t node = static_cast<size_t>(b) * (N + 1) + k, stage = static_cast<size_t>(b) * N + k;
  __shared__ double red[128][3];
  const int nut = d.qp.nu[stage];
  const double* dx = d.qp.dx + node * NX;
  const double* dut = d.qp.du + stage * NUT_MAX;
  double* du = d.du + stage * NU;
  double arm = 0.0, dxn = 0.0, dun = 0.0;
  // remapProjectedInput (ocs2_oc/src/multiple_shooting/Helpers.cpp:38-48): du = Pu dut + Px dx + u0.  35 outputs x 81 terms: three threads per
  // output take every third term (fixed partition, so the result is deterministic), the operand vector is staged once.
  __shared__ double zsh[NUT_MAX + NX], part[3][NU];
  for (int j = threadIdx.x; j < nut + NX; j += blockDim.x) zsh[j] = j < nut ? dut[j] : dx[j - nut];
  __syncthreads();
  if (nut > 0 && threadIdx.x < 3 * NU) {
    const int i = threadIdx.x % NU, p = threadIdx.x / NU;
    const double* Pu = d.Pu + stage * NU * NUT_MAX;
    const double* Px = d.Px + stage * NU * NX;
    double acc = 0.0;
    for (int j = p; j < nut + NX; j += 3) acc = fma(j < nut ? Pu[i + NU * j] : Px[i + NU * (j - nut)], zsh[j], acc);
    part[p][i] = acc;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < NU; i += blockDim.x) {
    const double s = nut > 0 ? ((d.u0p[stage * NU + i] + part[0][i]) + part[1][i]) + part[2][i] : 0.0;
    du[i] = s;
    dun = fma(s, s, dun);
  }
  for (int i = threadIdx.x; i < NX; i += blockDim.x) {
    arm = fma(d.qp.q[node * NX + i], dx[i], arm);
    dxn = fma(dx[i], dx[i], dxn);
    if (k == N - 1) {  // terminal node terms
      const double dxe = d.qp.dx[(node + 1) * NX + i];
      arm = fma(d.qp.q[(node + 1) * NX + i], dxe, arm);
      dxn = fma(dxe, dxe, dxn);
    }
  }
  for (int i = threadIdx.x; i < nut; i += blockDim.x) arm = fma(d.qp.r[stage * NUT_MAX + i], dut[i], arm);
  if (d.Kre && nut > 0) {
    // remapProjectedGain (Helpers.cpp:50-58): K = Pu Kt + Px
    const double* Pu = d.Pu + stage * NU * NUT_MAX;
    const double* Px = d.Px + stage * NU * NX;
    const double* Kt = d.qp.K + stage * NUT_MAX * NX;
    double* Ko = d.Kre + stage * NU * NX;
    for (int it = threadIdx.x; it < NU * NX; it += blockDim.x) {
      const int i = it % NU, j = it / NU;
      double s = Px[it];
      for (int l = 0; l < nut; ++l) s = fma(Pu[i + NU * l], Kt[l + NUT_MAX * j], s);
      Ko[it] = s;
    }
  } else if (d.Kre) {
    for (int it = threadIdx.x; it < NU * NX; it += blockDim.x) d.Kre[stage * NU * NX + it] = 0.0;
  }
  red[threadIdx.x][0] = arm;
  red[threadIdx.x][1] = dxn;
  red[threadIdx.x][2] = dun;
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0, x2 = 0, u2 = 0;
    for (int i = 0; i < blockDim.x; ++i) {
      a += red[i][0];
      x2 += red[i][1];
      u2 += red[i][2];
    }
    double* o = d.lsNode + node * 4;
    o[0] = a;
    o[1] = x2;
    o[2] = u2;
  }
}

// ---- K4b: per-instance reductions and line-search logic (one CTA per instance) ------------------------------------------------------------
__device__ __forceinline__ double blockSum(double v, double* sh) {
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  const double r = sh[0];
  __syncthreads();
  return r;
}

// mode 0: baseline PerformanceIndex from perfNode (after K1).  mode 1: Armijo/norm sums from lsNode (after remap) + line-search init.
__global__ void __launch_bounds__(128) prep_kernel(WbDev d, int mode) {
  const int b = blockIdx.x;
  if (d.flags[b * F_NF + F_CONVERGED]) return;
  __shared__ double sh[128];
  const int N = d.N;
  const double* src = (mode == 0 ? d.perfNode : d.lsNode) + static_cast<size_t>(b) * (N + 1) * 4;
  double a0 = 0, a1 = 0, a2 = 0;
  const int cnt = (mode == 0) ? N + 1 : N;
  for (int k = threadIdx.x; k < cnt; k += blockDim.x) {
    a0 += src[4 * k];
    a1 += src[4 * k + 1];
    a2 += src[4 * k + 2];
  }
  double x0d = 0.0;
  if (mode == 0)
    for (int i = threadIdx.x; i < NX; i += blockDim.x) {
      const double df = d.x0[b * NX + i] - d.x[static_cast<size_t>(b) * (N + 1) * NX + i];
      x0d = fma(df, df, x0d);
    }
  a0 = blockSum(a0, sh);
  a1 = blockSum(a1, sh);
  a2 = blockSum(a2, sh);
  x0d = blockSum(x0d, sh);
  if (mode == 0) {
    // delta_x0 = initState - x[0]  (SqpSolver.cpp:236)
    for (int i = threadIdx.x; i < NX; i += blockDim.x)
      const_cast<double*>(d.qp.dx0)[b * NX + i] = d.x0[b * NX + i] - d.x[static_cast<size_t>(b) * (N + 1) * NX + i];
  }
  if (threadIdx.x == 0) {
    double* in = d.inst + b * I_ND;
    if (mode == 0) {
      in[I_BASE_COST] = a0;
      in[I_BASE_DYN] = a1 + x0d;
      in[I_BASE_EQ] = a2;
      in[I_BASE_MERIT] = a0;  // merit = cost + Lagrangians (both zero here)
    } else {
      in[I_ARMIJO] = a0;
      in[I_DXN] = sqrt(a1);
      in[I_DUN] = sqrt(a2);
      in[I_ALPHA] = 1.0;
      in[I_STEP] = 0.0;
      d.flags[b * F_NF + F_LSDONE] = 0;
      if (d.flags[b * F_NF + F_RANKDEF]) {  // constraint Jacobian without full row rank (lu_kernel): the projected QP is not the reference's
        d.flags[b * F_NF + F_STATUS] = 2;
      } else if (d.qp.status[b]) {  // QP failed: no step, report through status
        d.flags[b * F_NF + F_STATUS] = 1;
      }
    }
  }
}

// K3.  RO_PACK shooting nodes per CTA (see RO_PACK above): every PHASE body is instantiated once per node on a slice of the threads rotated by
// 64 lanes; the nodes of a CTA share the barriers.
__device__ __forceinline__ void rolloutNodes(const WbDev& d, const WbDeviceModel& m, NodeIn* nsh, double* smem, int b, int k0) {
  const int tid = threadIdx.x;
  const int N = d.N;
  const double alpha = d.inst[b * I_ND + I_ALPHA];
  const size_t roStride = roWsDoubles();
  const size_t node0 = static_cast<size_t>(b) * (N + 1) + k0, stage0 = static_cast<size_t>(b) * N + k0;
  double* const perfBase = d.lsNode + node0 * 4;
  bool live[RO_PACK];
#pragma unroll
  for (int h = 0; h < RO_PACK; ++h) {
    const int k = k0 + h;
    live[h] = k <= N;
    if (!live[h]) continue;
    RoWs r;
    roWsMap(smem + h * roStride, r);
    if (tid == 0) {
      NodeIn n;
      loadNode(d, b, k, n);
      n.x = r.xa;
      n.u = r.ua;
      n.xnext = r.xna;
      nsh[h] = n;
    }
    for (int i = tid; i < NX; i += blockDim.x) {
      r.xa[i] = fma(alpha, d.qp.dx[(node0 + h) * NX + i], d.x[(node0 + h) * NX + i]);
      if (k < N) r.xna[i] = fma(alpha, d.qp.dx[(node0 + h + 1) * NX + i], d.x[(node0 + h + 1) * NX + i]);
    }
    if (k < N)
      for (int i = tid; i < NU; i += blockDim.x) r.ua[i] = fma(alpha, d.du[(stage0 + h) * NU + i], d.u[(stage0 + h) * NU + i]);
  }
  __syncthreads();
  // terminal and pre-event nodes: one short sum each, by the first thread of the node's slice
#pragma unroll
  for (int h = 0; h < RO_PACK; ++h) {
    if (!live[h]) continue;
    const int k = k0 + h;
    const NodeIn& n = nsh[h];
    if (k == N || n.event == 1) {
      live[h] = false;
      if (tid == 64 * h) {
        RoWs r;
        roWsMap(smem + h * roStride, r);
        double c = 0.0;
        for (int i = 0; i < NX; ++i) {
          if (k == N) {
            const double dx = r.xa[i] - n.xref[i];
            c += 0.5 * m.Qfd[i] * dx * dx;
          } else {
            const double df = r.xa[i] - r.xna[i];
            c += df * df;
          }
        }
        double* perfOut = perfBase + 4 * h;
        perfOut[0] = (k == N) ? c : 0.0;
        perfOut[1] = (k == N) ? 0.0 : c;
        perfOut[2] = 0.0;
      }
    }
  }
  bool any = false;
#pragma unroll
  for (int h = 0; h < RO_PACK; ++h) any = any || live[h];
  if (!any) return;
  PHASE_CLOCK_BEGIN(2)
#define RO_NODE(h_, ...)                                             \
  if (live[h_]) {                                                    \
    RoWs r;                                                          \
    roWsMap(smem + (h_) * roStride, r);                              \
    const NodeIn& n = nsh[h_];                                       \
    DynWs& W = *r.dyn;                                               \
    double* const perfOut = perfBase + 4 * (h_);                     \
    const Par P = rot(Par{tid, RO_THREADS}, 64 * (h_));              \
    (void)n;                                                         \
    (void)perfOut;                                                   \
    __VA_ARGS__                                                      \
  }
#undef PHASE
#if B200SQP_RO_PACK == 1
#define RO_NODES(...) RO_NODE(0, __VA_ARGS__)
#elif B200SQP_RO_PACK == 2
#define RO_NODES(...) RO_NODE(0, __VA_ARGS__) RO_NODE(1, __VA_ARGS__)
#else
#define RO_NODES(...) RO_NODE(0, __VA_ARGS__) RO_NODE(1, __VA_ARGS__) RO_NODE(2, __VA_ARGS__)
#endif
#define PHASE(...)           \
  { RO_NODES(__VA_ARGS__) }  \
  __syncthreads();           \
  PHASE_TICK()
#include "wb_rollout_body.inc"
#undef PHASE
#undef RO_NODES
#undef RO_NODE
}

// One CTA walks the instances b = blockIdx.y, blockIdx.y + gridDim.y, ...: the first trials of the line search are launched with one instance per
// CTA row; the later ones -- in which almost every instance has finished and its thread blocks would only be launched to return -- with an
// sixteenth of the rows (the asynchronous solve enqueues the whole back-tracking ladder, wb_capi.inc).
__global__ void __launch_bounds__(RO_THREADS, B200SQP_RO_CTAS) rollout_kernel(WbDev d) {
  extern __shared__ double smem[];
#if !B200SQP_RO_GLOBAL_MODEL
  __shared__ WbDeviceModel msh;
#endif
  __shared__ NodeIn nsh[RO_PACK];
  __shared__ int nAct, act[RO_THREADS];
  const int k0 = blockIdx.x * RO_PACK;
  // the instances of this CTA row that still search, found with ONE round of flag loads (a late trial walks sixteen instances per CTA and
  // nearly all of them have finished: sixteen dependent load pairs cost more than the rest of such a launch)
  if (threadIdx.x == 0) nAct = 0;
  __syncthreads();
  for (int j = threadIdx.x; blockIdx.y + j * gridDim.y < d.B; j += blockDim.x) {
    const int b = blockIdx.y + j * gridDim.y;
    if (!(d.flags[b * F_NF + F_CONVERGED] | d.flags[b * F_NF + F_LSDONE])) {
      const int slot = atomicAdd(&nAct, 1);
      if (slot < RO_THREADS) act[slot] = b;
    }
  }
  __syncthreads();
  const int n = nAct;
  if (n == 0) return;
  for (int a = 0; a < n; ++a) {   // (the instances of one CTA may carry different gains: the model is looked up per instance)
    const WbDeviceModel* const mb = d.instModel + static_cast<size_t>(act[a]) * d.modelStride;
#if B200SQP_RO_GLOBAL_MODEL
    const WbDeviceModel& msh = *mb;   // read through L1 (8.7 KB, shared by every CTA of the SM) instead of one copy per CTA
#else
    for (int i = threadIdx.x; i < static_cast<int>(sizeof(WbDeviceModel) / 8); i += blockDim.x)
      reinterpret_cast<double*>(&msh)[i] = reinterpret_cast<const double*>(mb)[i];
    __syncthreads();
#endif
    rolloutNodes(d, msh, nsh, smem, act[a], k0);
    __syncthreads();   // the workspace is reused by the next instance
  }
}

// trial PerformanceIndex of one instance at its current alpha (sums over the per-node results of K3) and the filter test
// (FilterLinesearch::acceptStep, FilterLinesearch.cpp:34-57)
struct TrialEval {
  double cost, dyn, eq, merit, g1;
  bool acc;
  int type;
};
__device__ __forceinline__ TrialEval evalTrial(const WbDev& d, int b, double alpha, double* sh) {
  const int N = d.N;
  const double* in = d.inst + b * I_ND;
  const double* src = d.lsNode + static_cast<size_t>(b) * (N + 1) * 4;
  double a0 = 0, a1 = 0, a2 = 0;
  for (int k = threadIdx.x; k <= N; k += blockDim.x) {
    a0 += src[4 * k];
    a1 += src[4 * k + 1];
    a2 += src[4 * k + 2];
  }
  double x0d = 0.0;
  for (int i = threadIdx.x; i < NX; i += blockDim.x) {
    // initState - xNew[0] with xNew[0] = x[0] + alpha (initState - x[0])
    const double df = (1.0 - alpha) * d.qp.dx0[b * NX + i];
    x0d = fma(df, df, x0d);
  }
  a0 = blockSum(a0, sh);
  a1 = blockSum(a1, sh);
  a2 = blockSum(a2, sh);
  x0d = blockSum(x0d, sh);
  const b200sqp_settings& st = d.st;
  TrialEval t;
  t.cost = a0;
  t.dyn = a1 + x0d;
  t.eq = a2;
  t.merit = a0;
  const double g0 = sqrt(in[I_BASE_DYN] + in[I_BASE_EQ]);
  t.g1 = sqrt(t.dyn + t.eq);
  const double arm = alpha * in[I_ARMIJO];
  if (d.flags[b * F_NF + F_STATUS]) {  // QP failure: never accept
    t.acc = false;
    t.type = 0;
  } else if (t.g1 > st.g_max) {
    t.acc = t.g1 < (1.0 - st.gamma_c) * g0;
    t.type = 1;  // CONSTRAINT
  } else if (t.g1 < st.g_min && g0 < st.g_min && arm < 0.0) {
    t.acc = t.merit < in[I_BASE_MERIT] + st.armijo_factor * arm;
    t.type = 3;  // COST
  } else {
    t.acc = t.merit < in[I_BASE_MERIT] - st.gamma_c * g0 || t.g1 < (1.0 - st.gamma_c) * g0;
    t.type = 2;  // DUAL
  }
  return t;
}

// FilterLinesearch::acceptStep + takeStep bookkeeping + checkConvergence for one instance (SqpSolver.cpp:484-602).
// forced = 0: per-instance back-tracking (reference semantics); 1: take the current (globally chosen) alpha; 2: take a zero step.
__global__ void __launch_bounds__(256) accept_kernel(WbDev d, int forced) {
  const int b = blockIdx.x;
  int* fl = d.flags + b * F_NF;
  if (fl[F_CONVERGED] || fl[F_LSDONE]) return;
  __shared__ double sh[256];
  __shared__ int decision;  // 0 continue, 1 accepted, 2 give up (zero step)
  const int N = d.N;
  double* in = d.inst + b * I_ND;
  const double alpha = in[I_ALPHA];
  const TrialEval t = evalTrial(d, b, alpha, sh);
  const b200sqp_settings& st = d.st;
  if (threadIdx.x == 0) {
    int dec = 0;
    const bool take = (forced == 1) ? !fl[F_STATUS] : (forced == 2 ? false : t.acc);
    if (take) {
      dec = 1;
      in[I_STEP] = alpha;
      in[I_STEPTYPE] = t.type;
      in[I_NEW_MERIT] = t.merit;
      in[I_NEW_COST] = t.cost;
      in[I_NEW_DYN] = t.dyn;
      in[I_NEW_EQ] = t.eq;
    } else {
      const double next = alpha * st.alpha_decay;
      if (forced || fl[F_STATUS] || (next * in[I_DXN] < st.delta_tol && next * in[I_DUN] < st.delta_tol) || !(next >= st.alpha_min)) {
        dec = 2;
        in[I_STEP] = 0.0;
        in[I_STEPTYPE] = 4;  // ZERO
        in[I_NEW_MERIT] = in[I_BASE_MERIT];
        in[I_NEW_COST] = in[I_BASE_COST];
        in[I_NEW_DYN] = in[I_BASE_DYN];
        in[I_NEW_EQ] = in[I_BASE_EQ];
      } else {
        in[I_ALPHA] = next;
      }
    }
    decision = dec;
  }
  __syncthreads();
  if (decision == 0) return;
  if (decision == 1) {  // x <- x + alpha dx, u <- u + alpha du
    for (size_t i = threadIdx.x; i < static_cast<size_t>(N + 1) * NX; i += blockDim.x) {
      const size_t g = static_cast<size_t>(b) * (N + 1) * NX + i;
      d.x[g] = fma(alpha, d.qp.dx[g], d.x[g]);
    }
    for (size_t i = threadIdx.x; i < static_cast<size_t>(N) * NU; i += blockDim.x) {
      const size_t g = static_cast<size_t>(b) * N * NU + i;
      d.u[g] = fma(alpha, d.du[g], d.u[g]);
    }
  }
  if (threadIdx.x == 0) {
    fl[F_LSDONE] = 1;
    atomicSub(d.pending, 1);
    const int iter = fl[F_ITER];
    const double step = in[I_STEP];
    const double dxn = step * in[I_DXN], dun = step * in[I_DUN];
    // checkConvergence (SqpSolver.cpp:583-602)
    int conv = 0;
    if (iter + 1 >= st.sqp_iteration) conv = 1;  // ITERATIONS
    else if (step < st.alpha_min) conv = 2;        // STEPSIZE
    else if (fabs(in[I_NEW_MERIT] - in[I_BASE_MERIT]) < st.cost_tol && sqrt(in[I_NEW_DYN] + in[I_NEW_EQ]) < st.g_min) conv = 3;  // METRICS
    else if (dxn < st.delta_tol && dun < st.delta_tol) conv = 4;  // PRIMAL
    if (iter < d.maxIter) {
      b200sqp_iter_log& L = d.log[static_cast<size_t>(b) * d.maxIter + iter];
      L.base_merit = in[I_BASE_MERIT];
      L.base_cost = in[I_BASE_COST];
      L.base_dyn_sse = in[I_BASE_DYN];
      L.base_eq_sse = in[I_BASE_EQ];
      L.merit = in[I_NEW_MERIT];
      L.cost = in[I_NEW_COST];
      L.dyn_sse = in[I_NEW_DYN];
      L.eq_sse = in[I_NEW_EQ];
      L.step_size = step;
      L.step_type = in[I_STEPTYPE];
      L.dx_norm = dxn;
      L.du_norm = dun;
      L.armijo = in[I_ARMIJO];
      L.convergence = conv;
      L.pad[0] = L.pad[1] = 0.0;
    }
    fl[F_ITER] = iter + 1;
    fl[F_CONVCODE] = conv;
    if (conv) fl[F_CONVERGED] = 1;
  }
}

// ---- global-step mode (SURVEY.md section 8e) ------------------------------------------------------------------------------------------------
// every active instance gets the same trial step size
__global__ void __launch_bounds__(256) set_alpha_kernel(WbDev d, double alpha) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= d.B || d.flags[b * F_NF + F_CONVERGED]) return;
  d.inst[b * I_ND + I_ALPHA] = alpha;
  d.flags[b * F_NF + F_LSDONE] = 0;
}
// candidate j of the ladder: filter test of every active instance, no state change; statistics accumulated with atomics
__global__ void __launch_bounds__(256) ladder_eval_kernel(WbDev d, int j) {
  const int b = blockIdx.x;
  const int* fl = d.flags + b * F_NF;
  if (fl[F_CONVERGED] || fl[F_STATUS]) return;
  __shared__ double sh[256];
  const TrialEval t = evalTrial(d, b, d.inst[b * I_ND + I_ALPHA], sh);
  if (threadIdx.x == 0) {
    double* s = d.gstats + 4 * j;
    if (t.acc) {
      atomicAdd(s, 1.0);
      atomicAdd(s + 1, t.merit);
    }
    // max of non-negative doubles = max of their bit patterns
    atomicMax(reinterpret_cast<unsigned long long*>(s + 2), static_cast<unsigned long long>(__double_as_longlong(t.g1)));
    atomicAdd(s + 3, 1.0);
  }
}

// extractValueFunction (SqpSolver.cpp:321-329): p_i -= P_i x_i with x the linearisation trajectory (before the step); one CTA per node
__global__ void __launch_bounds__(64) value_function_kernel(WbDev d) {
  const int k = blockIdx.x, b = blockIdx.y;
  if (d.flags[b * F_NF + F_CONVERGED]) return;
  const size_t node = static_cast<size_t>(b) * (d.N + 1) + k;
  const double* Pm = d.qp.P + node * NX * NX;
  const double* x = d.x + node * NX;
  for (int i = threadIdx.x; i < NX; i += blockDim.x) {
    double s = 0.0;
    for (int j = 0; j < NX; ++j) s = fma(Pm[i + NX * j], x[j], s);
    d.qp.p[node * NX + i] -= s;
  }
}

__global__ void __launch_bounds__(256) count_active_kernel(WbDev d) {
  // pending = number of instances that have not converged (they enter the next line search)
  __shared__ int cnt[256];
  int c = 0;
  for (int b = threadIdx.x; b < d.B; b += blockDim.x) c += !d.flags[b * F_NF + F_CONVERGED];
  cnt[threadIdx.x] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int i = 0; i < blockDim.x; ++i) t += cnt[i];
    *d.pending = t;
  }
}

#undef PHASE
#undef PHASE_TICK
#undef PHASE_CLOCK_BEGIN

}  // namespace b200sqp
