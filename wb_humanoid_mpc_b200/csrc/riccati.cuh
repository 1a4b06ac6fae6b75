// K2: batched Riccati backward factorisation + forward substitution, one persistent CTA per QP instance.
//
// Replaces HpipmInterface::solve + getRiccatiFeedback/Feedforward/CostToGo
// (lib/ocs2_ros2/ocs2_sqp/hpipm_catkin/src/HpipmInterface.cpp:166-455), i.e. HPIPM's unconstrained-QP path
// (one Riccati factorisation + one substitution; reg_prim on the Hessian diagonals).
//
// Data layout: include/b200sqp.h section (1).  P and p live in shared memory for the whole backward sweep.  Each stage record
// is streamed from HBM exactly once in the backward sweep; the copy of stage k-1 is issued with cp.async as soon as its
// destination buffers are dead and overlaps the factorisation of stage k.  The 58-wide contractions run on the fp64 tensor
// path (DMMA m8n8k4).  The forward sweep double-buffers (A|B), K, k, b the same way.
#pragma once
#include <cuda_pipeline.h>

#include "dense.cuh"
#include "dense_par.cuh"

namespace b200sqp {

// development aid (tools/phase_clock.py, -DB200SQP_PHASE_CLOCK): cycles of instance 0 accumulated per barrier slot over all stages
#ifdef B200SQP_PHASE_CLOCK
__device__ long long g_ricClk[32][2];
#define RIC_TICK(slot)                                                   \
  if (threadIdx.x == 0 && blockIdx.x == 0) {                             \
    const long long now_ = clock64();                                    \
    g_ricClk[slot][0] = __LINE__;                                        \
    g_ricClk[slot][1] += now_ - ricT_;                                   \
    ricT_ = now_;                                                        \
  }
#define RIC_CLOCK_BEGIN()                                                \
  long long ricT_ = clock64();                                           \
  if (threadIdx.x == 0 && blockIdx.x == 0)                               \
    for (int i_ = 0; i_ < 32; ++i_) g_ricClk[i_][0] = g_ricClk[i_][1] = 0;
#else
#define RIC_TICK(slot)
#define RIC_CLOCK_BEGIN()
#endif

struct QpDeviceView {
  int B, N, nx, numax;
  const double *A, *Bm, *b, *Q, *S, *R, *q, *r, *dx0;
  const int* nu;  // [B][N] or nullptr
  double *K, *kff, *P, *p, *dx, *du;
  int* status;  // [B]
  int keepP;
  double reg;
  // optional per-instance skip flags (the SQP solver's F_CONVERGED word, stride skipStride ints): a converged instance keeps the QP outputs
  // of the iteration it converged in -- in particular its re-centred cost-to-go (SqpSolver::extractValueFunction)
  const int* skip;
  int skipStride;
};

// The granularity of a batch array: one row per instance, per node (N + 1 per instance) or per stage (N per instance), or one block for the
// whole handle.  batchRows: the rows of B instances of `nodes` nodes each.
enum RowKind { ROW_INST, ROW_NODE, ROW_STAGE, ROW_HANDLE };
__host__ __device__ inline size_t batchRows(RowKind k, size_t B, int nodes) {
  return k == ROW_INST ? B : k == ROW_NODE ? B * nodes : k == ROW_STAGE ? B * (nodes - 1) : 1;
}

// The arrays of a QP batch, in allocation order: f(field, row kind, width in elements).  withP: the cost-to-go matrices, which only a solve
// that keeps them needs.
template <class F>
void forEachQpArray(QpDeviceView& v, bool withP, F&& f) {
  const int nx = v.nx, nm = v.numax;
  f(v.A, ROW_STAGE, nx * nx);
  f(v.Bm, ROW_STAGE, nx * nm);
  f(v.b, ROW_STAGE, nx);
  f(v.Q, ROW_NODE, nx * nx);
  f(v.S, ROW_STAGE, nm * nx);
  f(v.R, ROW_STAGE, nm * nm);
  f(v.q, ROW_NODE, nx);
  f(v.r, ROW_STAGE, nm);
  f(v.dx0, ROW_INST, nx);
  f(v.nu, ROW_STAGE, 1);
  f(v.K, ROW_STAGE, nm * nx);
  f(v.kff, ROW_STAGE, nm);
  f(v.p, ROW_NODE, nx);
  if (withP) f(v.P, ROW_NODE, nx * nx);
  f(v.dx, ROW_NODE, nx);
  f(v.du, ROW_STAGE, nm);
  f(v.status, ROW_INST, 1);
}

__host__ __device__ inline int even_up(int n) { return (n + 1) & ~1; }

struct RicLayout {
  int pq, ab, w, y, rs, linv, vec, total;  // sizes in doubles
  int kout;   // offset of [K | k] inside W
};
// Vectors ride along as extra matrix columns so that every matrix-vector product is folded into a tensor-core GEMM:
//   PQ = [P | p] (nx x (nx+1)),  AB = [A | b | B] (nx x (nx+1+nm)),  Y = [S | r] (nm x (nx+1))
// The scratch W first holds P [A | b | B] (the shape of AB), later [Yl | yl] (nm x (nx+1), at the leading dimension of Y) followed by
// [K | k] (nm x (nx+1), leading dimension nm): it is sized for the larger of the two uses (the second one, roughly, once nm >= nx).
__host__ __device__ inline RicLayout riccati_layout(int nx, int nm) {
  RicLayout L;
  L.pq = even_up(nx * (nx + 1));
  L.ab = even_up(nx * (nx + 1 + nm));
  L.kout = even_up(nm * (nx + 1));
  const int ylk = L.kout + even_up(nm * (nx + 1));   // [Yl | yl] and [K | k]
  L.w = ylk > L.ab ? ylk : L.ab;
  L.y = even_up(nm * (nx + 1));
  L.rs = even_up(nm * nm);
  L.linv = even_up(nm * nm);
  L.vec = even_up(nx) * 2 + even_up(nm) * 3 + 8;
  L.total = 2 * L.pq + 2 * L.ab + L.w + 2 * L.y + 2 * L.rs + L.linv + L.vec;
  return L;
}
// Leading dimensions of the shared-memory operands of the one-CTA kernel: ld = 4 (mod 8) makes every DMMA fragment load conflict free.  A
// fragment load reads, per half-warp, the doubles {r + ld*c : r, c in 0..3} (or {c + ld*r}); with 16 eight-byte banks these are 16 distinct
// banks iff 4*ld = +-8... i.e. ld = 4 or 12 (mod 16); nx = 58 (ld 58 = 10 mod 16) paid a two-way conflict on every operand fetch.
__host__ __device__ inline int ric_pad(int n) { return ((n + 3) & ~7) + 4; }
__host__ __device__ inline RicLayout riccati_layout_padded(int nx, int nm) {
  const int lx = ric_pad(nx), lm = ric_pad(nm);
  RicLayout L;
  L.pq = even_up(lx * (nx + 1));
  L.ab = even_up(lx * (nx + 1 + nm));
  L.kout = even_up(lm * (nx + 1));
  const int ylk = L.kout + even_up(nm * (nx + 1));   // [Yl | yl] and [K | k]
  L.w = ylk > L.ab ? ylk : L.ab;
  L.y = even_up(lm * (nx + 1));
  L.rs = even_up(lm * nm);
  L.linv = even_up(lm * nm);
  L.vec = even_up(nx) * 2 + even_up(nm) * 3 + 8;
  L.total = 2 * L.pq + 2 * L.ab + L.w + 2 * L.y + 2 * L.rs + L.linv + L.vec;
  return L;
}
__host__ __device__ inline size_t riccati_smem_doubles(int nx, int numax) { return static_cast<size_t>(riccati_layout_padded(nx, numax).total); }

// asynchronous global -> shared copy of n doubles by the whole block (16-byte chunks when both sides allow it)
__device__ __forceinline__ void async_copy(double* dst, const double* src, int n) {
  const bool wide = ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0 && (n & 1) == 0;
  if (wide) {
    for (int i = threadIdx.x; i < (n >> 1); i += blockDim.x) __pipeline_memcpy_async(dst + 2 * i, src + 2 * i, 16);
  } else {
    for (int i = threadIdx.x; i < n; i += blockDim.x) __pipeline_memcpy_async(dst + i, src + i, 8);
  }
}

// the same for a (rows x cols) column-major block with source / destination leading dimensions lds / ldd
__device__ __forceinline__ void async_copy_cols(double* dst, int ldd, const double* src, int lds, int rows, int cols) {
  const bool wide = ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0 && ((rows | lds | ldd) & 1) == 0;
  if (wide) {
    const int h = rows >> 1;
    for (int i = threadIdx.x; i < h * cols; i += blockDim.x) {
      const int c = i / h, r = 2 * (i - c * h);
      __pipeline_memcpy_async(dst + r + c * ldd, src + r + c * lds, 16);
    }
  } else {
    for (int i = threadIdx.x; i < rows * cols; i += blockDim.x) {
      const int c = i / rows, r = i - c * rows;
      __pipeline_memcpy_async(dst + r + c * ldd, src + r + c * lds, 8);
    }
  }
}

// NXT / NMT > 0: sizes fixed at compile time (the whole-body instantiation <58, 23>: index arithmetic folds to shifts and multiplies);
// 0: read from the view (generic QP interface)
template <int NXT, int NMT>
__global__ void __launch_bounds__(256, 1) riccati_kernel(QpDeviceView v) {
  extern __shared__ double sm[];
  const int inst = blockIdx.x;
  if (v.skip && v.skip[inst * v.skipStride]) return;
  const int nx = NXT ? NXT : v.nx, nm = NMT ? NMT : v.numax, N = v.N, nx1 = nx + 1;
  const RicLayout L = riccati_layout_padded(nx, nm);
  const int lx = ric_pad(nx), lm = ric_pad(nm);   // leading dimensions of the nx-row / nm-row operands in the backward sweep
  double* PQ[2] = {sm, sm + L.pq};
  double* AB[2] = {sm + 2 * L.pq, sm + 2 * L.pq + L.ab};
  double* W = AB[1] + L.ab;
  double* Y[2] = {W + L.w, W + L.w + L.y};
  double* Rs[2] = {Y[1] + L.y, Y[1] + L.y + L.rs};
  double* Linv = Rs[1] + L.rs;
  double* vec = Linv + L.linv;
  const int ex = even_up(nx), em = even_up(nm);
  double* xv = vec;            // forward state [x; 1; u] is assembled in xa
  double* tv = vec + ex;
  double* uv = vec + 2 * ex;
  double* kb[2] = {vec + 2 * ex + em, vec + 2 * ex + 2 * em};
  __shared__ int ok;
  if (threadIdx.x == 0) ok = 1;
  const Par P{static_cast<int>(threadIdx.x), static_cast<int>(blockDim.x)};

  const size_t iN = static_cast<size_t>(inst) * N, iN1 = static_cast<size_t>(inst) * (N + 1);
  int cur = 0;
  // terminal stage: [P_N | p_N] = [Q_N + reg I | q_N]
  {
    const double* QN = v.Q + (iN1 + N) * nx * nx;
    for (int i = threadIdx.x; i < nx * nx; i += blockDim.x) {
      const int r = i % nx, c = i / nx;
      PQ[cur][r + c * lx] = QN[i] + (r == c ? v.reg : 0.0);
    }
    block_copy(nx, v.q + (iN1 + N) * nx, PQ[cur] + lx * nx);
    __syncthreads();
    if (v.keepP) {
      for (int i = threadIdx.x; i < nx * nx; i += blockDim.x) v.P[(iN1 + N) * nx * nx + i] = PQ[cur][(i % nx) + (i / nx) * lx];
      block_copy(nx, PQ[cur] + lx * nx, v.p + (iN1 + N) * nx);
    }
  }
  auto prefetch = [&](int k, int set, double* qdst) {
    const size_t sk = iN + k;
    const int nu = v.nu ? v.nu[sk] : nm;
    async_copy_cols(AB[set], lx, v.A + sk * nx * nx, nx, nx, nx);
    async_copy(AB[set] + lx * nx, v.b + sk * nx, nx);
    if (nu > 0) {
      async_copy_cols(AB[set] + lx * nx1, lx, v.Bm + sk * nx * nm, nx, nx, nu);
      async_copy_cols(Y[set], lm, v.S + sk * nm * nx, nm, nm, nx);
      async_copy(Y[set] + lm * nx, v.r + sk * nm, nu);
      async_copy_cols(Rs[set], lm, v.R + sk * nm * nm, nm, nm, nm);
    }
    async_copy_cols(qdst, lx, v.Q + (iN1 + k) * nx * nx, nx, nx, nx);
    async_copy(qdst + lx * nx, v.q + (iN1 + k) * nx, nx);
    __pipeline_commit();
  };
  prefetch(N - 1, 0, PQ[1 - cur]);
  RIC_CLOCK_BEGIN()

  for (int k = N - 1; k >= 0; --k) {
    const int set = (N - 1 - k) & 1;
    const int nu = v.nu ? v.nu[iN + k] : nm;
    const size_t sk = iN + k;
    double* Pc = PQ[cur];
    double* Pn = PQ[1 - cur];
    double* ABk = AB[set];
    double* Yk = Y[set];
    double* Rk = Rs[set];
    __pipeline_wait_prior(0);
    __syncthreads();
    RIC_TICK(1)
    // ---- W = P [A | b | B] ; then W_b += p  (v = P b + p) ----------------------------------------------------------
    par_mma_gemm<false, false, 4>(P, nx, nx1 + nu, nx, 1.0, Pc, lx, ABk, lx, W, lx);
    __syncthreads();
    RIC_TICK(2)
    for (int i = threadIdx.x; i < nx; i += blockDim.x) W[lx * nx + i] += Pc[lx * nx + i];
    __syncthreads();
    RIC_TICK(3)
    // [P | p] is dead: start streaming stage k-1 (its [Q | q] goes into that buffer)
    if (k > 0) prefetch(k - 1, 1 - set, Pc);
    // ---- [Q~ | q~] = [Q | q] + A'[W_A | v] (+reg), [S~ | r~] = [S | r] + B'[W_A | v], R~ = R + B'W_B (+reg) ----------------
    par_mma_gemm<true, true, 4>(P, nx, nx1, nx, 1.0, ABk, lx, W, lx, Pn, lx);
    if (nu > 0) {
      par_mma_gemm<true, true, 4>(P, nu, nx1, nx, 1.0, ABk + lx * nx1, lx, W, lx, Yk, lm);
      par_mma_gemm<true, true, 3>(P, nu, nu, nx, 1.0, ABk + lx * nx1, lx, W + lx * nx1, lx, Rk, lm);
    }
    __syncthreads();
    RIC_TICK(4)
    for (int i = threadIdx.x; i < nx; i += blockDim.x) Pn[i + i * lx] += v.reg;
    for (int i = threadIdx.x; i < nu; i += blockDim.x) Rk[i + i * lm] += v.reg;
    __syncthreads();
    RIC_TICK(5)
    if (nu > 0) {
      // ---- R~ = L L', Linv = L^-1: fused, register resident, warp 0 ---------------------------------------------------------------
      if (threadIdx.x < 32) {
        if (nm <= 8) warp_chol_inverse<8>(nu, Rk, lm, Linv, lm, &ok);
        else if (nm <= 16) warp_chol_inverse<16>(nu, Rk, lm, Linv, lm, &ok);
        else if (nm <= 24) warp_chol_inverse<24>(nu, Rk, lm, Linv, lm, &ok);
        else warp_chol_inverse<32>(nu, Rk, lm, Linv, lm, &ok);
      }
      __syncthreads();
      RIC_TICK(6)
      // ---- [Yl | yl] = L^-1 [S~ | r~] (into W) ---------------------------------------------------------------------------------
      double* Yl = W;
      double* Kout = W + L.kout;   // [K | k] keeps the dense leading dimension nm of its destination in HBM
      par_mma_gemm<false, false, 4>(P, nu, nx1, nu, 1.0, Linv, lm, Yk, lm, Yl, lm);
      __syncthreads();
    RIC_TICK(8)
      // ---- [P | p] = [Q~ | q~] - Yl'[Yl | yl] ; [K | k] = -L^-T [Yl | yl] ---------------------------------------------------
      par_mma_gemm<true, true, 4>(P, nx, nx1, nu, -1.0, Yl, lm, Yl, lm, Pn, lx);
      par_mma_gemm<true, false, 4>(P, nu, nx1, nu, -1.0, Linv, lm, Yl, lm, Kout, nm);
      __syncthreads();
    RIC_TICK(9)
      for (int t = threadIdx.x; t < nm * nx; t += blockDim.x) v.K[sk * nm * nx + t] = (t % nm < nu) ? Kout[t] : 0.0;
      for (int t = threadIdx.x; t < nu; t += blockDim.x) v.kff[sk * nm + t] = Kout[nm * nx + t];
    }
    // symmetrise the P part in place (pairs), rotate buffers
    for (int t = threadIdx.x; t < nx * nx; t += blockDim.x) {
      const int i = t % nx, j = t / nx;
      if (i > j) {
        const double m = 0.5 * (Pn[i + j * lx] + Pn[j + i * lx]);
        Pn[i + j * lx] = m;
        Pn[j + i * lx] = m;
      }
    }
    cur = 1 - cur;
    __syncthreads();
    RIC_TICK(10)
    if (v.keepP) {
      for (int i = threadIdx.x; i < nx * nx; i += blockDim.x) v.P[(iN1 + k) * nx * nx + i] = PQ[cur][(i % nx) + (i / nx) * lx];
      block_copy(nx, PQ[cur] + lx * nx, v.p + (iN1 + k) * nx);
    }
  }
  __syncthreads();
    RIC_TICK(11)
  // ---- forward substitution, double-buffered: x+ = [A | b | B] [x; 1; u] ----------------------------------------------------------------
  auto prefetchF = [&](int k, int set) {
    const size_t sk = iN + k;
    const int nu = v.nu ? v.nu[sk] : nm;
    async_copy(AB[set], v.A + sk * nx * nx, nx * nx);
    async_copy(AB[set] + nx * nx, v.b + sk * nx, nx);
    if (nu > 0) {
      async_copy(AB[set] + nx * nx1, v.Bm + sk * nx * nm, nx * nu);
      async_copy(Y[set], v.K + sk * nm * nx, nm * nx);
      async_copy(kb[set], v.kff + sk * nm, nu);
    }
    __pipeline_commit();
  };
  block_copy(nx, v.dx0 + static_cast<size_t>(inst) * nx, xv);
  prefetchF(0, 0);
  __syncthreads();
    RIC_TICK(12)
  block_copy(nx, xv, v.dx + iN1 * nx);
  for (int k = 0; k < N; ++k) {
    const int set = k & 1;
    const int nu = v.nu ? v.nu[iN + k] : nm;
    const size_t sk = iN + k;
    __pipeline_wait_prior(0);
    __syncthreads();
    RIC_TICK(13)
    if (k + 1 < N) prefetchF(k + 1, 1 - set);
    // du = K x + k : 8 lanes per row, shuffle-reduced
    {
      const int row = threadIdx.x >> 3, sub = threadIdx.x & 7;
      double s = 0.0;
      if (row < nu)
        for (int j = sub; j < nx; j += 8) s = fma(Y[set][row + j * nm], xv[j], s);
      s += __shfl_xor_sync(0xffffffffu, s, 4);
      s += __shfl_xor_sync(0xffffffffu, s, 2);
      s += __shfl_xor_sync(0xffffffffu, s, 1);
      if (sub == 0 && row < nm) {
        const double r = (row < nu) ? s + kb[set][row] : 0.0;
        uv[row] = r;
        v.du[sk * nm + row] = r;
      }
    }
    __syncthreads();
    RIC_TICK(14)
    // x+ = A x + b + B u : 4 lanes per row
    {
      const int row = threadIdx.x >> 2, sub = threadIdx.x & 3;
      const double* Ak = AB[set];
      double s = 0.0;
      if (row < nx) {
        for (int j = sub; j < nx; j += 4) s = fma(Ak[row + j * nx], xv[j], s);
        for (int j = sub; j < nu; j += 4) s = fma(Ak[nx * nx1 + row + j * nx], uv[j], s);
      }
      s += __shfl_xor_sync(0xffffffffu, s, 2);
      s += __shfl_xor_sync(0xffffffffu, s, 1);
      if (sub == 0 && row < nx) tv[row] = s + Ak[nx * nx + row];
    }
    __syncthreads();
    RIC_TICK(15)
    for (int i = threadIdx.x; i < nx; i += blockDim.x) {
      xv[i] = tv[i];
      v.dx[(iN1 + k + 1) * nx + i] = tv[i];
    }
  }
  __syncthreads();
    RIC_TICK(16)
  if (threadIdx.x == 0) {
    int bad = !ok;
    for (int i = 0; i < nx; ++i) bad |= !isfinite(xv[i]);
    v.status[inst] = bad;
  }
}

}  // namespace b200sqp
