// K2, low-latency variant for small batches: one thread-block CLUSTER of RC CTAs (RC SMs) per QP instance.
//
// The Riccati recursion is sequential in the stages, so a single instance keeps one SM busy and the others idle.  Here the
// stage's contractions are split by COLUMNS over the CTAs of a cluster and the small results every CTA needs in full are exchanged through
// distributed shared memory (plain stores to cluster.map_shared_rank pointers, then cluster.sync()):
//   W[:, J]  = P [A|b|B][:, J]                                   own columns J, P replicated
//   Q~[:, J] += A' W[:, J] ;  S~[:, J] += B' W[:, J] ;  R~[:, Jb] += B' W_B[:, Jb]
//   all-gather R~ and S~ (one exchange)                -> every CTA factorises R~ = L L', L^-1 and forms Yl = L^-1 S~ itself
//   P[:, J]  = Q~[:, J] - Yl' Yl[:, J] ;  [K|k][:, J] = -L^-T Yl[:, J] -> global
//   all-gather P                                                 (two cluster barriers per stage)
// Arithmetic per entry is identical to riccati_kernel (same DMMA tiles), so the results agree bit for bit up to the symmetrisation order.
// The forward substitution is run by rank 0 alone (matrix-vector work, latency bound either way).
#pragma once
#include <cooperative_groups.h>

#include "riccati.cuh"

namespace b200sqp {

namespace cg = cooperative_groups;
constexpr int RC = 4;  // CTAs per instance
__host__ __device__ inline size_t riccati_cluster_smem_doubles(int nx, int numax) {
  const RicLayout L = riccati_layout(nx, numax);
  return static_cast<size_t>(L.total) + L.rs + L.y;
}

// The dynamic shared memory one block of a generic Riccati kernel may take: the 227 KB a block can opt into on sm_90, less the kernels' 16
// bytes of static shared memory (the `ok` flag, padded).
constexpr size_t RIC_SMEM_BYTES_MAX = 227 * 1024 - 16;
// The sizes b200sqp_qp_create accepts.  nu_max <= 32: warp_chol_inverse keeps one column per lane, and the forward sweep has 8 lanes per row of
// u in a 256-thread block; nx <= 64: 4 lanes per row of x.  launch_riccati picks the one-CTA or the cluster kernel by the batch size alone, so
// the layouts of both must fit.
__host__ __device__ inline bool riccati_sizes_supported(int nx, int nm) {
  if (nx <= 0 || nx > 64 || nm <= 0 || nm > 32) return false;
  return riccati_smem_doubles(nx, nm) * sizeof(double) <= RIC_SMEM_BYTES_MAX &&
         riccati_cluster_smem_doubles(nx, nm) * sizeof(double) <= RIC_SMEM_BYTES_MAX;
}

__device__ __forceinline__ int sliceLo(int n, int r) { return (n * r) / RC; }

// copy columns [c0, c1) of a column-major (rows x *) block from the local buffer to the same place in every peer's buffer
__device__ __forceinline__ void gather_columns(cg::cluster_group& cluster, double* buf, int rows, int ld, int c0, int c1) {
  const unsigned me = cluster.block_rank();
  const int n = rows * (c1 - c0);
  for (unsigned r = 0; r < RC; ++r) {
    if (r == me) continue;
    double* remote = cluster.map_shared_rank(buf, r);
    for (int t = threadIdx.x; t < n; t += blockDim.x) {
      const int i = t % rows, j = c0 + t / rows;
      remote[i + j * ld] = buf[i + j * ld];
    }
  }
}

template <int NXT, int NMT>
__global__ void __cluster_dims__(RC, 1, 1) __launch_bounds__(256, 1) riccati_cluster_kernel(QpDeviceView v) {
  extern __shared__ double sm[];
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = static_cast<int>(cluster.block_rank());
  const int inst = blockIdx.x / RC;
  if (v.skip && v.skip[inst * v.skipStride]) return;   // uniform over the cluster (same instance), before any cluster barrier
  const int nx = NXT ? NXT : v.nx, nm = NMT ? NMT : v.numax, N = v.N, nx1 = nx + 1;
  const RicLayout L = riccati_layout(nx, nm);
  double* PQ[2] = {sm, sm + L.pq};
  double* AB[2] = {sm + 2 * L.pq, sm + 2 * L.pq + L.ab};
  double* W = AB[1] + L.ab;
  double* Y[2] = {W + L.w, W + L.w + L.y};
  double* Rs[2] = {Y[1] + L.y, Y[1] + L.y + L.rs};
  double* Linv = Rs[1] + L.rs;
  double* vec = Linv + L.linv;
  const int ex = even_up(nx), em = even_up(nm);
  double* xv = vec;
  double* tv = vec + ex;
  double* uv = vec + 2 * ex;
  double* kb[2] = {vec + 2 * ex + em, vec + 2 * ex + 2 * em};
  double* Rg = vec + L.vec;   // gathered R~ and [S~ | r~] (own buffers: Rs[] / Y[] are cp.async targets of the prefetch, remote stores could race)
  double* Yg = Rg + L.rs;
  __shared__ int ok;
  if (threadIdx.x == 0) ok = 1;
  const Par P{static_cast<int>(threadIdx.x), static_cast<int>(blockDim.x)};
  const int xc0 = sliceLo(nx1, rank), xc1 = sliceLo(nx1, rank + 1);   // own columns of the [x | 1] part

  const size_t iN = static_cast<size_t>(inst) * N, iN1 = static_cast<size_t>(inst) * (N + 1);
  int cur = 0;
  {
    const double* QN = v.Q + (iN1 + N) * nx * nx;
    for (int i = threadIdx.x; i < nx * nx; i += blockDim.x) PQ[cur][i] = QN[i] + ((i % nx) == (i / nx) ? v.reg : 0.0);
    block_copy(nx, v.q + (iN1 + N) * nx, PQ[cur] + nx * nx);
    __syncthreads();
    if (v.keepP && rank == 0) {
      block_copy(nx * nx, PQ[cur], v.P + (iN1 + N) * nx * nx);
      block_copy(nx, PQ[cur] + nx * nx, v.p + (iN1 + N) * nx);
    }
  }
  auto prefetch = [&](int k, int set, double* qdst) {
    const size_t sk = iN + k;
    const int nu = v.nu ? v.nu[sk] : nm;
    async_copy(AB[set], v.A + sk * nx * nx, nx * nx);
    async_copy(AB[set] + nx * nx, v.b + sk * nx, nx);
    if (nu > 0) {
      async_copy(AB[set] + nx * nx1, v.Bm + sk * nx * nm, nx * nu);
      async_copy(Y[set], v.S + sk * nm * nx, nm * nx);
      async_copy(Y[set] + nm * nx, v.r + sk * nm, nu);
      async_copy(Rs[set], v.R + sk * nm * nm, nm * nm);
    }
    async_copy(qdst, v.Q + (iN1 + k) * nx * nx, nx * nx);
    async_copy(qdst + nx * nx, v.q + (iN1 + k) * nx, nx);
    __pipeline_commit();
  };
  prefetch(N - 1, 0, PQ[1 - cur]);
  cluster.sync();   // every CTA of the cluster is resident before the first remote store

  for (int k = N - 1; k >= 0; --k) {
    const int set = (N - 1 - k) & 1;
    const int nu = v.nu ? v.nu[iN + k] : nm;
    const int bc0 = sliceLo(nu, rank), bc1 = sliceLo(nu, rank + 1);   // own columns of the B part
    const size_t sk = iN + k;
    double* Pc = PQ[cur];
    double* Pn = PQ[1 - cur];
    double* ABk = AB[set];
    double* Yk = Y[set];
    double* Rk = Rs[set];
    __pipeline_wait_prior(0);
    __syncthreads();
    // ---- W[:, J] = P [A | b | B][:, J] ; v = P b + p on the owner of column nx ------------------------------------------------------------
    par_mma_gemm<false, false, 2>(P, nx, xc1 - xc0, nx, 1.0, Pc, nx, ABk + nx * xc0, nx, W + nx * xc0, nx);
    if (bc1 > bc0) par_mma_gemm<false, false, 2>(rot(P, 128), nx, bc1 - bc0, nx, 1.0, Pc, nx, ABk + nx * (nx1 + bc0), nx, W + nx * (nx1 + bc0), nx);
    __syncthreads();
    if (xc0 <= nx && nx < xc1)
      for (int i = threadIdx.x; i < nx; i += blockDim.x) W[nx * nx + i] += Pc[nx * nx + i];
    __syncthreads();
    if (k > 0) prefetch(k - 1, 1 - set, Pc);
    // ---- Q~[:, J] += A' W[:, J] ; S~[:, J] += B' W[:, J] ; R~[:, Jb] += B' W_B[:, Jb] ---------------------------------------------------
    par_mma_gemm<true, true, 2>(P, nx, xc1 - xc0, nx, 1.0, ABk, nx, W + nx * xc0, nx, Pn + nx * xc0, nx);
    if (nu > 0) {
      par_mma_gemm<true, true, 2>(rot(P, 128), nu, xc1 - xc0, nx, 1.0, ABk + nx * nx1, nx, W + nx * xc0, nx, Yk + nm * xc0, nm);
      if (bc1 > bc0) par_mma_gemm<true, true, 1>(rot(P, 64), nu, bc1 - bc0, nx, 1.0, ABk + nx * nx1, nx, W + nx * (nx1 + bc0), nx, Rk + nm * bc0, nm);
    }
    __syncthreads();
    for (int i = xc0 + threadIdx.x; i < xc1 && i < nx; i += blockDim.x) Pn[i + i * nx] += v.reg;
    for (int i = bc0 + threadIdx.x; i < bc1; i += blockDim.x) Rk[i + i * nm] += v.reg;
    __syncthreads();
    double* Yl = W;
    double* Kout = W + L.kout;
    if (nu > 0) {
      // ---- all-gather R~ and [S~ | r~] in one exchange, factorise and form Yl = L^-1 [S~ | r~] everywhere (identical arithmetic) ---------------
      for (int t = threadIdx.x; t < nm * (bc1 - bc0); t += blockDim.x) Rg[(t % nm) + nm * (bc0 + t / nm)] = Rk[(t % nm) + nm * (bc0 + t / nm)];
      for (int t = threadIdx.x; t < nm * (xc1 - xc0); t += blockDim.x) Yg[(t % nm) + nm * (xc0 + t / nm)] = Yk[(t % nm) + nm * (xc0 + t / nm)];
      __syncthreads();
      if (bc1 > bc0) gather_columns(cluster, Rg, nm, nm, bc0, bc1);
      gather_columns(cluster, Yg, nu, nm, xc0, xc1);
      cluster.sync();
      if (threadIdx.x < 32) {
        if (nm <= 8) warp_chol_inverse<8>(nu, Rg, nm, Linv, nm, &ok);
        else if (nm <= 16) warp_chol_inverse<16>(nu, Rg, nm, Linv, nm, &ok);
        else if (nm <= 24) warp_chol_inverse<24>(nu, Rg, nm, Linv, nm, &ok);
        else warp_chol_inverse<32>(nu, Rg, nm, Linv, nm, &ok);
      }
      __syncthreads();
      par_mma_gemm<false, false, 4>(P, nu, nx1, nu, 1.0, Linv, nm, Yg, nm, Yl, nm);
      __syncthreads();
      // ---- P[:, J] = Q~[:, J] - Yl' Yl[:, J] ; [K | k][:, J] = -L^-T Yl[:, J] ------------------------------------------------------------------
      par_mma_gemm<true, true, 2>(P, nx, xc1 - xc0, nu, -1.0, Yl, nm, Yl + nm * xc0, nm, Pn + nx * xc0, nx);
      par_mma_gemm<true, false, 2>(rot(P, 128), nu, xc1 - xc0, nu, -1.0, Linv, nm, Yl + nm * xc0, nm, Kout + nm * xc0, nm);
      __syncthreads();
      for (int t = threadIdx.x; t < nm * (xc1 - xc0); t += blockDim.x) {
        const int i = t % nm, c = xc0 + t / nm;
        const double val = (i < nu) ? Kout[i + nm * c] : 0.0;
        if (c < nx) v.K[sk * nm * nx + i + nm * c] = val;
        else if (i < nu) v.kff[sk * nm + i] = val;
      }
    } else {
      // nu == 0 (event node): no exchange is needed before the P gather, but a peer must not store into this CTA's Pn while the prefetch of
      // [Q | q] into it may still be in flight here (it is only known complete after this CTA's wait at the top of the stage)
      cluster.sync();
      for (int t = threadIdx.x; t < nm * (xc1 - xc0); t += blockDim.x) {
        const int i = t % nm, c = xc0 + t / nm;
        if (c < nx) v.K[sk * nm * nx + i + nm * c] = 0.0;
      }
    }
    // ---- all-gather P, symmetrise (every CTA, identical), rotate --------------------------------------------------------------------------------
    gather_columns(cluster, Pn, nx, nx, xc0, xc1);
    cluster.sync();
    for (int t = threadIdx.x; t < nx * nx; t += blockDim.x) {
      const int i = t % nx, j = t / nx;
      if (i > j) {
        const double m = 0.5 * (Pn[i + j * nx] + Pn[j + i * nx]);
        Pn[i + j * nx] = m;
        Pn[j + i * nx] = m;
      }
    }
    cur = 1 - cur;
    __syncthreads();
    if (v.keepP && rank == 0) {
      block_copy(nx * nx, PQ[cur], v.P + (iN1 + k) * nx * nx);
      block_copy(nx, PQ[cur] + nx * nx, v.p + (iN1 + k) * nx);
    }
    // the next stage's gathers write into the buffer peers are still symmetrising only after the next stage's first cluster barrier... no:
    // they write into Rk / Yl / Pn of the NEXT stage, none of which is PQ[cur]; the P gather of the next stage targets PQ[1 - cur], which every
    // CTA finished reading (as Pc) before it reached that stage's first cluster.sync()
  }
  cluster.sync();
  if (rank != 0) return;
  // ---- forward substitution by rank 0 (as in riccati_kernel) -----------------------------------------------------------------------------
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
  __threadfence();
  block_copy(nx, v.dx0 + static_cast<size_t>(inst) * nx, xv);
  prefetchF(0, 0);
  __syncthreads();
  block_copy(nx, xv, v.dx + iN1 * nx);
  for (int k = 0; k < N; ++k) {
    const int set = k & 1;
    const int nu = v.nu ? v.nu[iN + k] : nm;
    const size_t sk = iN + k;
    __pipeline_wait_prior(0);
    __syncthreads();
    if (k + 1 < N) prefetchF(k + 1, 1 - set);
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
    for (int i = threadIdx.x; i < nx; i += blockDim.x) {
      xv[i] = tv[i];
      v.dx[(iN1 + k + 1) * nx + i] = tv[i];
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int bad = !ok;
    for (int i = 0; i < nx; ++i) bad |= !isfinite(xv[i]);
    v.status[inst] = bad;
  }
}

}  // namespace b200sqp
