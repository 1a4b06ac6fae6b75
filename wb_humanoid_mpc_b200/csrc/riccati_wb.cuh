// K2 for the whole-body sizes (nx = 58, nu_max = 23), large batches: the Riccati recursion of HpipmInterface::solve
// (lib/ocs2_ros2/ocs2_sqp/hpipm_catkin/src/HpipmInterface.cpp:166-455) as TWO kernels.
//
//   riccati_bwd_kernel  backward factorisation, one persistent CTA of two independent LANES, each running one instance (112 KB of shared
//                       memory per lane, one CTA per SM).  The sweep is bound by latency (the factorisation chain, barriers, fragment loads), so
//                       two instances side by side on one SM overlap: a batch of up to twice the SM count runs in one wave.  Batches no larger than
//                       the SM count run one lane per CTA, so that no SM idles.  A lane is five warps: four GEMM warps run the fp64 tensor-path
//                       contractions (DMMA m8n8k4) and one helper warp
//                       (a) streams the next stage's [A | b | B] with cp.async.bulk + an mbarrier once this stage's last read of it is done
//                       (it lands densely, leading dimension 58, exactly as it lies in HBM), prefetches Q, q, S, r of the next stage into L2 and
//                       R as 8-byte cp.async (its HBM address is only 8-byte aligned), (b) factorises R~ = L L' and inverts L, register resident,
//                       WHILE the GEMM warps form Q~ and S~ (the factorisation only needs R~, which is formed first and handed over through a
//                       named barrier), (c) writes the cost-to-go out when it is kept.  Q, q, S, r are never staged in shared memory: they are
//                       the addends of the epilogues that form Q~ and [S~ | r~], read from global memory.
//                       Per stage:  W = P [A | b | B], W_b += p           (P is kept as its lower triangle: the operand loads pick (max, min))
//                                   R~ = R + B'W_B  ->  helper: L, L^-1   ||  Q~ = Q + A'W_A (lower tiles only, over the dead P),
//                                                                             [S~ | r~] = [S | r] + B'[W_A | v] (over the dead W_B)
//                                   Yl = L^-1 [S~ | r~]
//                                   [P | p] = [Q~ | q~] - Yl'Yl (lower tiles only), [K | k] = -L^-T Yl
//   riccati_fwd_kernel  forward substitution, one small CTA per instance (two resident per SM, so the whole batch is in flight and the
//                       second, partial wave of the backward kernel does not serialise it): du = K dx + k, dx+ = A dx + B du + b with the
//                       stage operands double-buffered in shared memory by cp.async.bulk + mbarrier.
//
// Same arithmetic as riccati_kernel<58, 23> up to the order of two additions (reg_prim is added to the diagonal of P after the
// update instead of before; symmetric entries are computed once instead of twice and averaged).
#pragma once
#include <cuda_pipeline.h>

#include "riccati.cuh"

namespace b200sqp {
namespace ricwb {

#ifdef B200SQP_PHASE_CLOCK
#define WB_TICK(slot, who)                                               \
  if (threadIdx.x == (who) && blockIdx.x == 0) {                         \
    const long long now_ = clock64();                                    \
    g_ricClk[slot][0] = __LINE__;                                        \
    g_ricClk[slot][1] += now_ - wbT_;                                    \
    wbT_ = now_;                                                         \
  }
#define WB_CLOCK_BEGIN()                                                 \
  long long wbT_ = clock64();                                            \
  if (threadIdx.x == 0 && blockIdx.x == 0)                               \
    for (int i_ = 0; i_ < 32; ++i_) g_ricClk[i_][0] = g_ricClk[i_][1] = 0;
#else
#define WB_TICK(slot, who)
#define WB_CLOCK_BEGIN()
#endif

constexpr int NXR = 58, NX1R = 59, NMR = 23;
constexpr int LWR = 60, LMR = 28;                 // leading dimensions of the operands the kernel produces itself: = 4 (mod 8), conflict-free DMMA fragment loads
constexpr int LANES = 2, LANE_GEMM_WARPS = 4;
constexpr int LANE_THREADS = 32 * (LANE_GEMM_WARPS + 1), BWD_THREADS = LANES * LANE_THREADS;
constexpr int PQ_D = NXR * NX1R + 2;              // [P | p], dense (ld 58), lower triangle of P valid; [Q~ | q~] once W is complete
constexpr int AB_D = NXR * (NX1R + NMR);          // [A | b | B], dense (ld 58): a 58 x 82 matrix
constexpr int W_D = LWR * (NX1R + NMR);           // W (ld 60); later Yl (ld 28), [K | k] (ld 23) and [S~ | r~] (ld 23)
constexpr int R_D = LMR * NMR;                    // 23 x 23 at ld 28
constexpr int YL_D = LMR * NX1R;
constexpr int KOUT_OFF = YL_D;                    // [K | k] behind Yl inside the W region
constexpr int Y_OFF = LWR * NX1R;                 // [S~ | r~] in the columns of W_B, dead once R~ is formed
// the shared memory of one lane (doubles); the two lanes' maps follow each other, then one mbarrier per lane
constexpr int PQ_OFF = 0;
constexpr int AB_OFF = PQ_OFF + PQ_D;
constexpr int W_OFF = AB_OFF + AB_D;
constexpr int RT_OFF = W_OFF + W_D;               // R~, overwritten by L^-1 (the helper warp holds R~ in registers by then)
constexpr int RIN_OFF = RT_OFF + R_D;             // R, landing buffer of the cp.async (read by the epilogue of R~)
constexpr int LANE_D = RIN_OFF + R_D;
constexpr int BWD_SMEM_D = LANES * LANE_D + LANES;
constexpr size_t BWD_SMEM_BYTES = static_cast<size_t>(BWD_SMEM_D) * 8;
constexpr size_t BWD_STATIC_SMEM_BYTES = 16;   // the lanes' `ok` flags, as ptxas allots them
static_assert(PQ_D % 2 == 0 && AB_D % 2 == 0 && W_D % 2 == 0 && R_D % 2 == 0, "bulk-copy targets and lane bases start on 16-byte boundaries");
static_assert(YL_D <= KOUT_OFF && KOUT_OFF + NMR * NX1R <= Y_OFF, "Yl and [K | k] stay below the W_B columns that hold [S~ | r~]");
static_assert(Y_OFF + NMR * NX1R <= W_D, "[S~ | r~] (ld 23) fits the W_B columns");
static_assert(BWD_SMEM_BYTES + BWD_STATIC_SMEM_BYTES <= 227 * 1024, "two lanes fit a block's opt-in shared memory on sm_90");

// ---- mbarrier / bulk-copy primitives (sm_90+; SASS: SYNCS.*, UBLKCP) -------------------------------------------------------------------
__device__ __forceinline__ unsigned smem_u32(const void* p) { return static_cast<unsigned>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// global -> shared bulk copy (bytes: a multiple of 16; both addresses 16-byte aligned), completion counted on `bar`
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src),
               "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// global -> L2 prefetch (bytes: a multiple of 16; address 16-byte aligned), and of the one cache line that holds address p
__device__ __forceinline__ void bulk_prefetch_l2(const void* src, unsigned bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
// generic-proxy accesses of this thread before, async-proxy accesses after (a buffer read with ld.shared is about to be refilled by a bulk copy)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void named_arrive(int id, int count) { asm volatile("barrier.cta.arrive %0, %1;" ::"r"(id), "r"(count) : "memory"); }
__device__ __forceinline__ void named_sync(int id, int count) { asm volatile("barrier.cta.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }

// ---- one DMMA work item: an 8-row strip x NG column tiles -------------------------------------------------------------------------------------
// C(tile tm, tiles tn[0..NG)) = (ACC ? C : 0) + alpha * op(A) * B on column-major operands; op(A) = A (M x K) or A' (A stored K x M).
// KC > 0: contraction length known at compile time (the k loop unrolls completely and the scheduler hoists the fragment loads).
// NG is a compile-time count (mma_item dispatches on the number of tiles) so that the unrolled DMMA stream carries no per-tile branches.
// SYM_A (only with !TRANS_A, M = K): A is symmetric and only its lower triangle is valid: element (m, k) is read from (max, min).
// vadd != nullptr: without ACC, column vcol of the result additionally gets the vector vadd (W_b = P b + p without a separate pass); with ACC,
// vadd is the addend of column vcol in place of Cin's column (C-in [Q | q] from Q and q, which lie apart in HBM).
// ACC: C = alpha * op(A) * B + Cin, Cin = C unless given (leading dimension ldcin).  The addends are loaded before the contraction, so that the
// latency of a global Cin hides behind it.
// PERM_A / PERM_B: the operand has leading dimension 58 with the contraction index running fastest (A' stored K x M, or B): lane group fr then
// takes row / column perm8(fr) = (0, 2, 4, 6, 1, 3, 5, 7)[fr] of the tile instead of fr.  A half-warp's fragment load touches the doubles
// {k + 58 n : k = 0..3, n = four rows / columns}: with n = 0, 1, 2, 3 the bank offsets 10 n (mod 16) = 0, 10, 4, 14 make the 4-wide runs of
// n = 0 and n = 3 collide (a two-way conflict on every load); with n = 0, 2, 4, 6 (and 1, 3, 5, 7 in the other half-warp) they are 0, 4, 8, 12:
// conflict free.  Which tile row a lane group feeds is arbitrary as long as the result is stored accordingly, which the epilogue does.
__device__ __forceinline__ int perm8(int j) { return j < 4 ? 2 * j : 2 * (j - 4) + 1; }
template <bool TRANS_A, bool ACC, int NG, int KC, bool SYM_A, bool PERM_A, bool PERM_B>
__device__ __forceinline__ void mma_item_ng(int lane, int M, int N, int Krt, double alpha, const double* __restrict__ A, int lda, int tm,
                                            const double* __restrict__ B, int ldb, const int* tn, double* __restrict__ C, int ldc,
                                            const double* __restrict__ vadd, int vcol, const double* __restrict__ Cin, int ldcin) {
  const int K = KC ? KC : Krt;
  const int fr = lane >> 2, fk = lane & 3;
  const int Kmain = K & ~3;
  const int ar = (tm << 3) + (PERM_A ? perm8(fr) : fr);
  const bool arok = ar < M;
  const int arc = arok ? ar : 0;
  const double* Ap = TRANS_A ? A + fk + arc * lda : A + arc + fk * lda;
  const double* ApU = A + fk + arc * lda;   // SYM_A: the mirrored element (k, m)
  const int astep = TRANS_A ? 4 : 4 * lda;
  const int frB = PERM_B ? perm8(fr) : fr;
  const int cj0 = PERM_B ? perm8(2 * fk) : 2 * fk, cj1 = PERM_B ? perm8(2 * fk + 1) : 2 * fk + 1;   // tile columns of this lane's two results
  const double* Bp[NG];
  bool bok[NG];
  double c0[NG], c1[NG];
#pragma unroll
  for (int g = 0; g < NG; ++g) {
    const int bn = (tn[g] << 3) + frB;
    bok[g] = bn < N;
    Bp[g] = B + fk + (bok[g] ? bn : 0) * ldb;
    c0[g] = c1[g] = 0.0;
  }
  double in0[NG], in1[NG];
  if (ACC) {
    const double* ci = Cin ? Cin : C;
    const int ldi = Cin ? ldcin : ldc;
#pragma unroll
    for (int g = 0; g < NG; ++g) {
      const int cn0 = (tn[g] << 3) + cj0, cn1 = (tn[g] << 3) + cj1;
      in0[g] = (arok && cn0 < N) ? ((vadd && cn0 == vcol) ? vadd[ar] : ci[ar + cn0 * ldi]) : 0.0;
      in1[g] = (arok && cn1 < N) ? ((vadd && cn1 == vcol) ? vadd[ar] : ci[ar + cn1 * ldi]) : 0.0;
    }
  }
#pragma unroll
  for (int k0 = 0; k0 < Kmain; k0 += 4) {
    double a;
    if (SYM_A) {
      const double* ps = (k0 + fk <= arc) ? Ap : ApU + k0;
      a = arok ? *ps : 0.0;
    } else {
      a = arok ? *Ap : 0.0;
    }
    Ap += astep;
#pragma unroll
    for (int g = 0; g < NG; ++g) {
      const double b = bok[g] ? Bp[g][k0] : 0.0;
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0[g]), "+d"(c1[g]) : "d"(a), "d"(b));
    }
  }
  if (Kmain < K) {
    const bool kok = Kmain + fk < K;
    double a = 0.0;
    if (arok && kok) {
      if (SYM_A) a = (Kmain + fk <= arc) ? *Ap : ApU[Kmain];
      else a = *Ap;
    }
#pragma unroll
    for (int g = 0; g < NG; ++g) {
      const double b = (bok[g] && kok) ? Bp[g][Kmain] : 0.0;
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0[g]), "+d"(c1[g]) : "d"(a), "d"(b));
    }
  }
  if (arok) {
#pragma unroll
    for (int g = 0; g < NG; ++g) {
      const int cn0 = (tn[g] << 3) + cj0, cn1 = (tn[g] << 3) + cj1;
      if (cn0 < N) {
        double r = ACC ? fma(alpha, c0[g], in0[g]) : alpha * c0[g];
        if (!ACC && vadd && cn0 == vcol) r += vadd[ar];
        C[ar + cn0 * ldc] = r;
      }
      if (cn1 < N) {
        double r = ACC ? fma(alpha, c1[g], in1[g]) : alpha * c1[g];
        if (!ACC && vadd && cn1 == vcol) r += vadd[ar];
        C[ar + cn1 * ldc] = r;
      }
    }
  }
}
template <bool TRANS_A, bool ACC, int NG, int KC, bool SYM_A = false, bool PERM_A = false, bool PERM_B = false>
__device__ __forceinline__ void mma_item(int lane, int M, int N, int Krt, double alpha, const double* __restrict__ A, int lda, int tm,
                                         const double* __restrict__ B, int ldb, const int (&tn)[NG], int cnt, double* __restrict__ C, int ldc,
                                         const double* __restrict__ vadd = nullptr, int vcol = -1, const double* __restrict__ Cin = nullptr,
                                         int ldcin = 0) {
  // (warp-uniform dispatch; NG bounds the tile count)
  if (NG >= 4 && cnt == 4)
    mma_item_ng<TRANS_A, ACC, (NG >= 4 ? 4 : NG), KC, SYM_A, PERM_A, PERM_B>(lane, M, N, Krt, alpha, A, lda, tm, B, ldb, tn, C, ldc, vadd, vcol, Cin, ldcin);
  else if (NG >= 3 && cnt == 3)
    mma_item_ng<TRANS_A, ACC, (NG >= 3 ? 3 : NG), KC, SYM_A, PERM_A, PERM_B>(lane, M, N, Krt, alpha, A, lda, tm, B, ldb, tn, C, ldc, vadd, vcol, Cin, ldcin);
  else if (NG >= 2 && cnt == 2)
    mma_item_ng<TRANS_A, ACC, (NG >= 2 ? 2 : NG), KC, SYM_A, PERM_A, PERM_B>(lane, M, N, Krt, alpha, A, lda, tm, B, ldb, tn, C, ldc, vadd, vcol, Cin, ldcin);
  else if (cnt == 1) mma_item_ng<TRANS_A, ACC, 1, KC, SYM_A, PERM_A, PERM_B>(lane, M, N, Krt, alpha, A, lda, tm, B, ldb, tn, C, ldc, vadd, vcol, Cin, ldcin);
}

// Work items of a symmetric 58 x 59 update (the [P | p] shape): row strip m needs the column tiles 0..m of the lower triangle plus tile 7,
// which holds the vector column 58 (the entries of the upper triangle inside those tiles come for free and are never read).
// 13 items, 43 of 64 tiles; items 13..18 of the schedules below are the six 4-tile items of a 23 x 59 product (strip it/2, tile group it%2).
struct SymItem {
  unsigned char m, cnt, n[4];
};
__constant__ SymItem kSymItems[13] = {
    {7, 4, {0, 1, 2, 3}}, {7, 4, {4, 5, 6, 7}}, {6, 4, {0, 1, 2, 3}}, {6, 4, {4, 5, 6, 7}}, {5, 4, {0, 1, 2, 3}}, {4, 4, {0, 1, 2, 3}}, {3, 4, {0, 1, 2, 3}},
    {2, 4, {0, 1, 2, 7}}, {5, 3, {4, 5, 7, 0}},   {1, 3, {0, 1, 7, 0}},   {4, 2, {4, 7, 0, 0}},   {0, 2, {0, 7, 0, 0}},   {3, 1, {7, 0, 0, 0}}};
// Item tables of a lane's four GEMM warps, by rank: rank 0 is the warp that shares its scheduler (and its fp64 / shuffle issue slots) with the
// lane's helper warp, ranks 1-3 are the other three, which form R~ first (one 3-tile row strip each) and hand it to the helper.
// P1b: the rest of W, column tiles 0..6 of the eight row strips (item = 2 * row strip + {0: column tiles 0-3, 1: column tiles 4-6}).
__constant__ signed char kP1bItems[LANE_GEMM_WARPS][4] = {{0, 2, 4, 6}, {8, 1, 3, 5}, {10, 7, 9, 11}, {12, 14, 13, 15}};
// P2: Q~ (the 13 symmetric items) and [S~ | r~] (items 13..18), 17 tiles for each R~ warp and 16 for rank 0; -1 ends
__constant__ signed char kP2Sched[LANE_GEMM_WARPS][5] = {{0, 1, 2, 3, -1}, {4, 5, 6, 7, 12}, {13, 14, 15, 8, 10}, {16, 17, 18, 9, 11}};
// stages without inputs (event nodes): only the 13 symmetric items
__constant__ signed char kP2SchedNoInput[LANE_GEMM_WARPS][4] = {{0, 1, 12, -1}, {2, 3, 8, -1}, {4, 5, 9, -1}, {6, 7, 10, 11}};

template <int NMAX>
__device__ __forceinline__ void warp_chol_inverse_reg(int n, const double* A, int lda, double reg, double* Linv, int ldl, int* ok);

// pairOff > 0: lane 1 of CTA c runs instance c + pairOff (the launch pairs instance c with c + ceil(B / 2)); pairOff = 0: lane 1 is idle.
__global__ void __launch_bounds__(BWD_THREADS, 1) riccati_bwd_kernel(QpDeviceView v, int pairOff) {
  extern __shared__ double sm[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // warps 4 ln .. 4 ln + 3: the GEMM warps of lane ln; warp 8 + ln: its helper warp, on scheduler ln, which only one of its GEMM warps shares
  const bool gemmWarp = warp < LANES * LANE_GEMM_WARPS;
  const int ln = gemmWarp ? warp / LANE_GEMM_WARPS : warp - LANES * LANE_GEMM_WARPS;
  const int lw = warp % LANE_GEMM_WARPS;                          // (GEMM warps) the warp's index in its lane = its scheduler
  const int rank = lw == ln ? 0 : 1 + lw - (lw > ln);             // (GEMM warps) row of the item tables; ranks 1-3 form R~
  const int lt = gemmWarp ? tid - 32 * LANE_GEMM_WARPS * ln : 32 * LANE_GEMM_WARPS + lane;   // thread index in the lane
  if (ln == 1 && pairOff == 0) return;
  const int inst = blockIdx.x + ln * pairOff;
  if (inst >= v.B || (v.skip && v.skip[inst * v.skipStride])) return;
  // every barrier below is the lane's own, so that a lane that returned above, or runs stages of another kind, never stalls the other one
  const int barLane = 1 + 3 * ln, barRt = barLane + 1, barW = barLane + 2;
  const auto laneSync = [&]() { named_sync(barLane, LANE_THREADS); };
  const int N = v.N;
  double* const P = sm + ln * LANE_D + PQ_OFF;
  double* const AB = sm + ln * LANE_D + AB_OFF;
  double* const W = sm + ln * LANE_D + W_OFF;
  double* const Rt = sm + ln * LANE_D + RT_OFF;
  double* const Rin = sm + ln * LANE_D + RIN_OFF;
  const double* const Bk = AB + NXR * NX1R;
  unsigned long long* bar = reinterpret_cast<unsigned long long*>(sm + LANES * LANE_D) + ln;   // [A | b | B] of the next stage
  __shared__ int okLane[LANES];
  int* const ok = &okLane[ln];
  const size_t iN = static_cast<size_t>(inst) * N, iN1 = static_cast<size_t>(inst) * (N + 1);

  if (lt == 0) {
    *ok = 1;
    mbar_init(bar, 1);
    mbar_fence_init();
  }
  // terminal stage: [P_N | p_N] = [Q_N + reg I | q_N]
  {
    const double* QN = v.Q + (iN1 + N) * NXR * NXR;
    for (int i = lt; i < NXR * NXR; i += LANE_THREADS) P[i] = QN[i] + ((i % NXR == i / NXR) ? v.reg : 0.0);
    for (int i = lt; i < NXR; i += LANE_THREADS) P[NXR * NXR + i] = v.q[(iN1 + N) * NXR + i];
  }
  laneSync();
  // the cost-to-go of stage kk, symmetric from its lower triangle
  auto storeP = [&](int kk, int t0, int nt) {
    for (int i = t0; i < NXR * NXR; i += nt) {
      const int r = i % NXR, c = i / NXR;
      v.P[(iN1 + kk) * NXR * NXR + i] = r >= c ? P[r + c * NXR] : P[c + r * NXR];
    }
    for (int i = t0; i < NXR; i += nt) v.p[(iN1 + kk) * NXR + i] = P[NXR * NXR + i];
  };
  if (v.keepP) storeP(N, lt, LANE_THREADS);
  // Stage record k, issued by the helper warp only, in three parts: the bulk copies of [A | b | B] (one lane) once the buffer is free, after
  // the last read of the previous stage's; the L2 prefetch of the epilogue addends Q, q, S, r; the 8-byte cp.async of R (whose HBM address is
  // only 8-byte aligned) after the factorisation, which is the last read of the previous R.
  auto prefetchBulk = [&](int k) {
    const size_t sk = iN + k;
    const int nu = v.nu ? v.nu[sk] : NMR;
    if (lane == 0) {
      fence_proxy_async();
      mbar_expect_tx(bar, static_cast<unsigned>((NXR * NX1R + NXR * nu) * 8));
      bulk_g2s(AB, v.A + sk * NXR * NXR, NXR * NXR * 8, bar);
      bulk_g2s(AB + NXR * NXR, v.b + sk * NXR, NXR * 8, bar);
      if (nu > 0) bulk_g2s(AB + NXR * NX1R, v.Bm + sk * NXR * NMR, static_cast<unsigned>(NXR * nu * 8), bar);
    }
  };
  auto prefetchAddends = [&](int k) {
    const size_t sk = iN + k;
    const int nu = v.nu ? v.nu[sk] : NMR;
    if (lane == 0) {
      bulk_prefetch_l2(v.Q + (iN1 + k) * NXR * NXR, NXR * NXR * 8);
      bulk_prefetch_l2(v.q + (iN1 + k) * NXR, NXR * 8);
      if (nu > 0) bulk_prefetch_l2(v.S + sk * NMR * NXR, NMR * NXR * 8);
    } else if (lane < 3 && nu > 0) {
      prefetch_l2(v.r + sk * NMR + (lane == 1 ? 0 : NMR - 1));   // r: 184 bytes, on at most two lines
    }
  };
  auto prefetchR = [&](int k) {
    const size_t sk = iN + k;
    const int nu = v.nu ? v.nu[sk] : NMR;
    if (nu > 0) {
      const double* Rg = v.R + sk * NMR * NMR;
      int c = 0, r = lane;   // (r, c) of element i = lane + 32 j, without divisions
      for (int i = lane; i < NMR * NMR; i += 32) {
        while (r >= NMR) {
          r -= NMR;
          ++c;
        }
        __pipeline_memcpy_async(Rin + r + c * LMR, Rg + i, 8);
        r += 32;
      }
    }
    __pipeline_commit();
  };
  unsigned parity = 0;
  if (!gemmWarp) {
    prefetchBulk(N - 1);
    prefetchAddends(N - 1);
    prefetchR(N - 1);
  }
  WB_CLOCK_BEGIN()

  for (int k = N - 1; k >= 0; --k) {
    const size_t sk = iN + k;
    const int nu = v.nu ? v.nu[sk] : NMR;
    const int tilesN = (NX1R + nu + 7) >> 3;
    // ---- [A | b | B] and R of this stage have landed ------------------------------------------------------------------------------------------
    if (!gemmWarp) __pipeline_wait_prior(0);
    mbar_wait(bar, parity);
    parity ^= 1;
    laneSync();
    WB_TICK(1, 0)
    WB_TICK(20, 256)
    // ---- P1a: the columns of W = P [A | b | B] that R~ needs first: column tiles 7.. = [A_56 A_57 | b | B] (column b additionally gets p) --------
    if (gemmWarp) {
      const int tn[4] = {7, 8, 9, 10};
      for (int strip = lw; strip < 8; strip += LANE_GEMM_WARPS)
        mma_item<false, false, 4, NXR, true, false, true>(lane, NXR, NX1R + nu, 0, 1.0, P, NXR, strip, AB, NXR, tn, tilesN - 7, W, LWR, P + NXR * NXR, NXR);
    } else if (v.keepP && k < N - 1) {
      storeP(k + 1, lane, 32);   // (the cost-to-go of stage k+1 is complete and read-only until Q~ replaces it in P2)
    }
    laneSync();
    WB_TICK(2, 0)
    WB_TICK(21, 256)
    // ---- P1b / P2: helper warp: factorise R~ as soon as three GEMM warps hand it over -- the factorisation (latency bound, one warp) runs
    //      WHILE the GEMM warps finish W (column tiles 0..6), and form Q~ (lower tiles) and [S~ | r~]
    if (!gemmWarp) {
      if (k > 0) prefetchAddends(k - 1);
      WB_TICK(22, 256)
      if (nu > 0) {
        named_sync(barRt, 128);
        WB_TICK(23, 256)
        warp_chol_inverse_reg<24>(nu, Rt, LMR, v.reg, Rt, LMR, ok);
        WB_TICK(24, 256)
      }
      if (k > 0) prefetchR(k - 1);
      WB_TICK(27, 256)
    } else {
      if (nu > 0 && rank > 0) {   // R~ = R + B'W_B
        const int tn[3] = {0, 1, 2};
        mma_item<true, true, 3, NXR, false, true, false>(lane, nu, nu, 0, 1.0, Bk, NXR, rank - 1, W + LWR * NX1R, LWR, tn, 3, Rt, LMR, nullptr, -1, Rin,
                                                         LMR);
        __threadfence_block();
        named_arrive(barRt, 128);
      }
      for (int j = 0; j < 4; ++j) {
        const int it = kP1bItems[rank][j];
        const int strip = it >> 1;
        if (it & 1) {
          const int tb[4] = {4, 5, 6, 0};
          mma_item<false, false, 4, NXR, true, false, true>(lane, NXR, NX1R + nu, 0, 1.0, P, NXR, strip, AB, NXR, tb, 3, W, LWR);
        } else {
          const int ta[4] = {0, 1, 2, 3};
          mma_item<false, false, 4, NXR, true, false, true>(lane, NXR, NX1R + nu, 0, 1.0, P, NXR, strip, AB, NXR, ta, 4, W, LWR);
        }
      }
      named_sync(barW, 32 * LANE_GEMM_WARPS);   // W is complete: P and W_B are dead
      WB_TICK(7, 32)
      const double* Qg = v.Q + (iN1 + k) * NXR * NXR;
      const double* qg = v.q + (iN1 + k) * NXR;
      const double* Sg = v.S + sk * NMR * NXR;
      const double* rg = v.r + sk * NMR;
      const signed char* sched = nu > 0 ? kP2Sched[rank] : kP2SchedNoInput[rank];
      const int nSched = nu > 0 ? 5 : 4;
      for (int j = 0; j < nSched; ++j) {
        const int id = sched[j];
        if (id < 0) break;
        if (id < 13) {   // Q~ = Q + A'W_A, q~ = q + A'v, over P
          const SymItem s = kSymItems[id];
          const int tn[4] = {s.n[0], s.n[1], s.n[2], s.n[3]};
          mma_item<true, true, 4, NXR, false, true, false>(lane, NXR, NX1R, 0, 1.0, AB, NXR, s.m, W, LWR, tn, s.cnt, P, NXR, qg, NXR, Qg, NXR);
        } else {         // [S~ | r~] = [S | r] + B'[W_A | v], over W_B
          const int tm = (id - 13) >> 1, g = ((id - 13) & 1) * 4;
          const int tn[4] = {g, g + 1, g + 2, g + 3};
          mma_item<true, true, 4, NXR, false, true, false>(lane, nu, NX1R, 0, 1.0, Bk, NXR, tm, W, LWR, tn, 4, W + Y_OFF, NMR, rg, NXR, Sg, NMR);
        }
      }
    }
    WB_TICK(8, 0)
    laneSync();
    WB_TICK(3, 0)
    WB_TICK(25, 256)
    // [A | b | B] of this stage is dead now: its buffer takes stage k-1's, which lands behind P3 .. P5 (and behind the other lane)
    if (!gemmWarp && k > 0) prefetchBulk(k - 1);
    double* Yl = W;
    double* Kout = W + KOUT_OFF;
    if (nu > 0) {
      // ---- P3: [Yl | yl] = L^-1 [S~ | r~] (into the W region) -----------------------------------------------------------------------------
      if (gemmWarp) {
        for (int it = lw; it < 6; it += LANE_GEMM_WARPS) {
          const int tm = it >> 1, g = (it & 1) * 4;
          const int tn[4] = {g, g + 1, g + 2, g + 3};
          mma_item<false, false, 4, 0>(lane, nu, NX1R, nu, 1.0, Rt, LMR, tm, W + Y_OFF, NMR, tn, 4, Yl, LMR);
        }
      }
      laneSync();
      WB_TICK(4, 0)
      // ---- P4: [P | p] = [Q~ | q~] - Yl'[Yl | yl] (lower tiles) ; [K | k] = -L^-T [Yl | yl] -------------------------------------------------
      if (gemmWarp) {
        for (int it = lw; it < 19; it += LANE_GEMM_WARPS) {
          if (it < 8 || it >= 14) {
            const SymItem s = kSymItems[it < 8 ? it : it - 6];
            const int tn[4] = {s.n[0], s.n[1], s.n[2], s.n[3]};
            mma_item<true, true, 4, 0>(lane, NXR, NX1R, nu, -1.0, Yl, LMR, s.m, Yl, LMR, tn, s.cnt, P, NXR);
          } else {
            const int j = it - 8, tm = j >> 1, g = (j & 1) * 4;
            const int tn[4] = {g, g + 1, g + 2, g + 3};
            mma_item<true, false, 4, 0>(lane, nu, NX1R, nu, -1.0, Rt, LMR, tm, Yl, LMR, tn, 4, Kout, NMR);
          }
        }
      }
      laneSync();
      WB_TICK(5, 0)
    }
    // ---- P5: reg_prim on the diagonal, gains out -------------------------------------------------------------------------------------------
    if (lt < NXR) P[lt + lt * NXR] += v.reg;
    if (nu > 0) {
      for (int t = lt; t < NMR * NXR; t += LANE_THREADS) v.K[sk * NMR * NXR + t] = (t % NMR < nu) ? Kout[t] : 0.0;
      for (int t = lt; t < nu; t += LANE_THREADS) v.kff[sk * NMR + t] = Kout[NMR * NXR + t];
    }
    WB_TICK(6, 0)
    WB_TICK(26, 256)
    // (the barrier at the top of the next stage orders this phase before the next GEMM)
  }
  laneSync();
  if (v.keepP) storeP(0, lt, LANE_THREADS);
  if (lt == 0) v.status[inst] = !*ok;
}

// warp_chol_inverse (dense.cuh) with reg added to the diagonal while loading.  Linv may be A: each lane consumes all its loads of A in the
// shuffles of column 0, which no lane completes before every lane has reached them, and the stores come after the last column.
template <int NMAX>
__device__ __forceinline__ void warp_chol_inverse_reg(int n, const double* A, int lda, double reg, double* Linv, int ldl, int* ok) {
  const int lane = threadIdx.x & 31;
  double a[NMAX], z[NMAX];
#pragma unroll
  for (int i = 0; i < NMAX; ++i) {
    const int r = i > lane ? i : lane, c = i > lane ? lane : i;
    a[i] = (i < n && lane < n) ? A[r + c * lda] + (i == lane ? reg : 0.0) : ((i == lane) ? 1.0 : 0.0);
    z[i] = (i == lane) ? 1.0 : 0.0;
  }
  bool good = true;
#pragma unroll
  for (int k = 0; k < NMAX; ++k) {
    double d = __shfl_sync(0xffffffffu, a[k], k);
    if (!(d > 0.0)) {
      good = false;
      d = 1.0;
    }
    const double inv = rsqrt(d);
    const double ljk = a[k] * inv;
    z[k] *= inv;
#pragma unroll
    for (int i = k + 1; i < NMAX; ++i) {
      const double vv = __shfl_sync(0xffffffffu, a[i], k) * inv;
      a[i] = fma(-vv, ljk, a[i]);
      z[i] = fma(-vv, z[k], z[i]);
    }
  }
#pragma unroll
  for (int i = 0; i < NMAX; ++i)
    if (i < n && lane < n) Linv[i + lane * ldl] = z[i];
  if (lane == 0 && !good) *ok = 0;
}

// ---- forward substitution ---------------------------------------------------------------------------------------------------------------
constexpr int FWD_THREADS = 128;
constexpr int FWD_A = NXR * NXR, FWD_B = NXR * NMR, FWD_K = NMR * NXR;
constexpr int FWD_SET = FWD_A + NXR + FWD_B + FWD_K + 24;   // A | b | B | K | k (padded to an even count)
constexpr size_t FWD_SMEM_BYTES = static_cast<size_t>(2 * FWD_SET) * 8;

__global__ void __launch_bounds__(FWD_THREADS) riccati_fwd_kernel(QpDeviceView v) {
  extern __shared__ double sm[];
  const int inst = blockIdx.x;
  if (v.skip && v.skip[inst * v.skipStride]) return;
  const int N = v.N, tid = threadIdx.x;
  __shared__ unsigned long long bar[2];
  __shared__ double xv[NXR], uv[24], part[4][64];
  const size_t iN = static_cast<size_t>(inst) * N, iN1 = static_cast<size_t>(inst) * (N + 1);
  if (tid == 0) {
    mbar_init(&bar[0], 1);
    mbar_init(&bar[1], 1);
    mbar_fence_init();
  }
  for (int i = tid; i < NXR; i += blockDim.x) {
    const double x0 = v.dx0[static_cast<size_t>(inst) * NXR + i];
    xv[i] = x0;
    v.dx[iN1 * NXR + i] = x0;
  }
  __syncthreads();
  auto prefetch = [&](int k, int set) {   // one thread: four bulk copies (A, b, B, K are contiguous, 16-byte multiples); k rides as plain loads
    const size_t sk = iN + k;
    double* s = sm + set * FWD_SET;
    const int nu = v.nu ? v.nu[sk] : NMR;
    fence_proxy_async();
    mbar_expect_tx(&bar[set], static_cast<unsigned>((FWD_A + NXR + (nu > 0 ? FWD_B + FWD_K : 0)) * 8));
    bulk_g2s(s, v.A + sk * FWD_A, FWD_A * 8, &bar[set]);
    bulk_g2s(s + FWD_A, v.b + sk * NXR, NXR * 8, &bar[set]);
    if (nu > 0) {
      bulk_g2s(s + FWD_A + NXR, v.Bm + sk * FWD_B, FWD_B * 8, &bar[set]);
      bulk_g2s(s + FWD_A + NXR + FWD_B, v.K + sk * FWD_K, FWD_K * 8, &bar[set]);
    }
  };
  if (tid == 0) prefetch(0, 0);
  unsigned parity[2] = {0, 0};
  const int w = tid >> 5, lane = tid & 31;
  for (int k = 0; k < N; ++k) {
    const int set = k & 1;
    const size_t sk = iN + k;
    const int nu = v.nu ? v.nu[sk] : NMR;
    const double* s = sm + set * FWD_SET;
    const double* Ak = s;
    const double* bk = s + FWD_A;
    const double* Bk = s + FWD_A + NXR;
    const double* Kk = s + FWD_A + NXR + FWD_B;
    if (tid == 0 && k + 1 < N) prefetch(k + 1, 1 - set);   // (the other set was last read before the barrier that ended stage k-1)
    const double kffv = (w == 0 && lane < nu) ? v.kff[sk * NMR + lane] : 0.0;
    mbar_wait(&bar[set], parity[set]);
    parity[set] ^= 1;
    // du = K dx + k: row = lane (23 of 32), the 58 columns split over the four warps
    if (nu > 0) {
      double s0 = 0.0, s1 = 0.0;
      if (lane < nu) {
        const int c0 = w * 15, c1 = (c0 + 15 < NXR) ? c0 + 15 : NXR;
        int c = c0;
        for (; c + 1 < c1; c += 2) {
          s0 = fma(Kk[lane + c * NMR], xv[c], s0);
          s1 = fma(Kk[lane + (c + 1) * NMR], xv[c + 1], s1);
        }
        if (c < c1) s0 = fma(Kk[lane + c * NMR], xv[c], s0);
      }
      part[w][lane] = s0 + s1;
    }
    __syncthreads();
    if (tid < NMR) {
      const double r = (tid < nu) ? (part[0][tid] + part[1][tid]) + (part[2][tid] + part[3][tid]) + kffv : 0.0;
      uv[tid] = r;
      v.du[sk * NMR + tid] = r;
    }
    __syncthreads();
    // dx+ = A dx + B du + b: rows 0..57 on 64 threads x 2 column halves of [A | B]
    {
      const int row = tid & 63, half = tid >> 6;
      double s0 = 0.0, s1 = 0.0;
      if (row < NXR) {
        if (half == 0) {
          for (int c = 0; c < 40; c += 2) {
            s0 = fma(Ak[row + c * NXR], xv[c], s0);
            s1 = fma(Ak[row + (c + 1) * NXR], xv[c + 1], s1);
          }
        } else {
          for (int c = 40; c < NXR; c += 2) {
            s0 = fma(Ak[row + c * NXR], xv[c], s0);
            s1 = fma(Ak[row + (c + 1) * NXR], xv[c + 1], s1);
          }
          for (int c = 0; c < nu; ++c) s0 = fma(Bk[row + c * NXR], uv[c], s0);
          s0 += bk[row];
        }
      }
      part[half][row] = s0 + s1;
    }
    __syncthreads();
    if (tid < NXR) {
      const double r = part[0][tid] + part[1][tid];
      xv[tid] = r;
      v.dx[(iN1 + k + 1) * NXR + tid] = r;
    }
    __syncthreads();
  }
  if (tid == 0) {
    int bad = 0;
    for (int i = 0; i < NXR; ++i) bad |= !isfinite(xv[i]);
    if (bad) v.status[inst] = 1;
  }
}

}  // namespace ricwb
}  // namespace b200sqp
