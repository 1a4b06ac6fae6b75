// Fleets (b200sqp_fleet_*): a batch whose instances may differ in node count, solved as one group per node count.  Every cycle the builder's
// grid pass runs over all instances in caller order; the partition below sorts them stably by node count (a counting sort in one CTA), and each
// group is solved as a view into the handle's batch allocation: slots [first, first + count) of the batch, instance arrays at the stride of the
// batch's node capacity.  The kernels here move the state that must survive a cycle between the two orders:
//   carry    the iterate of every view -> the builder's caller-order previous solution (per-instance length, rows strided by the capacity);
//   permute  caller order <-> slot order for the roll-out / joint-action inputs and outputs and the simulated state.
#pragma once
#include "wb_batch.cuh"
#include "wb_builder.cuh"

namespace b200sqp {

// ---- the partition, as phases of one CTA (tid, nt), so that the CPU harness can run the same functions thread by thread ---------------------------
// key[i] = node count of instance i (clamped into [0, nBins)); cnt[nBins] is the histogram, then the running offsets
// group table gtab = {G, (nodes, first slot, count) * G} in increasing node count; slotInst[s] = the instance in slot s.
HD void fleetCountAdd(int* p) {
#ifdef __CUDA_ARCH__
  atomicAdd(p, 1);
#else
  ++*p;
#endif
}
HD void fleetHistogram(const int* key, int B, int* cnt, int tid, int nt) {
  for (int i = tid; i < B; i += nt) fleetCountAdd(&cnt[key[i]]);
}
// one thread: histogram -> exclusive offsets, and the group table
HD void fleetOffsets(int* cnt, int nBins, int* gtab) {
  int g = 0, off = 0;
  for (int n = 0; n < nBins; ++n) {
    const int c = cnt[n];
    if (c) {
      gtab[1 + 3 * g] = n;
      gtab[2 + 3 * g] = off;
      gtab[3 + 3 * g] = c;
      ++g;
    }
    cnt[n] = off;
    off += c;
  }
  gtab[0] = g;
}
// tile [tile, tile + nt): instance i goes behind the instances of its node count in earlier tiles and in front of later ones of this tile (stable)
HD void fleetPlace(const int* key, int B, const int* off, int* slotInst, int tile, int tid) {
  const int i = tile + tid;
  if (i >= B) return;
  const int k = key[i];
  int r = 0;
  for (int j = tile; j < i; ++j) r += key[j] == k;
  slotInst[off[k] + r] = i;
}
HD void fleetAdvance(const int* key, int B, int* off, int tile, int tid) {
  const int i = tile + tid;
  if (i < B) fleetCountAdd(&off[key[i]]);
}

// group g of the table: the slot range and node count of a slot s (G is small: one entry per distinct node count)
HD int fleetGroupOf(const int* gtab, int s) {
  int g = 0;
  while (g + 1 < gtab[0] && s >= gtab[2 + 3 * (g + 1)]) ++g;
  return g;
}
// slot s of a batch of B instances allocated at capNodes nodes each: its group's node count, first slot and size (gtab null: a plain handle,
// one group of B instances at capNodes nodes), and the slot's first node and stage rows in the allocation (groupView's rows, then the slot's
// position in its group)
struct FleetSlot {
  int n, first, count;
  size_t node, stage;
};
HD FleetSlot fleetSlot(const int* gtab, int B, int capNodes, int s) {
  FleetSlot r{capNodes, 0, B, 0, 0};
  if (gtab) {
    const int g = fleetGroupOf(gtab, s);
    r.n = gtab[1 + 3 * g];
    r.first = gtab[2 + 3 * g];
    r.count = gtab[3 + 3 * g];
  }
  r.node = batchRows(ROW_NODE, r.first, capNodes) + batchRows(ROW_NODE, s - r.first, r.n);
  r.stage = batchRows(ROW_STAGE, r.first, capNodes) + batchRows(ROW_STAGE, s - r.first, r.n);
  return r;
}

#ifdef __CUDACC__
// one CTA; dynamic shared memory: nBins ints
__global__ void fleet_partition_kernel(const BldScratch* sc, int B, int nBins, int* key, int* slotInst, int* gtab) {
  extern __shared__ int cnt[];
  const int tid = threadIdx.x, nt = blockDim.x;
  for (int n = tid; n < nBins; n += nt) cnt[n] = 0;
  for (int i = tid; i < B; i += nt) key[i] = min(max(sc[i].nNodes, 0), nBins - 1);
  __syncthreads();
  fleetHistogram(key, B, cnt, tid, nt);
  __syncthreads();
  if (tid == 0) fleetOffsets(cnt, nBins, gtab);
  __syncthreads();
  for (int tile = 0; tile < B; tile += nt) {
    fleetPlace(key, B, cnt, slotInst, tile, tid);
    __syncthreads();
    fleetAdvance(key, B, cnt, tile, tid);
    __syncthreads();
  }
}

// carry: slot s of the last solve's group table (its view's iterate x / u, grid t / event, at the batch's capacity stride) -> row slotInst[s] of
// the caller-order previous solution (stride cap), prevLen = the group's node count.  One CTA per slot.
__global__ void __launch_bounds__(128) fleet_carry_kernel(WbDev base, int capNodes, const int* gtab, const int* slotInst, double* prevX, double* prevU,
                                                          double* prevT, uint8_t* prevE, int* prevLen) {
  const int s = blockIdx.x;
  const FleetSlot sl = fleetSlot(gtab, gridDim.x, capNodes, s);
  const int n = sl.n, i = slotInst[s];
  const size_t node0 = sl.node, stage0 = sl.stage;
  const size_t dst = static_cast<size_t>(i) * capNodes;
  for (size_t j = threadIdx.x; j < static_cast<size_t>(n) * NX; j += blockDim.x) prevX[dst * NX + j] = base.x[node0 * NX + j];
  for (size_t j = threadIdx.x; j < static_cast<size_t>(n - 1) * NU; j += blockDim.x) prevU[dst * NU + j] = base.u[stage0 * NU + j];
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    prevT[dst + j] = base.t[node0 + j];
    prevE[dst + j] = base.event[node0 + j];
  }
  if (threadIdx.x == 0) prevLen[i] = n;
}

// rows of `width` entries: scatter = 1: src row r -> dst row inst[r] (slot -> caller order); scatter = 0: src row inst[r] -> dst row r
template <class T>
__global__ void __launch_bounds__(64) fleet_permute_kernel(const T* src, int srcStride, T* dst, int dstStride, int width, const int* inst, int scatter) {
  const int r = blockIdx.x, i = inst[r];
  const T* a = src + static_cast<size_t>(scatter ? r : i) * srcStride;
  T* o = dst + static_cast<size_t>(scatter ? i : r) * dstStride;
  for (int j = threadIdx.x; j < width; j += blockDim.x) o[j] = a[j];
}
#endif

}  // namespace b200sqp
