// The shared-memory map of riccati_wb.cuh's riccati_bwd_kernel, for tests/test_emu_riccati_wb_layout.py (CPU only).
#include "../../wb_humanoid_mpc_b200/csrc/riccati_wb.cuh"

extern "C" {
// out: {lanes, lane_d, pq_off, ab_off, w_off, rt_off, rin_off, smem_d, smem_bytes, static_bytes, ldw, ldm, yl_d, kout_off, y_off, threads,
//       lane_threads}
void emu_ricwb_layout(long long* out) {
  using namespace b200sqp::ricwb;
  const long long v[] = {LANES, LANE_D, PQ_OFF, AB_OFF, W_OFF, RT_OFF, RIN_OFF, BWD_SMEM_D, static_cast<long long>(BWD_SMEM_BYTES),
                         static_cast<long long>(BWD_STATIC_SMEM_BYTES), LWR, LMR, YL_D, KOUT_OFF, Y_OFF, BWD_THREADS, LANE_THREADS};
  for (int i = 0; i < static_cast<int>(sizeof(v) / sizeof(v[0])); ++i) out[i] = v[i];
}
}
