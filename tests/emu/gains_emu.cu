// DEVELOPMENT HARNESS (tests only, never linked into libb200sqp.so): the row of gains_apply_kernel (wb_gains.cuh) on the CPU -- the check,
// the copy of the handle's model by 128 threads visited in reverse order, and the gain fields -- so that tests/test_emu_gains.py can compare
// the model it makes with the model the handle's constructor makes from a description carrying the same gains.
#include <cstdio>
#include <cstring>

#include "../../wb_humanoid_mpc_b200/csrc/cen_host.cuh"
#include "../../wb_humanoid_mpc_b200/csrc/wb_gains.cuh"
#include "../../wb_humanoid_mpc_b200/csrc/wb_host.cuh"

using namespace b200sqp;

namespace {
template <class M>
int gainsRow(const M& base, const b200sqp_gains* g, bool cen, void* out, int64_t* bytes) {
  *bytes = sizeof(M);
  if (!g) {
    std::memcpy(out, &base, sizeof(M));
    return 0;
  }
  if (const int st = gainsStatus(*g, cen)) return st;
  static M inst;
  std::memset(&inst, 0xA5, sizeof(M));   // a word the copy misses shows as a mismatch
  for (int tid = 127; tid >= 0; --tid) gainsCopyBase(base, inst, tid, 128);
  gainsWrite(*g, inst);
  std::memcpy(out, &inst, sizeof(M));
  return 0;
}
}  // namespace

extern "C" {

// the model of d (c = null: whole-body, else centroidal) after the gains row g -> out [*bytes]; g = null: the model of d itself.
// Returns the row status (0 applied, 1 not finite, 2 out of range), or -1 for a description the model constructor refuses.
int emu_gains_model(const b200sqp_model_desc* d, const b200sqp_cen_desc* c, const b200sqp_gains* g, void* out, int64_t* bytes) {
  static WbDeviceModel wm;
  static CenDevModel cm;
  const char* e = c ? makeCenDeviceModel(*d, *c, cm) : makeDeviceModel(*d, wm);
  if (e) {
    std::fprintf(stderr, "emu: %s\n", e);
    return -1;
  }
  return c ? gainsRow(cm, g, true, out, bytes) : gainsRow(wm, g, false, out, bytes);
}
}
