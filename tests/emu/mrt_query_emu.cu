// DEVELOPMENT HARNESS (tests only, never linked into libb200sqp.so): the MRT queries (wb_query.cuh: mrtQuery) executed on the CPU, with a
// phase runner of 24 slices visited one after another, in reverse.  Built into tests/emu/libmrtqueryemu.so by tests/test_emu_mrt_query.py.
// The product has no CPU path.
#include "../../wb_humanoid_mpc_b200/csrc/wb_query.cuh"

using namespace b200sqp;

namespace {
struct EmuQueryPhase {   // 24 slices: a width other than the kernel's, so that a result that depends on the split shows up
  static constexpr int slots = 24;
  template <class F>
  void operator()(F&& f) const {
    for (int t = slots - 1; t >= 0; --t) f(Par{t, slots});
  }
};
}  // namespace

extern "C" {

// one instance on the device layout: t [n], event [n], K [n-1][NU*NX] column-major (or NULL), P [n][NX*NX] column-major and p [n][NX] (or
// NULL), sx the ABI state width (58 or 35), x [sx] -> dfdxx [sx*sx], dfdx [sx], Kq [NU*sx], each may be NULL.  Returns the segment index.
int emu_mrt_query(int n, const double* t, const uint8_t* event, const double* K, const double* P, const double* p, int sx, double tq, const double* x,
                  double* dfdxx, double* dfdx, double* Kq) {
  const SimPlan plan{n, t, event, nullptr, nullptr, nullptr, K};
  mrtQuery(EmuQueryPhase{}, plan, P, p, sx, tq, x, dfdxx, dfdx, Kq);
  int idx;
  double alpha;
  simTimeSegment(t, n, tq, idx, alpha);
  return idx;
}

}  // extern "C"
