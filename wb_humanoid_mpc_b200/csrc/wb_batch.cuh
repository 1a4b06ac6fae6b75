// The batch layout of a handle: the device arrays of WbDev, with the row kind and width of each and the conditions under which it exists.
// set_batch allocates by walking it, and a fleet's group views (groupView) offset by walking it.
#pragma once
#include "wb_solver.cuh"

namespace b200sqp {

// f(field, row kind, width in elements, zero) for every array of the batch allocation, in allocation order.  The table decides which arrays
// exist: the cost-to-go matrices P with settings.create_value_function, the remapped gains Kre with settings.use_feedback_policy, the K1a /
// K1b records mid, luRec and luPerm on whole-body handles (cen false), the raw stage blocks with raw capture on.  zero: the padded state rows
// of a centroidal handle, zero-filled at allocation; they stay zero for the lifetime of the batch.  The widths of log and raw are d.maxIter
// and d.rawPer.
template <class F>
void forEachBatchArray(WbDev& d, bool cen, bool raw, F&& f) {
  const auto a = [&](auto*& p, RowKind k, size_t w) { f(p, k, w, false); };
  f(d.x0, ROW_INST, NX, cen);
  f(d.x, ROW_NODE, NX, cen);
  a(d.u, ROW_STAGE, NU);
  a(d.xInit, ROW_NODE, NX);
  a(d.uInit, ROW_STAGE, NU);
  a(d.t, ROW_NODE, 1);
  a(d.swing, ROW_NODE, 6);
  a(d.impact, ROW_NODE, 2);
  a(d.arm, ROW_NODE, 1);
  f(d.xref, ROW_NODE, NX, cen);
  a(d.event, ROW_NODE, 1);
  a(d.contact, ROW_NODE, 2);
  forEachQpArray(d.qp, d.st.create_value_function != 0, a);
  a(d.Pu, ROW_STAGE, NU * NUT_MAX);
  a(d.Px, ROW_STAGE, NU * NX);
  a(d.u0p, ROW_STAGE, NU);
  a(d.du, ROW_STAGE, NU);
  if (d.st.use_feedback_policy) a(d.Kre, ROW_STAGE, NU * NX);
  a(d.perfNode, ROW_NODE, 4);
  a(d.lsNode, ROW_NODE, 4);
  a(d.inst, ROW_INST, I_ND);
  a(d.flags, ROW_INST, F_NF);
  a(d.pending, ROW_HANDLE, 1);
  a(d.log, ROW_INST, d.maxIter);
  if (!cen) {
    a(d.mid, ROW_STAGE, Mid::SIZE);
    a(d.luRec, ROW_STAGE, LU_REC);
    a(d.luPerm, ROW_STAGE, LU_PERM);
  }
  a(d.gstats, ROW_HANDLE, 32 * 4 + 8);   // + [8]: all-reduced copy of the current candidate
  if (raw) a(d.raw, ROW_STAGE, d.rawPer);
}
// Both structs are kernel parameters, so their members keep their order.  A member added to either changes its size here: give it its place
// in the table above (or in forEachQpArray), then update the size.
static_assert(sizeof(QpDeviceView) == 184, "QpDeviceView changed: place the new member in forEachQpArray");
static_assert(sizeof(WbDev) == 560, "WbDev changed: place the new member in forEachBatchArray");

// Slots [first, first + count) of a batch allocated at capNodes nodes per instance, as a batch of their own with n nodes per instance: every
// instance, node and stage array offset to the slot range's first row (the instances of the view are packed at its own node count inside),
// and the view's line-search counter.  Handle-wide arrays and the models stay the base's.
inline WbDev groupView(const WbDev& base, int capNodes, int n, int first, int count, int* pending) {
  WbDev v = base;
  v.B = v.qp.B = count;
  v.N = v.qp.N = n - 1;
  forEachBatchArray(v, false, true, [&](auto*& p, RowKind k, size_t w, bool) {   // (every array the table knows; the absent ones are null)
    if (p && k != ROW_HANDLE) p += batchRows(k, first, capNodes) * w;
  });
  v.qp.skip = v.flags + F_CONVERGED;
  v.pending = pending;
  return v;
}

}  // namespace b200sqp
