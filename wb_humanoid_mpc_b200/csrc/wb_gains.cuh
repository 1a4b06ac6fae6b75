// Per-instance gains (b200sqp_set_gains): the cost weights and soft-constraint penalties of one instance written into its own copy of the
// handle's device model, for whole-body (WbDeviceModel) and centroidal (CenDevModel) handles.  The OCP kernels read instance b's model at
// instModel[b * modelStride] / instCen[b * modelStride] (WbDev); the stride is 0, and the pointer the handle's model, until gains are set.
// The row functions are __host__ __device__ so that the CPU harness runs the code of gains_apply_kernel.
#pragma once
#include <cstring>

#include "cen_solver.cuh"
#include "wb_model.cuh"

namespace b200sqp {

constexpr int GAINS_OK = 0, GAINS_NOT_FINITE = 1, GAINS_OUT_OF_RANGE = 2;

// The check of one record (the status of b200sqp_set_gains_dev): 1 when a used entry is not finite, else 2 when one is out of range, else 0.
// Used entries: nx / nu of Q, Qf / R, 18 (whole-body) or 12 (centroidal) foot weights, the 12 task-space weights on centroidal handles.
HD int gainsStatus(const b200sqp_gains& g, bool cen) {
  const int nx = cen ? CNX : NX, nu = cen ? CNU : NU, nFoot = cen ? 12 : 18, nTorso = cen ? 12 : 0;
  const double pen[10] = {g.jlim_mu, g.jlim_delta, g.coll_mu, g.coll_delta, g.coll_r_foot, g.coll_r_knee, g.fric_mu, g.fric_delta, g.momxy_mu, g.momxy_delta};
  bool finite = true, range = true;
  auto nonNeg = [&](double v) {
    finite &= v - v == 0.0;
    range &= v >= 0.0;
  };
  for (int i = 0; i < nx; ++i) {
    nonNeg(g.Q_diag[i]);
    nonNeg(g.Qf_diag[i]);
  }
  for (int i = 0; i < nu; ++i) {
    finite &= g.R_diag[i] - g.R_diag[i] == 0.0;
    range &= g.R_diag[i] > 0.0;
  }
  for (int k = 0; k < nFoot; ++k) nonNeg(g.foot_cost_w[k]);
  for (int k = 0; k < nTorso; ++k) nonNeg(g.torso_w[k]);
  for (int k = 0; k < 10; ++k) nonNeg(pen[k]);
  range &= g.jlim_delta > 0.0 && g.coll_delta > 0.0 && g.fric_delta > 0.0 && g.momxy_delta > 0.0;
  const int32_t flags[7] = {g.final_cost_active, g.foot_cost_active, g.torso_cost_active, g.joint_limits_active, g.foot_collision_active,
                            g.friction_cone_active, g.contact_moment_active};
  for (int k = 0; k < 7; ++k) range &= flags[k] == 0 || flags[k] == 1;
  return !finite ? GAINS_NOT_FINITE : !range ? GAINS_OUT_OF_RANGE : GAINS_OK;
}

// phase 1 (threads tid of nt): the instance's model starts as the handle's
template <class M>
HD void gainsCopyBase(const M& base, M& out, int tid, int nt) {
  static_assert(sizeof(M) % 8 == 0, "the models are copied as 8-byte words");
  const unsigned long long* s = reinterpret_cast<const unsigned long long*>(&base);
  unsigned long long* o = reinterpret_cast<unsigned long long*>(&out);
  for (int i = tid; i < static_cast<int>(sizeof(M) / 8); i += nt) o[i] = s[i];
}

// phase 2 (one thread): the gain fields and what is derived from them, as makeDeviceModel / makeCenDeviceModel derive it; an inactive term
// gets zero weights (costs) or a zero mu (penalties), so that it adds exactly zero
HD void gainsWrite(const b200sqp_gains& g, WbDeviceModel& m) {
  for (int i = 0; i < NX; ++i) {
    m.Qd[i] = g.Q_diag[i];
    m.Qfd[i] = g.final_cost_active ? g.Qf_diag[i] : 0.0;
  }
  for (int i = 0; i < NU; ++i) m.Rd[i] = g.R_diag[i];
  for (int k = 0; k < 18; ++k) m.footSqrtW[k] = g.foot_cost_active ? sqrt(g.foot_cost_w[k]) : 0.0;
  m.jlMu = g.joint_limits_active ? g.jlim_mu : 0.0;
  m.jlDelta = g.jlim_delta;
  m.collMu = g.foot_collision_active ? g.coll_mu : 0.0;
  m.collDelta = g.coll_delta;
  m.rFoot = g.coll_r_foot;
  m.rKnee = g.coll_r_knee;
  m.fricMu = g.friction_cone_active ? g.fric_mu : 0.0;
  m.fricDelta = g.fric_delta;
  m.momMu = g.contact_moment_active ? g.momxy_mu : 0.0;
  m.momDelta = g.momxy_delta;
}
HD void gainsWrite(const b200sqp_gains& g, CenDevModel& c) {
  CenOcpModel& m = c.ocp;
  for (int i = 0; i < CNX; ++i) {
    m.Qd[i] = g.Q_diag[i];
    m.Qfd[i] = c.QfdPad[i] = g.final_cost_active ? g.Qf_diag[i] : 0.0;
  }
  for (int i = 0; i < CNU; ++i) m.Rd[i] = g.R_diag[i];
  for (int k = 0; k < 12; ++k) {
    m.torsoSqrtW[k] = g.torso_cost_active ? sqrt(g.torso_w[k]) : 0.0;
    m.footSqrtW[k] = g.foot_cost_active ? sqrt(g.foot_cost_w[k]) : 0.0;
  }
  m.jlMu = g.joint_limits_active ? g.jlim_mu : 0.0;
  m.jlDelta = g.jlim_delta;
  m.collMu = g.foot_collision_active ? g.coll_mu : 0.0;
  m.collDelta = g.coll_delta;
  m.rFoot = g.coll_r_foot;
  m.rKnee = g.coll_r_knee;
  m.fricMu = g.friction_cone_active ? g.fric_mu : 0.0;
  m.fricDelta = g.fric_delta;
  m.momMu = g.contact_moment_active ? g.momxy_mu : 0.0;
  m.momDelta = g.momxy_delta;
}

// The record of the model description's values, every term active (b200sqp_default_gains); cen: the centroidal description, or null.
inline b200sqp_gains gainsFromDesc(const b200sqp_model_desc& d, const b200sqp_cen_desc* cen) {
  b200sqp_gains g;
  std::memset(&g, 0, sizeof(g));
  std::memcpy(g.Q_diag, d.Q_diag, sizeof(g.Q_diag));
  std::memcpy(g.R_diag, d.R_diag, sizeof(g.R_diag));
  std::memcpy(g.Qf_diag, d.Qf_diag, sizeof(g.Qf_diag));
  std::memcpy(g.foot_cost_w, d.foot_cost_w, sizeof(g.foot_cost_w));
  if (cen) std::memcpy(g.torso_w, cen->torso_w, sizeof(g.torso_w));
  g.jlim_mu = d.jlim_mu;
  g.jlim_delta = d.jlim_delta;
  g.coll_mu = d.coll_mu;
  g.coll_delta = d.coll_delta;
  g.coll_r_foot = d.coll_r_foot;
  g.coll_r_knee = d.coll_r_knee;
  g.fric_mu = d.fric_mu;
  g.fric_delta = d.fric_delta;
  g.momxy_mu = d.momxy_mu;
  g.momxy_delta = d.momxy_delta;
  g.final_cost_active = g.foot_cost_active = g.torso_cost_active = g.joint_limits_active = g.foot_collision_active = g.friction_cone_active =
      g.contact_moment_active = 1;
  return g;
}

#ifdef __CUDACC__
static_assert(sizeof(b200sqp_gains) % 8 == 0, "the records are copied as 8-byte words");

// One CTA per listed row r: instance idx[r] gets the record in[r].  A row that fails the check writes its status and leaves the instance
// unchanged; status may be null.  restore = 1: the instance goes back to the handle's model unchecked (in[r] is then the default record).
template <class M>
__global__ void __launch_bounds__(128) gains_apply_kernel(const M* base, M* inst, const b200sqp_gains* in, const int* idx, b200sqp_gains* rec,
                                                          int* custom, int restore, int* status, int cen) {
  const int r = blockIdx.x, i = idx[r];
  const b200sqp_gains& g = in[r];
  __shared__ int st;
  if (threadIdx.x == 0) {
    st = restore ? GAINS_OK : gainsStatus(g, cen != 0);
    if (status) status[r] = st;
  }
  __syncthreads();
  if (st != GAINS_OK) return;
  gainsCopyBase(*base, inst[i], threadIdx.x, blockDim.x);
  const unsigned long long* gs = reinterpret_cast<const unsigned long long*>(&g);
  unsigned long long* go = reinterpret_cast<unsigned long long*>(rec + i);
  for (int j = threadIdx.x; j < static_cast<int>(sizeof(b200sqp_gains) / 8); j += blockDim.x) go[j] = gs[j];
  __syncthreads();
  if (threadIdx.x == 0) {
    if (!restore) gainsWrite(g, inst[i]);
    custom[i] = !restore;
  }
}
#endif

}  // namespace b200sqp
