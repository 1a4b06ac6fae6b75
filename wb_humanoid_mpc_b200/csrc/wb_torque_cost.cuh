// Joint-torque cost of the whole-body OCP (reference: JointTorqueCostCppAd, humanoid_nmpc/humanoid_wb_mpc/src/cost/JointTorqueCostCppAd.cpp,
// wired in WBMpcInterface.cpp, commented out in the shipped interface): a Gauss-Newton StateInputCost of every intermediate node with the residual
//   r(x, u) = sqrt(w) .* tau(x, u),   tau = computeJointTorques(x, u)   (wb_torque.cuh: the same map as the MRT controllers)
// value 1/2 |r|^2, gradient J' r, Hessian J' J (no second-order term), J = dr/d(x, u) (NJ x 93), all scaled by the node's dt.
//
// Own formulation.  The term is optional, so it lives in kernels of its own that the solve launches only while it is on; K1a and K1b are not
// touched.  Two facts shape them:
//   * the raw Hessian of a node never exists as dense blocks in memory: K1b part 2 forms S and R in shared memory from the K1a record and
//     writes only the projected blocks.  The change of input variables (u = Px dx + Pu du~ + u0, changeOfInputVariables) is linear in the cost
//     approximation, so the term's own approximation, projected, is ADDED to K1b's output: with the residual written in the projected inputs,
//       r + J [dx; du] = r' + Ax dx + Au du~,   r' = r + Ju u0,  Ax = Jx + Ju Px,  Au = Ju Pu,
//     Q~ += dt Ax'Ax, S~ += dt Au'Ax, R~ += dt Au'Au, q~ += dt Ax'r', r~ += dt Au'r' and the projected cost offset += dt (r'Ju u0 + 1/2 |Ju u0|^2).
//     That is exactly what projecting (raw blocks + term) gives, up to the order of the floating-point sums.
//   * J by forward mode: lane d of a 96-thread CTA carries tangent direction d (x then u) through the value recursion of wb_torque.cuh in
//     single-tangent duals (D1), both Newton-Euler passes and the block-diagonal M_bb inverse of the base acceleration included -- so dtau/dz
//     carries M_jb dqdd_b/dz as computeJointTorques' CppAD tape does.  One instruction stream for all lanes, no closed forms to keep in step.
// Line search: jt_trial_kernel adds dt * 1/2 |r|^2 of every intermediate node of every searching instance to K3's per-node trial cost.
#pragma once
#include "wb_solver.cuh"
#include "wb_torque.cuh"

namespace b200sqp {

constexpr int JT_THREADS = 96;   // >= NZ tangent lanes

struct JtWeights {   // sqrt(joint_torque_weights), MPC joint order (JointTorqueCostCppAd::getParameters)
  double sw[NJ];
};

struct JtBody {
  DM3 R;
  DV3 p, w, al, a, ax;
};
HD DV3 dc3(const double* p) { return dconst(p[0], p[1], p[2]); }
HD DM3 dcm3(const double* A) {
  DM3 M;
#pragma unroll
  for (int i = 0; i < 9; ++i) M.m[i] = dmk(A[i]);
  return M;
}
HD DM3 dtr3(const DM3& A) {
  DM3 T;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) T.m[3 * i + j] = A.m[3 * j + i];
  return T;
}

// tqInverseDynamics (wb_torque.cuh) on single-tangent duals: generalized forces for the base acceleration qddb (null: zero) minus the contact
// wrenches, out[0..6) base, out[6..) joints; with Mang: the base block M_ang = S' (R' Ic R) S of the block-diagonal M_bb
HD void jtInverseDynamics(const WbDeviceModel& m, const D1* q, const D1* qd, const D1* u, const D1* qddb, JtBody* B, D1* out, DM3* Mang) {
  const D1 c0 = dcos(q[3]), s0 = dsin(q[3]), c1 = dcos(q[4]), s1 = dsin(q[4]), c2 = dcos(q[5]), s2 = dsin(q[5]);
  DM3 S;
  B[0].R.m[0] = c0 * c1; B[0].R.m[1] = c0 * s1 * s2 - s0 * c2; B[0].R.m[2] = c0 * s1 * c2 + s0 * s2;
  B[0].R.m[3] = s0 * c1; B[0].R.m[4] = s0 * s1 * s2 + c0 * c2; B[0].R.m[5] = s0 * s1 * c2 - c0 * s2;
  B[0].R.m[6] = -s1;     B[0].R.m[7] = c1 * s2;                B[0].R.m[8] = c1 * c2;
  S.m[0] = -s1;     S.m[1] = dmk(0.0); S.m[2] = dmk(1.0);
  S.m[3] = c1 * s2; S.m[4] = c2;       S.m[5] = dmk(0.0);
  S.m[6] = c1 * c2; S.m[7] = -s2;      S.m[8] = dmk(0.0);
  B[0].p = DV3{q[0], q[1], q[2]};
  B[0].w = B[0].R * (S * DV3{qd[3], qd[4], qd[5]});
  {
    const D1 d0 = qd[3], d1 = qd[4], d2 = qd[5];
    const DV3 bias{-(c1 * d1 * d0), (-(s1 * s2 * d1) + c1 * c2 * d2) * d0 - s2 * d2 * d1, (-(s1 * c2 * d1) - c1 * s2 * d2) * d0 - c2 * d2 * d1};
    const DV3 sdd = qddb ? S * DV3{qddb[3], qddb[4], qddb[5]} : dconst(0, 0, 0);
    B[0].al = B[0].R * (bias + sdd);
  }
  B[0].a = (qddb ? DV3{qddb[0], qddb[1], qddb[2]} : dconst(0, 0, 0)) + dconst(0, 0, m.gravity);
  B[0].ax = dconst(0, 0, 0);
  for (int i = 1; i < NB; ++i) {
    const int pa = m.parent[i];
    const double* a = m.axis[i];
    const D1 th = q[5 + i], c = dcos(th), s = dsin(th), t = dmk(1.0) - c;
    DM3 Rq;
    Rq.m[0] = t * (a[0] * a[0]) + c;   Rq.m[1] = t * (a[0] * a[1]) - s * a[2]; Rq.m[2] = t * (a[0] * a[2]) + s * a[1];
    Rq.m[3] = t * (a[0] * a[1]) + s * a[2]; Rq.m[4] = t * (a[1] * a[1]) + c;   Rq.m[5] = t * (a[1] * a[2]) - s * a[0];
    Rq.m[6] = t * (a[0] * a[2]) - s * a[1]; Rq.m[7] = t * (a[1] * a[2]) + s * a[0]; Rq.m[8] = t * (a[2] * a[2]) + c;
    B[i].R = B[pa].R * (dcm3(m.jR[i]) * Rq);
    const DV3 r = B[pa].R * dc3(m.jp[i]);
    B[i].p = B[pa].p + r;
    B[i].ax = B[i].R * dc3(a);
    const D1 qdi = qd[5 + i], qddi = u[12 + (i - 1)];
    B[i].w = B[pa].w + qdi * B[i].ax;
    B[i].al = B[pa].al + qddi * B[i].ax + qdi * dcross(B[pa].w, B[i].ax);
    B[i].a = B[pa].a + dcross(B[pa].al, r) + dcross(B[pa].w, dcross(B[pa].w, r));
  }
  DV3 F[NB], Mo[NB];
  DM3 Ic;   // composite rotational inertia about the base origin, world axes
  for (int k = 0; k < 9; ++k) Ic.m[k] = dmk(0.0);
  for (int i = 0; i < NB; ++i) {
    const DV3 rc = B[i].R * dc3(m.com[i]);
    const DV3 cw = B[i].p + rc;
    const DV3 ac = B[i].a + dcross(B[i].al, rc) + dcross(B[i].w, dcross(B[i].w, rc));
    const DM3 Iw = B[i].R * dcm3(m.Icom[i]) * dtr3(B[i].R);
    F[i] = m.mass[i] * ac;
    Mo[i] = Iw * B[i].al + dcross(B[i].w, Iw * B[i].w) + dcross(cw, F[i]);
    if (Mang) {
      const DV3 d = cw - B[0].p;
      const D1 dd = ddot(d, d), dv[3] = {d.x, d.y, d.z};
      for (int r = 0; r < 3; ++r)
        for (int k = 0; k < 3; ++k) Ic.m[3 * r + k] = Ic.m[3 * r + k] + Iw.m[3 * r + k] + m.mass[i] * ((r == k ? dd : dmk(0.0)) - dv[r] * dv[k]);
    }
  }
  for (int c = 0; c < 2; ++c) {
    const int b = m.frameBody[3 * c];
    const DV3 pf = B[b].p + B[b].R * dc3(m.frameP[3 * c]);
    const DV3 Fe{u[6 * c], u[6 * c + 1], u[6 * c + 2]}, Me{u[6 * c + 3], u[6 * c + 4], u[6 * c + 5]};
    F[b] = F[b] - Fe;
    Mo[b] = Mo[b] - (Me + dcross(pf, Fe));
  }
  for (int i = NB - 1; i >= 1; --i) {
    out[5 + i] = ddot(B[i].ax, Mo[i] - dcross(B[i].p, F[i]));
    F[m.parent[i]] = F[m.parent[i]] + F[i];
    Mo[m.parent[i]] = Mo[m.parent[i]] + Mo[i];
  }
  out[0] = F[0].x;
  out[1] = F[0].y;
  out[2] = F[0].z;
  const DV3 nb = dtr3(S) * (dtr3(B[0].R) * (Mo[0] - dcross(B[0].p, F[0])));
  out[3] = nb.x;
  out[4] = nb.y;
  out[5] = nb.z;
  if (Mang) *Mang = dtr3(S) * (dtr3(B[0].R) * Ic * B[0].R) * S;
}

// wbJointTorques (wb_torque.cuh) along tangent direction dir of z = (x, u): tau[j].v the torques, tau[j].d their derivative
HD void jtTorquesTangent(const WbDeviceModel& m, const double* x, const double* u, int dir, D1* tau) {
  D1 xs[NX], us[NU], g[NV], qddb[6];
  for (int i = 0; i < NX; ++i) xs[i] = dmk(x[i], i == dir ? 1.0 : 0.0);
  for (int i = 0; i < NU; ++i) us[i] = dmk(u[i], NX + i == dir ? 1.0 : 0.0);
  JtBody B[NB];
  DM3 Mang;
  jtInverseDynamics(m, xs, xs + NV, us, nullptr, B, g, &Mang);
  const DM3 Mai = dinv3(Mang);
  const D1 im = dmk(1.0) / dmk(m.mtot);
  for (int k = 0; k < 3; ++k) {
    qddb[k] = -(g[k] * im);
    qddb[3 + k] = -(Mai.m[3 * k] * g[3] + Mai.m[3 * k + 1] * g[4] + Mai.m[3 * k + 2] * g[5]);
  }
  jtInverseDynamics(m, xs, xs + NV, us, qddb, B, g, nullptr);
  for (int j = 0; j < NJ; ++j) tau[j] = g[6 + j];
}

// ---- phases of jt_lq_kernel (Par: any width, any order of the work items) -----------------------------------------------------------------
// J (NJ x NZ, ld NJ) = sqrt(w) .* dtau/dz, one tangent per work item; r (NJ) = sqrt(w) .* tau from direction 0
HD void jtPhaseJacobian(Par P, const WbDeviceModel& m, const JtWeights& w, const double* x, const double* u, double* J, double* r) {
  for (int dir = P.tid; dir < NZ; dir += P.nt) {
    D1 tau[NJ];
    jtTorquesTangent(m, x, u, dir, tau);
    for (int j = 0; j < NJ; ++j) J[j + NJ * dir] = w.sw[j] * tau[j].d;
    if (dir == 0)
      for (int j = 0; j < NJ; ++j) r[j] = w.sw[j] * tau[j].v;
  }
}
// the residual in the projected inputs: A = [Ax | Au] (NJ x (NX + nut), ld NJ), v = Ju u0.  Pu (ld NU), Px (ld NU), u0: the node's projection.
HD void jtPhaseProject(Par P, int nut, const double* J, const double* Pu, const double* Px, const double* u0, double* A, double* v) {
  const double* Ju = J + NJ * NX;
  for (int it = P.tid; it < NJ * (NX + nut + 1); it += P.nt) {
    const int j = it % NJ, c = it / NJ;
    const double* col = c < NX ? Px + NU * c : (c < NX + nut ? Pu + NU * (c - NX) : u0);
    double s = c < NX ? J[j + NJ * c] : 0.0;
    for (int i = 0; i < NU; ++i) s = fma(Ju[j + NJ * i], col[i], s);
    if (c < NX + nut) A[j + NJ * c] = s;
    else v[j] = s;
  }
}
// Sum_j L[j, a] R[j, b] (ld NJ) in a fixed order
HD double jtDot(const double* L, int a, const double* R, int b) {
  double s = 0.0;
  for (int j = 0; j < NJ; ++j) s = fma(L[j + NJ * a], R[j + NJ * b], s);
  return s;
}
HD double jtDotVec(const double* L, int a, const double* r, const double* v) {
  double s = 0.0;
  for (int j = 0; j < NJ; ++j) s = fma(L[j + NJ * a], v ? r[j] + v[j] : r[j], s);
  return s;
}
// adds the projected term to the node's QP blocks (Q ld NX, St / Rt ld NUT_MAX) and its performance-index entries
HD void jtPhaseAccumulate(Par P, int nut, double dt, const double* A, const double* r, const double* v, double* Q, double* St, double* Rt,
                          double* q, double* rt, double* perf) {
  const int nQ = NX * NX, nS = nut * NX, nR = nut * nut;
  for (int it = P.tid; it < nQ + nS + nR + NX + nut + 1; it += P.nt) {
    if (it < nQ) {
      Q[it] += dt * jtDot(A, it % NX, A, it / NX);
    } else if (it < nQ + nS) {
      const int e = it - nQ, l = e % nut, c = e / nut;
      St[l + NUT_MAX * c] += dt * jtDot(A, NX + l, A, c);
    } else if (it < nQ + nS + nR) {
      const int e = it - nQ - nS, l = e % nut, c = e / nut;
      Rt[l + NUT_MAX * c] += dt * jtDot(A, NX + l, A, NX + c);
    } else if (it < nQ + nS + nR + NX) {
      const int a = it - nQ - nS - nR;
      q[a] += dt * jtDotVec(A, a, r, v);
    } else if (it < nQ + nS + nR + NX + nut) {
      const int l = it - nQ - nS - nR - NX;
      rt[l] += dt * jtDotVec(A, NX + l, r, v);
    } else {
      double rr = 0.0, rv = 0.0, vv = 0.0;
      for (int j = 0; j < NJ; ++j) {
        rr = fma(r[j], r[j], rr);
        rv = fma(r[j], v[j], rv);
        vv = fma(v[j], v[j], vv);
      }
      perf[0] += dt * 0.5 * rr;
      perf[3] += dt * (rv + 0.5 * vv);
    }
  }
}
// adds the raw (pre-projection) term to the optional raw block dump (oracle layout, wb_lq.cuh pjPhaseRawA): Q, S (ld NU), R, q, r, c
HD void jtPhaseRaw(Par P, double dt, const double* J, const double* r, double* raw) {
  double* Q = raw + NX * NZ + NX;
  double* S = Q + NX * NX;
  double* R = S + NU * NX;
  double* q = R + NU * NU;
  double* rr = q + NX;
  double* c = rr + NU;
  for (int it = P.tid; it < NZ * NZ - NX * NU + NZ + 1; it += P.nt) {
    if (it < NX * NX) {
      Q[it] += dt * jtDot(J, it % NX, J, it / NX);
    } else if (it < NX * NX + NU * NX) {
      const int e = it - NX * NX;
      S[e] += dt * jtDot(J, NX + e % NU, J, e / NU);
    } else if (it < NX * NX + NU * NX + NU * NU) {
      const int e = it - NX * NX - NU * NX;
      R[e] += dt * jtDot(J, NX + e % NU, J, NX + e / NU);
    } else if (it < NX * NX + NU * NX + NU * NU + NZ) {
      const int a = it - NX * NX - NU * NX - NU * NU;
      (a < NX ? q[a] : rr[a - NX]) += dt * jtDotVec(J, a, r, nullptr);
    } else {
      double s = 0.0;
      for (int j = 0; j < NJ; ++j) s = fma(r[j], r[j], s);
      c[0] += dt * 0.5 * s;
    }
  }
}
// value of the term at (x, u), before dt: 1/2 |sqrt(w) .* tau|^2
HD double jtCostValue(const WbDeviceModel& m, const JtWeights& w, const double* x, const double* u) {
  double tau[NJ], s = 0.0;
  wbJointTorques(m, x, u, tau, nullptr);
  for (int j = 0; j < NJ; ++j) {
    const double r = w.sw[j] * tau[j];
    s = fma(r, r, s);
  }
  return 0.5 * s;
}

#ifdef __CUDACC__
// after K1b (lq_proj_kernel), before prep_kernel: one CTA per (instance, stage), intermediate nodes only
__global__ void __launch_bounds__(JT_THREADS) jt_lq_kernel(WbDev d, JtWeights w) {
  const int k = blockIdx.x, b = blockIdx.y;
  if (d.flags[b * F_NF + F_CONVERGED]) return;
  const size_t node = static_cast<size_t>(b) * (d.N + 1) + k, stage = static_cast<size_t>(b) * d.N + k;
  if (d.event[node] == 1) return;
  __shared__ double J[NJ * NZ], A[NJ * (NX + NUT_MAX)], r[NJ], v[NJ];
  const WbDeviceModel& m = d.instModel[static_cast<size_t>(b) * d.modelStride];
  const double dt = d.mid[stage * Mid::SIZE + Mid::META + 3];
  const Par P{static_cast<int>(threadIdx.x), static_cast<int>(blockDim.x)};
  const NodeOut out = nodeOut(d, node, stage);
  const int nut = *out.nut;
  jtPhaseJacobian(P, m, w, d.x + node * NX, d.u + stage * NU, J, r);
  __syncthreads();
  if (out.raw) jtPhaseRaw(P, dt, J, r, out.raw);
  jtPhaseProject(P, nut, J, out.Pu, out.Px, out.u0, A, v);
  __syncthreads();
  jtPhaseAccumulate(P, nut, dt, A, r, v, out.Q, out.St, out.Rt, out.q, out.rt, out.perf);
}

// after each K3 trial (rollout_kernel): one thread per (instance, stage); adds the term to the trial cost of the intermediate nodes of every
// instance that still searches (the instances K3 evaluated)
__global__ void __launch_bounds__(64) jt_trial_kernel(WbDev d, JtWeights w) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (k >= d.N || (d.flags[b * F_NF + F_CONVERGED] | d.flags[b * F_NF + F_LSDONE])) return;
  const size_t node = static_cast<size_t>(b) * (d.N + 1) + k, stage = static_cast<size_t>(b) * d.N + k;
  if (d.event[node] == 1) return;
  NodeIn n;
  loadNode(d, b, k, n);
  const double alpha = d.inst[b * I_ND + I_ALPHA];
  double xa[NX], ua[NU];
  for (int i = 0; i < NX; ++i) xa[i] = fma(alpha, d.qp.dx[node * NX + i], d.x[node * NX + i]);
  for (int i = 0; i < NU; ++i) ua[i] = fma(alpha, d.du[stage * NU + i], d.u[stage * NU + i]);
  d.lsNode[node * 4] += n.dt * jtCostValue(d.instModel[static_cast<size_t>(b) * d.modelStride], w, xa, ua);
}
#endif

}  // namespace b200sqp
