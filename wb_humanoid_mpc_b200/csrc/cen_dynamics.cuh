// Centroidal flow map of the humanoid centroidal MPC and its Jacobians (SURVEY.md section 8 row a8c), batched over instances.
//
// Reference path: PinocchioCentroidalDynamicsAD::getValueCppAd (ocs2_centroidal_model/src/PinocchioCentroidalDynamicsAD.cpp:75-94) =
//   updateCentroidalDynamics -> pinocchio::computeCentroidalMap (Ag, com)            (ModelHelperFunctions.cpp:46-58)
//   getNormalizedCentroidalMomentumRate                                               (ModelHelperFunctions.cpp:167-194)
//   CentroidalModelPinocchioMapping::getPinocchioJointVelocity with the block inverse (CentroidalModelPinocchioMapping.cpp:84-107,
//                                                                                      implementation/ModelHelperFunctionsImpl.h:40-47)
// differentiated by CppAD in the reference.  Layout: x = [h/m (lin 3, ang 3); base position 3; Euler ZYX 3; joints nj],
// u = [wrench_l (f, tau); wrench_r; qdot_j].
//
// Own formulation (not a port of Pinocchio): world axes, positions measured from the base position (the map is invariant to it), so that
// column k of the centroidal momentum matrix is a closed form of the composite of the subtree moved by coordinate k -- mass M, first moment
// mu = sum m c, second moment about the base position J = sum (Ic + m (|c|^2 1 - c c')) -- for a unit rotation w about an axis through p:
//   h_lin = w x (mu - M p),   L_O = J w - mu x (w x p),   L_G = L_O - G x h_lin      (translations: h_lin = m e_k, L_G = 0)
// One warp per instance: lane 0 evaluates the value and the analytic columns (the map is affine in hbar, the wrenches and qdot_j and
// invariant to the base position), lanes 1..26 each carry one tangent (3 Euler angles + 23 joints) through the same code as a
// single-tangent dual, i.e. all lanes run one instruction stream.
#pragma once
#include "wb_model.cuh"

namespace b200sqp {

constexpr int CEN_NX = 12 + NJ, CEN_NU = 12 + NJ;

struct CenModel {  // subset of b200sqp_model_desc the flow map reads
  int parent[NB];
  double jR[NB][9], jp[NB][3], axis[NB][3], mass[NB], com[NB][3], Icom[NB][9];
  double mtot;
  int contactBody[2];
  double contactP[2][3];
  // CentroidalModelInfo::centroidalModelType (0 full centroidal dynamics, 1 single rigid body) with the nominal inertia / com offset of the
  // latter; read by cenKinematics (cen_ocp.cuh).  cen_flow_kernel below always evaluates the full model.
  int modelType;
  double inertiaNominal[9], comToBaseNominal[3];
};

struct CenEval {      // what one lane produces
  D1 xdot[CEN_NX];
  D1 Ab22i[9], Ab12[9];   // blocks of the floating-base momentum matrix (value lane: analytic columns)
  D1 Aj[6][NJ];
  D1 r[2][3];             // com -> contact point
};

// the flow map with one tangent seeded on generalized coordinate `dir` (0..28; < 0: none)
HD void cenFlowDual(const CenModel& m, const double* x, const double* u, int dir, CenEval& e) {
  D1 q[NV];
#pragma unroll 1
  for (int i = 0; i < NV; ++i) q[i] = D1{x[6 + i], i == dir ? 1.0 : 0.0};
  // ---- world-frame kinematics and body composites -----------------------------------------------------------------------------------
  DM3 R[NB];
  DV3 p[NB], ax[NB];
  D1 M[NB];
  DV3 mu[NB];
  D1 J[NB][6];   // symmetric: xx xy xz yy yz zz
  {
    const D1 c0 = dcos(q[3]), s0 = dsin(q[3]), c1 = dcos(q[4]), s1 = dsin(q[4]), c2 = dcos(q[5]), s2 = dsin(q[5]);
    R[0].m[0] = c0 * c1; R[0].m[1] = c0 * s1 * s2 - s0 * c2; R[0].m[2] = c0 * s1 * c2 + s0 * s2;
    R[0].m[3] = s0 * c1; R[0].m[4] = s0 * s1 * s2 + c0 * c2; R[0].m[5] = s0 * s1 * c2 - c0 * s2;
    R[0].m[6] = -s1;     R[0].m[7] = c1 * s2;                R[0].m[8] = c1 * c2;
    // positions are measured from the base position: the map is invariant to it, and second moments J about a distant world origin would
    // cancel digits in L_G (a base 1 km out lost 7 of them)
    p[0] = dconst(0, 0, 0);
    ax[0] = dconst(0, 0, 0);
  }
#pragma unroll 1
  for (int i = 1; i < NB; ++i) {
    const int pa = m.parent[i];
    const double* a = m.axis[i];
    const D1 c = dcos(q[5 + i]), s = dsin(q[5 + i]), t = dmk(1.0) - c;
    DM3 Rq, Rj;
    Rq.m[0] = t * (a[0] * a[0]) + c;        Rq.m[1] = t * (a[0] * a[1]) - s * a[2]; Rq.m[2] = t * (a[0] * a[2]) + s * a[1];
    Rq.m[3] = t * (a[0] * a[1]) + s * a[2]; Rq.m[4] = t * (a[1] * a[1]) + c;        Rq.m[5] = t * (a[1] * a[2]) - s * a[0];
    Rq.m[6] = t * (a[0] * a[2]) - s * a[1]; Rq.m[7] = t * (a[1] * a[2]) + s * a[0]; Rq.m[8] = t * (a[2] * a[2]) + c;
#pragma unroll
    for (int k = 0; k < 9; ++k) Rj.m[k] = dmk(m.jR[i][k]);
    R[i] = R[pa] * (Rj * Rq);
    p[i] = p[pa] + R[pa] * dconst(m.jp[i][0], m.jp[i][1], m.jp[i][2]);
    ax[i] = R[i] * dconst(a[0], a[1], a[2]);
  }
#pragma unroll 1
  for (int i = 0; i < NB; ++i) {
    const DV3 c = p[i] + R[i] * dconst(m.com[i][0], m.com[i][1], m.com[i][2]);
    DM3 Ib, Rt;
#pragma unroll
    for (int k = 0; k < 9; ++k) Ib.m[k] = dmk(m.Icom[i][k]);
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int k = 0; k < 3; ++k) Rt.m[3 * r + k] = R[i].m[3 * k + r];
    const DM3 Iw = R[i] * (Ib * Rt);
    const double ms = m.mass[i];
    const D1 cc = ddot(c, c);
    M[i] = dmk(ms);
    mu[i] = ms * c;
    J[i][0] = Iw.m[0] + ms * (cc - c.x * c.x);
    J[i][1] = Iw.m[1] - ms * (c.x * c.y);
    J[i][2] = Iw.m[2] - ms * (c.x * c.z);
    J[i][3] = Iw.m[4] + ms * (cc - c.y * c.y);
    J[i][4] = Iw.m[5] - ms * (c.y * c.z);
    J[i][5] = Iw.m[8] + ms * (cc - c.z * c.z);
  }
#pragma unroll 1
  for (int i = NB - 1; i >= 1; --i) {   // subtree composites: children are numbered after their parents
    const int pa = m.parent[i];
    M[pa] = M[pa] + M[i];
    mu[pa] = mu[pa] + mu[i];
#pragma unroll
    for (int k = 0; k < 6; ++k) J[pa][k] = J[pa][k] + J[i][k];
  }
  const D1 mass = M[0];
  const DV3 G = (dmk(1.0) / mass) * mu[0];
  // ---- centroidal momentum matrix: columns 3..28 (the translation columns are [m 1; 0]) -------------------------------------------------------
  D1 Ag[6][NV - 3];
  const D1 c1 = dcos(q[4]), s1 = dsin(q[4]), c2 = dcos(q[5]), s2 = dsin(q[5]);
  const DV3 Scol[3] = {DV3{-s1, c1 * s2, c1 * c2}, DV3{dmk(0.0), c2, -s2}, DV3{dmk(1.0), dmk(0.0), dmk(0.0)}};   // columns of the ZYX subspace
#pragma unroll 1
  for (int k = 3; k < NV; ++k) {
    const int b = (k < 6) ? 0 : k - 5;
    const DV3 w = (k < 6) ? R[0] * Scol[k - 3] : ax[b];
    const DV3 hl = dcross(w, mu[b] - M[b] * p[b]);
    const D1* Jb = J[b];
    const DV3 Jw{Jb[0] * w.x + Jb[1] * w.y + Jb[2] * w.z, Jb[1] * w.x + Jb[3] * w.y + Jb[4] * w.z, Jb[2] * w.x + Jb[4] * w.y + Jb[5] * w.z};
    const DV3 LG = Jw - dcross(mu[b], dcross(w, p[b])) - dcross(G, hl);
    Ag[0][k - 3] = hl.x; Ag[1][k - 3] = hl.y; Ag[2][k - 3] = hl.z;
    Ag[3][k - 3] = LG.x; Ag[4][k - 3] = LG.y; Ag[5][k - 3] = LG.z;
  }
  // ---- normalized momentum rate ----------------------------------------------------------------------------------------------------------
  DV3 lin = DV3{dmk(0.0), dmk(0.0), dmk(-9.81) * mass}, ang = dconst(0, 0, 0);
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    const int b = m.contactBody[c];
    const DV3 r = p[b] + R[b] * dconst(m.contactP[c][0], m.contactP[c][1], m.contactP[c][2]) - G;
    const DV3 F = dconst(u[6 * c], u[6 * c + 1], u[6 * c + 2]), T = dconst(u[6 * c + 3], u[6 * c + 4], u[6 * c + 5]);
    lin = lin + F;
    ang = ang + dcross(r, F) + T;
    e.r[c][0] = r.x; e.r[c][1] = r.y; e.r[c][2] = r.z;
  }
  const D1 im = dmk(1.0) / mass;
  e.xdot[0] = im * lin.x; e.xdot[1] = im * lin.y; e.xdot[2] = im * lin.z;
  e.xdot[3] = im * ang.x; e.xdot[4] = im * ang.y; e.xdot[5] = im * ang.z;
  // ---- generalized velocity: v_b = Ab^-1 (m hbar - Aj qdot_j) with the block inverse; qdot_j from the input -------------------------------
  D1 mom[6];
#pragma unroll 1
  for (int r = 0; r < 6; ++r) {
    D1 s = mass * x[r];
    for (int j = 0; j < NJ; ++j) {
      s = s - Ag[r][3 + j] * u[12 + j];
      e.Aj[r][j] = Ag[r][3 + j];
    }
    mom[r] = s;
  }
  DM3 Ab22, Ab12;
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      Ab22.m[3 * r + k] = Ag[3 + r][k];
      Ab12.m[3 * r + k] = Ag[r][k];
    }
  const DM3 Ab22i = dinv3(Ab22);
  const DV3 wb = Ab22i * DV3{mom[3], mom[4], mom[5]};
  const DV3 t = Ab12 * wb;
  e.xdot[6] = im * mom[0] - im * t.x;
  e.xdot[7] = im * mom[1] - im * t.y;
  e.xdot[8] = im * mom[2] - im * t.z;
  e.xdot[9] = wb.x; e.xdot[10] = wb.y; e.xdot[11] = wb.z;
  for (int j = 0; j < NJ; ++j) e.xdot[12 + j] = dmk(u[12 + j]);
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    e.Ab22i[k] = Ab22i.m[k];
    e.Ab12[k] = Ab12.m[k];
  }
}

// One warp per instance.  xdot [B][35]; dfdx [B][35*35], dfdu [B][35*35] column-major (either may be null).
__global__ void __launch_bounds__(32) cen_flow_kernel(CenModel m, int batch, const double* __restrict__ x, const double* __restrict__ u,
                                                      double* __restrict__ xdot, double* __restrict__ dfdx, double* __restrict__ dfdu) {
  const int b = blockIdx.x, lane = threadIdx.x;
  if (b >= batch) return;
  const bool deriv = dfdx != nullptr || dfdu != nullptr;
  if (lane > 26 || (!deriv && lane > 0)) return;
  const double* xb = x + static_cast<size_t>(b) * CEN_NX;
  const double* ub = u + static_cast<size_t>(b) * CEN_NU;
  CenEval e;
  cenFlowDual(m, xb, ub, lane == 0 ? -1 : 2 + lane, e);   // lanes 1..26 -> generalized coordinates 3..28
  constexpr int NXc = CEN_NX, NUc = CEN_NU;
  if (lane == 0) {
    for (int i = 0; i < NXc; ++i) xdot[static_cast<size_t>(b) * NXc + i] = e.xdot[i].v;
    const double mass = m.mtot, im = 1.0 / mass;
    if (dfdx) {
      double* A = dfdx + static_cast<size_t>(b) * NXc * NXc;
      // columns hbar (0..5): d v_b / d hbar = m Ab^-1 ; base position (6..8): translation invariance
      for (int j = 0; j < 9; ++j)
        for (int i = 0; i < NXc; ++i) A[i + NXc * j] = 0.0;
      for (int k = 0; k < 3; ++k) {
        A[(6 + k) + NXc * k] = 1.0;   // (1/m) * m
        for (int r = 0; r < 3; ++r) {
          double t = 0.0;             // -(1/m) Ab12 Ab22^-1 * m
          for (int s = 0; s < 3; ++s) t -= e.Ab12[3 * r + s].v * e.Ab22i[3 * s + k].v;
          A[(6 + r) + NXc * (3 + k)] = t;
          A[(9 + r) + NXc * (3 + k)] = mass * e.Ab22i[3 * r + k].v;
        }
      }
    }
    if (dfdu) {
      double* Bm = dfdu + static_cast<size_t>(b) * NXc * NUc;
      for (int j = 0; j < NUc; ++j)
        for (int i = 0; i < NXc; ++i) Bm[i + NXc * j] = 0.0;
      for (int c = 0; c < 2; ++c) {
        const double r[3] = {e.r[c][0].v, e.r[c][1].v, e.r[c][2].v};
        const double rx[9] = {0, -r[2], r[1], r[2], 0, -r[0], -r[1], r[0], 0};
        for (int k = 0; k < 3; ++k) {
          Bm[k + NXc * (6 * c + k)] = im;                                             // d hbar_lin / d F
          for (int i = 0; i < 3; ++i) Bm[(3 + i) + NXc * (6 * c + k)] = im * rx[3 * i + k];   // d hbar_ang / d F = [r]x / m
          Bm[(3 + k) + NXc * (6 * c + 3 + k)] = im;                                   // d hbar_ang / d tau
        }
      }
      // d v_b / d qdot_j = -Ab^-1 Aj ; d qdot_j / d qdot_j = 1
      for (int j = 0; j < NJ; ++j) {
        double w[3], t[3];
        for (int r = 0; r < 3; ++r) w[r] = -(e.Ab22i[3 * r].v * e.Aj[3][j].v + e.Ab22i[3 * r + 1].v * e.Aj[4][j].v + e.Ab22i[3 * r + 2].v * e.Aj[5][j].v);
        for (int r = 0; r < 3; ++r) t[r] = e.Ab12[3 * r].v * w[0] + e.Ab12[3 * r + 1].v * w[1] + e.Ab12[3 * r + 2].v * w[2];
        for (int r = 0; r < 3; ++r) {
          Bm[(6 + r) + NXc * (12 + j)] = -im * e.Aj[r][j].v - im * t[r];
          Bm[(9 + r) + NXc * (12 + j)] = w[r];
        }
        Bm[(12 + j) + NXc * (12 + j)] = 1.0;
      }
    }
  } else if (dfdx) {
    double* A = dfdx + static_cast<size_t>(b) * NXc * NXc + static_cast<size_t>(NXc) * (8 + lane);   // state column 6 + (2 + lane)
    for (int i = 0; i < NXc; ++i) A[i] = e.xdot[i].d;
  }
}

}  // namespace b200sqp
