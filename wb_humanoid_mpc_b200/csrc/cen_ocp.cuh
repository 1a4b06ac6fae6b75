// LQ approximation of one shooting node of the humanoid CENTROIDAL OCP (BASELINE configs 0-1), device side.
//
// Reference: CentroidalMpcInterface::setupOptimalControlProblem (humanoid_nmpc/humanoid_centroidal_mpc/src/CentroidalMpcInterface.cpp:150-237)
// wires the terms below; every one of them obtains its derivatives from CppAD in the reference.  Term sources:
//   dynamics + RK4 sensitivity   cen_dynamics.cuh; ocs2_core/src/integration/SensitivityIntegratorImpl.cpp:130-169
//   quadratic tracking           humanoid_common_mpc/src/cost/StateInputQuadraticCost.cpp:67-78, SwitchedModelReferenceManager.cpp:110-135
//   task-space link cost         humanoid_common_mpc/src/cost/EndEffectorKinematicsQuadraticCost.cpp:76-128 (quaternionDistance / matrixToQuaternion:
//                                ocs2_robotic_tools/common/RotationTransforms.h:51-53,215-245)
//   ICP cost                     humanoid_centroidal_mpc/src/cost/ICPCost.cpp:78-108
//   foot tracking cost           humanoid_centroidal_mpc/src/cost/CentroidalMpcEndEffectorFootCost.cpp:91-147
//   external torque cost         humanoid_common_mpc/src/cost/ExternalTorqueQuadraticCostAD.cpp:84-131
//   joint limits / collision     humanoid_common_mpc/src/constraint/JointLimitsSoftConstraint.cpp:69-100, FootCollisionConstraint.cpp:80-144
//   friction cone / moment XY    humanoid_common_mpc/src/constraint/FrictionForceConeConstraint.cpp:80-224, ContactMomentXYConstraintCppAd.cpp:86-104
//   zero wrench                  humanoid_common_mpc/src/constraint/ZeroWrenchConstraint.cpp:59-84
//   zero velocity (stance)       humanoid_common_mpc/src/constraint/EndEffectorKinematicsTwistConstraint.cpp:79-131, CentroidalMpcInterface.cpp:246-268
//   normal velocity (swing)      humanoid_common_mpc/src/constraint/EndEffectorKinematicsLinearVelConstraint.cpp:71-111, HumanoidPreComputation.cpp:100-121
//
// Own formulation: forward-mode differentiation in SIMT form.  One CTA per node; thread t < 70 carries tangent direction t (x_0..x_34,
// u_0..u_34) as a single-tangent dual through the WHOLE node -- the four RK4 stages (so its x+ dual is column t of [A | B], no chain-rule
// GEMMs), the constraint rows and the Gauss-Newton residual rows -- in world-frame closed-form kinematics (cen_dynamics.cuh).  All threads
// execute one instruction stream; the only exchanges are the Jacobian rows gathered in shared memory for the Hessian J'J.  This is the
// correctness-first version of the centroidal path (configs 0-1 are single-instance correctness configurations): it spends ~70x redundant
// value arithmetic, which a later revision can remove by splitting the tangents by structure as cen_flow_kernel already does.
#pragma once
#include "cen_dynamics.cuh"
#include "wb_lq.cuh"

namespace b200sqp {

constexpr int CNX = CEN_NX, CNU = CEN_NU, CNZ = CEN_NX + CEN_NU;  // 35, 35, 70
constexpr int CEN_NFRAMES = NFRAMES + 1;                          // the whole-body frame table + the task-space link
constexpr int CEN_MAX_RES = 12 + 2 + 2 * 12 + 2 * 6;              // Gauss-Newton residual rows: torso, ICP, 2 x foot, 2 x external torque
constexpr int CEN_PEN_ROWS = 8 + 16;                              // first-order penalty rows: 2 x 4 contact moment, 16 collision distances
constexpr int CEN_ROWS = CEN_MAX_RES + CEN_PEN_ROWS;              // 74
constexpr int CEN_THREADS = 96;

struct CenOcpModel {
  CenModel kin;
  int frameBody[CEN_NFRAMES];
  double frameP[CEN_NFRAMES][3];
  int torsoFrame;
  double torsoR[9], torsoSqrtW[12], icpSqrtW;
  int tqJoint[2][6];
  double tqSqrtW[2][6];
  double Qd[CNX], Rd[CNU], Qfd[CNX];
  double gPosZ, gOri, footSqrtW[12];
  double fricCoeff, fricMu, fricDelta, fricReg, fricShift, momMu, momDelta, jlMu, jlDelta, collMu, collDelta, rFoot, rKnee;
  double rect[4];
  int armJoint[4];
  double qlo[NJ], qhi[NJ];
};

// ---- kinematics on duals: world placements, subtree composites, centroidal momentum matrix ----------------------------------------------------
struct CenKin {
  DM3 R[NB];
  DV3 p[NB], ax[NB];
  D1 M[NB];
  DV3 mu[NB];
  D1 J[NB][6];
  DV3 G, Sw[3];      // centre of mass as the dynamics see it (data.com[0]); world axes of the three Euler-rate columns
  DV3 Gcom;          // pinocchio::centerOfMass(q) (= G for the full model; the SRBD model carries a nominal offset in G instead)
  D1 mass;
  D1 Ag[6][NV - 3];  // columns 3..28 (translation columns are [m 1; 0])
};

HD void cenKinematics(const CenModel& m, const D1* q, CenKin& k) {
  // placements are formed relative to the base position and moved to the world at the end: the subtree second moments J are taken about the
  // base, so that a base far from the world origin (|c|^2 of 1e6 m^2 at 1 km) does not cancel digits in the centroidal momentum matrix
  const DV3 base{q[0], q[1], q[2]};
  {
    const D1 c0 = dcos(q[3]), s0 = dsin(q[3]), c1 = dcos(q[4]), s1 = dsin(q[4]), c2 = dcos(q[5]), s2 = dsin(q[5]);
    k.R[0].m[0] = c0 * c1; k.R[0].m[1] = c0 * s1 * s2 - s0 * c2; k.R[0].m[2] = c0 * s1 * c2 + s0 * s2;
    k.R[0].m[3] = s0 * c1; k.R[0].m[4] = s0 * s1 * s2 + c0 * c2; k.R[0].m[5] = s0 * s1 * c2 - c0 * s2;
    k.R[0].m[6] = -s1;     k.R[0].m[7] = c1 * s2;                k.R[0].m[8] = c1 * c2;
    k.p[0] = dconst(0, 0, 0);
    k.ax[0] = dconst(0, 0, 0);
    const DV3 Scol[3] = {DV3{-s1, c1 * s2, c1 * c2}, DV3{dmk(0.0), c2, -s2}, DV3{dmk(1.0), dmk(0.0), dmk(0.0)}};
    for (int e = 0; e < 3; ++e) k.Sw[e] = k.R[0] * Scol[e];
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
    for (int e = 0; e < 9; ++e) Rj.m[e] = dmk(m.jR[i][e]);
    k.R[i] = k.R[pa] * (Rj * Rq);
    k.p[i] = k.p[pa] + k.R[pa] * dconst(m.jp[i][0], m.jp[i][1], m.jp[i][2]);
    k.ax[i] = k.R[i] * dconst(a[0], a[1], a[2]);
  }
  if (m.modelType == 1) {
#pragma unroll 1
    for (int i = 0; i < NB; ++i) k.p[i] = k.p[i] + base;
    // updateCentroidalDynamics, SingleRigidBodyDynamics branch (ocs2_centroidal_model/src/ModelHelperFunctions.cpp:61-79): Ag = [Ab 0] from the
    // nominal centroidal inertia and com offset carried with the base; the frame placements above still follow the full kinematics
    const DV3 rw = k.R[0] * dconst(m.comToBaseNominal[0], m.comToBaseNominal[1], m.comToBaseNominal[2]);
    DM3 In, Rt;
#pragma unroll
    for (int e = 0; e < 9; ++e) In.m[e] = dmk(m.inertiaNominal[e]);
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int e = 0; e < 3; ++e) Rt.m[3 * r + e] = k.R[0].m[3 * e + r];
    const DM3 Iw = (k.R[0] * In) * Rt;
    k.mass = dmk(m.mtot);
    k.G = k.p[0] - rw;
    DV3 mu = dconst(0, 0, 0);
    for (int i = 0; i < NB; ++i) mu = mu + m.mass[i] * (k.p[i] + k.R[i] * dconst(m.com[i][0], m.com[i][1], m.com[i][2]));
    k.Gcom = (1.0 / m.mtot) * mu;
    for (int c = 3; c < NV; ++c)
      for (int r = 0; r < 6; ++r) k.Ag[r][c - 3] = dmk(0.0);
    for (int e = 0; e < 3; ++e) {
      const DV3 hl = m.mtot * dcross(rw, k.Sw[e]);
      const DV3 LG = Iw * k.Sw[e];
      k.Ag[0][e] = hl.x; k.Ag[1][e] = hl.y; k.Ag[2][e] = hl.z;
      k.Ag[3][e] = LG.x; k.Ag[4][e] = LG.y; k.Ag[5][e] = LG.z;
    }
    return;
  }
#pragma unroll 1
  for (int i = 0; i < NB; ++i) {
    const DV3 c = k.p[i] + k.R[i] * dconst(m.com[i][0], m.com[i][1], m.com[i][2]);
    DM3 Ib, Rt;
#pragma unroll
    for (int e = 0; e < 9; ++e) Ib.m[e] = dmk(m.Icom[i][e]);
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int e = 0; e < 3; ++e) Rt.m[3 * r + e] = k.R[i].m[3 * e + r];
    const DM3 Iw = k.R[i] * (Ib * Rt);
    const double ms = m.mass[i];
    const D1 cc = ddot(c, c);
    k.M[i] = dmk(ms);
    k.mu[i] = ms * c;
    k.J[i][0] = Iw.m[0] + ms * (cc - c.x * c.x);
    k.J[i][1] = Iw.m[1] - ms * (c.x * c.y);
    k.J[i][2] = Iw.m[2] - ms * (c.x * c.z);
    k.J[i][3] = Iw.m[4] + ms * (cc - c.y * c.y);
    k.J[i][4] = Iw.m[5] - ms * (c.y * c.z);
    k.J[i][5] = Iw.m[8] + ms * (cc - c.z * c.z);
  }
#pragma unroll 1
  for (int i = NB - 1; i >= 1; --i) {
    const int pa = m.parent[i];
    k.M[pa] = k.M[pa] + k.M[i];
    k.mu[pa] = k.mu[pa] + k.mu[i];
#pragma unroll
    for (int e = 0; e < 6; ++e) k.J[pa][e] = k.J[pa][e] + k.J[i][e];
  }
  k.mass = k.M[0];
  const DV3 Grel = (dmk(1.0) / k.mass) * k.mu[0];
#pragma unroll 1
  for (int c = 3; c < NV; ++c) {
    const int b = (c < 6) ? 0 : c - 5;
    const DV3 w = (c < 6) ? k.Sw[c - 3] : k.ax[b];
    const DV3 hl = dcross(w, k.mu[b] - k.M[b] * k.p[b]);
    const D1* Jb = k.J[b];
    const DV3 Jw{Jb[0] * w.x + Jb[1] * w.y + Jb[2] * w.z, Jb[1] * w.x + Jb[3] * w.y + Jb[4] * w.z, Jb[2] * w.x + Jb[4] * w.y + Jb[5] * w.z};
    const DV3 LG = Jw - dcross(k.mu[b], dcross(w, k.p[b])) - dcross(Grel, hl);
    k.Ag[0][c - 3] = hl.x; k.Ag[1][c - 3] = hl.y; k.Ag[2][c - 3] = hl.z;
    k.Ag[3][c - 3] = LG.x; k.Ag[4][c - 3] = LG.y; k.Ag[5][c - 3] = LG.z;
  }
  // world placements and centre of mass (mu and J stay about the base: nothing after this reads them)
#pragma unroll 1
  for (int i = 0; i < NB; ++i) k.p[i] = k.p[i] + base;
  k.G = Grel + base;
  k.Gcom = k.G;
}

// flow map on duals given the kinematics of q = x[6..35)
HD void cenFlowFromKin(const CenModel& m, const CenKin& k, const D1* x, const D1* u, D1* xdot) {
  DV3 lin = DV3{dmk(0.0), dmk(0.0), dmk(-9.81) * k.mass}, ang = dconst(0, 0, 0);
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    const int b = m.contactBody[c];
    const DV3 r = k.p[b] + k.R[b] * dconst(m.contactP[c][0], m.contactP[c][1], m.contactP[c][2]) - k.G;
    const DV3 F{u[6 * c], u[6 * c + 1], u[6 * c + 2]}, T{u[6 * c + 3], u[6 * c + 4], u[6 * c + 5]};
    lin = lin + F;
    ang = ang + dcross(r, F) + T;
  }
  const D1 im = dmk(1.0) / k.mass;
  xdot[0] = im * lin.x; xdot[1] = im * lin.y; xdot[2] = im * lin.z;
  xdot[3] = im * ang.x; xdot[4] = im * ang.y; xdot[5] = im * ang.z;
  D1 mom[6];
#pragma unroll 1
  for (int r = 0; r < 6; ++r) {
    D1 s = k.mass * x[r];
    for (int j = 0; j < NJ; ++j) s = s - k.Ag[r][3 + j] * u[12 + j];
    mom[r] = s;
  }
  DM3 Ab22, Ab12;
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int e = 0; e < 3; ++e) {
      Ab22.m[3 * r + e] = k.Ag[3 + r][e];
      Ab12.m[3 * r + e] = k.Ag[r][e];
    }
  const DM3 Ab22i = dinv3(Ab22);
  const DV3 wb = Ab22i * DV3{mom[3], mom[4], mom[5]};
  const DV3 t = Ab12 * wb;
  xdot[6] = im * mom[0] - im * t.x;
  xdot[7] = im * mom[1] - im * t.y;
  xdot[8] = im * mom[2] - im * t.z;
  xdot[9] = wb.x; xdot[10] = wb.y; xdot[11] = wb.z;
  for (int j = 0; j < NJ; ++j) xdot[12 + j] = u[12 + j];
}

// LOCAL_WORLD_ALIGNED velocity of a point pf fixed on `body` for generalized velocity qd (translation, Euler rates, joints)
HD void cenFrameVelocity(const CenModel& m, const CenKin& k, int body, DV3 pf, const D1* qd, DV3& vlin, DV3& vang) {
  vlin = DV3{qd[0], qd[1], qd[2]};
  vang = dconst(0, 0, 0);
#pragma unroll
  for (int e = 0; e < 3; ++e) {
    vang = vang + qd[3 + e] * k.Sw[e];
    vlin = vlin + qd[3 + e] * dcross(k.Sw[e], pf - k.p[0]);
  }
  for (int a = body; a >= 1; a = m.parent[a]) {
    vang = vang + qd[5 + a] * k.ax[a];
    vlin = vlin + qd[5 + a] * dcross(k.ax[a], pf - k.p[a]);
  }
}

// rotationMatrixDistanceToPlane(R, e_z) = -vec(shortest-arc quaternion from R e_z to e_z)   (RotationTransforms.h:98-113,396-405)
HD DV3 cenOriErrToPlane(const DM3& R) {
  const D1 ax = R.m[2], ay = R.m[5], az = R.m[8];
  const D1 cx = ay, cy = -ax;  // a x e_z
  const D1 w = dmk(1.0) + az;
  const D1 nrm = dsqrt(cx * cx + cy * cy + w * w);
  return DV3{-(cx / nrm), -(cy / nrm), dmk(0.0)};
}
// matrixToQuaternion, CppAD flavour: conditional expressions on values (RotationTransforms.h:215-245); q = (x, y, z, w)
HD void cenMatrixToQuaternion(const DM3& R, D1* q) {
  const D1 r00 = R.m[0], r01 = R.m[1], r02 = R.m[2], r10 = R.m[3], r11 = R.m[4], r12 = R.m[5], r20 = R.m[6], r21 = R.m[7], r22 = R.m[8];
  const bool gt = r00.v > r11.v, lt = r00.v < -r11.v, neg = r22.v < 0.0;
  const D1 one = dmk(1.0);
  const D1 t1 = gt ? one + r00 - r11 - r22 : one - r00 + r11 - r22;
  const D1 t2 = lt ? one - r00 - r11 + r22 : one + r00 + r11 + r22;
  const D1 t = neg ? t1 : t2;
  const D1 x1 = gt ? t : r10 + r01, x2 = lt ? r02 + r20 : r21 - r12;
  const D1 y1 = gt ? r10 + r01 : t, y2 = lt ? r21 + r12 : r02 - r20;
  const D1 z1 = gt ? r02 + r20 : r21 + r12, z2 = lt ? t : r10 - r01;
  const D1 w1 = gt ? r21 - r12 : r02 - r20, w2 = lt ? r10 - r01 : t;
  const D1 sc = dmk(0.5) / dsqrt(t);
  q[0] = (neg ? x1 : x2) * sc;
  q[1] = (neg ? y1 : y2) * sc;
  q[2] = (neg ? z1 : z2) * sc;
  q[3] = (neg ? w1 : w2) * sc;
}

struct CenTask {  // task-space quantities at (x, u)
  DV3 footPos[2], footVlin[2], footVang[2], footOri[2];
  DM3 footR[2];
  DV3 torsoPos, torsoVlin, torsoVang;
  D1 torsoQuat[4];
  DV3 framePos[NFRAMES];
};
HD void cenTaskSpace(const CenOcpModel& m, const CenKin& k, const D1* qd, CenTask& t) {
  for (int f = 0; f < NFRAMES; ++f) {
    const int b = m.frameBody[f];
    t.framePos[f] = k.p[b] + k.R[b] * dconst(m.frameP[f][0], m.frameP[f][1], m.frameP[f][2]);
  }
  for (int c = 0; c < 2; ++c) {
    const int b = m.frameBody[3 * c];
    t.footPos[c] = t.framePos[3 * c];
    t.footR[c] = k.R[b];
    t.footOri[c] = cenOriErrToPlane(k.R[b]);
    cenFrameVelocity(m.kin, k, b, t.footPos[c], qd, t.footVlin[c], t.footVang[c]);
  }
  const int tb = m.frameBody[m.torsoFrame];
  t.torsoPos = k.p[tb] + k.R[tb] * dconst(m.frameP[m.torsoFrame][0], m.frameP[m.torsoFrame][1], m.frameP[m.torsoFrame][2]);
  cenFrameVelocity(m.kin, k, tb, t.torsoPos, qd, t.torsoVlin, t.torsoVang);
  DM3 Rf;
#pragma unroll
  for (int e = 0; e < 9; ++e) Rf.m[e] = dmk(m.torsoR[e]);
  cenMatrixToQuaternion(k.R[tb] * Rf, t.torsoQuat);
}

// reference cost element of the task-space link at (xref, u = 0): position 3, quaternion xyzw 4, linear velocity 3, angular velocity 3.
// Value-only; evaluated once per node (EndEffectorKinematicsQuadraticCost::getParameters does the same with the double model).
HD void cenTorsoReference(const CenOcpModel& m, const double* xref, CenKin& k, double* ref) {
  D1 x[CNX], u[CNU], xd[CNX];
  for (int i = 0; i < CNX; ++i) x[i] = dmk(xref[i]);
  for (int i = 0; i < CNU; ++i) u[i] = dmk(0.0);
  cenKinematics(m.kin, x + 6, k);
  cenFlowFromKin(m.kin, k, x, u, xd);
  const int tb = m.frameBody[m.torsoFrame];
  const DV3 pos = k.p[tb] + k.R[tb] * dconst(m.frameP[m.torsoFrame][0], m.frameP[m.torsoFrame][1], m.frameP[m.torsoFrame][2]);
  DV3 vl, va;
  cenFrameVelocity(m.kin, k, tb, pos, xd + 6, vl, va);
  DM3 Rf;
#pragma unroll
  for (int e = 0; e < 9; ++e) Rf.m[e] = dmk(m.torsoR[e]);
  D1 q[4];
  cenMatrixToQuaternion(k.R[tb] * Rf, q);
  ref[0] = pos.x.v; ref[1] = pos.y.v; ref[2] = pos.z.v;
  for (int e = 0; e < 4; ++e) ref[3 + e] = q[e].v;
  ref[7] = vl.x.v; ref[8] = vl.y.v; ref[9] = vl.z.v;
  ref[10] = va.x.v; ref[11] = va.y.v; ref[12] = va.z.v;
}

HD int cenConstraintRows(const NodeIn& n) { return (n.contact[0] ? 6 : 7) + (n.contact[1] ? 6 : 7); }
HD int cenResidualRows(const NodeIn& n) { return 12 + 2 + 24 + 6 * (n.contact[0] + n.contact[1]); }

// Everything one tangent direction contributes to an intermediate node.  dir in [0, 70): seeded variable (x then u); dir < 0: values only.
struct CenDirOut {
  D1 xplus[CNX];       // RK4 image; .d = column dir of [A | B]
  D1 g[NC_MAX];        // state-input equality constraints, collection order: per foot {zeroWrench | zeroVelocity | normalVelocity}
  D1 res[CEN_MAX_RES]; // Gauss-Newton residuals: torso 12, ICP 2, per foot {tracking 12, external torque 6 if stance}
  D1 pen[CEN_PEN_ROWS];  // first-order penalty constraints h: contact moment XY (4 per stance foot, slots 4c..4c+3), collision 16 (slots 8..23)
};

HD void cenNodeDual(const CenOcpModel& m, const NodeIn& n, const double* torsoRef, int dir, CenKin& k, CenDirOut& o) {
  D1 x[CNX], u[CNU], xs[CNX], f[CNX];
  for (int i = 0; i < CNX; ++i) x[i] = D1{n.x[i], dir == i ? 1.0 : 0.0};
  for (int i = 0; i < CNU; ++i) u[i] = D1{n.u[i], dir == CNX + i ? 1.0 : 0.0};
  for (int e = 0; e < CEN_PEN_ROWS; ++e) o.pen[e] = dmk(0.0);   // inactive rows stay exact zeros (their weights are zero too)
  // ---- stage 1 at (x, u): also the linearisation point of every cost / constraint term ----------------------------------------------------------
  cenKinematics(m.kin, x + 6, k);
  cenFlowFromKin(m.kin, k, x, u, f);
  {
    CenTask t;
    cenTaskSpace(m, k, f + 6, t);
    // equality constraints
    int r = 0;
    for (int c = 0; c < 2; ++c) {
      if (!n.contact[c]) {
        for (int e = 0; e < 6; ++e) o.g[r++] = u[6 * c + e];
        const double b = -n.swing[c][1] - m.gPosZ * n.swing[c][0];
        o.g[r++] = dmk(b) + t.footVlin[c].z + m.gPosZ * t.footPos[c].z;
      } else {
        o.g[r++] = t.footVlin[c].x;
        o.g[r++] = t.footVlin[c].y;
        o.g[r++] = t.footVlin[c].z + m.gPosZ * t.footPos[c].z;
        o.g[r++] = t.footVang[c].x + m.gOri * t.footOri[c].x;
        o.g[r++] = t.footVang[c].y + m.gOri * t.footOri[c].y;
        o.g[r++] = t.footVang[c].z + m.gOri * t.footOri[c].z;
      }
    }
    // Gauss-Newton residuals
    r = 0;
    {
      const D1* q = t.torsoQuat;
      const double* qr = torsoRef + 3;
      const DV3 qv{q[0], q[1], q[2]}, rv = dconst(qr[0], qr[1], qr[2]);
      const DV3 cr = dcross(qv, rv);
      const DV3 oe{q[3] * qr[0] - qr[3] * q[0] + cr.x, q[3] * qr[1] - qr[3] * q[1] + cr.y, q[3] * qr[2] - qr[3] * q[2] + cr.z};
      const double* w = m.torsoSqrtW;
      o.res[r++] = w[0] * (t.torsoPos.x - dmk(torsoRef[0]));
      o.res[r++] = w[1] * (t.torsoPos.y - dmk(torsoRef[1]));
      o.res[r++] = w[2] * (t.torsoPos.z - dmk(torsoRef[2]));
      o.res[r++] = w[3] * oe.x;
      o.res[r++] = w[4] * oe.y;
      o.res[r++] = w[5] * oe.z;
      o.res[r++] = w[6] * (t.torsoVlin.x - dmk(torsoRef[7]));
      o.res[r++] = w[7] * (t.torsoVlin.y - dmk(torsoRef[8]));
      o.res[r++] = w[8] * (t.torsoVlin.z - dmk(torsoRef[9]));
      o.res[r++] = w[9] * (t.torsoVang.x - dmk(torsoRef[10]));
      o.res[r++] = w[10] * (t.torsoVang.y - dmk(torsoRef[11]));
      o.res[r++] = w[11] * (t.torsoVang.z - dmk(torsoRef[12]));
    }
    o.res[r++] = m.icpSqrtW * (0.5 * (t.footPos[0].x + t.footPos[1].x) - k.Gcom.x);
    o.res[r++] = m.icpSqrtW * (0.5 * (t.footPos[0].y + t.footPos[1].y) - k.Gcom.y);
    for (int c = 0; c < 2; ++c) {
      const double* w = m.footSqrtW;
      o.res[r++] = w[0] * t.footPos[c].x;
      o.res[r++] = w[1] * t.footPos[c].y;
      o.res[r++] = w[2] * t.footPos[c].z;
      o.res[r++] = w[3] * t.footOri[c].x;
      o.res[r++] = w[4] * t.footOri[c].y;
      o.res[r++] = w[5] * t.footOri[c].z;
      o.res[r++] = (n.impact[c] * w[6]) * t.footVlin[c].x;
      o.res[r++] = (n.impact[c] * w[7]) * t.footVlin[c].y;
      o.res[r++] = (n.impact[c] * w[8]) * t.footVlin[c].z;
      o.res[r++] = w[9] * t.footVang[c].x;
      o.res[r++] = w[10] * t.footVang[c].y;
      o.res[r++] = w[11] * t.footVang[c].z;
      if (n.contact[c]) {
        const DV3 F{u[6 * c], u[6 * c + 1], u[6 * c + 2]}, Mo{u[6 * c + 3], u[6 * c + 4], u[6 * c + 5]};
        const int fb = m.frameBody[3 * c];
        const double mid = 1.0 - n.impact[1 - c];
        for (int e = 0; e < 6; ++e) {
          const int body = m.tqJoint[c][e] + 1;
          bool onPath = false;
          for (int a = fb; a >= 1; a = m.kin.parent[a]) onPath = onPath || (a == body);
          D1 tau = dmk(0.0);
          if (onPath) tau = ddot(k.ax[body], Mo + dcross(t.footPos[c] - k.p[body], F));
          o.res[r++] = (m.tqSqrtW[c][e] * mid) * tau;
        }
      }
    }
    // first-order penalty constraints
    for (int c = 0; c < 2; ++c)
      if (n.contact[c]) {
        const DM3& R = t.footR[c];
        const D1 F0 = u[6 * c], F1 = u[6 * c + 1], F2 = u[6 * c + 2], M0 = u[6 * c + 3], M1 = u[6 * c + 4], M2 = u[6 * c + 5];
        const D1 lfz = R.m[2] * F0 + R.m[5] * F1 + R.m[8] * F2;
        const D1 lmx = R.m[0] * M0 + R.m[3] * M1 + R.m[6] * M2;
        const D1 lmy = R.m[1] * M0 + R.m[4] * M1 + R.m[7] * M2;
        o.pen[4 * c + 0] = lmx - m.rect[2] * lfz;
        o.pen[4 * c + 1] = -lmx + m.rect[3] * lfz;
        o.pen[4 * c + 2] = -lmy - m.rect[0] * lfz;
        o.pen[4 * c + 3] = lmy + m.rect[1] * lfz;
      }
    if (!(n.contact[0] && n.contact[1]))
      for (int e = 0; e < 16; ++e) {
        int a, b;
        bool knee;
        collisionPair(e, a, b, knee);
        const DV3 dv = t.framePos[a] - t.framePos[b];
        o.pen[8 + e] = dsqrt(ddot(dv, dv)) - dmk(2.0 * (knee ? m.rKnee : m.rFoot));
      }
  }
  // ---- RK4 (rk4SensitivityDiscretization restated as forward mode through the integrator) ---------------------------------------------------
  const double h = n.dt, h2 = 0.5 * n.dt;
  for (int i = 0; i < CNX; ++i) {
    o.xplus[i] = x[i] + (h / 6.0) * f[i];
    xs[i] = x[i] + h2 * f[i];
  }
  cenKinematics(m.kin, xs + 6, k);
  cenFlowFromKin(m.kin, k, xs, u, f);
  for (int i = 0; i < CNX; ++i) {
    o.xplus[i] = o.xplus[i] + (h / 3.0) * f[i];
    xs[i] = x[i] + h2 * f[i];
  }
  cenKinematics(m.kin, xs + 6, k);
  cenFlowFromKin(m.kin, k, xs, u, f);
  for (int i = 0; i < CNX; ++i) {
    o.xplus[i] = o.xplus[i] + (h / 3.0) * f[i];
    xs[i] = x[i] + h * f[i];
  }
  cenKinematics(m.kin, xs + 6, k);
  cenFlowFromKin(m.kin, k, xs, u, f);
  for (int i = 0; i < CNX; ++i) o.xplus[i] = o.xplus[i] + (h / 6.0) * f[i];
}

}  // namespace b200sqp
