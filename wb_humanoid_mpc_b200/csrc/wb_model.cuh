// Device-side constants of the whole-body OCP and small 3D/6D vector helpers.
#pragma once
#include <cuda_runtime.h>

#include "../../include/b200sqp.h"

#ifndef HD
#define HD __host__ __device__ __forceinline__
#endif

namespace b200sqp {

constexpr int NJ = 23;            // actuated joints of the G1 MPC model
constexpr int NB = NJ + 1;        // bodies (0 = floating base)
constexpr int NV = 6 + NJ;        // generalized velocity dimension (29)
constexpr int NX = 2 * NV;        // 58
constexpr int NU = 12 + NJ;       // 35
constexpr int NZ = NX + NU;       // 93 tangent directions (x then u)
constexpr int NC_MAX = 14;        // state-input equality constraint rows (12 / 13 / 14)
constexpr int NUT_MAX = NU - 12;  // 23 projected inputs (double stance)
constexpr int NFRAMES = 10;
constexpr int LEG_LEN = 6;

struct WbDeviceModel {
  int parent[NB];
  unsigned subtree[NB];  // bit j set <=> body j is in the subtree of body i (including i)
  int pathLen[NB], path[NB][8];  // joints from the base to body i (inclusive), root side first
  double jR[NB][9], jp[NB][3], axis[NB][3];
  double mass[NB], com[NB][3], Icom[NB][9];
  double mtot, gravity;
  double qlo[NJ], qhi[NJ];
  int frameBody[NFRAMES];
  double frameP[NFRAMES][3];
  int legBody[2][LEG_LEN];  // bodies from hip to ankle-roll of each contact
  double rect[4];
  double Qd[NX], Rd[NU], Qfd[NX];
  double gPosZ, gOri, gLinVelZ, gLinVelXY, gAngVel, gLinAccZ, gLinAccXY, gAngAcc;
  double footSqrtW[18];
  double fricCoeff, fricMu, fricDelta, fricReg, fricShift;
  double momMu, momDelta, jlMu, jlDelta, collMu, collDelta, rFoot, rKnee;
  int armJoint[4];
};

// ---- 3-vectors -------------------------------------------------------------------------------------------------------
struct V3 {
  double x, y, z;
};
HD V3 mk(double x, double y, double z) { return V3{x, y, z}; }
HD V3 ld3(const double* p) { return V3{p[0], p[1], p[2]}; }
HD void st3(double* p, V3 v) {
  p[0] = v.x;
  p[1] = v.y;
  p[2] = v.z;
}
HD V3 operator+(V3 a, V3 b) { return V3{a.x + b.x, a.y + b.y, a.z + b.z}; }
HD V3 operator-(V3 a, V3 b) { return V3{a.x - b.x, a.y - b.y, a.z - b.z}; }
HD V3 operator-(V3 a) { return V3{-a.x, -a.y, -a.z}; }
HD V3 operator*(double s, V3 a) { return V3{s * a.x, s * a.y, s * a.z}; }
HD V3 cross(V3 a, V3 b) { return V3{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
HD double dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
// row-major 3x3 times vector / transposed
HD V3 mv(const double* R, V3 v) {
  return V3{R[0] * v.x + R[1] * v.y + R[2] * v.z, R[3] * v.x + R[4] * v.y + R[5] * v.z, R[6] * v.x + R[7] * v.y + R[8] * v.z};
}
HD V3 mtv(const double* R, V3 v) {
  return V3{R[0] * v.x + R[3] * v.y + R[6] * v.z, R[1] * v.x + R[4] * v.y + R[7] * v.z, R[2] * v.x + R[5] * v.y + R[8] * v.z};
}
HD void mm3(const double* A, const double* B, double* C) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}

// ---- spatial 6-vectors [lin; ang] ------------------------------------------------------------------------------------------
struct V6 {
  V3 l, a;
};
HD V6 ld6(const double* p) { return V6{ld3(p), ld3(p + 3)}; }
HD void st6(double* p, V6 v) {
  st3(p, v.l);
  st3(p + 3, v.a);
}
HD V6 operator+(V6 a, V6 b) { return V6{a.l + b.l, a.a + b.a}; }
HD V6 operator-(V6 a, V6 b) { return V6{a.l - b.l, a.a - b.a}; }
HD V6 operator*(double s, V6 a) { return V6{s * a.l, s * a.a}; }
HD V6 mcross(V6 a, V6 b) { return V6{cross(a.a, b.l) + cross(a.l, b.a), cross(a.a, b.a)}; }   // motion x motion
HD V6 fcross(V6 a, V6 f) { return V6{cross(a.a, f.l), cross(a.a, f.a) + cross(a.l, f.l)}; }   // motion x* force
// 6x6 (row-major, [lin;ang]) times 6-vector
HD V6 m6v(const double* M, V6 v) {
  double in[6] = {v.l.x, v.l.y, v.l.z, v.a.x, v.a.y, v.a.z}, o[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    double s = 0.0;
#pragma unroll
    for (int j = 0; j < 6; ++j) s = fma(M[6 * i + j], in[j], s);
    o[i] = s;
  }
  return V6{V3{o[0], o[1], o[2]}, V3{o[3], o[4], o[5]}};
}
HD V6 basis6(int k) {
  double e[6] = {0, 0, 0, 0, 0, 0};
  e[k] = 1.0;
  return V6{V3{e[0], e[1], e[2]}, V3{e[3], e[4], e[5]}};
}

// single-tangent dual number for the closed-form output maps (the recursive part is differentiated analytically)
struct D1 {
  double v, d;
};
HD D1 dmk(double v, double d = 0.0) { return D1{v, d}; }
HD D1 operator+(D1 a, D1 b) { return D1{a.v + b.v, a.d + b.d}; }
HD D1 operator-(D1 a, D1 b) { return D1{a.v - b.v, a.d - b.d}; }
HD D1 operator-(D1 a) { return D1{-a.v, -a.d}; }
HD D1 operator*(D1 a, D1 b) { return D1{a.v * b.v, fma(a.d, b.v, a.v * b.d)}; }
HD D1 operator*(double s, D1 a) { return D1{s * a.v, s * a.d}; }
HD D1 operator/(D1 a, D1 b) {
  const double inv = 1.0 / b.v, q = a.v * inv;
  return D1{q, (a.d - q * b.d) * inv};
}
HD D1 dsqrt(D1 a) {
  const double s = sqrt(a.v);
  return D1{s, 0.5 * a.d / s};
}
struct DV3 {
  D1 x, y, z;
};
HD DV3 dv3(V3 v, V3 d) { return DV3{D1{v.x, d.x}, D1{v.y, d.y}, D1{v.z, d.z}}; }
HD DV3 operator+(DV3 a, DV3 b) { return DV3{a.x + b.x, a.y + b.y, a.z + b.z}; }
HD DV3 operator-(DV3 a, DV3 b) { return DV3{a.x - b.x, a.y - b.y, a.z - b.z}; }
HD DV3 dcross(DV3 a, DV3 b) { return DV3{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
HD V3 val(DV3 a) { return V3{a.x.v, a.y.v, a.z.v}; }
HD V3 tan_(DV3 a) { return V3{a.x.d, a.y.d, a.z.d}; }
// (R, dR) row-major 3x3 dual times dual vector
HD DV3 dmv(const double* R, const double* dR, DV3 v) {
  D1 r[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) r[i] = D1{R[i], dR[i]};
  return DV3{r[0] * v.x + r[1] * v.y + r[2] * v.z, r[3] * v.x + r[4] * v.y + r[5] * v.z, r[6] * v.x + r[7] * v.y + r[8] * v.z};
}
HD DV3 dmtv(const double* R, const double* dR, DV3 v) {
  D1 r[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) r[i] = D1{R[i], dR[i]};
  return DV3{r[0] * v.x + r[3] * v.y + r[6] * v.z, r[1] * v.x + r[4] * v.y + r[7] * v.z, r[2] * v.x + r[5] * v.y + r[8] * v.z};
}

HD D1 dsin(D1 a) { return D1{sin(a.v), cos(a.v) * a.d}; }
HD D1 dcos(D1 a) { return D1{cos(a.v), -sin(a.v) * a.d}; }
HD D1 operator*(D1 a, double s) { return D1{a.v * s, a.d * s}; }
HD D1 ddot(DV3 a, DV3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
HD DV3 operator*(D1 s, DV3 a) { return DV3{s * a.x, s * a.y, s * a.z}; }
HD DV3 operator*(double s, DV3 a) { return DV3{s * a.x, s * a.y, s * a.z}; }
HD DV3 dconst(double x, double y, double z) { return DV3{dmk(x), dmk(y), dmk(z)}; }
struct DM3 {  // row-major
  D1 m[9];
};
HD DV3 operator*(const DM3& A, DV3 v) {
  return DV3{A.m[0] * v.x + A.m[1] * v.y + A.m[2] * v.z, A.m[3] * v.x + A.m[4] * v.y + A.m[5] * v.z, A.m[6] * v.x + A.m[7] * v.y + A.m[8] * v.z};
}
HD DM3 operator*(const DM3& A, const DM3& B) {
  DM3 C;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) C.m[3 * i + j] = A.m[3 * i] * B.m[j] + A.m[3 * i + 1] * B.m[3 + j] + A.m[3 * i + 2] * B.m[6 + j];
  return C;
}
HD DM3 dinv3(const DM3& A) {
  const D1 c00 = A.m[4] * A.m[8] - A.m[5] * A.m[7], c01 = A.m[5] * A.m[6] - A.m[3] * A.m[8], c02 = A.m[3] * A.m[7] - A.m[4] * A.m[6];
  const D1 id = dmk(1.0) / (A.m[0] * c00 + A.m[1] * c01 + A.m[2] * c02);
  DM3 R;
  R.m[0] = c00 * id; R.m[1] = (A.m[2] * A.m[7] - A.m[1] * A.m[8]) * id; R.m[2] = (A.m[1] * A.m[5] - A.m[2] * A.m[4]) * id;
  R.m[3] = c01 * id; R.m[4] = (A.m[0] * A.m[8] - A.m[2] * A.m[6]) * id; R.m[5] = (A.m[2] * A.m[3] - A.m[0] * A.m[5]) * id;
  R.m[6] = c02 * id; R.m[7] = (A.m[1] * A.m[6] - A.m[0] * A.m[7]) * id; R.m[8] = (A.m[0] * A.m[4] - A.m[1] * A.m[3]) * id;
  return R;
}

}  // namespace b200sqp
