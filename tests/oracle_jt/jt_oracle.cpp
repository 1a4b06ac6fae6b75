// ORACLE extension (test infrastructure only) -- the joint-torque cost of the whole-body OCP (JointTorqueCostCppAd,
// humanoid_nmpc/humanoid_wb_mpc/src/cost/JointTorqueCostCppAd.cpp) on top of the CPU oracle of oracle/: the oracle's C entry points plus a
// whole-body OCP whose intermediate-node cost carries the term.  Built into tests/oracle_jt/libjtoracle.so by tests/jt_oracle_lib.py.
//
// computeJointTorques is restated on a template scalar (the oracle's wbJointTorques is double-only), so that the Jacobian of the residual comes
// from the oracle's own dual numbers -- independent of the forward-mode lanes of the CUDA path.  The oracle's SQP calls cost / costQuad at
// intermediate nodes only (PreEvent and terminal nodes have their own setup), which is where the reference's StateInputCost applies.
#include "../../oracle/capi.cpp"

namespace orc {

// computeJointTorques (humanoid_common_mpc/src/pinocchio_model/DynamicsHelperFunctions.cpp:232-270), as the oracle's wbJointTorques:
// tau_j = M_j [qdd_b; qdd_j] + nle_j - (J' W)_j with qdd_b from computeBaseAcceleration (block-diagonal M_bb inverse)
template <class S>
void wbJointTorquesT(const WbParams& P, const S* x, const S* u, S* tau) {
  const RobotModel& m = P.model;
  const int nv = m.nv();
  S qddb[6];
  KinData<S> kd;
  wbBaseAcceleration<S>(P, x, u, qddb, &kd);
  std::vector<S> a(nv, S(0.0)), full(nv);
  for (int k = 0; k < 6; ++k) a[k] = qddb[k];
  for (int j = 0; j < m.nj; ++j) a[6 + j] = u[12 + j];
  rnea<S>(m, x, x + nv, a.data(), full.data());
  for (int c = 0; c < 2; ++c) {
    const FrameKin<S> fk = frameKinematics(m, kd, P.contactFrame[c]);
    const V3<S> F(u[6 * c], u[6 * c + 1], u[6 * c + 2]), Mo(u[6 * c + 3], u[6 * c + 4], u[6 * c + 5]);
    for (int b = m.frameBody[P.contactFrame[c]]; b > 0; b = m.parent[b]) {
      const V3<S> ax = kd.oMi[b].R * V3<S>(S(m.axis[b][0]), S(m.axis[b][1]), S(m.axis[b][2]));
      full[5 + b] = full[5 + b] - dot(ax, Mo + cross(fk.pos - kd.oMi[b].p, F));
    }
  }
  for (int j = 0; j < m.nj; ++j) tau[j] = full[6 + j];
}

class WbJtOcp : public WbOcp {
 public:
  std::vector<double> sw;   // sqrt(joint_torque_weights); empty: the term is off

  WbJtOcp(WbParams p, std::vector<double> sqrtW) : WbOcp(std::move(p)), sw(std::move(sqrtW)) {}

  // r = sqrt(w) .* tau at (x, u) on scalar S
  template <class S>
  void residual(const S* x, const S* u, S* r) const {
    std::vector<S> tau(P.nj);
    wbJointTorquesT<S>(P, x, u, tau.data());
    for (int j = 0; j < P.nj; ++j) r[j] = S(sw[j]) * tau[j];
  }

  double cost(int k, double t, const Vec& x, const Vec& u) override {
    double f = WbOcp::cost(k, t, x, u);
    if (sw.empty()) return f;
    std::vector<double> r(P.nj);
    residual<double>(x.data(), u.data(), r.data());
    double s = 0.0;
    for (double v : r) s += v * v;
    return f + 0.5 * s;
  }

  // Gauss-Newton: value 1/2 |r|^2, gradient J' r, Hessian J' J (StateInputGaussNewtonCostAd)
  QuadApprox costQuad(int k, double t, const Vec& x, const Vec& u) override {
    QuadApprox c = WbOcp::costQuad(k, t, x, u);
    if (sw.empty()) return c;
    std::vector<D> xs(nx), us(nu), r(P.nj);
    for (int i = 0; i < nx; ++i) xs[i] = D::variable(x[i], i);
    for (int i = 0; i < nu; ++i) us[i] = D::variable(u[i], nx + i);
    residual<D>(xs.data(), us.data(), r.data());
    for (const D& rr : r) {
      c.f += 0.5 * rr.v * rr.v;
      for (int i = 0; i < nx; ++i) c.dfdx[i] += rr.v * rr.d[i];
      for (int i = 0; i < nu; ++i) c.dfdu[i] += rr.v * rr.d[nx + i];
      for (int j = 0; j < nx; ++j) {
        for (int i = 0; i < nx; ++i) c.dfdxx(i, j) += rr.d[i] * rr.d[j];
        for (int i = 0; i < nu; ++i) c.dfdux(i, j) += rr.d[nx + i] * rr.d[j];
      }
      for (int j = 0; j < nu; ++j)
        for (int i = 0; i < nu; ++i) c.dfduu(i, j) += rr.d[nx + i] * rr.d[nx + j];
    }
    return c;
  }
};

}  // namespace orc

extern "C" {

// a whole-body oracle handle (the orc_wb_* entry points apply) whose OCP carries the joint-torque cost with weights w [nj]; w = NULL: off
void* orc_jt_create(const b200sqp_model_desc* d, const double* w) {
  std::vector<double> sw;
  if (w)
    for (int j = 0; j < d->nj; ++j) sw.push_back(std::sqrt(w[j]));
  auto* h = new WbHandle;
  h->ocp = std::make_unique<WbJtOcp>(paramsFromDesc(d), std::move(sw));
  return h;
}

// torques of the templated restatement (double)
void orc_jt_torques(void* hv, const double* x, const double* u, double* tau) {
  wbJointTorquesT<double>(static_cast<WbHandle*>(hv)->ocp->P, x, u, tau);
}

// residual r [nj] and its Jacobian J [nj][nx + nu] (row-major) from the dual numbers; needs weights
int orc_jt_residual(void* hv, const double* x, const double* u, double* r, double* J) {
  auto* o = dynamic_cast<WbJtOcp*>(static_cast<WbHandle*>(hv)->ocp.get());
  if (!o || o->sw.empty()) return -1;
  using D = WbOcp::D;
  const int nx = o->nx, nu = o->nu, nz = nx + nu;
  std::vector<D> xs(nx), us(nu), res(o->P.nj);
  for (int i = 0; i < nx; ++i) xs[i] = D::variable(x[i], i);
  for (int i = 0; i < nu; ++i) us[i] = D::variable(u[i], nx + i);
  o->residual<D>(xs.data(), us.data(), res.data());
  for (int j = 0; j < o->P.nj; ++j) {
    r[j] = res[j].v;
    std::memcpy(J + static_cast<size_t>(j) * nz, res[j].d, sizeof(double) * nz);
  }
  return 0;
}

}  // extern "C"
