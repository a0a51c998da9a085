// oracle/shim/robotoc/robot/robot.hpp -- TEST INFRASTRUCTURE.  Stand-in for robotoc::Robot (the reference's class wraps
// pinocchio::Model / Data; Pinocchio is not in this image).  It carries the DIMENSIONS the hot-path sources query
// (include/robotoc/robot/robot.hpp: dimq, dimv, dimu, max_dimf, dim_passive, hasFloatingBase, maxNumContacts,
// contactTypes) and a dense restatement of the one piece of Pinocchio arithmetic that sits on the path,
// Robot::computeMJtJinv (include/robotoc/robot/robot.hxx:642-683: [[M, J^T], [J, 0]]^-1 through Cholesky of M and of
// J M^-1 J^T).  Rigid-body producers (RNEA, kinematics, SE(3) integration) are declared so that the reference's
// dynamics sources compile unmodified, and abort if ever called: they are outside the hot path (SURVEY.md 8, OUT-OF-SCOPE).
#ifndef ROBOTOC_ROBOT_HPP_
#define ROBOTOC_ROBOT_HPP_

#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "Eigen/Core"
#include "Eigen/LU"

#include "robotoc/robot/se3.hpp"
#include "robotoc/robot/contact_status.hpp"
#include "robotoc/robot/impact_status.hpp"
#include "robotoc/utils/aligned_vector.hpp"

namespace robotoc {

class Robot {
 public:
  using Vector6d = Eigen::Matrix<double, 6, 1>;

  Robot() : dimq_(0), dimv_(0), dimu_(0), dim_passive_(0), max_dimf_(0), floating_(false) {}
  /// floating base: dimq = dimv + 1 (quaternion), dim_passive = 6, dimu = dimv - 6
  Robot(int dimv, bool floating_base, int n_point_contacts)
      : dimq_(dimv + (floating_base ? 1 : 0)), dimv_(dimv), dimu_(dimv - (floating_base ? 6 : 0)),
        dim_passive_(floating_base ? 6 : 0), max_dimf_(3 * n_point_contacts), floating_(floating_base),
        contact_types_(size_t(n_point_contacts), ContactType::PointContact) {
    for (int i = 0; i < n_point_contacts; ++i) contact_frame_names_.push_back("contact_" + std::to_string(i));
  }

  int dimq() const { return dimq_; }
  int dimv() const { return dimv_; }
  int dimu() const { return dimu_; }
  int max_dimf() const { return max_dimf_; }
  int dim_passive() const { return dim_passive_; }
  bool hasFloatingBase() const { return floating_; }
  int maxNumContacts() const { return int(contact_types_.size()); }
  int maxNumPointContacts() const { return int(contact_types_.size()); }
  int maxNumSurfaceContacts() const { return 0; }
  ContactType contactType(const int i) const { return contact_types_[size_t(i)]; }
  const std::vector<ContactType>& contactTypes() const { return contact_types_; }
  std::vector<int> contactFrames() const { std::vector<int> f; for (size_t i = 0; i < contact_types_.size(); ++i) f.push_back(int(i)); return f; }
  ContactStatus createContactStatus() const { return ContactStatus(contact_types_, contact_frame_names_); }
  ImpactStatus createImpactStatus() const { return ImpactStatus(contact_types_, contact_frame_names_); }

  /// Dense restatement of robot.hxx:642-683 (Pinocchio's sparse Cholesky of M replaced by a dense one).
  template <typename MatrixType1, typename MatrixType2, typename MatrixType3>
  void computeMJtJinv(const Eigen::MatrixBase<MatrixType1>& M, const Eigen::MatrixBase<MatrixType2>& J,
                      const Eigen::MatrixBase<MatrixType3>& MJtJinv) {
    const int dimf = int(J.rows());
    Eigen::LLT<Eigen::MatrixXd> llt_M, llt_S;
    llt_M.compute(M);
    assert(llt_M.info() == Eigen::Success);
    const Eigen::MatrixXd Minv = llt_M.solve(Eigen::MatrixXd::Identity(dimv_, dimv_));
    Eigen::MatrixBase<MatrixType3>& out = const_cast<Eigen::MatrixBase<MatrixType3>&>(MJtJinv);
    if (dimf == 0) {
      out.topLeftCorner(dimv_, dimv_) = Minv;
      return;
    }
    const Eigen::MatrixXd MinvJt = llt_M.solve(Eigen::MatrixXd(J.transpose()));
    const Eigen::MatrixXd S = J * MinvJt;
    llt_S.compute(S);
    assert(llt_S.info() == Eigen::Success);
    const Eigen::MatrixXd Sinv = llt_S.solve(Eigen::MatrixXd::Identity(dimf, dimf));
    const Eigen::MatrixXd topRight = MinvJt * Sinv;
    out.topLeftCorner(dimv_, dimv_) = Minv - topRight * MinvJt.transpose();
    out.topRightCorner(dimv_, dimf) = topRight;
    out.bottomLeftCorner(dimf, dimv_) = topRight.transpose();
    out.bottomRightCorner(dimf, dimf) = -Sinv;
  }

  // ---- rigid-body producers: outside the hot path; present only so that the reference's sources compile and link
#define RBT_SHIM_UNREACHABLE(NAME) { std::fprintf(stderr, "oracle/shim Robot::" NAME " called: Pinocchio is not available\n"); std::abort(); }
  template <typename... A> void RNEA(const A&...) RBT_SHIM_UNREACHABLE("RNEA")
  template <typename... A> void RNEADerivatives(const A&...) RBT_SHIM_UNREACHABLE("RNEADerivatives")
  /// Test hook for a fixed-base robot: UnconstrDynamics keeps ID_ and dID_d* private and fills them only through
  /// RNEA / RNEADerivatives (unconstr_dynamics.cpp:46-60).  These overloads (exact matches for the VectorXd / MatrixXd members,
  /// so they win over the aborting templates above) return the injected values, which are INPUTS of the hot path (sections
  /// l_ID, l_dIDd* of the unconstrained linearization record).
  void injectRNEA(const Eigen::VectorXd& ID, const Eigen::MatrixXd& dq, const Eigen::MatrixXd& dv, const Eigen::MatrixXd& da) {
    inj_ID_ = ID; inj_dq_ = dq; inj_dv_ = dv; inj_da_ = da; has_inj_rnea_ = true;
  }
  void RNEA(const Eigen::VectorXd&, const Eigen::VectorXd&, const Eigen::VectorXd&, Eigen::VectorXd& tau) {
    if (!has_inj_rnea_) RBT_SHIM_UNREACHABLE("RNEA without injected values")
    tau = inj_ID_;
  }
  void RNEADerivatives(const Eigen::VectorXd&, const Eigen::VectorXd&, const Eigen::VectorXd&, Eigen::MatrixXd& dq,
                       Eigen::MatrixXd& dv, Eigen::MatrixXd& da) {
    if (!has_inj_rnea_) RBT_SHIM_UNREACHABLE("RNEADerivatives without injected values")
    dq = inj_dq_; dv = inj_dv_; da = inj_da_;
  }
  template <typename... A> void RNEAImpact(const A&...) RBT_SHIM_UNREACHABLE("RNEAImpact")
  template <typename... A> void RNEAImpactDerivatives(const A&...) RBT_SHIM_UNREACHABLE("RNEAImpactDerivatives")
  template <typename... A> void updateKinematics(const A&...) RBT_SHIM_UNREACHABLE("updateKinematics")
  template <typename... A> void updateFrameKinematics(const A&...) RBT_SHIM_UNREACHABLE("updateFrameKinematics")
  template <typename... A> void setContactForces(const A&...) RBT_SHIM_UNREACHABLE("setContactForces")
  template <typename... A> void setImpactForces(const A&...) RBT_SHIM_UNREACHABLE("setImpactForces")
  template <typename... A> void computeBaumgarteResidual(const A&...) RBT_SHIM_UNREACHABLE("computeBaumgarteResidual")
  template <typename... A> void computeBaumgarteDerivatives(const A&...) RBT_SHIM_UNREACHABLE("computeBaumgarteDerivatives")
  template <typename... A> void computeImpactVelocityResidual(const A&...) RBT_SHIM_UNREACHABLE("computeImpactVelocityResidual")
  template <typename... A> void computeImpactVelocityDerivatives(const A&...) RBT_SHIM_UNREACHABLE("computeImpactVelocityDerivatives")
  template <typename... A> void computeContactPositionResidual(const A&...) RBT_SHIM_UNREACHABLE("computeContactPositionResidual")
  template <typename... A> void computeContactPositionDerivative(const A&...) RBT_SHIM_UNREACHABLE("computeContactPositionDerivative")
  /// q <- q (+) step * dq for the JOINT coordinates only (vector space); the free-flyer part (SE(3) exponential, Pinocchio) is
  /// left untouched -- the wrapper's callers compare only the joint part of q.
  template <typename V, typename Q>
  void integrateConfiguration(const Eigen::MatrixBase<V>& dq, const double step, const Eigen::MatrixBase<Q>& q) const {
    Eigen::MatrixBase<Q>& qq = const_cast<Eigen::MatrixBase<Q>&>(q);
    const int nb_q = floating_ ? 7 : 0, nb_v = floating_ ? 6 : 0;
    for (int i = 0; i < dimv_ - nb_v; ++i) qq.coeffRef(nb_q + i) += step * dq.coeff(nb_v + i);
  }
  template <typename... A> void subtractConfiguration(const A&...) const RBT_SHIM_UNREACHABLE("subtractConfiguration")
  template <typename... A> void dSubtractConfiguration_dqf(const A&...) const RBT_SHIM_UNREACHABLE("dSubtractConfiguration_dqf")
  /// Test hook: the reference's correctLinearize(Impact)StateEquation re-evaluates dSubtract/dq0 (a Pinocchio call) in the middle
  /// of the linear algebra (state_equation.cpp:77, impact_state_equation.cpp:63); the wrapper queues the 6x6 block that call
  /// has to return (it is an INPUT of the hot path: section l_se3 of the linearization record).
  void injectdSubtractConfiguration_dq0(const Eigen::MatrixXd& top_left_6x6) { injected_ = top_left_6x6; has_injected_ = true; }
  template <typename Q1, typename Q2, typename M>
  void dSubtractConfiguration_dq0(const Q1&, const Q2&, const Eigen::MatrixBase<M>& out) const {
    if (!has_injected_) { std::fprintf(stderr, "oracle/shim Robot::dSubtractConfiguration_dq0 called without an injected block\n"); std::abort(); }
    Eigen::MatrixBase<M>& o = const_cast<Eigen::MatrixBase<M>&>(out);
    o.topLeftCorner(6, 6) = injected_;
  }
  template <typename... A> void dIntegrateTransport_dq(const A&...) const RBT_SHIM_UNREACHABLE("dIntegrateTransport_dq")
  template <typename... A> void dIntegrateTransport_dv(const A&...) const RBT_SHIM_UNREACHABLE("dIntegrateTransport_dv")
  template <typename... A> void normalizeConfiguration(const A&...) const RBT_SHIM_UNREACHABLE("normalizeConfiguration")
  template <typename... A> void transformFromLocalToWorld(const A&...) const RBT_SHIM_UNREACHABLE("transformFromLocalToWorld")
  template <typename... A> void getJacobianTransformFromLocalToWorld(const A&...) RBT_SHIM_UNREACHABLE("getJacobianTransformFromLocalToWorld")
  const Eigen::Matrix3d& frameRotation(const int) const RBT_SHIM_UNREACHABLE("frameRotation")
  Eigen::VectorXd jointEffortLimit() const { return limit_effort_; }
  Eigen::VectorXd jointVelocityLimit() const { return limit_velocity_; }
  Eigen::VectorXd lowerJointPositionLimit() const { return limit_qmin_; }
  Eigen::VectorXd upperJointPositionLimit() const { return limit_qmax_; }
  void setJointLimits(const Eigen::VectorXd& effort, const Eigen::VectorXd& velocity, const Eigen::VectorXd& qmin,
                      const Eigen::VectorXd& qmax) {
    limit_effort_ = effort; limit_velocity_ = velocity; limit_qmin_ = qmin; limit_qmax_ = qmax;
  }
#undef RBT_SHIM_UNREACHABLE

 private:
  int dimq_, dimv_, dimu_, dim_passive_, max_dimf_;
  bool floating_;
  std::vector<ContactType> contact_types_;
  std::vector<std::string> contact_frame_names_;
  Eigen::VectorXd limit_effort_, limit_velocity_, limit_qmin_, limit_qmax_;
  Eigen::MatrixXd injected_;
  bool has_injected_ = false;
  Eigen::VectorXd inj_ID_;
  Eigen::MatrixXd inj_dq_, inj_dv_, inj_da_;
  bool has_inj_rnea_ = false;
};

}  // namespace robotoc

#endif  // ROBOTOC_ROBOT_HPP_
