// oracle/ref_wrap/ref_ustage_wrap.cpp -- TEST INFRASTRUCTURE.  One grid point of the UNCONSTRAINED (fixed-base) path through the
// REFERENCE's own stage-layer code (compiled unmodified from robotoc/src/dynamics/unconstr_dynamics.cpp, src/constraints, src/core;
// oracle/Makefile.ref), in the order UnconstrIntermediateStage / UnconstrTerminalStage use it
// (src/unconstr/unconstr_intermediate_stage.cpp:70-144, unconstr_terminal_stage.cpp:69-132):
//   createConstraintsData(robot, stage) -> Constraints::condenseSlackAndDual -> UnconstrDynamics::condenseUnconstrDynamics
//   -> expandPrimal -> expandDual -> Constraints::expandSlackAndDual -> maxSlackStepSize / maxDualStepSize
//   -> SplitSolution::integrate -> Constraints::updateSlack / updateDual
// Inputs and outputs are the packed records of include/rbt_ustage_layout.h / rbt_layout.h (rbt_ulayout), so tests hand the same
// arrays to the oracle (oracle/unconstr_stage_oracle.c) and to this wrapper.  ID and dID/d(q, v, a) are INPUTS of the hot path;
// they reach UnconstrDynamics through the shim's injected Robot::RNEA / RNEADerivatives, with u = 0 and beta = 0 so that
// linearizeUnconstrDynamics adds nothing to the gradients the linearization record already holds.
#include <cstring>
#include <memory>

#include "Eigen/Core"
#include "robotoc/robot/robot.hpp"
#include "robotoc/core/split_kkt_matrix.hpp"
#include "robotoc/core/split_kkt_residual.hpp"
#include "robotoc/core/split_direction.hpp"
#include "robotoc/core/split_solution.hpp"
#include "robotoc/dynamics/unconstr_dynamics.hpp"
#include "robotoc/constraints/constraints.hpp"
#include "robotoc/constraints/pdipm.hpp"
#include "robotoc/constraints/joint_position_lower_limit.hpp"
#include "robotoc/constraints/joint_position_upper_limit.hpp"
#include "robotoc/constraints/joint_velocity_lower_limit.hpp"
#include "robotoc/constraints/joint_velocity_upper_limit.hpp"
#include "robotoc/constraints/joint_torques_lower_limit.hpp"
#include "robotoc/constraints/joint_torques_upper_limit.hpp"
#include "robotoc/constraints/joint_acceleration_lower_limit.hpp"
#include "robotoc/constraints/joint_acceleration_upper_limit.hpp"

#include "../../include/rbt_layout.h"
#include "../../include/rbt_ustage_layout.h"

namespace {
using namespace robotoc;

template <class M> void put_m(M&& dst, const double* src, int rows, int cols) {
  for (int j = 0; j < cols; ++j) for (int i = 0; i < rows; ++i) dst(i, j) = src[i + size_t(j) * rows];
}
template <class V> void put_v(V&& dst, const double* src, int n) { for (int i = 0; i < n; ++i) dst(i) = src[i]; }
template <class M> void get_m(const M& src, double* dst, int rows, int cols) {
  for (int j = 0; j < cols; ++j) for (int i = 0; i < rows; ++i) dst[i + size_t(j) * rows] = src(i, j);
}
template <class V> void get_v(const V& src, double* dst, int n) { for (int i = 0; i < n; ++i) dst[i] = src(i); }

// Number of components (6: the joint limits of examples/iiwa14/unconstr_ocp_benchmark.cpp:45-60; 8: + joint acceleration
// lower / upper limits) when the table is exactly what the reference can express, in component order; 0 otherwise.
int components(int nv, const rbt_constraint_table* tab) {
  const int var[8] = {RBT_VAR_Q, RBT_VAR_Q, RBT_VAR_V, RBT_VAR_V, RBT_VAR_U, RBT_VAR_U, RBT_VAR_A, RBT_VAR_A};
  const int nk = tab->n_box / nv;
  if (tab->n_contacts != 0 || (nk != 6 && nk != 8) || nk * nv != tab->n_box) return 0;
  for (int r = 0; r < tab->n_box; ++r) {
    const int k = r / nv;
    if (tab->box[r].var != var[k] || tab->box[r].idx != r % nv || tab->box[r].sign != (k % 2 ? 1 : -1)) return 0;
  }
  return nk;
}

// component k of the table order -> its ConstraintComponentData (Constraints::add sorts components by kinematics level and
// keeps the order of addition within a level)
ConstraintComponentData& component(ConstraintsData& d, int k) {
  return k < 2 ? d.position_level_data[k] : k < 4 ? d.velocity_level_data[k - 2] : d.acceleration_level_data[k - 4];
}
bool component_valid(const ConstraintsData& d, int k) {
  return k < 2 ? d.isPositionLevelValid() : k < 4 ? d.isVelocityLevelValid() : d.isAccelerationLevelValid();
}
}  // namespace

extern "C" {

// One grid point `stage` (GridInfo::stage, as UnconstrOCPSolver sets it: unconstr_ocp_solver.cpp:41-50) of an OCP with N
// intervals of length dt.  Returns 0, or 1 if the table is not one the reference can express.
// phase: 1 = condensing only (kkt, ex, con cmpl | cond), 2 = + expansion (xd du | dbeta, con dslack | ddual) and this grid
// point's max step sizes (steps_stage[2]), 3 = + SplitSolution::integrate with (alpha_p, d) and the slack / dual update.
// d: the direction record (rbt_ulayout d_dx, d_dlmdgmm, d_da) of this grid point.
// Records of a constraint level that is not valid on this grid point are left as they came in.
int ref_ustage(int nv, const rbt_constraint_table* tab, int stage, int N, double dt, const double* lin, double* con,
               double* kkt, double* ex, const double* d, double* xd, double* sol, double* steps_stage, double alpha_p,
               double alpha_d, int phase) {
  const int nk = components(nv, tab);
  if (!nk) return 1;
  rbt_ustage_layout S;
  rbt_make_ustage_layout(nv, tab->n_box, &S);
  rbt_ulayout K;
  rbt_make_ulayout(nv, &K);
  const int nx = 2 * nv;
  const bool terminal = stage == N;
  Robot robot(nv, false, 0);
  {
    Eigen::VectorXd lim = Eigen::VectorXd::Constant(nv, 1.0);
    robot.setJointLimits(lim, lim, -lim, lim);
  }
  SplitKKTMatrix km(robot);
  SplitKKTResidual kr(robot);
  put_m(km.Qxx, lin + S.l_Qxx, nx, nx);
  put_v(kr.lx, lin + S.l_lx, nx);
  SplitDirection dd(robot);
  put_v(dd.dx, d + K.d_dx, nx);
  put_v(dd.dlmdgmm, d + K.d_dlmdgmm, nx);
  steps_stage[0] = steps_stage[1] = 1.0;
  if (terminal) {  // UnconstrTerminalStage: the cost is the KKT record; no constraints, no dynamics (:69-132)
    get_m(km.Qxx, kkt + K.k_Qxx, nx, nx);
    get_v(kr.lx, kkt + K.k_lx, nx);
    if (phase >= 3) {
      SplitSolution s(robot);
      put_v(s.q, sol + S.s_q, nv); put_v(s.v, sol + S.s_v, nv); put_v(s.a, sol + S.s_a, nv); put_v(s.u, sol + S.s_u, nv);
      put_v(s.beta, sol + S.s_beta, nv); put_v(s.lmd, sol + S.s_lmd, nv); put_v(s.gmm, sol + S.s_gmm, nv);
      s.integrate(robot, alpha_p, dd);
      get_v(s.q, sol + S.s_q, nv); get_v(s.v, sol + S.s_v, nv); get_v(s.a, sol + S.s_a, nv); get_v(s.u, sol + S.s_u, nv);
      get_v(s.beta, sol + S.s_beta, nv); get_v(s.lmd, sol + S.s_lmd, nv); get_v(s.gmm, sol + S.s_gmm, nv);
    }
    return 0;
  }
  put_m(km.Qaa, lin + S.l_Qaa, nv, nv);
  put_m(km.Quu, lin + S.l_Quu, nv, nv);
  put_v(kr.la, lin + S.l_la, nv);
  put_v(kr.lu, lin + S.l_lu, nv);
  put_v(kr.Fx, lin + S.l_Fx, nx);
  {
    Eigen::VectorXd ID(nv);
    Eigen::MatrixXd Dq(nv, nv), Dv(nv, nv), Da(nv, nv);
    put_v(ID, lin + S.l_ID, nv);
    put_m(Dq, lin + S.l_dIDdq, nv, nv);
    put_m(Dv, lin + S.l_dIDdv, nv, nv);
    put_m(Da, lin + S.l_dIDda, nv, nv);
    robot.injectRNEA(ID, Dq, Dv, Da);
  }
  UnconstrDynamics ud(robot);
  {
    SplitSolution s0(robot);  // u = 0, beta = 0: ID_ is the injected ID and the gradients stay as the record holds them
    s0.u.setZero();
    s0.beta.setZero();
    ud.linearizeUnconstrDynamics(robot, dt, s0, kr);
  }
  // ---- constraints: slack, dual, residual from the PDIPM record; cmpl as evalConstraint leaves it (pdipm.hxx:27-31)
  auto constraints = std::make_shared<Constraints>(tab->barrier, tab->fraction_to_boundary);
  constraints->add("joint_position_lower", std::make_shared<JointPositionLowerLimit>(robot));
  constraints->add("joint_position_upper", std::make_shared<JointPositionUpperLimit>(robot));
  constraints->add("joint_velocity_lower", std::make_shared<JointVelocityLowerLimit>(robot));
  constraints->add("joint_velocity_upper", std::make_shared<JointVelocityUpperLimit>(robot));
  constraints->add("joint_torques_lower", std::make_shared<JointTorquesLowerLimit>(robot));
  constraints->add("joint_torques_upper", std::make_shared<JointTorquesUpperLimit>(robot));
  if (nk == 8) {
    const Eigen::VectorXd amax = Eigen::VectorXd::Constant(nv, 1.0);
    constraints->add("joint_acceleration_lower", std::make_shared<JointAccelerationLowerLimit>(robot, -amax));
    constraints->add("joint_acceleration_upper", std::make_shared<JointAccelerationUpperLimit>(robot, amax));
  }
  ConstraintsData cdata = constraints->createConstraintsData(robot, stage);
  for (int k = 0; k < nk; ++k) {
    ConstraintComponentData& cc = component(cdata, k);
    put_v(cc.slack, con + S.c_slack + k * nv, nv);
    put_v(cc.dual, con + S.c_dual + k * nv, nv);
    put_v(cc.residual, con + S.c_res + k * nv, nv);
    pdipm::computeComplementarySlackness(tab->barrier, cc);
  }
  ContactStatus contact_status = robot.createContactStatus();
  constraints->condenseSlackAndDual(contact_status, cdata, km, kr);
  get_v(kr.lu, ex + S.e_lu, nv);  // the expansion record: lu, Quu after the constraints (read by expandDual)
  get_m(km.Quu, ex + S.e_Quu, nv, nv);
  ud.condenseUnconstrDynamics(km, kr);
  get_m(km.Qxx, kkt + K.k_Qxx, nx, nx);
  get_m(km.Qxu, kkt + K.k_Qxu, nx, nv);
  get_m(km.Qaa, kkt + K.k_Qaa, nv, nv);
  get_v(kr.Fx, kkt + K.k_Fx, nx);
  get_v(kr.lx, kkt + K.k_lx, nx);
  get_v(kr.la, kkt + K.k_la, nv);
  for (int k = 0; k < nk; ++k) {
    if (!component_valid(cdata, k)) continue;  // the reference does not touch the data of a level that is not valid here
    get_v(component(cdata, k).cmpl, con + S.c_cmpl + k * nv, nv);
    get_v(component(cdata, k).cond, con + S.c_cond + k * nv, nv);
  }
  if (phase < 2) return 0;

  // ---- expansion and step sizes (unconstr_intermediate_stage.cpp:103-122)
  put_v(dd.da(), d + K.d_da, nv);
  ud.expandPrimal(dd);
  UnconstrDynamics::expandDual(dt, km, kr, dd);
  constraints->expandSlackAndDual(contact_status, cdata, dd);
  get_v(dd.du, xd + S.x_du, nv);
  get_v(dd.dbeta(), xd + S.x_dbeta, nv);
  steps_stage[0] = constraints->maxSlackStepSize(cdata);
  steps_stage[1] = constraints->maxDualStepSize(cdata);
  for (int k = 0; k < nk; ++k) {
    if (!component_valid(cdata, k)) continue;
    get_v(component(cdata, k).dslack, con + S.c_dslack + k * nv, nv);
    get_v(component(cdata, k).ddual, con + S.c_ddual + k * nv, nv);
  }
  if (phase < 3) return 0;

  // ---- updatePrimal / updateDual (:125-144)
  SplitSolution s(robot);
  put_v(s.q, sol + S.s_q, nv); put_v(s.v, sol + S.s_v, nv); put_v(s.a, sol + S.s_a, nv); put_v(s.u, sol + S.s_u, nv);
  put_v(s.beta, sol + S.s_beta, nv); put_v(s.lmd, sol + S.s_lmd, nv); put_v(s.gmm, sol + S.s_gmm, nv);
  s.integrate(robot, alpha_p, dd);
  get_v(s.q, sol + S.s_q, nv); get_v(s.v, sol + S.s_v, nv); get_v(s.a, sol + S.s_a, nv); get_v(s.u, sol + S.s_u, nv);
  get_v(s.beta, sol + S.s_beta, nv); get_v(s.lmd, sol + S.s_lmd, nv); get_v(s.gmm, sol + S.s_gmm, nv);
  Constraints::updateSlack(cdata, alpha_p);
  Constraints::updateDual(cdata, alpha_d);
  for (int k = 0; k < nk; ++k) {
    if (!component_valid(cdata, k)) continue;
    get_v(component(cdata, k).slack, con + S.c_slack + k * nv, nv);
    get_v(component(cdata, k).dual, con + S.c_dual + k * nv, nv);
  }
  return 0;
}

}  // extern "C"
