// oracle/ref_wrap/ref_stage_wrap.cpp -- TEST INFRASTRUCTURE.  One OCP stage through the REFERENCE's own stage-layer code
// (compiled unmodified from robotoc/src/dynamics, src/constraints, src/core; oracle/Makefile.ref), in the order
// {Intermediate,Impact}Stage use it (src/ocp/intermediate_stage.cpp:133-203, impact_stage.cpp:115-169):
//   Constraints::condenseSlackAndDual -> condenseContactDynamics | condenseImpactDynamics -> correctLinearize(Impact)StateEquation
//   -> [STO scaling of intermediate_stage.cpp:140-148, seven scalings restated here: they are lines of a member function that
//      also evaluates costs] -> expandContactDynamicsPrimal -> Constraints::expandSlackAndDual -> maxSlackStepSize / maxDualStepSize
//   -> expandContactDynamicsDual -> correctCostateDirection -> Constraints::updateSlack / updateDual
// Inputs and outputs are the packed records of include/rbt_stage_layout.h / rbt_layout.h, so tests hand the same arrays to
// the oracle (oracle/condense_oracle.c) and to this wrapper.  Pinocchio-side quantities are INPUTS of the hot path (they are
// sections of the linearization record); Robot::computeMJtJinv is the shim's dense restatement.
#include <cassert>
#include <cmath>
#include <cstring>
#include <iostream>
#include <limits>
#include <memory>
#include <random>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "Eigen/Core"
#include "Eigen/LU"
#include "robotoc/robot/robot.hpp"
#include "robotoc/core/split_kkt_matrix.hpp"
#include "robotoc/core/split_kkt_residual.hpp"
#include "robotoc/core/split_direction.hpp"
#include "robotoc/core/split_solution.hpp"
#include "robotoc/dynamics/contact_dynamics.hpp"
#include "robotoc/dynamics/impact_dynamics.hpp"
#include "robotoc/dynamics/state_equation.hpp"
#include "robotoc/dynamics/impact_state_equation.hpp"
#include "robotoc/dynamics/terminal_state_equation.hpp"
#include "robotoc/constraints/constraints.hpp"
#include "robotoc/constraints/pdipm.hpp"
#include "robotoc/constraints/joint_position_lower_limit.hpp"
#include "robotoc/constraints/joint_position_upper_limit.hpp"
#include "robotoc/constraints/joint_velocity_lower_limit.hpp"
#include "robotoc/constraints/joint_velocity_upper_limit.hpp"
#include "robotoc/constraints/joint_torques_lower_limit.hpp"
#include "robotoc/constraints/joint_torques_upper_limit.hpp"
#include "robotoc/constraints/friction_cone.hpp"
#include "robotoc/constraints/impact_friction_cone.hpp"
#include "robotoc/line_search/line_search_filter.hpp"

#include "../../include/rbt_layout.h"
#include "../../include/rbt_stage_layout.h"

namespace {
using namespace robotoc;

template <class M> void put_m(M&& dst, const double* src, int rows, int cols, int ld) {
  for (int j = 0; j < cols; ++j) for (int i = 0; i < rows; ++i) dst(i, j) = src[i + size_t(j) * ld];
}
template <class V> void put_v(V&& dst, const double* src, int n) { for (int i = 0; i < n; ++i) dst(i) = src[i]; }
template <class M> void get_m(const M& src, double* dst, int rows, int cols, int ld) {
  for (int j = 0; j < cols; ++j) for (int i = 0; i < rows; ++i) dst[i + size_t(j) * ld] = src(i, j);
}
template <class V> void get_v(const V& src, double* dst, int n) { for (int i = 0; i < n; ++i) dst[i] = src(i); }

// the six joint-limit components + the friction cone of examples/anymal/trot.cpp:131-148, in the row order of the table
std::shared_ptr<Constraints> make_constraints(const Robot& robot, const rbt_constraint_table* tab) {
  auto c = std::make_shared<Constraints>(tab->barrier, tab->fraction_to_boundary);
  c->add("joint_position_lower", std::make_shared<JointPositionLowerLimit>(robot));
  c->add("joint_position_upper", std::make_shared<JointPositionUpperLimit>(robot));
  c->add("joint_velocity_lower", std::make_shared<JointVelocityLowerLimit>(robot));
  c->add("joint_velocity_upper", std::make_shared<JointVelocityUpperLimit>(robot));
  c->add("joint_torques_lower", std::make_shared<JointTorquesLowerLimit>(robot));
  c->add("joint_torques_upper", std::make_shared<JointTorquesUpperLimit>(robot));
  c->add("friction_cone", std::make_shared<FrictionCone>(robot));
  if (tab->impact_friction_cone) c->add("impact_friction_cone", std::make_shared<ImpactFrictionCone>(robot));  // run.cpp:173-181
  return c;
}

// component k of the table order -> its ConstraintComponentData inside ConstraintsData
ConstraintComponentData& component(ConstraintsData& d, int k) {
  switch (k) {
    case 0: return d.position_level_data[0];
    case 1: return d.position_level_data[1];
    case 2: return d.velocity_level_data[0];
    case 3: return d.velocity_level_data[1];
    case 4: return d.acceleration_level_data[0];
    case 5: return d.acceleration_level_data[1];
    default: return d.acceleration_level_data[2];
  }
}
}  // namespace

// {cost_barrier, primal_feasibility, dual_feasibility, kkt_error} of the last ref_stage call, summarised BEFORE "Forms linear
// system" with the reference's own member functions, exactly as {Intermediate,Impact,Terminal}Stage::evalKKT do
// (intermediate_stage.cpp:124-132, impact_stage.cpp:104-113, terminal_stage.cpp:94-100)
static double g_last_perf[4] = {0, 0, 0, 0};

extern "C" {

void ref_last_perf(double* out) { for (int q = 0; q < 4; ++q) out[q] = g_last_perf[q]; }

// Returns 0.  phase: 1 = condensing only, 2 = + primal expansion and step sizes, 3 = + dual expansion and slack / dual update.
// con: slack | dual | residual in; cmpl, cond, dslack, ddual and the updated slack | dual out.  d is updated like the reference
// updates SplitDirection (costate correction).  steps_stage[2] = this stage's max primal / dual step size.
int ref_stage(const rbt_stage_dims* sd, const rbt_constraint_table* tab, const rbt_stage_ctrl* c, const double* lin, double* con,
              double* kkt, double* ex, double* d, const double* d_next, double* xd, double* steps_stage, double alpha_p,
              double alpha_d, int phase) {
  rbt_stage_layout S;
  rbt_make_stage_layout(sd, &S);
  rbt_dims kd = {sd->nv, sd->nu, sd->ns_max, sd->n_passive};
  rbt_layout K;
  rbt_make_layout(&kd, &K);
  const int nv = S.nv, nu = S.nu, nx = S.nx, np = S.np, nfm = S.nfm, nvfm = S.nvf;
  const bool impact = c->type == RBT_IMPACT;
  const int nf = c->nf, nvf = nv + nf, ns = impact ? 0 : c->ns;
  Robot robot(nv, np == 6, tab->n_contacts);
  if (c->type == RBT_TERMINAL) {
    // TerminalStage::evalKKT tail / expandDual (terminal_stage.cpp:102-106, 139-143): the cost Hessian and gradient are the KKT
    // record; correctLinearizeTerminalStateEquation leaves Fqq_prev_inv for the costate correction
    memcpy(kkt + K.k_Qxx, lin + S.l_Qxx, sizeof(double) * nx * nx);
    memcpy(kkt + K.k_lx, lin + S.l_lx, sizeof(double) * nx);
    StateEquationData se(robot);
    SplitKKTMatrix km(robot);
    if (np == 6) put_m(se.Fqq_prev.topLeftCorner(6, 6), lin + S.l_se3 + 36, 6, 6, 6);
    correctLinearizeTerminalStateEquation(se, km);
    if (np == 6) get_m(se.Fqq_prev_inv, ex + S.e_Fqqpi, 6, 6, 6);
    {  // terminal_stage.cpp:94-100: only the cost gradient lx (the state-equation residual of the last interval lives on N-1)
      SplitKKTResidual krT(robot);
      put_v(krT.lx, lin + S.l_lx, nx);
      g_last_perf[0] = 0.0;
      g_last_perf[1] = krT.primalFeasibility<1>();
      g_last_perf[2] = krT.dualFeasibility<1>();
      g_last_perf[3] = krT.KKTError();
    }
    steps_stage[0] = steps_stage[1] = 1.0;
    if (phase >= 3) {
      SplitDirection dd(robot);
      put_v(dd.dlmdgmm, d + K.d_dlmdgmm, nx);
      correctCostateDirection(se, dd);
      get_v(dd.dlmdgmm, d + K.d_dlmdgmm, nx);
    }
    return 0;
  }
  {
    Eigen::VectorXd lim = Eigen::VectorXd::Constant(nu, 1.0);
    robot.setJointLimits(lim, lim, -lim, lim);
  }
  ContactStatus contact_status = robot.createContactStatus();
  ImpactStatus impact_status = robot.createImpactStatus();
  for (int ci = 0; ci < tab->n_contacts; ++ci)
    if ((c->contact_mask >> ci) & 1) {
      if (impact) impact_status.activateImpact(ci); else contact_status.activateContact(ci);
    }
  SplitKKTMatrix km(robot);
  SplitKKTResidual kr(robot);
  km.setContactDimension(nf); kr.setContactDimension(nf);
  km.setSwitchingConstraintDimension(ns); kr.setSwitchingConstraintDimension(ns);
  put_m(km.Qxx, lin + S.l_Qxx, nx, nx, nx);
  put_v(kr.lx, lin + S.l_lx, nx);
  put_v(kr.Fx, lin + S.l_Fx, nx);
  for (int i = 0; i < nv; ++i) (impact ? km.Qdvdv : km.Qaa)(i, i) = lin[S.l_Qaa + i];
  put_m(km.Qff(), lin + S.l_Qff, nf, nf, nfm);
  put_m(km.Qqf(), lin + S.l_Qqf, nv, nf, nv);
  put_v(impact ? kr.ldv : kr.la, lin + S.l_la, nv);
  put_v(kr.lf(), lin + S.l_lf, nf);
  // the state after linearize(Impact)StateEquation: Fqq = dSubtract/dqf (identity outside the floating-base block), Fqv = dt I
  for (int i = 0; i < nv; ++i) km.Fqq()(i, i) = 1.0;
  if (np == 6) put_m(km.Fqq().topLeftCorner(6, 6), lin + S.l_se3, 6, 6, 6);
  if (!impact) {
    for (int i = 0; i < nv; ++i) km.Fqv()(i, i) = c->dt;
    put_m(km.Quu, lin + S.l_Quu, nu, nu, nu);
    put_v(kr.lu, lin + S.l_lu, nu);
    put_v(km.ha, lin + S.l_ha, nv);
    put_v(km.hf(), lin + S.l_hf, nf);
    put_v(km.hx, lin + S.l_hx, nx);
    put_v(km.hu, lin + S.l_hu, nu);
    put_v(km.fx, lin + S.l_fx, nx);
    kr.h = lin[S.l_sc + 0];
    km.Qtt = lin[S.l_sc + 1];
    if (ns > 0) {
      put_m(km.Phix(), lin + S.l_Phix, ns, nx, ns);
      put_m(km.Phia(), lin + S.l_Phia, ns, nv, ns);
      put_v(kr.P(), lin + S.l_p, ns);
      put_v(km.Phit(), lin + S.l_Phit, ns);
    }
  }
  ContactDynamicsData cd(robot);
  cd.setContactDimension(nf);
  cd.setSwitchingConstraintDimension(ns);
  put_m(impact ? cd.dIDddv : cd.dIDda, lin + S.l_M, nv, nv, nv);
  put_m(cd.dCda(), lin + S.l_J, nf, nv, nfm);
  put_m(cd.dIDCdqv(), lin + S.l_D, nvf, nx, nvfm);
  put_v(cd.IDC(), lin + S.l_IDC, nvf);
  if (!impact && np > 0) put_v(cd.lu_passive, lin + S.l_lup, np);
  StateEquationData se(robot);
  if (np == 6) {
    put_m(se.Fqq_prev.topLeftCorner(6, 6), lin + S.l_se3 + 36, 6, 6, 6);
    Eigen::MatrixXd cur(6, 6);
    put_m(cur, lin + S.l_se3 + 72, 6, 6, 6);
    robot.injectdSubtractConfiguration_dq0(cur);
  }
  // ---- constraints: slack, dual, residual from the PDIPM record; cmpl as evalConstraint leaves it (pdipm.hxx:27-63)
  std::shared_ptr<Constraints> constraints = make_constraints(robot, tab);
  // GridInfo::stage decides which constraint levels act (ConstraintsData::setTimeStage, constraints_data.cpp:20-45); the control
  // word carries max(0, 2 - stage)
  ConstraintsData cdata = constraints->createConstraintsData(robot, impact ? -1 : 2 - c->ineq_gate);
  auto comp_valid = [&](int k) { return k >= 4 || (k >= 2 ? c->ineq_gate <= 1 : c->ineq_gate == 0); };
  const int nj = nu;  // rows per joint-limit component
  if (!impact) {
    for (int k = 0; k < 7; ++k) {
      ConstraintComponentData& cc = component(cdata, k);
      const int off = k * nj, n = (k < 6) ? nj : 5 * tab->n_contacts;
      put_v(cc.slack, con + S.c_slack + off, n);
      put_v(cc.dual, con + S.c_dual + off, n);
      put_v(cc.residual, con + S.c_res + off, n);
      if (k < 6) {
        pdipm::computeComplementarySlackness(tab->barrier, cc);
      } else {
        cc.cmpl.setZero();
        for (int ci = 0; ci < tab->n_contacts; ++ci) {
          if (!((c->contact_mask >> ci) & 1)) {
            cc.residual.template segment<5>(5 * ci).setZero();  // FrictionCone::evalConstraint zeroes inactive contacts (:122-123)
            continue;
          }
          pdipm::computeComplementarySlackness<5>(tab->barrier, cc, 5 * ci);
          put_m(cc.J[ci], lin + S.l_dgdq + size_t(ci) * 5 * nv, 5, nv, 5);                       // dg_dq
          put_m(cc.J[tab->n_contacts + ci], lin + S.l_dgdf + size_t(ci) * 15, 5, 3, 5);          // dg_df
        }
      }
    }
  }
  const bool icone = impact && tab->impact_friction_cone;
  if (icone) {  // the ImpactFrictionCone component: same record rows, same J slots (impact_friction_cone.hpp:140-148)
    ConstraintComponentData& cc = cdata.impact_level_data[0];
    const int off = 6 * nj, n = 5 * tab->n_contacts;
    put_v(cc.slack, con + S.c_slack + off, n);
    put_v(cc.dual, con + S.c_dual + off, n);
    put_v(cc.residual, con + S.c_res + off, n);
    cc.cmpl.setZero();
    for (int ci = 0; ci < tab->n_contacts; ++ci) {
      if (!((c->contact_mask >> ci) & 1)) {
        cc.residual.template segment<5>(5 * ci).setZero();  // ImpactFrictionCone::evalConstraint zeroes inactive contacts
        continue;
      }
      pdipm::computeComplementarySlackness<5>(tab->barrier, cc, 5 * ci);
      put_m(cc.J[ci], lin + S.l_dgdq + size_t(ci) * 5 * nv, 5, nv, 5);
      put_m(cc.J[tab->n_contacts + ci], lin + S.l_dgdf + size_t(ci) * 15, 5, 3, 5);
    }
  }
  {  // PerformanceIndex as evalKKT summarises it before condensing: log barrier per valid component (what evalConstraint
     // accumulates, constraint_component_base / friction_cone.cpp:122-139), then the members of OCPData and SplitKKTResidual
    for (int k = 0; k < 6; ++k) component(cdata, k).log_barrier = pdipm::logBarrier(tab->barrier, component(cdata, k).slack);
    ConstraintComponentData& cone = impact ? (icone ? cdata.impact_level_data[0] : component(cdata, 6)) : component(cdata, 6);
    cone.log_barrier = 0.0;
    for (int ci = 0; ci < tab->n_contacts; ++ci)
      if ((c->contact_mask >> ci) & 1) cone.log_barrier += pdipm::logBarrier(tab->barrier, cone.slack.template segment<5>(5 * ci));
    g_last_perf[0] = cdata.logBarrier();
    g_last_perf[1] = cdata.primalFeasibility<1>() + cd.primalFeasibility<1>() + kr.primalFeasibility<1>();
    g_last_perf[2] = cdata.dualFeasibility<1>() + cd.dualFeasibility<1>() + kr.dualFeasibility<1>();
    g_last_perf[3] = cdata.KKTError() + cd.KKTError() + kr.KKTError();
  }
  // ---- "Forms linear system"
  SplitSolution s_dummy(robot), s_next_dummy(robot);
  if (!impact) {
    constraints->condenseSlackAndDual(contact_status, cdata, km, kr);
    condenseContactDynamics(robot, contact_status, c->dt, cd, km, kr);
    correctLinearizeStateEquation(robot, c->dt, s_dummy, s_next_dummy, se, km, kr);
    const double g1 = 1.0 / c->ngrids_in_phase;                    // intermediate_stage.cpp:140-148
    kr.h *= g1;
    km.hx.array() *= g1;
    km.hu.array() *= g1;
    km.fx.array() *= g1;
    km.Qtt *= g1 * g1;
    km.Qtt_prev = -km.Qtt;
    if (ns > 0) km.Phit().array() *= g1;
  } else {
    constraints->condenseSlackAndDual(impact_status, cdata, km, kr);
    condenseImpactDynamics(robot, impact_status, cd, km, kr);
    correctLinearizeImpactStateEquation(robot, s_dummy, s_next_dummy, se, km, kr);
  }
  // ---- pack: KKT record, expansion record, PDIPM cmpl | cond
  get_m(km.Fxx, kkt + K.k_Fxx, nx, nx, nx);
  get_m(km.Qxx, kkt + K.k_Qxx, nx, nx, nx);
  get_v(kr.Fx, kkt + K.k_Fx, nx);
  get_v(kr.lx, kkt + K.k_lx, nx);
  get_m(cd.MJtJinv(), ex + S.e_Z, nvf, nvf, nvfm);
  get_m(cd.MJtJinv_dIDCdqv(), ex + S.e_R, nvf, nx, nvfm);
  get_v(cd.MJtJinv_IDC(), ex + S.e_r, nvf);
  get_m(cd.Qafqv(), ex + S.e_Qafqv, nvf, nx, nvfm);
  get_v(cd.laf(), ex + S.e_laf, nvf);
  if (np == 6) get_m(se.Fqq_prev_inv, ex + S.e_Fqqpi, 6, 6, 6);
  if (!impact) {
    get_m(km.Fvu, kkt + K.k_Fvu, nv, nu, nv);
    get_m(km.Qxu, kkt + K.k_Qxu, nx, nu, nx);
    get_m(km.Quu, kkt + K.k_Quu, nu, nu, nu);
    get_v(kr.lu, kkt + K.k_lu, nu);
    get_v(km.fx, kkt + K.k_fx, nx);
    get_v(km.hx, kkt + K.k_hx, nx);
    get_v(km.hu, kkt + K.k_hu, nu);
    kkt[K.k_sc + 0] = km.Qtt; kkt[K.k_sc + 1] = km.Qtt_prev; kkt[K.k_sc + 2] = kr.h;
    if (ns > 0) {
      get_m(km.Phix(), kkt + K.k_Phix, ns, nx, ns);
      get_m(km.Phiu(), kkt + K.k_Phiu, ns, nu, ns);
      get_v(kr.P(), kkt + K.k_p, ns);
      get_v(km.Phit(), kkt + K.k_Phit, ns);
      get_m(cd.Phia(), ex + S.e_Phia, ns, nv, ns);
    }
    get_m(cd.Qafu_full(), ex + S.e_Qafu, nvf, nv, nvfm);
    get_v(cd.haf(), ex + S.e_haf, nvf);
    if (np > 0) {
      get_m(cd.Qxu_passive, ex + S.e_Qxup, nx, np, nx);
      get_m(cd.Quu_passive_topRight, ex + S.e_Quup, np, nu, np);
      get_v(cd.lu_passive, ex + S.e_lup, np);
    }
    for (int k = 0; k < 7; ++k) {
      if (!comp_valid(k)) continue;  // the reference does not touch the data of a level that is not valid on this grid point
      ConstraintComponentData& cc = component(cdata, k);
      const int off = k * nj, n = (k < 6) ? nj : 5 * tab->n_contacts;
      get_v(cc.cmpl, con + S.c_cmpl + off, n);
      get_v(cc.cond, con + S.c_cond + off, n);
    }
  }
  if (icone) {
    ConstraintComponentData& cc = cdata.impact_level_data[0];
    get_v(cc.cmpl, con + S.c_cmpl + 6 * nj, 5 * tab->n_contacts);
    get_v(cc.cond, con + S.c_cond + 6 * nj, 5 * tab->n_contacts);
  }
  if (phase < 2) return 0;

  // ---- primal expansion + step sizes
  SplitDirection dd(robot), dn(robot);
  dd.setContactDimension(nf);
  dd.setSwitchingConstraintDimension(ns);
  put_v(dd.dx, d + K.d_dx, nx);
  put_v(dd.dlmdgmm, d + K.d_dlmdgmm, nx);
  dd.dts = d[K.d_dts];
  dd.dts_next = d[K.d_dts + 1];
  if (!impact) {
    put_v(dd.du, d + K.d_du, nu);
    if (ns > 0) put_v(dd.dxi(), d + K.d_dxi, ns);
    expandContactDynamicsPrimal(cd, dd);
    constraints->expandSlackAndDual(contact_status, cdata, dd);
  } else {
    expandImpactDynamicsPrimal(cd, dd);
    constraints->expandSlackAndDual(impact_status, cdata, dd);
  }
  get_v(impact ? dd.ddvf() : dd.daf(), xd + S.x_daf, nvf);
  steps_stage[0] = constraints->maxSlackStepSize(cdata);
  steps_stage[1] = constraints->maxDualStepSize(cdata);
  if (!impact)
    for (int k = 0; k < 7; ++k) {
      if (!comp_valid(k)) continue;
      ConstraintComponentData& cc = component(cdata, k);
      const int off = k * nj, n = (k < 6) ? nj : 5 * tab->n_contacts;
      get_v(cc.dslack, con + S.c_dslack + off, n);
      get_v(cc.ddual, con + S.c_ddual + off, n);
    }
  if (icone) {
    ConstraintComponentData& cc = cdata.impact_level_data[0];
    get_v(cc.dslack, con + S.c_dslack + 6 * nj, 5 * tab->n_contacts);
    get_v(cc.ddual, con + S.c_ddual + 6 * nj, 5 * tab->n_contacts);
  }
  if (phase < 3) return 0;

  // ---- dual expansion, costate correction, slack / dual update
  put_v(dn.dlmdgmm, d_next + K.d_dlmdgmm, nx);
  if (!impact) {
    double dts = 0.0;
    if (c->ngrids_in_phase > 0) dts = (dd.dts_next - dd.dts) / c->ngrids_in_phase;   // intermediate_stage.cpp:168-171
    expandContactDynamicsDual(c->dt, dts, cd, dn, dd);
  } else {
    expandImpactDynamicsDual(cd, dn, dd);
  }
  correctCostateDirection(se, dd);
  get_v(cd.laf(), ex + S.e_laf, nvf);  // expand*Dual completes laf / ldvf in place (contact_dynamics.cpp:180-188, impact_dynamics.cpp:92-94)
  get_v(dd.dbetamu(), xd + S.x_dbetamu, nvf);
  if (!impact && np > 0) get_v(dd.dnu_passive, xd + S.x_dnup, np);
  get_v(dd.dlmdgmm, d + K.d_dlmdgmm, nx);
  if (!impact) {
    Constraints::updateSlack(cdata, alpha_p);
    Constraints::updateDual(cdata, alpha_d);
    for (int k = 0; k < 7; ++k) {
      if (!comp_valid(k)) continue;
      ConstraintComponentData& cc = component(cdata, k);
      const int off = k * nj, n = (k < 6) ? nj : 5 * tab->n_contacts;
      get_v(cc.slack, con + S.c_slack + off, n);
      get_v(cc.dual, con + S.c_dual + off, n);
    }
  }
  if (icone) {  // ImpactStage::updatePrimal / updateDual (impact_stage.cpp:151-165)
    Constraints::updateSlack(cdata, alpha_p);
    Constraints::updateDual(cdata, alpha_d);
    ConstraintComponentData& cc = cdata.impact_level_data[0];
    get_v(cc.slack, con + S.c_slack + 6 * nj, 5 * tab->n_contacts);
    get_v(cc.dual, con + S.c_dual + 6 * nj, 5 * tab->n_contacts);
  }
  return 0;
}

// Constraints::linearizeConstraints (constraints.cpp:283-306) over the six joint-limit components of the reference, for one grid
// point: residual of the valid levels -> con (c_res rows), gradient terms -> the lx / la / lu sections of the linearization record.
// bound: limit of each box row in the table order of make_constraints (q lower | q upper | v lower | v upper | u lower | u upper;
// the reference's velocity / torque limits are symmetric: bound[v lower] == -bound[v upper]).
int ref_linearize_joint_limits(const rbt_stage_dims* sd, const rbt_constraint_table* tab, const rbt_stage_ctrl* c, const double* bound,
                               const double* sol, double* lin, double* con) {
  rbt_stage_layout S;
  rbt_make_stage_layout(sd, &S);
  const int nv = S.nv, nu = S.nu, nx = S.nx, np = S.np;
  if (c->type == RBT_TERMINAL || c->type == RBT_IMPACT) return 0;
  Robot robot(nv, np == 6, tab->n_contacts);
  Eigen::VectorXd effort(nu), velocity(nu), qmin(nu), qmax(nu);
  for (int j = 0; j < nu; ++j) {
    qmin(j) = bound[j]; qmax(j) = bound[nu + j];
    velocity(j) = bound[3 * nu + j]; effort(j) = bound[5 * nu + j];
    if (bound[2 * nu + j] != -velocity(j) || bound[4 * nu + j] != -effort(j)) return 1;
  }
  robot.setJointLimits(effort, velocity, qmin, qmax);
  auto constraints = std::make_shared<Constraints>(tab->barrier, tab->fraction_to_boundary);
  constraints->add("joint_position_lower", std::make_shared<JointPositionLowerLimit>(robot));
  constraints->add("joint_position_upper", std::make_shared<JointPositionUpperLimit>(robot));
  constraints->add("joint_velocity_lower", std::make_shared<JointVelocityLowerLimit>(robot));
  constraints->add("joint_velocity_upper", std::make_shared<JointVelocityUpperLimit>(robot));
  constraints->add("joint_torques_lower", std::make_shared<JointTorquesLowerLimit>(robot));
  constraints->add("joint_torques_upper", std::make_shared<JointTorquesUpperLimit>(robot));
  ConstraintsData cdata = constraints->createConstraintsData(robot, 2 - c->ineq_gate);
  auto comp = [&](int k) -> ConstraintComponentData& {
    return k < 2 ? cdata.position_level_data[k] : (k < 4 ? cdata.velocity_level_data[k - 2] : cdata.acceleration_level_data[k - 4]);
  };
  for (int k = 0; k < 6; ++k) {
    put_v(comp(k).slack, con + S.c_slack + k * nu, nu);
    put_v(comp(k).dual, con + S.c_dual + k * nu, nu);
  }
  SplitSolution s(robot);
  put_v(s.q, sol + S.s_q, S.nq);
  put_v(s.v, sol + S.s_v, nv);
  put_v(s.a, sol + S.s_a, nv);
  put_v(s.u, sol + S.s_u, nu);
  SplitKKTResidual kr(robot);
  put_v(kr.lx, lin + S.l_lx, nx);
  put_v(kr.la, lin + S.l_la, nv);
  put_v(kr.lu, lin + S.l_lu, nu);
  ContactStatus contact_status = robot.createContactStatus();
  constraints->linearizeConstraints(robot, contact_status, cdata, s, kr);
  get_v(kr.lx, lin + S.l_lx, nx);
  get_v(kr.la, lin + S.l_la, nv);
  get_v(kr.lu, lin + S.l_lu, nu);
  for (int k = 0; k < 6; ++k) {
    const bool valid = k >= 4 || (k >= 2 ? c->ineq_gate <= 1 : c->ineq_gate == 0);
    if (valid) get_v(comp(k).residual, con + S.c_res + k * nu, nu);
  }
  return 0;
}

// robotoc::LineSearchFilter (src/line_search/line_search_filter.cpp, compiled unmodified) driven like
// LineSearch::lineSearchFilterMethod drives it (line_search.cpp:58-86) for ONE OCP over `rounds` consecutive line searches with
// n_trials pre-evaluated candidates each: cost0/viol0 [rounds], cost/viol [rounds][n_trials] (barrier already included).
// out_step[round], out_k[round].
int ref_filter_line_search(int rounds, int n_trials, double rate, double min_step, double cost_rate, double viol_rate,
                           const double* alpha_max, const double* cost0, const double* viol0, const double* cost, const double* viol,
                           double* out_step, int* out_k) {
  robotoc::LineSearchFilter filter(cost_rate, viol_rate);
  for (int r = 0; r < rounds; ++r) {
    if (filter.isEmpty()) filter.augment(cost0[r], viol0[r]);
    double alpha = alpha_max[r];
    int k = 0, acc = -1;
    while (alpha > min_step && k < n_trials) {
      const double c = cost[size_t(r) * n_trials + k], v = viol[size_t(r) * n_trials + k];
      if (filter.isAccepted(c, v)) {
        filter.augment(c, v);
        acc = k;
        break;
      }
      alpha *= rate;
      ++k;
    }
    out_step[r] = alpha;
    out_k[r] = acc;
  }
  return 0;
}

}  // extern "C"
