/*
 * robotoc_b200.h -- C ABI of the H100-native Riccati / KKT inner loop (librobotoc_b200.so).
 *
 * This is the drop-in boundary behind robotoc::OCPSolver / UnconstrOCPSolver.  The reference has no
 * FFI seam; the seam is the C++ member API of its solver classes.  Every entry point below names
 * the reference interface it replaces (paths relative to the reference tree, commit d30d404).
 *
 * Conventions
 *  - plain C types only: opaque handle, int return codes (0 = RBT_OK), double* buffers, void* stream
 *    (a cudaStream_t; NULL = the legacy default stream).  No C++/torch types cross this boundary.
 *  - all arithmetic is IEEE fp64; records are laid out by rbt_layout.h, arrays are [batch][grid][record].
 *  - "host" pointers may be pageable or pinned; "dev" pointers are CUDA device pointers on the handle's
 *    device.  All work is stream-ordered; call rbt_sync() (or synchronise the stream) before reading
 *    host outputs.
 *  - there is NO CPU fallback: every compute entry point fails with RBT_ERR_CUDA if no usable
 *    sm_90 device is present.
 */
#ifndef ROBOTOC_B200_H_
#define ROBOTOC_B200_H_

#include "rbt_layout.h"
#include "rbt_stage_layout.h"
#include "rbt_ustage_layout.h"

#ifdef __cplusplus
extern "C" {
#endif

enum {
  RBT_OK = 0,
  RBT_ERR_ARG = 1,     /* invalid argument (reference: std::out_of_range / std::invalid_argument, ocp_solver.cpp:29-49) */
  RBT_ERR_CUDA = 2,    /* CUDA runtime / no device */
  RBT_ERR_STATE = 3,   /* call order (e.g. no schedule set) */
  RBT_ERR_NUMERIC = 4  /* non-positive pivot met in a Cholesky (reference: assert(llt_.info()==Success), riccati_factorizer.cpp:50) */
};

/* which buffer, for rbt_dev_ptr / rbt_download / rbt_upload */
enum {
  RBT_BUF_KKT = 0,   /* KKT records          (input)  */
  RBT_BUF_RIC = 1,   /* Riccati records      (output of backward) */
  RBT_BUF_FACT = 2,  /* factorized KKT F,H,G,lu (optional output of backward; the reference mutates kkt in place) */
  RBT_BUF_DIR = 3,   /* direction records    (output of forward) */
  RBT_BUF_DX0 = 4,   /* initial state direction dx0, [batch][nx] (input of forward) */
  RBT_BUF_INFO = 5,  /* per-OCP int status flags, [batch] (as doubles are not used: int32) */
  /* stage layer (rbt_stage_setup): records of include/rbt_stage_layout.h */
  RBT_BUF_LIN = 6,   /* linearization records (input of condensing) */
  RBT_BUF_CON = 7,   /* PDIPM records: slack, dual, residual in; cmpl, cond, dslack, ddual out; slack, dual updated */
  RBT_BUF_EXP = 8,   /* expansion records (MJtJinv, MJtJinv_dIDCdqv, ... kept by condensing for the expansion) */
  RBT_BUF_SOL = 9,   /* solution records (q, v, a, dv, u, f, lmd, gmm, beta, mu, nu_passive, xi), updated in place */
  RBT_BUF_XDIR = 10, /* expanded direction records (daf, dbetamu, dnu_passive) */
  RBT_BUF_STEPS = 11,/* [batch][2] max primal / dual step size over the horizon */
  RBT_BUF_PERF = 12, /* [batch][8] PerformanceIndex of rbt_eval_kkt: {cost (0: not evaluated on this path), cost_barrier,
                        primal_feasibility, dual_feasibility, kkt_error, sqrt(kkt_error) = OCPSolver::KKTError(), 0, 0} */
  RBT_BUF_CONTACT_POS = 13, /* [batch][n_grid][n_contacts][3] desired contact positions of rbt_linearize_contact_kinematics
                               (ContactStatus::contactPosition of each grid point's phase); allocated by its first upload */
  RBT_BUF_Q0 = 14           /* [batch][nq] measured configuration q0 of OCPSolver::solve(t, q, v), the q_prev of grid point 0 in
                               rbt_linearize_state_equation; allocated by its first upload */
};

typedef struct rbt_handle rbt_handle;

/* Layout query by field name (e.g. "k_Fxx", "r_stride"); returns -1 for an unknown name. */
int rbt_layout_get(const rbt_dims* dims, const char* field);
int rbt_ulayout_get(int nv, const char* field);

/* Library / device probe: returns RBT_OK and fills sm (e.g. 100) and n_sm when a CUDA device is usable. */
int rbt_device_info(int device, int* sm, int* n_sm, char* name, int name_len);
const char* rbt_version(void);

/* ---------------------------------------------------------------------------------------------
 * Constrained path -- replaces robotoc::RiccatiRecursion
 *   ctor RiccatiRecursion(const OCP&, double max_dts0)            include/robotoc/riccati/riccati_recursion.hpp:35
 *   (data sized N+1+reserved events; here n_grid_max)             src/riccati/riccati_recursion.cpp:10-16
 * --------------------------------------------------------------------------------------------- */
int rbt_create(const rbt_dims* dims, int n_grid_max, int batch, int device, rbt_handle** out);
int rbt_destroy(rbt_handle* h);

/* Stage control table for the whole horizon (n_grid = time_discretization.size(), i.e. N+1 grid points,
 * last one Terminal) and the STO regularisation.
 *   replaces: the TimeDiscretization& argument of backward/forwardRiccatiRecursion (riccati_recursion.hpp:66-84)
 *             and RiccatiRecursion::setRegularization(max_dts0)   (riccati_recursion.hpp:58) */
int rbt_set_schedule(rbt_handle* h, const rbt_stage_ctrl* ctrl, int n_grid, double max_dts0);

/* Device buffers owned by the handle (so a GPU producer can fill KKT records in place). */
double* rbt_dev_ptr(rbt_handle* h, int which);
long long rbt_buf_doubles(rbt_handle* h, int which); /* size of that buffer in doubles for the current schedule */

/* Use a caller-owned device buffer (>= rbt_buf_doubles(h, which) doubles) instead of the handle's own; NULL restores
 * the internal one.  The reference's solver owns its containers (OCPSolver members kkt_matrix_, riccati_factorization_,
 * d_; include/robotoc/solver/ocp_solver.hpp:219-236); this lets a GPU front-end or an NCCL all-gather work in place. */
int rbt_bind_buffer(rbt_handle* h, int which, double* dev);

/* RBT_BUF_KKT, RBT_BUF_DX0, RBT_BUF_LIN, RBT_BUF_CON (input fields slack | dual | residual only), RBT_BUF_SOL */
int rbt_upload(rbt_handle* h, int which, const double* host, void* stream);
int rbt_download(rbt_handle* h, int which, double* host, void* stream);       /* any output buffer */
/* bytes rbt_upload(h, which, ..) actually moves host->device (KKT uploads skip record padding and, on stages without
 * a switching constraint / STO, the unused switching+STO sections) */
long long rbt_upload_bytes(rbt_handle* h, int which);
int rbt_download_info(rbt_handle* h, int* host_flags, void* stream);          /* per-OCP Cholesky status */
/* Synchronises `stream` and turns the per-OCP flags into a return code: RBT_OK if every factorization of the last
 * condense / backward sweep succeeded, RBT_ERR_NUMERIC otherwise (rbt_last_error names the first failing OCP and the flag:
 * 1 = Quu + B^T P B not positive definite, 2 = switching-constraint Schur complement, 4 = M, 8 = J M^-1 J^T in the
 * condensing).  The reference only asserts here (assert(llt_.info() == Eigen::Success), riccati_factorizer.cpp:50,64):
 * the other OCPs of the batch are unaffected and their results are valid.  *first_bad (may be NULL) = index or -1. */
int rbt_check_info(rbt_handle* h, int* first_bad, void* stream);

/* Structure of the state-equation blocks Fxx of the KKT records handed to rbt_riccati_backward.  Every linearisation robotoc
 * produces has Fqq = I and Fqv = dt I outside their top-left dim_passive x dim_passive blocks (src/dynamics/state_equation.cpp:
 * 52-55 and, for a floating base, :68-87; impact stages: Fqv = 0, impact_state_equation.cpp) -- the backward sweep has an
 * instance that skips those rows of the two nx^3 products.  RBT_FXX_AUTO (default): the records are inspected on the device at
 * every sweep and the general instance runs if any Fxx deviates (records written by rbt_condense are known to conform and are
 * not inspected).  RBT_FXX_MECHANICAL: the caller guarantees the structure (no inspection).  RBT_FXX_GENERAL: arbitrary Fxx. */
enum { RBT_FXX_AUTO = 0, RBT_FXX_MECHANICAL = 1, RBT_FXX_GENERAL = 2 };
int rbt_set_fxx_structure(rbt_handle* h, int mode);

/* Time-parallel Riccati sweeps.  Without switching-time optimisation the backward sweep carries only (P, s) from grid i+1 to
 * grid i and the forward sweep only dx (src/riccati/riccati_recursion.cpp:32-131 with every sto flag false), so the horizon
 * can be split into `segments` contiguous pieces that run on separate CTAs: the (P, s) at every segment end comes from an
 * associative combine of per-stage value-function elements and dx at every segment start from composed closed-loop maps,
 * then each segment runs the serial per-stage algebra.  Same outputs up to rounding; worth it only when the batch leaves
 * most SMs idle.  0 = automatic (default: chosen from the handle's batch, the SM count and the schedule), 1 = serial,
 * k > 1 = k segments.  Returns RBT_ERR_ARG for k > n_grid - 1 of the current schedule (set the schedule first) or for k > 1 on
 * a schedule with switching-time optimisation; such schedules always run serially, and a later schedule with fewer stages
 * clamps k.  Applies to rbt_riccati_backward / forward and every host path built on them. */
int rbt_set_time_segments(rbt_handle* h, int segments);

/* RiccatiRecursion::backwardRiccatiRecursion(time_discretization, kkt_matrix, kkt_residual, factorization)
 *   src/riccati/riccati_recursion.cpp:32-80.  Reads RBT_BUF_KKT, writes RBT_BUF_RIC (P,s,K,k,M,m,STO terms,
 *   STOPolicy) and, if write_fact != 0, RBT_BUF_FACT (the values the reference leaves in Qxx,Qxu,Quu,lu). */
int rbt_riccati_backward(rbt_handle* h, int write_fact, void* stream);

/* RiccatiRecursion::forwardRiccatiRecursion(time_discretization, kkt_matrix, kkt_residual, factorization, d)
 *   src/riccati/riccati_recursion.cpp:83-131.  Reads RBT_BUF_KKT, RBT_BUF_RIC, RBT_BUF_DX0; writes RBT_BUF_DIR. */
int rbt_riccati_forward(rbt_handle* h, void* stream);

/* One call with HOST buffers: upload kkt + dx0, backward, forward, download what is asked for (NULL = skip).
 * This is the call an OCPSolver::updateSolution (src/solver/ocp_solver.cpp:118-123) adaptor makes. */
int rbt_riccati_solve_host(rbt_handle* h, const double* kkt_host, const double* dx0_host, double* ric_host,
                           double* dir_host, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Stage layer -- the condensing tail of evalKKT and the expansion / step-size / update half of
 * robotoc::DirectMultipleShooting (include/robotoc/ocp/direct_multiple_shooting.hpp:86-199)
 * --------------------------------------------------------------------------------------------- */
int rbt_stage_layout_get(const rbt_stage_dims* sdims, const char* field);
/* Allocates the stage-layer buffers.  `table` = the constraints of the OCP (robotoc::Constraints with its joint limits
 * and friction cones, src/constraints/constraints.cpp); barrier / fraction-to-boundary as in constraint_component_base.hpp:44-45. */
int rbt_stage_setup(rbt_handle* h, const rbt_stage_dims* sdims, const rbt_constraint_table* table);
/* "Forms linear system" of {Intermediate,Impact,Terminal}Stage::evalKKT (intermediate_stage.cpp:133-148, impact_stage.cpp:115-121,
 * terminal_stage.cpp:102-106): Constraints::condenseSlackAndDual, condenseContactDynamics / condenseImpactDynamics,
 * correctLinearizeStateEquation, STO scaling.  Reads RBT_BUF_LIN, RBT_BUF_CON; writes RBT_BUF_KKT, RBT_BUF_EXP, RBT_BUF_CON. */
int rbt_condense(rbt_handle* h, void* stream);
/* Measurement aid: rbt_condense issues two kernels (MJtJinv, then the condensing proper); a caller-owned cudaEvent_t given
 * here is recorded between them so each can be timed on its own (NULL switches it off). */
int rbt_set_condense_event(rbt_handle* h, void* cuda_event);
/* DirectMultipleShooting::computeStepSizes + maxPrimalStepSize / maxDualStepSize (direct_multiple_shooting.cpp:174-209):
 * expandPrimal of every stage, slack/dual directions, fraction-to-boundary, min over the horizon.
 * Reads RBT_BUF_DIR, RBT_BUF_EXP, RBT_BUF_LIN; writes RBT_BUF_XDIR (daf), RBT_BUF_CON (dslack, ddual), RBT_BUF_STEPS. */
int rbt_expand_and_step_sizes(rbt_handle* h, void* stream);
/* DirectMultipleShooting::integrateSolution (direct_multiple_shooting.cpp:212-241) with the step sizes of RBT_BUF_STEPS:
 * expandDual, correctCostateDirection, SplitSolution::integrate, updateSlack / updateDual. */
int rbt_update(rbt_handle* h, void* stream);

/* The PerformanceIndex that {Intermediate,Impact,Terminal}Stage::evalKKT summarise before condensing and
 * DirectMultipleShooting::evalKKT sums over the horizon (src/ocp/intermediate_stage.cpp:128-132, impact_stage.cpp:109-113,
 * terminal_stage.cpp:97-100, src/ocp/direct_multiple_shooting.cpp:155-158): squared KKT error (SplitKKTResidual::KKTError,
 * split_kkt_residual.hxx:90-104, + contact dynamics + constraints), primal / dual feasibility (l1), log barrier
 * (pdipm.hxx:194-200) -- per OCP into RBT_BUF_PERF, whose entry 5 is OCPSolver::KKTError() (ocp_solver.cpp:429-431), the
 * quantity the SQP loop compares with kkt_tol (ocp_solver.cpp:183-208).  Reads RBT_BUF_LIN and RBT_BUF_CON as uploaded (it does
 * not depend on rbt_condense having run).  The stage cost itself belongs to the cost evaluation (out of scope): entry 0 is 0. */
int rbt_eval_kkt(rbt_handle* h, void* stream);
/* pdipm::setSlackAndDualPositive (include/robotoc/constraints/pdipm.hxx:13-24) on RBT_BUF_CON: slack <- max(slack, sqrt(barrier)),
 * dual <- barrier / slack -- what Constraints::setSlackAndDual applies when a solver is initialised (initConstraints). */
int rbt_set_slack_and_dual_positive(rbt_handle* h, void* stream);
/* SURVEY.md 8f-2, first slice -- the joint-limit half of Constraints::linearizeConstraints (src/constraints/constraints.cpp:283-306
 * over JointPosition / Velocity / Torques Lower / Upper Limit, joint_*_limit.cpp:47-63) on the device, from the solution records
 * the library already holds: for every box row whose level is valid on the grid point,
 *   residual = sign (x - bound) + slack  -> RBT_BUF_CON (evalConstraint),   l_x += sign dual -> the gradient section of RBT_BUF_LIN
 * (evalDerivatives).  A host that uses it uploads linearisation records whose gradients lack the joint-limit terms and PDIPM
 * residuals for the friction-cone rows only (those need frame kinematics).  rbt_set_joint_limits: bound_host[n_box] = the limit
 * of each box row of the constraint table (qmin / qmax, -vmax / vmax, -umax / umax of the robot model); call once.
 * Order: rbt_upload(LIN, CON, SOL) -> rbt_linearize_joint_limits -> rbt_eval_kkt / rbt_condense. */
int rbt_set_joint_limits(rbt_handle* h, const double* bound_host);
int rbt_linearize_joint_limits(rbt_handle* h, void* stream);

/* Robot model of the inverse-dynamics linearisation (SURVEY.md 8f-1, first slice): what pinocchio::Model holds for a floating-base
 * tree of revolute joints, in Pinocchio's depth-first joint order.  Body b is Pinocchio joint b + 1 (joint 0 is the universe):
 * body 0 is the free-flyer root, bodies 1 .. n_bodies-1 are revolute joints.  All frames are Pinocchio's joint frames.
 *   parent[b]            parent body (parent[0] = -1, else 0 <= parent[b] < b)               model.parents[b+1] - 1
 *   axis[b]              unit rotation axis of a revolute joint in its own frame (body 0: unused)  JointModelRevolute(Unaligned) axis
 *   placement[b]         joint frame in the parent joint frame: R (column-major 3x3) | p     model.jointPlacements[b+1]
 *   mass, com, inertia   Inertia of the body with the children of fixed joints merged in, rotational inertia about the centre of
 *                        mass (column-major 3x3, symmetric positive definite)               model.inertias[b+1]
 *   contact_parent[c], contact_placement[c]   parent body and placement jXf of point contact c    PointContact (point_contact.cpp)
 *   gravity              model.gravity.linear()
 * n_bodies = nv - 5 (six free-flyer velocities + one per revolute joint). */
#define RBT_MAX_BODIES 32
typedef struct rbt_robot_model {
  int nv, n_bodies, n_contacts, pad_;
  int parent[RBT_MAX_BODIES];
  double axis[RBT_MAX_BODIES][3];
  double placement[RBT_MAX_BODIES][12];
  double mass[RBT_MAX_BODIES];
  double com[RBT_MAX_BODIES][3];
  double inertia[RBT_MAX_BODIES][9];
  int contact_parent[RBT_MAX_CONTACTS];
  double contact_placement[RBT_MAX_CONTACTS][12];
  double gravity[3];
} rbt_robot_model;
/* Copies the model to the device; call once after rbt_stage_setup.  RBT_ERR_ARG if nv or n_contacts disagree with the handle,
 * a parent is not earlier in the order, a mass is not positive, an inertia is not symmetric positive definite or an axis is not
 * a unit vector (rbt_last_error names the entry). */
int rbt_set_robot_model(rbt_handle* h, const rbt_robot_model* model);
/* The inverse-dynamics rows of linearizeContactDynamics (src/dynamics/contact_dynamics.cpp:22-44: Robot::setContactForces, RNEA,
 * RNEADerivatives, robot.hxx:494-580, fext[parent] = jXf.act(Force(f, 0)) per active point contact, point_contact.cpp:55-60) on
 * Intermediate and Lift grid points and of linearizeImpactDynamics (impact_dynamics.cpp:17-35: RNEAImpact /
 * RNEAImpactDerivatives, robot.hxx:589-622 -- v = 0, dv for a, the impulse as external force, no gravity) on Impact grid points,
 * from q, v, a | dv, f, beta of RBT_BUF_SOL.  Writes into RBT_BUF_LIN: the nv ID rows of IDC (RNEA - [0; u]; impact: RNEA),
 * the ID rows [dIDdq | dIDdv] of dIDCdqv (impact: [dIDdq | 0]), M = dIDda (impact: dIDddv), symmetrised from its upper
 * triangle like Robot::RNEADerivatives, and adds lq += dIDdq^T beta, lv += dIDdv^T beta, la (impact: ldv) += M^T beta
 * (contact_dynamics.cpp:31-33, impact_dynamics.cpp:24-25).  Derivatives in q are taken in the tangent space, q (+) dq =
 * integrate(q, dq) with the free flyer as [p | quaternion xyzw] and the local SE(3) exponential.  Terminal grid points are
 * untouched.  Order: rbt_upload(LIN, CON, SOL) -> (rbt_linearize_joint_limits) -> rbt_linearize_inverse_dynamics ->
 * rbt_eval_kkt / rbt_condense; the uploaded records' ID sections are ignored and their gradients lack the beta terms.
 * RBT_ERR_STATE before rbt_set_robot_model. */
int rbt_linearize_inverse_dynamics(rbt_handle* h, void* stream);
/* Baumgarte gains of the point contacts (SURVEY.md 8f-1, second slice): gains_host[n_contacts][2] = {baumgarte_position_gain,
 * baumgarte_velocity_gain} of ContactModelInfo (include/robotoc/robot/contact_model_info.hpp), as each PointContact holds them
 * (point_contact.hxx:29-33).  RBT_ERR_ARG if a gain is negative or not finite (PointContact's constructor throws,
 * src/robot/point_contact.cpp:27-34); RBT_ERR_STATE before rbt_stage_setup. */
int rbt_set_contact_gains(rbt_handle* h, const double* gains_host);
/* The contact rows of linearizeContactDynamics (src/dynamics/contact_dynamics.cpp:12-52: Robot::computeBaumgarteResidual /
 * computeBaumgarteDerivatives, robot.hxx:291-360, PointContact, point_contact.hxx:16-86) on Intermediate and Lift grid points,
 * kinematics at (q, v, a) without gravity (intermediate_stage.cpp:94), and of linearizeImpactDynamics (impact_dynamics.cpp:8-35:
 * computeImpactVelocityResidual / Derivatives, point_contact.hxx:89-117) on Impact grid points, kinematics at (q, v + dv)
 * (impact_stage.cpp:61,89).  Per active point contact, in contact order, three rows:
 *   Intermediate / Lift: C = a_cl + kv v_f,lin + kp (oMf.p - p_des) with a_cl = a_f,lin + w_f x v_f,lin (LOCAL frame),
 *                        p_des from RBT_BUF_CONTACT_POS; J = dC/da = J_lin; [dC/dq | dC/dv];
 *   Impact:              C = v_f,lin; J = dC/dv = J_lin; [dv_f,lin/dq | J_lin].
 * Writes J (ld nf_max), rows nv .. nv+nf-1 of dIDCdqv and of IDC into RBT_BUF_LIN, full width, and updates the gradients:
 * lf -= J beta, lq += dCdq^T mu, lv += dCdv^T mu, la (impact: ldv) += J^T mu (contact_dynamics.cpp:34-36,47-51,
 * impact_dynamics.cpp:27-31).  Derivatives in q in the tangent space, as rbt_linearize_inverse_dynamics.  Inactive rows,
 * grid points without contacts, terminal grid points and every other section are untouched.
 * Order: rbt_upload(LIN, CON, SOL) -> (rbt_linearize_joint_limits) -> (rbt_linearize_inverse_dynamics) ->
 * rbt_linearize_contact_kinematics -> rbt_eval_kkt / rbt_condense.  RBT_ERR_STATE until rbt_set_robot_model,
 * rbt_set_contact_gains and one rbt_upload(RBT_BUF_CONTACT_POS) have been made. */
int rbt_linearize_contact_kinematics(rbt_handle* h, void* stream);
/* The state-equation rows (SURVEY.md 8f-1, third slice): linearizeStateEquation (src/dynamics/state_equation.cpp:30-65) on
 * Intermediate and Lift grid points, linearizeImpactStateEquation (impact_state_equation.cpp:26-54) on Impact grid points and
 * linearizeTerminalStateEquation (terminal_state_equation.cpp:8-28) on the terminal one, with q_prev = q0 (RBT_BUF_Q0) on grid
 * point 0 and s[i-1].q otherwise, s_next = s[i+1] (direct_multiple_shooting.cpp:129-159).  Writes Fx = [Fq | Fv], the three
 * SE(3) blocks at l_se3 (Fqq = dSubtractConfiguration_dqf(q, q_next), Fqq_prev = dSubtractConfiguration_dq0(q_prev, q),
 * Fqq_cur = dSubtractConfiguration_dq0(q, q_next), state_equation.cpp:78) and, on the terminal grid point, Fqq_prev only; adds
 * the costate terms to lq, lv and la (impact: ldv); on schedules with a switching-time stage, Intermediate and Lift grid
 * points also get the STO terms: fx = [v | a] is written, lmd_next . v + gmm_next . a is added to h, lmd_next to hv and
 * gmm_next to ha.  Every other section is untouched.
 * Order: rbt_upload(LIN, SOL) -> (rbt_linearize_inverse_dynamics) -> (rbt_linearize_contact_kinematics) ->
 * rbt_linearize_state_equation -> rbt_eval_kkt / rbt_condense.  RBT_ERR_STATE before rbt_stage_setup or before one
 * rbt_upload(RBT_BUF_Q0). */
int rbt_linearize_state_equation(rbt_handle* h, void* stream);
/* computeInitialStateDirection (src/dynamics/state_equation.cpp:98-109) into RBT_BUF_DX0.  dq0_v0_host: [batch][2 nv] =
 * {q0 (-) s[0].q from Robot::subtractConfiguration (the robot model stays on the host), v0}; uses the stage-0 Fqq_prev_inv that
 * rbt_condense left in RBT_BUF_EXP and s[0].v of RBT_BUF_SOL, so call it after rbt_condense and before rbt_riccati_forward. */
int rbt_initial_state_direction(rbt_handle* h, const double* dq0_v0_host, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Line search (SURVEY.md 8f-3) -- the model-free half of robotoc::LineSearch::lineSearchFilterMethod
 * (src/line_search/line_search.cpp:58-86), with the backtracking step sizes alpha_k = alpha_max * rate^k as an extra batch axis.
 * rbt_line_search_trials: DirectMultipleShooting::integratePrimalSolution (direct_multiple_shooting.cpp:244-266) for n_trials
 *   step sizes at once, after rbt_expand_and_step_sizes (alpha_max = the max primal step of RBT_BUF_STEPS) and BEFORE rbt_update.
 *   Writes trial primal records [n_trials][batch][n_grid][rbt_trial_doubles() = 80] = {q (nq, padded to 20) | v | a or dv | u | f}
 *   on the device (rbt_line_search_trial_dev; also to trial_host if not NULL), alphas [n_trials][batch], and the log-barrier of
 *   the trial slacks (pdipm.hxx:194-200 on slack + alpha dslack) summed over the horizon, barrier [n_trials][batch].
 *   evalOCP at the trial points -- stage costs, dynamics residuals -- needs the robot model: the caller (or a GPU front-end)
 *   evaluates cost[k][b] and violation[k][b] from the trial records.
 * rbt_line_search_filter: LineSearchFilter (src/line_search/line_search_filter.cpp:25-56) per OCP over those evaluations:
 *   empty filter -> augment(cost0, violation0); the first trial k with alpha_k > min_step_size that the filter accepts is taken
 *   (and augments the filter), otherwise the first alpha_k <= min_step_size is returned -- exactly the reference's loop.
 *   cost_host excludes the barrier part (added here from rbt_line_search_trials).  The per-OCP filters persist across calls;
 *   rbt_line_search_clear_history = LineSearch::clearHistory. */
int rbt_trial_doubles(void);
int rbt_line_search_trials(rbt_handle* h, int n_trials, double step_size_reduction_rate, double* alphas_host, double* barrier_host,
                           double* trial_host, void* stream);
double* rbt_line_search_trial_dev(rbt_handle* h);
int rbt_line_search_filter(rbt_handle* h, int n_trials, double step_size_reduction_rate, double min_step_size,
                           double filter_cost_reduction_rate, double filter_constraint_violation_reduction_rate,
                           const double* cost0_host, const double* violation0_host, const double* cost_host,
                           const double* violation_host, double* step_host, int* accepted_trial_host, void* stream);
int rbt_line_search_clear_history(rbt_handle* h, void* stream);

/* One hot-path iteration with HOST buffers -- the linear-algebra body of OCPSolver::updateSolution
 * (src/solver/ocp_solver.cpp:118-144) given the stage linearisations: upload lin / con / sol / dx0, condense, backward and
 * forward Riccati, step sizes, update, download the updated solution, the PDIPM data and the step sizes (NULL = skip). */
int rbt_iteration_host(rbt_handle* h, const double* lin_host, const double* con_host, const double* sol_host,
                       const double* dx0_host, double* sol_out, double* con_out, double* steps_out, void* stream);
/* Bytes one rbt_iteration_host call moves over PCIe.  Only what the kernels read and what persists is moved: record padding
 * never, the switching-constraint section of a linearization record only on stages that carry one, of the PDIPM record
 * slack | dual | residual go up and the updated slack | dual come back (the other PDIPM fields are per-iteration scratch that
 * the reference keeps inside ConstraintComponentData; con_out's remaining fields are left untouched).  The call is
 * pipelined over chunks of the batch (upload of chunk c+1, kernels of chunk c, download of chunk c-1 overlap on three
 * streams); `stream` is ordered after the last download, so rbt_sync(h, stream) covers everything. */
int rbt_iteration_host_bytes(rbt_handle* h, int mode /* 0 dense records, 1 wire, 2 wire + resident state */, long long* h2d_bytes,
                             long long* d2h_bytes);
/* The same call with the linearization records in the host wire format of rbt_stage_layout.h: per grid point only what a
 * robotoc linearisation of that grid point holds -- packed upper triangles of the symmetric blocks M, Qff, Qxx, Quu; contact
 * blocks sized by the active contact dimension nf and the active contacts (as the reference's own dimf-sized containers); no
 * padding; no Qqf (zero until the friction-cone condensing fills it); the STO section only when the schedule has a
 * switching-time stage; Qxx, lx and one SE(3) block on the terminal grid point.  ANYmal trot N=40: 42 % fewer bytes over PCIe
 * than the dense records.  One OCP's wire records are concatenated in grid order: wire_host is [batch][rbt_wire_doubles].
 * `lin_host_switching` = classic records, of which only the switching-constraint sections of the stages that carry one are
 * read (NULL if the schedule has none).  rbt_pack_wire is the host-side packing helper (what an adaptor does while copying
 * out of SplitKKTMatrix::Qxx etc.; rbt_wire_layout_get gives the segment table of grid point i for an adaptor that fills the
 * wire records directly); `ctrl` / `n_grid` must be the schedule in force (rbt_set_schedule). */
int rbt_iteration_host_wire(rbt_handle* h, const double* wire_host, const double* lin_host_switching, const double* con_host,
                            const double* sol_host, const double* dx0_host, double* sol_out, double* con_out,
                            double* steps_out, void* stream);
/* The iteration as OCPSolver itself runs it: the solution s_ and the slack / dual variables are solver STATE (members of
 * OCPSolver / ConstraintComponentData that only updateSolution modifies), so they stay resident on the device between
 * iterations -- initialise them once with rbt_upload(RBT_BUF_SOL / RBT_BUF_CON) (or rbt_iteration_host_wire) -- and one
 * iteration moves only what the host recomputed at the new linearisation point: the wire records, the PDIPM residuals
 * res_host [batch][n_grid][ncp] (= g(x) + slack, ConstraintComponentData::residual; ncp = rbt_stage_layout.ncp) and dx0.
 * Back come (NULL = skip) the updated solution records sol_out [batch][n_grid][s_stride], the updated slack | dual
 * slack_dual_out [batch][n_grid][2 ncp] (compact: every transfer of this call is one contiguous DMA per chunk -- strided
 * 2-D copies of ~1 KB rows cost the copy engine as much per row as 4 KB of payload) and the step sizes. */
int rbt_iteration_host_resident(rbt_handle* h, const double* wire_host, const double* lin_host_switching, const double* res_host,
                                const double* dx0_host, double* sol_out, double* slack_dual_out, double* steps_out, void* stream);
/* cost_structure (RBT_COST_GENERAL / RBT_COST_ROBOTOC, rbt_stage_layout.h): with RBT_COST_ROBOTOC the wire records carry the
 * cost Hessians the way every cost component robotoc ships produces them -- Qqq dense, Qvv / Quu / Qff diagonal, Qqv = 0
 * (configuration_space_cost.cpp:308-322, task_space_*_cost.cpp, com_cost.cpp, local_contact_force_cost.cpp:130) -- 23 % fewer
 * bytes again; a problem with user-defined cost components that fill other entries uses RBT_COST_GENERAL (default).
 * rbt_set_wire_cost_structure tells the handle which of the two the host's wire records are in.
 * RBT_WIRE_DEVICE_ID OR-ed into cost_structure (rbt_stage_layout.h): the device computes the inverse-dynamics rows
 * (rbt_linearize_inverse_dynamics, after rbt_set_robot_model), so the wire records drop M, the ID rows of dIDCdqv and of IDC,
 * and their gradients lack the beta terms; rbt_iteration_host_wire / _resident run the kernel right after the unpack and
 * rbt_iteration_host_bytes counts the smaller records.  RBT_WIRE_DEVICE_CONTACT, alone or with RBT_WIRE_DEVICE_ID: the device
 * computes the contact rows (rbt_linearize_contact_kinematics, after rbt_set_robot_model, rbt_set_contact_gains and an upload of
 * RBT_BUF_CONTACT_POS), so the records drop J and the contact rows of dIDCdqv and IDC and their gradients lack the multiplier
 * terms of the contact rows; the kernel runs right after the inverse-dynamics kernel (or the unpack).  RBT_WIRE_DEVICE_STATE,
 * alone or with the other two: the device computes the state-equation rows (rbt_linearize_state_equation, after an upload of
 * RBT_BUF_Q0), so non-terminal records drop Fx and the three SE(3) blocks (144 doubles for nv = 18) and terminal records the
 * Fqq_prev block (36), and the gradients and the STO section lack the costate terms; the kernel runs last, after the
 * inverse-dynamics and the contact kernels (ID -> contact -> state, the order the gradient additions keep). */
int rbt_set_wire_cost_structure(rbt_handle* h, int cost_structure);
int rbt_wire_doubles(const rbt_stage_dims* sdims, const rbt_stage_ctrl* ctrl, int n_grid, int cost_structure);   /* doubles per OCP */
int rbt_wire_layout_get(const rbt_stage_dims* sdims, const rbt_stage_ctrl* ctrl, int n_grid, int cost_structure, int i,
                        rbt_wire_layout* out);
int rbt_pack_wire(const rbt_stage_dims* sdims, const rbt_stage_ctrl* ctrl, int n_grid, int cost_structure, const double* lin_host,
                  double* wire_host, long long n_ocps);

/* Multi-GPU (SURVEY.md 8e): OCP instances are independent, so a batch is sharded over ranks without any data-path collective;
 * the one exchange is the Newton step of every OCP on every rank, e.g. for a host that advances all trajectories.
 * rbt_allgather_step packs this rank's direction records to their used prefix -- rbt_step_doubles(h) = dx | du | dlmd,dgmm | dxi |
 * dts,dts_next per grid point (98 of the 112-double record stride for ANYmal) -- and issues ONE ncclAllGather on `stream`:
 * all_dev receives [nranks][batch][n_grid][rbt_step_doubles] doubles (device memory of this rank).  `nccl_comm` is the caller's
 * ncclComm_t; NCCL is looked up in the calling process (dlsym, then libnccl.so.2), the library does not link against it.
 * Put the call on its own stream to overlap it with the next iteration's condensing / backward sweep: the direction records are
 * only overwritten by the next rbt_riccati_forward. */
int rbt_step_doubles(rbt_handle* h);
/* only the packing ([batch][n_grid][rbt_step_doubles] doubles into packed_dev), for a host that owns the collective itself
 * (e.g. torch.distributed); the gather then reads the packed copy, so the next forward sweep need not wait for it */
int rbt_pack_step(rbt_handle* h, double* packed_dev, void* stream);
int rbt_allgather_step(rbt_handle* h, void* nccl_comm, double* all_dev, void* stream);

int rbt_sync(rbt_handle* h, void* stream);
const char* rbt_last_error(rbt_handle* h);
/* number of kernel launches issued by this handle since creation (bench.py's gpu_launches) */
long long rbt_launch_count(rbt_handle* h);

/* ---------------------------------------------------------------------------------------------
 * Unconstrained path -- replaces robotoc::UnconstrRiccatiRecursion
 *   include/robotoc/riccati/unconstr_riccati_recursion.hpp, src/riccati/unconstr_riccati_recursion.cpp:9-48
 *   (N stages + terminal, constant dt = T/N, control = acceleration)
 * --------------------------------------------------------------------------------------------- */
typedef struct rbt_uhandle rbt_uhandle;
int rbt_unconstr_create(int nv, int N, double dt, int batch, int device, rbt_uhandle** out);
int rbt_unconstr_destroy(rbt_uhandle* h);
double* rbt_unconstr_dev_ptr(rbt_uhandle* h, int which);
long long rbt_unconstr_buf_doubles(rbt_uhandle* h, int which);
int rbt_unconstr_upload(rbt_uhandle* h, int which, const double* host, void* stream);
int rbt_unconstr_download(rbt_uhandle* h, int which, double* host, void* stream);
int rbt_unconstr_download_info(rbt_uhandle* h, int* host_flags, void* stream);
/* UnconstrRiccatiRecursion::backwardRiccatiRecursion  unconstr_riccati_recursion.cpp:26-35 */
int rbt_unconstr_backward(rbt_uhandle* h, int write_fact, void* stream);
/* UnconstrRiccatiRecursion::forwardRiccatiRecursion   unconstr_riccati_recursion.cpp:37-46 */
int rbt_unconstr_forward(rbt_uhandle* h, void* stream);
int rbt_unconstr_solve_host(rbt_uhandle* h, const double* kkt_host, const double* dx0_host, double* ric_host,
                            double* dir_host, void* stream);
/* Stage layer of the unconstrained path -- the condensing tail of UnconstrIntermediateStage::evalKKT and the expansion /
 * step-size / update half of robotoc::UnconstrDirectMultipleShooting
 * (include/robotoc/unconstr/unconstr_direct_multiple_shooting.hpp; src/unconstr/unconstr_direct_multiple_shooting.cpp:88-179).
 * Records: include/rbt_ustage_layout.h.  `table` holds the joint position / velocity / acceleration / torque limits
 * (n_contacts must be 0). */
int rbt_unconstr_stage_layout_get(int nv, int n_box, const char* field);
int rbt_unconstr_stage_setup(rbt_uhandle* h, const rbt_constraint_table* table);
/* Constraints::condenseSlackAndDual + UnconstrDynamics::condenseUnconstrDynamics (src/dynamics/unconstr_dynamics.cpp:67-87)
 * on every stage; terminal stage: Qxx, lx.  Reads RBT_BUF_LIN, RBT_BUF_CON; writes RBT_BUF_KKT, RBT_BUF_EXP, RBT_BUF_CON.
 * As ConstraintsData::setTimeStage does for GridInfo::stage = i (constraints_data.cpp:20-45), a table row acts on stage i iff
 * i >= 2 for RBT_VAR_Q, i >= 1 for RBT_VAR_V, always for RBT_VAR_A / RBT_VAR_U; the PDIPM record of a row that does not act is
 * left untouched by this call, rbt_unconstr_expand_and_step_sizes (which also leaves it out of the step sizes) and
 * rbt_unconstr_update. */
int rbt_unconstr_condense(rbt_uhandle* h, void* stream);
/* UnconstrDirectMultipleShooting::computeStepSizes + maxPrimalStepSize / maxDualStepSize (:128-156): expandPrimal, expandDual
 * (unconstr_dynamics.cpp:90-104), slack/dual directions, fraction-to-boundary, min over the horizon -> RBT_BUF_STEPS. */
int rbt_unconstr_expand_and_step_sizes(rbt_uhandle* h, void* stream);
/* UnconstrDirectMultipleShooting::integrateSolution (:159-179) with the step sizes of RBT_BUF_STEPS. */
int rbt_unconstr_update(rbt_uhandle* h, void* stream);
/* The linear-algebra body of UnconstrOCPSolver::updateSolution (src/solver/unconstr_ocp_solver.cpp:101-118) with HOST buffers. */
int rbt_unconstr_iteration_host(rbt_uhandle* h, const double* lin_host, const double* con_host, const double* sol_host,
                                const double* dx0_host, double* sol_out, double* con_out, double* steps_out, void* stream);
int rbt_unconstr_sync(rbt_uhandle* h, void* stream);
const char* rbt_unconstr_last_error(rbt_uhandle* h);
long long rbt_unconstr_launch_count(rbt_uhandle* h);

#ifdef __cplusplus
}
#endif
#endif /* ROBOTOC_B200_H_ */
