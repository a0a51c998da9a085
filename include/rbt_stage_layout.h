/*
 * rbt_stage_layout.h -- packed fp64 records of the per-stage "condense / expand / update" layer (SURVEY.md 8a rows a10-a16).
 *
 * These records carry what the reference keeps in
 *   ContactDynamicsData        include/robotoc/dynamics/contact_dynamics_data.hpp   (M=dIDda, J=dCda, dIDCdqv, IDC, MJtJinv, ...)
 *   StateEquationData          include/robotoc/dynamics/state_equation_data.hpp      (Fqq_prev, Fqq_inv, Fqq_prev_inv 6x6 blocks)
 *   ConstraintComponentData    include/robotoc/constraints/constraint_component_data.hpp (slack,dual,residual,cmpl,cond,dslack,ddual)
 *   SplitSolution              include/robotoc/core/split_solution.hpp
 *   SplitDirection (daf, dbetamu, dnu_passive)   src/core/split_direction.cpp:7-22
 * The linearization record is the INPUT boundary of the hot path: it is what the (out-of-scope, Pinocchio-based)
 * linearize* halves produce before condensing starts (intermediate_stage.cpp:94-132).
 *
 * All blocks are column-major with FIXED leading dimensions (nvf = nv + nf_max rows for the stacked [a;f] blocks,
 * nf_max for J/Qff, 5 for the friction-cone Jacobians), except the switching-constraint blocks which use ld = ns of
 * the stage like the KKT record.  Offsets are multiples of 2 doubles, strides multiples of 16.
 */
#ifndef RBT_STAGE_LAYOUT_H_
#define RBT_STAGE_LAYOUT_H_

#include "rbt_layout.h"

#ifdef __cplusplus
extern "C" {
#endif

#define RBT_MAX_BOX_ROWS 128
#define RBT_MAX_CONTACTS 8

/* variable a box limit acts on */
enum { RBT_VAR_Q = 0, RBT_VAR_V = 1, RBT_VAR_A = 2, RBT_VAR_U = 3 };

/* One inequality row  sign*(x[idx] - bound) + slack = 0  (sign = -1: lower limit, +1: upper limit), i.e. J = sign*e_idx.
 * Mirrors JointPosition/Velocity/Acceleration/TorquesLower/UpperLimit (src/constraints/joint_*_limit.cpp:68-90). */
typedef struct rbt_box_row {
  int var;
  int idx;  /* index inside dq / dv / da / du */
  int sign;
} rbt_box_row;

/* Constraint table shared by the batch (examples/anymal/trot.cpp:135-148: 6 box limits x 12 joints + friction cones). */
typedef struct rbt_constraint_table {
  int n_box;
  int n_contacts;           /* max point contacts; each active one contributes 5 friction-cone rows (friction_cone.cpp) */
  int impact_friction_cone; /* != 0: impact stages carry the same 5 rows per active impact (ImpactFrictionCone,
                               src/constraints/impact_friction_cone.cpp; examples/anymal/run.cpp:173-181); box limits never act
                               on impact stages (Constraints::condenseSlackAndDual(impact_status, ...), constraints.cpp:347-354) */
  int pad_;
  double barrier;           /* mu  (constraint_component_base.hpp:44) */
  double fraction_to_boundary;  /* tau (constraint_component_base.hpp:45) */
  rbt_box_row box[RBT_MAX_BOX_ROWS];
} rbt_constraint_table;

typedef struct rbt_stage_dims {
  int nv, nu, n_passive, nf_max, ns_max, n_contacts, n_box;
} rbt_stage_dims;

typedef struct rbt_stage_layout {
  int nv, nu, nx, np, nfm, nvf, nsm, ncon, nbox, nc, ncp, nq;
  /* ---- linearization record (input) */
  int l_M, l_J, l_D, l_IDC, l_Qaa, l_Qff, l_Qqf, l_Qxx, l_Quu, l_lx, l_la, l_lf, l_lu, l_Fx, l_lup, l_se3;
  int l_Phix, l_Phia, l_p, l_Phit, l_ha, l_hf, l_hx, l_hu, l_fx, l_sc, l_dgdq, l_dgdf, l_stride;
  /* ---- expansion record (written by condense, read by expand / update) */
  int e_Z, e_R, e_r, e_Qafqv, e_Qafu, e_laf, e_Qxup, e_Quup, e_lup, e_Phia, e_haf, e_Fqqpi, e_Qaf, e_Quf, e_Qaa, e_stride;
  /* ---- PDIPM record */
  int c_slack, c_dual, c_res, c_cmpl, c_cond, c_dslack, c_ddual, c_stride;
  /* ---- solution record */
  int s_q, s_v, s_a, s_dv, s_u, s_f, s_lmd, s_gmm, s_beta, s_mu, s_nup, s_xi, s_stride;
  /* ---- expanded direction record (beyond the Riccati direction record) */
  int x_daf, x_dbetamu, x_dnup, x_stride;
} rbt_stage_layout;

static inline RBT_HD void rbt_make_stage_layout(const rbt_stage_dims* d, rbt_stage_layout* L) {
  const int nv = d->nv, nu = d->nu, nx = 2 * nv, np = d->n_passive, nfm = d->nf_max, nvf = nv + nfm, nsm = d->ns_max;
  const int ncon = d->n_contacts, nbox = d->n_box, nc = nbox + 5 * ncon, ncp = rbt_up2(nc);
  int o = 0;
  L->nv = nv; L->nu = nu; L->nx = nx; L->np = np; L->nfm = nfm; L->nvf = nvf; L->nsm = nsm; L->ncon = ncon;
  L->nbox = nbox; L->nc = nc; L->ncp = ncp; L->nq = nv + (np == 6 ? 1 : 0);
  L->l_M = o; o += rbt_up2(nv * nv);
  L->l_J = o; o += rbt_up2(nfm * nv);
  L->l_D = o; o += rbt_up2(nvf * nx);
  L->l_IDC = o; o += rbt_up2(nvf);
  L->l_Qaa = o; o += rbt_up2(nv);
  L->l_Qff = o; o += rbt_up2(nfm * nfm);
  L->l_Qqf = o; o += rbt_up2(nv * nfm);
  L->l_Qxx = o; o += rbt_up2(nx * nx);
  L->l_Quu = o; o += rbt_up2(nu * nu);
  L->l_lx = o; o += rbt_up2(nx);
  L->l_la = o; o += rbt_up2(nv);
  L->l_lf = o; o += rbt_up2(nfm);
  L->l_lu = o; o += rbt_up2(nu);
  L->l_Fx = o; o += rbt_up2(nx);
  L->l_lup = o; o += rbt_up2(np);
  L->l_se3 = o; o += 3 * 36; /* Fqq top-left (dSub/dqf), Fqq_prev (dSub/dq0 at i-1), Fqq_cur (dSub/dq0 at i): 6x6 each */
  L->l_Phix = o; o += rbt_up2(nsm * nx);
  L->l_Phia = o; o += rbt_up2(nsm * nv);
  L->l_p = o; o += rbt_up2(nsm);
  L->l_Phit = o; o += rbt_up2(nsm);
  L->l_ha = o; o += rbt_up2(nv);
  L->l_hf = o; o += rbt_up2(nfm);
  L->l_hx = o; o += rbt_up2(nx);
  L->l_hu = o; o += rbt_up2(nu);
  L->l_fx = o; o += rbt_up2(nx);
  L->l_sc = o; o += 4; /* {h, Qtt, 0, 0} */
  L->l_dgdq = o; o += rbt_up2(ncon * 5 * nv);
  L->l_dgdf = o; o += rbt_up2(ncon * 15);
  L->l_stride = rbt_up16(o);

  o = 0;
  L->e_Z = o; o += rbt_up2(nvf * nvf);
  L->e_R = o; o += rbt_up2(nvf * nx);
  L->e_r = o; o += rbt_up2(nvf);
  L->e_Qafqv = o; o += rbt_up2(nvf * nx);
  L->e_Qafu = o; o += rbt_up2(nvf * nv);
  L->e_laf = o; o += rbt_up2(nvf);
  L->e_Qxup = o; o += rbt_up2(nx * np);
  L->e_Quup = o; o += rbt_up2(np * nu);
  L->e_lup = o; o += rbt_up2(np);
  L->e_Phia = o; o += rbt_up2(nsm * nv);
  L->e_haf = o; o += rbt_up2(nvf);
  L->e_Fqqpi = o; o += 36;
  /* What the CUDA path keeps of Qafqv / Qafu_full (contact_dynamics.cpp:68-86): their contact rows, Qaf (nfm x nx, ld nfm) |
   * Quf (nfm x nv, ld nfm), and diag(Qaa) after the PDIPM terms -- the acceleration rows are -diag(Qaa) R_a and diag(Qaa) Z_aa
   * and are never materialised (the dual expansion uses Qaa o (da + r_a) for them).  e_Qafqv / e_Qafu (the full matrices) are
   * written by the CPU oracle and the reference wrapper only. */
  L->e_Qaf = o; o += rbt_up2(nfm * nx);
  L->e_Quf = o; o += rbt_up2(nfm * nv);
  L->e_Qaa = o; o += rbt_up2(nv);
  L->e_stride = rbt_up16(o);

  o = 0;
  L->c_slack = o; o += ncp;
  L->c_dual = o; o += ncp;
  L->c_res = o; o += ncp;
  L->c_cmpl = o; o += ncp;
  L->c_cond = o; o += ncp;
  L->c_dslack = o; o += ncp;
  L->c_ddual = o; o += ncp;
  L->c_stride = rbt_up16(o);

  o = 0;
  L->s_q = o; o += rbt_up2(L->nq);
  L->s_v = o; o += rbt_up2(nv);
  L->s_a = o; o += rbt_up2(nv);
  L->s_dv = o; o += rbt_up2(nv);
  L->s_u = o; o += rbt_up2(nu);
  L->s_f = o; o += rbt_up2(nfm);
  L->s_lmd = o; o += rbt_up2(nv);
  L->s_gmm = o; o += rbt_up2(nv);
  L->s_beta = o; o += rbt_up2(nv);
  L->s_mu = o; o += rbt_up2(nfm);
  L->s_nup = o; o += rbt_up2(np);
  L->s_xi = o; o += rbt_up2(nsm);
  L->s_stride = rbt_up16(o);

  o = 0;
  L->x_daf = o; o += rbt_up2(nvf);
  L->x_dbetamu = o; o += rbt_up2(nvf);
  L->x_dnup = o; o += rbt_up2(np);
  L->x_stride = rbt_up16(o);
}


/* ---------------- host wire format of the linearization records (the PCIe-facing form used by rbt_iteration_host_wire /
 * rbt_iteration_host_resident).  Only what a robotoc linearisation of THAT grid point holds travels, so the wire record of a
 * grid point depends on the stage control word (type, nf, contact mask) -- like the reference's own containers, whose contact
 * blocks are dimf-sized (SplitKKTMatrix::setContactDimension):
 *  - the symmetric blocks M, Qff (nf x nf), Qxx, Quu as packed upper triangles (column-major packed, element (i,j), i <= j, at
 *    j(j+1)/2 + i -- BLAS "UPLO=U" packed storage);
 *  - J = dCda as nf x nv, dIDCdqv as (nv+nf) x nx, IDC as nv+nf (column-major, leading dimension = the active row count);
 *  - the friction-cone Jacobians dg/dq (5 x nv), dg/df (5 x 3) of the ACTIVE contacts only, in contact order;
 *  - Qqf is NOT part of the wire record: no cost writes it, it is zero until the friction-cone condensing fills it
 *    (src/constraints/friction_cone.cpp:219 is the only writer; cost_function.cpp:194 only scales it) -- the device zero-fills it;
 *  - the STO section [ha | hf | hx | hu | fx | {h, Qtt}] only if the schedule has a switching-time stage (with_sto; the
 *    kernels read it on such stages only) -- otherwise the device zero-fills it;
 *  - cost_structure RBT_COST_ROBOTOC: the cost Hessians as every cost component robotoc ships produces them -- Qqq dense
 *    (packed), Qvv / Quu / Qff DIAGONAL, Qqv = 0 (src/cost/configuration_space_cost.cpp:308-322, task_space_*_cost.cpp, com_cost.cpp
 *    and local_contact_force_cost.cpp:130 are the only writers; nothing writes Qqv or an off-diagonal of Qvv / Quu / Qff before
 *    the condensing) -- RBT_COST_GENERAL sends Qxx, Quu, Qff as full packed triangles (user-defined cost components);
 *  - a Terminal grid point sends Qxx, lx and the Fqq_prev block only (terminal_stage.cpp:94-106);
 *  - neither padding nor the switching-constraint section (sent separately, only for stages that carry one).
 * One OCP's wire records are concatenated in grid order (rbt_wire_layout::ocp_off = offset of the grid point inside the OCP's
 * block; the OCP stride is the sum).  A host adaptor fills them straight from the reference's Eigen members; the device
 * expands them back into the rbt_stage_layout records (inactive rows / contacts of the device record are never read). */
typedef struct rbt_wire_seg { int lin_off, wire_off, rows, cols, ld, sym; } rbt_wire_seg;
  /* sym 0: rows x cols dense (ld rows on the wire) -> leading dimension ld ; 1: rows x rows packed upper triangle -> dense, ld ;
     2: the diagonal of a rows x rows block (rows doubles on the wire) -> element (k,k), ld */
typedef struct rbt_wire_zero { int lin_off, n; } rbt_wire_zero;   /* sections of the record the device zero-fills (first) */
enum { RBT_COST_GENERAL = 0, RBT_COST_ROBOTOC = 1 };
/* OR-ed into cost_structure: the device fills the inverse-dynamics rows (rbt_linearize_inverse_dynamics), so non-terminal wire
 * records carry neither M nor the first nv rows of dIDCdqv and IDC -- only their nf contact rows */
#define RBT_WIRE_DEVICE_ID 2
/* OR-ed into cost_structure: the device fills the contact rows (rbt_linearize_contact_kinematics), so non-terminal wire records
 * carry neither J nor the nf contact rows of dIDCdqv and IDC; alone or together with RBT_WIRE_DEVICE_ID */
#define RBT_WIRE_DEVICE_CONTACT 4
/* OR-ed into cost_structure: the device fills the state-equation rows (rbt_linearize_state_equation), so non-terminal wire
 * records carry neither Fx nor the three SE(3) blocks (the lx .. SE(3) segment splits around them) and terminal records no
 * Fqq_prev block; the STO section still travels with the cost's share of h, hv, ha (the device adds the costate terms and
 * overwrites fx).  Alone or together with the other two bits */
#define RBT_WIRE_DEVICE_STATE 16
#define RBT_WIRE_MAX_SEGS 20
#define RBT_WIRE_MAX_ZERO 5
typedef struct rbt_wire_layout {
  int nseg, nzero, w_doubles, ocp_off;
  rbt_wire_seg seg[RBT_WIRE_MAX_SEGS];
  rbt_wire_zero zero[RBT_WIRE_MAX_ZERO];
} rbt_wire_layout;

static inline RBT_HD void rbt_wire_add_(rbt_wire_layout* W, int lin_off, int rows, int cols, int ld, int sym) {
  rbt_wire_seg* g = &W->seg[W->nseg++];
  g->lin_off = lin_off; g->wire_off = W->w_doubles; g->rows = rows; g->cols = cols; g->ld = ld; g->sym = sym;
  W->w_doubles += rbt_up2(sym == 1 ? rows * (rows + 1) / 2 : (sym == 2 ? rows : rows * cols));
}
static inline RBT_HD void rbt_wire_zero_(rbt_wire_layout* W, int lin_off, int n) {
  W->zero[W->nzero].lin_off = lin_off; W->zero[W->nzero].n = n; W->nzero++;
}
/* Qxx of a grid point: full packed triangle, or Qqq packed + diag(Qvv) with the rest zero-filled */
static inline RBT_HD void rbt_wire_add_qxx_(const rbt_stage_layout* L, int cost_structure, rbt_wire_layout* W) {
  const int nv = L->nv, nx = L->nx;
  if (cost_structure == RBT_COST_ROBOTOC) {
    rbt_wire_zero_(W, L->l_Qxx, nx * nx);
    rbt_wire_add_(W, L->l_Qxx, nv, nv, nx, 1);
    rbt_wire_add_(W, L->l_Qxx + nv * nx + nv, nv, nv, nx, 2);
  } else {
    rbt_wire_add_(W, L->l_Qxx, nx, nx, nx, 1);
  }
}

static inline RBT_HD void rbt_make_wire_layout(const rbt_stage_layout* L, const rbt_stage_ctrl* c, int with_sto, int cost_structure,
                                               rbt_wire_layout* W) {
  const int nv = L->nv, nx = L->nx, nf = c->nf, nvf = nv + nf;
  const int dc = ((cost_structure & RBT_COST_ROBOTOC) != 0), did = ((cost_structure & RBT_WIRE_DEVICE_ID) != 0);
  const int dcon = ((cost_structure & RBT_WIRE_DEVICE_CONTACT) != 0);
  const int dst = ((cost_structure & RBT_WIRE_DEVICE_STATE) != 0);
  int ci;
  cost_structure &= RBT_COST_ROBOTOC;
  W->nseg = 0; W->nzero = 0; W->w_doubles = 0; W->ocp_off = 0;
  if (c->type == RBT_TERMINAL) {
    rbt_wire_add_qxx_(L, cost_structure, W);
    rbt_wire_add_(W, L->l_lx, nx, 1, nx, 0);
    if (!dst) rbt_wire_add_(W, L->l_se3 + 36, 36, 1, 36, 0);
    return;
  }
  if (!did && dcon) {  /* ID rows only: M, [dIDdq | dIDdv], ID */
    rbt_wire_add_(W, L->l_M, nv, nv, nv, 1);
    rbt_wire_add_(W, L->l_D, nv, nx, L->nvf, 0);
    rbt_wire_add_(W, L->l_IDC, nv, 1, nv, 0);
  } else if (!did) {
    rbt_wire_add_(W, L->l_M, nv, nv, nv, 1);
    if (nf > 0) rbt_wire_add_(W, L->l_J, nf, nv, L->nfm, 0);
    rbt_wire_add_(W, L->l_D, nvf, nx, L->nvf, 0);
    rbt_wire_add_(W, L->l_IDC, nvf, 1, nvf, 0);
  } else if (nf > 0 && !dcon) {  /* contact rows only: dCda, [dCdq | dCdv], C */
    rbt_wire_add_(W, L->l_J, nf, nv, L->nfm, 0);
    rbt_wire_add_(W, L->l_D + nv, nf, nx, L->nvf, 0);
    rbt_wire_add_(W, L->l_IDC + nv, nf, 1, nf, 0);
  }
  rbt_wire_add_(W, L->l_Qaa, nv, 1, nv, 0);
  if (dc) rbt_wire_zero_(W, L->l_Qff, L->nfm * L->nfm);
  if (nf > 0) rbt_wire_add_(W, L->l_Qff, nf, nf, L->nfm, dc ? 2 : 1);
  rbt_wire_add_qxx_(L, cost_structure, W);
  if (dc) rbt_wire_zero_(W, L->l_Quu, L->nu * L->nu);
  rbt_wire_add_(W, L->l_Quu, L->nu, L->nu, L->nu, dc ? 2 : 1);
  if (dst) {  /* lx | la | lf | lu, then lup */
    rbt_wire_add_(W, L->l_lx, L->l_Fx - L->l_lx, 1, L->l_Fx - L->l_lx, 0);
    rbt_wire_add_(W, L->l_lup, L->l_se3 - L->l_lup, 1, L->l_se3 - L->l_lup, 0);
  } else {
    rbt_wire_add_(W, L->l_lx, L->l_Phix - L->l_lx, 1, L->l_Phix - L->l_lx, 0);   /* lx | la | lf | lu | Fx | lup | SE(3) blocks */
  }
  for (ci = 0; ci < L->ncon; ++ci)
    if ((c->contact_mask >> ci) & 1) {
      rbt_wire_add_(W, L->l_dgdq + ci * 5 * nv, 5 * nv, 1, 5 * nv, 0);
      rbt_wire_add_(W, L->l_dgdf + ci * 15, 15, 1, 15, 0);
    }
  if (with_sto) rbt_wire_add_(W, L->l_ha, L->l_dgdq - L->l_ha, 1, L->l_dgdq - L->l_ha, 0);
  rbt_wire_zero_(W, L->l_Qqf, L->l_Qxx - L->l_Qqf);
  if (!with_sto) rbt_wire_zero_(W, L->l_ha, L->l_dgdq - L->l_ha);
}

/* one record: rbt_stage_layout linearization record -> wire record (reads the upper triangles) */
static inline void rbt_pack_wire_record(const rbt_wire_layout* W, const double* lin, double* wire) {
  int k, i, j;
  for (k = 0; k < W->nseg; ++k) {
    const rbt_wire_seg* g = &W->seg[k];
    double* dst = wire + g->wire_off;
    const double* src = lin + g->lin_off;
    if (!g->sym) {
      for (j = 0; j < g->cols; ++j)
        for (i = 0; i < g->rows; ++i) dst[i + j * g->rows] = src[i + j * g->ld];
      continue;
    }
    if (g->sym == 2) { for (i = 0; i < g->rows; ++i) dst[i] = src[i * (g->ld + 1)]; continue; }
    for (j = 0; j < g->rows; ++j)
      for (i = 0; i <= j; ++i) dst[j * (j + 1) / 2 + i] = src[i + j * g->ld];
  }
}
/* wire record -> linearization record (what the device kernel does; used by the CPU tests) */
static inline void rbt_unpack_wire_record(const rbt_wire_layout* W, const double* wire, double* lin) {
  int k, i, j;
  for (k = 0; k < W->nzero; ++k)
    for (i = 0; i < W->zero[k].n; ++i) lin[W->zero[k].lin_off + i] = 0.0;
  for (k = 0; k < W->nseg; ++k) {
    const rbt_wire_seg* g = &W->seg[k];
    const double* src = wire + g->wire_off;
    double* dst = lin + g->lin_off;
    if (!g->sym) {
      for (j = 0; j < g->cols; ++j)
        for (i = 0; i < g->rows; ++i) dst[i + j * g->ld] = src[i + j * g->rows];
      continue;
    }
    if (g->sym == 2) { for (i = 0; i < g->rows; ++i) dst[i * (g->ld + 1)] = src[i]; continue; }
    for (j = 0; j < g->rows; ++j)
      for (i = 0; i < g->rows; ++i) dst[i + j * g->ld] = (i <= j) ? src[j * (j + 1) / 2 + i] : src[i * (i + 1) / 2 + j];
  }
}

#define RBT_STAGE_LAYOUT_FIELDS(X) \
  X(nv) X(nu) X(nx) X(np) X(nfm) X(nvf) X(nsm) X(ncon) X(nbox) X(nc) X(ncp) X(nq) \
  X(l_M) X(l_J) X(l_D) X(l_IDC) X(l_Qaa) X(l_Qff) X(l_Qqf) X(l_Qxx) X(l_Quu) X(l_lx) X(l_la) X(l_lf) X(l_lu) X(l_Fx) \
  X(l_lup) X(l_se3) X(l_Phix) X(l_Phia) X(l_p) X(l_Phit) X(l_ha) X(l_hf) X(l_hx) X(l_hu) X(l_fx) X(l_sc) X(l_dgdq) \
  X(l_dgdf) X(l_stride) \
  X(e_Z) X(e_R) X(e_r) X(e_Qafqv) X(e_Qafu) X(e_laf) X(e_Qxup) X(e_Quup) X(e_lup) X(e_Phia) X(e_haf) X(e_Fqqpi) X(e_Qaf) X(e_Quf) X(e_Qaa) X(e_stride) \
  X(c_slack) X(c_dual) X(c_res) X(c_cmpl) X(c_cond) X(c_dslack) X(c_ddual) X(c_stride) \
  X(s_q) X(s_v) X(s_a) X(s_dv) X(s_u) X(s_f) X(s_lmd) X(s_gmm) X(s_beta) X(s_mu) X(s_nup) X(s_xi) X(s_stride) \
  X(x_daf) X(x_dbetamu) X(x_dnup) X(x_stride)

static inline int rbt_stage_layout_field(const rbt_stage_layout* L, const char* name) {
#define X(f) if (rbt_streq_(name, #f)) return L->f;
  RBT_STAGE_LAYOUT_FIELDS(X)
#undef X
  return -1;
}

#ifdef __cplusplus
}
#endif
#endif /* RBT_STAGE_LAYOUT_H_ */
