/*
 * unconstr_stage_oracle.c -- CPU restatement of the stage layer of robotoc's UNCONSTRAINED path (iiwa14-type robots).
 *
 * TEST INFRASTRUCTURE ONLY: used by tests/, __graft_entry__.smoke() and bench.py's CPU legs as the checker.  The product
 * (librobotoc_b200.so) never links or calls it.
 *
 * Parity pinning: tests/golden/golden_ref_ustage.npz holds what the reference's own stage-layer code computes on these records
 * (oracle/ref_wrap/ref_ustage_wrap.cpp, built by oracle/Makefile.ref), and tests/test_golden_ref_ustage.py compares this file
 * with it block by block.  tests/test_oracle_unconstr_stage.py adds reference-independent identities: the condensed (q,v,a)
 * model equals the (q,v,a,u) model with u = ID + dID*[dq;dv;da] substituted (value, gradient, Hessian), the PDIPM rows equal
 * J^T W J / J^T cond, and the expansion reproduces the Newton step of the full stage KKT system.
 *
 * Which rows act on grid point i (GridInfo::stage = i, unconstr_ocp_solver.cpp:41-50): ConstraintsData::setTimeStage
 * (constraints_data.cpp:20-45) turns position-level components off on stages 0 and 1 and velocity-level components off on
 * stage 0, and every Constraints member skips a level that is not valid.  So a row of level l (2: q, 1: v, 0: a and u) acts
 * iff i >= l; a row that does not act adds nothing to the KKT and expansion records, takes no part in the step sizes, and
 * its PDIPM record (slack, dual, res, cmpl, cond, dslack, ddual) is left as it came in.
 *
 * Records: include/rbt_ustage_layout.h (stage layer), rbt_ulayout in include/rbt_layout.h (KKT / direction).
 */
#include <float.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "../include/rbt_ustage_layout.h"

#define IDX(i, j, ld) ((size_t)(i) + (size_t)(j) * (size_t)(ld))

/* ConstraintsData::setTimeStage: does box row b act on grid point `stage`? */
static int row_acts(const rbt_box_row* b, int stage) {
  return stage >= (b->var == RBT_VAR_Q ? 2 : b->var == RBT_VAR_V ? 1 : 0);
}

/* C(m x n) (+)= A^T(m x k) * diag(w) * B(k x n) ; all column-major with leading dimension ld = k or given */
static void atdb(int m, int n, int k, const double* A, const double* w, const double* B, double beta, double* C, int ldc) {
  for (int j = 0; j < n; ++j)
    for (int i = 0; i < m; ++i) {
      double acc = 0.0;
      for (int l = 0; l < k; ++l) acc += A[IDX(l, i, k)] * (w ? w[l] : 1.0) * B[IDX(l, j, k)];
      C[IDX(i, j, ldc)] = beta * C[IDX(i, j, ldc)] + acc;
    }
}

/*
 * UnconstrIntermediateStage::evalKKT "Forms linear system" tail         src/unconstr/unconstr_intermediate_stage.cpp:96-98
 *   pdipm::computeComplementarySlackness / condenseSlackAndDual          pdipm.hxx:27-100, joint_*_limit.cpp:68-83
 *   UnconstrDynamics::condenseUnconstrDynamics                           src/dynamics/unconstr_dynamics.cpp:67-87
 * UnconstrTerminalStage::evalKKT has no constraints and no dynamics      src/unconstr/unconstr_terminal_stage.cpp:69-94
 * terminal != 0: kkt gets Qxx, lx only.  stage: GridInfo::stage of the grid point (row_acts).
 */
void orc_ustage_condense_at(int nv, const rbt_constraint_table* tab, int stage, int terminal, const double* lin, double* con,
                            double* kkt, double* ex) {
  rbt_ustage_layout S;
  rbt_ulayout K;
  rbt_make_ustage_layout(nv, tab->n_box, &S);
  rbt_make_ulayout(nv, &K);
  const int nx = 2 * nv;
  memset(kkt, 0, sizeof(double) * K.k_stride);
  memset(ex, 0, sizeof(double) * S.e_stride);
  double* Qxx = kkt + K.k_Qxx;
  double* lx = kkt + K.k_lx;
  memcpy(Qxx, lin + S.l_Qxx, sizeof(double) * nx * nx);
  memcpy(lx, lin + S.l_lx, sizeof(double) * nx);
  if (terminal) return;
  double* Qxu = kkt + K.k_Qxu;
  double* Qaa = kkt + K.k_Qaa;
  double* la = kkt + K.k_la;
  double* lu = ex + S.e_lu;
  double* Quu = ex + S.e_Quu;
  memcpy(Qaa, lin + S.l_Qaa, sizeof(double) * nv * nv);
  memcpy(la, lin + S.l_la, sizeof(double) * nv);
  memcpy(lu, lin + S.l_lu, sizeof(double) * nv);
  memcpy(Quu, lin + S.l_Quu, sizeof(double) * nv * nv);
  memcpy(kkt + K.k_Fx, lin + S.l_Fx, sizeof(double) * nx);
  /* PDIPM */
  double* slack = con + S.c_slack;
  double* dual = con + S.c_dual;
  double* res = con + S.c_res;
  double* cmpl = con + S.c_cmpl;
  double* cond = con + S.c_cond;
  for (int r = 0; r < tab->n_box; ++r) {
    const rbt_box_row* b = &tab->box[r];
    if (!row_acts(b, stage)) continue;
    cmpl[r] = slack[r] * dual[r] - tab->barrier;                        /* pdipm.hxx:27-31 */
    cond[r] = (dual[r] * res[r] - cmpl[r]) / slack[r];                  /* pdipm.hxx:66-70 */
    const double w = dual[r] / slack[r];
    switch (b->var) {                                                   /* joint_*_limit.cpp:68-75 */
      case RBT_VAR_Q: Qxx[IDX(b->idx, b->idx, nx)] += w; lx[b->idx] += b->sign * cond[r]; break;
      case RBT_VAR_V: Qxx[IDX(nv + b->idx, nv + b->idx, nx)] += w; lx[nv + b->idx] += b->sign * cond[r]; break;
      case RBT_VAR_A: Qaa[IDX(b->idx, b->idx, nv)] += w; la[b->idx] += b->sign * cond[r]; break;
      default: Quu[IDX(b->idx, b->idx, nv)] += w; lu[b->idx] += b->sign * cond[r]; break;
    }
  }
  /* condenseUnconstrDynamics  unconstr_dynamics.cpp:67-87 */
  const double* Dq = lin + S.l_dIDdq;
  const double* Dv = lin + S.l_dIDdv;
  const double* Da = lin + S.l_dIDda;
  const double* ID = lin + S.l_ID;
  double* w = (double*)malloc(sizeof(double) * 2 * nv);
  double* luc = w + nv;
  for (int i = 0; i < nv; ++i) {
    w[i] = Quu[IDX(i, i, nv)];                                          /* Quu.diagonal() */
    luc[i] = lu[i] + w[i] * ID[i];                                      /* :70-71 */
  }
  for (int j = 0; j < nv; ++j) {                                        /* :72-74 */
    double aq = 0.0, av = 0.0, aa = 0.0;
    for (int l = 0; l < nv; ++l) {
      aq += Dq[IDX(l, j, nv)] * luc[l];
      av += Dv[IDX(l, j, nv)] * luc[l];
      aa += Da[IDX(l, j, nv)] * luc[l];
    }
    lx[j] += aq;
    lx[nv + j] += av;
    la[j] += aa;
  }
  atdb(nv, nv, nv, Dq, w, Dq, 1.0, Qxx, nx);                            /* Qqq += dIDdq^T Quu dIDdq  :79 */
  atdb(nv, nv, nv, Dq, w, Dv, 1.0, Qxx + IDX(0, nv, nx), nx);           /* Qqv += ..                 :80 */
  for (int j = 0; j < nv; ++j)                                          /* Qvq = Qqv^T               :81 */
    for (int i = 0; i < nv; ++i) Qxx[IDX(nv + i, j, nx)] = Qxx[IDX(j, nv + i, nx)];
  atdb(nv, nv, nv, Dv, w, Dv, 1.0, Qxx + IDX(nv, nv, nx), nx);          /* Qvv += ..                 :82 */
  atdb(nv, nv, nv, Da, w, Da, 1.0, Qaa, nv);                            /* Qaa += ..                 :83 */
  atdb(nv, nv, nv, Dq, w, Da, 0.0, Qxu, nx);                            /* Qqu() = (Quu dIDdq)^T dIDda :85 */
  atdb(nv, nv, nv, Dv, w, Da, 0.0, Qxu + nv, nx);                       /* Qvu() = (Quu dIDdv)^T dIDda :86 */
  free(w);
}

/* pdipm::fractionToBoundary  pdipm.hxx:121-142, over the rows that act on grid point `stage` */
static double fraction_to_boundary(const rbt_constraint_table* tab, int stage, const double* v, const double* dv) {
  double m = 1.0;
  for (int i = 0; i < tab->n_box; ++i) {
    if (!row_acts(&tab->box[i], stage)) continue;
    const double f = -tab->fraction_to_boundary * (v[i] / dv[i]);
    if (f > 0 && f < 1 && f < m) m = f;
  }
  return m;
}

/*
 * UnconstrIntermediateStage::expandPrimalAndDual + max{Primal,Dual}StepSize   unconstr_intermediate_stage.cpp:103-122
 *   UnconstrDynamics::expandPrimal / expandDual                               unconstr_dynamics.cpp:90-104
 *   Constraints::expandSlackAndDual                                           joint_*_limit.cpp:78-83, pdipm.hxx:159-164
 * d: direction record (rbt_ulayout d_dx, d_da).  steps = {primal, dual}.  (The terminal stage returns 1.0, 1.0 and
 * touches nothing: unconstr_terminal_stage.cpp:97-112 -- the caller skips it.)
 */
void orc_ustage_expand_at(int nv, const rbt_constraint_table* tab, int stage, double dt, const double* lin, const double* ex,
                          const double* d, double* con, double* xd, double* steps) {
  rbt_ustage_layout S;
  rbt_ulayout K;
  rbt_make_ustage_layout(nv, tab->n_box, &S);
  rbt_make_ulayout(nv, &K);
  const double* dq = d + K.d_dx;
  const double* dv = dq + nv;
  const double* da = d + K.d_da;
  double* du = xd + S.x_du;
  double* dbeta = xd + S.x_dbeta;
  for (int i = 0; i < nv; ++i) {
    double acc = lin[S.l_ID + i];                                                         /* du = ID_  :91 */
    for (int j = 0; j < nv; ++j)
      acc += lin[S.l_dIDdq + IDX(i, j, nv)] * dq[j] + lin[S.l_dIDdv + IDX(i, j, nv)] * dv[j] +
             lin[S.l_dIDda + IDX(i, j, nv)] * da[j];                                       /* :92-94 */
    du[i] = acc;
  }
  for (int i = 0; i < nv; ++i) {
    double acc = ex[S.e_lu + i];
    for (int j = 0; j < nv; ++j) acc += ex[S.e_Quu + IDX(i, j, nv)] * du[j];
    dbeta[i] = acc / dt;                                                                   /* :103 */
  }
  double* slack = con + S.c_slack;
  double* dual = con + S.c_dual;
  for (int r = 0; r < tab->n_box; ++r) {
    const rbt_box_row* b = &tab->box[r];
    if (!row_acts(b, stage)) continue;
    const double* var = b->var == RBT_VAR_Q ? dq : b->var == RBT_VAR_V ? dv : b->var == RBT_VAR_A ? da : du;
    con[S.c_dslack + r] = -b->sign * var[b->idx] - con[S.c_res + r];
    con[S.c_ddual + r] = -(dual[r] * con[S.c_dslack + r] + con[S.c_cmpl + r]) / slack[r];
  }
  steps[0] = fraction_to_boundary(tab, stage, slack, con + S.c_dslack);
  steps[1] = fraction_to_boundary(tab, stage, dual, con + S.c_ddual);
}

/* updatePrimal + updateDual  unconstr_intermediate_stage.cpp:125-144, unconstr_terminal_stage.cpp:115-132,
 * SplitSolution::integrate split_solution.cpp:58-90 (fixed base: q += step*dq). */
void orc_ustage_update_at(int nv, const rbt_constraint_table* tab, int stage, int terminal, const double* d, const double* xd,
                          double* con, double* sol, double primal_step, double dual_step) {
  rbt_ustage_layout S;
  rbt_ulayout K;
  rbt_make_ustage_layout(nv, tab->n_box, &S);
  rbt_make_ulayout(nv, &K);
  for (int i = 0; i < nv; ++i) {
    sol[S.s_q + i] += primal_step * d[K.d_dx + i];
    sol[S.s_v + i] += primal_step * d[K.d_dx + nv + i];
    sol[S.s_lmd + i] += primal_step * d[K.d_dlmdgmm + i];
    sol[S.s_gmm + i] += primal_step * d[K.d_dlmdgmm + nv + i];
  }
  if (terminal) return;
  for (int i = 0; i < nv; ++i) {
    sol[S.s_a + i] += primal_step * d[K.d_da + i];
    sol[S.s_u + i] += primal_step * xd[S.x_du + i];
    sol[S.s_beta + i] += primal_step * xd[S.x_dbeta + i];
  }
  for (int r = 0; r < tab->n_box; ++r) {
    if (!row_acts(&tab->box[r], stage)) continue;
    con[S.c_slack + r] += primal_step * con[S.c_dslack + r];
    con[S.c_dual + r] += dual_step * con[S.c_ddual + r];
  }
}

/* The same three steps on a grid point from stage 2 on, where every row of the table acts. */
void orc_ustage_condense(int nv, const rbt_constraint_table* tab, int terminal, const double* lin, double* con, double* kkt,
                         double* ex) {
  orc_ustage_condense_at(nv, tab, 2, terminal, lin, con, kkt, ex);
}
void orc_ustage_expand(int nv, const rbt_constraint_table* tab, double dt, const double* lin, const double* ex, const double* d,
                       double* con, double* xd, double* steps) {
  orc_ustage_expand_at(nv, tab, 2, dt, lin, ex, d, con, xd, steps);
}
void orc_ustage_update(int nv, const rbt_constraint_table* tab, int terminal, const double* d, const double* xd, double* con,
                       double* sol, double primal_step, double dual_step) {
  orc_ustage_update_at(nv, tab, 2, terminal, d, xd, con, sol, primal_step, dual_step);
}

/* ---------------- batched horizon drivers (UnconstrDirectMultipleShooting::{evalKKT tail, computeStepSizes,
 * maxPrimal/DualStepSize, integrateSolution}  src/unconstr/unconstr_direct_multiple_shooting.cpp:88-179) */
void orc_ucondense_batch(int nv, const rbt_constraint_table* tab, int N, int batch, const double* lin, double* con,
                         double* kkt, double* ex) {
  rbt_ustage_layout S;
  rbt_ulayout K;
  rbt_make_ustage_layout(nv, tab->n_box, &S);
  rbt_make_ulayout(nv, &K);
#pragma omp parallel for schedule(static)
  for (int b = 0; b < batch; ++b)
    for (int i = 0; i <= N; ++i) {
      const size_t o = (size_t)b * (N + 1) + i;
      orc_ustage_condense_at(nv, tab, i, i == N, lin + o * S.l_stride, con + o * S.c_stride, kkt + o * K.k_stride, ex + o * S.e_stride);
    }
}

void orc_uexpand_batch(int nv, const rbt_constraint_table* tab, int N, double dt, int batch, const double* lin,
                       const double* ex, const double* dir, double* con, double* xd, double* steps) {
  rbt_ustage_layout S;
  rbt_ulayout K;
  rbt_make_ustage_layout(nv, tab->n_box, &S);
  rbt_make_ulayout(nv, &K);
#pragma omp parallel for schedule(static)
  for (int b = 0; b < batch; ++b) {
    double mp = 1.0, md = 1.0;
    for (int i = 0; i < N; ++i) {
      const size_t o = (size_t)b * (N + 1) + i;
      double st[2];
      orc_ustage_expand_at(nv, tab, i, dt, lin + o * S.l_stride, ex + o * S.e_stride, dir + o * K.d_stride, con + o * S.c_stride,
                        xd + o * S.x_stride, st);
      if (st[0] < mp) mp = st[0];
      if (st[1] < md) md = st[1];
    }
    steps[2 * b] = mp;
    steps[2 * b + 1] = md;
  }
}

void orc_uupdate_batch(int nv, const rbt_constraint_table* tab, int N, int batch, const double* dir, const double* xd,
                       double* con, double* sol, const double* steps) {
  rbt_ustage_layout S;
  rbt_ulayout K;
  rbt_make_ustage_layout(nv, tab->n_box, &S);
  rbt_make_ulayout(nv, &K);
#pragma omp parallel for schedule(static)
  for (int b = 0; b < batch; ++b)
    for (int i = 0; i <= N; ++i) {
      const size_t o = (size_t)b * (N + 1) + i;
      orc_ustage_update_at(nv, tab, i, i == N, dir + o * K.d_stride, xd + o * S.x_stride, con + o * S.c_stride,
                        sol + o * S.s_stride, steps[2 * b], steps[2 * b + 1]);
    }
}

int orc_ustage_layout_get(int nv, int n_box, const char* field) {
  rbt_ustage_layout S;
  rbt_make_ustage_layout(nv, n_box, &S);
  return rbt_ustage_layout_field(&S, field);
}
