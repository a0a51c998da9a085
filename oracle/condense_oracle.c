/*
 * condense_oracle.c -- TEST INFRASTRUCTURE ONLY (parity oracle / CPU baseline) for SURVEY.md 8a rows a10-a16:
 * PDIPM slack/dual condensing, contact / impact dynamics condensing, floating-base state-equation correction,
 * primal / dual expansion, fraction-to-boundary step sizes and the primal/dual update.
 *
 * Plain-C restatement of the reference (robotoc @ d30d404), every function citing the lines it follows.
 * PARITY STATUS: PINNED against the reference's own code.  robotoc/src/dynamics/{contact_dynamics,impact_dynamics,
 * state_equation,impact_state_equation,terminal_state_equation,...}.cpp, src/constraints/{constraints,friction_cone,joint_*_limit,
 * constraint_component_*}.cpp and src/core are compiled UNMODIFIED (oracle/Makefile.ref, Eigen / Robot stand-ins of oracle/shim)
 * and driven stage by stage in the order Intermediate/Impact/TerminalStage use them (oracle/ref_wrap/ref_stage_wrap.cpp);
 * tests/test_golden_ref_stage.py compares a FULL iteration of this file + riccati_oracle.c with a full iteration of that code
 * (condensed KKT records, every expansion block, cmpl / cond / dslack / ddual, step sizes, dual expansion, costate correction,
 * updated slack / dual) on event schedules with and without STO and on the BASELINE trot N=40 schedule: agreement < 1e-10
 * (measured 1e-14), and against the committed reference output tests/golden/golden_ref_stage_r2.npz.  Not covered by the
 * reference code here: Robot::computeMJtJinv (Pinocchio; dense restatement on both sides) and SplitSolution::integrate's SE(3)
 * exponential (Pinocchio; pinned against scipy's Rotation in tests/test_oracle_condense.py, and against a 100-digit expm in
 * tests/test_stage_mp.py).  The exponential here takes 1 - cos th as 2 sin^2(th/2), as the CUDA kernel does, where pinocchio's
 * exp6 writes (1 - cos th) / th^2: the same function, without the cancellation that costs the difference form up to 2u / th^2
 * of it just above the small-angle branch.  This is a choice of accuracy, not a departure from the reference's mathematics.
 * Additionally pinned by identities that do not reuse its formulas (tests/test_oracle_condense.py): MJtJinv == dense inverse;
 * condensed quadratic model == uncondensed model with (a, f) substituted; PDIPM condensing == J^T diag(z/s) J; the expansions
 * satisfy the linearised contact dynamics / make the uncondensed stage Lagrangian stationary; STO sensitivities == substituted
 * Hamiltonian derivatives; SE(3) corrections satisfy E*F = -G.
 * Robot::computeMJtJinv uses Pinocchio's sparse Cholesky of M; here M is factorised densely (same mathematics, different
 * rounding).  Where the reference itself departs from the exact expressions (dnu_passive has no dxi / dts term) the
 * departure is restated and documented in the tests.
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <float.h>
#include "../include/rbt_stage_layout.h"

#define IDX(i, j, ld) ((i) + (size_t)(j) * (ld))

#include "orc_linalg.h"  /* gemm(): register-blocked small GEMM shared by the oracle sources */

static int chol_lower(int n, double* A, int lda) {
  for (int j = 0; j < n; ++j) {
    double d = A[IDX(j, j, lda)];
    for (int k = 0; k < j; ++k) d -= A[IDX(j, k, lda)] * A[IDX(j, k, lda)];
    if (!(d > 0.0)) return 1;
    d = sqrt(d);
    A[IDX(j, j, lda)] = d;
    for (int i = j + 1; i < n; ++i) {
      double v = A[IDX(i, j, lda)];
      for (int k = 0; k < j; ++k) v -= A[IDX(i, k, lda)] * A[IDX(j, k, lda)];
      A[IDX(i, j, lda)] = v / d;
    }
  }
  return 0;
}

static void chol_solve(int n, const double* L, int ldl, int nrhs, double* B, int ldb) {
  for (int c = 0; c < nrhs; ++c) {
    double* b = B + (size_t)c * ldb;
    for (int i = 0; i < n; ++i) {
      double v = b[i];
      for (int k = 0; k < i; ++k) v -= L[IDX(i, k, ldl)] * b[k];
      b[i] = v / L[IDX(i, i, ldl)];
    }
    for (int i = n - 1; i >= 0; --i) {
      double v = b[i];
      for (int k = i + 1; k < n; ++k) v -= L[IDX(k, i, ldl)] * b[k];
      b[i] = v / L[IDX(i, i, ldl)];
    }
  }
}

/* Robot::computeMJtJinv  include/robotoc/robot/robot.hxx:642-683 (dense restatement; contact_inv_damping = 0).
 * Z ((nv+nf) x (nv+nf), ld ldz) = [[M, J^T],[J, 0]]^-1.  Returns nonzero if a Cholesky fails. */
static int mjtjinv(int nv, int nf, const double* M, const double* J, int ldj, double* Z, int ldz, double* ws) {
  double* Lm = ws;                 /* nv x nv */
  double* Minv = Lm + nv * nv;     /* nv x nv */
  double* JMi = Minv + nv * nv;    /* nf x nv : J Minv  (bottomLeft before the final overwrite) */
  double* S = JMi + nf * nv;       /* nf x nf */
  double* Sinv = S + nf * nf;      /* nf x nf */
  int info = 0;
  memcpy(Lm, M, sizeof(double) * nv * nv);
  if (chol_lower(nv, Lm, nv)) info |= 1;
  memset(Minv, 0, sizeof(double) * nv * nv);
  for (int i = 0; i < nv; ++i) Minv[IDX(i, i, nv)] = 1.0;
  chol_solve(nv, Lm, nv, nv, Minv, nv);                                   /* topLeft = M^-1               :676 */
  for (int j = 0; j < nv; ++j)
    for (int i = 0; i < nv; ++i) Z[IDX(i, j, ldz)] = Minv[IDX(i, j, nv)];
  if (nf == 0) return info;
  gemm(0, 0, nf, nv, nv, 1.0, J, ldj, Minv, nv, 0.0, JMi, nf);            /* bottomLeft = J * topLeft     :677 */
  gemm(0, 1, nf, nf, nv, 1.0, JMi, nf, J, ldj, 0.0, S, nf);               /* JMinvJt = J M^-1 J^T         :661-663 */
  memcpy(Sinv, S, sizeof(double) * nf * nf);
  if (chol_lower(nf, S, nf)) info |= 2;                                   /* llt_JMinvJt                  :667 */
  memset(Sinv, 0, sizeof(double) * nf * nf);
  for (int i = 0; i < nf; ++i) Sinv[IDX(i, i, nf)] = 1.0;
  chol_solve(nf, S, nf, nf, Sinv, nf);                                    /* -bottomRight = (J M^-1 J^T)^-1 :674-675 */
  for (int j = 0; j < nf; ++j)
    for (int i = 0; i < nf; ++i) Z[IDX(nv + i, nv + j, ldz)] = -Sinv[IDX(i, j, nf)];
  /* topRight = bottomLeft^T * (-bottomRight) = M^-1 J^T S^-1              :678 */
  for (int j = 0; j < nf; ++j)
    for (int i = 0; i < nv; ++i) {
      double acc = 0.0;
      for (int l = 0; l < nf; ++l) acc += JMi[IDX(l, i, nf)] * Sinv[IDX(l, j, nf)];
      Z[IDX(i, nv + j, ldz)] = acc;
    }
  /* topLeft -= topRight * bottomLeft                                     :679 */
  for (int j = 0; j < nv; ++j)
    for (int i = 0; i < nv; ++i) {
      double acc = 0.0;
      for (int l = 0; l < nf; ++l) acc += Z[IDX(i, nv + l, ldz)] * JMi[IDX(l, j, nf)];
      Z[IDX(i, j, ldz)] -= acc;
    }
  for (int j = 0; j < nv; ++j)                                            /* bottomLeft = topRight^T      :680 */
    for (int i = 0; i < nf; ++i) Z[IDX(nv + i, j, ldz)] = Z[IDX(j, nv + i, ldz)];
  return info;
}

static void inv3(const double* A, int lda, double* B, int ldb) {
  const double a = A[IDX(0, 0, lda)], b = A[IDX(0, 1, lda)], c = A[IDX(0, 2, lda)];
  const double d = A[IDX(1, 0, lda)], e = A[IDX(1, 1, lda)], f = A[IDX(1, 2, lda)];
  const double g = A[IDX(2, 0, lda)], h = A[IDX(2, 1, lda)], i = A[IDX(2, 2, lda)];
  const double det = a * (e * i - f * h) - b * (d * i - f * g) + c * (d * h - e * g);
  const double r = 1.0 / det;
  B[IDX(0, 0, ldb)] = (e * i - f * h) * r; B[IDX(0, 1, ldb)] = (c * h - b * i) * r; B[IDX(0, 2, ldb)] = (b * f - c * e) * r;
  B[IDX(1, 0, ldb)] = (f * g - d * i) * r; B[IDX(1, 1, ldb)] = (a * i - c * g) * r; B[IDX(1, 2, ldb)] = (c * d - a * f) * r;
  B[IDX(2, 0, ldb)] = (d * h - e * g) * r; B[IDX(2, 1, ldb)] = (b * g - a * h) * r; B[IDX(2, 2, ldb)] = (a * e - b * d) * r;
}

/* SE3JacobianInverse::compute  include/robotoc/robot/se3_jacobian_inverse.hxx:17-32  (6x6, ld 6; bottom-left stays 0) */
static void se3_jac_inverse(const double* Jac, double* Jinv) {
  double tmp[9];
  memset(Jinv, 0, sizeof(double) * 36);
  inv3(Jac, 6, Jinv, 6);
  inv3(Jac + IDX(3, 3, 6), 6, Jinv + IDX(3, 3, 6), 6);
  gemm(0, 0, 3, 3, 3, 1.0, Jac + IDX(0, 3, 6), 6, Jinv + IDX(3, 3, 6), 6, 0.0, tmp, 3);
  gemm(0, 0, 3, 3, 3, -1.0, Jinv, 6, tmp, 3, 0.0, Jinv + IDX(0, 3, 6), 6);
}

/* row r of the constraint table applied to the direction: J_r * d  (box: sign*d[var][idx]) */
static double* var_ptr(double* q, double* v, double* a, double* u, int var) {
  return var == RBT_VAR_Q ? q : var == RBT_VAR_V ? v : var == RBT_VAR_A ? a : u;
}

/* Does box row r act on this grid point?  Box limits never act on impact stages (constraints.cpp:347-354), and the position- /
 * velocity-level limits not on the first two grid points: ConstraintsData::setTimeStage (constraints_data.cpp:20-45) validates the
 * position level from GridInfo::stage >= 2, the velocity level from >= 1 (c->ineq_gate = max(0, 2 - stage)). */
static inline int box_row_on(const rbt_constraint_table* tab, const rbt_stage_ctrl* c, int r) {
  const int level = tab->box[r].var == RBT_VAR_Q ? 2 : (tab->box[r].var == RBT_VAR_V ? 1 : 0);
  return c->type != RBT_IMPACT && level + c->ineq_gate <= 2;
}

/*
 * One stage of "Forms linear system" (intermediate_stage.cpp:133-148 / impact_stage.cpp:115-121 / terminal_stage.cpp:102-106):
 *   pdipm::computeComplementarySlackness + Constraints::condenseSlackAndDual      pdipm.hxx:27-100, joint_*_limit.cpp:68-83,
 *                                                                                friction_cone.cpp:194-235
 *   condenseContactDynamics / condenseImpactDynamics                             contact_dynamics.cpp:55-164, impact_dynamics.cpp:38-80
 *   correctLinearize(Impact|Terminal)StateEquation                               state_equation.cpp:68-87, impact_state_equation.cpp:53-70
 *   STO scaling                                                                  intermediate_stage.cpp:140-148
 * Inputs: lin (read-only), con.{slack,dual,res}.  Outputs: kkt record, exp record, con.{cmpl,cond}.
 */
int orc_stage_condense(const rbt_stage_dims* sd, const rbt_constraint_table* tab, const rbt_stage_ctrl* c,
                       const double* lin, double* con, double* kkt, double* ex) {
  rbt_stage_layout S;
  rbt_make_stage_layout(sd, &S);
  rbt_dims kd = {sd->nv, sd->nu, sd->ns_max, sd->n_passive};
  rbt_layout K;
  rbt_make_layout(&kd, &K);
  const int nv = S.nv, nu = S.nu, nx = S.nx, np = S.np, nvfm = S.nvf, nfm = S.nfm;
  const int type = c->type;
  int info = 0;
  memset(kkt, 0, sizeof(double) * K.k_stride);
  memset(ex, 0, sizeof(double) * S.e_stride);
  if (type == RBT_TERMINAL) {
    /* terminal_stage.cpp:94-106: no constraints, no dynamics; only Fqq_prev_inv for the costate correction */
    memcpy(kkt + K.k_Qxx, lin + S.l_Qxx, sizeof(double) * nx * nx);
    memcpy(kkt + K.k_lx, lin + S.l_lx, sizeof(double) * nx);
    if (np == 6) se3_jac_inverse(lin + S.l_se3 + 36, ex + S.e_Fqqpi);
    return 0;
  }
  const int impact = (type == RBT_IMPACT);
  const int nf = c->nf, nvf = nv + nf, ns = impact ? 0 : c->ns;
  const double dt = c->dt;
  /* working copies of the blocks the constraints / condensing mutate */
  double* Qxx = kkt + K.k_Qxx;
  double* Qxu = kkt + K.k_Qxu;
  double* Quu = kkt + K.k_Quu;
  double* lx = kkt + K.k_lx;
  double* lu = kkt + K.k_lu;
  double* Fx = kkt + K.k_Fx;
  memcpy(Qxx, lin + S.l_Qxx, sizeof(double) * nx * nx);
  memcpy(Quu, lin + S.l_Quu, sizeof(double) * nu * nu);
  memcpy(lx, lin + S.l_lx, sizeof(double) * nx);
  memcpy(lu, lin + S.l_lu, sizeof(double) * nu);
  memcpy(Fx, lin + S.l_Fx, sizeof(double) * nx);
  /* per-stage scratch on the stack (a heap allocation per stage would be charged to the CPU baseline) */
  double Qaa[nv], Qff[(size_t)nfm * nfm + 1], Qqf[(size_t)nv * nfm + 1], la[nv], lf[nfm + 1];
  memset(Qaa, 0, sizeof(Qaa)); memset(Qff, 0, sizeof(Qff)); memset(Qqf, 0, sizeof(Qqf));
  memset(la, 0, sizeof(la)); memset(lf, 0, sizeof(lf));
  memcpy(Qaa, lin + S.l_Qaa, sizeof(double) * nv);
  memcpy(Qff, lin + S.l_Qff, sizeof(double) * nfm * nfm);
  memcpy(Qqf, lin + S.l_Qqf, sizeof(double) * nv * nfm);
  memcpy(la, lin + S.l_la, sizeof(double) * nv);
  memcpy(lf, lin + S.l_lf, sizeof(double) * nfm);

  /* ---------------- PDIPM: box limits on Intermediate / Lift stages; friction cones there and -- if the table registers
   * ImpactFrictionCone (impact_friction_cone.cpp:190-235, the same algebra on the impact forces) -- on Impact stages */
  const int cones = !impact || tab->impact_friction_cone;
  if (cones) {
    double* slack = con + S.c_slack;
    double* dual = con + S.c_dual;
    double* res = con + S.c_res;
    double* cmpl = con + S.c_cmpl;
    double* cond = con + S.c_cond;
    double* lq = lx;
    double* lv = lx + nv;
    for (int r = 0; r < tab->n_box; ++r) {
      if (!box_row_on(tab, c, r)) continue;
      const rbt_box_row* b = &tab->box[r];
      cmpl[r] = slack[r] * dual[r] - tab->barrier;                         /* pdipm.hxx:27-31 */
      cond[r] = (dual[r] * res[r] - cmpl[r]) / slack[r];                   /* pdipm.hxx:66-70 */
      const double w = dual[r] / slack[r];
      /* joint_*_limit.cpp:68-75: diagonal += dual/slack ; gradient -+ cond */
      switch (b->var) {
        case RBT_VAR_Q: Qxx[IDX(b->idx, b->idx, nx)] += w; lq[b->idx] += b->sign * cond[r]; break;
        case RBT_VAR_V: Qxx[IDX(nv + b->idx, nv + b->idx, nx)] += w; lv[b->idx] += b->sign * cond[r]; break;
        case RBT_VAR_A: Qaa[b->idx] += w; la[b->idx] += b->sign * cond[r]; break;
        default: Quu[IDX(b->idx, b->idx, nu)] += w; lu[b->idx] += b->sign * cond[r]; break;
      }
    }
    /* FrictionCone::condenseSlackAndDual  friction_cone.cpp:194-235 */
    int fstack = 0;
    for (int ci = 0; ci < tab->n_contacts; ++ci) {
      const int base = tab->n_box + 5 * ci;
      if (!((c->contact_mask >> ci) & 1)) {
        for (int r = 0; r < 5; ++r) { cond[base + r] = 0.0; }               /* data.cond.setZero()  :198 */
        continue;
      }
      const double* dgdq = lin + S.l_dgdq + (size_t)ci * 5 * nv; /* 5 x nv, ld 5 */
      const double* dgdf = lin + S.l_dgdf + (size_t)ci * 15;     /* 5 x 3,  ld 5 */
      double ri[5];
      for (int r = 0; r < 5; ++r) {
        cmpl[base + r] = slack[base + r] * dual[base + r] - tab->barrier;
        cond[base + r] = (dual[base + r] * res[base + r] - cmpl[base + r]) / slack[base + r];
        ri[r] = dual[base + r] / slack[base + r];
      }
      for (int j = 0; j < nv; ++j) {                                       /* lq += dg_dq^T cond  :207 */
        double acc = 0.0;
        for (int r = 0; r < 5; ++r) acc += dgdq[IDX(r, j, 5)] * cond[base + r];
        lq[j] += acc;
      }
      for (int j = 0; j < 3; ++j) {                                        /* lf += dg_df^T cond  :208-209 */
        double acc = 0.0;
        for (int r = 0; r < 5; ++r) acc += dgdf[IDX(r, j, 5)] * cond[base + r];
        lf[fstack + j] += acc;
      }
      for (int j = 0; j < nv; ++j)                                         /* Qqq += dg_dq^T diag(r) dg_dq :217-218 */
        for (int i = 0; i < nv; ++i) {
          double acc = 0.0;
          for (int r = 0; r < 5; ++r) acc += dgdq[IDX(r, i, 5)] * ri[r] * dgdq[IDX(r, j, 5)];
          Qxx[IDX(i, j, nx)] += acc;
        }
      for (int j = 0; j < 3; ++j)                                          /* Qqf += dg_dq^T diag(r) dg_df :219-220 */
        for (int i = 0; i < nv; ++i) {
          double acc = 0.0;
          for (int r = 0; r < 5; ++r) acc += dgdq[IDX(r, i, 5)] * ri[r] * dgdf[IDX(r, j, 5)];
          Qqf[IDX(i, fstack + j, nv)] += acc;
        }
      for (int j = 0; j < 3; ++j)                                          /* Qff += dg_df^T diag(r) dg_df :221-222 */
        for (int i = 0; i < 3; ++i) {
          double acc = 0.0;
          for (int r = 0; r < 5; ++r) acc += dgdf[IDX(r, i, 5)] * ri[r] * dgdf[IDX(r, j, 5)];
          Qff[IDX(fstack + i, fstack + j, nfm)] += acc;
        }
      fstack += 3;
    }
  }

  /* ---------------- condenseContactDynamics / condenseImpactDynamics */
  double* Z = ex + S.e_Z;        /* ld nvfm */
  double* R = ex + S.e_R;        /* ld nvfm */
  double* r_ = ex + S.e_r;
  double* Qafqv = ex + S.e_Qafqv;
  double* Qafu = ex + S.e_Qafu;  /* Qafu_full: nvf x nv, ld nvfm */
  double* laf = ex + S.e_laf;
  const double* D = lin + S.l_D; /* ld nvfm */
  const double* IDC = lin + S.l_IDC;
  double ws[(size_t)3 * nv * nv + 2 * nfm * nv + 2 * nfm * nfm + 16];
  memset(ws, 0, sizeof(ws));
  info |= mjtjinv(nv, nf, lin + S.l_M, lin + S.l_J, nfm, Z, nvfm, ws);    /* contact_dynamics.cpp:64 / impact :42 */
  gemm(0, 0, nvf, nx, nvf, 1.0, Z, nvfm, D, nvfm, 0.0, R, nvfm);          /* MJtJinv_dIDCdqv = Z dIDCdqv   :65 */
  gemm(0, 0, nvf, 1, nvf, 1.0, Z, nvfm, IDC, nvfm, 0.0, r_, nvfm);        /* MJtJinv_IDC = Z IDC           :66 */
  for (int j = 0; j < nx; ++j) {
    for (int i = 0; i < nv; ++i) Qafqv[IDX(i, j, nvfm)] = -Qaa[i] * R[IDX(i, j, nvfm)];                 /* :68-70 */
    for (int i = 0; i < nf; ++i) {                                                                       /* :71-72 */
      double acc = 0.0;
      for (int l = 0; l < nf; ++l) acc += Qff[IDX(i, l, nfm)] * R[IDX(nv + l, j, nvfm)];
      Qafqv[IDX(nv + i, j, nvfm)] = -acc;
    }
  }
  for (int j = 0; j < nv; ++j)                                                                           /* :73-74 */
    for (int i = 0; i < nf; ++i) Qafqv[IDX(nv + i, j, nvfm)] -= Qqf[IDX(j, i, nv)];
  if (!impact) {
    for (int j = 0; j < nv; ++j) {
      for (int i = 0; i < nv; ++i) Qafu[IDX(i, j, nvfm)] = Qaa[i] * Z[IDX(i, j, nvfm)];                  /* :75-77 */
      for (int i = 0; i < nf; ++i) {                                                                      /* :78-79 */
        double acc = 0.0;
        for (int l = 0; l < nf; ++l) acc += Qff[IDX(i, l, nfm)] * Z[IDX(nv + l, j, nvfm)];
        Qafu[IDX(nv + i, j, nvfm)] = acc;
      }
    }
  }
  for (int i = 0; i < nv; ++i) laf[i] = la[i] - Qaa[i] * r_[i];                                           /* :80,82-84 */
  for (int i = 0; i < nf; ++i) {                                                                          /* :81,85-86 */
    double acc = 0.0;
    for (int l = 0; l < nf; ++l) acc += Qff[IDX(i, l, nfm)] * r_[nv + l];
    laf[nv + i] = -lf[i] - acc;
  }
  gemm(1, 0, nx, nx, nvf, -1.0, R, nvfm, Qafqv, nvfm, 1.0, Qxx, nx);                                      /* Qxx -= R^T Qafqv :88-89 */
  gemm(0, 0, nv, nx, nf, 1.0, Qqf, nv, R + nv, nvfm, 1.0, Qxx, nx);                                       /* Qxx[:nv,:] += Qqf R_f :90-91 */
  if (!impact) {
    double* Qxup = ex + S.e_Qxup; /* nx x np */
    double* Quup = ex + S.e_Quup; /* np x nu */
    double* lup = ex + S.e_lup;
    if (np > 0) {
      gemm(1, 0, nx, np, nvf, -1.0, R, nvfm, Qafu, nvfm, 0.0, Qxup, nx);                                  /* :93-94 */
      gemm(0, 0, nv, np, nf, -1.0, Qqf, nv, Z + nv, nvfm, 1.0, Qxup, nx);                                 /* :95-96 */
    }
    gemm(1, 0, nx, nu, nvf, -1.0, R, nvfm, Qafu + (size_t)np * nvfm, nvfm, 1.0, Qxu, nx);                 /* :97-98 / :103-104 */
    gemm(0, 0, nv, nu, nf, -1.0, Qqf, nv, Z + nv + (size_t)np * nvfm, nvfm, 1.0, Qxu, nx);                /* :99-100 / :105-106 */
    gemm(1, 0, nx, 1, nvf, -1.0, R, nvfm, laf, nvfm, 1.0, lx, nx);                                        /* lx -= R^T laf :108-109 */
    gemm(0, 0, nv, 1, nf, 1.0, Qqf, nv, r_ + nv, nvfm, 1.0, lx, nx);                                      /* lq += Qqf r_f :110-111 */
    if (np > 0)
      gemm(0, 0, np, nu, nvf, 1.0, Z, nvfm, Qafu + (size_t)np * nvfm, nvfm, 0.0, Quup, np);               /* :114-115 */
    gemm(0, 0, nu, nu, nvf, 1.0, Z + np, nvfm, Qafu + (size_t)np * nvfm, nvfm, 1.0, Quu, nu);             /* :116-117 / :120-121 */
    if (np > 0) {
      memcpy(lup, lin + S.l_lup, sizeof(double) * np);
      gemm(0, 0, np, 1, nvf, 1.0, Z, nvfm, laf, nvfm, 1.0, lup, np);                                      /* :124-125 */
    }
    gemm(0, 0, nu, 1, nvf, 1.0, Z + np, nvfm, laf, nvfm, 1.0, lu, nu);                                    /* :127-128 */
  } else {
    gemm(1, 0, nx, 1, nvf, -1.0, R, nvfm, laf, nvfm, 1.0, lx, nx);                                        /* impact :67-68 */
    gemm(0, 0, nv, 1, nf, 1.0, Qqf, nv, r_ + nv, nvfm, 1.0, lx, nx);                                      /* impact :69-70 */
  }
  /* state equation blocks: Fqq, Fqv from linearizeStateEquation (state_equation.cpp:42-56), Fvq,Fvv,Fvu,Fv from condensing */
  double* Fxx = kkt + K.k_Fxx;
  for (int i = 0; i < nv; ++i) Fxx[IDX(i, i, nx)] = 1.0;
  if (np == 6)
    for (int j = 0; j < 6; ++j)
      for (int i = 0; i < 6; ++i) Fxx[IDX(i, j, nx)] = lin[S.l_se3 + IDX(i, j, 6)];   /* dSubtract/dqf top-left */
  if (!impact)
    for (int i = 0; i < nv; ++i) Fxx[IDX(i, nv + i, nx)] = dt;
  const double sdt = impact ? 1.0 : dt;
  for (int j = 0; j < nv; ++j)
    for (int i = 0; i < nv; ++i) {
      Fxx[IDX(nv + i, j, nx)] = -sdt * R[IDX(i, j, nvfm)];                                                /* Fvq :130 / impact :71 */
      Fxx[IDX(nv + i, nv + j, nx)] = -sdt * R[IDX(i, nv + j, nvfm)] + (i == j ? 1.0 : 0.0);               /* Fvv :131-133 / :72-73 */
    }
  if (!impact) {
    double* Fvu = kkt + K.k_Fvu;
    for (int j = 0; j < nu; ++j)
      for (int i = 0; i < nv; ++i) Fvu[IDX(i, j, nv)] = dt * Z[IDX(i, np + j, nvfm)];                     /* :134 */
  }
  for (int i = 0; i < nv; ++i) Fx[nv + i] -= sdt * r_[i];                                                 /* Fv -= dt r_a :135 / :74 */

  /* switching constraint   contact_dynamics.cpp:138-153 */
  if (ns > 0) {
    const double* Phia = lin + S.l_Phia; /* ns x nv, ld ns */
    double* Phix = kkt + K.k_Phix;
    double* Phiu = kkt + K.k_Phiu;
    double* pp = kkt + K.k_p;
    double* Phit = kkt + K.k_Phit;
    memcpy(ex + S.e_Phia, Phia, sizeof(double) * ns * nv);
    memcpy(Phix, lin + S.l_Phix, sizeof(double) * ns * nx);
    memcpy(pp, lin + S.l_p, sizeof(double) * ns);
    memcpy(Phit, lin + S.l_Phit, sizeof(double) * ns);
    gemm(0, 0, ns, nx, nv, -1.0, Phia, ns, R, nvfm, 1.0, Phix, ns);                                       /* :143-144 */
    gemm(0, 0, ns, nu, nv, 1.0, Phia, ns, Z + (size_t)np * nvfm, nvfm, 0.0, Phiu, ns);                    /* :145-146 */
    gemm(0, 0, ns, 1, nv, -1.0, Phia, ns, r_, nvfm, 1.0, Phit, ns);                                       /* :147-148 */
    gemm(0, 0, ns, 1, nv, -1.0, Phia, ns, r_, nvfm, 1.0, pp, ns);                                         /* :149-150 */
  }
  /* STO sensitivities   contact_dynamics.cpp:156-163 (skipped on impact stages: no dt) */
  double* haf = ex + S.e_haf;
  double hsc = lin[S.l_sc + 0], Qtt = lin[S.l_sc + 1];
  double* hx = kkt + K.k_hx;
  double* hu = kkt + K.k_hu;
  double* fx = kkt + K.k_fx;
  if (!impact) {
    memcpy(hx, lin + S.l_hx, sizeof(double) * nx);
    memcpy(hu, lin + S.l_hu, sizeof(double) * nu);
    memcpy(fx, lin + S.l_fx, sizeof(double) * nx);
    for (int i = 0; i < nv; ++i) haf[i] = lin[S.l_ha + i];
    for (int i = 0; i < nf; ++i) haf[nv + i] = -lin[S.l_hf + i];
    for (int i = 0; i < nvf; ++i) hsc -= r_[i] * haf[i];                                                  /* h -= r . haf :158 */
    gemm(1, 0, nx, 1, nvf, -1.0, R, nvfm, haf, nvfm, 1.0, hx, nx);                                        /* hx -= R^T haf :159 */
    gemm(0, 0, nv, 1, nf, 1.0 / dt, Qqf, nv, r_ + nv, nvfm, 1.0, hx, nx);                                 /* hq += (1/dt) Qqf r_f :160-161 */
    gemm(0, 0, nu, 1, nvf, 1.0, Z + np, nvfm, haf, nvfm, 1.0, hu, nu);                                    /* hu += Z[np:nv,:] haf :162-163 */
  }

  /* ---------------- floating base: correctLinearizeStateEquation  state_equation.cpp:68-87 / impact_state_equation.cpp:53-70 */
  if (np == 6) {
    double Fqq_inv[36], tmp[36], v6[6];
    se3_jac_inverse(lin + S.l_se3 + 36, ex + S.e_Fqqpi);      /* Fqq_prev_inv  :76 */
    se3_jac_inverse(lin + S.l_se3 + 72, Fqq_inv);             /* Fqq_inv       :77-78 */
    for (int j = 0; j < 6; ++j)
      for (int i = 0; i < 6; ++i) tmp[IDX(i, j, 6)] = Fxx[IDX(i, j, nx)];
    for (int j = 0; j < 6; ++j)
      for (int i = 0; i < 6; ++i) {
        double acc = 0.0;
        for (int l = 0; l < 6; ++l) acc += Fqq_inv[IDX(i, l, 6)] * tmp[IDX(l, j, 6)];
        Fxx[IDX(i, j, nx)] = -acc;                                                                         /* :80 */
        if (!impact) Fxx[IDX(i, nv + j, nx)] = -dt * Fqq_inv[IDX(i, j, 6)];                                /* :81 */
      }
    for (int i = 0; i < 6; ++i) v6[i] = Fx[i];
    for (int i = 0; i < 6; ++i) {
      double acc = 0.0;
      for (int l = 0; l < 6; ++l) acc += Fqq_inv[IDX(i, l, 6)] * v6[l];
      Fx[i] = -acc;                                                                                        /* :83 */
    }
    if (!impact) {
      for (int i = 0; i < 6; ++i) v6[i] = fx[i];
      for (int i = 0; i < 6; ++i) {
        double acc = 0.0;
        for (int l = 0; l < 6; ++l) acc += Fqq_inv[IDX(i, l, 6)] * v6[l];
        fx[i] = -acc;                                                                                      /* :85 */
      }
    }
  }
  /* ---------------- STO scaling   intermediate_stage.cpp:140-148 */
  if (!impact) {
    const double g1 = 1.0 / c->ngrids_in_phase;
    hsc *= g1;
    for (int i = 0; i < nx; ++i) { hx[i] *= g1; fx[i] *= g1; }
    for (int i = 0; i < nu; ++i) hu[i] *= g1;
    Qtt *= g1 * g1;
    kkt[K.k_sc + 0] = Qtt;
    kkt[K.k_sc + 1] = -Qtt;
    kkt[K.k_sc + 2] = hsc;
    if (ns > 0)
      for (int i = 0; i < ns; ++i) kkt[K.k_Phit + i] *= g1;
  }

  return info;
}

/* pdipm::fractionToBoundary  pdipm.hxx:121-142 */
static double fraction_to_boundary(int n, double rate, const double* v, const double* dv) {
  double m = 1.0;
  for (int i = 0; i < n; ++i) {
    const double f = -rate * (v[i] / dv[i]);
    if (f > 0 && f < 1 && f < m) m = f;
  }
  return m;
}

/*
 * expandPrimal + step sizes for one stage:
 *   expandContactDynamicsPrimal / expandImpactDynamicsPrimal   contact_dynamics.cpp:167-174, impact_dynamics.cpp:83-88
 *   Constraints::expandSlackAndDual                            joint_*_limit.cpp:78-83, friction_cone.cpp:238-268, pdipm.hxx:159-164
 *   maxSlackStepSize / maxDualStepSize                         constraint_component_base.hxx:13-22
 * d: Riccati direction record of this stage; xd: expanded direction record (daf written); steps[2] = {primal, dual}.
 */
void orc_stage_expand_primal(const rbt_stage_dims* sd, const rbt_constraint_table* tab, const rbt_stage_ctrl* c,
                             const double* lin, const double* ex, const double* d, double* con, double* xd,
                             double* steps) {
  rbt_stage_layout S;
  rbt_make_stage_layout(sd, &S);
  rbt_dims kd = {sd->nv, sd->nu, sd->ns_max, sd->n_passive};
  rbt_layout K;
  rbt_make_layout(&kd, &K);
  const int nv = S.nv, nu = S.nu, nx = S.nx, np = S.np, nvfm = S.nvf;
  steps[0] = 1.0;
  steps[1] = 1.0;
  if (c->type == RBT_TERMINAL) return;                        /* terminal_stage.cpp:109-136 */
  const int impact = (c->type == RBT_IMPACT);
  const int nf = c->nf, nvf = nv + nf;
  const double* dx = d + K.d_dx;
  const double* du = d + K.d_du;
  double* daf = xd + S.x_daf;
  gemm(0, 0, nvf, 1, nx, -1.0, ex + S.e_R, nvfm, dx, nx, 0.0, daf, nvfm);                                 /* daf = -R dx :169 */
  if (!impact) gemm(0, 0, nvf, 1, nu, 1.0, ex + S.e_Z + (size_t)np * nvfm, nvfm, du, nu, 1.0, daf, nvfm); /* += Z[:,np:np+nu] du :170-171 */
  for (int i = 0; i < nvf; ++i) daf[i] -= ex[S.e_r + i];                                                  /* -= r :172 */
  for (int i = 0; i < nf; ++i) daf[nv + i] *= -1.0;                                                       /* df *= -1 :173 */
  if (impact && !tab->impact_friction_cone) return;           /* no impact-level constraints in the table */
  double* slack = con + S.c_slack;
  double* dual = con + S.c_dual;
  double* res = con + S.c_res;
  double* cmpl = con + S.c_cmpl;
  double* dslack = con + S.c_dslack;
  double* ddual = con + S.c_ddual;
  double* dq = (double*)dx;
  double* dv = (double*)dx + nv;
  for (int r = 0; r < tab->n_box; ++r) {
    if (!box_row_on(tab, c, r)) continue;
    const rbt_box_row* b = &tab->box[r];
    const double* var = var_ptr(dq, dv, daf, (double*)du, b->var);
    dslack[r] = -b->sign * var[b->idx] - res[r];                                                          /* joint_*_limit.cpp:78-82 */
    ddual[r] = -(dual[r] * dslack[r] + cmpl[r]) / slack[r];                                               /* pdipm.hxx:159-164 */
  }
  int fstack = 0;
  for (int ci = 0; ci < tab->n_contacts; ++ci) {
    const int base = tab->n_box + 5 * ci;
    for (int r = 0; r < 5; ++r) { dslack[base + r] = 1.0; ddual[base + r] = 1.0; }                        /* friction_cone.cpp:244-245 */
    if (!((c->contact_mask >> ci) & 1)) continue;
    const double* dgdq = lin + S.l_dgdq + (size_t)ci * 5 * nv;
    const double* dgdf = lin + S.l_dgdf + (size_t)ci * 15;
    for (int r = 0; r < 5; ++r) {
      double acc = 0.0;
      for (int j = 0; j < nv; ++j) acc += dgdq[IDX(r, j, 5)] * dq[j];
      for (int j = 0; j < 3; ++j) acc += dgdf[IDX(r, j, 5)] * daf[nv + fstack + j];
      dslack[base + r] = -acc - res[base + r];                                                            /* :253-256 */
      ddual[base + r] = -(dual[base + r] * dslack[base + r] + cmpl[base + r]) / slack[base + r];          /* :257 */
    }
    fstack += 3;
  }
  /* rows that do not act on this grid point (box rows of an impact stage, gated levels) take no part: maxSlackStepSize /
   * maxDualStepSize only visit the valid levels (constraints.cpp:397-440) */
  steps[0] = 1.0; steps[1] = 1.0;
  for (int r = 0; r < S.nc; ++r) {
    if (r < tab->n_box && !box_row_on(tab, c, r)) continue;
    const double fp = fraction_to_boundary(1, tab->fraction_to_boundary, slack + r, dslack + r);
    const double fd = fraction_to_boundary(1, tab->fraction_to_boundary, dual + r, ddual + r);
    if (fp < steps[0]) steps[0] = fp;
    if (fd < steps[1]) steps[1] = fd;
  }
}

/* free-flyer part of Robot::integrateConfiguration: q(p, quat xyzw) <- q (+) step*dq, textbook SE(3) exponential */
static void integrate_free_flyer(double* q, const double* dq, double step) {
  const double vx = step * dq[0], vy = step * dq[1], vz = step * dq[2];
  const double wx = step * dq[3], wy = step * dq[4], wz = step * dq[5];
  const double th2 = wx * wx + wy * wy + wz * wz, th = sqrt(th2);
  double b, cc; /* (1-cos th)/th^2, (th - sin th)/th^3 */
  if (th < 1e-6) {
    b = 0.5 - th2 / 24.0; cc = 1.0 / 6.0 - th2 / 120.0;
  } else {
    /* 1 - cos th = 2 sin^2(th/2): the difference form loses up to 2u / th^2 of b (9e-5 relative just above th = 1e-6) */
    const double s2 = sin(0.5 * th), c2 = cos(0.5 * th);
    b = 2.0 * s2 * s2 / th2; cc = (th - 2.0 * s2 * c2) / (th2 * th);
  }
  /* t = V v,  V = I + b [w]x + cc [w]x^2 */
  const double cx = wy * vz - wz * vy, cy = wz * vx - wx * vz, cz = wx * vy - wy * vx;
  const double ccx = wy * cz - wz * cy, ccy = wz * cx - wx * cz, ccz = wx * cy - wy * cx;
  const double tx = vx + b * cx + cc * ccx, ty = vy + b * cy + cc * ccy, tz = vz + b * cz + cc * ccz;
  /* rotate t by the current quaternion and add to p */
  const double qx = q[3], qy = q[4], qz = q[5], qw = q[6];
  const double ux = qy * tz - qz * ty, uy = qz * tx - qx * tz, uz = qx * ty - qy * tx;
  const double u2x = qy * uz - qz * uy, u2y = qz * ux - qx * uz, u2z = qx * uy - qy * ux;
  q[0] += tx + 2.0 * (qw * ux + u2x);
  q[1] += ty + 2.0 * (qw * uy + u2y);
  q[2] += tz + 2.0 * (qw * uz + u2z);
  /* quaternion of exp(w): (sin(th/2)/th * w, cos(th/2)) */
  double sh, ch;
  if (th < 1e-6) { sh = 0.5 - th2 / 48.0; ch = 1.0 - th2 / 8.0; } else { sh = sin(0.5 * th) / th; ch = cos(0.5 * th); }
  const double ex_ = sh * wx, ey = sh * wy, ez = sh * wz, ew = ch;
  double nx_ = qw * ex_ + qx * ew + qy * ez - qz * ey;
  double ny = qw * ey - qx * ez + qy * ew + qz * ex_;
  double nz = qw * ez + qx * ey - qy * ex_ + qz * ew;
  double nw = qw * ew - qx * ex_ - qy * ey - qz * ez;
  const double nrm = 1.0 / sqrt(nx_ * nx_ + ny * ny + nz * nz + nw * nw);
  q[3] = nx_ * nrm; q[4] = ny * nrm; q[5] = nz * nrm; q[6] = nw * nrm;
}

/*
 * expandDual + update for one stage (DirectMultipleShooting::integrateSolution, direct_multiple_shooting.cpp:212-241):
 *   expandContactDynamicsDual / expandImpactDynamicsDual    contact_dynamics.cpp:177-202, impact_dynamics.cpp:91-96
 *   correctCostateDirection                                 state_equation.cpp:90-95
 *   SplitSolution::integrate                                src/core/split_solution.cpp:58-90
 *   updateSlack / updateDual                                constraint_component_base.hxx:25-36
 * d (mutable: dlmd head corrected), dn = direction record of stage i+1 (NULL on the terminal stage), ex is mutated (laf) as
 * the reference mutates data.laf().
 */
void orc_stage_expand_dual_update(const rbt_stage_dims* sd, const rbt_constraint_table* tab, const rbt_stage_ctrl* c,
                                  double* ex, double* d, const double* dn, double* xd, double* con, double* sol,
                                  double primal_step, double dual_step) {
  rbt_stage_layout S;
  rbt_make_stage_layout(sd, &S);
  rbt_dims kd = {sd->nv, sd->nu, sd->ns_max, sd->n_passive};
  rbt_layout K;
  rbt_make_layout(&kd, &K);
  const int nv = S.nv, nu = S.nu, nx = S.nx, np = S.np, nvfm = S.nvf;
  const int type = c->type;
  const int impact = (type == RBT_IMPACT), terminal = (type == RBT_TERMINAL);
  const int nf = terminal ? 0 : c->nf, nvf = nv + nf, ns = (impact || terminal) ? 0 : c->ns;
  const double* dx = d + K.d_dx;
  const double* du = d + K.d_du;
  double* dbm = xd + S.x_dbetamu;
  if (!terminal) {
    const double* dgmm_n = dn + K.d_dlmdgmm + nv;
    double* laf = ex + S.e_laf;
    if (!impact) {
      const double dt = c->dt;
      double dts = 0.0;                                                                                    /* intermediate_stage.cpp:167-170 */
      if (c->ngrids_in_phase > 0) dts = (d[K.d_dts + 1] - d[K.d_dts]) / c->ngrids_in_phase;
      if (np > 0) {                                                                                        /* contact_dynamics.cpp:182-190 */
        double* dnup = xd + S.x_dnup;
        for (int i = 0; i < np; ++i) dnup[i] = -ex[S.e_lup + i];
        gemm(0, 0, np, 1, nu, -1.0, ex + S.e_Quup, np, du, nu, 1.0, dnup, np);
        gemm(1, 0, np, 1, nx, -1.0, ex + S.e_Qxup, nx, dx, nx, 1.0, dnup, np);
        gemm(0, 0, np, 1, nv, -dt, ex + S.e_Z, nvfm, dgmm_n, nv, 1.0, dnup, np);
      }
      gemm(0, 0, nvf, 1, nx, 1.0, ex + S.e_Qafqv, nvfm, dx, nx, 1.0, laf, nvfm);                           /* :191 */
      gemm(0, 0, nvf, 1, nu, 1.0, ex + S.e_Qafu + (size_t)np * nvfm, nvfm, du, nu, 1.0, laf, nvfm);        /* :192 */
      for (int i = 0; i < nv; ++i) laf[i] += dt * dgmm_n[i];                                               /* :193 */
      if (ns > 0) gemm(1, 0, nv, 1, ns, 1.0, ex + S.e_Phia, ns, d + K.d_dxi, ns, 1.0, laf, nvfm);          /* :194-197 */
      if (dts < -DBL_EPSILON || dts > DBL_EPSILON)                                                         /* :198-201 */
        for (int i = 0; i < nvf; ++i) laf[i] += dts * ex[S.e_haf + i];
    } else {
      gemm(0, 0, nvf, 1, nx, 1.0, ex + S.e_Qafqv, nvfm, dx, nx, 1.0, laf, nvfm);                           /* impact_dynamics.cpp:93 */
      for (int i = 0; i < nv; ++i) laf[i] += dgmm_n[i];                                                    /* :94 */
    }
    gemm(0, 0, nvf, 1, nvf, -1.0, ex + S.e_Z, nvfm, laf, nvfm, 0.0, dbm, nvfm);                            /* dbetamu = -Z laf :202 / :95 */
  }
  if (np == 6) {                                                                                           /* correctCostateDirection */
    double tmp[6];
    double* dl = d + K.d_dlmdgmm;
    for (int i = 0; i < 6; ++i) {
      double acc = 0.0;
      for (int l = 0; l < 6; ++l) acc += ex[S.e_Fqqpi + IDX(l, i, 6)] * dl[l];
      tmp[i] = acc;
    }
    for (int i = 0; i < 6; ++i) dl[i] = -tmp[i];
  }
  /* SplitSolution::integrate   split_solution.cpp:58-90 */
  const double a_ = primal_step;
  double* q = sol + S.s_q;
  if (np == 6) {
    integrate_free_flyer(q, dx, a_);
    for (int i = 6; i < nv; ++i) q[i + 1] += a_ * dx[i];
  } else {
    for (int i = 0; i < nv; ++i) q[i] += a_ * dx[i];
  }
  for (int i = 0; i < nv; ++i) sol[S.s_v + i] += a_ * dx[nv + i];
  const double* daf = xd + S.x_daf;
  if (terminal) {
    /* terminal: d.da, d.du are zero-sized/zero in the reference's direction; only q,v,lmd,gmm move */
  } else if (!impact) {
    for (int i = 0; i < nv; ++i) sol[S.s_a + i] += a_ * daf[i];
    for (int i = 0; i < nv; ++i) sol[S.s_dv + i] = 0.0;
    for (int i = 0; i < nu; ++i) sol[S.s_u + i] += a_ * du[i];
  } else {
    for (int i = 0; i < nv; ++i) sol[S.s_a + i] = 0.0;
    for (int i = 0; i < nv; ++i) sol[S.s_dv + i] += a_ * daf[i];
    for (int i = 0; i < nu; ++i) sol[S.s_u + i] = 0.0;
  }
  for (int i = 0; i < nv; ++i) sol[S.s_lmd + i] += a_ * d[K.d_dlmdgmm + i];
  for (int i = 0; i < nv; ++i) sol[S.s_gmm + i] += a_ * d[K.d_dlmdgmm + nv + i];
  if (!terminal) {
    for (int i = 0; i < nv; ++i) sol[S.s_beta + i] += a_ * dbm[i];
    if (np > 0 && !impact)
      for (int i = 0; i < np; ++i) sol[S.s_nup + i] += a_ * xd[S.x_dnup + i];
    for (int i = 0; i < nf; ++i) sol[S.s_f + i] += a_ * daf[nv + i];
    for (int i = 0; i < nf; ++i) sol[S.s_mu + i] += a_ * dbm[nv + i];
    if (ns > 0)
      for (int i = 0; i < ns; ++i) sol[S.s_xi + i] += a_ * d[K.d_dxi + i];
    if (!impact || tab->impact_friction_cone) {
      for (int r = 0; r < S.nc; ++r) {
        if (r < S.nbox && !box_row_on(tab, c, r)) continue;
        con[S.c_slack + r] += primal_step * con[S.c_dslack + r];
        con[S.c_dual + r] += dual_step * con[S.c_ddual + r];
      }
    }
  }
}

/* ---------------- batched drivers (OpenMP over OCP instances; the reference's own OpenMP loop is over stages) */
#ifdef _OPENMP
#include <omp.h>
#endif

int orc_condense_batch(const rbt_stage_dims* sd, const rbt_constraint_table* tab, const rbt_stage_ctrl* ctrl, int n_grid,
                       int batch, const double* lin, double* con, double* kkt, double* ex, int nthreads) {
  rbt_stage_layout S;
  rbt_make_stage_layout(sd, &S);
  rbt_dims kd = {sd->nv, sd->nu, sd->ns_max, sd->n_passive};
  rbt_layout K;
  rbt_make_layout(&kd, &K);
  int info = 0;
#ifdef _OPENMP
  if (nthreads > 0) omp_set_num_threads(nthreads);
#endif
#pragma omp parallel for schedule(dynamic) reduction(| : info)
  for (int b = 0; b < batch; ++b)
    for (int i = 0; i < n_grid; ++i) {
      const size_t o = (size_t)b * n_grid + i;
      info |= orc_stage_condense(sd, tab, &ctrl[i], lin + o * S.l_stride, con + o * S.c_stride, kkt + o * K.k_stride,
                                 ex + o * S.e_stride);
    }
  return info;
}

/* computeStepSizes + min over the horizon (direct_multiple_shooting.cpp:174-209): steps[b] = {primal, dual} */
void orc_expand_batch(const rbt_stage_dims* sd, const rbt_constraint_table* tab, const rbt_stage_ctrl* ctrl, int n_grid,
                      int batch, const double* lin, const double* ex, const double* d, double* con, double* xd,
                      double* steps, int nthreads) {
  rbt_stage_layout S;
  rbt_make_stage_layout(sd, &S);
  rbt_dims kd = {sd->nv, sd->nu, sd->ns_max, sd->n_passive};
  rbt_layout K;
  rbt_make_layout(&kd, &K);
#ifdef _OPENMP
  if (nthreads > 0) omp_set_num_threads(nthreads);
#endif
#pragma omp parallel for schedule(dynamic)
  for (int b = 0; b < batch; ++b) {
    double mp = 1.0, md = 1.0;
    for (int i = 0; i < n_grid; ++i) {
      const size_t o = (size_t)b * n_grid + i;
      double st[2];
      orc_stage_expand_primal(sd, tab, &ctrl[i], lin + o * S.l_stride, ex + o * S.e_stride, d + o * K.d_stride,
                              con + o * S.c_stride, xd + o * S.x_stride, st);
      if (st[0] < mp) mp = st[0];
      if (st[1] < md) md = st[1];
    }
    steps[2 * b] = mp;
    steps[2 * b + 1] = md;
  }
}

void orc_update_batch(const rbt_stage_dims* sd, const rbt_constraint_table* tab, const rbt_stage_ctrl* ctrl, int n_grid,
                      int batch, double* ex, double* d, double* xd, double* con, double* sol, const double* steps,
                      int nthreads) {
  rbt_stage_layout S;
  rbt_make_stage_layout(sd, &S);
  rbt_dims kd = {sd->nv, sd->nu, sd->ns_max, sd->n_passive};
  rbt_layout K;
  rbt_make_layout(&kd, &K);
#ifdef _OPENMP
  if (nthreads > 0) omp_set_num_threads(nthreads);
#endif
#pragma omp parallel for schedule(dynamic)
  for (int b = 0; b < batch; ++b) {
    /* stage i reads dgmm of stage i+1 BEFORE the costate correction touches dlmd (only dlmd's head changes, dgmm never) */
    for (int i = 0; i < n_grid; ++i) {
      const size_t o = (size_t)b * n_grid + i;
      const double* dn = (i + 1 < n_grid) ? d + (o + 1) * K.d_stride : NULL;
      orc_stage_expand_dual_update(sd, tab, &ctrl[i], ex + o * S.e_stride, d + o * K.d_stride, dn, xd + o * S.x_stride,
                                   con + o * S.c_stride, sol + o * S.s_stride, steps[2 * b], steps[2 * b + 1]);
    }
  }
}

int orc_stage_layout_get(const rbt_stage_dims* sd, const char* field) {
  rbt_stage_layout S;
  rbt_make_stage_layout(sd, &S);
  return rbt_stage_layout_field(&S, field);
}

/* exposed for the identity tests */
int orc_mjtjinv(int nv, int nf, const double* M, const double* J, int ldj, double* Z, int ldz) {
  double* ws = (double*)calloc((size_t)3 * nv * nv + 2 * (nf + 1) * nv + 2 * (nf + 1) * (nf + 1) + 16, 8);
  int info = mjtjinv(nv, nf, M, J, ldj, Z, ldz, ws);
  free(ws);
  return info;
}

/* ---------------- whole hot-path iteration drivers (CPU baseline of bench.py; BASELINE.md section 3) ----------------
 * The linear-algebra body of OCPSolver::updateSolution (src/solver/ocp_solver.cpp:118-144) for a batch of OCPs:
 *   mode 0  "batch-parallel" (best-case CPU): OpenMP over OCP instances, each thread runs condense -> backward -> forward ->
 *           step sizes -> update for its OCP back to back (records stay in its cache), `nthreads` threads;
 *   mode 1  "reference-faithful": one OCP after the other; the stage loops are `omp parallel for num_threads(nthreads)` like
 *           DirectMultipleShooting (src/ocp/direct_multiple_shooting.cpp:135-154, 184-199, 218-241; the examples use
 *           nthreads = 4) and the Riccati recursion is serial (src/riccati/riccati_recursion.cpp:39,94).
 * Returns the OR of the Cholesky flags. */
int orc_riccati_backward(const rbt_dims* dims, const rbt_stage_ctrl* ctrl, int n_grid, double max_dts0, double* kkt, double* ric);
void orc_riccati_forward(const rbt_dims* dims, const rbt_stage_ctrl* ctrl, int n_grid, const double* kkt, const double* ric, double* d);

int orc_iteration_batch(const rbt_stage_dims* sd, const rbt_constraint_table* tab, const rbt_stage_ctrl* ctrl, int n_grid,
                        int batch, double max_dts0, const double* lin, double* con, double* kkt, double* ex, double* ric,
                        const double* dx0, double* d, double* xd, double* sol, double* steps, int mode, int nthreads) {
  rbt_stage_layout S;
  rbt_make_stage_layout(sd, &S);
  rbt_dims kd = {sd->nv, sd->nu, sd->ns_max, sd->n_passive};
  rbt_layout K;
  rbt_make_layout(&kd, &K);
  int info = 0;
  if (nthreads < 1) nthreads = 1;
  if (mode == 0) {
#pragma omp parallel for schedule(dynamic) reduction(| : info) num_threads(nthreads)
    for (int b = 0; b < batch; ++b) {
      const size_t o0 = (size_t)b * n_grid;
      for (int i = 0; i < n_grid; ++i)
        info |= orc_stage_condense(sd, tab, &ctrl[i], lin + (o0 + i) * S.l_stride, con + (o0 + i) * S.c_stride,
                                   kkt + (o0 + i) * K.k_stride, ex + (o0 + i) * S.e_stride);
      info |= orc_riccati_backward(&kd, ctrl, n_grid, max_dts0, kkt + o0 * K.k_stride, ric + o0 * K.r_stride);
      memcpy(d + o0 * K.d_stride + K.d_dx, dx0 + (size_t)b * K.nx, sizeof(double) * K.nx);
      orc_riccati_forward(&kd, ctrl, n_grid, kkt + o0 * K.k_stride, ric + o0 * K.r_stride, d + o0 * K.d_stride);
      double mp = 1.0, md = 1.0;
      for (int i = 0; i < n_grid; ++i) {
        double st[2];
        orc_stage_expand_primal(sd, tab, &ctrl[i], lin + (o0 + i) * S.l_stride, ex + (o0 + i) * S.e_stride,
                                d + (o0 + i) * K.d_stride, con + (o0 + i) * S.c_stride, xd + (o0 + i) * S.x_stride, st);
        if (st[0] < mp) mp = st[0];
        if (st[1] < md) md = st[1];
      }
      steps[2 * b] = mp;
      steps[2 * b + 1] = md;
      for (int i = 0; i < n_grid; ++i) {
        const double* dn = (i + 1 < n_grid) ? d + (o0 + i + 1) * K.d_stride : NULL;
        orc_stage_expand_dual_update(sd, tab, &ctrl[i], ex + (o0 + i) * S.e_stride, d + (o0 + i) * K.d_stride, dn,
                                     xd + (o0 + i) * S.x_stride, con + (o0 + i) * S.c_stride, sol + (o0 + i) * S.s_stride, mp, md);
      }
    }
    return info;
  }
  for (int b = 0; b < batch; ++b) {
    const size_t o0 = (size_t)b * n_grid;
#pragma omp parallel for reduction(| : info) num_threads(nthreads)
    for (int i = 0; i < n_grid; ++i)
      info |= orc_stage_condense(sd, tab, &ctrl[i], lin + (o0 + i) * S.l_stride, con + (o0 + i) * S.c_stride,
                                 kkt + (o0 + i) * K.k_stride, ex + (o0 + i) * S.e_stride);
    info |= orc_riccati_backward(&kd, ctrl, n_grid, max_dts0, kkt + o0 * K.k_stride, ric + o0 * K.r_stride);
    memcpy(d + o0 * K.d_stride + K.d_dx, dx0 + (size_t)b * K.nx, sizeof(double) * K.nx);
    orc_riccati_forward(&kd, ctrl, n_grid, kkt + o0 * K.k_stride, ric + o0 * K.r_stride, d + o0 * K.d_stride);
    double mp = 1.0, md = 1.0;
#pragma omp parallel for reduction(min : mp, md) num_threads(nthreads)
    for (int i = 0; i < n_grid; ++i) {
      double st[2];
      orc_stage_expand_primal(sd, tab, &ctrl[i], lin + (o0 + i) * S.l_stride, ex + (o0 + i) * S.e_stride,
                              d + (o0 + i) * K.d_stride, con + (o0 + i) * S.c_stride, xd + (o0 + i) * S.x_stride, st);
      if (st[0] < mp) mp = st[0];
      if (st[1] < md) md = st[1];
    }
    steps[2 * b] = mp;
    steps[2 * b + 1] = md;
    /* as in the reference's own stage-parallel integrateSolution: stage i reads dgmm of stage i+1, which the costate
     * correction of stage i+1 never writes (it only rewrites the head of dlmd) */
#pragma omp parallel for num_threads(nthreads)
    for (int i = 0; i < n_grid; ++i) {
      const double* dn = (i + 1 < n_grid) ? d + (o0 + i + 1) * K.d_stride : NULL;
      orc_stage_expand_dual_update(sd, tab, &ctrl[i], ex + (o0 + i) * S.e_stride, d + (o0 + i) * K.d_stride, dn,
                                   xd + (o0 + i) * S.x_stride, con + (o0 + i) * S.c_stride, sol + (o0 + i) * S.s_stride, mp, md);
    }
  }
  return info;
}

/* ---------------- rows a12 / a13 / a16 of SURVEY.md 8a: what a device-resident SQP loop needs to terminate on its own ----------
 * Stage part of the PerformanceIndex (include/robotoc/core/performance_index.hpp) as {Intermediate,Impact,Terminal}Stage::evalKKT
 * summarise it BEFORE condensing (intermediate_stage.cpp:128-132, impact_stage.cpp:109-113, terminal_stage.cpp:97-100):
 *   kkt_error          = SplitKKTResidual::KKTError() (split_kkt_residual.hxx:90-104: |Fx|^2 + |P|^2 + |lx|^2 + |lu|^2 + |la|^2 +
 *                        |ldv|^2 + |lf|^2) + ContactDynamicsData::KKTError() (|IDC|^2 + |lu_passive|^2, contact_dynamics_data.hpp:204)
 *                        + sum over constraint components of |residual|^2 + |cmpl|^2 (constraint_component_data.hpp:122)
 *   primal_feasibility = |Fx|_1 + |P|_1 + |IDC|_1 + |residual|_1          (the <1> instantiations)
 *   dual_feasibility   = |lx|_1 + |la|_1 + |ldv|_1 + |lf|_1 + |lu|_1 + |lu_passive|_1 + |cmpl|_1
 *   cost_barrier       = - barrier * sum log(slack)                        (pdipm.hxx:194-200; active rows only, friction_cone.cpp:122-139)
 * out = {cost_barrier, primal_feasibility, dual_feasibility, kkt_error}.  The stage cost itself comes from the (out-of-scope)
 * cost evaluation.  cmpl = slack * dual - barrier (pdipm.hxx:27-63) is recomputed here, so the call does not depend on the
 * condensing having run. */
void orc_stage_perf_index(const rbt_stage_dims* sd, const rbt_constraint_table* tab, const rbt_stage_ctrl* c, const double* lin,
                          const double* con, double* out) {
  rbt_stage_layout S;
  rbt_make_stage_layout(sd, &S);
  const int nv = S.nv, nu = S.nu, nx = S.nx, np = S.np, nf = c->nf;
  double kkt = 0.0, pf = 0.0, df = 0.0, lb = 0.0;
#define ORC_ACC_P(ptr, n) for (int q_ = 0; q_ < (n); ++q_) { const double v_ = (ptr)[q_]; kkt += v_ * v_; pf += fabs(v_); }
#define ORC_ACC_D(ptr, n) for (int q_ = 0; q_ < (n); ++q_) { const double v_ = (ptr)[q_]; kkt += v_ * v_; df += fabs(v_); }
  ORC_ACC_D(lin + S.l_lx, nx)
  if (c->type != RBT_TERMINAL) {
    const int impact = c->type == RBT_IMPACT;
    ORC_ACC_P(lin + S.l_Fx, nx)
    ORC_ACC_D(lin + S.l_la, nv)           /* la on a control stage, ldv on an impact stage (same slot of the record) */
    ORC_ACC_D(lin + S.l_lf, nf)
    ORC_ACC_P(lin + S.l_IDC, nv + nf)
    if (!impact) {
      ORC_ACC_D(lin + S.l_lu, nu)
      ORC_ACC_D(lin + S.l_lup, np)
      ORC_ACC_P(lin + S.l_p, c->ns)
    }
    if (!impact || tab->impact_friction_cone) {
      for (int r = 0; r < S.nc; ++r) {
        const int cone = r >= S.nbox;
        if (cone && !((c->contact_mask >> ((r - S.nbox) / 5)) & 1)) continue;  /* inactive contact: residual = cmpl = 0 */
        if (!cone && !box_row_on(tab, c, r)) continue;                         /* level not valid on this grid point */
        const double sl = con[S.c_slack + r], du = con[S.c_dual + r], res = con[S.c_res + r];
        const double cm = sl * du - tab->barrier;
        kkt += res * res + cm * cm;
        pf += fabs(res);
        df += fabs(cm);
        lb -= tab->barrier * log(sl);
      }
    }
  }
#undef ORC_ACC_P
#undef ORC_ACC_D
  out[0] = lb; out[1] = pf; out[2] = df; out[3] = kkt;
}

/* DirectMultipleShooting::evalKKT's sum over the horizon (direct_multiple_shooting.cpp:155-158), stage order 0..N, and
 * OCPSolver::KKTError() = sqrt(kkt_error) (ocp_solver.cpp:429-431; no STO part here).
 * perf[b] = {cost (0: not evaluated on this path), cost_barrier, primal_feasibility, dual_feasibility, kkt_error, sqrt(kkt_error), 0, 0} */
void orc_perf_index_batch(const rbt_stage_dims* sd, const rbt_constraint_table* tab, const rbt_stage_ctrl* ctrl, int n_grid,
                          int batch, const double* lin, const double* con, double* perf) {
  rbt_stage_layout S;
  rbt_make_stage_layout(sd, &S);
  for (int b = 0; b < batch; ++b) {
    double acc[4] = {0, 0, 0, 0};
    for (int i = 0; i < n_grid; ++i) {
      const size_t o = (size_t)b * n_grid + i;
      double st[4];
      orc_stage_perf_index(sd, tab, &ctrl[i], lin + o * S.l_stride, con + o * S.c_stride, st);
      for (int q = 0; q < 4; ++q) acc[q] += st[q];
    }
    double* p = perf + (size_t)b * 8;
    p[0] = 0.0; p[1] = acc[0]; p[2] = acc[1]; p[3] = acc[2]; p[4] = acc[3]; p[5] = sqrt(acc[3]); p[6] = 0.0; p[7] = 0.0;
  }
}

/* pdipm::setSlackAndDualPositive (pdipm.hxx:13-24) on every inequality row of every constrained stage:
 * slack <- max(slack, sqrt(barrier)), dual <- barrier / slack. */
void orc_set_slack_dual_positive_batch(const rbt_stage_dims* sd, const rbt_constraint_table* tab, const rbt_stage_ctrl* ctrl,
                                       int n_grid, int batch, double* con) {
  rbt_stage_layout S;
  rbt_make_stage_layout(sd, &S);
  const double sb = sqrt(tab->barrier);
  for (int b = 0; b < batch; ++b)
    for (int i = 0; i < n_grid; ++i) {
      if (ctrl[i].type == RBT_TERMINAL || (ctrl[i].type == RBT_IMPACT && !tab->impact_friction_cone)) continue;
      double* cc = con + ((size_t)b * n_grid + i) * S.c_stride;
      for (int r = 0; r < S.nc; ++r) {
        if (r < S.nbox && !box_row_on(tab, &ctrl[i], r)) continue;
        if (cc[S.c_slack + r] < sb) cc[S.c_slack + r] = sb;
        cc[S.c_dual + r] = tab->barrier / cc[S.c_slack + r];
      }
    }
}

/* computeInitialStateDirection (src/dynamics/state_equation.cpp:98-109) given dq_raw = q0 (-) s0.q from the robot model
 * (Robot::subtractConfiguration is Pinocchio's, out of scope): dq[0:6] = -Fqq_prev_inv dq_raw[0:6] for a floating base,
 * dv = v0 - s0.v.  ex0 / sol0 = expansion / solution record of stage 0 of this OCP; dx0 has nx entries. */
void orc_initial_state_direction(const rbt_stage_dims* sd, const double* ex0, const double* sol0, const double* dq_raw,
                                 const double* v0, double* dx0) {
  rbt_stage_layout S;
  rbt_make_stage_layout(sd, &S);
  const int nv = S.nv;
  for (int i = 0; i < nv; ++i) dx0[i] = dq_raw[i];
  if (S.np == 6)
    for (int i = 0; i < 6; ++i) {
      double a = 0.0;
      for (int l = 0; l < 6; ++l) a += ex0[S.e_Fqqpi + IDX(i, l, 6)] * dq_raw[l];
      dx0[i] = -a;
    }
  for (int i = 0; i < nv; ++i) dx0[nv + i] = v0[i] - sol0[S.s_v + i];
}

/* ---------------- SURVEY.md 8f-3: the model-free half of the line search, batched over trial step sizes --------------------
 * LineSearch::lineSearchFilterMethod (src/line_search/line_search.cpp:58-86) tries alpha_k = alpha_max * rate^k (rate 0.75,
 * line_search_settings.hpp) one after the other: integratePrimalSolution (direct_multiple_shooting.cpp:244-266 ->
 * SplitSolution::integrate + Constraints::updateSlack), evalOCP, filter test.  The trial solutions of ALL k are independent of
 * each other, so they form an extra batch axis; evalOCP needs the robot model (out of scope) except for the log-barrier of the
 * trial slacks, which is computed here.
 * Trial record (t_stride = 80 doubles): {q (nq, padded to 20) | v (18) | a or dv (18) | u (12) | f (12)} -- the primal variables
 * evalOCP reads.  out_barrier = - barrier * sum log(slack + alpha dslack) over the active inequality rows of the stage. */
#define ORC_T_Q 0
#define ORC_T_V 20
#define ORC_T_A 38
#define ORC_T_U 56
#define ORC_T_F 68
#define ORC_T_STRIDE 80
void orc_stage_trial(const rbt_stage_dims* sd, const rbt_constraint_table* tab, const rbt_stage_ctrl* c, const double* sol,
                     const double* d, const double* xd, const double* con, double alpha, double* trial, double* out_barrier) {
  rbt_stage_layout S;
  rbt_make_stage_layout(sd, &S);
  rbt_dims kd = {sd->nv, sd->nu, sd->ns_max, sd->n_passive};
  rbt_layout K;
  rbt_make_layout(&kd, &K);
  const int nv = S.nv, nu = S.nu, np = S.np;
  const int terminal = c->type == RBT_TERMINAL, impact = c->type == RBT_IMPACT;
  const double* dx = d + K.d_dx;
  memset(trial, 0, sizeof(double) * ORC_T_STRIDE);
  double* q = trial + ORC_T_Q;
  memcpy(q, sol + S.s_q, sizeof(double) * S.nq);
  if (np == 6) {
    integrate_free_flyer(q, dx, alpha);
    for (int i = 6; i < nv; ++i) q[i + 1] += alpha * dx[i];
  } else {
    for (int i = 0; i < nv; ++i) q[i] += alpha * dx[i];
  }
  for (int i = 0; i < nv; ++i) trial[ORC_T_V + i] = sol[S.s_v + i] + alpha * dx[nv + i];
  *out_barrier = 0.0;
  if (terminal) return;
  const double* daf = xd + S.x_daf;
  for (int i = 0; i < nv; ++i) trial[ORC_T_A + i] = (impact ? sol[S.s_dv + i] : sol[S.s_a + i]) + alpha * daf[i];
  if (!impact)
    for (int i = 0; i < nu; ++i) trial[ORC_T_U + i] = sol[S.s_u + i] + alpha * d[K.d_du + i];
  for (int i = 0; i < c->nf; ++i) trial[ORC_T_F + i] = sol[S.s_f + i] + alpha * daf[nv + i];
  if (!impact || tab->impact_friction_cone) {
    double lb = 0.0;
    for (int r = 0; r < S.nc; ++r) {
      if (r >= S.nbox && !((c->contact_mask >> ((r - S.nbox) / 5)) & 1)) continue;
      if (r < S.nbox && !box_row_on(tab, c, r)) continue;
      lb -= tab->barrier * log(con[S.c_slack + r] + alpha * con[S.c_dslack + r]);
    }
    *out_barrier = lb;
  }
}

/* alphas[k][b] = steps[b].primal * rate^k;  trial[k][b][i][80];  barrier[k][b] = sum over the horizon (stage order) */
void orc_trial_batch(const rbt_stage_dims* sd, const rbt_constraint_table* tab, const rbt_stage_ctrl* ctrl, int n_grid, int batch,
                     int n_trials, double rate, const double* sol, const double* d, const double* xd, const double* con,
                     const double* steps, double* alphas, double* trial, double* barrier) {
  rbt_stage_layout S;
  rbt_make_stage_layout(sd, &S);
  rbt_dims kd = {sd->nv, sd->nu, sd->ns_max, sd->n_passive};
  rbt_layout K;
  rbt_make_layout(&kd, &K);
  for (int k = 0; k < n_trials; ++k)
    for (int b = 0; b < batch; ++b) {
      double a = steps[2 * b];
      for (int q = 0; q < k; ++q) a *= rate;
      alphas[(size_t)k * batch + b] = a;
      double acc = 0.0;
      for (int i = 0; i < n_grid; ++i) {
        const size_t o = (size_t)b * n_grid + i;
        double lb;
        orc_stage_trial(sd, tab, &ctrl[i], sol + o * S.s_stride, d + o * K.d_stride, xd + o * S.x_stride, con + o * S.c_stride, a,
                        trial + (((size_t)k * batch + b) * n_grid + i) * ORC_T_STRIDE, &lb);
        acc += lb;
      }
      barrier[(size_t)k * batch + b] = acc;
    }
}

/* LineSearchFilter (src/line_search/line_search_filter.cpp:25-56) with a fixed-capacity store: filt[2*cap] pairs, *n entries. */
static int filter_accepted(const double* filt, int n, double cr, double vr, double cost, double viol) {
  if (n == 0) return 1;
  for (int e = 0; e < n; ++e)
    if (cost < filt[2 * e] - cr * filt[2 * e + 1] || viol < (1.0 - vr) * filt[2 * e + 1]) return 1;
  return 0;
}
static void filter_augment(double* filt, int* n, int cap, double cr, double vr, double cost, double viol) {
  if (!filter_accepted(filt, *n, cr, vr, cost, viol)) return;
  int w = 0;
  for (int e = 0; e < *n; ++e)
    if (!(filt[2 * e] <= cost && filt[2 * e + 1] <= viol)) { filt[2 * w] = filt[2 * e]; filt[2 * w + 1] = filt[2 * e + 1]; ++w; }
  if (w < cap) { filt[2 * w] = cost; filt[2 * w + 1] = viol; ++w; }
  *n = w;
}
/* lineSearchFilterMethod (line_search.cpp:58-86) for every OCP, given cost[k][b] (stage costs summed by the evaluator; the barrier
 * part barrier[k][b] is added here) and violation[k][b] of the trials and cost0/viol0 of the current iterate:
 *   if the filter is empty: augment(cost0, viol0);   alpha = alpha_max;
 *   while (alpha > min_step): [trial k] if accepted -> augment, return alpha;  alpha *= rate;     return alpha
 * filt: [batch][2*cap], nfilt: [batch].  out_step[b], out_k[b] (-1: none accepted). */
void orc_line_search_filter(int batch, int n_trials, double rate, double min_step, double cr, double vr, int cap,
                            const double* steps, const double* cost0, const double* viol0, const double* cost,
                            const double* barrier, const double* viol, double* filt, int* nfilt, double* out_step, int* out_k) {
  for (int b = 0; b < batch; ++b) {
    double* f = filt + (size_t)b * 2 * cap;
    if (nfilt[b] == 0) filter_augment(f, &nfilt[b], cap, cr, vr, cost0[b], viol0[b]);
    double alpha = steps[2 * b];
    int k = 0, acc = -1;
    while (alpha > min_step && k < n_trials) {
      const double c = cost[(size_t)k * batch + b] + barrier[(size_t)k * batch + b], v = viol[(size_t)k * batch + b];
      if (filter_accepted(f, nfilt[b], cr, vr, c, v)) {
        filter_augment(f, &nfilt[b], cap, cr, vr, c, v);
        acc = k;
        break;
      }
      alpha *= rate;
      ++k;
    }
    out_step[b] = alpha;
    out_k[b] = acc;
  }
}


/* ---------------- SURVEY.md 8f-2 (first slice): Constraints::linearizeConstraints for the joint-limit components
 * (constraints.cpp:283-306 -> joint_{position,velocity,torques}_{lower,upper}_limit.cpp:47-63):
 *   evalConstraint:    residual = sign * (x - bound) + slack        (lower: qmin - q + slack, upper: q - qmax + slack)
 *   evalDerivatives:   l_x += sign * dual                          (lower: lq.tail -= dual, upper: lq.tail += dual)
 * for every box row whose level is valid on the grid point; x = s.q (joint part), s.v, s.a or s.u of the solution record.
 * bound[r] = the limit of row r (from the robot model).  The friction cones need frame kinematics and stay with the host. */
void orc_linearize_joint_limits_batch(const rbt_stage_dims* sd, const rbt_constraint_table* tab, const rbt_stage_ctrl* ctrl,
                                      int n_grid, int batch, const double* bound, const double* sol, double* lin, double* con) {
  rbt_stage_layout S;
  rbt_make_stage_layout(sd, &S);
  const int nv = S.nv;
  for (int b = 0; b < batch; ++b)
    for (int i = 0; i < n_grid; ++i) {
      const rbt_stage_ctrl* c = &ctrl[i];
      if (c->type == RBT_TERMINAL || c->type == RBT_IMPACT) continue;
      const size_t o = (size_t)b * n_grid + i;
      const double* s = sol + o * S.s_stride;
      double* l = lin + o * S.l_stride;
      double* cc = con + o * S.c_stride;
      for (int r = 0; r < tab->n_box; ++r) {
        if (!box_row_on(tab, c, r)) continue;
        const rbt_box_row* br = &tab->box[r];
        double x, *g;
        switch (br->var) {
          case RBT_VAR_Q: x = s[S.s_q + br->idx + (S.np == 6 ? 1 : 0)]; g = l + S.l_lx + br->idx; break;  /* q has one more entry (quaternion) */
          case RBT_VAR_V: x = s[S.s_v + br->idx]; g = l + S.l_lx + nv + br->idx; break;
          case RBT_VAR_A: x = s[S.s_a + br->idx]; g = l + S.l_la + br->idx; break;
          default: x = s[S.s_u + br->idx]; g = l + S.l_lu + br->idx; break;
        }
        cc[S.c_res + r] = br->sign * (x - bound[r]) + cc[S.c_slack + r];
        *g += br->sign * cc[S.c_dual + r];
      }
    }
}
