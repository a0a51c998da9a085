/*
 * riccati_oracle.c -- TEST INFRASTRUCTURE ONLY (parity oracle / CPU baseline).
 *
 * Plain-C, single-threaded-per-OCP restatement of the reference's Riccati recursion
 * (robotoc @ d30d404).  Nothing in the product path (robotoc_b200/, include/) may
 * call into this file; only tests/, __graft_entry__.smoke() and bench.py's CPU legs do.
 *
 * PARITY STATUS: PINNED against the reference's own code.  robotoc/src/riccati/ (all .cpp files) and src/core/split_{kkt_matrix,kkt_residual,direction}.cpp are
 * compiled UNMODIFIED (oracle/Makefile.ref) against a self-written stand-in for the Eigen3 / Robot API (oracle/shim/) into
 * oracle/_ref/libref_riccati.so; tests/test_golden_ref.py compares this file with that library on every field of every
 * Riccati / direction record and of the mutated KKT blocks (event schedules with and without switching-time optimisation,
 * BASELINE trot N=40 and jump STO N=80, iiwa14): agreement 1e-15 .. 3e-15.  tests/golden/golden_ref_r2.npz holds outputs of
 * that library (tests/golden/make_golden_ref.py), so the pin also holds where no robotoc tree is available.
 * Besides: the reference tests' algebraic identities re-run with fixed seeds and an independent dense solve of the full block
 * KKT system in numpy (tests/test_oracle_kkt.py; for the STO path with the switching-time increments as unknowns: exact up to
 * the three places where the reference itself departs from the exact Newton step, all restated here and documented at
 * orc_debug_exact_*).
 *
 * Each function cites the reference file:line it restates.  The order of the floating
 * point operations follows the reference's expression order (Eigen evaluates each
 * `noalias() =` as a plain inner-product GEMM; we use the k-inner triple loop).
 * All matrices are column-major; records are laid out by include/rbt_layout.h.
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <float.h>
#include "../include/rbt_layout.h"

#define IDX(i, j, ld) ((i) + (size_t)(j) * (ld))

int orc_debug_exact_chi = 0; /* see the switching-constraint STO terms below; never set outside the tests */
int orc_debug_exact_transition = 0; /* phase transition with the rank-one term of P (tests only), see phase_transition() */
int orc_debug_exact_impact_costate = 0; /* costate at an impact grid with -Phi * (this event's dts) (tests only) */

#include "orc_linalg.h"  /* gemm(): register-blocked small GEMM shared by the oracle sources */

static double dot(int n, const double* a, const double* b) {
  double s = 0.0;
  for (int i = 0; i < n; ++i) s += a[i] * b[i];
  return s;
}

/* Lower Cholesky A = L L^T in place (what Eigen::LLT<MatrixXd> computes; riccati_factorizer.hpp:152).
 * Returns 0 on success, 1 if a non-positive pivot is met (Eigen::NumericalIssue). */
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

/* B <- (L L^T)^{-1} B, B is n x nrhs (Eigen LLT::solve). */
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

typedef struct {
  double *AtP, *BtP, *GK, *K, *Ginv, *DGinv, *S, *SinvDGinv, *DtM, *KtDtM, *Pf, *Lg, *tmp, *m_rec;
} orc_ws;

static orc_ws* ws_new(const rbt_layout* L) {
  const int nx = L->nx, nu = L->nu, ns = L->ns_max > 0 ? L->ns_max : 1;
  orc_ws* w = (orc_ws*)calloc(1, sizeof(orc_ws));
  w->AtP = (double*)calloc((size_t)nx * nx, 8);
  w->BtP = (double*)calloc((size_t)nu * nx, 8);
  w->GK = (double*)calloc((size_t)nu * nx, 8);
  w->K = (double*)calloc((size_t)nu * nx, 8);
  w->Ginv = (double*)calloc((size_t)nu * nu, 8);
  w->DGinv = (double*)calloc((size_t)ns * nu, 8);
  w->S = (double*)calloc((size_t)ns * ns, 8);
  w->SinvDGinv = (double*)calloc((size_t)ns * nu, 8);
  w->DtM = (double*)calloc((size_t)nu * nx, 8);
  w->KtDtM = (double*)calloc((size_t)nx * nx, 8);
  w->Pf = (double*)calloc((size_t)nx, 8);
  w->Lg = (double*)calloc((size_t)nu * nu, 8);
  w->tmp = (double*)calloc((size_t)(nx > nu ? nx : nu) * (ns > nu ? ns : nu) + nx * nx, 8);
  w->m_rec = (double*)calloc((size_t)L->r_stride, 8);
  return w;
}

static void ws_free(orc_ws* w) {
  free(w->AtP); free(w->BtP); free(w->GK); free(w->K); free(w->Ginv); free(w->DGinv); free(w->S);
  free(w->SinvDGinv); free(w->DtM); free(w->KtDtM); free(w->Pf); free(w->Lg); free(w->tmp); free(w->m_rec);
  free(w);
}

/*
 * Full backward step (Intermediate / Lift stage).
 *   RiccatiFactorizer::backwardRiccatiRecursion              riccati_factorizer.cpp:44-90   (LQR part)
 *   RiccatiFactorizer::backwardRiccatiRecursion (sto flags)  riccati_factorizer.cpp:93-142  (STO part)
 *   BackwardRiccatiRecursionFactorizer::factorizeKKTMatrix   backward_riccati_recursion_factorizer.cpp:31-45
 *   ...::factorizeHamiltonian :48-66, ...::factorizeRiccatiFactorization :78-91, ...::factorizeSTOFactorization :94-143
 * kkt is mutated in place exactly like the reference mutates Qxx,Qxu,Quu,lu.
 * `ric` must be zero-initialised by the caller (a freshly constructed SplitRiccatiFactorization):
 * the reference does not reset Phi,rho,iota when !sto (riccati_factorizer.cpp:99-105).
 * Returns 0, or 1/2 if the Cholesky of G / S fails (reference: assert only).
 */
static int backward_full(const rbt_layout* L, orc_ws* w, int ns, int sto, int sto_next, const double* rn,
                         double* kkt, double* ric) {
  const int nx = L->nx, nu = L->nu, nv = L->nv;
  const double* A = kkt + L->k_Fxx;
  const double* Bv = kkt + L->k_Fvu; /* nv x nu */
  double* F = kkt + L->k_Qxx;
  double* H = kkt + L->k_Qxu;
  double* G = kkt + L->k_Quu;
  const double* Fx = kkt + L->k_Fx;
  const double* lx = kkt + L->k_lx;
  double* lu = kkt + L->k_lu;
  const double* Pn = rn + L->r_P;
  const double* sn = rn + L->r_s;
  double* K = w->K; /* nu x nx col-major */
  double* kvec = ric + L->r_k;
  int info = 0;

  /* factorizeKKTMatrix: backward_riccati_recursion_factorizer.cpp:34-44 */
  gemm(1, 0, nx, nx, nx, 1.0, A, nx, Pn, nx, 0.0, w->AtP, nx);             /* AtP = A^T Pn            :34 */
  gemm(1, 0, nu, nx, nv, 1.0, Bv, nv, Pn + nv, nx, 0.0, w->BtP, nu);       /* BtP = Bv^T Pn[nv:,:]    :35 */
  gemm(0, 0, nx, nx, nx, 1.0, w->AtP, nx, A, nx, 1.0, F, nx);              /* Qxx += AtP A            :37 */
  gemm(0, 0, nx, nu, nv, 1.0, w->AtP + (size_t)nv * nx, nx, Bv, nv, 1.0, H, nx); /* Qxu += AtP[:,nv:] Bv :39 */
  gemm(0, 0, nu, nu, nv, 1.0, w->BtP + (size_t)nv * nu, nu, Bv, nv, 1.0, G, nu); /* Quu += BtP[:,nv:] Bv :41 */
  gemm(0, 0, nu, 1, nx, 1.0, w->BtP, nu, Fx, nx, 1.0, lu, nu);             /* lu += BtP Fx            :43 */
  gemm(1, 0, nu, 1, nv, -1.0, Bv, nv, sn + nv, nv, 1.0, lu, nu);           /* lu -= Bv^T sn[nv:]      :44 */

  /* LLT of G: riccati_factorizer.cpp:49 */
  memcpy(w->Lg, G, sizeof(double) * nu * nu);
  if (chol_lower(nu, w->Lg, nu)) info = 1;

  if (ns == 0) {
    /* K = -G^-1 H^T ; k = -G^-1 lu   :55-56 */
    for (int j = 0; j < nx; ++j)
      for (int i = 0; i < nu; ++i) K[IDX(i, j, nu)] = H[IDX(j, i, nx)];
    chol_solve(nu, w->Lg, nu, nx, K, nu);
    for (int i = 0; i < nu * nx; ++i) K[i] = -K[i];
    memcpy(kvec, lu, sizeof(double) * nu);
    chol_solve(nu, w->Lg, nu, 1, kvec, nu);
    for (int i = 0; i < nu; ++i) kvec[i] = -kvec[i];
  } else {
    /* Schur-complement path :58-77.  D = Phiu (ns x nu), C = Phix (ns x nx), p = residual P() */
    const double* D = kkt + L->k_Phiu;
    const double* C = kkt + L->k_Phix;
    const double* p = kkt + L->k_p;
    double* M = ric + L->r_M; /* ns x nx, ld = ns */
    double* mvec = ric + L->r_m;
    double* Dt = w->tmp; /* nu x ns */
    memset(w->Ginv, 0, sizeof(double) * nu * nu);
    for (int i = 0; i < nu; ++i) w->Ginv[IDX(i, i, nu)] = 1.0;
    chol_solve(nu, w->Lg, nu, nu, w->Ginv, nu);                            /* Ginv = G^-1                :60 */
    for (int j = 0; j < ns; ++j)
      for (int i = 0; i < nu; ++i) Dt[IDX(i, j, nu)] = D[IDX(j, i, ns)];
    chol_solve(nu, w->Lg, nu, ns, Dt, nu);                                 /* DGinv^T = G^-1 D^T         :61 */
    for (int j = 0; j < nu; ++j)
      for (int i = 0; i < ns; ++i) w->DGinv[IDX(i, j, ns)] = Dt[IDX(j, i, nu)];
    gemm(0, 1, ns, ns, nu, 1.0, w->DGinv, ns, D, ns, 0.0, w->S, ns);       /* S = DGinv D^T              :62 */
    if (chol_lower(ns, w->S, ns)) info = 2;                                /* llt_s_                     :63 */
    memcpy(w->SinvDGinv, w->DGinv, sizeof(double) * ns * nu);
    chol_solve(ns, w->S, ns, nu, w->SinvDGinv, ns);                        /* SinvDGinv = S^-1 DGinv     :65 */
    gemm(1, 0, nu, nu, ns, -1.0, w->SinvDGinv, ns, w->DGinv, ns, 1.0, w->Ginv, nu); /* Ginv -= SDG^T DG  :66 */
    gemm(0, 1, nu, nx, nu, -1.0, w->Ginv, nu, H, nx, 0.0, K, nu);          /* K  = -Ginv H^T             :67 */
    gemm(1, 0, nu, nx, ns, -1.0, w->SinvDGinv, ns, C, ns, 1.0, K, nu);     /* K -= SDG^T C               :68 */
    gemm(0, 0, nu, 1, nu, -1.0, w->Ginv, nu, lu, nu, 0.0, kvec, nu);       /* k  = -Ginv lu              :69 */
    gemm(1, 0, nu, 1, ns, -1.0, w->SinvDGinv, ns, p, ns, 1.0, kvec, nu);   /* k -= SDG^T p               :70 */
    memcpy(M, C, sizeof(double) * ns * nx);
    chol_solve(ns, w->S, ns, nx, M, ns);                                   /* M  = S^-1 C                :71 */
    gemm(0, 1, ns, nx, nu, -1.0, w->SinvDGinv, ns, H, nx, 1.0, M, ns);     /* M -= SDG H^T               :72 */
    memcpy(mvec, p, sizeof(double) * ns);
    chol_solve(ns, w->S, ns, 1, mvec, ns);                                 /* m  = S^-1 p                :73 */
    gemm(0, 0, ns, 1, nu, -1.0, w->SinvDGinv, ns, lu, nu, 1.0, mvec, ns);  /* m -= SDG lu                :74 */
  }

  /* factorizeRiccatiFactorization: backward_riccati_recursion_factorizer.cpp:82-90 */
  double* P = ric + L->r_P;
  double* s = ric + L->r_s;
  gemm(0, 0, nu, nx, nu, 1.0, G, nu, K, nu, 0.0, w->GK, nu);               /* GK = G K                   :82 */
  gemm(1, 0, nx, nx, nu, -1.0, K, nu, w->GK, nu, 1.0, F, nx);              /* Qxx -= K^T GK              :83 */
  for (int j = 0; j < nx; ++j)
    for (int i = 0; i < nx; ++i) P[IDX(i, j, nx)] = 0.5 * (F[IDX(i, j, nx)] + F[IDX(j, i, nx)]); /* :85 */
  gemm(1, 0, nx, 1, nx, 1.0, A, nx, sn, nx, 0.0, s, nx);                   /* s  = A^T sn                :87 */
  gemm(0, 0, nx, 1, nx, -1.0, w->AtP, nx, Fx, nx, 1.0, s, nx);             /* s -= AtP Fx                :88 */
  for (int i = 0; i < nx; ++i) s[i] -= lx[i];                              /* s -= lx                    :89 */
  gemm(0, 0, nx, 1, nu, -1.0, H, nx, kvec, nu, 1.0, s, nx);                /* s -= Qxu k                 :90 */

  if (ns > 0) {
    /* riccati_factorizer.cpp:83-89 */
    const double* D = kkt + L->k_Phiu;
    const double* C = kkt + L->k_Phix;
    gemm(1, 0, nu, nx, ns, 1.0, D, ns, ric + L->r_M, ns, 0.0, w->DtM, nu); /* DtM = D^T M                :84 */
    gemm(1, 0, nx, nx, nu, 1.0, K, nu, w->DtM, nu, 0.0, w->KtDtM, nx);     /* KtDtM = K^T DtM            :85 */
    for (int j = 0; j < nx; ++j)
      for (int i = 0; i < nx; ++i) P[IDX(i, j, nx)] -= w->KtDtM[IDX(i, j, nx)];
    for (int j = 0; j < nx; ++j)
      for (int i = 0; i < nx; ++i) P[IDX(i, j, nx)] -= w->KtDtM[IDX(j, i, nx)];
    gemm(1, 0, nx, 1, ns, -1.0, C, ns, ric + L->r_m, ns, 1.0, s, nx);      /* s -= C^T m                 :88 */
  }

  /* store K (record holds the reference's row-major nu x nx K == col-major nx x nu K^T) */
  {
    double* Kt = ric + L->r_K;
    for (int j = 0; j < nx; ++j)
      for (int i = 0; i < nu; ++i) Kt[IDX(j, i, nx)] = K[IDX(i, j, nu)];
  }

  double* sc = ric + L->r_sc; /* xi, chi, rho, eta, iota */
  double* Psi = ric + L->r_Psi;
  double* Phi = ric + L->r_Phi;
  if (!sto) { /* riccati_factorizer.cpp:99-105 */
    memset(Psi, 0, sizeof(double) * nx);
    sc[0] = 0.0; sc[1] = 0.0; sc[3] = 0.0;
    return info;
  }

  /* factorizeHamiltonian: backward_riccati_recursion_factorizer.cpp:48-66 */
  const double* f = kkt + L->k_fx;
  const double* hx = kkt + L->k_hx;
  const double* hu = kkt + L->k_hu;
  const double* ksc = kkt + L->k_sc; /* Qtt, Qtt_prev, h */
  const double* Psin = rn + L->r_Psi;
  const double* Phin = rn + L->r_Phi;
  const double* scn = rn + L->r_sc;
  double* psix = ric + L->r_psix;
  double* psiu = ric + L->r_psiu;
  double* phix = ric + L->r_phix;
  double* phiu = ric + L->r_phiu;
  double* T = ric + L->r_T;
  double* W = ric + L->r_W;
  gemm(0, 0, nx, 1, nx, 1.0, w->AtP, nx, f, nx, 0.0, psix, nx);            /* psi_x = AtP fx   :52 */
  gemm(0, 0, nu, 1, nx, 1.0, w->BtP, nu, f, nx, 0.0, psiu, nu);            /* psi_u = BtP fx   :53 */
  for (int i = 0; i < nx; ++i) psix[i] += hx[i];                           /* :54 */
  for (int i = 0; i < nu; ++i) psiu[i] += hu[i];                           /* :55 */
  gemm(1, 0, nx, 1, nx, 1.0, A, nx, Psin, nx, 1.0, psix, nx);              /* psi_x += A^T Psin :56 */
  gemm(1, 0, nu, 1, nv, 1.0, Bv, nv, Psin + nv, nv, 1.0, psiu, nu);        /* psi_u += Bv^T Psin[nv:] :57 */
  if (sto_next) {
    gemm(1, 0, nx, 1, nx, 1.0, A, nx, Phin, nx, 0.0, phix, nx);            /* :59 */
    gemm(1, 0, nu, 1, nv, 1.0, Bv, nv, Phin + nv, nv, 0.0, phiu, nu);      /* :60 */
  } else {
    memset(phix, 0, sizeof(double) * nx);
    memset(phiu, 0, sizeof(double) * nu);
  }
  /* riccati_factorizer.cpp:109-129 */
  memset(W, 0, sizeof(double) * nu);
  if (ns > 0) {
    const double* ct = kkt + L->k_Phit;
    double* mt = ric + L->r_mt;
    double* mtn = ric + L->r_mtn;
    gemm(0, 0, nu, 1, nu, -1.0, w->Ginv, nu, psiu, nu, 0.0, T, nu);        /* T  = -Ginv psi_u :111 */
    gemm(1, 0, nu, 1, ns, -1.0, w->SinvDGinv, ns, ct, ns, 1.0, T, nu);     /* T -= SDG^T Phit  :112 */
    if (sto_next) gemm(0, 0, nu, 1, nu, -1.0, w->Ginv, nu, phiu, nu, 0.0, W, nu); /* :114 */
    memcpy(mt, ct, sizeof(double) * ns);
    chol_solve(ns, w->S, ns, 1, mt, ns);                                   /* mt = S^-1 Phit   :116 */
    gemm(0, 0, ns, 1, nu, -1.0, w->SinvDGinv, ns, psiu, nu, 1.0, mt, ns);  /* mt -= SDG psi_u  :117 */
    if (sto_next) gemm(0, 0, ns, 1, nu, -1.0, w->SinvDGinv, ns, phiu, nu, 0.0, mtn, ns); /* :119 */
    else memset(mtn, 0, sizeof(double) * ns);
  } else {
    memcpy(T, psiu, sizeof(double) * nu);
    chol_solve(nu, w->Lg, nu, 1, T, nu);
    for (int i = 0; i < nu; ++i) T[i] = -T[i];                             /* T = -G^-1 psi_u  :126 */
    if (sto_next) {
      memcpy(W, phiu, sizeof(double) * nu);
      chol_solve(nu, w->Lg, nu, 1, W, nu);
      for (int i = 0; i < nu; ++i) W[i] = -W[i];                           /* :128 */
    }
  }
  /* factorizeSTOFactorization: backward_riccati_recursion_factorizer.cpp:94-143 */
  memcpy(Psi, psix, sizeof(double) * nx);
  gemm(1, 0, nx, 1, nu, 1.0, K, nu, psiu, nu, 1.0, Psi, nx);               /* Psi = psi_x + K^T psi_u :100-101 */
  if (sto_next) {
    memcpy(Phi, phix, sizeof(double) * nx);
    gemm(1, 0, nx, 1, nu, 1.0, K, nu, phiu, nu, 1.0, Phi, nx);             /* :103-104 */
  } else {
    memset(Phi, 0, sizeof(double) * nx);
  }
  gemm(0, 0, nx, 1, nx, 1.0, Pn, nx, f, nx, 0.0, w->Pf, nx);               /* Pf = Pn fx :110 */
  double xi = dot(nx, f, w->Pf);
  xi += ksc[0];
  xi += 2 * dot(nx, Psin, f);
  xi += dot(nu, T, psiu);
  xi += scn[0];
  double chi = 0.0, rho = 0.0, iota = 0.0;
  if (sto_next) {
    chi = ksc[1];
    chi += dot(nx, Phin, f);
    chi += dot(nu, T, phiu);
    chi += scn[1];
    rho = dot(nu, W, phiu);
    rho += scn[2];
  }
  gemm(0, 0, nx, 1, nx, 1.0, Pn, nx, Fx, nx, 0.0, w->Pf, nx);              /* Pf = Pn Fx - sn :129 */
  for (int i = 0; i < nx; ++i) w->Pf[i] -= sn[i];
  double eta = dot(nx, f, w->Pf);
  eta += ksc[2];
  eta += dot(nx, Psin, Fx);
  eta += dot(nu, psiu, kvec);
  eta += scn[3];
  if (sto_next) {
    iota = dot(nx, Phin, Fx);
    iota += dot(nu, phiu, kvec);
    iota += scn[4];
  }
  if (ns > 0) { /* riccati_factorizer.cpp:136-141 */
    const double* ct = kkt + L->k_Phit;
    gemm(1, 0, nx, 1, ns, 1.0, ric + L->r_M, ns, ct, ns, 1.0, Psi, nx);    /* Psi += M^T Phit */
    xi += dot(ns, ric + L->r_mt, ct);
    /* NB: T already contains -SDG^T Phit, so T.phi_u above already carries Phit^T mt_next; the reference adds it once
     * more here (riccati_factorizer.cpp:139).  Restated as it is; orc_debug_exact_chi = 1 (tests only) leaves it out,
     * which makes the recursion the exact elimination of the KKT system (tests/test_oracle_kkt.py). */
    if (sto_next && !orc_debug_exact_chi) chi += dot(ns, ric + L->r_mtn, ct);
    eta += dot(ns, ric + L->r_m, ct);
  }
  sc[0] = xi; sc[1] = chi; sc[2] = rho; sc[3] = eta; sc[4] = iota;
  return info;
}

/*
 * Impact-stage backward step: riccati_factorizer.cpp:178-197,
 * backward_riccati_recursion_factorizer.cpp:69-75 (factorizeKKTMatrix), :146-157, :160-174 (STO).
 */
static void backward_impact(const rbt_layout* L, orc_ws* w, int sto, const double* rn, double* kkt, double* ric) {
  const int nx = L->nx;
  const double* A = kkt + L->k_Fxx;
  double* F = kkt + L->k_Qxx;
  const double* Fx = kkt + L->k_Fx;
  const double* lx = kkt + L->k_lx;
  const double* Pn = rn + L->r_P;
  const double* sn = rn + L->r_s;
  double* P = ric + L->r_P;
  double* s = ric + L->r_s;
  gemm(1, 0, nx, nx, nx, 1.0, A, nx, Pn, nx, 0.0, w->AtP, nx);
  gemm(0, 0, nx, nx, nx, 1.0, w->AtP, nx, A, nx, 1.0, F, nx);
  for (int j = 0; j < nx; ++j)
    for (int i = 0; i < nx; ++i) P[IDX(i, j, nx)] = 0.5 * (F[IDX(i, j, nx)] + F[IDX(j, i, nx)]);
  gemm(1, 0, nx, 1, nx, 1.0, A, nx, sn, nx, 0.0, s, nx);
  gemm(0, 0, nx, 1, nx, -1.0, w->AtP, nx, Fx, nx, 1.0, s, nx);
  for (int i = 0; i < nx; ++i) s[i] -= lx[i];
  if (sto) {
    double* sc = ric + L->r_sc;
    const double* scn = rn + L->r_sc;
    memset(ric + L->r_Psi, 0, sizeof(double) * nx);
    gemm(1, 0, nx, 1, nx, 1.0, A, nx, rn + L->r_Phi, nx, 0.0, ric + L->r_Phi, nx);
    sc[0] = 0.0; sc[1] = 0.0; sc[2] = scn[2]; sc[3] = 0.0;
    sc[4] = scn[4] + dot(nx, rn + L->r_Phi, Fx);
  }
}

/*
 * Phase transition: riccati_factorizer.cpp:145-175.  `pol` is the record whose STOPolicy
 * section (dtsdx, dtsdts, dts0) receives the policy.
 */
static void phase_transition(const rbt_layout* L, double max_dts0, const double* r, double* m, double* pol,
                             int sto_next) {
  const int nx = L->nx;
  const double eps = sqrt(DBL_EPSILON);
  const double* sc = r + L->r_sc;
  double* msc = m + L->r_sc;
  memcpy(m + L->r_P, r + L->r_P, sizeof(double) * nx * nx);
  memcpy(m + L->r_s, r + L->r_s, sizeof(double) * nx);
  memset(m + L->r_Psi, 0, sizeof(double) * nx);
  memcpy(m + L->r_Phi, r + L->r_Psi, sizeof(double) * nx);
  msc[0] = 0.0; msc[1] = 0.0; msc[2] = sc[0]; msc[3] = 0.0; msc[4] = sc[3];
  if (sto_next) {
    const double xi = sc[0], chi = sc[1], rho = sc[2], eta = sc[3], iota = sc[4];
    double sgm = xi - 2.0 * chi + rho;
    if ((sgm * max_dts0) < fabs(eta - iota) || sgm < eps) sgm = fabs(sgm) + fabs(eta - iota) / max_dts0;
    const double* Psi = r + L->r_Psi;
    const double* Phi = r + L->r_Phi;
    double* dtsdx = pol + L->r_dtsdx;
    for (int i = 0; i < nx; ++i) dtsdx[i] = -(1.0 / sgm) * (Psi[i] - Phi[i]);
    pol[L->r_stosc + 0] = (1.0 / sgm) * (xi - chi);
    pol[L->r_stosc + 1] = -(1.0 / sgm) * (eta - iota);
    for (int i = 0; i < nx; ++i) m[L->r_s + i] += (1.0 / sgm) * (Psi[i] - Phi[i]) * (eta - iota);
    for (int i = 0; i < nx; ++i) m[L->r_Phi + i] -= (1.0 / sgm) * (Psi[i] - Phi[i]) * (xi - chi);
    msc[2] = xi - (1.0 / sgm) * (xi - chi) * (xi - chi);
    msc[4] = eta - (1.0 / sgm) * (xi - chi) * (eta - iota);
    /* NB: minimising over the next switching time also gives P_m = P - (Psi-Phi)(Psi-Phi)^T / sgm; the reference keeps
     * riccati_m.P = riccati.P (:149).  Restated as it is; orc_debug_exact_transition = 1 (tests only) adds the term. */
    if (orc_debug_exact_transition) {
      double* P_m = m + L->r_P;
      for (int j = 0; j < nx; ++j)
        for (int i = 0; i < nx; ++i) P_m[IDX(i, j, nx)] -= (1.0 / sgm) * (Psi[i] - Phi[i]) * (Psi[j] - Phi[j]);
    }
  }
}

/*
 * RiccatiRecursion::backwardRiccatiRecursion  riccati_recursion.cpp:32-80.
 * n_grid = time_discretization.size() = N+1 grid points; kkt/ric are [n_grid][stride] for ONE OCP.
 * ric must be zero-initialised.  kkt is mutated in place.  Returns the OR of Cholesky failures.
 */
int orc_riccati_backward(const rbt_dims* dims, const rbt_stage_ctrl* ctrl, int n_grid, double max_dts0,
                         double* kkt, double* ric) {
  rbt_layout L;
  rbt_make_layout(dims, &L);
  orc_ws* w = ws_new(&L);
  const int N = n_grid - 1;
  const int nx = L.nx;
  int info = 0;
  double* ricN = ric + (size_t)N * L.r_stride;
  const double* kktN = kkt + (size_t)N * L.k_stride;
  memcpy(ricN + L.r_P, kktN + L.k_Qxx, sizeof(double) * nx * nx);           /* :37 */
  for (int i = 0; i < nx; ++i) ricN[L.r_s + i] = -kktN[L.k_lx + i];         /* :38 */
  for (int i = N - 1; i >= 0; --i) {
    const rbt_stage_ctrl* g = &ctrl[i];
    double* kk = kkt + (size_t)i * L.k_stride;
    double* rr = ric + (size_t)i * L.r_stride;
    const double* rn = ric + (size_t)(i + 1) * L.r_stride;
    if (g->type == RBT_IMPACT) {
      if (ctrl[i - 1].sto || g->sto) {                                      /* :42-48 */
        memset(w->m_rec, 0, sizeof(double) * L.r_stride);
        phase_transition(&L, max_dts0, rn, w->m_rec, rr, g->sto_next);
        backward_impact(&L, w, g->sto, w->m_rec, kk, rr);
      } else {
        backward_impact(&L, w, g->sto, rn, kk, rr);
      }
    } else if (ctrl[i + 1].type == RBT_LIFT) {
      if (g->sto || g->sto_next) {                                          /* :56-62 */
        memset(w->m_rec, 0, sizeof(double) * L.r_stride);
        phase_transition(&L, max_dts0, rn, w->m_rec, ric + (size_t)(i + 1) * L.r_stride, g->sto_next);
        info |= backward_full(&L, w, g->ns, g->sto, g->sto_next, w->m_rec, kk, rr);
      } else {
        info |= backward_full(&L, w, g->ns, g->sto, g->sto_next, rn, kk, rr);
      }
    } else {
      info |= backward_full(&L, w, g->ns, g->sto, g->sto_next, rn, kk, rr);
    }
  }
  if (ctrl[0].sto) {                                                        /* :75-79 */
    memset(w->m_rec, 0, sizeof(double) * L.r_stride);
    phase_transition(&L, max_dts0, ric, w->m_rec, ric, ctrl[0].sto_next);
  }
  ws_free(w);
  return info;
}

/* computeSwitchingTimeDirection: riccati_factorizer.cpp:237-243 */
static void switching_time_direction(const rbt_layout* L, const double* pol, double* d, int sto_prev) {
  double v = dot(L->nx, pol + L->r_dtsdx, d + L->d_dx) + pol[L->r_stosc + 1];
  if (sto_prev) v += pol[L->r_stosc + 0] * d[L->d_dts + 0];
  d[L->d_dts + 1] = v;
}

/* computeCostateDirection (4-arg form): riccati_factorizer.cpp:246-256; the 3-arg (impact) form :259-266 */
static void costate_direction(const rbt_layout* L, const double* r, double* d, int sto, int sto_next, int impact_form) {
  const int nx = L->nx;
  double* dl = d + L->d_dlmdgmm;
  gemm(0, 0, nx, 1, nx, 1.0, r + L->r_P, nx, d + L->d_dx, nx, 0.0, dl, nx);
  for (int i = 0; i < nx; ++i) dl[i] -= r[L->r_s + i];
  const double dts = d[L->d_dts], dtsn = d[L->d_dts + 1];
  if (impact_form) {
    /* NB: at the impact grid the forward sweep holds (dts, dts_next) = (this event's increment, 0 or the next event's), and
     * the value function there depends on THIS event's increment through Phi; the reference multiplies Phi by dts_next
     * (:262-264).  Restated as it is; orc_debug_exact_impact_costate = 1 (tests only) uses dts, which makes the costate
     * the multiplier of the KKT system (tests/test_oracle_condense.py, test_oracle_kkt.py). */
    if (sto) for (int i = 0; i < nx; ++i) dl[i] -= r[L->r_Phi + i] * (orc_debug_exact_impact_costate ? dts : dtsn);
  } else if (sto) {
    for (int i = 0; i < nx; ++i) dl[i] += r[L->r_Psi + i] * (dtsn - dts);
    if (sto_next) for (int i = 0; i < nx; ++i) dl[i] -= r[L->r_Phi + i] * dtsn;
  }
}

/* forwardRiccatiRecursion (with LQR policy): riccati_factorizer.cpp:200-221 */
static void forward_full(const rbt_layout* L, const double* kkt, const double* r, double* d, double* dn, int sto,
                         int sto_next) {
  const int nx = L->nx, nu = L->nu, nv = L->nv;
  const double* Kt = r + L->r_K; /* nx x nu col-major = K^T */
  double* du = d + L->d_du;
  const double* dx = d + L->d_dx;
  const double dts = d[L->d_dts], dtsn = d[L->d_dts + 1];
  gemm(1, 0, nu, 1, nx, 1.0, Kt, nx, dx, nx, 0.0, du, nu);
  for (int i = 0; i < nu; ++i) du[i] += r[L->r_k + i];
  if (sto) {
    for (int i = 0; i < nu; ++i) du[i] += r[L->r_T + i] * (dtsn - dts);
    if (sto_next) for (int i = 0; i < nu; ++i) du[i] -= r[L->r_W + i] * dtsn;
  }
  double* dxn = dn + L->d_dx;
  memcpy(dxn, kkt + L->k_Fx, sizeof(double) * nx);
  gemm(0, 0, nx, 1, nx, 1.0, kkt + L->k_Fxx, nx, dx, nx, 1.0, dxn, nx);
  gemm(0, 0, nv, 1, nu, 1.0, kkt + L->k_Fvu, nv, du, nu, 1.0, dxn + nv, nv);
  if (sto) for (int i = 0; i < nx; ++i) dxn[i] += kkt[L->k_fx + i] * (dtsn - dts);
  dn[L->d_dts] = dts;
  dn[L->d_dts + 1] = dtsn;
}

/* forwardRiccatiRecursion (impact): riccati_factorizer.cpp:224-232 */
static void forward_impact(const rbt_layout* L, const double* kkt, const double* d, double* dn) {
  const int nx = L->nx;
  double* dxn = dn + L->d_dx;
  memcpy(dxn, kkt + L->k_Fx, sizeof(double) * nx);
  gemm(0, 0, nx, 1, nx, 1.0, kkt + L->k_Fxx, nx, d + L->d_dx, nx, 1.0, dxn, nx);
  dn[L->d_dts] = d[L->d_dts];
  dn[L->d_dts + 1] = d[L->d_dts + 1];
}

/* computeLagrangeMultiplierDirection: riccati_factorizer.cpp:269-281 */
static void multiplier_direction(const rbt_layout* L, int ns, const double* r, double* d, int sto, int sto_next) {
  double* dxi = d + L->d_dxi;
  gemm(0, 0, ns, 1, L->nx, 1.0, r + L->r_M, ns, d + L->d_dx, L->nx, 0.0, dxi, ns);
  for (int i = 0; i < ns; ++i) dxi[i] += r[L->r_m + i];
  if (sto) {
    const double dts = d[L->d_dts], dtsn = d[L->d_dts + 1];
    for (int i = 0; i < ns; ++i) dxi[i] += r[L->r_mt + i] * (dtsn - dts);
    if (sto_next) for (int i = 0; i < ns; ++i) dxi[i] -= r[L->r_mtn + i] * dtsn;
  }
}

/*
 * RiccatiRecursion::forwardRiccatiRecursion  riccati_recursion.cpp:83-131.
 * kkt here is the UNMUTATED-or-mutated record (only Fxx,Fvu,Fx,fx are read).  d[0].dx must hold dx0.
 */
void orc_riccati_forward(const rbt_dims* dims, const rbt_stage_ctrl* ctrl, int n_grid, const double* kkt,
                         const double* ric, double* d) {
  rbt_layout L;
  rbt_make_layout(dims, &L);
  const int N = n_grid - 1;
  d[L.d_dts] = 0.0;
  d[L.d_dts + 1] = 0.0;
  if (ctrl[0].sto) switching_time_direction(&L, ric, d, 0);                 /* :90-93 */
  for (int i = 0; i < N; ++i) {
    const rbt_stage_ctrl* g = &ctrl[i];
    const double* kk = kkt + (size_t)i * L.k_stride;
    const double* rr = ric + (size_t)i * L.r_stride;
    double* di = d + (size_t)i * L.d_stride;
    double* dn = d + (size_t)(i + 1) * L.d_stride;
    if (g->type == RBT_IMPACT) {                                            /* :96-108 */
      const double* dp = d + (size_t)(i - 1) * L.d_stride;
      di[L.d_dts] = dp[L.d_dts + 1];
      di[L.d_dts + 1] = 0.0;
      forward_impact(&L, kk, di, dn);
      if (g->sto_next) {
        dn[L.d_dts] = dp[L.d_dts + 1];
        dn[L.d_dts + 1] = 0.0;
        switching_time_direction(&L, rr, dn, g->sto);
        di[L.d_dts] = dn[L.d_dts];
        di[L.d_dts + 1] = dn[L.d_dts + 1];
      }
      costate_direction(&L, rr, di, g->sto, 0, 1);
    } else if (g->type == RBT_LIFT) {                                       /* :109-118 */
      const double* dp = d + (size_t)(i - 1) * L.d_stride;
      di[L.d_dts] = dp[L.d_dts + 1];
      di[L.d_dts + 1] = 0.0;
      if (g->sto_next) switching_time_direction(&L, rr, di, g->sto);
      forward_full(&L, kk, rr, di, dn, g->sto, g->sto_next);
      costate_direction(&L, rr, di, g->sto, g->sto_next, 0);
    } else {                                                                /* :119-123 */
      forward_full(&L, kk, rr, di, dn, g->sto, g->sto_next);
      costate_direction(&L, rr, di, g->sto, g->sto_next, 0);
    }
    if (g->ns > 0) multiplier_direction(&L, g->ns, rr, di, g->sto, g->sto_next); /* :124-126 */
  }
  costate_direction(&L, ric + (size_t)N * L.r_stride, d + (size_t)N * L.d_stride, 0, 0, 0); /* :128-130 */
}

/* ------------------------------------------------------------------------------------------
 * Unconstrained variant: unconstr_riccati_recursion.cpp:26-48, unconstr_riccati_factorizer.cpp:26-58,
 * unconstr_backward_riccati_recursion_factorizer.cpp:27-70.   A=[[I,dt I],[0,I]], B=[0;dt I] implicit.
 * ------------------------------------------------------------------------------------------ */
int orc_unconstr_backward(int nv, int N, double dt, double* kkt, double* ric) {
  rbt_ulayout L;
  rbt_make_ulayout(nv, &L);
  const int nx = L.nx;
  int info = 0;
  double* GK = (double*)calloc((size_t)nv * nx, 8);
  double* K = (double*)calloc((size_t)nv * nx, 8);
  double* Lg = (double*)calloc((size_t)nv * nv, 8);
  double* ricN = ric + (size_t)N * L.r_stride;
  const double* kktN = kkt + (size_t)N * L.k_stride;
  memcpy(ricN + L.r_P, kktN + L.k_Qxx, sizeof(double) * nx * nx);
  for (int i = 0; i < nx; ++i) ricN[L.r_s + i] = -kktN[L.k_lx + i];
  for (int st = N - 1; st >= 0; --st) {
    double* kk = kkt + (size_t)st * L.k_stride;
    double* rr = ric + (size_t)st * L.r_stride;
    const double* rn = ric + (size_t)(st + 1) * L.r_stride;
    const double* Pn = rn + L.r_P;
    const double* sn = rn + L.r_s;
    double* F = kk + L.k_Qxx;
    double* H = kk + L.k_Qxu; /* nx x nv */
    double* G = kk + L.k_Qaa;
    const double* Fx = kk + L.k_Fx;
    const double* lx = kk + L.k_lx;
    double* la = kk + L.k_la;
    /* factorizeKKTMatrix: unconstr_backward_riccati_recursion_factorizer.cpp:31-50 */
    for (int j = 0; j < nx; ++j)
      for (int i = 0; i < nx; ++i) F[IDX(i, j, nx)] += Pn[IDX(i, j, nx)];                      /* :32 */
    for (int j = 0; j < nx; ++j)
      for (int i = 0; i < nv; ++i) F[IDX(nv + i, j, nx)] += dt * Pn[IDX(i, j, nx)];            /* :33-34 */
    for (int j = 0; j < nv; ++j)
      for (int i = 0; i < nx; ++i) F[IDX(i, nv + j, nx)] += dt * Pn[IDX(i, j, nx)];            /* :35-36 */
    for (int j = 0; j < nv; ++j)
      for (int i = 0; i < nv; ++i) F[IDX(nv + i, nv + j, nx)] += (dt * dt) * Pn[IDX(i, j, nx)]; /* :37-38 */
    for (int j = 0; j < nv; ++j)
      for (int i = 0; i < nx; ++i) H[IDX(i, j, nx)] += dt * Pn[IDX(i, nv + j, nx)];            /* :40 */
    for (int j = 0; j < nv; ++j)
      for (int i = 0; i < nv; ++i) H[IDX(nv + i, j, nx)] += (dt * dt) * Pn[IDX(i, nv + j, nx)]; /* :41 */
    for (int j = 0; j < nv; ++j)
      for (int i = 0; i < nv; ++i) G[IDX(i, j, nv)] += (dt * dt) * Pn[IDX(nv + i, nv + j, nx)]; /* :43 */
    for (int i = 0; i < nv; ++i) {                                                             /* :45-47 */
      double acc = 0.0;
      for (int l = 0; l < nx; ++l) acc += Pn[IDX(nv + i, l, nx)] * Fx[l];
      la[i] += dt * acc;
    }
    for (int i = 0; i < nv; ++i) la[i] -= dt * sn[nv + i];
    /* unconstr_riccati_factorizer.cpp:33-36 */
    memcpy(Lg, G, sizeof(double) * nv * nv);
    if (chol_lower(nv, Lg, nv)) info = 1;
    for (int j = 0; j < nx; ++j)
      for (int i = 0; i < nv; ++i) K[IDX(i, j, nv)] = H[IDX(j, i, nx)];
    chol_solve(nv, Lg, nv, nx, K, nv);
    for (int i = 0; i < nv * nx; ++i) K[i] = -K[i];
    double* kvec = rr + L.r_k;
    memcpy(kvec, la, sizeof(double) * nv);
    chol_solve(nv, Lg, nv, 1, kvec, nv);
    for (int i = 0; i < nv; ++i) kvec[i] = -kvec[i];
    /* factorizeRiccatiFactorization: unconstr_backward_riccati_recursion_factorizer.cpp:59-69 */
    double* P = rr + L.r_P;
    double* s = rr + L.r_s;
    gemm(0, 0, nv, nx, nv, 1.0, G, nv, K, nv, 0.0, GK, nv);
    gemm(1, 0, nx, nx, nv, -1.0, K, nv, GK, nv, 1.0, F, nx);
    for (int j = 0; j < nx; ++j)
      for (int i = 0; i < nx; ++i) P[IDX(i, j, nx)] = 0.5 * (F[IDX(i, j, nx)] + F[IDX(j, i, nx)]);
    memcpy(s, sn, sizeof(double) * nx);                                                        /* :63 */
    for (int i = 0; i < nv; ++i) s[nv + i] += dt * sn[i];                                      /* :64 */
    gemm(0, 0, nx, 1, nx, -1.0, Pn, nx, Fx, nx, 1.0, s, nx);                                   /* :65 */
    for (int i = 0; i < nv; ++i) {                                                             /* :66-67 */
      double acc = 0.0;
      for (int l = 0; l < nx; ++l) acc += Pn[IDX(i, l, nx)] * Fx[l];
      s[nv + i] -= dt * acc;
    }
    for (int i = 0; i < nx; ++i) s[i] -= lx[i];                                                /* :68 */
    gemm(0, 0, nx, 1, nv, -1.0, H, nx, kvec, nv, 1.0, s, nx);                                  /* :69 */
    double* Kt = rr + L.r_K;
    for (int j = 0; j < nx; ++j)
      for (int i = 0; i < nv; ++i) Kt[IDX(j, i, nx)] = K[IDX(i, j, nv)];
  }
  free(GK); free(K); free(Lg);
  return info;
}

/* UnconstrRiccatiRecursion::forwardRiccatiRecursion unconstr_riccati_recursion.cpp:37-46,
 * UnconstrRiccatiFactorizer::forwardRiccatiRecursion unconstr_riccati_factorizer.cpp:43-52, costate :55-58 */
void orc_unconstr_forward(int nv, int N, double dt, const double* kkt, const double* ric, double* d) {
  rbt_ulayout L;
  rbt_make_ulayout(nv, &L);
  const int nx = L.nx;
  for (int st = 0; st <= N; ++st) {
    const double* rr = ric + (size_t)st * L.r_stride;
    double* di = d + (size_t)st * L.d_stride;
    const double* dx = di + L.d_dx;
    if (st < N) {
      const double* kk = kkt + (size_t)st * L.k_stride;
      double* dn = d + (size_t)(st + 1) * L.d_stride;
      double* da = di + L.d_da;
      gemm(1, 0, nv, 1, nx, 1.0, rr + L.r_K, nx, dx, nx, 0.0, da, nv);
      for (int i = 0; i < nv; ++i) da[i] += rr[L.r_k + i];
      for (int i = 0; i < nx; ++i) dn[L.d_dx + i] = kk[L.k_Fx + i] + dx[i];
      for (int i = 0; i < nv; ++i) dn[L.d_dx + i] += dt * dx[nv + i];
      for (int i = 0; i < nv; ++i) dn[L.d_dx + nv + i] += dt * da[i];
    }
    double* dl = di + L.d_dlmdgmm;
    gemm(0, 0, nx, 1, nx, 1.0, rr + L.r_P, nx, dx, nx, 0.0, dl, nx);
    for (int i = 0; i < nx; ++i) dl[i] -= rr[L.r_s + i];
  }
}

/* ---------------- batched drivers (CPU baseline): OpenMP over OCP instances, serial inside each OCP,
 * i.e. BASELINE.md 3 mode (ii) "best-case CPU".  nthreads<=0 -> OpenMP default. */
#ifdef _OPENMP
#include <omp.h>
#endif

int orc_riccati_batch(const rbt_dims* dims, const rbt_stage_ctrl* ctrl, int n_grid, double max_dts0, int batch,
                      double* kkt, double* ric, const double* dx0, double* d, int nthreads) {
  rbt_layout L;
  rbt_make_layout(dims, &L);
  int info = 0;
#ifdef _OPENMP
  if (nthreads > 0) omp_set_num_threads(nthreads);
#endif
#pragma omp parallel for schedule(dynamic) reduction(| : info)
  for (int b = 0; b < batch; ++b) {
    double* kk = kkt + (size_t)b * n_grid * L.k_stride;
    double* rr = ric + (size_t)b * n_grid * L.r_stride;
    info |= orc_riccati_backward(dims, ctrl, n_grid, max_dts0, kk, rr);
    if (d) {
      double* dd = d + (size_t)b * n_grid * L.d_stride;
      memcpy(dd + L.d_dx, dx0 + (size_t)b * L.nx, sizeof(double) * L.nx);
      orc_riccati_forward(dims, ctrl, n_grid, kk, rr, dd);
    }
  }
  return info;
}

int orc_unconstr_batch(int nv, int N, double dt, int batch, double* kkt, double* ric, const double* dx0, double* d,
                       int nthreads) {
  rbt_ulayout L;
  rbt_make_ulayout(nv, &L);
  int info = 0;
#ifdef _OPENMP
  if (nthreads > 0) omp_set_num_threads(nthreads);
#endif
#pragma omp parallel for schedule(dynamic) reduction(| : info)
  for (int b = 0; b < batch; ++b) {
    double* kk = kkt + (size_t)b * (N + 1) * L.k_stride;
    double* rr = ric + (size_t)b * (N + 1) * L.r_stride;
    info |= orc_unconstr_backward(nv, N, dt, kk, rr);
    if (d) {
      double* dd = d + (size_t)b * (N + 1) * L.d_stride;
      memcpy(dd + L.d_dx, dx0 + (size_t)b * L.nx, sizeof(double) * L.nx);
      orc_unconstr_forward(nv, N, dt, kk, rr, dd);
    }
  }
  return info;
}

int orc_max_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

/* single-step entry points for unit tests of the factorizer identities */
int orc_backward_full_step(const rbt_dims* dims, int ns, int sto, int sto_next, const double* ric_next, double* kkt,
                           double* ric) {
  rbt_layout L;
  rbt_make_layout(dims, &L);
  orc_ws* w = ws_new(&L);
  int info = backward_full(&L, w, ns, sto, sto_next, ric_next, kkt, ric);
  ws_free(w);
  return info;
}

void orc_backward_impact_step(const rbt_dims* dims, int sto, const double* ric_next, double* kkt, double* ric) {
  rbt_layout L;
  rbt_make_layout(dims, &L);
  orc_ws* w = ws_new(&L);
  backward_impact(&L, w, sto, ric_next, kkt, ric);
  ws_free(w);
}

void orc_phase_transition_step(const rbt_dims* dims, double max_dts0, const double* ric, double* ric_m, double* pol,
                               int sto_next) {
  rbt_layout L;
  rbt_make_layout(dims, &L);
  phase_transition(&L, max_dts0, ric, ric_m, pol, sto_next);
}

/* layout queries for the test side */
int orc_layout_get(const rbt_dims* dims, const char* field) {
  rbt_layout L;
  rbt_make_layout(dims, &L);
  return rbt_layout_field(&L, field);
}
int orc_ulayout_get(int nv, const char* field) {
  rbt_ulayout L;
  rbt_make_ulayout(nv, &L);
  return rbt_ulayout_field(&L, field);
}
