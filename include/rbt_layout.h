/*
 * rbt_layout.h -- packed fp64 record layout for one OCP stage (HBM / host staging).
 *
 * Plain C (usable from gcc, g++ and nvcc).  The records mirror the reference's
 * per-stage containers, block by block, as contiguous column-major doubles:
 *
 *   KKT record      <-> robotoc::SplitKKTMatrix   (robotoc/src/core/split_kkt_matrix.cpp:7-34)
 *                       robotoc::SplitKKTResidual (robotoc/src/core/split_kkt_residual.cpp:7-20)
 *   Riccati record  <-> robotoc::SplitRiccatiFactorization (include/robotoc/riccati/split_riccati_factorization.hpp),
 *                       robotoc::LQRPolicy (include/robotoc/riccati/lqr_policy.hpp:16-126; K is ROW-major there,
 *                       i.e. the same memory as a column-major nx x nu K^T, which is what we store),
 *                       robotoc::STOPolicy (include/robotoc/riccati/sto_policy.hpp)
 *   Direction record<-> robotoc::SplitDirection   (robotoc/src/core/split_direction.cpp:7-22)
 *
 * Arrays are [batch][stage][record]; every section offset is a multiple of 2 doubles (16 B,
 * the cp.async.bulk granule) and every record stride a multiple of 16 doubles (128 B).
 * Variable-size blocks (switching constraint, ns rows) are stored compactly with
 * leading dimension = ns of that stage inside a section sized for ns_max.
 */
#ifndef RBT_LAYOUT_H_
#define RBT_LAYOUT_H_

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__CUDACC__)
#define RBT_HD __host__ __device__
#else
#define RBT_HD
#endif

/* Grid types: same order as robotoc::GridType (include/robotoc/ocp/grid_info.hpp:14-19). */
enum { RBT_INTERMEDIATE = 0, RBT_IMPACT = 1, RBT_LIFT = 2, RBT_TERMINAL = 3 };

/* Robot dimensions (src/robot/robot.cpp:33-60): nv=dimv, nu=dimu, nx=2*nv, ns_max=max_dimf,
 * n_passive = dim_passive (6 for a floating base, else 0). */
typedef struct rbt_dims {
  int nv;
  int nu;
  int ns_max;
  int n_passive;
} rbt_dims;

/* Per-stage control word, derived from robotoc::GridInfo (grid_info.hpp:25-92); shared by the batch. */
typedef struct rbt_stage_ctrl {
  int type;            /* RBT_INTERMEDIATE / IMPACT / LIFT / TERMINAL */
  int sto;             /* GridInfo::sto */
  int sto_next;        /* GridInfo::sto_next */
  int ns;              /* switching-constraint dimension (0 if !switching_constraint) */
  int nf;              /* active contact dimension dimf of this stage's phase (impact dimf on Impact) */
  int ngrids_in_phase; /* GridInfo::num_grids_in_phase */
  int contact_mask;    /* bit c set: point contact c is active in this stage's phase (ContactStatus::isContactActive);
                          on an Impact stage: the contacts of the ImpactStatus */
  int ineq_gate;       /* which inequality levels act on this grid point (ConstraintsData::setTimeStage, constraints_data.cpp:20-45):
                          0 = all; 1 = no position-level limits (GridInfo::stage == 1); 2 = neither position- nor velocity-level
                          (GridInfo::stage == 0).  = max(0, 2 - GridInfo::stage); acceleration-level rows (torque limits,
                          friction cones) always act */
  double dt;           /* GridInfo::dt */
} rbt_stage_ctrl;

typedef struct rbt_layout {
  int nv, nu, nx, ns_max;
  /* ---- KKT record (input of the Riccati recursion; mutated blocks are NOT written back here) */
  int k_Fxx, k_Fvu, k_Qxx, k_Qxu, k_Quu, k_Fx, k_lx, k_lu; /* core */
  int k_Phix, k_Phiu, k_p;                                 /* switching constraint (ld = ns) */
  int k_fx, k_hx, k_hu, k_Phit, k_sc;                      /* STO: sc = {Qtt, Qtt_prev, h, 0} */
  int k_stage_size;  /* doubles of the leading [Fxx|Fvu|Fx|lx|lu] part (one bulk copy to shared memory) */
  int k_core_size;   /* doubles of the core section (what every stage transfers) */
  int k_extra_size;  /* doubles of the switching + STO sections [Phix|Phiu|p|fx|hx|hu|Phit|sc] */
  int k_stride;
  /* ---- Riccati record (output of backward) */
  int r_P, r_s, r_K, r_k;
  int r_M, r_m;
  int r_Psi, r_Phi, r_T, r_W, r_psix, r_psiu, r_phix, r_phiu, r_mt, r_mtn;
  int r_sc;          /* {xi, chi, rho, eta, iota, 0,0,0} */
  int r_dtsdx, r_stosc; /* STOPolicy: dtsdx (nx), {dtsdts, dts0} */
  int r_core_size;   /* [P|s|K|k] */
  int r_extra_size;  /* everything after the core */
  int r_stride;
  /* ---- factorized-KKT record (optional write-back of the mutated Qxx,Qxu,Quu,lu = F,H,G,lu) */
  int f_F, f_H, f_G, f_lu, f_stride;
  /* ---- direction record (output of forward) */
  int d_dx, d_du, d_dlmdgmm, d_dxi, d_dts; /* d_dts: {dts, dts_next} */
  int d_stride;
} rbt_layout;

static inline RBT_HD int rbt_up2(int x) { return (x + 1) & ~1; }
static inline RBT_HD int rbt_up16(int x) { return (x + 15) & ~15; }

static inline RBT_HD void rbt_make_layout(const rbt_dims* d, rbt_layout* L) {
  const int nv = d->nv, nu = d->nu, nx = 2 * d->nv, ns = d->ns_max;
  int o = 0;
  L->nv = nv; L->nu = nu; L->nx = nx; L->ns_max = ns;
  /* blocks staged through shared memory by one bulk copy come first ... */
  L->k_Fxx = o; o += rbt_up2(nx * nx);
  L->k_Fvu = o; o += rbt_up2(nv * nu);
  L->k_Fx = o; o += rbt_up2(nx);
  L->k_lx = o; o += rbt_up2(nx);
  L->k_lu = o; o += rbt_up2(nu);
  L->k_stage_size = o;
  /* ... then the Hessian blocks, which go straight to accumulator registers */
  L->k_Qxx = o; o += rbt_up2(nx * nx);
  L->k_Qxu = o; o += rbt_up2(nx * nu);
  L->k_Quu = o; o += rbt_up2(nu * nu);
  L->k_core_size = o;
  L->k_Phix = o; o += rbt_up2(ns * nx);
  L->k_Phiu = o; o += rbt_up2(ns * nu);
  L->k_p = o; o += rbt_up2(ns);
  L->k_fx = o; o += rbt_up2(nx);
  L->k_hx = o; o += rbt_up2(nx);
  L->k_hu = o; o += rbt_up2(nu);
  L->k_Phit = o; o += rbt_up2(ns);
  L->k_sc = o; o += 4;
  L->k_extra_size = o - L->k_core_size;
  L->k_stride = rbt_up16(o);

  o = 0;
  L->r_P = o; o += rbt_up2(nx * nx);
  L->r_s = o; o += rbt_up2(nx);
  L->r_K = o; o += rbt_up2(nu * nx);
  L->r_k = o; o += rbt_up2(nu);
  L->r_core_size = o;
  L->r_M = o; o += rbt_up2(ns * nx);
  L->r_m = o; o += rbt_up2(ns);
  L->r_Psi = o; o += rbt_up2(nx);
  L->r_Phi = o; o += rbt_up2(nx);
  L->r_T = o; o += rbt_up2(nu);
  L->r_W = o; o += rbt_up2(nu);
  L->r_psix = o; o += rbt_up2(nx);
  L->r_psiu = o; o += rbt_up2(nu);
  L->r_phix = o; o += rbt_up2(nx);
  L->r_phiu = o; o += rbt_up2(nu);
  L->r_mt = o; o += rbt_up2(ns);
  L->r_mtn = o; o += rbt_up2(ns);
  L->r_sc = o; o += 8;
  L->r_dtsdx = o; o += rbt_up2(nx);
  L->r_stosc = o; o += 2;
  L->r_extra_size = o - L->r_core_size;
  L->r_stride = rbt_up16(o);

  o = 0;
  L->f_F = o; o += rbt_up2(nx * nx);
  L->f_H = o; o += rbt_up2(nx * nu);
  L->f_G = o; o += rbt_up2(nu * nu);
  L->f_lu = o; o += rbt_up2(nu);
  L->f_stride = rbt_up16(o);

  o = 0;
  L->d_dx = o; o += rbt_up2(nx);
  L->d_du = o; o += rbt_up2(nu);
  L->d_dlmdgmm = o; o += rbt_up2(nx);
  L->d_dxi = o; o += rbt_up2(ns);
  L->d_dts = o; o += 2;
  L->d_stride = rbt_up16(o);
}

/* ---------------- unconstrained (fixed-base, no contacts) path: implicit A=[[I,dt I],[0,I]], B=[0;dt I];
 * control = acceleration a (dim nv).  Mirrors what UnconstrRiccatiRecursion touches
 * (robotoc/src/riccati/unconstr_riccati_recursion.cpp:26-48): Qxx,Qxu,Qaa,Fx,lx,la. */
typedef struct rbt_ulayout {
  int nv, nx;
  int k_Qxx, k_Qxu, k_Qaa, k_Fx, k_lx, k_la, k_stride;
  int r_P, r_s, r_K, r_k, r_stride;
  int f_F, f_H, f_G, f_la, f_stride;
  int d_dx, d_da, d_dlmdgmm, d_stride;
} rbt_ulayout;

static inline RBT_HD void rbt_make_ulayout(int nv, rbt_ulayout* L) {
  const int nx = 2 * nv;
  int o = 0;
  L->nv = nv; L->nx = nx;
  L->k_Qxx = o; o += rbt_up2(nx * nx);
  L->k_Qxu = o; o += rbt_up2(nx * nv);
  L->k_Qaa = o; o += rbt_up2(nv * nv);
  L->k_Fx = o; o += rbt_up2(nx);
  L->k_lx = o; o += rbt_up2(nx);
  L->k_la = o; o += rbt_up2(nv);
  L->k_stride = rbt_up16(o);
  o = 0;
  L->r_P = o; o += rbt_up2(nx * nx);
  L->r_s = o; o += rbt_up2(nx);
  L->r_K = o; o += rbt_up2(nv * nx);
  L->r_k = o; o += rbt_up2(nv);
  L->r_stride = rbt_up16(o);
  o = 0;
  L->f_F = o; o += rbt_up2(nx * nx);
  L->f_H = o; o += rbt_up2(nx * nv);
  L->f_G = o; o += rbt_up2(nv * nv);
  L->f_la = o; o += rbt_up2(nv);
  L->f_stride = rbt_up16(o);
  o = 0;
  L->d_dx = o; o += rbt_up2(nx);
  L->d_da = o; o += rbt_up2(nv);
  L->d_dlmdgmm = o; o += rbt_up2(nx);
  L->d_stride = rbt_up16(o);
}


/* ---------------- field lookup by name (host only; used by the ctypes / test side) */
#define RBT_LAYOUT_FIELDS(X) \
  X(nv) X(nu) X(nx) X(ns_max) \
  X(k_Fxx) X(k_Fvu) X(k_Qxx) X(k_Qxu) X(k_Quu) X(k_Fx) X(k_lx) X(k_lu) X(k_Phix) X(k_Phiu) X(k_p) \
  X(k_fx) X(k_hx) X(k_hu) X(k_Phit) X(k_sc) X(k_stage_size) X(k_core_size) X(k_extra_size) X(k_stride) \
  X(r_P) X(r_s) X(r_K) X(r_k) X(r_M) X(r_m) X(r_Psi) X(r_Phi) X(r_T) X(r_W) X(r_psix) X(r_psiu) \
  X(r_phix) X(r_phiu) X(r_mt) X(r_mtn) X(r_sc) X(r_dtsdx) X(r_stosc) X(r_core_size) X(r_extra_size) X(r_stride) \
  X(f_F) X(f_H) X(f_G) X(f_lu) X(f_stride) \
  X(d_dx) X(d_du) X(d_dlmdgmm) X(d_dxi) X(d_dts) X(d_stride)
#define RBT_ULAYOUT_FIELDS(X) \
  X(nv) X(nx) X(k_Qxx) X(k_Qxu) X(k_Qaa) X(k_Fx) X(k_lx) X(k_la) X(k_stride) \
  X(r_P) X(r_s) X(r_K) X(r_k) X(r_stride) X(f_F) X(f_H) X(f_G) X(f_la) X(f_stride) \
  X(d_dx) X(d_da) X(d_dlmdgmm) X(d_stride)

static inline int rbt_streq_(const char* a, const char* b) {
  while (*a && *a == *b) { ++a; ++b; }
  return *a == *b;
}
static inline int rbt_layout_field(const rbt_layout* L, const char* name) {
#define X(f) if (rbt_streq_(name, #f)) return L->f;
  RBT_LAYOUT_FIELDS(X)
#undef X
  return -1;
}
static inline int rbt_ulayout_field(const rbt_ulayout* L, const char* name) {
#define X(f) if (rbt_streq_(name, #f)) return L->f;
  RBT_ULAYOUT_FIELDS(X)
#undef X
  return -1;
}

#ifdef __cplusplus
}
#endif
#endif /* RBT_LAYOUT_H_ */
