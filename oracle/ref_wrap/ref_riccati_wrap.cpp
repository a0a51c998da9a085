// oracle/ref_wrap/ref_riccati_wrap.cpp -- TEST INFRASTRUCTURE.  C entry points around the REFERENCE's own Riccati classes,
// compiled unmodified from robotoc/src/riccati/*.cpp and src/core/split_*.cpp (see oracle/Makefile.ref) against the
// Eigen / Robot stand-ins of oracle/shim/.  Records in and out use the packed layout of include/rbt_layout.h, exactly like
// the oracle's orc_riccati_batch / orc_unconstr_batch, so a test can hand the same arrays to both and compare.
//   robotoc::RiccatiRecursion::backwardRiccatiRecursion / forwardRiccatiRecursion   src/riccati/riccati_recursion.cpp:32-131
//   robotoc::UnconstrRiccatiRecursion                                               src/riccati/unconstr_riccati_recursion.cpp:26-48
#include <cstring>
#include <vector>
#include <cassert>
#include <cmath>
#include <iostream>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <memory>
#include <limits>
#include <random>
#include <chrono>

#include "Eigen/Core"
#include "Eigen/LU"
#include "robotoc/robot/robot.hpp"
#include "robotoc/core/kkt_matrix.hpp"
#include "robotoc/core/kkt_residual.hpp"
#include "robotoc/core/direction.hpp"
#include "robotoc/ocp/ocp.hpp"
#include "robotoc/ocp/time_discretization.hpp"
// The STO policies are a private member of RiccatiRecursion without a getter (riccati_recursion.hpp:114-117); the
// wrapper reads them to compare dtsdx / dtsdts / dts0.  Only this translation unit sees the relaxed access; the
// reference's own sources are compiled as they are.
#define private public
#include "robotoc/riccati/riccati_recursion.hpp"
#undef private
#include "robotoc/riccati/unconstr_riccati_recursion.hpp"

#include "../../include/rbt_layout.h"

namespace {

using robotoc::GridInfo;
using robotoc::GridType;

void put_mat(Eigen::MatrixXd& M, const double* src, int rows, int cols) {
  for (int j = 0; j < cols; ++j) for (int i = 0; i < rows; ++i) M(i, j) = src[i + j * rows];
}
template <class V> void put_vec(V&& v, const double* src, int n) { for (int i = 0; i < n; ++i) v(i) = src[i]; }
template <class M> void get_mat(const M& m, double* dst, int rows, int cols) {
  for (int j = 0; j < cols; ++j) for (int i = 0; i < rows; ++i) dst[i + j * rows] = m(i, j);
}
template <class V> void get_vec(const V& v, double* dst, int n) { for (int i = 0; i < n; ++i) dst[i] = v(i); }

robotoc::TimeDiscretization make_td(const rbt_stage_ctrl* ctrl, int n_grid) {
  std::vector<GridInfo> g(static_cast<size_t>(n_grid));
  for (int i = 0; i < n_grid; ++i) {
    g[i].type = static_cast<GridType>(ctrl[i].type);
    g[i].dt = ctrl[i].dt;
    g[i].sto = ctrl[i].sto != 0;
    g[i].sto_next = ctrl[i].sto_next != 0;
    g[i].switching_constraint = ctrl[i].ns > 0;
    g[i].num_grids_in_phase = ctrl[i].ngrids_in_phase;
    g[i].stage = i;
  }
  return robotoc::TimeDiscretization(g);
}

}  // namespace

extern "C" {

// One OCP after the other (the reference is single-OCP).  kkt is mutated in place like the reference mutates its
// SplitKKTMatrix / SplitKKTResidual (Qxx, Qxu, Quu, lu <- F, H, G, lu').  Returns 0.
int ref_riccati_batch(const rbt_dims* dims, const rbt_stage_ctrl* ctrl, int n_grid, double max_dts0, int batch, double* kkt,
                      double* ric, const double* dx0, double* dir) {
  rbt_layout L;
  rbt_make_layout(dims, &L);
  const int nv = L.nv, nu = L.nu, nx = L.nx;
  const int N = n_grid - 1;
  robotoc::OCP ocp;
  ocp.robot = robotoc::Robot(nv, dims->n_passive == 6, dims->ns_max / 3);
  assert(ocp.robot.dimu() == nu);
  ocp.N = N;
  ocp.reserved_num_discrete_events = 0;
  const robotoc::TimeDiscretization td = make_td(ctrl, n_grid);
  for (int b = 0; b < batch; ++b) {
    robotoc::KKTMatrix kkt_matrix(static_cast<size_t>(n_grid), robotoc::SplitKKTMatrix(ocp.robot));
    robotoc::KKTResidual kkt_residual(static_cast<size_t>(n_grid), robotoc::SplitKKTResidual(ocp.robot));
    robotoc::RiccatiFactorization factorization(static_cast<size_t>(n_grid), robotoc::SplitRiccatiFactorization(ocp.robot));
    robotoc::Direction d(static_cast<size_t>(n_grid), robotoc::SplitDirection(ocp.robot));
    double* kkt_b = kkt + size_t(b) * n_grid * L.k_stride;
    for (int i = 0; i < n_grid; ++i) {
      const double* rec = kkt_b + size_t(i) * L.k_stride;
      robotoc::SplitKKTMatrix& km = kkt_matrix[i];
      robotoc::SplitKKTResidual& kr = kkt_residual[i];
      put_mat(km.Qxx, rec + L.k_Qxx, nx, nx);
      put_vec(kr.lx, rec + L.k_lx, nx);
      if (ctrl[i].type == RBT_TERMINAL) continue;
      put_mat(km.Fxx, rec + L.k_Fxx, nx, nx);
      put_vec(kr.Fx, rec + L.k_Fx, nx);
      if (ctrl[i].type == RBT_IMPACT) continue;
      put_mat(km.Fvu, rec + L.k_Fvu, nv, nu);
      put_mat(km.Qxu, rec + L.k_Qxu, nx, nu);
      put_mat(km.Quu, rec + L.k_Quu, nu, nu);
      put_vec(kr.lu, rec + L.k_lu, nu);
      const int ns = ctrl[i].ns;
      km.setSwitchingConstraintDimension(ns);
      kr.setSwitchingConstraintDimension(ns);
      if (ns > 0) {
        for (int j = 0; j < nx; ++j) for (int r = 0; r < ns; ++r) km.Phix()(r, j) = rec[L.k_Phix + r + j * ns];
        for (int j = 0; j < nu; ++j) for (int r = 0; r < ns; ++r) km.Phiu()(r, j) = rec[L.k_Phiu + r + j * ns];
        for (int r = 0; r < ns; ++r) kr.P()(r) = rec[L.k_p + r];
      }
      if (ctrl[i].sto) {
        put_vec(km.fx, rec + L.k_fx, nx);
        put_vec(km.hx, rec + L.k_hx, nx);
        put_vec(km.hu, rec + L.k_hu, nu);
        for (int r = 0; r < ns; ++r) km.Phit()(r) = rec[L.k_Phit + r];
        km.Qtt = rec[L.k_sc + 0];
        km.Qtt_prev = rec[L.k_sc + 1];
        kr.h = rec[L.k_sc + 2];
      }
    }
    robotoc::RiccatiRecursion rr(ocp, max_dts0);
    rr.backwardRiccatiRecursion(td, kkt_matrix, kkt_residual, factorization);
    if (dx0) {
      put_vec(d[0].dx, dx0 + size_t(b) * nx, nx);
      rr.forwardRiccatiRecursion(td, kkt_matrix, kkt_residual, factorization, d);
    }
    // ---- unpack
    double* ric_b = ric + size_t(b) * n_grid * L.r_stride;
    const robotoc::aligned_vector<robotoc::LQRPolicy>& pol = rr.getLQRPolicy();
    for (int i = 0; i < n_grid; ++i) {
      double* r = ric_b + size_t(i) * L.r_stride;
      double* rec = kkt_b + size_t(i) * L.k_stride;
      const robotoc::SplitRiccatiFactorization& f = factorization[i];
      get_mat(f.P, r + L.r_P, nx, nx);
      get_vec(f.s, r + L.r_s, nx);
      get_vec(f.Psi, r + L.r_Psi, nx);
      get_vec(f.Phi, r + L.r_Phi, nx);
      r[L.r_sc + 0] = f.xi; r[L.r_sc + 1] = f.chi; r[L.r_sc + 2] = f.rho; r[L.r_sc + 3] = f.eta; r[L.r_sc + 4] = f.iota;
      // STO policies live at the index the recursion used (riccati_recursion.cpp:42-78)
      get_vec(rr.sto_policy_[i].dtsdx, r + L.r_dtsdx, nx);
      r[L.r_stosc + 0] = rr.sto_policy_[i].dtsdts;
      r[L.r_stosc + 1] = rr.sto_policy_[i].dts0;
      if (ctrl[i].type == RBT_TERMINAL) continue;
      get_mat(kkt_matrix[i].Qxx, rec + L.k_Qxx, nx, nx);  // mutated in place (F, or F - K^T G K on control stages)
      if (ctrl[i].type == RBT_IMPACT) continue;
      get_mat(kkt_matrix[i].Qxu, rec + L.k_Qxu, nx, nu);
      get_mat(kkt_matrix[i].Quu, rec + L.k_Quu, nu, nu);
      get_vec(kkt_residual[i].lu, rec + L.k_lu, nu);
      for (int u = 0; u < nu; ++u) for (int j = 0; j < nx; ++j) r[L.r_K + j + u * nx] = pol[i].K(u, j);  // row-major K == col-major K^T
      get_vec(pol[i].k, r + L.r_k, nu);
      get_vec(pol[i].T, r + L.r_T, nu);
      get_vec(pol[i].W, r + L.r_W, nu);
      get_vec(f.psi_x, r + L.r_psix, nx);
      get_vec(f.psi_u, r + L.r_psiu, nu);
      get_vec(f.phi_x, r + L.r_phix, nx);
      get_vec(f.phi_u, r + L.r_phiu, nu);
      const int ns = ctrl[i].ns;
      if (ns > 0) {
        for (int j = 0; j < nx; ++j) for (int q = 0; q < ns; ++q) r[L.r_M + q + j * ns] = f.M()(q, j);
        for (int q = 0; q < ns; ++q) {
          r[L.r_m + q] = f.m()(q);
          r[L.r_mt + q] = f.mt()(q);
          r[L.r_mtn + q] = f.mt_next()(q);
        }
      }
    }
    if (dx0) {
      double* dir_b = dir + size_t(b) * n_grid * L.d_stride;
      for (int i = 0; i < n_grid; ++i) {
        double* r = dir_b + size_t(i) * L.d_stride;
        get_vec(d[i].dx, r + L.d_dx, nx);
        get_vec(d[i].dlmdgmm, r + L.d_dlmdgmm, nx);
        r[L.d_dts] = d[i].dts;
        r[L.d_dts + 1] = d[i].dts_next;
        if (ctrl[i].type == RBT_TERMINAL || ctrl[i].type == RBT_IMPACT) continue;
        get_vec(d[i].du, r + L.d_du, nu);
        for (int q = 0; q < ctrl[i].ns; ++q) r[L.d_dxi + q] = d[i].dxi()(q);
      }
    }
  }
  return 0;
}

// Unconstrained recursion (iiwa14-style fixed base, control = acceleration).  Records: rbt_ulayout.
int ref_unconstr_batch(int nv, int N, double dt, int batch, double* kkt, double* ric, const double* dx0, double* dir) {
  rbt_ulayout L;
  rbt_make_ulayout(nv, &L);
  const int nx = 2 * nv;
  robotoc::OCP ocp;
  ocp.robot = robotoc::Robot(nv, false, 0);
  ocp.N = N;
  ocp.T = dt * N;
  for (int b = 0; b < batch; ++b) {
    robotoc::KKTMatrix kkt_matrix(static_cast<size_t>(N + 1), robotoc::SplitKKTMatrix(ocp.robot));
    robotoc::KKTResidual kkt_residual(static_cast<size_t>(N + 1), robotoc::SplitKKTResidual(ocp.robot));
    robotoc::UnconstrRiccatiFactorization factorization(static_cast<size_t>(N + 1), robotoc::SplitRiccatiFactorization(ocp.robot));
    robotoc::Direction d(static_cast<size_t>(N + 1), robotoc::SplitDirection(ocp.robot));
    double* kkt_b = kkt + size_t(b) * (N + 1) * L.k_stride;
    for (int i = 0; i <= N; ++i) {
      const double* rec = kkt_b + size_t(i) * L.k_stride;
      put_mat(kkt_matrix[i].Qxx, rec + L.k_Qxx, nx, nx);
      put_vec(kkt_residual[i].lx, rec + L.k_lx, nx);
      if (i == N) continue;
      put_mat(kkt_matrix[i].Qxu, rec + L.k_Qxu, nx, nv);
      put_mat(kkt_matrix[i].Qaa, rec + L.k_Qaa, nv, nv);
      put_vec(kkt_residual[i].Fx, rec + L.k_Fx, nx);
      put_vec(kkt_residual[i].la, rec + L.k_la, nv);
    }
    robotoc::UnconstrRiccatiRecursion rr(ocp);
    rr.backwardRiccatiRecursion(kkt_matrix, kkt_residual, factorization);
    if (dx0) {
      put_vec(d[0].dx, dx0 + size_t(b) * nx, nx);
      rr.forwardRiccatiRecursion(kkt_residual, factorization, d);
    }
    double* ric_b = ric + size_t(b) * (N + 1) * L.r_stride;
    const std::vector<robotoc::LQRPolicy>& pol = rr.getLQRPolicy();
    for (int i = 0; i <= N; ++i) {
      double* r = ric_b + size_t(i) * L.r_stride;
      double* rec = kkt_b + size_t(i) * L.k_stride;
      get_mat(factorization[i].P, r + L.r_P, nx, nx);
      get_vec(factorization[i].s, r + L.r_s, nx);
      if (i == N) continue;
      for (int a = 0; a < nv; ++a) for (int j = 0; j < nx; ++j) r[L.r_K + j + a * nx] = pol[i].K(a, j);
      get_vec(pol[i].k, r + L.r_k, nv);
      get_mat(kkt_matrix[i].Qxx, rec + L.k_Qxx, nx, nx);
      get_mat(kkt_matrix[i].Qxu, rec + L.k_Qxu, nx, nv);
      get_mat(kkt_matrix[i].Qaa, rec + L.k_Qaa, nv, nv);
      get_vec(kkt_residual[i].la, rec + L.k_la, nv);
    }
    if (dx0) {
      double* dir_b = dir + size_t(b) * (N + 1) * L.d_stride;
      for (int i = 0; i <= N; ++i) {
        double* r = dir_b + size_t(i) * L.d_stride;
        get_vec(d[i].dx, r + L.d_dx, nx);
        get_vec(d[i].dlmdgmm, r + L.d_dlmdgmm, nx);
        if (i < N) get_vec(d[i].da(), r + L.d_da, nv);
      }
    }
  }
  return 0;
}

const char* ref_version(void) { return "robotoc reference sources (d30d404) compiled unmodified against oracle/shim"; }

}  // extern "C"
