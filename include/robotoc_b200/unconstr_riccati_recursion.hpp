// robotoc_b200/unconstr_riccati_recursion.hpp -- C++ host-side adaptors for the unconstrained (fixed-base, no contacts) path with
// the reference's class and method names on top of the C ABI (include/robotoc_b200.h).  Header-only, C++14, no Eigen.
//
//   robotoc::UnconstrRiccatiRecursion          include/robotoc/riccati/unconstr_riccati_recursion.hpp:22-70
//                                              src/riccati/unconstr_riccati_recursion.cpp:9-48
//   robotoc::UnconstrDirectMultipleShooting    include/robotoc/unconstr/unconstr_direct_multiple_shooting.hpp
//                                              src/unconstr/unconstr_direct_multiple_shooting.cpp:88-179 (hot-path half)
//
// The containers are the Matrix / Vector types of riccati_recursion.hpp (column-major like Eigen::MatrixXd); the members
// carry the reference's names (Qxx, Qxu, Qaa, Fx, lx, la; P, s; K row-major nv x nx == column-major K^T; dx, da, dlmdgmm).
#pragma once
#include "riccati_recursion.hpp"

namespace robotoc_b200 {

struct UnconstrSplitKKTMatrix {
  Matrix Qxx, Qxu, Qaa;  // nx x nx, nx x nv, nv x nv
  UnconstrSplitKKTMatrix() = default;
  explicit UnconstrSplitKKTMatrix(int nv) : Qxx(2 * nv, 2 * nv), Qxu(2 * nv, nv), Qaa(nv, nv) {}
};
struct UnconstrSplitKKTResidual {
  Vector Fx, lx, la;
  UnconstrSplitKKTResidual() = default;
  explicit UnconstrSplitKKTResidual(int nv) : Fx(2 * nv), lx(2 * nv), la(nv) {}
};
struct UnconstrSplitDirection {
  Vector dx, da, dlmdgmm;
  UnconstrSplitDirection() = default;
  explicit UnconstrSplitDirection(int nv) : dx(2 * nv), da(nv), dlmdgmm(2 * nv) {}
};
struct UnconstrLQRPolicy {
  Matrix Kt;  // K^T column-major == the reference's row-major nv x nx K
  Vector k;
  UnconstrLQRPolicy() = default;
  explicit UnconstrLQRPolicy(int nv) : Kt(2 * nv, nv), k(nv) {}
  double K(int a, int j) const { return Kt(j, a); }
};
struct UnconstrSplitRiccatiFactorization {
  Matrix P;
  Vector s;
  UnconstrSplitRiccatiFactorization() = default;
  explicit UnconstrSplitRiccatiFactorization(int nv) : P(2 * nv, 2 * nv), s(2 * nv) {}
};

/// Drop-in for robotoc::UnconstrRiccatiRecursion, ONE OCP (batch = 1): N stages + terminal, dt = T / N.
class UnconstrRiccatiRecursion {
 public:
  /// UnconstrRiccatiRecursion(const OCP& ocp): nv = ocp.robot.dimv(), N = ocp.N, T = ocp.T   (unconstr_riccati_recursion.cpp:9-14)
  UnconstrRiccatiRecursion(int nv, int N, double T, int device = 0) : nv_(nv), N_(N) {
    if (N <= 0) throw std::out_of_range("[UnconstrRiccatiRecursion] invalid argument: 'N' must be positive!");
    if (T <= 0) throw std::out_of_range("[UnconstrRiccatiRecursion] invalid argument: 'T' must be positive!");
    rbt_make_ulayout(nv, &L_);
    const int rc = rbt_unconstr_create(nv, N, T / N, 1, device, &h_);
    if (rc != RBT_OK) {
      const std::string msg = h_ ? rbt_unconstr_last_error(h_) : "unsupported robot dimension";
      if (h_) rbt_unconstr_destroy(h_);
      h_ = nullptr;
      throw std::runtime_error("[UnconstrRiccatiRecursion] cannot create the device handle: " + msg);
    }
    lqr_policy_.assign(size_t(N) + 1, UnconstrLQRPolicy(nv));
  }
  ~UnconstrRiccatiRecursion() { if (h_) rbt_unconstr_destroy(h_); }
  UnconstrRiccatiRecursion(const UnconstrRiccatiRecursion&) = delete;
  UnconstrRiccatiRecursion& operator=(const UnconstrRiccatiRecursion&) = delete;

  /// unconstr_riccati_recursion.cpp:26-35.  kkt_matrix / kkt_residual are mutated like the reference (Qxx, Qxu, Qaa, la <- F, H, G, la').
  void backwardRiccatiRecursion(std::vector<UnconstrSplitKKTMatrix>& kkt_matrix, std::vector<UnconstrSplitKKTResidual>& kkt_residual,
                                std::vector<UnconstrSplitRiccatiFactorization>& factorization) {
    const int nx = 2 * nv_;
    if (int(kkt_matrix.size()) != N_ + 1 || int(kkt_residual.size()) != N_ + 1)
      throw std::invalid_argument("[UnconstrRiccatiRecursion] invalid argument: horizon containers must hold N+1 stages");
    kkt_.assign(size_t(N_ + 1) * L_.k_stride, 0.0);
    for (int i = 0; i <= N_; ++i) {
      double* rec = kkt_.data() + size_t(i) * L_.k_stride;
      std::memcpy(rec + L_.k_Qxx, kkt_matrix[i].Qxx.data(), sizeof(double) * nx * nx);
      std::memcpy(rec + L_.k_lx, kkt_residual[i].lx.data(), sizeof(double) * nx);
      if (i == N_) continue;
      std::memcpy(rec + L_.k_Qxu, kkt_matrix[i].Qxu.data(), sizeof(double) * nx * nv_);
      std::memcpy(rec + L_.k_Qaa, kkt_matrix[i].Qaa.data(), sizeof(double) * nv_ * nv_);
      std::memcpy(rec + L_.k_Fx, kkt_residual[i].Fx.data(), sizeof(double) * nx);
      std::memcpy(rec + L_.k_la, kkt_residual[i].la.data(), sizeof(double) * nv_);
    }
    check(rbt_unconstr_upload(h_, RBT_BUF_KKT, kkt_.data(), nullptr));
    check(rbt_unconstr_backward(h_, /*write_fact=*/1, nullptr));
    ric_.resize(size_t(N_ + 1) * L_.r_stride);
    fact_.resize(size_t(N_ + 1) * L_.f_stride);
    check(rbt_unconstr_download(h_, RBT_BUF_RIC, ric_.data(), nullptr));
    check(rbt_unconstr_download(h_, RBT_BUF_FACT, fact_.data(), nullptr));
    check(rbt_unconstr_sync(h_, nullptr));
    int flag = 0;
    check(rbt_unconstr_download_info(h_, &flag, nullptr));
    check(rbt_unconstr_sync(h_, nullptr));
    if (flag) throw std::runtime_error("[UnconstrRiccatiRecursion] Qaa + B^T P B is not positive definite (the reference asserts llt_.info() == Eigen::Success)");
    factorization.resize(size_t(N_) + 1);
    for (int i = 0; i <= N_; ++i) {
      const double* r = ric_.data() + size_t(i) * L_.r_stride;
      if (factorization[i].P.rows() != nx) factorization[i] = UnconstrSplitRiccatiFactorization(nv_);
      std::memcpy(factorization[i].P.data(), r + L_.r_P, sizeof(double) * nx * nx);
      std::memcpy(factorization[i].s.data(), r + L_.r_s, sizeof(double) * nx);
      if (i == N_) continue;
      std::memcpy(lqr_policy_[i].Kt.data(), r + L_.r_K, sizeof(double) * nx * nv_);
      std::memcpy(lqr_policy_[i].k.data(), r + L_.r_k, sizeof(double) * nv_);
      const double* fc = fact_.data() + size_t(i) * L_.f_stride;
      std::memcpy(kkt_matrix[i].Qxx.data(), fc + L_.f_F, sizeof(double) * nx * nx);
      std::memcpy(kkt_matrix[i].Qxu.data(), fc + L_.f_H, sizeof(double) * nx * nv_);
      std::memcpy(kkt_matrix[i].Qaa.data(), fc + L_.f_G, sizeof(double) * nv_ * nv_);
      std::memcpy(kkt_residual[i].la.data(), fc + L_.f_la, sizeof(double) * nv_);
    }
  }

  /// unconstr_riccati_recursion.cpp:37-46; d[0].dx holds the initial state direction.
  void forwardRiccatiRecursion(const std::vector<UnconstrSplitKKTResidual>&, const std::vector<UnconstrSplitRiccatiFactorization>&,
                               std::vector<UnconstrSplitDirection>& d) {
    const int nx = 2 * nv_;
    check(rbt_unconstr_upload(h_, RBT_BUF_DX0, d[0].dx.data(), nullptr));
    check(rbt_unconstr_forward(h_, nullptr));
    dir_.resize(size_t(N_ + 1) * L_.d_stride);
    check(rbt_unconstr_download(h_, RBT_BUF_DIR, dir_.data(), nullptr));
    check(rbt_unconstr_sync(h_, nullptr));
    for (int i = 0; i <= N_; ++i) {
      const double* r = dir_.data() + size_t(i) * L_.d_stride;
      std::memcpy(d[i].dx.data(), r + L_.d_dx, sizeof(double) * nx);
      std::memcpy(d[i].dlmdgmm.data(), r + L_.d_dlmdgmm, sizeof(double) * nx);
      if (i < N_) std::memcpy(d[i].da.data(), r + L_.d_da, sizeof(double) * nv_);
    }
  }

  const std::vector<UnconstrLQRPolicy>& getLQRPolicy() const { return lqr_policy_; }  // unconstr_riccati_recursion.hpp:66
  rbt_uhandle* handle() { return h_; }
  const rbt_ulayout& layout() const { return L_; }
  int N() const { return N_; }
  int dimv() const { return nv_; }
  void check(int rc) {
    if (rc == RBT_OK) return;
    const std::string msg = rbt_unconstr_last_error(h_);
    if (rc == RBT_ERR_ARG) throw std::invalid_argument("[UnconstrRiccatiRecursion] invalid argument: " + msg);
    throw std::runtime_error("[UnconstrRiccatiRecursion] " + msg);
  }

 private:
  int nv_, N_;
  rbt_ulayout L_;
  rbt_uhandle* h_ = nullptr;
  std::vector<UnconstrLQRPolicy> lqr_policy_;
  std::vector<double> kkt_, ric_, fact_, dir_;
};

/// The hot-path half of robotoc::UnconstrDirectMultipleShooting over the records of include/rbt_ustage_layout.h, sharing the
/// device buffers of an UnconstrRiccatiRecursion (as UnconstrOCPSolver owns both, src/solver/unconstr_ocp_solver.cpp:101-118):
///   dms.evalKKT(lin, con);  riccati backward / forward on the device-resident KKT;  dms.computeStepSizes();
///   dms.maxPrimalStepSize(); dms.maxDualStepSize();  dms.integrateSolution(sol);
class UnconstrDirectMultipleShooting {
 public:
  UnconstrDirectMultipleShooting(UnconstrRiccatiRecursion& riccati, const rbt_constraint_table& constraints) : rr_(riccati) {
    rbt_make_ustage_layout(rr_.dimv(), constraints.n_box, &S_);
    rr_.check(rbt_unconstr_stage_setup(rr_.handle(), &constraints));
  }
  /// condensing tail of UnconstrIntermediateStage::evalKKT (unconstr_intermediate_stage.cpp:96-98) for every stage
  void evalKKT(const std::vector<double>& lin, const std::vector<double>& con) {
    expect(lin, S_.l_stride, "lin");
    expect(con, S_.c_stride, "con");
    rr_.check(rbt_unconstr_upload(rr_.handle(), RBT_BUF_LIN, lin.data(), nullptr));
    rr_.check(rbt_unconstr_upload(rr_.handle(), RBT_BUF_CON, con.data(), nullptr));
    rr_.check(rbt_unconstr_condense(rr_.handle(), nullptr));
  }
  void backwardRiccatiRecursion() { rr_.check(rbt_unconstr_backward(rr_.handle(), 0, nullptr)); }
  void forwardRiccatiRecursion(const std::vector<double>& dx0) {
    if (int(dx0.size()) != 2 * rr_.dimv()) throw std::invalid_argument("[UnconstrDirectMultipleShooting] invalid argument: dx0 size");
    rr_.check(rbt_unconstr_upload(rr_.handle(), RBT_BUF_DX0, dx0.data(), nullptr));
    rr_.check(rbt_unconstr_forward(rr_.handle(), nullptr));
  }
  void computeStepSizes() {  // unconstr_direct_multiple_shooting.cpp:128-146
    rr_.check(rbt_unconstr_expand_and_step_sizes(rr_.handle(), nullptr));
    steps_.assign(2, 1.0);
    rr_.check(rbt_unconstr_download(rr_.handle(), RBT_BUF_STEPS, steps_.data(), nullptr));
    rr_.check(rbt_unconstr_sync(rr_.handle(), nullptr));
  }
  double maxPrimalStepSize() const { return steps_.at(0); }  // :149-152
  double maxDualStepSize() const { return steps_.at(1); }    // :153-156
  /// integrateSolution (:159-179) with the step sizes left on the device; `sol` is updated in place
  void integrateSolution(std::vector<double>& sol) {
    expect(sol, S_.s_stride, "sol");
    rr_.check(rbt_unconstr_upload(rr_.handle(), RBT_BUF_SOL, sol.data(), nullptr));
    rr_.check(rbt_unconstr_update(rr_.handle(), nullptr));
    rr_.check(rbt_unconstr_download(rr_.handle(), RBT_BUF_SOL, sol.data(), nullptr));
    rr_.check(rbt_unconstr_sync(rr_.handle(), nullptr));
  }
  const rbt_ustage_layout& layout() const { return S_; }

 private:
  void expect(const std::vector<double>& a, int stride, const char* what) const {
    if (a.size() != size_t(rr_.N() + 1) * stride)
      throw std::invalid_argument(std::string("[UnconstrDirectMultipleShooting] invalid argument: size of '") + what + "'");
  }
  UnconstrRiccatiRecursion& rr_;
  rbt_ustage_layout S_;
  std::vector<double> steps_;
};

}  // namespace robotoc_b200
