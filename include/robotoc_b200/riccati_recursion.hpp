// robotoc_b200/riccati_recursion.hpp -- C++ host-side adaptor with the reference's class and method names on top of the
// C ABI (include/robotoc_b200.h).  Header-only, C++14, no Eigen: the containers below are the subset of the reference's
// Split* types that the Riccati path touches, with the reference's member names, column-major like Eigen::MatrixXd
// (LQRPolicy::K row-major like include/robotoc/riccati/lqr_policy.hpp:18-19).  A reference build would keep its own
// Eigen-based types and use the pack/unpack helpers with `.data()` pointers (see INTEGRATION.md).
//
//   robotoc::RiccatiRecursion                 include/robotoc/riccati/riccati_recursion.hpp:26-119
//   robotoc::SplitKKTMatrix / SplitKKTResidual  src/core/split_kkt_matrix.cpp:7-34, src/core/split_kkt_residual.cpp:7-20
//   robotoc::SplitRiccatiFactorization, LQRPolicy, SplitDirection, GridInfo
#pragma once
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

extern "C" {
#include "../robotoc_b200.h"
}

namespace robotoc_b200 {

struct Matrix {  // column-major, like Eigen::MatrixXd
  int rows_ = 0, cols_ = 0;
  std::vector<double> a;
  Matrix() = default;
  Matrix(int r, int c) : rows_(r), cols_(c), a(size_t(r) * c, 0.0) {}
  double& operator()(int i, int j) { return a[size_t(i) + size_t(j) * rows_]; }
  double operator()(int i, int j) const { return a[size_t(i) + size_t(j) * rows_]; }
  double* data() { return a.data(); }
  const double* data() const { return a.data(); }
  int rows() const { return rows_; }
  int cols() const { return cols_; }
  size_t size() const { return a.size(); }
};
using Vector = std::vector<double>;

enum class GridType { Intermediate, Impact, Lift, Terminal };  // grid_info.hpp:14-19

struct GridInfo {  // grid_info.hpp:25-92 (fields read on this path)
  GridType type = GridType::Intermediate;
  double dt = 0;
  bool sto = false, sto_next = false, switching_constraint = false;
  int num_grids_in_phase = 1;
  int dims = 0;  // dimension of the switching constraint attached to this grid (impact dimf), 0 if none
  int dimf = 0;  // active contact dimension
  int contact_mask = -1;  // bit per point contact that is closed on this grid (ContactStatus::isContactActive); must be given
                          // whenever dimf > 0 -- the library never guesses which feet are on the ground
  int stage = -1;         // GridInfo::stage (index of the grid point): the reference gates the position- / velocity-level
                          // inequality constraints on stages 0 and 1 with it; -1 = all levels act
};
using TimeDiscretization = std::vector<GridInfo>;  // size() == N+1 grid points, last one Terminal

struct SplitKKTMatrix {
  Matrix Fxx, Fvu, Qxx, Qxu, Quu, Phix_, Phiu_;
  Vector fx, hx, hu, Phit_;
  double Qtt = 0, Qtt_prev = 0;
  int dims_ = 0;
  SplitKKTMatrix() = default;
  SplitKKTMatrix(int nv, int nu, int ns_max)
      : Fxx(2 * nv, 2 * nv), Fvu(nv, nu), Qxx(2 * nv, 2 * nv), Qxu(2 * nv, nu), Quu(nu, nu), Phix_(ns_max, 2 * nv),
        Phiu_(ns_max, nu), fx(2 * nv), hx(2 * nv), hu(nu), Phit_(ns_max) {}
  void setSwitchingConstraintDimension(int dims) {
    dims_ = dims;
    Phix_ = Matrix(dims, Fxx.rows());
    Phiu_ = Matrix(dims, Quu.rows());
    Phit_.assign(dims, 0.0);
  }
  int dims() const { return dims_; }
  Matrix& Phix() { return Phix_; }
  Matrix& Phiu() { return Phiu_; }
  Vector& Phit() { return Phit_; }
};

struct SplitKKTResidual {
  Vector Fx, lx, lu, P_;
  double h = 0;
  SplitKKTResidual() = default;
  SplitKKTResidual(int nv, int nu) : Fx(2 * nv), lx(2 * nv), lu(nu) {}
  Vector& P() { return P_; }
};

struct SplitRiccatiFactorization {
  Matrix P, M_;
  Vector s, Psi, Phi, m_;
  double xi = 0, chi = 0, rho = 0, eta = 0, iota = 0;
  SplitRiccatiFactorization() = default;
  explicit SplitRiccatiFactorization(int nv) : P(2 * nv, 2 * nv), s(2 * nv), Psi(2 * nv), Phi(2 * nv) {}
  Matrix& M() { return M_; }
  Vector& m() { return m_; }
};

struct LQRPolicy {
  Matrix Kt;  // stores K^T column-major == the reference's row-major nu x nx K
  Vector k, T, W;
  LQRPolicy() = default;
  LQRPolicy(int nv, int nu) : Kt(2 * nv, nu), k(nu), T(nu), W(nu) {}
  double K(int u, int j) const { return Kt(j, u); }
};

struct SplitDirection {
  Vector dx, du, dlmdgmm, dxi_;
  double dts = 0, dts_next = 0;
  SplitDirection() = default;
  SplitDirection(int nv, int nu) : dx(2 * nv), du(nu), dlmdgmm(2 * nv) {}
  Vector& dxi() { return dxi_; }
};

using KKTMatrix = std::vector<SplitKKTMatrix>;
using KKTResidual = std::vector<SplitKKTResidual>;
using RiccatiFactorization = std::vector<SplitRiccatiFactorization>;
using Direction = std::vector<SplitDirection>;

/// Drop-in for robotoc::RiccatiRecursion (riccati_recursion.hpp:26-119) for ONE OCP (batch = 1).  Batched callers use
/// the C ABI (or the Python mirror) directly.
class RiccatiRecursion {
 public:
  /// RiccatiRecursion(const OCP& ocp, double max_dts0) -- `dims` and `n_grid_max` (= N+1+reserved events) stand for the OCP.
  RiccatiRecursion(const rbt_dims& dims, int n_grid_max, double max_dts0 = 0.1, int device = 0)
      : dims_(dims), n_grid_max_(n_grid_max), max_dts0_(max_dts0) {
    if (max_dts0 <= 0) throw std::out_of_range("[RiccatiRecursion] invalid argument: 'max_dts0' must be positive!");
    rbt_make_layout(&dims_, &L_);
    const int rc = rbt_create(&dims_, n_grid_max, 1, device, &h_);
    if (rc != RBT_OK) {
      const std::string msg = h_ ? rbt_last_error(h_) : "unsupported robot dimensions";
      if (h_) rbt_destroy(h_);
      h_ = nullptr;
      throw std::runtime_error("[RiccatiRecursion] cannot create the device handle: " + msg);
    }
    lqr_policy_.assign(n_grid_max, LQRPolicy(dims_.nv, dims_.nu));
  }
  ~RiccatiRecursion() {
    if (h_) rbt_destroy(h_);
  }
  RiccatiRecursion(const RiccatiRecursion&) = delete;
  RiccatiRecursion& operator=(const RiccatiRecursion&) = delete;

  void setRegularization(double max_dts0) {  // riccati_recursion.hpp:58
    if (max_dts0 <= 0) throw std::out_of_range("[RiccatiRecursion] invalid argument: 'max_dts0' must be positive!");
    max_dts0_ = max_dts0;
  }

  /// Time-parallel sweeps (rbt_set_time_segments): 0 = automatic (default), 1 = serial, k > 1 = k segments of the horizon on
  /// separate CTAs.  Checked against the time discretization of every following sweep: k > 1 throws std::invalid_argument on
  /// a horizon with fewer than k stages or with switching-time optimisation.
  void setTimeSegments(int segments) {
    if (segments < 0) throw std::invalid_argument("[RiccatiRecursion] invalid argument: 'segments' must be non-negative!");
    segments_ = segments;
  }

  /// riccati_recursion.cpp:32-80.  kkt_matrix / kkt_residual are mutated like the reference (Qxx,Qxu,Quu,lu <- F,H,G,lu').
  void backwardRiccatiRecursion(const TimeDiscretization& td, KKTMatrix& kkt_matrix, KKTResidual& kkt_residual,
                                RiccatiFactorization& factorization) {
    const int n_grid = int(td.size());
    setSchedule(td);
    const int nx = L_.nx, nu = L_.nu, nv = L_.nv;
    kkt_.assign(size_t(n_grid) * L_.k_stride, 0.0);
    for (int i = 0; i < n_grid; ++i) {
      double* rec = kkt_.data() + size_t(i) * L_.k_stride;
      SplitKKTMatrix& km = kkt_matrix[i];
      SplitKKTResidual& kr = kkt_residual[i];
      put(rec + L_.k_Qxx, km.Qxx.data(), nx * nx);
      put(rec + L_.k_lx, kr.lx.data(), nx);
      if (td[i].type == GridType::Terminal) continue;
      put(rec + L_.k_Fxx, km.Fxx.data(), nx * nx);
      put(rec + L_.k_Fx, kr.Fx.data(), nx);
      if (td[i].type == GridType::Impact) continue;
      put(rec + L_.k_Fvu, km.Fvu.data(), nv * nu);
      put(rec + L_.k_Qxu, km.Qxu.data(), nx * nu);
      put(rec + L_.k_Quu, km.Quu.data(), nu * nu);
      put(rec + L_.k_lu, kr.lu.data(), nu);
      const int ns = ctrl_[i].ns;
      if (ns > 0) {
        put(rec + L_.k_Phix, km.Phix_.data(), ns * nx);
        put(rec + L_.k_Phiu, km.Phiu_.data(), ns * nu);
        put(rec + L_.k_p, kr.P_.data(), ns);
      }
      if (td[i].sto) {
        put(rec + L_.k_fx, km.fx.data(), nx);
        put(rec + L_.k_hx, km.hx.data(), nx);
        put(rec + L_.k_hu, km.hu.data(), nu);
        if (ns > 0) put(rec + L_.k_Phit, km.Phit_.data(), ns);
        rec[L_.k_sc + 0] = km.Qtt;
        rec[L_.k_sc + 1] = km.Qtt_prev;
        rec[L_.k_sc + 2] = kr.h;
      }
    }
    check(rbt_upload(h_, RBT_BUF_KKT, kkt_.data(), nullptr));
    check(rbt_riccati_backward(h_, /*write_fact=*/1, nullptr));
    ric_.resize(size_t(n_grid) * L_.r_stride);
    fact_.resize(size_t(n_grid) * L_.f_stride);
    check(rbt_download(h_, RBT_BUF_RIC, ric_.data(), nullptr));
    check(rbt_download(h_, RBT_BUF_FACT, fact_.data(), nullptr));
    check(rbt_sync(h_, nullptr));
    factorization.resize(n_grid);
    for (int i = 0; i < n_grid; ++i) {
      const double* r = ric_.data() + size_t(i) * L_.r_stride;
      SplitRiccatiFactorization& f = factorization[i];
      if (f.P.rows() != nx) f = SplitRiccatiFactorization(nv);
      get(f.P.data(), r + L_.r_P, nx * nx);
      get(f.s.data(), r + L_.r_s, nx);
      get(f.Psi.data(), r + L_.r_Psi, nx);
      get(f.Phi.data(), r + L_.r_Phi, nx);
      f.xi = r[L_.r_sc + 0]; f.chi = r[L_.r_sc + 1]; f.rho = r[L_.r_sc + 2]; f.eta = r[L_.r_sc + 3]; f.iota = r[L_.r_sc + 4];
      if (td[i].type == GridType::Terminal) continue;
      const double* fc = fact_.data() + size_t(i) * L_.f_stride;  // in-place mutation semantics of the reference
      get(kkt_matrix[i].Qxx.data(), fc + L_.f_F, nx * nx);        // (impact stages too: riccati_factorizer.cpp:178-186)
      if (td[i].type == GridType::Impact) continue;
      LQRPolicy& pol = lqr_policy_[i];
      get(pol.Kt.data(), r + L_.r_K, nx * nu);
      get(pol.k.data(), r + L_.r_k, nu);
      get(pol.T.data(), r + L_.r_T, nu);
      get(pol.W.data(), r + L_.r_W, nu);
      const int ns = ctrl_[i].ns;
      if (ns > 0) {
        f.M_ = Matrix(ns, nx);
        f.m_.assign(ns, 0.0);
        get(f.M_.data(), r + L_.r_M, ns * nx);
        get(f.m_.data(), r + L_.r_m, ns);
      }
      get(kkt_matrix[i].Qxu.data(), fc + L_.f_H, nx * nu);
      get(kkt_matrix[i].Quu.data(), fc + L_.f_G, nu * nu);
      get(kkt_residual[i].lu.data(), fc + L_.f_lu, nu);
    }
  }

  /// riccati_recursion.cpp:83-131; d[0].dx must hold the initial state direction.
  void forwardRiccatiRecursion(const TimeDiscretization& td, const KKTMatrix&, const KKTResidual&,
                               const RiccatiFactorization&, Direction& d) {
    const int n_grid = int(td.size());
    check(rbt_upload(h_, RBT_BUF_DX0, d[0].dx.data(), nullptr));
    check(rbt_riccati_forward(h_, nullptr));
    dir_.resize(size_t(n_grid) * L_.d_stride);
    check(rbt_download(h_, RBT_BUF_DIR, dir_.data(), nullptr));
    check(rbt_sync(h_, nullptr));
    for (int i = 0; i < n_grid; ++i) {
      const double* r = dir_.data() + size_t(i) * L_.d_stride;
      get(d[i].dx.data(), r + L_.d_dx, L_.nx);
      get(d[i].du.data(), r + L_.d_du, L_.nu);
      get(d[i].dlmdgmm.data(), r + L_.d_dlmdgmm, L_.nx);
      d[i].dts = r[L_.d_dts];
      d[i].dts_next = r[L_.d_dts + 1];
      if (ctrl_[i].ns > 0) {
        d[i].dxi_.assign(ctrl_[i].ns, 0.0);
        get(d[i].dxi_.data(), r + L_.d_dxi, ctrl_[i].ns);
      }
    }
  }

  const std::vector<LQRPolicy>& getLQRPolicy() const { return lqr_policy_; }  // riccati_recursion.hpp:104
  const rbt_layout& layout() const { return L_; }

 private:
  static void put(double* dst, const double* src, int n) { std::memcpy(dst, src, sizeof(double) * size_t(n)); }
  static void get(double* dst, const double* src, int n) { std::memcpy(dst, src, sizeof(double) * size_t(n)); }
  void check(int rc) {
    if (rc == RBT_OK) return;
    const std::string msg = rbt_last_error(h_);
    if (rc == RBT_ERR_ARG) throw std::invalid_argument("[RiccatiRecursion] invalid argument: " + msg);
    throw std::runtime_error("[RiccatiRecursion] " + msg);
  }
  void setSchedule(const TimeDiscretization& td) {
    if (int(td.size()) > n_grid_max_) throw std::out_of_range("[RiccatiRecursion] invalid argument: horizon longer than reserved");
    ctrl_.assign(td.size(), rbt_stage_ctrl());
    for (size_t i = 0; i < td.size(); ++i) {
      rbt_stage_ctrl& c = ctrl_[i];
      c.type = int(td[i].type);
      c.sto = td[i].sto;
      c.sto_next = td[i].sto_next;
      c.ns = td[i].switching_constraint ? td[i].dims : 0;
      c.nf = td[i].dimf;
      c.ngrids_in_phase = td[i].num_grids_in_phase;
      if (td[i].contact_mask < 0 && td[i].dimf > 0)
        throw std::invalid_argument("[RiccatiRecursion] invalid argument: GridInfo::contact_mask must be set when dimf > 0");
      c.contact_mask = td[i].contact_mask < 0 ? 0 : td[i].contact_mask;
      c.ineq_gate = td[i].stage < 0 ? 0 : (td[i].stage >= 2 ? 0 : 2 - td[i].stage);  // constraints_data.cpp:20-45
      c.dt = td[i].dt;
    }
    check(rbt_set_schedule(h_, ctrl_.data(), int(td.size()), max_dts0_));
    check(rbt_set_time_segments(h_, segments_));
  }

  rbt_dims dims_;
  rbt_layout L_;
  int n_grid_max_;
  double max_dts0_;
  int segments_ = 0;
  rbt_handle* h_ = nullptr;
  std::vector<rbt_stage_ctrl> ctrl_;
  std::vector<LQRPolicy> lqr_policy_;
  std::vector<double> kkt_, ric_, fact_, dir_;
};

}  // namespace robotoc_b200

// ---------------------------------------------------------------------------------------------------------------------
// robotoc_b200::DirectMultipleShooting -- the part of robotoc::DirectMultipleShooting that is on the hot path
// (include/robotoc/ocp/direct_multiple_shooting.hpp:86-199), over the stage-layer records of include/rbt_stage_layout.h.
// It shares the handle (and so the KKT / direction buffers on the device) of a RiccatiRecursion, exactly as the
// reference's OCPSolver owns both and passes kkt_matrix_ / d_ between them (src/solver/ocp_solver.cpp:118-144):
//
//   dms.evalKKT(lin, con);                 // condensing tail of evalKKT              direct_multiple_shooting.cpp:129-159
//   riccati.backwardRiccatiRecursion();    // on the device-resident KKT records
//   riccati.forwardRiccatiRecursion(dx0);
//   dms.computeStepSizes();                //                                         :174-199
//   dms.maxPrimalStepSize(); dms.maxDualStepSize();                                //  :202-209
//   dms.integrateSolution(sol, con);       //                                         :212-241
namespace robotoc_b200 {

class DeviceRiccatiRecursion {  // batch-of-one-or-more variant that keeps everything on the device between calls
 public:
  DeviceRiccatiRecursion(const rbt_dims& dims, const std::vector<rbt_stage_ctrl>& ctrl, int batch, double max_dts0 = 0.1,
                         int device = 0)
      : dims_(dims), n_grid_(int(ctrl.size())), batch_(batch) {
    if (max_dts0 <= 0) throw std::out_of_range("[RiccatiRecursion] invalid argument: 'max_dts0' must be positive!");
    if (rbt_create(&dims_, n_grid_, batch, device, &h_) != RBT_OK) {
      const std::string msg = h_ ? rbt_last_error(h_) : "unsupported robot dimensions";
      if (h_) rbt_destroy(h_);
      throw std::runtime_error("[RiccatiRecursion] cannot create the device handle: " + msg);
    }
    const int rc = rbt_set_schedule(h_, ctrl.data(), n_grid_, max_dts0);
    if (rc != RBT_OK) {  // the destructor does not run when a constructor throws: release the handle here
      const std::string msg = rbt_last_error(h_);
      rbt_destroy(h_);
      h_ = nullptr;
      if (rc == RBT_ERR_ARG) throw std::invalid_argument("[robotoc_b200] invalid argument: " + msg);
      throw std::runtime_error("[robotoc_b200] " + msg);
    }
  }
  ~DeviceRiccatiRecursion() { if (h_) rbt_destroy(h_); }
  DeviceRiccatiRecursion(const DeviceRiccatiRecursion&) = delete;
  DeviceRiccatiRecursion& operator=(const DeviceRiccatiRecursion&) = delete;
  void backwardRiccatiRecursion() { check(rbt_riccati_backward(h_, 0, nullptr)); }
  void forwardRiccatiRecursion(const std::vector<double>& dx0) {
    if (dx0.size() != size_t(batch_) * 2 * dims_.nv) throw std::invalid_argument("[RiccatiRecursion] invalid argument: dx0 size");
    check(rbt_upload(h_, RBT_BUF_DX0, dx0.data(), nullptr));
    check(rbt_riccati_forward(h_, nullptr));
  }
  std::vector<double> download(int which) {
    std::vector<double> out(size_t(rbt_buf_doubles(h_, which)));
    check(rbt_download(h_, which, out.data(), nullptr));
    check(rbt_sync(h_, nullptr));
    return out;
  }
  rbt_handle* handle() { return h_; }
  int batch() const { return batch_; }
  int n_grid() const { return n_grid_; }
  void check(int rc) {
    if (rc == RBT_OK) return;
    const std::string msg = rbt_last_error(h_);
    if (rc == RBT_ERR_ARG) throw std::invalid_argument("[robotoc_b200] invalid argument: " + msg);
    throw std::runtime_error("[robotoc_b200] " + msg);
  }

 private:
  rbt_dims dims_;
  int n_grid_, batch_;
  rbt_handle* h_ = nullptr;
};

class DirectMultipleShooting {
 public:
  DirectMultipleShooting(DeviceRiccatiRecursion& riccati, const rbt_stage_dims& sdims, const rbt_constraint_table& constraints)
      : rr_(riccati), sdims_(sdims) {
    rbt_make_stage_layout(&sdims_, &S_);
    rr_.check(rbt_stage_setup(rr_.handle(), &sdims_, &constraints));
  }
  /// The condensing tail of evalKKT for every stage of every OCP ("Forms linear system", intermediate_stage.cpp:133-148).
  void evalKKT(const std::vector<double>& lin, const std::vector<double>& con) {
    expect(lin, S_.l_stride, "lin");
    expect(con, S_.c_stride, "con");
    rr_.check(rbt_upload(rr_.handle(), RBT_BUF_LIN, lin.data(), nullptr));
    rr_.check(rbt_upload(rr_.handle(), RBT_BUF_CON, con.data(), nullptr));
    rr_.check(rbt_condense(rr_.handle(), nullptr));
  }
  void computeStepSizes() {
    rr_.check(rbt_expand_and_step_sizes(rr_.handle(), nullptr));
    steps_ = rr_.download(RBT_BUF_STEPS);
  }
  /// per OCP of the batch (the reference's scalar is entry 0 for batch 1)
  double maxPrimalStepSize(int ocp = 0) const { return steps_.at(2 * size_t(ocp)); }
  double maxDualStepSize(int ocp = 0) const { return steps_.at(2 * size_t(ocp) + 1); }
  /// integrateSolution with the step sizes computeStepSizes left on the device; `sol` is updated in place.
  void integrateSolution(std::vector<double>& sol) {
    expect(sol, S_.s_stride, "sol");
    rr_.check(rbt_upload(rr_.handle(), RBT_BUF_SOL, sol.data(), nullptr));
    rr_.check(rbt_update(rr_.handle(), nullptr));
    rr_.check(rbt_download(rr_.handle(), RBT_BUF_SOL, sol.data(), nullptr));
    rr_.check(rbt_sync(rr_.handle(), nullptr));
  }
  /// OCPSolver::KKTError() of every OCP (ocp_solver.cpp:429-431): the PerformanceIndex that evalKKT summarises before condensing
  /// (direct_multiple_shooting.cpp:155-158), from the records uploaded by evalKKT.  perf(ocp) = {cost (0: the cost evaluation is
  /// not on this path), cost_barrier, primal_feasibility, dual_feasibility, kkt_error, sqrt(kkt_error), 0, 0}.
  void evalPerformanceIndex() {
    rr_.check(rbt_eval_kkt(rr_.handle(), nullptr));
    perf_ = rr_.download(RBT_BUF_PERF);
  }
  double KKTError(int ocp = 0) const { return perf_.at(8 * size_t(ocp) + 5); }
  const double* performanceIndex(int ocp = 0) const { return perf_.data() + 8 * size_t(ocp); }
  /// pdipm::setSlackAndDualPositive on the uploaded PDIPM records (Constraints::setSlackAndDual at initConstraints); `con` is
  /// uploaded, adjusted on the device and read back.
  void setSlackAndDualPositive(std::vector<double>& con) {
    expect(con, S_.c_stride, "con");
    rr_.check(rbt_upload(rr_.handle(), RBT_BUF_CON, con.data(), nullptr));
    rr_.check(rbt_set_slack_and_dual_positive(rr_.handle(), nullptr));
    rr_.check(rbt_download(rr_.handle(), RBT_BUF_CON, con.data(), nullptr));
    rr_.check(rbt_sync(rr_.handle(), nullptr));
  }
  /// computeInitialStateDirection (state_equation.cpp:98-109): dq0_v0 = [batch][2 nv] = {q0 (-) s[0].q, v0}; call after evalKKT
  /// (and with the solution uploaded, e.g. by a previous integrateSolution) and before forwardRiccatiRecursion.
  void computeInitialStateDirection(const std::vector<double>& dq0_v0) {
    if (dq0_v0.size() != size_t(rr_.batch()) * 2 * S_.nv) throw std::invalid_argument("[DirectMultipleShooting] invalid argument: size of 'dq0_v0'");
    rr_.check(rbt_initial_state_direction(rr_.handle(), dq0_v0.data(), nullptr));
  }
  /// The robot model of the inverse-dynamics linearisation (rbt_robot_model, filled from pinocchio::Model; INTEGRATION.md 5b).
  void setRobotModel(const rbt_robot_model& model) { rr_.check(rbt_set_robot_model(rr_.handle(), &model)); }
  /// The inverse-dynamics rows of linearizeContactDynamics / linearizeImpactDynamics on the device (rbt_linearize_inverse_dynamics):
  /// `lin` (records without the ID rows and without the beta terms of the gradients) and `sol` are uploaded, `lin` is read back
  /// with IDC / dIDCdqv ID rows, M and the beta terms filled in.
  void linearizeInverseDynamics(std::vector<double>& lin, const std::vector<double>& sol) {
    expect(lin, S_.l_stride, "lin");
    expect(sol, S_.s_stride, "sol");
    rr_.check(rbt_upload(rr_.handle(), RBT_BUF_LIN, lin.data(), nullptr));
    rr_.check(rbt_upload(rr_.handle(), RBT_BUF_SOL, sol.data(), nullptr));
    rr_.check(rbt_linearize_inverse_dynamics(rr_.handle(), nullptr));
    rr_.check(rbt_download(rr_.handle(), RBT_BUF_LIN, lin.data(), nullptr));
    rr_.check(rbt_sync(rr_.handle(), nullptr));
  }
  /// Baumgarte gains of the point contacts, [n_contacts][2] = {baumgarte_position_gain, baumgarte_velocity_gain} of
  /// ContactModelInfo (rbt_set_contact_gains; INTEGRATION.md 5b).
  void setContactGains(const std::vector<double>& gains) {
    if (gains.size() != size_t(2) * sdims_.n_contacts)
      throw std::invalid_argument("[DirectMultipleShooting] invalid argument: gains must hold 2 values per contact");
    rr_.check(rbt_set_contact_gains(rr_.handle(), gains.data()));
  }
  /// Desired contact positions [batch][n_grid][n_contacts][3] (ContactStatus::contactPosition of each grid point's phase),
  /// uploaded to RBT_BUF_CONTACT_POS; they stay on the device until the next call.
  void setContactPositions(const std::vector<double>& pos) {
    if (pos.size() != size_t(rr_.batch()) * rr_.n_grid() * sdims_.n_contacts * 3)
      throw std::invalid_argument("[DirectMultipleShooting] invalid argument: contact positions must be [batch][n_grid][n_contacts][3]");
    rr_.check(rbt_upload(rr_.handle(), RBT_BUF_CONTACT_POS, pos.data(), nullptr));
    rr_.check(rbt_sync(rr_.handle(), nullptr));
  }
  /// The contact rows of linearizeContactDynamics / linearizeImpactDynamics on the device (rbt_linearize_contact_kinematics):
  /// `lin` and `sol` are uploaded, `lin` is read back with J, the contact rows of dIDCdqv / IDC and the multiplier terms of the
  /// gradients filled in.
  void linearizeContactKinematics(std::vector<double>& lin, const std::vector<double>& sol) {
    expect(lin, S_.l_stride, "lin");
    expect(sol, S_.s_stride, "sol");
    rr_.check(rbt_upload(rr_.handle(), RBT_BUF_LIN, lin.data(), nullptr));
    rr_.check(rbt_upload(rr_.handle(), RBT_BUF_SOL, sol.data(), nullptr));
    rr_.check(rbt_linearize_contact_kinematics(rr_.handle(), nullptr));
    rr_.check(rbt_download(rr_.handle(), RBT_BUF_LIN, lin.data(), nullptr));
    rr_.check(rbt_sync(rr_.handle(), nullptr));
  }
  /// The measured configuration q0 [batch][nq] of OCPSolver::solve(t, q, v), uploaded to RBT_BUF_Q0: grid point 0's q_prev in
  /// linearizeStateEquation and the device-side state-equation rows of the wire paths.  It stays on the device until the next call.
  void setInitialConfiguration(const std::vector<double>& q0) {
    if (q0.size() != size_t(rr_.batch()) * S_.nq)
      throw std::invalid_argument("[DirectMultipleShooting] invalid argument: q0 must be [batch][nq]");
    rr_.check(rbt_upload(rr_.handle(), RBT_BUF_Q0, q0.data(), nullptr));
    rr_.check(rbt_sync(rr_.handle(), nullptr));
  }
  /// The state-equation rows of linearizeStateEquation / linearizeImpactStateEquation / linearizeTerminalStateEquation on the
  /// device (rbt_linearize_state_equation): `lin` and `sol` are uploaded, `lin` is read back with Fx, the SE(3) blocks, the
  /// costate terms of the gradients and, on schedules with a switching-time stage, the STO terms filled in.
  void linearizeStateEquation(std::vector<double>& lin, const std::vector<double>& sol) {
    expect(lin, S_.l_stride, "lin");
    expect(sol, S_.s_stride, "sol");
    rr_.check(rbt_upload(rr_.handle(), RBT_BUF_LIN, lin.data(), nullptr));
    rr_.check(rbt_upload(rr_.handle(), RBT_BUF_SOL, sol.data(), nullptr));
    rr_.check(rbt_linearize_state_equation(rr_.handle(), nullptr));
    rr_.check(rbt_download(rr_.handle(), RBT_BUF_LIN, lin.data(), nullptr));
    rr_.check(rbt_sync(rr_.handle(), nullptr));
  }
  /// Host wire records of the schedule in force (rbt_stage_layout.h): what an adaptor sends instead of the dense records.
  /// device_inverse_dynamics: the records leave M and the ID rows of dIDCdqv / IDC to the device (RBT_WIRE_DEVICE_ID).
  /// device_contact_kinematics: the records leave J and the contact rows of dIDCdqv / IDC to the device (RBT_WIRE_DEVICE_CONTACT).
  /// device_state_equation: the records leave Fx and the SE(3) blocks to the device (RBT_WIRE_DEVICE_STATE).
  void setWireCostStructure(bool robotoc_costs, bool device_inverse_dynamics = false, bool device_contact_kinematics = false,
                            bool device_state_equation = false) {
    cost_structure_ = (robotoc_costs ? RBT_COST_ROBOTOC : RBT_COST_GENERAL) | (device_inverse_dynamics ? RBT_WIRE_DEVICE_ID : 0) |
                      (device_contact_kinematics ? RBT_WIRE_DEVICE_CONTACT : 0) | (device_state_equation ? RBT_WIRE_DEVICE_STATE : 0);
    rr_.check(rbt_set_wire_cost_structure(rr_.handle(), cost_structure_));
  }
  std::vector<double> packWire(const std::vector<double>& lin, const std::vector<rbt_stage_ctrl>& ctrl) const {
    expect(lin, S_.l_stride, "lin");
    const int w = rbt_wire_doubles(&sdims_, ctrl.data(), int(ctrl.size()), cost_structure_);
    std::vector<double> wire(size_t(rr_.batch()) * w);
    rr_.check(rbt_pack_wire(&sdims_, ctrl.data(), int(ctrl.size()), cost_structure_, lin.data(), wire.data(), rr_.batch()));
    return wire;
  }
  /// Uploads the solver state (solution, slack / dual) that rbt_iteration_host_resident keeps on the device between iterations.
  void setState(const std::vector<double>& sol, const std::vector<double>& con) {
    expect(sol, S_.s_stride, "sol");
    expect(con, S_.c_stride, "con");
    rr_.check(rbt_upload(rr_.handle(), RBT_BUF_SOL, sol.data(), nullptr));
    rr_.check(rbt_upload(rr_.handle(), RBT_BUF_CON, con.data(), nullptr));
  }
  /// One iteration from host memory with the solver state resident on the device: wire records, PDIPM residuals [batch][n_grid][ncp]
  /// and dx0 in; updated solution records, slack | dual [batch][n_grid][2 ncp] and the step sizes out.
  void iterationHostResident(const std::vector<double>& wire, const std::vector<double>& lin_switching, const std::vector<double>& res,
                             const std::vector<double>& dx0, std::vector<double>& sol_out, std::vector<double>& slack_dual_out) {
    expect(res, S_.ncp, "res");
    sol_out.resize(size_t(rr_.batch()) * rr_.n_grid() * S_.s_stride);
    slack_dual_out.resize(size_t(rr_.batch()) * rr_.n_grid() * 2 * S_.ncp);
    steps_.resize(2 * size_t(rr_.batch()));
    rr_.check(rbt_iteration_host_resident(rr_.handle(), wire.data(), lin_switching.empty() ? nullptr : lin_switching.data(), res.data(),
                                          dx0.data(), sol_out.data(), slack_dual_out.data(), steps_.data(), nullptr));
    rr_.check(rbt_sync(rr_.handle(), nullptr));
  }
  const rbt_stage_layout& layout() const { return S_; }

 private:
  void expect(const std::vector<double>& a, int stride, const char* what) const {
    if (a.size() != size_t(rr_.batch()) * rr_.n_grid() * stride)
      throw std::invalid_argument(std::string("[DirectMultipleShooting] invalid argument: size of '") + what + "'");
  }
  DeviceRiccatiRecursion& rr_;
  rbt_stage_dims sdims_;
  rbt_stage_layout S_;
  std::vector<double> steps_, perf_;
  int cost_structure_ = RBT_COST_GENERAL;
};

}  // namespace robotoc_b200
