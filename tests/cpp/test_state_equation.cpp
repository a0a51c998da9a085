// C++ drop-in test of the device state-equation rows: robotoc_b200::DirectMultipleShooting::setInitialConfiguration /
// linearizeStateEquation and the resident wire path with the inverse dynamics, the contact rows and the state equation left to
// the device.
//   argv[1]: an rbt_robot_model as raw bytes; argv[2]: a directory for ctrl.bin, sol.bin, q0.bin, lin_in.bin, lin_out.bin, which
//   the calling test compares with the numpy restatement tests/state_ref.py.
// Checks here: linearizeStateEquation before setInitialConfiguration throws std::runtime_error (RBT_ERR_STATE), a q0 of the wrong
// size throws std::invalid_argument; the resident wire path with RBT_WIRE_DEVICE_ID | RBT_WIRE_DEVICE_CONTACT |
// RBT_WIRE_DEVICE_STATE reproduces, bit for bit, linearizeInverseDynamics -> linearizeContactKinematics -> linearizeStateEquation
// -> evalKKT -> backward -> forward -> step sizes -> integrateSolution, and its wire records are 144 doubles per non-terminal and
// 36 per terminal grid point smaller than with the first two bits.
#include <cmath>
#include <cstdio>
#include <stdexcept>
#include <string>
#include <vector>

#include "robotoc_b200/riccati_recursion.hpp"

using namespace robotoc_b200;

static unsigned long long g_state = 93ULL;
static double urand() {
  g_state = g_state * 6364136223846793005ULL + 1442695040888963407ULL;
  return double((g_state >> 11) & ((1ULL << 53) - 1)) / double(1ULL << 52) - 1.0;
}
static double pos() { return 0.01 + 0.495 * (urand() + 1.0); }

template <class T>
static bool dump(const std::string& path, const T* p, size_t n) {
  FILE* f = std::fopen(path.c_str(), "wb");
  if (!f) return false;
  const bool ok = std::fwrite(p, sizeof(T), n, f) == n;
  return std::fclose(f) == 0 && ok;
}

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  rbt_robot_model model;
  FILE* mf = std::fopen(argv[1], "rb");
  if (!mf || std::fread(&model, sizeof(model), 1, mf) != 1) return 2;
  std::fclose(mf);
  const std::string out = argv[2];

  const int nv = 18, nu = 12, nx = 36, batch = 2, n_grid = 7;
  rbt_dims dims = {nv, nu, 12, 6};
  rbt_constraint_table tab = {};
  tab.n_contacts = 4; tab.barrier = 1e-3; tab.fraction_to_boundary = 0.995;
  int r = 0;
  const int vars[3] = {RBT_VAR_Q, RBT_VAR_V, RBT_VAR_U}, offs[3] = {6, 6, 0};
  for (int v = 0; v < 3; ++v)
    for (int sgn = -1; sgn <= 1; sgn += 2)
      for (int j = 0; j < 12; ++j) { tab.box[r].var = vars[v]; tab.box[r].idx = offs[v] + j; tab.box[r].sign = sgn; ++r; }
  tab.n_box = r;
  rbt_stage_dims sd = {nv, nu, 6, 12, 12, 4, tab.n_box};
  rbt_stage_layout S; rbt_make_stage_layout(&sd, &S);
  // Intermediate grid points with four, two and no contacts, an impact of one foot, and the terminal grid point
  const int types[n_grid] = {RBT_INTERMEDIATE, RBT_INTERMEDIATE, RBT_IMPACT, RBT_INTERMEDIATE, RBT_INTERMEDIATE, RBT_INTERMEDIATE,
                             RBT_TERMINAL};
  const int masks[n_grid] = {0xF, 0x5, 0x2, 0x7, 0x0, 0xF, 0xF};
  std::vector<rbt_stage_ctrl> ctrl(n_grid);
  for (int i = 0; i < n_grid; ++i) {
    ctrl[i] = rbt_stage_ctrl();
    ctrl[i].type = types[i];
    ctrl[i].contact_mask = masks[i];
    int nf = 0;
    for (int c = 0; c < 4; ++c) nf += 3 * ((masks[i] >> c) & 1);
    ctrl[i].nf = nf; ctrl[i].ngrids_in_phase = 1; ctrl[i].dt = (types[i] == RBT_TERMINAL || types[i] == RBT_IMPACT) ? 0.0 : 0.05;
  }
  const size_t per = size_t(batch) * n_grid;
  std::vector<double> lin(per * S.l_stride, 0.0), con(per * S.c_stride, 0.0), sol(per * S.s_stride, 0.0), dx0(size_t(batch) * nx);
  auto putspd = [&](double* dst, int n, int ld, double diag, double sc) {
    std::vector<double> t(size_t(n) * n);
    for (auto& x : t) x = urand();
    for (int j = 0; j < n; ++j)
      for (int i = 0; i < n; ++i) {
        double acc = (i == j) ? diag : 0.0;
        for (int k = 0; k < n; ++k) acc += sc * t[i + size_t(k) * n] * t[j + size_t(k) * n];
        dst[i + size_t(j) * ld] = acc;
      }
    for (int j = 0; j < n; ++j)
      for (int i = j + 1; i < n; ++i) dst[i + size_t(j) * ld] = dst[j + size_t(i) * ld];
  };
  for (size_t o = 0; o < per; ++o) {
    const rbt_stage_ctrl& c = ctrl[o % n_grid];
    const int nf = c.nf;
    const bool impact = c.type == RBT_IMPACT;
    double* rec = lin.data() + o * S.l_stride;
    putspd(rec + S.l_Qxx, nx, nx, 1.0, 1.0 / nx);
    for (int i = 0; i < nx; ++i) rec[S.l_lx + i] = urand();
    for (int k = 0; k < 3; ++k)
      for (int j = 0; j < 6; ++j)
        for (int i = 0; i < 6; ++i) {
          double v = 0.0;
          if ((i < 3) == (j < 3)) v = ((i == j) ? 1.0 : 0.0) + 0.1 * urand();
          else if (i < 3) v = 0.1 * urand();
          rec[S.l_se3 + 36 * k + i + 6 * j] = (k == 0) ? -v : v;
        }
    double* s = sol.data() + o * S.s_stride;
    // neighbouring configurations a few degrees and centimetres apart, as along a trajectory
    for (int i = 0; i < S.nq; ++i) s[S.s_q + i] = (i == 6 ? 1.0 : 0.0) + 0.05 * urand();
    double nrm = 0; for (int i = 3; i < 7; ++i) nrm += s[S.s_q + i] * s[S.s_q + i];
    for (int i = 3; i < 7; ++i) s[S.s_q + i] /= std::sqrt(nrm);
    for (int i = 0; i < nv; ++i) {
      s[S.s_v + i] = urand(); s[S.s_a + i] = urand(); s[S.s_dv + i] = urand(); s[S.s_lmd + i] = urand(); s[S.s_gmm + i] = urand();
      s[S.s_beta + i] = urand();
    }
    for (int i = 0; i < nu; ++i) s[S.s_u + i] = urand();
    for (int i = 0; i < 12; ++i) { s[S.s_f + i] = 20.0 * urand(); s[S.s_mu + i] = urand(); }
    for (int i = 0; i < 6; ++i) s[S.s_nup + i] = urand();
    if (c.type == RBT_TERMINAL) continue;
    // the ID and contact rows are left as noise: the device overwrites them
    for (int j = 0; j < nv; ++j) for (int i = 0; i < nf; ++i) rec[S.l_J + i + 12 * j] = urand();
    for (int j = 0; j < nx; ++j) for (int i = 0; i < S.nvf; ++i) rec[S.l_D + i + S.nvf * j] = 0.5 * urand();
    if (impact)  // dCdv of an impact is the contact Jacobian (impact_dynamics.cpp:40)
      for (int j = 0; j < nv; ++j) for (int i = 0; i < nf; ++i) rec[S.l_D + nv + i + S.nvf * (nv + j)] = rec[S.l_J + i + 12 * j];
    for (int i = 0; i < S.nvf; ++i) rec[S.l_IDC + i] = 0.5 * urand();
    for (int i = 0; i < nv * nv; ++i) rec[S.l_M + i] = urand();
    for (int i = 0; i < nv; ++i) { rec[S.l_Qaa + i] = pos(); rec[S.l_la + i] = urand(); }
    for (int i = 0; i < nf; ++i) { rec[S.l_Qff + i + 12 * i] = 1e-3; rec[S.l_lf + i] = urand(); }
    for (int i = 0; i < nx; ++i) rec[S.l_Fx + i] = 0.1 * urand();
    if (impact) continue;
    putspd(rec + S.l_Quu, nu, nu, 0.1, 1.0 / nu);
    for (int i = 0; i < nu; ++i) rec[S.l_lu + i] = urand();
    for (int i = 0; i < 6; ++i) rec[S.l_lup + i] = urand();
    rec[S.l_sc + 1] = 1.0;
    for (int ci = 0; ci < 4; ++ci) {
      if (!((c.contact_mask >> ci) & 1)) continue;
      for (int e = 0; e < 5 * nv; ++e) rec[S.l_dgdq + ci * 5 * nv + e] = 0.3 * urand();
      for (int e = 0; e < 15; ++e) rec[S.l_dgdf + ci * 15 + e] = urand();
    }
    double* c_ = con.data() + o * S.c_stride;
    for (int i = 0; i < S.nc; ++i) { c_[S.c_slack + i] = pos(); c_[S.c_dual + i] = pos(); c_[S.c_res + i] = 0.1 * urand(); }
  }
  for (auto& x : dx0) x = 0.1 * urand();

  std::vector<double> q0(size_t(batch) * S.nq);
  for (int b = 0; b < batch; ++b) {
    for (int i = 0; i < S.nq; ++i) q0[b * S.nq + i] = sol[size_t(b) * n_grid * S.s_stride + S.s_q + i] + 0.01 * urand();
    double nrm = 0; for (int i = 3; i < 7; ++i) nrm += q0[b * S.nq + i] * q0[b * S.nq + i];
    for (int i = 3; i < 7; ++i) q0[b * S.nq + i] /= std::sqrt(nrm);
  }
  std::vector<double> gains(8), pos(per * 4 * 3);
  for (int c = 0; c < 4; ++c) { gains[2 * c] = 30.0 + 5.0 * c; gains[2 * c + 1] = 8.0 + 2.0 * c; }
  for (auto& x : pos) x = urand();

  DeviceRiccatiRecursion riccati_recursion(dims, ctrl, batch, 0.1);
  DirectMultipleShooting dms(riccati_recursion, sd, tab);
  dms.setRobotModel(model);
  dms.setContactGains(gains);
  dms.setContactPositions(pos);
  bool threw = false;
  std::vector<double> lin_d = lin;
  try { dms.linearizeStateEquation(lin_d, sol); } catch (const std::runtime_error&) { threw = true; }
  if (!threw) { std::printf("linearizeStateEquation before setInitialConfiguration did not throw\n"); return 3; }
  threw = false;
  try { dms.setInitialConfiguration(std::vector<double>(q0.size() - 1)); } catch (const std::invalid_argument&) { threw = true; }
  if (!threw) { std::printf("a q0 of the wrong size was accepted\n"); return 3; }
  dms.setInitialConfiguration(q0);
  lin_d = lin;
  dms.linearizeStateEquation(lin_d, sol);
  if (!dump(out + "/ctrl.bin", ctrl.data(), ctrl.size()) || !dump(out + "/sol.bin", sol.data(), sol.size()) ||
      !dump(out + "/q0.bin", q0.data(), q0.size()) || !dump(out + "/lin_in.bin", lin.data(), lin.size()) ||
      !dump(out + "/lin_out.bin", lin_d.data(), lin_d.size()))
    return 2;

  // step by step: ID, contact and state-equation rows from the device, then the iteration
  const std::vector<double> sol_in = sol, con_in = con;
  lin_d = lin;
  dms.linearizeInverseDynamics(lin_d, sol);
  dms.linearizeContactKinematics(lin_d, sol);
  dms.linearizeStateEquation(lin_d, sol);
  dms.evalKKT(lin_d, con);
  riccati_recursion.backwardRiccatiRecursion();
  riccati_recursion.forwardRiccatiRecursion(dx0);
  dms.computeStepSizes();
  std::vector<double> steps(2 * batch);
  for (int b = 0; b < batch; ++b) { steps[2 * b] = dms.maxPrimalStepSize(b); steps[2 * b + 1] = dms.maxDualStepSize(b); }
  dms.integrateSolution(sol);

  // resident wire path, the ID, contact and state-equation rows left to the device
  std::vector<double> sol_r, sd_r, res(per * S.ncp, 0.0);
  for (size_t o = 0; o < per; ++o)
    for (int i = 0; i < S.ncp; ++i) res[o * S.ncp + i] = con_in[o * S.c_stride + S.c_res + i];
  dms.setWireCostStructure(false, true, true);
  const size_t id_contact = dms.packWire(lin, ctrl).size();
  dms.setWireCostStructure(false, true, true, true);
  const std::vector<double> wire = dms.packWire(lin, ctrl);
  dms.setState(sol_in, con_in);
  dms.iterationHostResident(wire, std::vector<double>(), res, dx0, sol_r, sd_r);
  const int used = S.s_xi + S.nsm;
  bool same = true, finite = true;
  for (size_t o = 0; o < per; ++o)
    for (int i = 0; i < used; ++i) {
      same = same && (sol_r[o * S.s_stride + i] == sol[o * S.s_stride + i]);
      finite = finite && std::isfinite(sol[o * S.s_stride + i]);
    }
  for (int b = 0; b < batch; ++b)
    same = same && dms.maxPrimalStepSize(b) == steps[2 * b] && dms.maxDualStepSize(b) == steps[2 * b + 1];
  const size_t drop = size_t(batch) * (144 * (n_grid - 1) + 36);
  std::printf("resident wire path with device ID, contact and state-equation rows %s the step-by-step path (%zu vs %zu wire "
              "doubles per batch)\n", same ? "reproduces" : "DIFFERS FROM", wire.size(), id_contact);
  return (same && finite && id_contact - wire.size() == drop) ? 0 : 1;
}
