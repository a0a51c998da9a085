// state_kernels.cuh -- the state-equation rows of the linearisation (SURVEY.md 8f-1, third slice):
//   linearize_state_equation_kernel   linearizeStateEquation (src/dynamics/state_equation.cpp:30-65),
//       linearizeImpactStateEquation (impact_state_equation.cpp:26-54), linearizeTerminalStateEquation
//       (terminal_state_equation.cpp:8-28), and the third SE(3) block of correctLinearizeStateEquation (state_equation.cpp:78)
//
// With M(q) the free-flyer placement of q, Sub(qf, q0) = Robot::subtractConfiguration = log6(M(q0)^-1 M(qf)) on the base,
// qf - q0 on the joints (robot.hxx:97-139), q_prev = q0 (the measured configuration, RBT_BUF_Q0) on grid point 0 and
// s[i-1].q otherwise (direct_multiple_shooting.cpp:129-159):
//   Intermediate / Lift: Fq = Sub(q, q_next) + dt v,  Fv = v + dt a - v_next
//   Impact:              Fq = Sub(q, q_next),         Fv = v + dv - v_next
//   l_se3 blocks:        Fqq = dSub/dqf(q, q_next) = Jlog6(M),  Fqq_prev = dSub/dq0(q_prev, q),  Fqq_cur = dSub/dq0(q, q_next)
//   costate terms:       lq[0:6] += Fqq^T lmd_next[0:6] + Fqq_prev^T lmd[0:6],  lq[6:] += lmd_next[6:] - lmd[6:],
//                        lv += dt lmd_next + gmm_next - gmm (impact: no dt),  la += dt gmm_next (impact: ldv += gmm_next)
//   STO terms (schedules with a switching-time stage, Intermediate / Lift only):
//                        h += lmd_next . v + gmm_next . a,  hv += lmd_next,  ha += gmm_next,  fq = v,  fv = a
//   Terminal:            Fqq_prev,  lq[0:6] += Fqq_prev^T lmd[0:6],  lq[6:] -= lmd[6:],  lv -= gmm
// The SE(3) log, Jlog6 and Ad live next to the free-flyer exponential in spatial.cuh.
#pragma once
#include "spatial.cuh"
#include "stage_kernels.cuh"  // StageParams

namespace rbt {

struct StateCfg {
  static constexpr int NW = 4;  // grid points (one warp each) per CTA
};

// One warp per (OCP, grid point), no CTA barrier.  Lane 0 takes M = M(q_next)^-1 M(q) (Fq head, Fqq, Fqq_cur), lane 1
// M = M(q)^-1 M(q_prev) (Fqq_prev): log6, Jlog6 and Ad(M^-1) into shared memory.  Then the lanes form the three 6x6 blocks
// (entries of -Jlog6 Ad(M^-1)) and lane k < NV the rows of direction k; h is a warp sum.  Each OCP's grid points lie in one
// batch window, so the neighbours s[i-1], s[i+1] are records of the same window.
template <int NV>
__global__ void __launch_bounds__(32 * StateCfg::NW)
    linearize_state_equation_kernel(const StageParams p, const double* __restrict__ q0, int with_sto) {
  constexpr int NW = StateCfg::NW, NQ = NV + 1;
  static_assert(NV <= 32, "one lane per row");
  __shared__ double sJ[NW][2][36], sAd[NW][2][36], sF[NW][3][36], sxi[NW][6];
  const rbt_stage_layout& S = p.S;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const size_t st = size_t(blockIdx.x) * NW + wid;
  if (st >= size_t(p.batch) * p.n_grid) return;  // the whole warp
  const int i = int(st % p.n_grid);
  const rbt_stage_ctrl c = p.ctrl[i];
  const bool terminal = c.type == RBT_TERMINAL, impact = c.type == RBT_IMPACT;
  const double* s = p.sol + st * S.s_stride;
  const double* sn = s + S.s_stride;  // read on non-terminal grid points only
  const double* q_prev = i == 0 ? q0 + (st / p.n_grid) * NQ : s - S.s_stride + S.s_q;
  double* l = const_cast<double*>(p.lin) + st * S.l_stride;
  if (lane < 2 && (lane == 1 || !terminal)) {
    double xi[6], R[9], pt[3], coef[3];
    se3_log6_dev(lane == 0 ? sn + S.s_q : s + S.s_q, lane == 0 ? s + S.s_q : q_prev, xi, R, pt, coef);
    se3_jlog6_dev(xi, pt, coef, sJ[wid][lane]);
    se3_ad_inv_dev(R, pt, sAd[wid][lane]);
    if (lane == 0)
      for (int r = 0; r < 6; ++r) sxi[wid][r] = xi[r];
  }
  __syncwarp();
  // block 0: Fqq = J_0; block 1: Fqq_prev = -J_1 Ad_1; block 2: Fqq_cur = -J_0 Ad_0 (column-major)
  for (int e = lane; e < 108; e += 32) {
    const int k = e / 36, ij = e % 36, r = ij % 6, col = ij / 6, m = k == 1 ? 1 : 0;
    if (terminal && k != 1) continue;
    double v = sJ[wid][0][ij];
    if (k != 0) {
      double acc = 0.0;
      for (int t = 0; t < 6; ++t) acc = fma(sJ[wid][m][r + 6 * t], sAd[wid][m][t + 6 * col], acc);
      v = -acc;
    }
    sF[wid][k][ij] = v;
    l[S.l_se3 + e] = v;
  }
  __syncwarp();
  double hsum = 0.0;
  if (lane < NV) {
    const int k = lane;
    const double lmd = s[S.s_lmd + k], gmm = s[S.s_gmm + k];
    double lq_add = 0.0;
    if (k < 6)
      for (int r = 0; r < 6; ++r) lq_add = fma(sF[wid][1][r + 6 * k], s[S.s_lmd + r], lq_add);
    if (terminal) {
      l[S.l_lx + k] += k < 6 ? lq_add : -lmd;
      l[S.l_lx + NV + k] -= gmm;
    } else {
      const double lmd_n = sn[S.s_lmd + k], gmm_n = sn[S.s_gmm + k], v = s[S.s_v + k], v_n = sn[S.s_v + k];
      double Fq = k < 6 ? sxi[wid][k] : s[S.s_q + k + 1] - sn[S.s_q + k + 1], Fv;
      if (impact) {
        Fv = v + s[S.s_dv + k] - v_n;
      } else {
        Fq += c.dt * v;
        Fv = v + c.dt * s[S.s_a + k] - v_n;
      }
      l[S.l_Fx + k] = Fq;
      l[S.l_Fx + NV + k] = Fv;
      if (k < 6) {
        double acc = 0.0;
        for (int r = 0; r < 6; ++r) acc = fma(sF[wid][0][r + 6 * k], sn[S.s_lmd + r], acc);
        lq_add += acc;
      } else {
        lq_add = lmd_n - lmd;
      }
      l[S.l_lx + k] += lq_add;
      if (impact) {
        l[S.l_lx + NV + k] += gmm_n - gmm;
        l[S.l_la + k] += gmm_n;
      } else {
        const double a = s[S.s_a + k];
        l[S.l_lx + NV + k] += c.dt * lmd_n + gmm_n - gmm;
        l[S.l_la + k] += c.dt * gmm_n;
        if (with_sto) {
          hsum = lmd_n * v + gmm_n * a;
          l[S.l_hx + NV + k] += lmd_n;
          l[S.l_ha + k] += gmm_n;
          l[S.l_fx + k] = v;
          l[S.l_fx + NV + k] = a;
        }
      }
    }
  }
  if (with_sto && !terminal && !impact) {  // warp-uniform
    for (int o = 16; o > 0; o >>= 1) hsum += __shfl_xor_sync(0xffffffffu, hsum, o);
    if (lane == 0) l[S.l_sc] += hsum;
  }
}

}  // namespace rbt
