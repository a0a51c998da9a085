// contact_kernels.cuh -- the contact rows of the contact / impact dynamics linearisation (SURVEY.md 8f-1, second slice):
//   linearize_contact_kinematics_kernel   linearizeContactDynamics / linearizeImpactDynamics, their contact part
//       (src/dynamics/contact_dynamics.cpp:12-52, impact_dynamics.cpp:8-35; Robot::computeBaumgarteResidual / Derivatives,
//        computeImpactVelocityResidual / Derivatives, include/robotoc/robot/robot.hxx:291-360; PointContact,
//        include/robotoc/robot/point_contact.hxx:16-117)
//
// Kinematics without gravity (pinocchio::forwardKinematics): body velocities and classical accelerations at (q, v, a) on
// Intermediate / Lift grid points, velocities at (q, v + dv) on Impact grid points.  Per active point contact c, with v_f, a_f
// the LOCAL spatial velocity / acceleration of the contact frame and oMf its world placement:
//   Intermediate / Lift:  C_c = a_f,lin + w_f x v_f,lin + kv v_f,lin + kp (oMf.p - p_des,c)
//   Impact:               C_c = v_f,lin
// and their derivatives, forward mode: one lane per (active contact, tangent direction k) carries the q- and the v-tangent of
// the velocity and acceleration along the contact's chain from the joint of direction k to the contact's parent body, in
// registers (q (+) eps e_k = integrate(q, eps e_k), as in rnea_kernels.cuh).  The v-tangent of v_f,lin is the column k of the
// contact Jacobian J_lin, which is also dC/da on Intermediate / Lift and dC/dv on Impact grid points.
#pragma once
#include "spatial.cuh"
#include "stage_kernels.cuh"  // StageParams

namespace rbt {

template <int NV>
struct ContactCfg {
  static constexpr int NB = NV - 5;
  static constexpr int NTHR = 96;  // >= 3 NV + 3 RBT_MAX_CONTACTS: the gradient lanes of the last phase
  static constexpr int NFM = 3 * RBT_MAX_CONTACTS;
};

// One CTA per (OCP, grid point).  Phase 1: joint placements (one body per lane) and the chain of every active contact.
// Phase 2: one lane per active contact walks its chain: v, a (no gravity) and the world placement, then the contact frame and
// C.  Phase 3: one lane per (active contact, direction k) walks the chain from the joint of k: q- and v-tangents in registers.
// Phase 4: the rows, stacked in contact order, and the multiplier terms of the gradients.
template <int NV>
__global__ void __launch_bounds__(ContactCfg<NV>::NTHR)
    linearize_contact_kinematics_kernel(const StageParams p, const RneaModel* __restrict__ gm, const double* __restrict__ gains,
                                        const double* __restrict__ cpos) {
  using C = ContactCfg<NV>;
  constexpr int NB = C::NB, NFM = C::NFM, NT = C::NTHR;
  __shared__ double sR[NB][9], sp[NB][3], sq[NV + 1], sqd[NV], sqdd[NV], sbeta[NV], smu[NFM];
  __shared__ double sv[RBT_MAX_CONTACTS][NB][6], sa[RBT_MAX_CONTACTS][NB][6];  // along each active contact's chain
  __shared__ double svf[RBT_MAX_CONTACTS][6], soRf[RBT_MAX_CONTACTS][9];       // contact frame: LOCAL velocity, world rotation
  __shared__ double sJ[NFM][NV], sDq[NFM][NV], sDv[NFM][NV], sC[NFM];
  __shared__ int schain[RBT_MAX_CONTACTS][NB], sdepth[RBT_MAX_CONTACTS], sct[RBT_MAX_CONTACTS];
  const rbt_stage_layout& S = p.S;
  const int tid = threadIdx.x;
  const size_t st = blockIdx.x;
  const rbt_stage_ctrl c = p.ctrl[int(st % p.n_grid)];
  if (c.type == RBT_TERMINAL || c.nf == 0) return;
  const bool impact = c.type == RBT_IMPACT;
  const int nf = c.nf, nact = nf / 3;
  const RneaModel& m = *gm;
  const double* sol = p.sol + st * S.s_stride;
  for (int e = tid; e < NV + 1; e += NT) sq[e] = sol[S.s_q + e];
  for (int e = tid; e < NV; e += NT) {
    sqd[e] = impact ? sol[S.s_v + e] + sol[S.s_dv + e] : sol[S.s_v + e];
    sqdd[e] = impact ? 0.0 : sol[S.s_a + e];
    sbeta[e] = sol[S.s_beta + e];
  }
  for (int e = tid; e < nf; e += NT) smu[e] = sol[S.s_mu + e];
  if (tid < nact) {  // slot tid: the tid-th active contact, and its chain root .. parent body
    int ci = -1;
    for (int k = 0; k <= tid; ++k) ci = __ffs(c.contact_mask & ~((1 << (ci + 1)) - 1)) - 1;
    sct[tid] = ci;
    int d = 0;
    for (int b = m.cparent[ci]; b >= 0; b = m.parent[b]) ++d;
    sdepth[tid] = d;
    for (int b = m.cparent[ci]; b >= 0; b = m.parent[b]) schain[tid][--d] = b;
  }
  __syncthreads();
  for (int b = tid; b < NB; b += NT) joint_placement(m, sq, b, sR[b], sp[b]);
  __syncthreads();
  if (tid < nact) {
    const int a = tid, ci = sct[a], depth = sdepth[a];
    double v[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0}, acc[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    double oR[9] = {1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0}, op[3] = {0.0, 0.0, 0.0};
    for (int j = 0; j < depth; ++j) {
      const int b = schain[a][j];
      double t[3];
      forward_step(m, b, sR[b], sp[b], sqd, sqdd, v, acc, v, acc);
      for (int r = 0; r < 6; ++r) { sv[a][j][r] = v[r]; sa[a][j][r] = acc[r]; }
      // oMi = oMparent * liMi
      rot_mul(oR, sp[b], t);
      for (int r = 0; r < 3; ++r) op[r] += t[r];
      double Rn[9];
      for (int k = 0; k < 3; ++k) rot_mul(oR, &sR[b][3 * k], Rn + 3 * k);
      for (int r = 0; r < 9; ++r) oR[r] = Rn[r];
    }
    // contact frame: v_f = fXi^-1 v, a_f = fXi^-1 a, oMf = oMi * jXf
    const double* cR = m.cR[ci];
    double vf[6], af[6], t[3];
    motion_act_inv(cR, m.cp[ci], v, vf);
    motion_act_inv(cR, m.cp[ci], acc, af);
    rot_mul(oR, m.cp[ci], t);
    for (int r = 0; r < 3; ++r) op[r] += t[r];
    for (int k = 0; k < 3; ++k) rot_mul(oR, cR + 3 * k, &soRf[a][3 * k]);
    for (int r = 0; r < 6; ++r) svf[a][r] = vf[r];
    if (impact) {
      for (int r = 0; r < 3; ++r) sC[3 * a + r] = vf[r];
    } else {
      const double kp = gains[2 * ci], kv = gains[2 * ci + 1];
      const double* pd = cpos + (st * S.ncon + ci) * 3;
      cross3(vf + 3, vf, t);
      for (int r = 0; r < 3; ++r) sC[3 * a + r] = af[r] + t[r] + kv * vf[r] + kp * (op[r] - pd[r]);
    }
  }
  __syncthreads();
  // tangents: lane (slot a, direction k); zero columns for joints off the chain
  for (int e = tid; e < nact * NV; e += NT) {
    const int a = e / NV, k = e % NV, jb = k < 6 ? 0 : k - 5, ci = sct[a], depth = sdepth[a];
    int pos = -1;
    for (int j = 0; j < depth; ++j) pos = schain[a][j] == jb ? j : pos;
    double dq[3] = {0.0, 0.0, 0.0}, dv[3] = {0.0, 0.0, 0.0}, Jl[3] = {0.0, 0.0, 0.0};
    if (pos >= 0) {
      double s[6], vJ[6], w[6];
      double tvq[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0}, taq[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
      double tvv[6], tav[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
      joint_s(m, jb, k, s);
      joint_motion(m, jb, sqd, vJ);
      if (pos > 0) {  // d/deps exp(-eps s) X^-1 m = (X^-1 m) x s, for m = v_parent and a_parent (the root's are zero)
        motion_act_inv(sR[jb], sp[jb], sv[a][pos - 1], w);
        motion_cross_add(w, s, tvq);
        motion_act_inv(sR[jb], sp[jb], sa[a][pos - 1], w);
        motion_cross_add(w, s, taq);
      }
      motion_cross_add(tvq, vJ, taq);
      for (int r = 0; r < 6; ++r) tvv[r] = s[r];
      motion_cross_add(s, vJ, tav);
      motion_cross_add(sv[a][pos], s, tav);
      for (int j = pos + 1; j < depth; ++j) {
        const int b = schain[a][j];
        joint_motion(m, b, sqd, vJ);
        motion_act_inv(sR[b], sp[b], tvq, w);
        for (int r = 0; r < 6; ++r) tvq[r] = w[r];
        motion_act_inv(sR[b], sp[b], taq, w);
        motion_cross_add(tvq, vJ, w);
        for (int r = 0; r < 6; ++r) taq[r] = w[r];
        motion_act_inv(sR[b], sp[b], tvv, w);
        for (int r = 0; r < 6; ++r) tvv[r] = w[r];
        motion_act_inv(sR[b], sp[b], tav, w);
        motion_cross_add(tvv, vJ, w);
        for (int r = 0; r < 6; ++r) tav[r] = w[r];
      }
      const double* cR = m.cR[ci];
      double fvq[6], fvv[6];
      motion_act_inv(cR, m.cp[ci], tvq, fvq);
      motion_act_inv(cR, m.cp[ci], tvv, fvv);
      for (int r = 0; r < 3; ++r) Jl[r] = fvv[r];
      if (impact) {
        for (int r = 0; r < 3; ++r) { dq[r] = fvq[r]; dv[r] = fvv[r]; }
      } else {
        // dC = da_f,lin + w_f x dv_f,lin + dw_f x v_f,lin + kv dv_f,lin (+ kp oRf J_lin for a q-direction)
        const double kp = gains[2 * ci], kv = gains[2 * ci + 1];
        const double* vf = svf[a];
        double faq[6], fav[6], t1[3], t2[3], t3[3];
        motion_act_inv(cR, m.cp[ci], taq, faq);
        motion_act_inv(cR, m.cp[ci], tav, fav);
        rot_mul(soRf[a], Jl, t3);
        cross3(vf + 3, fvq, t1);
        cross3(fvq + 3, vf, t2);
        for (int r = 0; r < 3; ++r) dq[r] = faq[r] + t1[r] + t2[r] + kv * fvq[r] + kp * t3[r];
        cross3(vf + 3, fvv, t1);
        cross3(fvv + 3, vf, t2);
        for (int r = 0; r < 3; ++r) dv[r] = fav[r] + t1[r] + t2[r] + kv * fvv[r];
      }
    }
    for (int r = 0; r < 3; ++r) { sJ[3 * a + r][k] = Jl[r]; sDq[3 * a + r][k] = dq[r]; sDv[3 * a + r][k] = dv[r]; }
  }
  __syncthreads();
  // outputs: J (ld nfm), the contact rows of dIDCdqv (ld nvf) and IDC; lf -= J beta, lq += dCdq^T mu, lv += dCdv^T mu,
  // la (impact: ldv) += J^T mu
  double* l = const_cast<double*>(p.lin) + st * S.l_stride;
  const int nvf = S.nvf, nfm = S.nfm;
  for (int e = tid; e < nf * NV; e += NT) {
    const int r = e % nf, col = e / nf;
    l[S.l_J + r + col * nfm] = sJ[r][col];
    l[S.l_D + NV + r + col * nvf] = sDq[r][col];
    l[S.l_D + NV + r + (NV + col) * nvf] = sDv[r][col];
  }
  if (tid < 3 * NV) {
    const int kind = tid / NV, k = tid % NV;
    const double(*src)[NV] = kind == 0 ? sDq : (kind == 1 ? sDv : sJ);
    double acc = 0.0;
    for (int r = 0; r < nf; ++r) acc = fma(src[r][k], smu[r], acc);
    l[(kind == 2 ? S.l_la : S.l_lx + kind * NV) + k] += acc;
  } else if (tid < 3 * NV + nf) {
    const int r = tid - 3 * NV;
    double acc = 0.0;
    for (int k = 0; k < NV; ++k) acc = fma(sJ[r][k], sbeta[k], acc);
    l[S.l_IDC + NV + r] = sC[r];
    l[S.l_lf + r] -= acc;
  }
}

}  // namespace rbt
