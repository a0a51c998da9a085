// rnea_kernels.cuh -- the inverse-dynamics rows of the contact / impact dynamics linearisation (SURVEY.md 8f-1, first slice):
//   linearize_inverse_dynamics_kernel   linearizeContactDynamics / linearizeImpactDynamics, their RNEA part
//       (src/dynamics/contact_dynamics.cpp:22-44, impact_dynamics.cpp:17-35; Robot::RNEA / RNEADerivatives / RNEAImpact /
//        RNEAImpactDerivatives, include/robotoc/robot/robot.hxx:494-622; pinocchio::rnea with external forces)
//
// Spatial algebra in Pinocchio's conventions (spatial.cuh).  The derivatives are forward-mode directional derivatives of RNEA,
// one lane per tangent direction: 18 in q (q (+) eps e_k = integrate(q, eps e_k): a perturbation of joint j right-multiplies
// its liMi by exp(eps S e_k)), 18 in v and 18 in a.  The primal pass (velocities, accelerations, body forces) runs once per grid
// point and is shared through shared memory.  One CTA of 64 threads per grid point.
#pragma once
#include "spatial.cuh"
#include "stage_kernels.cuh"  // StageParams

namespace rbt {

template <int NV>
struct RneaCfg {
  static constexpr int NB = NV - 5;  // free flyer + one revolute joint per remaining velocity
  static constexpr int NDIR = 3 * NV;
  static constexpr int NTHR = 64;
};

// One CTA per (OCP, grid point).  Shared: joint transforms and the primal v_i, a_i, f_i (f_i = total body force after the
// children's forces were added), then the NDIR directional derivatives of tau.
template <int NV>
__global__ void __launch_bounds__(64) linearize_inverse_dynamics_kernel(const StageParams p, const RneaModel* __restrict__ gm) {
  using C = RneaCfg<NV>;
  constexpr int NB = C::NB, NDIR = C::NDIR;
  __shared__ RneaModel m;
  __shared__ double sR[NB][9], sp[NB][3], sv[NB][6], sa[NB][6], sf[NB][6], sfx[NB][6];
  __shared__ double sq[NV + 1], sqd[NV], sqdd[NV], sbeta[NV], stau[NV];
  __shared__ double sout[NDIR][NV];
  const rbt_stage_layout& S = p.S;
  const int tid = threadIdx.x;
  const size_t st = blockIdx.x;
  const rbt_stage_ctrl c = p.ctrl[int(st % p.n_grid)];
  if (c.type == RBT_TERMINAL) return;
  const bool impact = c.type == RBT_IMPACT;
  {
    const double* g = reinterpret_cast<const double*>(gm);
    double* d = reinterpret_cast<double*>(&m);
    for (int e = tid; e < int(sizeof(RneaModel) / 8); e += C::NTHR) d[e] = g[e];
  }
  const double* sol = p.sol + st * S.s_stride;
  for (int e = tid; e < NV + 1; e += C::NTHR) sq[e] = sol[S.s_q + e];
  for (int e = tid; e < NV; e += C::NTHR) {
    sqd[e] = impact ? 0.0 : sol[S.s_v + e];
    sqdd[e] = sol[(impact ? S.s_dv : S.s_a) + e];
    sbeta[e] = sol[S.s_beta + e];
  }
  __syncthreads();
  // joint placements liMi = placement * M_J(q), one body per thread; external forces of the contacts
  if (tid < NB) {
    joint_placement(m, sq, tid, sR[tid], sp[tid]);
    for (int r = 0; r < 6; ++r) sfx[tid][r] = 0.0;
  }
  __syncthreads();
  if (tid == 0) {
    // Robot::setContactForces / setImpactForces: fjoint[parent] = jXf.act(Force(f, 0)), zero for an inactive contact, in
    // contact order (a later contact on the same parent overwrites, as the reference's assignment does)
    int k = 0;
    for (int ci = 0; ci < m.ncon; ++ci) {
      double* fx = sfx[m.cparent[ci]];
      if ((c.contact_mask >> ci) & 1) {
        const double f3[3] = {sol[S.s_f + k], sol[S.s_f + k + 1], sol[S.s_f + k + 2]};
        k += 3;
        rot_mul(m.cR[ci], f3, fx);
        cross3(m.cp[ci], fx, fx + 3);
      } else {
        for (int r = 0; r < 6; ++r) fx[r] = 0.0;
      }
    }
    // primal RNEA: forward pass
    for (int b = 0; b < NB; ++b) {
      const int pa = m.parent[b];
      if (pa < 0) {  // root: the parent's velocity is zero and its acceleration -g (impact: no gravity)
        const double zero[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
        double ag[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
        if (!impact) { ag[0] = -m.gravity[0]; ag[1] = -m.gravity[1]; ag[2] = -m.gravity[2]; }
        forward_step(m, b, sR[b], sp[b], sqd, sqdd, zero, ag, sv[b], sa[b]);
      } else {
        forward_step(m, b, sR[b], sp[b], sqd, sqdd, sv[pa], sa[pa], sv[b], sa[b]);
      }
      // f_i = I a_i + v_i x* (I v_i) - fext_i
      double Iv[6], f[6];
      inertia_mul(m.mass[b], m.com[b], m.Ic[b], sv[b], Iv);
      inertia_mul(m.mass[b], m.com[b], m.Ic[b], sa[b], f);
      force_cross_add(sv[b], Iv, f);
      for (int r = 0; r < 6; ++r) sf[b][r] = f[r] - sfx[b][r];
    }
    // backward pass: tau_i = S^T f_i, f_parent += liMi f_i
    for (int b = NB - 1; b >= 0; --b) {
      if (b == 0) { for (int r = 0; r < 6; ++r) stau[r] = sf[0][r]; }
      else stau[b + 5] = m.axis[b][0] * sf[b][3] + m.axis[b][1] * sf[b][4] + m.axis[b][2] * sf[b][5];
      const int pa = m.parent[b];
      if (pa >= 0) {
        double t[6];
        force_act(sR[b], sp[b], sf[b], t);
        for (int r = 0; r < 6; ++r) sf[pa][r] += t[r];
      }
    }
  }
  __syncthreads();
  // directional derivatives: lane d < NV: e_d in q, < 2 NV: in v, < 3 NV: in a
  if (tid < NDIR) {
    const int kind = tid / NV, k = tid % NV, jb = k < 6 ? 0 : k - 5;
    // s = column k of S, stored by index rather than by joint_s's selects: with the selects this kernel took 6.51 instead of
    // 6.20 ms per launch (H100 80GB HBM3, 700 W, ANYmal trot N=40, batch 1024)
    double s[6];
    for (int r = 0; r < 6; ++r) s[r] = 0.0;
    if (jb == 0) s[k] = 1.0;
    else { s[3] = m.axis[jb][0]; s[4] = m.axis[jb][1]; s[5] = m.axis[jb][2]; }
    double dv[NB][6], da[NB][6], df[NB][6];
    for (int b = 0; b < NB; ++b) {
      const int pa = m.parent[b];
      double w[6];
      for (int r = 0; r < 6; ++r) { dv[b][r] = 0.0; da[b][r] = 0.0; }
      if (pa >= 0) {
        motion_act_inv(sR[b], sp[b], dv[pa], dv[b]);
        motion_act_inv(sR[b], sp[b], da[pa], da[b]);
      }
      double vJ[6];
      joint_motion(m, b, sqd, vJ);
      const bool here = (b == jb);
      if (here && kind == 0) {  // d/deps exp(-eps s) X^-1 m = (X^-1 m) x s, for m = v_parent and a_parent
        if (pa >= 0) { motion_act_inv(sR[b], sp[b], sv[pa], w); motion_cross_add(w, s, dv[b]); }
        double ag[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
        if (pa < 0 && !impact) { ag[0] = -m.gravity[0]; ag[1] = -m.gravity[1]; ag[2] = -m.gravity[2]; }
        motion_act_inv(sR[b], sp[b], pa >= 0 ? sa[pa] : ag, w);
        motion_cross_add(w, s, da[b]);
      }
      if (here && kind == 1)
        for (int r = 0; r < 6; ++r) dv[b][r] += s[r];
      if (here && kind == 2)
        for (int r = 0; r < 6; ++r) da[b][r] += s[r];
      motion_cross_add(dv[b], vJ, da[b]);
      if (here && kind == 1) motion_cross_add(sv[b], s, da[b]);
      double Iv[6], Idv[6];
      inertia_mul(m.mass[b], m.com[b], m.Ic[b], da[b], df[b]);
      inertia_mul(m.mass[b], m.com[b], m.Ic[b], sv[b], Iv);
      inertia_mul(m.mass[b], m.com[b], m.Ic[b], dv[b], Idv);
      force_cross_add(dv[b], Iv, df[b]);
      force_cross_add(sv[b], Idv, df[b]);
    }
    double* out = sout[tid];
    for (int b = NB - 1; b >= 0; --b) {
      if (b == 0) { for (int r = 0; r < 6; ++r) out[r] = df[0][r]; }
      else out[b + 5] = m.axis[b][0] * df[b][3] + m.axis[b][1] * df[b][4] + m.axis[b][2] * df[b][5];
      const int pa = m.parent[b];
      if (pa >= 0) {
        double t[6];
        if (b == jb && kind == 0) force_cross_add(s, sf[b], df[b]);  // d/deps X exp(eps s) f = X (s x* f)
        force_act(sR[b], sp[b], df[b], t);
        for (int r = 0; r < 6; ++r) df[pa][r] += t[r];
      }
    }
  }
  __syncthreads();
  // outputs: IDC rows, [dIDdq | dIDdv] rows, M (upper triangle mirrored), and the beta terms of the gradients
  double* l = const_cast<double*>(p.lin) + st * S.l_stride;
  const int nvf = S.nvf;
  for (int e = tid; e < NV; e += C::NTHR)
    l[S.l_IDC + e] = (!impact && e >= 6) ? stau[e] - sol[S.s_u + e - 6] : stau[e];
  for (int e = tid; e < NV * 2 * NV; e += C::NTHR) {
    const int r = e % NV, col = e / NV;
    l[S.l_D + r + col * nvf] = (impact && col >= NV) ? 0.0 : sout[col][r];
  }
  for (int e = tid; e < NV * NV; e += C::NTHR) {
    const int r = e % NV, col = e / NV;
    l[S.l_M + r + col * NV] = r <= col ? sout[2 * NV + col][r] : sout[2 * NV + r][col];
  }
  if (tid < 3 * NV) {
    const int kind = tid / NV, k = tid % NV;
    double acc = 0.0;
    if (kind < 2) {
      for (int r = 0; r < NV; ++r) acc = fma(sout[tid][r], sbeta[r], acc);
    } else {
      for (int r = 0; r < NV; ++r) acc = fma(r <= k ? sout[2 * NV + k][r] : sout[2 * NV + r][k], sbeta[r], acc);
    }
    if (kind == 0) l[S.l_lx + k] += acc;
    else if (kind == 1) { if (!impact) l[S.l_lx + NV + k] += acc; }
    else l[S.l_la + k] += acc;
  }
}

}  // namespace rbt
