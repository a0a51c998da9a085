// rnea_kernels.cuh -- the inverse-dynamics rows of the contact / impact dynamics linearisation (SURVEY.md 8f-1, first slice):
//   linearize_inverse_dynamics_kernel   linearizeContactDynamics / linearizeImpactDynamics, their RNEA part
//       (src/dynamics/contact_dynamics.cpp:22-44, impact_dynamics.cpp:17-35; Robot::RNEA / RNEADerivatives / RNEAImpact /
//        RNEAImpactDerivatives, include/robotoc/robot/robot.hxx:494-622; pinocchio::rnea with external forces)
//
// Spatial algebra in Pinocchio's conventions: motion = [linear | angular], force = [linear | angular], every body quantity in
// its joint frame, liMi = jointPlacement * M_J(q).  The derivatives are forward-mode directional derivatives of RNEA, one lane
// per tangent direction: 18 in q (q (+) eps e_k = integrate(q, eps e_k): a perturbation of joint j right-multiplies its liMi by
// exp(eps S e_k)), 18 in v and 18 in a.  The primal pass (velocities, accelerations, body forces) runs once per grid point and
// is shared through shared memory.  One CTA of 64 threads per grid point.
#pragma once
#include "stage_kernels.cuh"

namespace rbt {

struct RneaModel {  // device copy of rbt_robot_model, as the kernel reads it
  int nb, ncon;
  int parent[RBT_MAX_BODIES];
  double axis[RBT_MAX_BODIES][3];
  double R[RBT_MAX_BODIES][9], p[RBT_MAX_BODIES][3];
  double mass[RBT_MAX_BODIES], com[RBT_MAX_BODIES][3], Ic[RBT_MAX_BODIES][9];
  int cparent[RBT_MAX_CONTACTS];
  double cR[RBT_MAX_CONTACTS][9], cp[RBT_MAX_CONTACTS][3];
  double gravity[3];
};

// ---- spatial algebra (6-vectors [lin | ang]; R column-major)
__device__ __forceinline__ void rot_mul(const double* R, const double* x, double* y) {  // y = R x
  y[0] = R[0] * x[0] + R[3] * x[1] + R[6] * x[2];
  y[1] = R[1] * x[0] + R[4] * x[1] + R[7] * x[2];
  y[2] = R[2] * x[0] + R[5] * x[1] + R[8] * x[2];
}
__device__ __forceinline__ void rot_tmul(const double* R, const double* x, double* y) {  // y = R^T x
  y[0] = R[0] * x[0] + R[1] * x[1] + R[2] * x[2];
  y[1] = R[3] * x[0] + R[4] * x[1] + R[5] * x[2];
  y[2] = R[6] * x[0] + R[7] * x[1] + R[8] * x[2];
}
__device__ __forceinline__ void cross3(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}
// m' = X^-1 m for X = (R, p) (SE3::actInv on a motion): w' = R^T w, v' = R^T (v - p x w)
__device__ __forceinline__ void motion_act_inv(const double* R, const double* p, const double* m, double* out) {
  double t[3], u[3];
  cross3(p, m + 3, t);
  u[0] = m[0] - t[0]; u[1] = m[1] - t[1]; u[2] = m[2] - t[2];
  rot_tmul(R, u, out);
  rot_tmul(R, m + 3, out + 3);
}
// f' = X f (SE3::act on a force): n' = R n + p x (R f)
__device__ __forceinline__ void force_act(const double* R, const double* p, const double* f, double* out) {
  double t[3];
  rot_mul(R, f, out);
  rot_mul(R, f + 3, out + 3);
  cross3(p, out, t);
  out[3] += t[0]; out[4] += t[1]; out[5] += t[2];
}
// out += a x m  (motion cross motion): [w x v_m + v x w_m | w x w_m]
__device__ __forceinline__ void motion_cross_add(const double* a, const double* m, double* out) {
  double t[3];
  cross3(a + 3, m, t); out[0] += t[0]; out[1] += t[1]; out[2] += t[2];
  cross3(a, m + 3, t); out[0] += t[0]; out[1] += t[1]; out[2] += t[2];
  cross3(a + 3, m + 3, t); out[3] += t[0]; out[4] += t[1]; out[5] += t[2];
}
// out += a x* f  (motion cross force): [w x f | w x n + v x f]
__device__ __forceinline__ void force_cross_add(const double* a, const double* f, double* out) {
  double t[3];
  cross3(a + 3, f, t); out[0] += t[0]; out[1] += t[1]; out[2] += t[2];
  cross3(a + 3, f + 3, t); out[3] += t[0]; out[4] += t[1]; out[5] += t[2];
  cross3(a, f, t); out[3] += t[0]; out[4] += t[1]; out[5] += t[2];
}
// f = I m for the spatial inertia (mass, com c, Ic about c): f_lin = mass (v - c x w), f_ang = Ic w + c x f_lin
__device__ __forceinline__ void inertia_mul(double mass, const double* c, const double* Ic, const double* m, double* f) {
  double t[3];
  cross3(c, m + 3, t);
  f[0] = mass * (m[0] - t[0]); f[1] = mass * (m[1] - t[1]); f[2] = mass * (m[2] - t[2]);
  rot_mul(Ic, m + 3, f + 3);
  cross3(c, f, t);
  f[3] += t[0]; f[4] += t[1]; f[5] += t[2];
}
// joint motion subspace column k of body b: the free flyer's S is the identity, a revolute joint's is [0 | axis]
__device__ __forceinline__ void joint_s(const RneaModel& m, int b, int k, double* s) {
  for (int r = 0; r < 6; ++r) s[r] = 0.0;
  if (b == 0) s[k] = 1.0;
  else { s[3] = m.axis[b][0]; s[4] = m.axis[b][1]; s[5] = m.axis[b][2]; }
}

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
    const int b = tid;
    double RJ[9], pJ[3] = {0.0, 0.0, 0.0};
    if (b == 0) {  // free flyer: q = [p | x y z w]
      const double x = sq[3], y = sq[4], z = sq[5], w = sq[6];
      RJ[0] = 1 - 2 * (y * y + z * z); RJ[3] = 2 * (x * y - z * w);     RJ[6] = 2 * (x * z + y * w);
      RJ[1] = 2 * (x * y + z * w);     RJ[4] = 1 - 2 * (x * x + z * z); RJ[7] = 2 * (y * z - x * w);
      RJ[2] = 2 * (x * z - y * w);     RJ[5] = 2 * (y * z + x * w);     RJ[8] = 1 - 2 * (x * x + y * y);
      pJ[0] = sq[0]; pJ[1] = sq[1]; pJ[2] = sq[2];
    } else {  // revolute about the unit axis u: Rodrigues
      const double th = sq[b + 6];  // q of body b >= 1 sits after the 7 free-flyer entries
      double sn, cs;
      sincos(th, &sn, &cs);
      const double ux = m.axis[b][0], uy = m.axis[b][1], uz = m.axis[b][2], t = 1.0 - cs;
      RJ[0] = cs + ux * ux * t;      RJ[3] = ux * uy * t - uz * sn; RJ[6] = ux * uz * t + uy * sn;
      RJ[1] = uy * ux * t + uz * sn; RJ[4] = cs + uy * uy * t;      RJ[7] = uy * uz * t - ux * sn;
      RJ[2] = uz * ux * t - uy * sn; RJ[5] = uz * uy * t + ux * sn; RJ[8] = cs + uz * uz * t;
    }
    const double* RP = m.R[b];
    for (int j = 0; j < 3; ++j) rot_mul(RP, RJ + 3 * j, &sR[b][3 * j]);
    rot_mul(RP, pJ, sp[b]);
    for (int r = 0; r < 3; ++r) sp[b][r] += m.p[b][r];
    for (int r = 0; r < 6; ++r) sfx[b][r] = 0.0;
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
      double vJ[6], s[6];
      if (b == 0) { for (int r = 0; r < 6; ++r) vJ[r] = sqd[r]; }
      else { joint_s(m, b, 0, s); for (int r = 0; r < 6; ++r) vJ[r] = s[r] * sqd[b + 5]; }
      double w[6], ag[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
      if (pa < 0) {
        for (int r = 0; r < 6; ++r) sv[b][r] = vJ[r];
        if (!impact) { ag[0] = -m.gravity[0]; ag[1] = -m.gravity[1]; ag[2] = -m.gravity[2]; }
        motion_act_inv(sR[b], sp[b], ag, w);
      } else {
        motion_act_inv(sR[b], sp[b], sv[pa], w);
        for (int r = 0; r < 6; ++r) sv[b][r] = w[r] + vJ[r];
        motion_act_inv(sR[b], sp[b], sa[pa], w);
      }
      // a_i = X^-1 a_p + S qdd + v_i x vJ
      if (b == 0) { for (int r = 0; r < 6; ++r) w[r] += sqdd[r]; }
      else { for (int r = 0; r < 6; ++r) w[r] += s[r] * sqdd[b + 5]; }
      motion_cross_add(sv[b], vJ, w);
      for (int r = 0; r < 6; ++r) sa[b][r] = w[r];
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
    double s[6];
    joint_s(m, jb, k < 6 ? k : 0, s);
    double dv[NB][6], da[NB][6], df[NB][6];
    for (int b = 0; b < NB; ++b) {
      const int pa = m.parent[b];
      double w[6];
      for (int r = 0; r < 6; ++r) { dv[b][r] = 0.0; da[b][r] = 0.0; }
      if (pa >= 0) {
        motion_act_inv(sR[b], sp[b], dv[pa], dv[b]);
        motion_act_inv(sR[b], sp[b], da[pa], da[b]);
      }
      double vJ[6], sb[6];
      if (b == 0) { for (int r = 0; r < 6; ++r) vJ[r] = sqd[r]; }
      else { joint_s(m, b, 0, sb); for (int r = 0; r < 6; ++r) vJ[r] = sb[r] * sqd[b + 5]; }
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
