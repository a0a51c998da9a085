// spatial.cuh -- rigid-body and SE(3) math of the device kernels, in Pinocchio's conventions:
//   q = [p | quaternion x y z w | revolute joints], motion = [linear | angular], force = [linear | angular], R column-major,
//   every body quantity in its joint frame, liMi = jointPlacement * M_J(q).
// The joint and spatial-algebra helpers serve the inverse-dynamics and contact rows; the free-flyer exponential, log, Jlog6,
// Ad(M^-1) and SE3JacobianInverse serve the condensing, the update, the line search and the state-equation rows.
#pragma once
#include "../../include/robotoc_b200.h"  // RBT_MAX_BODIES, RBT_MAX_CONTACTS

namespace rbt {

struct RneaModel {  // device copy of rbt_robot_model, as the kernels read it
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

// rotation of the unit quaternion (x, y, z, w): R = I + 2 w [v]x + 2 [v]x^2, v = (x, y, z)
__device__ __forceinline__ void quat_to_rot(double x, double y, double z, double w, double* R) {
  R[0] = 1.0 - 2.0 * (y * y + z * z); R[3] = 2.0 * (x * y - z * w);       R[6] = 2.0 * (x * z + y * w);
  R[1] = 2.0 * (x * y + z * w);       R[4] = 1.0 - 2.0 * (x * x + z * z); R[7] = 2.0 * (y * z - x * w);
  R[2] = 2.0 * (x * z - y * w);       R[5] = 2.0 * (y * z + x * w);       R[8] = 1.0 - 2.0 * (x * x + y * y);
}

// ---- joints: body 0 is the free flyer (q[0..6], qd[0..5]), body b >= 1 a revolute joint (q[b + 6], qd[b + 5])
// liMi = placement * M_J(q) of body b
__device__ __forceinline__ void joint_placement(const RneaModel& m, const double* q, int b, double* R, double* p) {
  double RJ[9], pJ[3] = {0.0, 0.0, 0.0};
  if (b == 0) {  // free flyer: q = [p | x y z w]
    quat_to_rot(q[3], q[4], q[5], q[6], RJ);
    pJ[0] = q[0]; pJ[1] = q[1]; pJ[2] = q[2];
  } else {  // revolute about the unit axis u: Rodrigues
    double sn, cs;
    sincos(q[b + 6], &sn, &cs);
    const double ux = m.axis[b][0], uy = m.axis[b][1], uz = m.axis[b][2], t = 1.0 - cs;
    RJ[0] = cs + ux * ux * t;      RJ[3] = ux * uy * t - uz * sn; RJ[6] = ux * uz * t + uy * sn;
    RJ[1] = uy * ux * t + uz * sn; RJ[4] = cs + uy * uy * t;      RJ[7] = uy * uz * t - ux * sn;
    RJ[2] = uz * ux * t - uy * sn; RJ[5] = uz * uy * t + ux * sn; RJ[8] = cs + uz * uz * t;
  }
  const double* RP = m.R[b];
  for (int j = 0; j < 3; ++j) rot_mul(RP, RJ + 3 * j, R + 3 * j);
  rot_mul(RP, pJ, p);
  for (int r = 0; r < 3; ++r) p[r] += m.p[b][r];
}
// joint motion subspace column k of body b: the free flyer's S is the identity, a revolute joint's is [0 | axis].  Every entry
// is selected rather than indexed, so s stays in registers.
__device__ __forceinline__ void joint_s(const RneaModel& m, int b, int k, double* s) {
  for (int r = 0; r < 6; ++r) s[r] = b == 0 ? (r == k ? 1.0 : 0.0) : (r < 3 ? 0.0 : m.axis[b][r - 3]);
}
// joint velocity S qd of body b
__device__ __forceinline__ void joint_motion(const RneaModel& m, int b, const double* qd, double* vJ) {
  if (b == 0) { for (int r = 0; r < 6; ++r) vJ[r] = qd[r]; }
  else { for (int r = 0; r < 3; ++r) { vJ[r] = 0.0; vJ[3 + r] = m.axis[b][r] * qd[b + 5]; } }
}
// One step of the forward recursion for body b with liMi = (R, p), from its parent's velocity vp and acceleration ap (the
// root's parent: zero, with -g in the acceleration where gravity acts):
//   v = liMi^-1 vp + vJ,  a = liMi^-1 ap + S qdd + v x vJ,  vJ = S qd.
// v and a may be vp and ap.
__device__ __forceinline__ void forward_step(const RneaModel& m, int b, const double* R, const double* p, const double* qd,
                                             const double* qdd, const double* vp, const double* ap, double* v, double* a) {
  double vJ[6], w[6];
  joint_motion(m, b, qd, vJ);
  motion_act_inv(R, p, vp, w);
  for (int r = 0; r < 6; ++r) v[r] = w[r] + vJ[r];
  motion_act_inv(R, p, ap, w);
  if (b == 0) { for (int r = 0; r < 6; ++r) w[r] += qdd[r]; }
  else { for (int r = 0; r < 3; ++r) w[3 + r] += m.axis[b][r] * qdd[b + 5]; }
  motion_cross_add(v, vJ, w);
  for (int r = 0; r < 6; ++r) a[r] = w[r];
}

// ---- SE(3) maps of the free flyer
// free-flyer part of Robot::integrateConfiguration (textbook SE(3) exponential; see oracle/condense_oracle.c)
__device__ __forceinline__ void integrate_free_flyer_dev(double* q, const double* dq, double step) {
  const double vx = step * dq[0], vy = step * dq[1], vz = step * dq[2];
  const double wx = step * dq[3], wy = step * dq[4], wz = step * dq[5];
  const double th2 = wx * wx + wy * wy + wz * wz, th = sqrt(th2);
  double bb, cc, s2 = 0.0, c2 = 1.0;  // one sincos of the half angle serves both the translation and the quaternion part
  if (th < 1e-6) {
    bb = 0.5 - th2 / 24.0; cc = 1.0 / 6.0 - th2 / 120.0;
  } else {
    sincos(0.5 * th, &s2, &c2);
    bb = 2.0 * s2 * s2 / th2; cc = (th - 2.0 * s2 * c2) / (th2 * th);
  }
  const double cx = wy * vz - wz * vy, cy = wz * vx - wx * vz, cz = wx * vy - wy * vx;
  const double ccx = wy * cz - wz * cy, ccy = wz * cx - wx * cz, ccz = wx * cy - wy * cx;
  const double tx = vx + bb * cx + cc * ccx, ty = vy + bb * cy + cc * ccy, tz = vz + bb * cz + cc * ccz;
  const double qx = q[3], qy = q[4], qz = q[5], qw = q[6];
  const double ux = qy * tz - qz * ty, uy = qz * tx - qx * tz, uz = qx * ty - qy * tx;
  const double u2x = qy * uz - qz * uy, u2y = qz * ux - qx * uz, u2z = qx * uy - qy * ux;
  q[0] += tx + 2.0 * (qw * ux + u2x);
  q[1] += ty + 2.0 * (qw * uy + u2y);
  q[2] += tz + 2.0 * (qw * uz + u2z);
  double sh, ch;
  if (th < 1e-6) { sh = 0.5 - th2 / 48.0; ch = 1.0 - th2 / 8.0; } else { sh = s2 / th; ch = c2; }
  const double ex_ = sh * wx, ey = sh * wy, ez = sh * wz, ew = ch;
  const double nx_ = qw * ex_ + qx * ew + qy * ez - qz * ey;
  const double ny = qw * ey - qx * ez + qy * ew + qz * ex_;
  const double nz = qw * ez + qx * ey - qy * ex_ + qz * ew;
  const double nw = qw * ew - qx * ex_ - qy * ey - qz * ez;
  const double nrm = 1.0 / sqrt(nx_ * nx_ + ny * ny + nz * nz + nw * nw);
  q[3] = nx_ * nrm; q[4] = ny * nrm; q[5] = nz * nrm; q[6] = nw * nrm;
}

// Free-flyer part of pinocchio::difference(q0, q1) = log6(M0^-1 M1), q = [p | x y z w], motion = [linear | angular].  The
// rotation comes from the relative quaternion e = conj(quat0) (x) quat1, re-signed to w >= 0: th = 2 atan2(|e_v|, e_w) lies in
// [0, pi] and needs no arccos (exact at th = 0 and well conditioned at pi).  Writes xi = log6(M), M's rotation R (column-major)
// and translation p = R0^T (p1 - p0), and coef = {alpha, beta, beta'(th) / th} for se3_jlog6_dev:
//   alpha = (th / 2) cot(th / 2),  beta = (1 - alpha) / th^2,  v = alpha p - w x p / 2 + beta (w . p) w.
// Below th = 0.1 the three coefficients are Taylor series in th^2 (their closed forms cancel there); tests/state_ref.py
// restates this function operation for operation.
__device__ __forceinline__ void se3_log6_dev(const double* q0, const double* q1, double* xi, double* R, double* p, double* coef) {
  const double ax = q0[3], ay = q0[4], az = q0[5], aw = q0[6], bx = q1[3], by = q1[4], bz = q1[5], bw = q1[6];
  double ex = aw * bx - ax * bw - ay * bz + az * by, ey = aw * by + ax * bz - ay * bw - az * bx;
  double ez = aw * bz - ax * by + ay * bx - az * bw, ew = aw * bw + ax * bx + ay * by + az * bz;
  if (ew < 0.0) { ex = -ex; ey = -ey; ez = -ez; ew = -ew; }
  const double s = sqrt(ex * ex + ey * ey + ez * ez);
  const double ratio = s < 1e-6 ? 2.0 / ew * (1.0 - s * s / (3.0 * ew * ew)) : 2.0 * atan2(s, ew) / s;
  const double wx = ratio * ex, wy = ratio * ey, wz = ratio * ez, th = ratio * s;
  {  // p = R(quat0)^T (p1 - p0) = d - 2 w0 (v0 x d) + 2 v0 x (v0 x d)
    const double dx = q1[0] - q0[0], dy = q1[1] - q0[1], dz = q1[2] - q0[2];
    const double ux = ay * dz - az * dy, uy = az * dx - ax * dz, uz = ax * dy - ay * dx;
    p[0] = dx - 2.0 * aw * ux + 2.0 * (ay * uz - az * uy);
    p[1] = dy - 2.0 * aw * uy + 2.0 * (az * ux - ax * uz);
    p[2] = dz - 2.0 * aw * uz + 2.0 * (ax * uy - ay * ux);
  }
  double alpha, beta, bdot;
  if (th < 0.1) {
    const double t = th * th;
    alpha = 1.0 - t * (1.0 / 12 + t * (1.0 / 720 + t * (1.0 / 30240 + t * (1.0 / 1209600))));
    beta = 1.0 / 12 + t * (1.0 / 720 + t * (1.0 / 30240 + t * (1.0 / 1209600 + t * (1.0 / 47900160))));
    bdot = 1.0 / 360 + t * (1.0 / 7560 + t * (1.0 / 201600 + t * (1.0 / 5987520)));
  } else {
    const double t = th * th;
    double sh, ch;
    sincos(0.5 * th, &sh, &ch);
    alpha = 0.5 * th * ch / sh;
    beta = (1.0 - alpha) / t;
    bdot = -2.0 / (t * t) + (1.0 + 2.0 * sh * ch / th) / (t * 4.0 * sh * sh);
  }
  coef[0] = alpha; coef[1] = beta; coef[2] = bdot;
  const double wp = wx * p[0] + wy * p[1] + wz * p[2];
  xi[0] = alpha * p[0] - 0.5 * (wy * p[2] - wz * p[1]) + beta * wp * wx;
  xi[1] = alpha * p[1] - 0.5 * (wz * p[0] - wx * p[2]) + beta * wp * wy;
  xi[2] = alpha * p[2] - 0.5 * (wx * p[1] - wy * p[0]) + beta * wp * wz;
  xi[3] = wx; xi[4] = wy; xi[5] = wz;
  quat_to_rot(ex, ey, ez, ew, R);
}

// pinocchio::Jlog6(M) (column-major 6x6) from se3_log6_dev's xi, p and coef: [[A, C A], [0, A]] with
//   A = Jlog3 = alpha I + [w]x / 2 + beta w w^T,
//   C = ((beta' / th)(w . p) w - (th^2 beta' / th + 2 beta) p) w^T + beta w p^T + beta (w . p) I + [p]x / 2.
// dDifference: ARG1 = Jlog6(M), ARG0 = -Jlog6(M) Ad(M^-1).
__device__ __forceinline__ void se3_jlog6_dev(const double* xi, const double* p, const double* coef, double* J) {
  const double alpha = coef[0], beta = coef[1], bdot = coef[2];
  const double w[3] = {xi[3], xi[4], xi[5]};
  const double th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2], wp = w[0] * p[0] + w[1] * p[1] + w[2] * p[2];
  const double u[3] = {bdot * wp * w[0] - (th2 * bdot + 2.0 * beta) * p[0], bdot * wp * w[1] - (th2 * bdot + 2.0 * beta) * p[1],
                       bdot * wp * w[2] - (th2 * bdot + 2.0 * beta) * p[2]};
  double A[9], C[9];
  for (int c = 0; c < 3; ++c)
    for (int r = 0; r < 3; ++r) {
      const int e = r + 3 * c;
      // [x]x (r, c) = -eps_rck x_k: (1,0) = x2, (0,1) = -x2, (2,0) = -x1, (0,2) = x1, (2,1) = x0, (1,2) = -x0
      const int k = 3 - r - c;
      const double sgn = (r == c) ? 0.0 : (((c - r + 3) % 3 == 1) ? -1.0 : 1.0);
      A[e] = (r == c ? alpha : 0.0) + (r == c ? 0.0 : 0.5 * sgn * w[k]) + beta * w[r] * w[c];
      C[e] = u[r] * w[c] + beta * w[r] * p[c] + (r == c ? wp * beta : 0.0) + (r == c ? 0.0 : 0.5 * sgn * p[k]);
    }
  for (int c = 0; c < 6; ++c)
    for (int r = 0; r < 6; ++r) {
      double v = 0.0;
      if (r < 3 && c < 3) v = A[r + 3 * c];
      else if (r >= 3 && c >= 3) v = A[(r - 3) + 3 * (c - 3)];
      else if (r < 3) v = C[r] * A[3 * (c - 3)] + C[r + 3] * A[1 + 3 * (c - 3)] + C[r + 6] * A[2 + 3 * (c - 3)];
      J[r + 6 * c] = v;
    }
}

// Ad(M^-1) (column-major 6x6) of M = (R, p) on motions [linear | angular]: [[R^T, -R^T [p]x], [0, R^T]]
__device__ __forceinline__ void se3_ad_inv_dev(const double* R, const double* p, double* Ad) {
  for (int c = 0; c < 6; ++c)
    for (int r = 0; r < 6; ++r) {
      double v = 0.0;
      if ((r < 3) == (c < 3)) {
        v = R[(c % 3) + 3 * (r % 3)];
      } else if (r < 3) {  // -(R^T [p]x)(r, c') = -sum_k R(k, r) [p]x(k, c')
        const int cc = c - 3;
        const double px[9] = {0.0, p[2], -p[1], -p[2], 0.0, p[0], p[1], -p[0], 0.0};  // [p]x column-major
        v = -(R[3 * r] * px[3 * cc] + R[1 + 3 * r] * px[1 + 3 * cc] + R[2 + 3 * r] * px[2 + 3 * cc]);
      }
      Ad[r + 6 * c] = v;
    }
}

__device__ __forceinline__ void inv3_dev(const double* A, int lda, double* B, int ldb) {
  const double a = A[0], b = A[lda], c = A[2 * lda], d = A[1], e = A[1 + lda], f = A[1 + 2 * lda], g = A[2], h = A[2 + lda],
               i = A[2 + 2 * lda];
  const double det = a * (e * i - f * h) - b * (d * i - f * g) + c * (d * h - e * g);
  const double r = 1.0 / det;
  B[0] = (e * i - f * h) * r; B[ldb] = (c * h - b * i) * r; B[2 * ldb] = (b * f - c * e) * r;
  B[1] = (f * g - d * i) * r; B[1 + ldb] = (a * i - c * g) * r; B[1 + 2 * ldb] = (c * d - a * f) * r;
  B[2] = (d * h - e * g) * r; B[2 + ldb] = (b * g - a * h) * r; B[2 + 2 * ldb] = (a * e - b * d) * r;
}

// SE3JacobianInverse::compute (se3_jacobian_inverse.hxx:17-32); one thread; Jac may be global, Jinv shared/global (ld 6)
__device__ __noinline__ void se3_jac_inverse_dev(const double* Jac, double* Jinv) {
  double tmp[9];
  for (int q = 0; q < 36; ++q) Jinv[q] = 0.0;
  inv3_dev(Jac, 6, Jinv, 6);
  inv3_dev(Jac + 3 + 18, 6, Jinv + 3 + 18, 6);
  for (int j = 0; j < 3; ++j)
    for (int i = 0; i < 3; ++i) {
      double acc = 0.0;
      for (int l = 0; l < 3; ++l) acc = fma(Jac[i + (3 + l) * 6], Jinv[(3 + l) + (3 + j) * 6], acc);
      tmp[i + 3 * j] = acc;
    }
  for (int j = 0; j < 3; ++j)
    for (int i = 0; i < 3; ++i) {
      double acc = 0.0;
      for (int l = 0; l < 3; ++l) acc = fma(Jinv[i + l * 6], tmp[l + 3 * j], acc);
      Jinv[i + (3 + j) * 6] = -acc;
    }
}

}  // namespace rbt
