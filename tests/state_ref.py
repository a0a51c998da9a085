"""numpy restatement of the state-equation rows of the linearisation: Pinocchio's free-flyer difference / dDifference
(q = [p | quaternion xyzw | revolute joints], motion = [linear | angular]) and robotoc's linearizeStateEquation
(src/dynamics/state_equation.cpp:30-65), linearizeImpactStateEquation (impact_state_equation.cpp:26-54) and
linearizeTerminalStateEquation (terminal_state_equation.cpp:8-28), with correctLinearizeStateEquation's third block
(state_equation.cpp:78).

  difference(q0, q1) = log6(M0^-1 M1) on the free flyer, q1 - q0 on the joints;
  dDifference ARG1   = Jlog6(M),  ARG0 = -Jlog6(M) Ad(M^-1),  M = M0^-1 M1;
  subtractConfiguration(qf, q0) = difference(q0, qf).

The log is taken from the relative quaternion conj(quat0) (x) quat1, re-signed to w >= 0, so the angle is 2 atan2(|v|, w) in
[0, pi] and needs no arccos.  Jlog3 = alpha I + [w]x / 2 + beta w w^T and Jlog6 = [[Jlog3, C Jlog3], [0, Jlog3]] with
alpha = (th / 2) cot(th / 2), beta = (1 - alpha) / th^2 and C as in Pinocchio's Jlog6; below th = 0.1 the three scalar
coefficients come from their Taylor series.  spatial.cuh (se3_log6_dev, se3_jlog6_dev, se3_ad_inv_dev) evaluates the
same expressions in the same order; tests/test_state_equation.py pins them by central differences, by round trips through
rbd_ref.integrate and by a 100-digit matrix log."""
import numpy as np

SERIES_TH = 0.1  # below this angle alpha, beta and beta'/th are evaluated by their Taylor series in th^2


def _quat_between(a, b):
    """conj(a) (x) b, xyzw."""
    ax, ay, az, aw = a[..., 0], a[..., 1], a[..., 2], a[..., 3]
    bx, by, bz, bw = b[..., 0], b[..., 1], b[..., 2], b[..., 3]
    return np.stack([aw * bx - ax * bw - ay * bz + az * by, aw * by + ax * bz - ay * bw - az * bx,
                     aw * bz - ax * by + ay * bx - az * bw, aw * bw + ax * bx + ay * by + az * bz], -1)


def _rot_t(a, d):
    """R(a)^T d = d - 2 w (v x d) + 2 v x (v x d) for the quaternion a = (v, w)."""
    v, w = a[..., :3], a[..., 3:4]
    u = np.cross(v, d)
    return d - 2.0 * w * u + 2.0 * np.cross(v, u)


def _skew(x):
    z = np.zeros(x.shape[:-1])
    return np.stack([np.stack([z, -x[..., 2], x[..., 1]], -1), np.stack([x[..., 2], z, -x[..., 0]], -1),
                     np.stack([-x[..., 1], x[..., 0], z], -1)], -2)


def _coefficients(th):
    """alpha, beta, beta'(th) / th of Pinocchio's log6 / Jlog6."""
    t = th * th
    small = th < SERIES_TH
    ts = np.where(small, t, 0.0)
    a_s = 1.0 - ts * (1.0 / 12 + ts * (1.0 / 720 + ts * (1.0 / 30240 + ts * (1.0 / 1209600))))
    b_s = 1.0 / 12 + ts * (1.0 / 720 + ts * (1.0 / 30240 + ts * (1.0 / 1209600 + ts * (1.0 / 47900160))))
    d_s = 1.0 / 360 + ts * (1.0 / 7560 + ts * (1.0 / 201600 + ts * (1.0 / 5987520)))
    thl = np.where(small, 1.0, th)
    tl = thl * thl
    sh, ch = np.sin(0.5 * thl), np.cos(0.5 * thl)
    a_l = 0.5 * thl * ch / sh
    b_l = (1.0 - a_l) / tl
    d_l = -2.0 / (tl * tl) + (1.0 + 2.0 * sh * ch / thl) / (tl * 4.0 * sh * sh)
    return np.where(small, a_s, a_l), np.where(small, b_s, b_l), np.where(small, d_s, d_l)


def log6(q0, q1):
    """(xi [B, 6], R [B, 3, 3], p [B, 3], (alpha, beta, bdot) [B]) of M = M(q0)^-1 M(q1), q = [p | x y z w] (at least 7)."""
    e = _quat_between(q0[..., 3:7], q1[..., 3:7])
    e = np.where(e[..., 3:4] < 0.0, -e, e)
    ev, ew = e[..., :3], e[..., 3]
    s = np.sqrt(np.sum(ev * ev, -1))
    ratio = np.where(s < 1e-6, 2.0 / ew * (1.0 - s * s / (3.0 * ew * ew)), 2.0 * np.arctan2(s, ew) / np.where(s < 1e-6, 1.0, s))
    w = ratio[..., None] * ev
    th = ratio * s
    p = _rot_t(q0[..., 3:7], q1[..., :3] - q0[..., :3])
    alpha, beta, bdot = _coefficients(th)
    wp = np.sum(w * p, -1)
    v = alpha[..., None] * p - 0.5 * np.cross(w, p) + (beta * wp)[..., None] * w
    K = _skew(ev)
    R = np.eye(3) + 2.0 * ew[..., None, None] * K + 2.0 * K @ K
    return np.concatenate([v, w], -1), R, p, (alpha, beta, bdot)


def jlog6(xi, p, coef):
    """Pinocchio's Jlog6 [B, 6, 6] from log6's outputs."""
    alpha, beta, bdot = coef
    w = xi[..., 3:]
    th2 = np.sum(w * w, -1)
    wp = np.sum(w * p, -1)
    A = alpha[..., None, None] * np.eye(3) + 0.5 * _skew(w) + beta[..., None, None] * w[..., :, None] * w[..., None, :]
    u = (bdot * wp)[..., None] * w - (th2 * bdot + 2.0 * beta)[..., None] * p
    C = u[..., :, None] * w[..., None, :] + beta[..., None, None] * w[..., :, None] * p[..., None, :]
    C = C + (wp * beta)[..., None, None] * np.eye(3) + 0.5 * _skew(p)
    J = np.zeros(xi.shape[:-1] + (6, 6))
    J[..., :3, :3] = A
    J[..., 3:, 3:] = A
    J[..., :3, 3:] = C @ A
    return J


def ad_inv(R, p):
    """Ad(M^-1) [B, 6, 6] of M = (R, p): [[R^T, -R^T [p]x], [0, R^T]]."""
    Rt = np.swapaxes(R, -1, -2)
    out = np.zeros(R.shape[:-2] + (6, 6))
    out[..., :3, :3] = Rt
    out[..., :3, 3:] = -Rt @ _skew(p)
    out[..., 3:, 3:] = Rt
    return out


def difference(q0, q1):
    """pinocchio::difference(q0, q1) [B, nv] = q1 (-) q0."""
    xi = log6(q0, q1)[0]
    return np.concatenate([xi, q1[..., 7:] - q0[..., 7:]], -1)


def d_difference(q0, q1, arg):
    """pinocchio::dDifference(q0, q1, ARG0 | ARG1) [B, nv, nv] (arg = 0 | 1)."""
    xi, R, p, coef = log6(q0, q1)
    J = jlog6(xi, p, coef)
    nv = q0.shape[-1] - 1
    out = np.zeros(q0.shape[:-1] + (nv, nv))
    out[..., 6:, 6:] = np.eye(nv - 6) * (1.0 if arg == 1 else -1.0)
    out[..., :6, :6] = J if arg == 1 else -J @ ad_inv(R, p)
    return out


def _put(r, off, blk):
    """6x6 blocks [B, 6, 6] into column-major record sections."""
    r[:, off:off + 36] = np.swapaxes(blk, -1, -2).reshape(-1, 36)


def linearize(S, ctrl, sol, lin, q0):
    """What rbt_linearize_state_equation writes, for records [batch, n_grid, ...] and the measured configuration q0
    [batch, nq]: returns the updated linearization records."""
    from robotoc_b200.grid import IMPACT, TERMINAL
    l = lin.copy()
    nv, nq = S.nv, S.nq
    with_sto = any(c.sto or c.sto_next for c in ctrl)
    for i, c in enumerate(ctrl):
        s = sol[:, i]
        q, lmd, gmm = s[:, S.s_q:S.s_q + nq], s[:, S.s_lmd:S.s_lmd + nv], s[:, S.s_gmm:S.s_gmm + nv]
        q_prev = q0 if i == 0 else sol[:, i - 1, S.s_q:S.s_q + nq]
        r = l[:, i]
        Fqq_prev = d_difference(q, q_prev, 0)[:, :6, :6]   # dSubtractConfiguration_dq0(q_prev, q)
        _put(r, S.l_se3 + 36, Fqq_prev)
        lq, lv = r[:, S.l_lx:S.l_lx + nv], r[:, S.l_lx + nv:S.l_lx + 2 * nv]
        if c.type == TERMINAL:
            lq[:, :6] += np.einsum("brk,br->bk", Fqq_prev, lmd[:, :6])
            lq[:, 6:] -= lmd[:, 6:]
            lv -= gmm
            continue
        impact = c.type == IMPACT
        sn = sol[:, i + 1]
        q_n, v_n = sn[:, S.s_q:S.s_q + nq], sn[:, S.s_v:S.s_v + nv]
        lmd_n, gmm_n = sn[:, S.s_lmd:S.s_lmd + nv], sn[:, S.s_gmm:S.s_gmm + nv]
        v, a, dv = s[:, S.s_v:S.s_v + nv], s[:, S.s_a:S.s_a + nv], s[:, S.s_dv:S.s_dv + nv]
        xi, R, p, coef = log6(q_n, q)                  # subtractConfiguration(q, q_next) = difference(q_next, q)
        J = jlog6(xi, p, coef)
        Fq = np.concatenate([xi, q[:, 7:] - q_n[:, 7:]], -1)
        if impact:
            Fv = v + dv - v_n
        else:
            Fq = Fq + c.dt * v
            Fv = v + c.dt * a - v_n
        r[:, S.l_Fx:S.l_Fx + nv], r[:, S.l_Fx + nv:S.l_Fx + 2 * nv] = Fq, Fv
        _put(r, S.l_se3, J)                              # Fqq top-left = dSubtractConfiguration_dqf(q, q_next)
        _put(r, S.l_se3 + 72, -J @ ad_inv(R, p))         # Fqq_cur = dSubtractConfiguration_dq0(q, q_next)
        lq[:, :6] += np.einsum("brk,br->bk", J, lmd_n[:, :6]) + np.einsum("brk,br->bk", Fqq_prev, lmd[:, :6])
        lq[:, 6:] += lmd_n[:, 6:] - lmd[:, 6:]
        la = r[:, S.l_la:S.l_la + nv]
        if impact:
            lv += gmm_n - gmm
            la += gmm_n
            continue
        lv += c.dt * lmd_n + gmm_n - gmm
        la += c.dt * gmm_n
        if with_sto:
            r[:, S.l_sc] += np.sum(lmd_n * v, -1) + np.sum(gmm_n * a, -1)
            r[:, S.l_hx + nv:S.l_hx + 2 * nv] += lmd_n
            r[:, S.l_ha:S.l_ha + nv] += gmm_n
            r[:, S.l_fx:S.l_fx + nv], r[:, S.l_fx + nv:S.l_fx + 2 * nv] = v, a
    return l


def random_q0(seed, batch, nq):
    """A measured configuration per OCP: position in [-1, 1]^3, a random unit quaternion, joints in [-1, 1]."""
    rng = np.random.default_rng(seed)
    q = rng.uniform(-1.0, 1.0, (batch, nq))
    quat = rng.normal(size=(batch, 4))
    q[:, 3:7] = quat / np.linalg.norm(quat, axis=1, keepdims=True)
    return q
