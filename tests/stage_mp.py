"""Extended-precision (mpmath) reference of two stage-layer kernels, independent of oracle/condense_oracle.c:

  - mjtjinv(M, J): Robot::computeMJtJinv (include/robotoc/robot/robot.hxx:642-683), Z = [[M, J^T], [J, 0]]^-1, taken as the
    exact inverse of the whole KKT matrix by mp LU (mp.inverse), not by the Cholesky of M and of the Schur complement
    J M^-1 J^T that both fp64 implementations use.
  - integrate_free_flyer(q, dq, step): the free-flyer part of SplitSolution::integrate (src/core/split_solution.cpp:58-90 ->
    Robot::integrateConfiguration -> pinocchio::integrate): M_new = M(q) * exp(step * dq[:6]) with the exponential taken by
    mp.expm of the 4x4 twist matrix, as tests/rbd_mp.py does.  The quaternion is q (x) (sin(th/2) w / th, cos(th/2)), the
    SU(2) exponential whose sign the kernels keep (it is not re-signed towards q for th > pi); the CPU tests check that its
    rotation is the expm rotation to 1e-40.

Every output comes with a scale, the size of what the fp64 arithmetic of that row is made of, so that a comparison holds each
row to the error its own arithmetic can make:
  - Z: the row's largest entry of |Z| |A| |Z|, the componentwise sensitivity of Z to one rounding of the KKT matrix A;
  - the translation rows: |p| + |R(q)| t_size, the terms of p + R(q) t with t_size = |v| + b |[w]x| |v| + c |[w]x|^2 |v| the
    terms of t = V(w) v, and |R(q)| = I + 2 |qw| |[qv]x| + 2 |[qv]x|^2 entrywise (the quaternion rotation the kernels
    evaluate);
  - the quaternion rows: the sum of |q_a| |e_b| over the terms of the Hamilton product, plus th / 2 sum |q_a|: the kernels
    round th (from step * dq and a square root) before they take sin(th / 2), cos(th / 2), and one rounding of th / 2 moves
    e by up to th / 2 of a unit;
  - the joint rows: |q_j| + |step dq_j|.
Every function works under mp.workdps(DPS) and leaves the process's precision alone."""
import numpy as np
from mpmath import mp

DPS = 100


def _m(A):
    return mp.matrix([[mp.mpf(float(x)) for x in row] for row in np.atleast_2d(A)])


def _f64(X, rows, cols):
    return np.array([[float(X[i, j]) for j in range(cols)] for i in range(rows)])


def kkt(M, J):
    """[[M, J^T], [J, 0]] as an mp matrix (exact in the fp64 entries)."""
    nv, nf = M.shape[0], J.shape[0]
    A = np.zeros((nv + nf, nv + nf))
    A[:nv, :nv], A[nv:, :nv], A[:nv, nv:] = M, J, J.T
    return _m(A)


def mjtjinv(M, J):
    """(Z, scale): Z [n, n] rounded once from the exact inverse, scale [n] = row max of |Z| |A| |Z|."""
    n = M.shape[0] + J.shape[0]
    with mp.workdps(DPS):
        A = kkt(M, J)
        Z = mp.inverse(A)
        aZ, aA = Z.apply(abs), A.apply(abs)
        S = aZ * aA * aZ
        return _f64(Z, n, n), np.array([float(max(S[i, j] for j in range(n))) for i in range(n)])


def _skew(w):
    return mp.matrix([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])


def _quat_mul(a, b):
    """Hamilton product of xyzw quaternions."""
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return [aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
            aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz]


def quat_rot(q):
    """R(q) = I + 2 qw [qv]x + 2 [qv]x^2, the rotation of a unit quaternion as the kernels apply it."""
    K = _skew(q[:3])
    return mp.eye(3) + 2 * q[3] * K + 2 * K * K


def _exp_quat(w):
    th = mp.sqrt(sum(x * x for x in w))
    if th == 0:
        return [mp.mpf(0)] * 3 + [mp.mpf(1)], th
    sh = mp.sin(th / 2) / th
    return [sh * w[0], sh * w[1], sh * w[2], mp.cos(th / 2)], th


def _integrate(q, dq, step):
    """mp values: (p_new [3], quat_new [4], expm rotation [3x3], R(q) [3x3], t [3], th)."""
    v = [step * mp.mpf(float(x)) for x in dq[:3]]
    w = [step * mp.mpf(float(x)) for x in dq[3:6]]
    T = mp.expm(mp.matrix([[0, -w[2], w[1], v[0]], [w[2], 0, -w[0], v[1]], [-w[1], w[0], 0, v[2]], [0, 0, 0, 0]]))
    qq = [mp.mpf(float(x)) for x in q[3:7]]
    R0 = quat_rot(qq)
    t = mp.matrix([T[0, 3], T[1, 3], T[2, 3]])
    p = R0 * t
    e, th = _exp_quat(w)
    n = _quat_mul(qq, e)
    nrm = mp.sqrt(sum(x * x for x in n))
    return [mp.mpf(float(q[k])) + p[k] for k in range(3)], [x / nrm for x in n], T[:3, :3], R0, t, th, v, w, e


def integrate_free_flyer(q, dq, step):
    """(q_new [nq], scale [nq]) of Robot::integrateConfiguration for a floating base: q = (p, quat xyzw, joints), dq [nv]."""
    q, dq = np.asarray(q, float), np.asarray(dq, float)
    out, sc = q.copy(), np.zeros_like(q)
    with mp.workdps(DPS):
        p1, n, _, R0, _, th, v, w, e = _integrate(q, dq, step)
        av = [abs(x) for x in v]
        Kw = _skew(w).apply(abs)
        b = (1 - mp.cos(th)) / th ** 2 if th != 0 else mp.mpf(0.5)
        c = (th - mp.sin(th)) / th ** 3 if th != 0 else mp.mpf(1) / 6
        tsz = mp.matrix(av) + b * (Kw * mp.matrix(av)) + c * (Kw * (Kw * mp.matrix(av)))
        aq = [abs(mp.mpf(float(x))) for x in q[3:7]]
        Kq = _skew(aq[:3]).apply(abs)
        Ra = mp.eye(3) + 2 * aq[3] * Kq + 2 * Kq * Kq
        rsz = Ra * tsz
        ae = [abs(x) for x in e]
        qx, qy, qz, qw = aq
        ex, ey, ez, ew = ae
        hq = th / 2 * (qx + qy + qz + qw)  # one rounding of the half angle th / 2 moves e by up to th / 2 of it
        qsz = [qw * ex + qx * ew + qy * ez + qz * ey + hq, qw * ey + qx * ez + qy * ew + qz * ex + hq,
               qw * ez + qx * ey + qy * ex + qz * ew + hq, qw * ew + qx * ex + qy * ey + qz * ez + hq]
        for k in range(3):
            out[k], sc[k] = float(p1[k]), float(abs(mp.mpf(float(q[k]))) + rsz[k])
        for k in range(4):
            out[3 + k], sc[3 + k] = float(n[k]), float(qsz[k])
    for j in range(7, q.size):
        out[j] = float(mp.mpf(float(q[j])) + mp.mpf(float(step)) * mp.mpf(float(dq[j - 1])))
        sc[j] = abs(q[j]) + abs(step * dq[j - 1])
    return out, sc


def row_errors(got, ref, scale, witness=None, a=4.0, b=16.0):
    """The comparison rule of a row r: e_dev(r) <= max(a e_orc(r), b 2^-53 C(r)), e = max over the row of |x - mp|.
    got, ref, witness: [..., rows, cols] (or [..., rows]); scale [..., rows].  Returns e_dev / bound per row; a row whose value,
    witness or scale is not finite gets inf, so it fails any bound (NaN would compare False against every bound)."""
    got, ref, scale = np.asarray(got, float), np.asarray(ref, float), np.asarray(scale, float)
    if got.ndim == scale.ndim:
        got, ref = got[..., None], ref[..., None]
        witness = None if witness is None else np.asarray(witness, float)[..., None]
    e = np.max(np.abs(got - ref), axis=-1)
    bound = b * 2.0 ** -53 * scale
    if witness is not None:
        bound = np.maximum(bound, a * np.max(np.abs(np.asarray(witness, float) - ref), axis=-1))
    r = np.where(e == 0, 0.0, e / np.where(bound > 0, bound, 1e-300))
    return np.where(np.isfinite(e) & np.isfinite(bound), r, np.inf)
