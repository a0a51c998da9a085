"""State-equation rows of the linearisation (rbt_linearize_state_equation), CPU side.

There is no Pinocchio here, so tests/state_ref.py restates difference / dDifference and the rows of linearizeStateEquation,
linearizeImpactStateEquation and linearizeTerminalStateEquation.  This file pins that restatement by
  - central differences in the tangent space, q (+) eps e_k with the free-flyer exponential of the update kernel, for Fqq,
    Fqq_prev and Fqq_cur;
  - difference(q, integrate(q, xi)) = xi for rotation angles up to pi - 1e-6;
  - Fqq_prev of grid point i + 1 being Fqq_cur of grid point i;
  - the costate and STO terms being the gradient of sum_i lmd_{i+1} . Fq_i + gmm_{i+1} . Fv_i over a whole horizon (q0 fixed);
  - a 100-digit evaluation with the matrix log and exp of 4x4 homogeneous transforms, held to the row-scale rule of
    tests/stage_mp.py.
It also checks the wire tables with RBT_WIRE_DEVICE_STATE: the segments, the 144 / 36 doubles they drop and the pack / unpack
round trip, alone and with the other two device bits."""
import ctypes
import zlib

import numpy as np
import pytest
from mpmath import mp

import state_ref as SR
from stage_mp import row_errors

NV, NQ = 18, 19


def _random_q(rng, B, pos=1.0):
    q = rng.uniform(-1.0, 1.0, (B, NQ))
    q[:, :3] *= pos
    quat = rng.normal(size=(B, 4))
    q[:, 3:7] = quat / np.linalg.norm(quat, axis=1, keepdims=True)
    return q


def exp_update(q, dq):
    """q (+) dq with the free-flyer exponential of update_kernel (integrate_free_flyer_dev, step 1), joints added."""
    out = q.copy()
    for b in range(q.shape[0]):
        v, w = dq[b, :3], dq[b, 3:6]
        th2 = float(w @ w)
        th = np.sqrt(th2)
        if th < 1e-6:
            bb, cc, sh, ch = 0.5 - th2 / 24.0, 1.0 / 6.0 - th2 / 120.0, 0.5 - th2 / 48.0, 1.0 - th2 / 8.0
        else:
            s2, c2 = np.sin(0.5 * th), np.cos(0.5 * th)
            bb, cc, sh, ch = 2.0 * s2 * s2 / th2, (th - 2.0 * s2 * c2) / (th2 * th), s2 / th, c2
        c1 = np.cross(w, v)
        t = v + bb * c1 + cc * np.cross(w, c1)
        qv, qw = q[b, 3:6], q[b, 6]
        u = np.cross(qv, t)
        out[b, :3] = q[b, :3] + t + 2.0 * (qw * u + np.cross(qv, u))
        e, ew = sh * w, ch
        n = np.concatenate([qw * e + ew * qv + np.cross(qv, e), [qw * ew - qv @ e]])
        out[b, 3:7] = n / np.linalg.norm(n)
        out[b, 7:] = q[b, 7:] + dq[b, 6:]
    return out


def _central(f, q, h=1e-6):
    """[B, m, nv] central differences of f(q) [B, m] in the tangent space of q."""
    B = q.shape[0]
    cols = []
    for k in range(NV):
        e = np.zeros((B, NV))
        e[:, k] = h
        cols.append((f(exp_update(q, e)) - f(exp_update(q, -e))) / (2 * h))
    return np.stack(cols, -1)


def test_jacobians_match_central_differences():
    rng = np.random.default_rng(1)
    q, q_n, q_p = (_random_q(rng, 6) for _ in range(3))
    # Fq = Sub(q, q_next) = difference(q_next, q): Fqq = d/dq, Fqq_cur = d/dq_next; Fqq_prev = d/dq Sub(q_prev, q)
    Fqq = SR.d_difference(q_n, q, 1)
    Fqq_cur = SR.d_difference(q_n, q, 0)
    Fqq_prev = SR.d_difference(q, q_p, 0)
    np.testing.assert_allclose(Fqq, _central(lambda x: SR.difference(q_n, x), q), rtol=0, atol=1e-8)
    np.testing.assert_allclose(Fqq_cur, _central(lambda x: SR.difference(x, q), q_n), rtol=0, atol=1e-8)
    np.testing.assert_allclose(Fqq_prev, _central(lambda x: SR.difference(x, q_p), q), rtol=0, atol=1e-8)


ANGLES = [0.0, 1e-12, 1e-6, np.nextafter(1e-6, 0.0), np.nextafter(1e-6, 1.0), 0.0999999, 0.1, 0.1000001, 1.0, 3.0,
          np.pi - 1e-6]


@pytest.mark.parametrize("th", ANGLES)
def test_difference_inverts_the_exponential(th):
    rng = np.random.default_rng(2)
    q = _random_q(rng, 4)
    xi = rng.uniform(-1.0, 1.0, (4, NV))
    axis = rng.normal(size=(4, 3))
    xi[:, 3:6] = th * axis / np.linalg.norm(axis, axis=1, keepdims=True)
    got = SR.difference(q, exp_update(q, xi))
    np.testing.assert_allclose(got, xi, rtol=0, atol=4e-15 * (1 + np.pi))


def _horizon(which):
    import helpers
    return {"small_sto": lambda: helpers.small_event_schedule(sto=True)[2], "trot": lambda: helpers.trot_schedule(12)[2]}[which]()


def _records(ctrl, batch, seed):
    from robotoc_b200 import ANYMAL, StageDims, StageLayout, anymal_constraint_table
    from synth import make_stage_inputs
    table = anymal_constraint_table()
    sd = StageDims(ANYMAL, nf_max=12, n_contacts=4, n_box=table.n_box)
    S = StageLayout(sd)
    lin, con, sol, dx0 = make_stage_inputs(sd, S, ctrl, batch, seed)
    return sd, S, lin, sol


def test_fqq_prev_is_the_previous_fqq_cur():
    ctrl = _horizon("small_sto")
    _, S, lin, sol = _records(ctrl, 3, 3)
    out = SR.linearize(S, ctrl, sol, lin, SR.random_q0(4, 3, S.nq))
    for i in range(len(ctrl) - 1):
        np.testing.assert_array_equal(out[:, i + 1, S.l_se3 + 36:S.l_se3 + 72], out[:, i, S.l_se3 + 72:S.l_se3 + 108])


@pytest.mark.parametrize("which", ["small_sto", "trot"])
def test_costate_terms_are_the_gradient_of_the_multiplier_terms(which):
    """linearize adds d/dx_i sum_j (lmd_{j+1} . Fq_j + gmm_{j+1} . Fv_j) to lq, lv, la | ldv (the terms of the Lagrangian that
    hold the state equation, q0 fixed) and, with STO, its dt_i derivative to h."""
    from robotoc_b200.grid import IMPACT, TERMINAL
    ctrl = _horizon(which)
    _, S, lin, sol = _records(ctrl, 2, 5)
    q0 = SR.random_q0(6, 2, S.nq)
    zero = np.zeros_like(lin)
    out = SR.linearize(S, ctrl, sol, zero, q0)
    nv, n = S.nv, len(ctrl)
    dts = np.array([c.dt for c in ctrl])

    def phi(sl, dt=dts):
        tot = np.zeros(sl.shape[0])
        for j in range(n - 1):
            s, sn = sl[:, j], sl[:, j + 1]
            q, qn = s[:, S.s_q:S.s_q + S.nq], sn[:, S.s_q:S.s_q + S.nq]
            v, vn = s[:, S.s_v:S.s_v + nv], sn[:, S.s_v:S.s_v + nv]
            Fq = SR.difference(qn, q)
            if ctrl[j].type == IMPACT:
                Fv = v + s[:, S.s_dv:S.s_dv + nv] - vn
            else:
                Fq = Fq + dt[j] * v
                Fv = v + dt[j] * s[:, S.s_a:S.s_a + nv] - vn
            tot += np.sum(sn[:, S.s_lmd:S.s_lmd + nv] * Fq, -1) + np.sum(sn[:, S.s_gmm:S.s_gmm + nv] * Fv, -1)
        # grid point 0's q_prev term: lmd_0 . Sub(q0, q_0), gmm_0 . (-v_0); then lmd_{j} for j >= 1 enter through Fq_{j-1}
        tot += np.sum(sl[:, 0, S.s_lmd:S.s_lmd + nv] * SR.difference(sl[:, 0, S.s_q:S.s_q + S.nq], q0), -1)
        tot -= np.sum(sl[:, 0, S.s_gmm:S.s_gmm + nv] * sl[:, 0, S.s_v:S.s_v + nv], -1)
        return tot

    h = 1e-6
    for i, c in enumerate(ctrl):
        r = out[:, i]
        for k in range(nv):
            e = np.zeros((2, NV))
            e[:, k] = h
            sp, sm = sol.copy(), sol.copy()
            sp[:, i, S.s_q:S.s_q + S.nq] = exp_update(sol[:, i, S.s_q:S.s_q + S.nq], e)
            sm[:, i, S.s_q:S.s_q + S.nq] = exp_update(sol[:, i, S.s_q:S.s_q + S.nq], -e)
            assert np.allclose(r[:, S.l_lx + k], (phi(sp) - phi(sm)) / (2 * h), rtol=1e-6, atol=1e-7), (i, "lq", k)
            offs = [(S.s_v, S.l_lx + nv)]
            if c.type != TERMINAL:
                offs.append((S.s_dv if c.type == IMPACT else S.s_a, S.l_la))
            for so, lo in offs:
                sp, sm = sol.copy(), sol.copy()
                sp[:, i, so + k] += h
                sm[:, i, so + k] -= h
                assert np.allclose(r[:, lo + k], (phi(sp) - phi(sm)) / (2 * h), rtol=1e-6, atol=1e-7), (i, lo, k)
        if any(cc.sto or cc.sto_next for cc in ctrl) and c.type not in (IMPACT, TERMINAL):
            dp, dm = dts.copy(), dts.copy()
            dp[i] += h
            dm[i] -= h
            assert np.allclose(r[:, S.l_sc], (phi(sol, dp) - phi(sol, dm)) / (2 * h), rtol=1e-6, atol=1e-7), i
            s = sol[:, i]
            np.testing.assert_array_equal(r[:, S.l_fx:S.l_fx + 2 * nv], np.concatenate([s[:, S.s_v:S.s_v + nv], s[:, S.s_a:S.s_a + nv]], -1))
            np.testing.assert_array_equal(r[:, S.l_hx + nv:S.l_hx + 2 * nv], sol[:, i + 1, S.s_lmd:S.s_lmd + nv])
            np.testing.assert_array_equal(r[:, S.l_ha:S.l_ha + nv], sol[:, i + 1, S.s_gmm:S.s_gmm + nv])


# ---- 100-digit reference: log and exp of 4x4 homogeneous transforms
DPS = 100


def _T(q):
    """4x4 mp transform of q = [p | x y z w] (the quaternion normalised in mp)."""
    x, y, z, w = (mp.mpf(float(c)) for c in q[3:7])
    n = mp.sqrt(x * x + y * y + z * z + w * w)
    x, y, z, w = x / n, y / n, z / n, w / n
    R = [[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
         [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
         [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]]
    return mp.matrix([R[0] + [mp.mpf(float(q[0]))], R[1] + [mp.mpf(float(q[1]))], R[2] + [mp.mpf(float(q[2]))], [0, 0, 0, 1]])


def _hat(xi):
    v, w = xi[:3], xi[3:]
    return mp.matrix([[0, -w[2], w[1], v[0]], [w[2], 0, -w[0], v[1]], [-w[1], w[0], 0, v[2]], [0, 0, 0, 0]])


def _vee(L):
    return [L[0, 3], L[1, 3], L[2, 3], L[2, 1], L[0, 2], L[1, 0]]


def _mp_difference(q0, q1, xi0):
    """(xi [6], J1 [6, 6], J0 [6, 6], |p|, th) of log6(M0^-1 M1) and its derivatives for right perturbations M exp(eps e_k) of
    M1 (J1) and of M0 (J0).  mp.logm picks a wrong branch near th = pi, so the log is the root of expm(hat(xi)) = M found by
    Newton from the fp64 value xi0, with logm taken only near the identity: xi += Jr(xi)^-1 vee(logm(expm(-hat(xi)) M)).  Jr and
    Jl, the right and left Jacobians of the exponential, are forward differences (eps = 1e-45) of logm near the identity, and
    J1 = Jr^-1, J0 = -Jl^-1 (exp(xi + d) = exp(Jl d) exp(xi) = exp(xi) exp(Jr d))."""
    with mp.workdps(DPS):
        M = mp.inverse(_T(q0)) * _T(q1)
        log = lambda A: [mp.re(x) for x in _vee(mp.logm(A))]  # noqa: E731  (real: drop round-off of the complex log)
        eps = mp.mpf("1e-45")

        def jac(xi, left):
            J = mp.matrix(6, 6)
            Ei = mp.expm(-_hat(xi))
            for k in range(6):
                e = list(xi)
                e[k] += eps
                d = log(mp.expm(_hat(e)) * Ei if left else Ei * mp.expm(_hat(e)))
                for r in range(6):
                    J[r, k] = d[r] / eps
            return J

        xi = [mp.mpf(float(x)) for x in xi0]
        for _ in range(2):
            Jr_inv = mp.inverse(jac(xi, False))
            for _ in range(3):
                d = Jr_inv * mp.matrix(log(mp.expm(-_hat(xi)) * M))
                xi = [xi[r] + d[r] for r in range(6)]
        res = max(abs(x) for x in log(mp.expm(-_hat(xi)) * M))
        assert res < mp.mpf("1e-80"), res
        J1, J0 = mp.inverse(jac(xi, False)), -mp.inverse(jac(xi, True))
        pn = float(mp.sqrt(M[0, 3] ** 2 + M[1, 3] ** 2 + M[2, 3] ** 2))
        th = float(mp.sqrt(xi[3] ** 2 + xi[4] ** 2 + xi[5] ** 2))
        assert th < mp.pi
        f = lambda A: np.array([[float(A[r, c]) for c in range(6)] for r in range(6)])  # noqa: E731
        return np.array([float(x) for x in xi]), f(J1), f(J0), pn, th


def _quat_mul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz])


def _case(name):
    """(q0, q1) of one configuration pair: e is the relative quaternion (sin(th/2) axis, cos(th/2)) rounded to fp64; with an
    identity base rotation q1 carries e exactly, so the fp64 neighbours of an angle reach the code as they are."""
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    ident = name.startswith("x:")
    if ident:
        axis = np.array([1.0, 0.0, 0.0])
    kind, val = name.split(":")[0], name.split(":")[1]
    th = {"0": 0.0, "1e-12": 1e-12, "1e-6": 1e-6, "1e-6-": np.nextafter(1e-6, 0.0), "1e-6+": np.nextafter(1e-6, 1.0),
          "0.1": 0.1, "1": 1.0, "pi-1e-6": np.pi - 1e-6}[val]
    e = np.concatenate([np.sin(0.5 * th) * axis, [np.cos(0.5 * th)]])
    if val.startswith("1e-6") and ident:  # the sine itself on the neighbours: s = 1e-6 / 2 and its fp64 neighbours
        e = np.array([{"1e-6": 5e-7, "1e-6-": np.nextafter(5e-7, 0.0), "1e-6+": np.nextafter(5e-7, 1.0)}[val], 0.0, 0.0, 1.0])
    q0 = np.zeros(NQ)
    q0[:3] = rng.uniform(-1, 1, 3) + (np.array([1e3, -1e3, 5e2]) if kind == "far" else 0.0)
    if ident:
        q0[3:7] = [0.0, 0.0, 0.0, 1.0]
    else:
        qq = rng.normal(size=4)
        q0[3:7] = qq / np.linalg.norm(qq)
    q1 = q0.copy()
    q1[:3] = q0[:3] + rng.uniform(-0.5, 0.5, 3)
    q1[3:7] = e if ident else _quat_mul(q0[3:7], e)
    if kind == "neg":  # the same rotation with w < 0
        q1[3:7] = -q1[3:7]
    return q0, q1


MP_CASES = ["x:0", "x:1e-12", "x:1e-6", "x:1e-6-", "x:1e-6+", "x:0.1", "r:1e-12", "r:1e-6", "r:1", "r:pi-1e-6", "neg:1",
            "neg:pi-1e-6", "neg:1e-6", "far:1", "far:1e-6", "far:pi-1e-6"]


@pytest.mark.parametrize("name", MP_CASES)
def test_difference_and_its_jacobians_match_100_digits(name):
    """Each row is held to 16 units of 2^-53 of its scale 1 + |p| + th (p: the relative translation): what the fp64 terms of
    log6, Jlog6 and Ad(M^-1) are made of, so a formulation that cancels large absolute positions fails the "far" cases."""
    q0, q1 = _case(name)
    got_xi = SR.difference(q0[None], q1[None])[0, :6]
    xi, J1, J0, pn, th = _mp_difference(q0, q1, got_xi)
    got_J1 = SR.d_difference(q0[None], q1[None], 1)[0, :6, :6]
    got_J0 = SR.d_difference(q0[None], q1[None], 0)[0, :6, :6]
    scale = np.full(6, 1.0 + pn + th)
    assert row_errors(got_xi, xi, scale).max() <= 1.0, (got_xi, xi)
    assert row_errors(got_J1, J1, scale).max() <= 1.0, np.abs(got_J1 - J1).max()
    assert row_errors(got_J0, J0, scale).max() <= 1.0, np.abs(got_J0 - J0).max()


# ---- wire segment tables with RBT_WIRE_DEVICE_STATE
class _seg(ctypes.Structure):
    _fields_ = [(f, ctypes.c_int) for f in ("lin_off", "wire_off", "rows", "cols", "ld", "sym")]


class _zero(ctypes.Structure):
    _fields_ = [("lin_off", ctypes.c_int), ("n", ctypes.c_int)]


class _wl(ctypes.Structure):
    _fields_ = [("nseg", ctypes.c_int), ("nzero", ctypes.c_int), ("w_doubles", ctypes.c_int), ("ocp_off", ctypes.c_int),
                ("seg", _seg * 20), ("zero", _zero * 5)]


def _unpack(W, wire, lin):
    """rbt_unpack_wire_record restated."""
    for k in range(W.nzero):
        z = W.zero[k]
        lin[z.lin_off:z.lin_off + z.n] = 0.0
    for k in range(W.nseg):
        g = W.seg[k]
        src = wire[g.wire_off:]
        for j in range(g.cols if g.sym == 0 else g.rows):
            for i in range(g.rows):
                if g.sym == 0:
                    lin[g.lin_off + i + j * g.ld] = src[i + j * g.rows]
                elif g.sym == 2:
                    if i == j:
                        lin[g.lin_off + i * (g.ld + 1)] = src[i]
                else:
                    lin[g.lin_off + i + j * g.ld] = src[j * (j + 1) // 2 + i] if i <= j else src[i * (i + 1) // 2 + j]


def _schedule(which):
    import helpers
    return {"trot": helpers.trot_schedule, "jump": helpers.jump_sto_schedule,
            "small_sto": lambda: helpers.small_event_schedule(sto=True)}[which]()[2]


@pytest.mark.parametrize("which", ["trot", "jump", "small_sto"])
@pytest.mark.parametrize("cs", [16, 17, 18, 20, 22, 23])
def test_wire_tables_with_device_state_equation(which, cs):
    from robotoc_b200._lib import lib
    from robotoc_b200.grid import TERMINAL
    from synth import symmetrize_lin
    ctrl = _schedule(which)
    sd, S, lin, _ = _records(ctrl, 1, 7)
    lin = symmetrize_lin(S, lin)[0]
    L = lib()
    csd = sd.c()
    n = len(ctrl)
    base = cs & ~16  # the same records with the state-equation rows on the wire
    total = {f: L.rbt_wire_doubles(ctypes.byref(csd), ctrl, n, f) for f in (base, cs)}
    wires = {}
    for f in (base, cs):
        wires[f] = np.zeros(total[f])
        assert L.rbt_pack_wire(ctypes.byref(csd), ctrl, n, f, lin.ctypes.data_as(ctypes.c_void_p),
                               wires[f].ctypes.data_as(ctypes.c_void_p), 1) == 0
    dropped = 0
    for i in range(n):
        w, w0 = _wl(), _wl()
        assert L.rbt_wire_layout_get(ctypes.byref(csd), ctrl, n, cs, i, ctypes.byref(w)) == 0
        assert L.rbt_wire_layout_get(ctypes.byref(csd), ctrl, n, base, i, ctypes.byref(w0)) == 0
        got = [(w.seg[k].lin_off, w.seg[k].rows, w.seg[k].cols, w.seg[k].ld, w.seg[k].sym) for k in range(w.nseg)]
        ref = [(w0.seg[k].lin_off, w0.seg[k].rows, w0.seg[k].cols, w0.seg[k].ld, w0.seg[k].sym) for k in range(w0.nseg)]
        device = np.zeros(S.l_stride, bool)  # what the device fills instead
        if ctrl[i].type == TERMINAL:
            assert got == ref[:-1] and ref[-1] == (S.l_se3 + 36, 36, 1, 36, 0)
            assert w0.w_doubles - w.w_doubles == 36
            dropped += 36
            device[S.l_se3 + 36:S.l_se3 + 72] = True
        else:
            # the lx .. SE(3) segment splits around Fx and the SE(3) blocks; every other segment stays
            k = ref.index((S.l_lx, S.l_Phix - S.l_lx, 1, S.l_Phix - S.l_lx, 0))
            assert got[:k] == ref[:k] and got[k + 2:] == ref[k + 1:]
            assert got[k:k + 2] == [(S.l_lx, S.l_Fx - S.l_lx, 1, S.l_Fx - S.l_lx, 0),
                                    (S.l_lup, S.l_se3 - S.l_lup, 1, S.l_se3 - S.l_lup, 0)]
            assert w0.w_doubles - w.w_doubles == 144
            dropped += 144
            device[S.l_Fx:S.l_Fx + S.nx] = True
            device[S.l_se3:S.l_se3 + 108] = True
        full, mine = np.full(S.l_stride, np.nan), np.full(S.l_stride, np.nan)
        _unpack(w0, wires[base][w0.ocp_off:], full)
        _unpack(w, wires[cs][w.ocp_off:], mine)
        assert np.isnan(mine[device]).all() and not np.isnan(full[device]).any()
        np.testing.assert_array_equal(mine[~device], full[~device])
    assert total[base] - total[cs] == dropped
