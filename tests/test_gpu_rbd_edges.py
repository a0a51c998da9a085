"""rbt_linearize_inverse_dynamics and rbt_linearize_contact_kinematics on the device against the extended-precision reference
tests/rbd_mp.py (tests/golden/rbd_mp_cases.npz), entry by entry, on the states where fp64 kernels go wrong: ANYmal standing
(the base rows a near-cancellation), trotting, touching down and 1e3 m from the origin (the Baumgarte position term a
near-cancellation), joint angles up to 1e12 rad (both argument reductions of fp64 sincos), quaternions with w = 0, 1e-9, < 0 and
-q; a 13-body chain and star with off-axis gravity, 1e-3 kg links, a contact on the base and two contacts on one body (robotoc's
assignment of fext: the later contact replaces the earlier, an inactive one writes zero).  Every state runs on Intermediate,
Lift and Impact grid points with four contact masks.

An entry passes when |kernel - reference| <= 1e-12 x its row's largest additive contribution (rbd_mp.row_scale, which
departs from it only for rows that vanish analytically and for the dtau/dq rows of a link far smaller than its block; the
gradient entries by the sum of the bounds of what they add), and every entry the kernels do not write keeps its bits.  Two
kernel-against-kernel checks hold bit for bit: q and -q give the same rows (the rotation of a quaternion is even in it), and
moving the base moves only C, by kp times the shift."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_rbd_mp  # noqa: E402
import rbd_mp  # noqa: E402
import rbd_ref as R  # noqa: E402
from synth import make_stage_inputs, symmetrize_lin  # noqa: E402

TOL = 1e-12
LIN = 6
KINDS = (0, 2, 1)   # Intermediate, Lift, Impact grid points (robotoc_b200.grid)
DATA = make_rbd_mp.load()
STATES = [str(s) for s in DATA["state"]]


def _states(name):
    return [s for s in range(len(STATES)) if str(DATA["model"][s]) == name]


def _inputs(s):
    return {k: DATA[k][s].copy() for k in ("q", "v", "a", "dv", "forces", "pdes")}


def _run(name, states):
    """Both kernels, in the order linearizeContactDynamics runs them, on one handle: batch entry b holds states[b] on grid
    points [Intermediate x 4 masks, Lift x 4 masks, Impact x 4 masks, Terminal].  Returns (S, ctrl, sol, lin in, lin out)."""
    from robotoc_b200 import ANYMAL, DirectMultipleShooting, RiccatiRecursion, StageDims, StageLayout, anymal_constraint_table
    from robotoc_b200.grid import plain_schedule
    s0 = _states(name)[0]
    masks, gains = [int(m) for m in DATA["masks"][s0]], DATA["gains"][s0]
    ctrl = plain_schedule(12, 0.02, 0)
    for i in range(12):
        ctrl[i].type, ctrl[i].contact_mask = KINDS[i // 4], masks[i % 4]
        ctrl[i].nf = 3 * bin(masks[i % 4]).count("1")
    table = anymal_constraint_table()
    sd = StageDims(ANYMAL, nf_max=12, n_contacts=4, n_box=table.n_box)
    S = StageLayout(sd)
    lin1, _, sol1, _ = make_stage_inputs(sd, S, ctrl, 1, 91)
    B = len(states)
    lin, sol = np.repeat(symmetrize_lin(S, lin1), B, 0), np.repeat(sol1, B, 0)
    pos = np.zeros((B, len(ctrl), 4, 3))
    for b, st in enumerate(states):
        for i in range(len(ctrl)):
            r = sol[b, i]
            r[S.s_q:S.s_q + S.nq], r[S.s_v:S.s_v + 18], r[S.s_a:S.s_a + 18], r[S.s_dv:S.s_dv + 18] = st["q"], st["v"], st["a"], st["dv"]
            if i < 12:
                r[S.s_f:S.s_f + ctrl[i].nf] = st["forces"][i % 4][:ctrl[i].nf]
            pos[b, i] = st["pdes"]
    rr = RiccatiRecursion(ANYMAL, len(ctrl), B)
    try:
        rr.setTimeDiscretization(ctrl)
        dms = DirectMultipleShooting(rr, sd, table)
        dms.setRobotModel(R.to_c(make_rbd_mp.model_of(DATA, name)))
        dms.setContactGains(gains)
        dms.setContactPositions(pos)
        dms._up(LIN, lin, S.l_stride, None)
        dms.setSolution(sol)
        dms.linearizeInverseDynamics()
        dms.linearizeContactKinematics()
        got = dms._down(LIN, lin.shape)
    finally:
        rr.close()
    return S, ctrl, sol, lin, got


def _expected(S, ctrl, sol, lin, s, b):
    """(expected records, per-entry scale, written mask) [n_grid, l_stride] of batch entry b holding npz state s."""
    nv, nvf, nfm = S.nv, S.nvf, S.nfm
    exp, sc, w = lin[b].copy(), np.zeros_like(lin[b]), np.zeros(lin[b].shape, bool)
    M, Msc = DATA["M"][s], rbd_mp.row_scale(DATA["M_scale"][s])
    J, Jsc = DATA["J"][s], rbd_mp.row_scale(DATA["J_scale"][s].reshape(-1)).reshape(4, 3)
    for i in range(12):
        c, g, j = ctrl[i], int(ctrl[i].type == 1), i % 4
        r, rs, rw = exp[i], sc[i], w[i]
        beta, mu, u = sol[b, i, S.s_beta:S.s_beta + nv], sol[b, i, S.s_mu:S.s_mu + c.nf], sol[b, i, S.s_u:S.s_u + S.nu]
        act = [ci for ci in range(4) if (c.contact_mask >> ci) & 1]
        tau, tsc = DATA["tau"][s, g, j].copy(), rbd_mp.row_scale(DATA["tau_scale"][s, g, j])
        dq, dqs = DATA["dtau_dq"][s, g, j], rbd_mp.row_scale(DATA["dtau_dq_scale"][s, g, j], rbd_mp.DQ_FLOOR)
        dv, dvs = DATA["dtau_dv"][s, g, j], DATA["dtau_dv_scale"][s, g, j]
        dvs = rbd_mp.row_scale(dvs) if g == 0 else dvs
        if g == 0:
            tau[6:] -= u
            tsc[6:] = np.maximum(tsc[6:], np.abs(u))
        Cq = np.concatenate([DATA["dC_dq"][s, g, ci] for ci in act])
        Cv = np.concatenate([DATA["dC_dv"][s, g, ci] for ci in act])
        Cqs = rbd_mp.row_scale(DATA["dC_dq_scale"][s, g].reshape(-1)).reshape(4, 3)
        Cvs = rbd_mp.row_scale(DATA["dC_dv_scale"][s, g].reshape(-1)).reshape(4, 3)
        Cs = rbd_mp.row_scale(DATA["C_scale"][s, g].reshape(-1)).reshape(4, 3)
        Ja = np.concatenate([J[ci] for ci in act])

        def put(off, rows, cols, ld, val, rowscale):
            for k in range(cols):
                r[off + k * ld:off + k * ld + rows] = val[:, k]
                rs[off + k * ld:off + k * ld + rows] = rowscale
                rw[off + k * ld:off + k * ld + rows] = True

        r[S.l_IDC:S.l_IDC + nv], rs[S.l_IDC:S.l_IDC + nv], rw[S.l_IDC:S.l_IDC + nv] = tau, tsc, True
        put(S.l_D, nv, nv, nvf, dq, dqs)
        put(S.l_D + nv * nvf, nv, nv, nvf, dv, dvs)
        put(S.l_M, nv, nv, nv, M, Msc)
        lx0, lv0, la0 = r[S.l_lx:S.l_lx + nv].copy(), r[S.l_lx + nv:S.l_lx + 2 * nv].copy(), r[S.l_la:S.l_la + nv].copy()
        lx, lxs = lx0 + dq.T @ beta, np.abs(lx0) + dqs @ np.abs(beta)
        lv, lvs = lv0 + (dv.T @ beta if g == 0 else 0.0), np.abs(lv0) + (dvs @ np.abs(beta) if g == 0 else 0.0)
        la, las = la0 + M @ beta, np.abs(la0) + Msc @ np.abs(beta)
        if act:
            nf = c.nf
            rows = lambda x: np.concatenate([x[ci] for ci in act])  # noqa: E731
            put(S.l_J, nf, nv, nfm, Ja, rows(Jsc))
            put(S.l_D + nv, nf, nv, nvf, Cq, rows(Cqs))
            put(S.l_D + nv + nv * nvf, nf, nv, nvf, Cv, rows(Cvs))
            o = S.l_IDC + nv
            r[o:o + nf] = np.concatenate([DATA["C"][s, g, ci] for ci in act])
            rs[o:o + nf], rw[o:o + nf] = rows(Cs), True
            lx, lxs = lx + Cq.T @ mu, lxs + rows(Cqs) @ np.abs(mu)
            lv, lvs = lv + Cv.T @ mu, lvs + rows(Cvs) @ np.abs(mu)
            la, las = la + Ja.T @ mu, las + rows(Jsc) @ np.abs(mu)
            lf0 = r[S.l_lf:S.l_lf + nf].copy()
            r[S.l_lf:S.l_lf + nf] = lf0 - Ja @ beta
            rs[S.l_lf:S.l_lf + nf], rw[S.l_lf:S.l_lf + nf] = np.abs(lf0) + rows(Jsc) * np.abs(beta).sum(), True
        for off, val, vs in ((S.l_lx, lx, lxs), (S.l_lx + nv, lv, lvs), (S.l_la, la, las)):
            r[off:off + nv], rs[off:off + nv], rw[off:off + nv] = val, vs, True
    return exp, sc, w


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["anymal", "chain", "star"])
def test_kernels_match_the_extended_precision_reference(name):
    idx = _states(name)
    S, ctrl, sol, lin, got = _run(name, [_inputs(s) for s in idx])
    nv = S.nv
    sections = {"IDC": (S.l_IDC, S.nvf), "D": (S.l_D, S.nvf * 2 * nv), "M": (S.l_M, nv * nv), "J": (S.l_J, S.nfm * nv),
                "lx": (S.l_lx, 2 * nv), "la": (S.l_la, nv), "lf": (S.l_lf, S.nfm)}
    worst = {}
    for b, s in enumerate(idx):
        exp, sc, w = _expected(S, ctrl, sol, lin, s, b)
        np.testing.assert_array_equal(got[b][~w], lin[b][~w], err_msg=STATES[s])   # nothing else is touched
        for key, (o, n) in sections.items():
            sl = slice(o, o + n)
            d = np.abs(got[b][:, sl] - exp[:, sl])
            e = float(np.max(np.where(d == 0, 0.0, d / np.where(sc[:, sl] > 0, sc[:, sl], 1e-300))))
            worst[(STATES[s], key)] = e
    for st in (STATES[s] for s in idx):
        print(st, " ".join(f"{k} {worst[(st, k)]:.1e}" for k in sections))
    bad = {k: e for k, e in worst.items() if not e <= TOL}
    assert not bad, bad


@pytest.mark.gpu
def test_sign_flipped_quaternion_gives_identical_bits():
    st = _inputs(STATES.index("trot"))
    neg = {k: x.copy() for k, x in st.items()}
    neg["q"][3:7] = -neg["q"][3:7]
    _, _, _, _, got = _run("anymal", [st, neg])
    np.testing.assert_array_equal(got[0], got[1])


@pytest.mark.gpu
def test_moving_the_base_moves_only_the_baumgarte_rows():
    st = _inputs(STATES.index("trot"))
    shift = np.array([1000.0, -500.0, 3.0])
    moved = {k: x.copy() for k, x in st.items()}
    moved["q"][:3] += shift
    S, ctrl, _, _, got = _run("anymal", [st, moved])
    kp = DATA["gains"][STATES.index("trot")][:, 0]
    for i, c in enumerate(ctrl):
        C = np.zeros(S.l_stride, bool)
        if c.type in (0, 2) and c.nf:
            C[S.l_IDC + S.nv:S.l_IDC + S.nv + c.nf] = True
            act = [ci for ci in range(4) if (c.contact_mask >> ci) & 1]
            dC = got[1, i, C] - got[0, i, C]
            want = np.concatenate([kp[ci] * shift for ci in act])
            bound = TOL * np.concatenate([kp[ci] * (np.abs(shift) + np.abs(st["pdes"][ci]) + 1.0) for ci in act])
            assert (np.abs(dC - want) <= bound).all(), (i, dC - want)
        np.testing.assert_array_equal(got[1, i, ~C], got[0, i, ~C], err_msg=str(i))
