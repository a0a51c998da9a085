"""Pins oracle/unconstr_stage_oracle.c by identities that do not depend on its code (numpy dense algebra):
UnconstrDynamics::condenseUnconstrDynamics / expandPrimal / expandDual (src/dynamics/unconstr_dynamics.cpp:67-104),
joint-limit PDIPM condensing (joint_*_limit.cpp:68-83, pdipm.hxx) -- cf. the reference's own
test/dynamics/unconstr_dynamics_test.cpp (condense vs explicit block formulas)."""
import ctypes

import numpy as np
import pytest

import oracle_lib
from oracle_lib import ptr
from robotoc_b200.layout import ULayout
from robotoc_b200.stage import VAR_A, VAR_Q, VAR_U, VAR_V
from robotoc_b200.unconstr_dms import UStageLayout, iiwa14_constraint_table
from synth import make_unconstr_stage_inputs

NV = 7


def _layouts(tab):
    lib = oracle_lib.load()
    S = UStageLayout(NV, tab.n_box, getter=lib.orc_ustage_layout_get)
    UL = ULayout(NV, getter=lib.orc_ulayout_get)
    return lib, S, UL


def _m(rec, off, m, n):
    return rec[off:off + m * n].reshape(n, m).T.copy()


def _jac(tab):
    """Constraint Jacobian of the table over z = (q, v, a, u)."""
    J = np.zeros((tab.n_box, 4 * NV))
    for r in range(tab.n_box):
        b = tab.box[r]
        J[r, {VAR_Q: 0, VAR_V: 1, VAR_A: 2, VAR_U: 3}[b.var] * NV + b.idx] = b.sign
    return J


def _acts(tab, stage):
    """Rows that act on grid point `stage` (ConstraintsData::setTimeStage, constraints_data.cpp:20-45): position rows from
    stage 2, velocity rows from stage 1, acceleration and torque rows everywhere."""
    return np.array([stage >= {VAR_Q: 2, VAR_V: 1}.get(tab.box[r].var, 0) for r in range(tab.n_box)])


def test_layout_matches_header_rules():
    tab = iiwa14_constraint_table()
    lib, S, UL = _layouts(tab)
    assert S.nbox == 42 and S.ncp == 42 and S.nx == 14
    for f in ("l_stride", "e_stride", "c_stride", "s_stride", "x_stride"):
        assert getattr(S, f) % 16 == 0
    assert S.l_stride == 512


def test_condensed_model_equals_substituted_model():
    _check_condensed_model(2)


@pytest.mark.parametrize("stage", [0, 1])
def test_condensed_model_on_grid_points_0_and_1_carries_only_the_rows_that_act(stage):
    """Grid point 0 carries the torque and acceleration rows, grid point 1 also the velocity rows; the PDIPM records of the
    other rows are left as they came in."""
    _check_condensed_model(stage)


def _check_condensed_model(stage):
    tab = iiwa14_constraint_table()
    tab.box[5].var = VAR_A  # make sure an acceleration row is exercised too
    lib, S, UL = _layouts(tab)
    lin, con, sol, dx0 = make_unconstr_stage_inputs(S, 1, 4, seed=5)
    nx = 2 * NV
    act = _acts(tab, stage)
    assert act.sum() == {0: 15, 1: 29, 2: 42}[stage]
    for b in range(4):
        l, c = lin[b, 0].copy(), con[b, 0].copy()
        c[S.c_cmpl:S.c_cmpl + tab.n_box] = c[S.c_cond:S.c_cond + tab.n_box] = np.nan  # rows that do not act stay untouched
        c_in = c.copy()
        kkt, ex = np.zeros(UL.k_stride), np.zeros(S.e_stride)
        lib.orc_ustage_condense_at(NV, ctypes.byref(tab), stage, 0, ptr(l), ptr(c), ptr(kkt), ptr(ex))
        # full model over z = (q, v, a, u) after the PDIPM terms of the rows that act
        slack, dual, res = (con[b, 0, o:o + tab.n_box][act] for o in (S.c_slack, S.c_dual, S.c_res))
        J = _jac(tab)[act]
        cmpl = slack * dual - tab.barrier
        cond = (dual * res - cmpl) / slack
        H = np.zeros((4 * NV, 4 * NV))
        H[:nx, :nx] = _m(l, S.l_Qxx, nx, nx)
        H[nx:nx + NV, nx:nx + NV] = _m(l, S.l_Qaa, NV, NV)
        H[3 * NV:, 3 * NV:] = _m(l, S.l_Quu, NV, NV)
        g = np.concatenate([l[S.l_lx:S.l_lx + nx], l[S.l_la:S.l_la + NV], l[S.l_lu:S.l_lu + NV]])
        H += J.T @ np.diag(dual / slack) @ J
        g += J.T @ cond
        np.testing.assert_allclose(c[S.c_cmpl:S.c_cmpl + tab.n_box][act], cmpl, rtol=1e-14)
        np.testing.assert_allclose(c[S.c_cond:S.c_cond + tab.n_box][act], cond, rtol=1e-13)
        for o in (S.c_cmpl, S.c_cond):
            np.testing.assert_array_equal(c[o:o + tab.n_box][~act], c_in[o:o + tab.n_box][~act])
        np.testing.assert_array_equal(np.delete(c, np.r_[S.c_cmpl:S.c_cmpl + tab.n_box, S.c_cond:S.c_cond + tab.n_box]),
                                      np.delete(c_in, np.r_[S.c_cmpl:S.c_cmpl + tab.n_box, S.c_cond:S.c_cond + tab.n_box]))
        # substitute du = ID + D y, y = (dq, dv, da)
        D = np.hstack([_m(l, S.l_dIDdq, NV, NV), _m(l, S.l_dIDdv, NV, NV), _m(l, S.l_dIDda, NV, NV)])
        ID = l[S.l_ID:S.l_ID + NV]
        T = np.vstack([np.eye(3 * NV), D])  # z = T y + [0; ID]
        Hc = T.T @ H @ T
        gc = T.T @ (g + H @ np.concatenate([np.zeros(3 * NV), ID]))
        Qxx = _m(kkt, UL.k_Qxx, nx, nx)
        Qxu = _m(kkt, UL.k_Qxu, nx, NV)
        Qaa = _m(kkt, UL.k_Qaa, NV, NV)
        scale = np.abs(Hc).max()
        assert np.abs(Qxx - Hc[:nx, :nx]).max() / scale < 1e-14
        assert np.abs(Qxu - Hc[:nx, nx:]).max() / scale < 1e-14
        assert np.abs(Qaa - Hc[nx:, nx:]).max() / scale < 1e-14
        np.testing.assert_allclose(kkt[UL.k_lx:UL.k_lx + nx], gc[:nx], rtol=1e-12, atol=1e-13)
        np.testing.assert_allclose(kkt[UL.k_la:UL.k_la + NV], gc[nx:], rtol=1e-12, atol=1e-13)
        np.testing.assert_array_equal(kkt[UL.k_Fx:UL.k_Fx + nx], l[S.l_Fx:S.l_Fx + nx])
        # expansion record = lu, Quu after the constraints
        np.testing.assert_allclose(ex[S.e_lu:S.e_lu + NV], g[3 * NV:], rtol=1e-13)
        np.testing.assert_allclose(_m(ex, S.e_Quu, NV, NV), H[3 * NV:, 3 * NV:], rtol=1e-13)


def test_only_the_diagonal_of_quu_is_condensed():
    """unconstr_dynamics.cpp:70-78 uses kkt_matrix.Quu.diagonal(); expandDual (:103) uses the full Quu."""
    tab = iiwa14_constraint_table()
    lib, S, UL = _layouts(tab)
    lin, con, sol, dx0 = make_unconstr_stage_inputs(S, 1, 1, seed=9)
    l = lin[0, 0].copy()
    k0, e0 = np.zeros(UL.k_stride), np.zeros(S.e_stride)
    lib.orc_ustage_condense(NV, ctypes.byref(tab), 0, ptr(l), ptr(con[0, 0].copy()), ptr(k0), ptr(e0))
    l2 = l.copy()
    l2[S.l_Quu + 1] += 0.37  # Quu(1,0)
    l2[S.l_Quu + NV] += 0.37  # Quu(0,1)
    k1, e1 = np.zeros(UL.k_stride), np.zeros(S.e_stride)
    lib.orc_ustage_condense(NV, ctypes.byref(tab), 0, ptr(l2), ptr(con[0, 0].copy()), ptr(k1), ptr(e1))
    np.testing.assert_array_equal(k0, k1)
    assert e1[S.e_Quu + 1] - e0[S.e_Quu + 1] == 0.37


def test_terminal_stage_copies_cost_only():
    tab = iiwa14_constraint_table()
    lib, S, UL = _layouts(tab)
    lin, con, sol, dx0 = make_unconstr_stage_inputs(S, 1, 1, seed=3)
    l = lin[0, 1].copy()
    c = con[0, 1].copy()
    kkt, ex = np.full(UL.k_stride, np.nan), np.full(S.e_stride, np.nan)
    lib.orc_ustage_condense(NV, ctypes.byref(tab), 1, ptr(l), ptr(c), ptr(kkt), ptr(ex))
    np.testing.assert_array_equal(kkt[UL.k_Qxx:UL.k_Qxx + 196], l[S.l_Qxx:S.l_Qxx + 196])
    np.testing.assert_array_equal(kkt[UL.k_lx:UL.k_lx + 14], l[S.l_lx:S.l_lx + 14])
    assert not kkt[UL.k_Qxu:UL.k_Fx].any() and not ex.any()
    np.testing.assert_array_equal(c, con[0, 1])


def test_expand_update_consistency():
    """One full iteration on the oracle; the expanded step satisfies the linearised stage equations it was eliminated from, on
    the rows that act on each grid point; the PDIPM records of the rows that do not act (position rows on grid points 0 and 1,
    velocity rows on grid point 0) come out bit-unchanged, and those rows take no part in the step sizes."""
    tab = iiwa14_constraint_table()
    lib, S, UL = _layouts(tab)
    N, dt, batch = 6, 0.05, 3
    lin, con, sol, dx0 = make_unconstr_stage_inputs(S, N, batch, seed=21)
    out = oracle_lib.unconstr_iteration(NV, UL, S, tab, N, dt, lin, con, sol, dx0)
    assert out["info"] == 0
    J = _jac(tab)
    nb = tab.n_box
    for b in range(batch):
        mins_p, mins_d = [], []
        for i in range(N):
            l, d, xd, ex = lin[b, i], out["dir"][b, i], out["xd"][b, i], out["ex"][b, i]
            dq, dv, da = d[UL.d_dx:UL.d_dx + NV], d[UL.d_dx + NV:UL.d_dx + 2 * NV], d[UL.d_da:UL.d_da + NV]
            du = l[S.l_ID:S.l_ID + NV] + _m(l, S.l_dIDdq, NV, NV) @ dq + _m(l, S.l_dIDdv, NV, NV) @ dv + _m(l, S.l_dIDda, NV, NV) @ da
            np.testing.assert_allclose(xd[S.x_du:S.x_du + NV], du, rtol=1e-12, atol=1e-13)
            # stationarity w.r.t. u of the stage Lagrangian: lu' + Quu' du - dt*dbeta = 0   (linearizeUnconstrDynamics :62)
            dbeta = xd[S.x_dbeta:S.x_dbeta + NV]
            np.testing.assert_allclose(ex[S.e_lu:S.e_lu + NV] + _m(ex, S.e_Quu, NV, NV) @ du - dt * dbeta, 0, atol=1e-11)
            act = _acts(tab, i)
            for rec in (out["con_condensed"], out["con_expanded"], out["con"]):
                rows = lambda c: c[:7 * S.ncp].reshape(7, S.ncp)[:, :nb][:, ~act]  # noqa: E731  (slack ... ddual)
                np.testing.assert_array_equal(rows(rec[b, i]), rows(con[b, i]))
            c0, c1 = out["con_condensed"][b, i], out["con_expanded"][b, i]
            slack, dual, res, cmpl = (c0[o:o + nb][act] for o in (S.c_slack, S.c_dual, S.c_res, S.c_cmpl))
            dslack, ddual = c1[S.c_dslack:S.c_dslack + nb][act], c1[S.c_ddual:S.c_ddual + nb][act]
            z = np.concatenate([dq, dv, da, du])
            np.testing.assert_allclose(J[act] @ z + dslack + res, 0, atol=1e-12)            # linearised g + slack = 0
            np.testing.assert_allclose(slack * ddual + dual * dslack + cmpl, 0, atol=1e-12)  # linearised complementarity
            fp = -tab.fraction_to_boundary * (slack / dslack)
            fd = -tab.fraction_to_boundary * (dual / ddual)
            mins_p.append(min([1.0] + [f for f in fp if 0 < f < 1]))
            mins_d.append(min([1.0] + [f for f in fd if 0 < f < 1]))
            ps, ds = out["steps"][b]
            np.testing.assert_allclose(out["con"][b, i, S.c_slack:S.c_slack + nb][act], slack + ps * dslack, rtol=1e-14)
            np.testing.assert_allclose(out["con"][b, i, S.c_dual:S.c_dual + nb][act], dual + ds * ddual, rtol=1e-14)
            assert (out["con"][b, i, S.c_slack:S.c_slack + nb] > 0).all() and (out["con"][b, i, S.c_dual:S.c_dual + nb] > 0).all()
            for off, dd in ((S.s_q, dq), (S.s_v, dv), (S.s_a, da), (S.s_u, du), (S.s_beta, dbeta)):
                np.testing.assert_allclose(out["sol"][b, i, off:off + NV], sol[b, i, off:off + NV] + ps * dd, rtol=1e-13, atol=1e-14)
        assert out["steps"][b, 0] == min(mins_p) and out["steps"][b, 1] == min(mins_d)
        # terminal stage: q, v, lmd, gmm move; a, u, beta and the PDIPM data do not
        dT = out["dir"][b, N]
        ps = out["steps"][b, 0]
        np.testing.assert_allclose(out["sol"][b, N, S.s_q:S.s_q + NV], sol[b, N, S.s_q:S.s_q + NV] + ps * dT[UL.d_dx:UL.d_dx + NV], rtol=1e-13)
        np.testing.assert_array_equal(out["sol"][b, N, S.s_a:S.s_a + NV], sol[b, N, S.s_a:S.s_a + NV])
        np.testing.assert_array_equal(out["con"][b, N], con[b, N])
