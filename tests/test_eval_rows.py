"""Rows a12 / a13 / a16 of SURVEY.md 8a: PerformanceIndex of evalKKT (KKT error, primal / dual feasibility, log barrier),
pdipm::setSlackAndDualPositive and computeInitialStateDirection.
CPU: the oracle against an independent numpy statement of the reference formulas; GPU: the CUDA path against the oracle."""
import ctypes

import numpy as np
import pytest

import oracle_lib
from iteration_check import oracle_perf_index as _oracle_perf
from helpers import contact_mask_walk_schedule, crawl_schedule, jump_sto_schedule, small_event_schedule, trot_schedule
from robotoc_b200 import ANYMAL, StageDims, StageLayout, anymal_constraint_table
from robotoc_b200.grid import IMPACT, TERMINAL
from synth import make_stage_inputs, mat


def _setup(sched, batch, seed, getter=None, impact_cones=False):
    lib = oracle_lib.load()
    table = anymal_constraint_table(impact_friction_cone=impact_cones)
    sd = StageDims(ANYMAL, nf_max=12, n_contacts=table.n_contacts, n_box=table.n_box)
    S = StageLayout(sd, getter=getter or lib.orc_stage_layout_get)
    td, ev, ctrl = sched
    lin, con, sol, dx0 = make_stage_inputs(sd, S, ctrl, batch, seed, impact_cones=impact_cones)
    # give the residual slots of the records something to measure
    rng = np.random.default_rng(seed + 1)
    for i, c in enumerate(ctrl):
        if c.type not in (IMPACT, TERMINAL):
            lin[:, i, S.l_p:S.l_p + c.ns] = rng.uniform(-1, 1, size=(batch, c.ns))
    lib.orc_perf_index_batch.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 3
    lib.orc_set_slack_dual_positive_batch.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    lib.orc_initial_state_direction.argtypes = [ctypes.c_void_p] + [ctypes.c_void_p] * 5
    return lib, table, sd, S, ctrl, lin, con, sol, dx0


def _numpy_perf(S, table, ctrl, lin, con):
    """The reference formulas, vectorised over the batch (intermediate_stage.cpp:128-132 and what it calls)."""
    b = lin.shape[0]
    kkt, pf, df, lb = np.zeros(b), np.zeros(b), np.zeros(b), np.zeros(b)
    sq = lambda x: np.sum(x * x, axis=1)  # noqa: E731
    l1 = lambda x: np.sum(np.abs(x), axis=1)  # noqa: E731
    for i, c in enumerate(ctrl):
        rec, cc = lin[:, i], con[:, i]
        lx = rec[:, S.l_lx:S.l_lx + S.nx]
        kkt += sq(lx); df += l1(lx)
        if c.type == TERMINAL:
            continue
        Fx, la, lf = rec[:, S.l_Fx:S.l_Fx + S.nx], rec[:, S.l_la:S.l_la + S.nv], rec[:, S.l_lf:S.l_lf + c.nf]
        IDC = rec[:, S.l_IDC:S.l_IDC + S.nv + c.nf]
        kkt += sq(Fx) + sq(la) + sq(lf) + sq(IDC)
        pf += l1(Fx) + l1(IDC)
        df += l1(la) + l1(lf)
        if c.type == IMPACT and not table.impact_friction_cone:
            continue
        if c.type != IMPACT:
            lu, lup, p = rec[:, S.l_lu:S.l_lu + S.nu], rec[:, S.l_lup:S.l_lup + S.np], rec[:, S.l_p:S.l_p + c.ns]
            kkt += sq(lu) + sq(lup) + sq(p)
            df += l1(lu) + l1(lup)
            pf += l1(p)
        act = np.ones(S.nc, dtype=bool)
        if c.type == IMPACT:
            act[:S.nbox] = False  # impact stages only carry the ImpactFrictionCone rows
        for r in range(S.nbox):  # ConstraintsData::setTimeStage: position level from stage 2, velocity level from stage 1 on
            level = {0: 2, 1: 1}.get(table.box[r].var, 0)
            if level + c.ineq_gate > 2:
                act[r] = False
        for ci in range(S.ncon):
            if not (c.contact_mask >> ci) & 1:
                act[S.nbox + 5 * ci:S.nbox + 5 * ci + 5] = False
        sl, du, res = cc[:, S.c_slack:S.c_slack + S.nc][:, act], cc[:, S.c_dual:S.c_dual + S.nc][:, act], cc[:, S.c_res:S.c_res + S.nc][:, act]
        cm = sl * du - table.barrier
        kkt += sq(res) + sq(cm)
        pf += l1(res)
        df += l1(cm)
        lb += -table.barrier * np.sum(np.log(sl), axis=1)
    return np.stack([np.zeros(b), lb, pf, df, kkt, np.sqrt(kkt), np.zeros(b), np.zeros(b)], axis=1)


@pytest.mark.parametrize("which", ["small", "small_sto", "trot", "trot_icone"])
def test_oracle_performance_index_matches_the_reference_formulas(which):
    sched = {"small": small_event_schedule(False), "small_sto": small_event_schedule(True), "trot": trot_schedule(40),
             "trot_icone": trot_schedule(40)}[which]
    lib, table, sd, S, ctrl, lin, con, sol, dx0 = _setup(sched, 3, 61, impact_cones=which.endswith("icone"))
    got = _oracle_perf(lib, sd, table, ctrl, lin, con)
    want = _numpy_perf(S, table, ctrl, lin, con)
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=0)
    assert (got[:, 4] > 0).all() and (got[:, 5] > 0).all()


def test_oracle_set_slack_and_dual_positive_and_initial_state_direction():
    lib, table, sd, S, ctrl, lin, con, sol, dx0 = _setup(small_event_schedule(False), 2, 62)
    rng = np.random.default_rng(5)
    con[:, :, S.c_slack:S.c_slack + S.nc] = rng.uniform(-0.5, 0.5, size=(2, len(ctrl), S.nc))  # infeasible start
    want = con.copy()
    csd = sd.c()
    lib.orc_set_slack_dual_positive_batch(ctypes.byref(csd), ctypes.byref(table), ctrl, len(ctrl), 2, oracle_lib.ptr(con))
    sb = np.sqrt(table.barrier)
    for i, c in enumerate(ctrl):
        if c.type in (IMPACT, TERMINAL):
            continue
        on = np.array([r >= S.nbox or {0: 2, 1: 1}.get(table.box[r].var, 0) + c.ineq_gate <= 2 for r in range(S.nc)])
        sl = np.maximum(want[:, i, S.c_slack:S.c_slack + S.nc], sb)
        want[:, i, S.c_slack:S.c_slack + S.nc] = np.where(on, sl, want[:, i, S.c_slack:S.c_slack + S.nc])
        want[:, i, S.c_dual:S.c_dual + S.nc] = np.where(on, table.barrier / sl, want[:, i, S.c_dual:S.c_dual + S.nc])
    np.testing.assert_array_equal(con, want)
    assert (con[:, 2:-1, S.c_slack:S.c_slack + S.nc][:, [i - 2 for i, c in enumerate(ctrl[:-1]) if i >= 2 and c.type != IMPACT]] >= sb).all()
    # initial state direction: dq[0:6] = -Fqq_prev_inv dq_raw[0:6], dv = v0 - v
    ex0 = rng.uniform(-1, 1, size=S.e_stride)
    dq_raw, v0 = rng.uniform(-1, 1, size=18), rng.uniform(-1, 1, size=18)
    out = np.zeros(36)
    P = oracle_lib.ptr
    lib.orc_initial_state_direction(ctypes.byref(csd), P(ex0), P(np.ascontiguousarray(sol[0, 0])), P(dq_raw), P(v0), P(out))
    Fi = mat(ex0, S.e_Fqqpi, 6, 6)
    want_dx = np.concatenate([-Fi @ dq_raw[:6], dq_raw[6:], v0 - sol[0, 0, S.s_v:S.s_v + 18]])
    np.testing.assert_allclose(out, want_dx, rtol=1e-14, atol=1e-15)


@pytest.mark.gpu
@pytest.mark.parametrize("which,batch", [("small_sto", 3), ("trot", 16), ("jump", 4), ("trot_icone", 5), ("crawl_icone", 4),
                                         ("mask_walk", 3)])
def test_cuda_eval_rows_match_the_oracle(which, batch):
    from robotoc_b200 import DirectMultipleShooting, RiccatiRecursion
    sched = {"small_sto": lambda: small_event_schedule(True), "trot": lambda: trot_schedule(40), "jump": lambda: jump_sto_schedule(80),
             "trot_icone": lambda: trot_schedule(40), "crawl_icone": lambda: crawl_schedule(54),
             "mask_walk": contact_mask_walk_schedule}[which]()
    lib, table, sd, S, ctrl, lin, con, sol, dx0 = _setup(sched, batch, 63, getter=None, impact_cones=which.endswith("icone"))
    S = StageLayout(sd)
    rr = RiccatiRecursion(ANYMAL, len(ctrl), batch)
    rr.setTimeDiscretization(ctrl)
    dms = DirectMultipleShooting(rr, sd, table)
    # PerformanceIndex / KKTError
    got = dms.evalKKT(lin, con)
    want = _oracle_perf(lib, sd, table, ctrl, lin, con)
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=0)
    np.testing.assert_allclose(dms.KKTError(), want[:, 5], rtol=1e-12)
    # setSlackAndDualPositive
    rng = np.random.default_rng(7)
    con2 = con.copy()
    con2[:, :, S.c_slack:S.c_slack + S.nc] = rng.uniform(-0.5, 0.5, size=(batch, len(ctrl), S.nc))
    dms.setSlackAndDualPositive(con2)
    got_con = dms.getConstraintData()
    csd = sd.c()
    lib.orc_set_slack_dual_positive_batch(ctypes.byref(csd), ctypes.byref(table), ctrl, len(ctrl), batch, oracle_lib.ptr(con2))
    for f in ("c_slack", "c_dual"):
        o = getattr(S, f)
        np.testing.assert_allclose(got_con[:, :, o:o + S.nc], con2[:, :, o:o + S.nc], rtol=1e-15, atol=0)
    # computeInitialStateDirection (needs the stage-0 Fqq_prev_inv of the condensing and s[0].v)
    dms.condense(lin, con)
    dms._up(9, sol, S.s_stride, None)
    dq0, v0 = rng.uniform(-1, 1, size=(batch, 18)), rng.uniform(-1, 1, size=(batch, 18))
    dms.computeInitialStateDirection(dq0, v0)
    got_dx0 = dms.getInitialStateDirection()
    ex = dms.getExpansionData()
    for b in range(batch):
        out = np.zeros(36)
        lib.orc_initial_state_direction(ctypes.byref(csd), oracle_lib.ptr(np.ascontiguousarray(ex[b, 0])),
                                        oracle_lib.ptr(np.ascontiguousarray(sol[b, 0])), oracle_lib.ptr(np.ascontiguousarray(dq0[b])),
                                        oracle_lib.ptr(np.ascontiguousarray(v0[b])), oracle_lib.ptr(out))
        np.testing.assert_allclose(got_dx0[b], out, rtol=1e-13, atol=1e-15)
    rr.close()
