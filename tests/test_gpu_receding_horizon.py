"""The device iteration on the schedules an MPC loop meets as its horizon slides over a gait (helpers.receding_horizon_schedules):
events in the first interval, on grid 1 and beside it, a hair after t0, at the last admissible grid points, steps far below
T / N, grid 0 already in a later phase, and n_grid changing from one call to the next on the same handle.  Everything goes
through the C ABI; the CPU oracle and the segmented-sweep comparison of test_gpu_parity are the references."""
import os
import sys

import numpy as np
import pytest

import oracle_lib
from helpers import RH_SETS, receding_horizon_schedules
from iteration_check import (_cmp, compare_final, compare_reference_records, compare_riccati, cuda_iteration_records, mask_unread_sto,
                             oracle_iteration, oracle_perf_index, oracle_sensitivity, oracle_trials, reference_view_of_expansion)
from robotoc_b200 import ANYMAL, DirectMultipleShooting, Layout, RiccatiRecursion, StageDims, StageLayout, anymal_constraint_table
from robotoc_b200.grid import IMPACT, TERMINAL
from robotoc_b200.stage import VAR_Q, VAR_V
from synth import make_kkt, make_stage_inputs, robotoc_cost_structure, symmetrize_lin

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_golden_ref_live as mgl  # noqa: E402
from golden_sample import load, restore  # noqa: E402

pytestmark = pytest.mark.gpu
TOL = 1e-8
RESERVED = 5  # events a handle is sized for (a crawl horizon holds five): n_grid_max = N + 1 + 3 * RESERVED, as the reference sizes its data


def _problem(impact_cones=False):
    table = anymal_constraint_table(impact_friction_cone=impact_cones)
    sd = StageDims(ANYMAL, nf_max=12, n_contacts=table.n_contacts, n_box=table.n_box)
    return table, sd, StageLayout(sd), Layout(ANYMAL)


def _handle(N, batch, sd, table):
    rr = RiccatiRecursion(ANYMAL, N + 1 + 3 * RESERVED, batch)
    return rr, DirectMultipleShooting(rr, sd, table)


def _acting_rows(table, S, c):
    """The PDIPM rows that act on grid point `c`: box rows whose level is valid there (not on impacts, position / velocity
    level not on grid 0 / 1), friction-cone rows of the closed contacts (on impacts: of the impact, if the table has
    ImpactFrictionCone).  The derived fields (cmpl, cond, ...) of the other rows are never rewritten, so on a handle that
    ran another schedule before they hold that schedule's values; nothing reads them."""
    rows = []
    for r in range(S.nc):
        if r < S.nbox:
            level = {VAR_Q: 2, VAR_V: 1}.get(table.box[r].var, 0)
            ok = c.type != IMPACT and level + c.ineq_gate <= 2
        else:
            ok = (c.type != IMPACT or table.impact_friction_cone) and (c.contact_mask >> ((r - S.nbox) // 5)) & 1
        if ok:
            rows.append(r)
    return np.array(rows, dtype=int)


def _mask_absent_sections(K, ctrl, kkt):
    """Zeroes (in place) the KKT sections a grid point does not have: the control rows and fx of an impact, the switching-
    constraint rows beyond its ns (impact and terminal grid points are compared on their own sections only).  The device never writes them, so on a reused handle they hold the previous schedule's
    values; the oracle writes zeros and nothing reads them."""
    nx, nu, nv, nsm = K.nx, K.nu, K.nv, ANYMAL.ns_max
    for i, c in enumerate(ctrl):
        if c.type == IMPACT:
            for off, n in ((K.k_Fvu, nv * nu), (K.k_Qxu, nx * nu), (K.k_Quu, nu * nu), (K.k_lu, nu), (K.k_fx, nx)):
                kkt[:, i, off:off + n] = 0.0
        ns = 0 if c.type == IMPACT else c.ns
        for off, w in ((K.k_Phix, nx), (K.k_Phiu, nu), (K.k_p, 1), (K.k_Phit, 1)):
            kkt[:, i, off + ns * w:off + nsm * w] = 0.0
    return kkt


def _tolerance(sd, S, K, table, td, ctrl, lin, con, sol, dx0, ref):
    """TOL per OCP; on a schedule with a step below 1e-3 T / N, the condition-aware bound of iteration_check (the
    oracle's own sensitivity to one rounding error of its inputs) where that is larger."""
    if min(c.dt for c in ctrl[:-1] if c.type != IMPACT) >= 1e-3 * td.T / td.N:
        return TOL, None
    sens = oracle_sensitivity(sd, S, K, table, ctrl, lin, con, sol, dx0, ref)
    return np.where(sens > 1e-3 * TOL, np.maximum(TOL, 1e3 * sens), TOL), sens


def _check_iteration(rr, dms, sd, S, K, table, td, ctrl, lin, con, sol, dx0, worst, reused):
    """condense -> backward -> forward -> step sizes -> update on the device, every block of every grid point after every
    call against the oracle (the blocks of test_gpu_stage); `worst` collects the largest error per block family.  On a
    handle that ran another schedule before (`reused`), sections and PDIPM rows the grid point does not have are left out:
    they hold that schedule's values (see _acting_rows, _mask_absent_sections); a fresh handle compares whole records."""
    ref = oracle_iteration(sd, S, K, table, ctrl, lin, con, sol, dx0)
    tol, sens = _tolerance(sd, S, K, table, td, ctrl, lin, con, sol, dx0, ref)

    def cmp(family, name, got, want):
        _cmp(name, got, want, tol, worst.setdefault(family, [0.0, TOL]))

    def cmp_rows(name, c, f, got, want):
        if reused:
            rows = _acting_rows(table, S, c)
        elif c.type != IMPACT:
            rows = np.arange(S.nc)
        else:
            rows = np.arange(S.nbox if table.impact_friction_cone else S.nc, S.nc)
        if rows.size:
            o = getattr(S, f)
            cmp("pdipm", name, got[:, o + rows], want[:, o + rows])

    rr.setTimeDiscretization(ctrl)
    dms.condense(lin, con)
    kkt = mask_unread_sto(K, S, ctrl, kkt=dms.getKKT())
    kkt_ref = mask_unread_sto(K, S, ctrl, kkt=ref["kkt"].copy())
    if reused:
        kkt, kkt_ref = _mask_absent_sections(K, ctrl, kkt), _mask_absent_sections(K, ctrl, kkt_ref)
    cc = dms.getConstraintData()
    nx = K.nx
    for i, c in enumerate(ctrl):
        if reused and c.type in (IMPACT, TERMINAL):  # the sections such a grid point has: Fxx, Fx (impact), Qxx, lx
            secs = ((K.k_Qxx, nx * nx), (K.k_lx, nx)) + (((K.k_Fxx, nx * nx), (K.k_Fx, nx)) if c.type == IMPACT else ())
            for off, n in secs:
                cmp("kkt", f"kkt[{i}]", kkt[:, i, off:off + n], kkt_ref[:, i, off:off + n])
        else:
            cmp("kkt", f"kkt[{i}]", kkt[:, i], kkt_ref[:, i])
        if c.type != TERMINAL:
            for f in ("c_cmpl", "c_cond"):
                cmp_rows(f"{f}[{i}]", c, f, cc[:, i], ref["cc_cond"][:, i])
    rr.backwardRiccatiRecursion()
    rr.forwardRiccatiRecursion(dx0)
    cmp("direction", "direction", rr.getDirection(), ref["d"])
    dms.computeStepSizes()
    xd, cc = dms.getExpandedDirection(), dms.getConstraintData()
    for i, c in enumerate(ctrl):
        if c.type == TERMINAL:
            continue
        cmp("expanded direction", f"daf[{i}]", xd[:, i, S.x_daf:S.x_daf + 18 + c.nf], ref["xd_exp"][:, i, S.x_daf:S.x_daf + 18 + c.nf])
        for f in ("c_dslack", "c_ddual"):
            cmp_rows(f"{f}[{i}]", c, f, cc[:, i], ref["cc_exp"][:, i])
    dms.integrateSolution(sol)
    assert int(rr.info().max()) == 0
    steps = np.stack([dms.maxPrimalStepSize(), dms.maxDualStepSize()], axis=1)
    ric, d, sol_g, cc = rr.getRiccatiFactorization(), rr.getDirection(), dms.getSolution(), dms.getConstraintData()
    w = worst.setdefault("riccati, direction, solution, step sizes", [0.0, TOL])
    w[0] = max(w[0], compare_final(S, K, ctrl, ref, ric, d, steps, sol_g, cc, TOL, sensitivity=sens))
    xd = dms.getExpandedDirection()
    ex = reference_view_of_expansion(S, dms.getExpansionData())
    for i, c in enumerate(ctrl):
        if c.type == TERMINAL:
            continue
        cmp("expanded direction", f"dbetamu[{i}]", xd[:, i, S.x_dbetamu:S.x_dbetamu + 18 + c.nf],
            ref["xd_upd"][:, i, S.x_dbetamu:S.x_dbetamu + 18 + c.nf])
        if c.type != IMPACT:
            cmp("expanded direction", f"dnup[{i}]", xd[:, i, S.x_dnup:S.x_dnup + 6], ref["xd_upd"][:, i, S.x_dnup:S.x_dnup + 6])
        nz = 1080 if c.type == IMPACT else 1080 + 540
        cmp("expansion", f"Qafqv|Qafu[{i}]", ex[:, i, S.e_Qafqv:S.e_Qafqv + nz], ref["ex_upd"][:, i, S.e_Qafqv:S.e_Qafqv + nz])
        for f, n in (("e_Z", 900), ("e_R", 1080), ("e_r", 30), ("e_laf", 30)):
            o = getattr(S, f)
            cmp("expansion", f"{f}[{i}]", ex[:, i, o:o + n], ref["ex_upd"][:, i, o:o + n])


def _report(what, worst):
    print(f"{what}: worst rel err vs oracle " + ", ".join(f"{k} {v[0]:.2e}" for k, v in sorted(worst.items())))


@pytest.mark.parametrize("gait,sto", RH_SETS)
def test_sweep_on_one_handle(gait, sto):
    """t0 over one gait cycle in steps of dt / 4 (crawl: dt / 2, its cycle is twice as long) on ONE handle sized for
    N + 1 + 3 * RESERVED grid points, as an MPC loop runs it: re-set the schedule, upload fresh records (batch 2), run the
    iteration, compare with the oracle."""
    table, sd, S, K = _problem()
    sched = receding_horizon_schedules(gait, sto, "sweep", per_dt=2 if gait == "crawl" else 4)
    rr, dms = _handle(sched[0][1].N, 2, sd, table)
    worst = {}
    for k, (t0, td, ev, ctrl) in enumerate(sched):
        lin, con, sol, dx0 = make_stage_inputs(sd, S, ctrl, 2, 9000 + k)
        try:
            _check_iteration(rr, dms, sd, S, K, table, td, ctrl, lin, con, sol, dx0, worst, reused=k > 0)
        except AssertionError as e:
            raise AssertionError(f"{gait} sto={sto} t0={t0!r} (n_grid {len(ctrl)}): {e}") from None
    rr.close()
    _report(f"sweep {gait} sto={sto}", worst)


def _edge_schedules(order_for_reuse=False):
    """The edge sets of RH_SETS; for reuse, ordered so that STO and non-STO schedules alternate and n_grid changes at every
    step."""
    sets = [(g, s, x) for g, s in RH_SETS for x in receding_horizon_schedules(g, s, "edge")]
    if not order_for_reuse:
        return sets
    pools = [[x for x in sets if x[1]], [x for x in sets if not x[1]]]
    out, prev = [], None
    while pools[0] or pools[1]:
        pool = pools[len(out) % 2] or pools[(len(out) + 1) % 2]
        k = next((j for j, x in enumerate(pool) if prev is None or len(x[2][3]) != prev), 0)
        x = pool.pop(k)
        out.append(x)
        prev = len(x[2][3])
    return out


def _all_paths(rr, dms, S, ctrl, lin_s, con, sol, dx0):
    """Step-by-step iteration, then the one-call wire and resident paths with both wire cost structures."""
    from iteration_check import run_device_iteration
    rr.setTimeDiscretization(ctrl)
    out = run_device_iteration(rr, dms, lin_s, con, sol, dx0)
    res = np.ascontiguousarray(con[:, :, S.c_res:S.c_res + S.ncp])
    for robotoc_costs in (False, True):
        lin = robotoc_cost_structure(S, lin_s) if robotoc_costs else lin_s
        dms.setWireCostStructure(robotoc_costs)
        w = dms.pack_wire(lin)
        out[f"wire{int(robotoc_costs)}"] = dms.iteration_host_wire(w, lin, con, sol, dx0)
        dms.setSolution(sol)
        dms.setConstraintData(con)
        out[f"resident{int(robotoc_costs)}"] = dms.iteration_host_resident(w, lin, res, dx0)
    dms.setWireCostStructure(False)
    return out


def test_reused_handle_matches_fresh_handles_on_the_edge_set():
    """Nothing a previous schedule leaves on a handle (RIC / DIR records, KKT, expansion and constraint records, wire segment
    tables, STO sections) leaks into the next one: the reused handle gives a fresh handle's bits on every edge schedule, with
    STO and non-STO schedules alternating and n_grid changing at every step."""
    table, sd, S, K = _problem()
    batch = 2
    seq = _edge_schedules(order_for_reuse=True)
    used = S.s_xi + S.nsm
    rr, dms = _handle(max(x[2][1].N for x in seq), batch, sd, table)
    for k, (gait, sto, (t0, td, ev, ctrl)) in enumerate(seq):
        lin, con, sol, dx0 = make_stage_inputs(sd, S, ctrl, batch, 7000 + k)
        lin = symmetrize_lin(S, lin)
        rf, df = _handle(td.N, batch, sd, table)
        want = _all_paths(rf, df, S, ctrl, lin, con, sol, dx0)
        rf.close()
        got = _all_paths(rr, dms, S, ctrl, lin, con, sol, dx0)
        msg = f"{gait} sto={sto} t0={t0!r} (n_grid {len(ctrl)})"
        assert int(want["info"].max()) == 0, msg
        for key in ("ric", "d", "steps", "sol", "info"):
            np.testing.assert_array_equal(got[key], want[key], err_msg=f"{msg}: {key}")
        for f in ("c_slack", "c_dual"):
            o = getattr(S, f)
            np.testing.assert_array_equal(got["cc"][:, :, o:o + S.nc], want["cc"][:, :, o:o + S.nc], err_msg=f"{msg}: {f}")
        for c in (0, 1):
            for a, b in zip(got[f"wire{c}"], want[f"wire{c}"]):
                np.testing.assert_array_equal(a, b, err_msg=f"{msg}: iteration_host_wire, cost structure {c}")
            for a, b in zip(got[f"resident{c}"], want[f"resident{c}"]):
                np.testing.assert_array_equal(a, b, err_msg=f"{msg}: iteration_host_resident, cost structure {c}")
            # the one-call paths give the step-by-step bits
            sol_w, con_w, steps_w = got[f"wire{c}"]
            if c == 0:
                np.testing.assert_array_equal(sol_w[:, :, :used], got["sol"][:, :, :used], err_msg=msg)
                np.testing.assert_array_equal(steps_w, got["steps"], err_msg=msg)
            sol_r, sd_r, steps_r = got[f"resident{c}"]
            np.testing.assert_array_equal(sol_r[:, :, :used], sol_w[:, :, :used], err_msg=f"{msg}: resident vs wire")
            np.testing.assert_array_equal(steps_r, steps_w, err_msg=f"{msg}: resident vs wire")
    rr.close()


@pytest.mark.parametrize("impact_cones", [False, True])
def test_edge_set_iteration_against_oracle(impact_cones):
    """Every edge schedule through the iteration, with and without ImpactFrictionCone rows on the impact stages."""
    table, sd, S, K = _problem(impact_cones)
    worst = {}
    seq = _edge_schedules(order_for_reuse=True)
    rr, dms = _handle(max(x[2][1].N for x in seq), 3, sd, table)
    for k, (gait, sto, (t0, td, ev, ctrl)) in enumerate(seq):
        lin, con, sol, dx0 = make_stage_inputs(sd, S, ctrl, 3, 8000 + k, impact_cones=impact_cones)
        try:
            _check_iteration(rr, dms, sd, S, K, table, td, ctrl, lin, con, sol, dx0, worst, reused=k > 0)
        except AssertionError as e:
            raise AssertionError(f"{gait} sto={sto} t0={t0!r} (n_grid {len(ctrl)}): {e}") from None
    rr.close()
    _report(f"edge set, impact cones {impact_cones}", worst)


@pytest.mark.parametrize("batch", [1, 3])
def test_time_parallel_sweeps_on_the_edge_set(batch):
    """Segmented Riccati sweeps (no STO) at MPC batch sizes: the segment bounds move with n_grid and the events sit at the
    ends of the horizon.  RIC, FACT and DIR against the oracle at S = 2, 3, 7 and n_grid - 1."""
    L = Layout(ANYMAL)
    seq = [x for x in _edge_schedules() if not x[1]]
    rr = RiccatiRecursion(ANYMAL, max(len(x[2][3]) for x in seq), batch)
    worst = 0.0
    for k, (gait, sto, (t0, td, ev, ctrl)) in enumerate(seq):
        kkt, dx0 = make_kkt(ANYMAL, L, ctrl, batch=batch, seed=6000 + k)
        kk, ric_o, d_o, info = oracle_lib.riccati_batch(ANYMAL, L, ctrl, kkt, dx0)
        assert info == 0
        rr.setTimeDiscretization(ctrl)
        for segs in (2, 3, 7, len(ctrl) - 1):
            rr.setTimeSegments(segs)
            rr.backwardRiccatiRecursion(kkt, write_fact=True)
            rr.forwardRiccatiRecursion(dx0)
            assert int(rr.info().max()) == 0
            try:
                worst = max(worst, compare_riccati(ANYMAL, L, ctrl, rr.getRiccatiFactorization(), ric_o, rr.getDirection(), d_o,
                                            rr.getFactorizedKKT(), kk))
            except AssertionError as e:
                raise AssertionError(f"{gait} t0={t0!r} (n_grid {len(ctrl)}) S={segs}: {e}") from None
    rr.close()
    print(f"time-parallel sweeps, batch {batch}: worst rel err vs oracle {worst:.2e}")


def test_cuda_reproduces_the_reference_on_horizon_edges():
    """The iteration against the reference's own code (golden_ref_horizon.npz, made by make_golden_ref_live.py) on the edge
    schedules of a lift and an impact of every gait set, impact friction cones on every other one; fresh handle, batch 1."""
    GH = load(mgl.HORIZON_PATH)
    for case in mgl.horizon_cases():
        table, sd, S, K, ctrl, lin, con, sol, dx0, icone = mgl.horizon_case(case)
        rr, dms = _handle(len(ctrl) - 1, 1, sd, table)
        rr.setTimeDiscretization(ctrl)
        got = cuda_iteration_records(rr, dms, S, lin, con, sol, dx0)
        rr.close()
        want = {k: restore(GH, f"h_{case[0]}_{k}", got[k]) for k in mgl.STAGE_KEYS if k in got}
        try:
            compare_reference_records(S, K, ctrl, got, want, TOL, impact_cones=icone)
        except AssertionError as e:
            raise AssertionError(f"{case[0]} t0={case[3]!r} (n_grid {len(ctrl)}): {e}") from None


def test_eval_kkt_and_line_search_on_the_edge_set():
    """rbt_eval_kkt (PerformanceIndex, KKT error) and the line-search trials on every edge schedule, on one reused handle,
    against the oracle as test_eval_rows / test_line_search check them (impact cones on, switching residuals nonzero)."""
    from robotoc_b200 import LineSearch
    lib = oracle_lib.load()
    table, sd, S, K = _problem(impact_cones=True)
    batch, n_trials = 2, 4
    seq = _edge_schedules(order_for_reuse=True)
    rr, dms = _handle(max(x[2][1].N for x in seq), batch, sd, table)
    ls = LineSearch(dms)
    rng = np.random.default_rng(11)
    for k, (gait, sto, (t0, td, ev, ctrl)) in enumerate(seq):
        msg = f"{gait} sto={sto} t0={t0!r} (n_grid {len(ctrl)})"
        lin, con, sol, dx0 = make_stage_inputs(sd, S, ctrl, batch, 5000 + k, impact_cones=True)
        for i, c in enumerate(ctrl):
            if c.type not in (IMPACT, TERMINAL):
                lin[:, i, S.l_p:S.l_p + c.ns] = rng.uniform(-1, 1, size=(batch, c.ns))
        rr.setTimeDiscretization(ctrl)
        perf = dms.evalKKT(lin, con)
        want = oracle_perf_index(lib, sd, table, ctrl, lin, con)
        np.testing.assert_allclose(perf, want, rtol=1e-12, atol=0, err_msg=msg)
        np.testing.assert_allclose(dms.KKTError(), want[:, 5], rtol=1e-12, err_msg=msg)
        ref = oracle_iteration(sd, S, K, table, ctrl, lin, con, sol, dx0)
        dms.condense(lin, con)
        rr.backwardRiccatiRecursion()
        rr.forwardRiccatiRecursion(dx0)
        dms.computeStepSizes()
        steps = np.stack([dms.maxPrimalStepSize(), dms.maxDualStepSize()], axis=1)
        np.testing.assert_allclose(steps, ref["steps"], rtol=1e-10, err_msg=msg)  # compare_final's bound on the step sizes
        dms.setSolution(sol)  # the current iterate: trials are generated before integrateSolution
        alphas, barrier, trial = ls.trialSolutions(n_trials)
        # the trials start from the device's own maximum step size: on the tiny-step schedules it differs from the oracle's
        # in the 13th digit (the direction's conditioning), which is not what this compares
        a_o, b_o, t_o = oracle_trials(lib, sd, table, ctrl, sol, dict(ref, steps=steps), n_trials)
        np.testing.assert_allclose(alphas, a_o, rtol=1e-14, err_msg=msg)
        np.testing.assert_allclose(barrier, b_o, rtol=1e-11, err_msg=msg)
        np.testing.assert_allclose(trial, t_o, rtol=0, atol=1e-11 * max(1.0, np.abs(t_o).max()), err_msg=msg)
    rr.close()

