"""The stage layer (condensing, expansion, step sizes, slack / dual update: SURVEY.md 8a rows a10-a16) pinned against the
reference's own code.  tests/golden/golden_ref_stage_r2.npz holds (a seeded sample of) one full iteration computed by robotoc's sources
(make_golden_ref_stage.py);
  CPU: the oracle reproduces it; it is also compared with the reference code on the BASELINE trot schedule and further seeds
       (a fixed sample of every record: tests/golden/golden_ref_live.npz, make_golden_ref_live.py);
  GPU: the CUDA path reproduces it through the C ABI."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_ref_stage as mg  # noqa: E402
from golden_sample import load, restore  # noqa: E402
import make_golden_ref_live as mgl  # noqa: E402

import oracle_lib  # noqa: E402
from iteration_check import compare_reference_records as _cmp_records, cuda_iteration_records as _cuda_iteration  # noqa: E402
from iteration_check import oracle_iteration  # noqa: E402

G = load(mg.PATH)


def _golden(got, impact_cones):
    """The stored reference iteration (a seeded sample of every record section), put into copies of the records under test."""
    pre = "ic_" if impact_cones else ""
    return {k: restore(G, pre + k, got[k]) for k in mg.KEYS if k in got}
TOL = 1e-10


@pytest.mark.parametrize("impact_cones", [False, True])
def test_oracle_reproduces_the_reference_iteration_golden(impact_cones):
    lib = oracle_lib.load()
    table, sd, S, K, ctrl, lin, con, sol, dx0 = mg.problem(lib.orc_stage_layout_get, lib.orc_layout_get, impact_cones)
    got = oracle_iteration(sd, S, K, table, ctrl, lin, con, sol, dx0)
    ref = _golden(got, impact_cones)
    if impact_cones:  # the impact cones must matter: the iteration differs from the one without them
        both, a, b = np.intersect1d(G["ic_ric#i"], G["ric#i"], return_indices=True)
        assert np.max(np.abs(G["ic_ric#v"][a] - G["ric#v"][b])) > 1e-6
    _cmp_records(S, K, ctrl, got, ref, TOL, impact_cones=impact_cones)


def _oracle_perf_stage(lib, sd, S, table, ctrl, lin, con):
    """orc_stage_perf_index per grid point: {cost_barrier, primal_feasibility, dual_feasibility, kkt_error}."""
    import ctypes
    lib.orc_stage_perf_index.argtypes = [ctypes.c_void_p] * 6
    out = np.zeros((lin.shape[0], len(ctrl), 4))
    csd = sd.c()
    for b in range(lin.shape[0]):
        for i, c in enumerate(ctrl):
            st = np.zeros(4)
            lib.orc_stage_perf_index(ctypes.byref(csd), ctypes.byref(table), ctypes.byref(c), oracle_lib.ptr(np.ascontiguousarray(lin[b, i])),
                                     oracle_lib.ptr(np.ascontiguousarray(con[b, i])), oracle_lib.ptr(st))
            out[b, i] = st
    return out


@pytest.mark.parametrize("impact_cones", [False, True])
def test_oracle_performance_index_equals_the_reference_evalKKT_summary(impact_cones):
    """PerformanceIndex of every grid point (log barrier, primal / dual feasibility, squared KKT error) as the reference's own
    members compute it before condensing (OCPData / SplitKKTResidual / ConstraintsData / ContactDynamicsData ::KKTError etc.,
    intermediate_stage.cpp:124-132, impact_stage.cpp:104-113, terminal_stage.cpp:94-100) -- golden fixtures."""
    lib = oracle_lib.load()
    table, sd, S, K, ctrl, lin, con, sol, dx0 = mg.problem(lib.orc_stage_layout_get, lib.orc_layout_get, impact_cones)
    got = _oracle_perf_stage(lib, sd, S, table, ctrl, lin, con)
    ref = G["ic_perf_stage" if impact_cones else "perf_stage"]
    np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-300)
    assert (ref[:, :, 3] > 0).all() and (ref[:, :-1, 0] != 0).any()
    table, ctrl, lin, con, dx0 = mgl.perf_case(sd, S, impact_cones)
    np.testing.assert_allclose(_oracle_perf_stage(lib, sd, S, table, ctrl, lin, con), load(mgl.PATH)[f"perf_icone{int(impact_cones)}"],
                               rtol=1e-12, atol=1e-300)


@pytest.mark.parametrize("which,seed", mgl.STAGE_CASES)
def test_oracle_equals_live_reference_stage_layer(which, seed):
    lib = oracle_lib.load()
    table, sd, S, K, ctrl, lin, con, sol, dx0, icone = mgl.stage_case(which, seed, lib.orc_stage_layout_get, lib.orc_layout_get)
    got = oracle_iteration(sd, S, K, table, ctrl, lin, con, sol, dx0)
    GL = load(mgl.fixture_path(which))
    ref = {k: restore(GL, f"stage_{which}_{k}", got[k]) for k in mgl.STAGE_KEYS}
    _cmp_records(S, K, ctrl, got, ref, TOL, impact_cones=icone)


def test_oracle_equals_live_reference_on_horizon_edges():
    """The receding-horizon edge schedules (t0 != 0, events on grid 1 and beside it, at the last admissible grid points, steps
    far below T / N; with and without impact cones): the oracle == the reference's code (golden_ref_horizon.npz)."""
    lib = oracle_lib.load()
    GH = load(mgl.HORIZON_PATH)
    for case in mgl.horizon_cases():
        table, sd, S, K, ctrl, lin, con, sol, dx0, icone = mgl.horizon_case(case, lib.orc_stage_layout_get, lib.orc_layout_get)
        got = oracle_iteration(sd, S, K, table, ctrl, lin, con, sol, dx0)
        ref = {k: restore(GH, f"h_{case[0]}_{k}", got[k]) for k in mgl.STAGE_KEYS}
        try:
            _cmp_records(S, K, ctrl, got, ref, TOL, impact_cones=icone)
        except AssertionError as e:
            raise AssertionError(f"{case[0]} t0={case[3]!r} (n_grid {len(ctrl)}): {e}") from None


def test_horizon_edge_cases_cover_the_edges():
    """The edge cases stored in golden_ref_horizon.npz reach the grid positions the kernels branch on."""
    from helpers import receding_horizon_coverage
    receding_horizon_coverage([(c[3], c[4], None, c[5]) for c in mgl.horizon_cases()])


@pytest.mark.gpu
@pytest.mark.parametrize("impact_cones", [False, True])
def test_cuda_reproduces_the_reference_iteration_golden(impact_cones):
    from robotoc_b200 import ANYMAL, DirectMultipleShooting, RiccatiRecursion
    table, sd, S, K, ctrl, lin, con, sol, dx0 = mg.problem(impact_cones=impact_cones)
    rr = RiccatiRecursion(ANYMAL, len(ctrl), lin.shape[0])
    rr.setTimeDiscretization(ctrl)
    dms = DirectMultipleShooting(rr, sd, table)
    # PerformanceIndex of evalKKT: {cost (not on this path), barrier, primal / dual feasibility, KKT error, sqrt} vs the reference's sums
    perf = dms.evalKKT(lin, con)
    pref = (G["ic_perf_stage"] if impact_cones else G["perf_stage"]).sum(axis=1)
    np.testing.assert_allclose(perf[:, 1:5], pref, rtol=1e-11)
    np.testing.assert_allclose(perf[:, 5], np.sqrt(pref[:, 3]), rtol=1e-11)
    got = _cuda_iteration(rr, dms, S, lin, con, sol, dx0)
    _cmp_records(S, K, ctrl, got, _golden(got, impact_cones), 1e-8, impact_cones=impact_cones)
    rr.close()


@pytest.mark.gpu
@pytest.mark.parametrize("which,seed", [(w, s) for w, s in mgl.STAGE_CASES if w in mgl.GAIT_CASES])
def test_cuda_reproduces_the_reference_iteration_gaits(which, seed):
    """The CUDA iteration against the reference's own on the crawl (with / without switching-time optimisation and impact
    cones) and contact-mask-walk schedules (golden_ref_gaits.npz)."""
    from robotoc_b200 import ANYMAL, DirectMultipleShooting, RiccatiRecursion
    table, sd, S, K, ctrl, lin, con, sol, dx0, icone = mgl.stage_case(which, seed, None, None)
    rr = RiccatiRecursion(ANYMAL, len(ctrl), lin.shape[0])
    rr.setTimeDiscretization(ctrl)
    got = _cuda_iteration(rr, DirectMultipleShooting(rr, sd, table), S, lin, con, sol, dx0)
    GL = load(mgl.GAITS_PATH)
    _cmp_records(S, K, ctrl, got, {k: restore(GL, f"stage_{which}_{k}", got[k]) for k in mgl.STAGE_KEYS if k in got},
                 1e-8, impact_cones=icone)
    rr.close()
