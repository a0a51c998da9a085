"""The CUDA stage layer of the unconstrained (fixed-base, iiwa14) path against the oracle and the reference's own iteration, block
by block on every grid point (iteration_check.compare_unconstr_records): horizon lengths that end inside the grid points where
joint limits are partly off, batch sizes that leave partial 4-warp CTAs, constraint tables the C ABI accepts beyond what the
reference can express, step sizes bound on chosen rows, a reused handle, and an OCP whose Riccati factorization fails in the
middle of a batch."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_ref_ustage as mu  # noqa: E402
from golden_sample import load, restore  # noqa: E402

import oracle_lib  # noqa: E402
from helpers import unconstr_step_coverage  # noqa: E402
from iteration_check import compare_unconstr_records  # noqa: E402
from robotoc_b200.layout import ULayout  # noqa: E402
from robotoc_b200.stage import RBT_MAX_BOX_ROWS, VAR_A, VAR_Q, VAR_U, VAR_V  # noqa: E402
from synth import iiwa14_rows, make_unconstr_stage_inputs, table_rows, unconstr_table  # noqa: E402

NV = 7
TOL = 1e-9
SHAPES = [(N, batch) for N in (1, 2, 3, 20, 50) for batch in (1, 3, 5, 256)]


def _oracle(tab, S, N, dt, lin, con, sol, dx0):
    out = oracle_lib.unconstr_iteration(NV, ULayout(NV, getter=oracle_lib.load().orc_ulayout_get), S, tab, N, dt, lin, con, sol, dx0)
    assert out["info"] == 0
    return out


def _device(rr, dms, lin, con, sol, dx0):
    """One iteration step by step through the C ABI, with every record read back after the call that writes it."""
    dms.condense(lin, con)
    dms.setSolution(sol)
    got = dict(kkt=dms.getKKT(), ex=dms.getExpansionData(), con_condensed=dms.getConstraintsData())
    rr.backwardRiccatiRecursion()
    rr.forwardRiccatiRecursion(dx0)
    got["dir"] = rr.getDirection()
    dms.computeStepSizes()
    got.update(xd=dms.getExpandedDirection(), con_expanded=dms.getConstraintsData(),
               steps=np.stack([dms.maxPrimalStepSize(), dms.maxDualStepSize()], axis=1))
    dms.integrateSolution()
    got.update(sol=dms.getSolution(), con=dms.getConstraintsData(), info=rr.info())
    return got


def _run(tab, N, batch, dt, seed, lin=None, con=None, sol=None, dx0=None, ref=None):
    """Device iteration vs the oracle (and `ref`, a reference iteration, if given); the one-call host path must give the
    step-by-step bits.  Returns the worst error per block family."""
    from robotoc_b200 import UnconstrDirectMultipleShooting, UnconstrRiccatiRecursion
    rr = UnconstrRiccatiRecursion(NV, N, dt, batch)
    dms = UnconstrDirectMultipleShooting(rr, tab)
    S = dms.layout
    if lin is None:
        lin, con, sol, dx0 = make_unconstr_stage_inputs(S, N, batch, seed)
    got = _device(rr, dms, lin, con, sol, dx0)
    assert int(got["info"].max()) == 0
    worst = compare_unconstr_records(S, rr.layout, got, _oracle(tab, S, N, dt, lin, con, sol, dx0), TOL)
    if ref is not None:
        compare_unconstr_records(S, rr.layout, got, ref, TOL)
    sol2, con2, steps2 = dms.iteration_host(lin, con, sol, dx0)
    np.testing.assert_array_equal(sol2, got["sol"])
    np.testing.assert_array_equal(con2, got["con"])
    np.testing.assert_array_equal(steps2, got["steps"])
    rr.close()
    return worst


def test_shapes_reach_the_cta_tails():
    """batch (N + 1) (ucondense, uupdate) and batch N (uexpand) both leave a partial 4-warp CTA on some shapes."""
    assert any(b * (N + 1) % 4 and b * N % 4 for N, b in SHAPES)
    assert {N for N, _ in SHAPES} >= {1, 2, 3} and max(b for _, b in SHAPES) >= 256


@pytest.mark.gpu
@pytest.mark.parametrize("N,batch", SHAPES)
def test_iiwa14_table_every_shape(N, batch):
    _run(unconstr_table(iiwa14_rows()), N, batch, 0.05 if N < 50 else 0.02, seed=1000 + 7 * N + batch)


def _tables():
    rng = np.random.default_rng(5)
    iiwa = iiwa14_rows()
    every = [(var, j, sign) for var in (VAR_Q, VAR_V, VAR_A, VAR_U) for sign in (-1, 1) for j in range(NV)]
    return {
        "acceleration_limits": iiwa14_rows(acceleration_limits=True),
        "permuted": [iiwa[k] for k in rng.permutation(len(iiwa))],
        "same_row_twice": iiwa + [(VAR_U, 3, 1), (VAR_Q, 0, -1), (VAR_V, 6, 1), (VAR_A, 2, -1), (VAR_A, 2, -1)],
        "joint_subset": [(var, j, sign) for var in (VAR_Q, VAR_V, VAR_U) for sign in (-1, 1) for j in (0, 2, 5)],
        "no_rows": [],
        "max_rows": [every[k] for k in rng.permutation(np.arange(RBT_MAX_BOX_ROWS) % len(every))],
    }


def test_tables_reach_their_edges():
    t = _tables()
    assert len(t["max_rows"]) == RBT_MAX_BOX_ROWS and len(t["acceleration_limits"]) > 32 and not t["no_rows"]
    assert len(set(t["same_row_twice"])) < len(t["same_row_twice"]) and t["permuted"] != iiwa14_rows()
    assert sorted(t["permuted"]) == sorted(iiwa14_rows())


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(_tables()))
@pytest.mark.parametrize("N,batch", [(20, 3), (2, 5)])
def test_tables_the_reference_cannot_express(name, N, batch):
    tab = unconstr_table(_tables()[name])
    assert table_rows(tab) == _tables()[name]
    _run(tab, N, batch, 0.05, seed=2000 + N + len(_tables()[name]))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(mu.CASES))
def test_reference_iteration(name):
    """The reference's own iteration (golden_ref_ustage.npz, whose oracle-vs-reference pin is test_golden_ref_ustage.py),
    including the step-size case: primal and dual steps bound on a torque row of grid 0, a velocity row of grid 1 and a row
    of grid N - 1, and a position row on grid 0 that would bind if it were counted."""
    tab, S, N, dt, lin, con, sol, dx0 = mu.problem(name)
    G = load(mu.PATH)
    ref_full = _oracle(tab, S, N, dt, lin, con, sol, dx0)
    ref = {k: restore(G, f"{name}_{k}", ref_full[k]) for k in mu.KEYS}
    if name == "bind":
        unconstr_step_coverage(S, tab, N, con, ref_full, dx0, mu.BINDS, mu.GATED)
    _run(tab, N, lin.shape[0], dt, None, lin, con, sol, dx0, ref=ref)


@pytest.mark.gpu
def test_reused_handle_resets_the_step_sizes():
    """Two consecutive iterations on one handle, each against the oracle: the first binds its steps near 1e-6, the second
    has steps four orders of magnitude larger, which a step-size buffer left over from the first call would cap."""
    from robotoc_b200 import UnconstrDirectMultipleShooting, UnconstrRiccatiRecursion
    tab, S, N, dt, lin1, con1, sol1, dx01 = mu.problem("bind")
    batch = lin1.shape[0]
    rr = UnconstrRiccatiRecursion(NV, N, dt, batch)
    dms = UnconstrDirectMultipleShooting(rr, tab)
    lin2, con2, sol2, dx02 = make_unconstr_stage_inputs(S, N, batch, seed=3001)
    steps = []
    for lin, con, sol, dx0 in ((lin1, con1, sol1, dx01), (lin2, con2, sol2, dx02)):
        got = _device(rr, dms, lin, con, sol, dx0)
        compare_unconstr_records(S, rr.layout, got, _oracle(tab, S, N, dt, lin, con, sol, dx0), TOL)
        steps.append(got["steps"])
    assert (steps[1] > 1e3 * steps[0]).all()
    rr.close()


@pytest.mark.gpu
def test_indefinite_G_flags_only_that_ocp():
    """Qaa <- -1e6 I on one grid point of the middle OCP: G = Qaa + B^T P B is negative definite whatever P is.  The flag comes
    back from rbt_unconstr_download_info, and the other OCPs still match the oracle."""
    from robotoc_b200 import UnconstrDirectMultipleShooting, UnconstrRiccatiRecursion
    tab = unconstr_table(iiwa14_rows())
    N, batch, dt, sick = 20, 5, 0.05, 2
    rr = UnconstrRiccatiRecursion(NV, N, dt, batch)
    dms = UnconstrDirectMultipleShooting(rr, tab)
    S = dms.layout
    lin, con, sol, dx0 = make_unconstr_stage_inputs(S, N, batch, seed=4001)
    lin[sick, 7, S.l_Qaa:S.l_Qaa + NV * NV] = (-1.0e6 * np.eye(NV)).reshape(-1)
    got = _device(rr, dms, lin, con, sol, dx0)
    assert got["info"][sick] != 0
    assert (np.delete(got["info"], sick) == 0).all()
    ok = [b for b in range(batch) if b != sick]
    ref = _oracle(tab, S, N, dt, *(np.ascontiguousarray(a[ok]) for a in (lin, con, sol, dx0)))
    compare_unconstr_records(S, rr.layout, {k: v[ok] for k, v in got.items() if k != "info"}, ref, TOL)
    rr.close()
