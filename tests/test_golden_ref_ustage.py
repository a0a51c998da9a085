"""The stage layer of the unconstrained (fixed-base, iiwa14) path pinned against the reference's own code.
tests/golden/golden_ref_ustage.npz holds (a seeded sample of) full iterations computed by robotoc's UnconstrDynamics, joint-limit
components, SplitSolution and UnconstrRiccatiRecursion (make_golden_ref_ustage.py): N = 1, 2, 3, 20, 50, the iiwa14 table with
and without joint acceleration limits, and inputs whose step sizes bind on chosen rows.  The oracle reproduces it block by block
on every grid point; where oracle/_ref/libref_riccati.so is built, also live."""
import ctypes
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_ref_ustage as mu  # noqa: E402
from golden_sample import load, restore  # noqa: E402

import oracle_lib  # noqa: E402
import ref_lib  # noqa: E402
from iteration_check import compare_unconstr_records  # noqa: E402
from robotoc_b200.layout import ULayout  # noqa: E402

G = load(mu.PATH)
TOL = 1e-12
NV = mu.NV


def _oracle(name):
    lib = oracle_lib.load()
    tab, S, N, dt, lin, con, sol, dx0 = mu.problem(name, lib.orc_ustage_layout_get)
    UL = ULayout(NV, getter=lib.orc_ulayout_get)
    out = oracle_lib.unconstr_iteration(NV, UL, S, tab, N, dt, lin, con, sol, dx0)
    assert out["info"] == 0
    return tab, S, UL, N, dt, lin, con, sol, dx0, out


def golden(name, got):
    """The stored reference iteration of case `name`, put into copies of the records under test."""
    return {k: restore(G, f"{name}_{k}", got[k]) for k in mu.KEYS}


@pytest.mark.parametrize("name", list(mu.CASES))
def test_oracle_reproduces_the_reference_unconstrained_iteration(name):
    tab, S, UL, N, dt, lin, con, sol, dx0, out = _oracle(name)
    compare_unconstr_records(S, UL, out, golden(name, out), TOL)


@pytest.mark.skipif(not ref_lib.available(), reason="the reference's stage layer is not built (set ROBOTOC_REFERENCE)")
@pytest.mark.parametrize("name", list(mu.CASES))
def test_oracle_equals_live_reference_unconstrained_iteration(name):
    tab, S, UL, N, dt, lin, con, sol, dx0, out = _oracle(name)
    ref = ref_lib.unconstr_iteration(NV, UL, S, tab, N, dt, lin, con, sol, dx0)
    compare_unconstr_records(S, UL, out, ref, TOL)


def test_the_fixture_pins_the_grid_gating():
    """On grid points 0 and 1 the reference's KKT blocks differ from a condensing that applies every row: the fixture would
    catch joint limits applied where ConstraintsData::setTimeStage turns them off."""
    lib = oracle_lib.load()
    for name in ("n20", "n1", "acc"):
        tab, S, UL, N, dt, lin, con, sol, dx0, out = _oracle(name)
        b_s, i_s, e_s = np.unravel_index(G[f"{name}_kkt#i"], tuple(G[f"{name}_kkt#shape"]))
        v_s = G[f"{name}_kkt#v"]
        for i in [i for i in (0, 1) if i < N]:  # grid point N is the terminal, which has no constraints
            diff, scale = 0.0, 0.0
            for b in range(lin.shape[0]):
                kkt, ex, c = np.zeros(UL.k_stride), np.zeros(S.e_stride), con[b, i].copy()
                lib.orc_ustage_condense(NV, ctypes.byref(tab), 0, oracle_lib.ptr(np.ascontiguousarray(lin[b, i])),
                                        oracle_lib.ptr(c), oracle_lib.ptr(kkt), oracle_lib.ptr(ex))  # every row acts
                for off, n in ((UL.k_Qxx, 4 * NV * NV), (UL.k_lx, 2 * NV)):
                    sel = (b_s == b) & (i_s == i) & (e_s >= off) & (e_s < off + n)
                    assert sel.any()
                    diff = max(diff, np.abs(kkt[e_s[sel]] - v_s[sel]).max())
                    scale = max(scale, np.abs(v_s[sel]).max())
            assert diff > 1e-3 * scale, (name, i)


def test_bind_case_covers_the_step_size_edges():
    """The "bind" case reaches what the step-size code branches on: primal and dual steps below 1 and different; primal steps
    bound by a torque row on grid 0, a velocity row on grid 1 and a row on grid N - 1; a position row on grid 0 that would bind
    far below the step if it were counted."""
    from helpers import unconstr_step_coverage
    tab, S, UL, N, dt, lin, con, sol, dx0, out = _oracle("bind")
    unconstr_step_coverage(S, tab, N, con, out, dx0, mu.BINDS, mu.GATED)
