"""The discretization restatement (schedule_fixture.TimeDiscretization) == the reference's own TimeDiscretization
(src/ocp/time_discretization.cpp, with ContactSequence from src/planner/, compiled unmodified into
oracle/_ref/libref_discretize.so by oracle/Makefile.ref), on every receding-horizon schedule the tests build: t0 swept over
a gait cycle and t0 placed at the event edges (tiny first steps, events on and beside grid boundaries, at the horizon's
last-interval margin and at t0 itself).  Every device test takes its control table from the restatement."""
import os

import pytest

import ref_lib
from helpers import RH_GAITS, RH_SETS, receding_horizon_coverage, receding_horizon_schedules, small_event_schedule
from schedule_fixture import TimeDiscretization

FLOATS = ("t0", "t", "dt", "dt_next")
INTS = ("type", "phase", "stage", "impact_index", "lift_index", "stage_in_phase", "num_grids_in_phase", "sto", "sto_next",
        "switching_constraint")

needs_ref = pytest.mark.skipif(not (os.path.exists(ref_lib.LIB_DISCRETIZE)
                                    or (ref_lib.REFERENCE and os.path.isdir(os.path.join(ref_lib.REFERENCE, "src", "ocp")))),
                               reason="oracle/_ref/libref_discretize.so is not built (set ROBOTOC_REFERENCE)")


def _compare(td, ref, what):
    assert len(ref) == td.size(), f"{what}: n_grid {td.size()} != reference {len(ref)}"
    for i, (g, r) in enumerate(zip(td.grid, ref)):
        for f in INTS:
            assert int(getattr(g, f)) == r[f], f"{what}: grid {i}: {f} = {int(getattr(g, f))}, reference {r[f]}"
        for f in FLOATS:
            assert abs(getattr(g, f) - r[f]) <= 1e-15, f"{what}: grid {i}: {f} = {getattr(g, f)!r}, reference {r[f]!r}"


def test_receding_horizon_schedules_cover_the_edges():
    """The sweep and the edge set together (and the edge set alone) reach every grid position the kernels branch on."""
    sets = {w: [s for g, sto in RH_SETS for s in receding_horizon_schedules(g, sto, w)] for w in ("sweep", "edge")}
    receding_horizon_coverage(sets["sweep"] + sets["edge"])
    receding_horizon_coverage(sets["edge"])


@needs_ref
@pytest.mark.parametrize("which", ["sweep", "edge"])
@pytest.mark.parametrize("gait,sto", RH_SETS)
def test_discretization_matches_reference(gait, sto, which):
    T, N = RH_GAITS[gait][2:]
    for t0, td, ev, ctrl in receding_horizon_schedules(gait, sto, which):
        _compare(td, ref_lib.discretize(T, N, ev, t0), f"{gait} sto={sto} t0={t0!r}")


@needs_ref
def test_discretization_without_step_correction_matches_reference():
    """discretize alone (DiscretizationMethod::GridBased): the raw grid, unequal steps around the events, no STO flags."""
    for gait, sto in RH_SETS:
        T, N = RH_GAITS[gait][2:]
        for t0, _, ev, _ in receding_horizon_schedules(gait, sto, "edge"):
            td = TimeDiscretization(T, N).discretize(ev, t0, sto=False)
            _compare(td, ref_lib.discretize(T, N, ev, t0, phase_based=False), f"{gait} sto={sto} t0={t0!r} grid-based")
    td, ev, _ = small_event_schedule(sto=True)
    _compare(td, ref_lib.discretize(td.T, td.N, ev, 0.0), "small event schedule")
