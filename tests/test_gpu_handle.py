"""Handle plumbing of the C ABI: caller-bound device buffers (the path bench.py runs on) and a stage setup that follows a
rejected one."""
import ctypes

import numpy as np
import pytest

from helpers import trot_schedule
from iteration_check import run_device_iteration
from robotoc_b200 import ANYMAL, DirectMultipleShooting, Layout, RiccatiRecursion, StageDims, StageLayout, anymal_constraint_table
from synth import make_stage_inputs, symmetrize_lin

pytestmark = pytest.mark.gpu
DIR, CON, SOL = 3, 7, 9  # RBT_BUF_*
BATCH = 8


def _problem():
    _, _, ctrl = trot_schedule(40)
    table = anymal_constraint_table()
    sd = StageDims(ANYMAL, nf_max=12, n_contacts=table.n_contacts, n_box=table.n_box)
    S = StageLayout(sd)
    lin, con, sol, dx0 = make_stage_inputs(sd, S, ctrl, BATCH, 7)
    return ctrl, table, sd, S, (symmetrize_lin(S, lin), con, sol, dx0)


def _handle(ctrl, sd, table):
    rr = RiccatiRecursion(ANYMAL, len(ctrl), BATCH)
    rr.setTimeDiscretization(ctrl)
    return rr, DirectMultipleShooting(rr, sd, table)


def _assert_same(got, ref):
    for k in ref:
        assert np.array_equal(got[k], ref[k]), k


def test_bound_buffers_give_the_bits_of_the_handles_own():
    torch = pytest.importorskip("torch")
    ctrl, table, sd, S, inputs = _problem()
    K, n_grid = Layout(ANYMAL), len(ctrl)
    ref = run_device_iteration(*_handle(ctrl, sd, table), *inputs)

    rr, dms = _handle(ctrl, sd, table)
    own = {w: rr.dev_ptr(w) for w in (DIR, CON, SOL)}
    bound = {w: torch.zeros((BATCH, n_grid, stride), dtype=torch.float64, device="cuda")
             for w, stride in ((DIR, K.d_stride), (CON, S.c_stride), (SOL, S.s_stride))}
    for w, t in bound.items():
        rr.bind_buffer(w, ctypes.c_void_p(t.data_ptr()))
        assert rr.dev_ptr(w) == t.data_ptr()
    got = run_device_iteration(rr, dms, *inputs)
    _assert_same(got, ref)
    torch.cuda.synchronize()
    # the outputs are in the caller's tensors
    assert np.array_equal(bound[DIR].cpu().numpy(), ref["d"])
    assert np.array_equal(bound[CON].cpu().numpy(), ref["cc"])
    assert np.array_equal(bound[SOL].cpu().numpy(), ref["sol"])

    for w in bound:
        rr.bind_buffer(w, None)
        assert rr.dev_ptr(w) == own[w]
    _assert_same(run_device_iteration(rr, dms, *inputs), ref)


def test_stage_setup_after_a_rejected_one():
    ctrl, table, sd, S, inputs = _problem()
    ref = run_device_iteration(*_handle(ctrl, sd, table), *inputs)

    rr = RiccatiRecursion(ANYMAL, len(ctrl), BATCH)
    rr.setTimeDiscretization(ctrl)
    few = anymal_constraint_table()
    few.n_contacts = 2  # the trot schedule has grid points with four contacts
    with pytest.raises(ValueError, match="more contacts than the stage layer"):
        DirectMultipleShooting(rr, StageDims(ANYMAL, nf_max=12, n_contacts=2, n_box=few.n_box), few)
    assert rr._lib.rbt_buf_doubles(rr._h, SOL) == -1
    dms = DirectMultipleShooting(rr, sd, table)
    _assert_same(run_device_iteration(rr, dms, *inputs), ref)
