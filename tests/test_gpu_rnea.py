"""rbt_linearize_inverse_dynamics on the device: the kernel against the numpy restatement tests/rbd_ref.py (itself pinned by
tests/test_rnea.py), a full iteration with the ID sections filled on the host against one where the device fills them, and the
resident wire path with RBT_WIRE_DEVICE_ID against the step-by-step calls."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_model_fixture  # noqa: E402
import rbd_ref as R  # noqa: E402
from helpers import contact_mask_walk_schedule, crawl_schedule, jump_sto_schedule, rel_err, trot_schedule  # noqa: E402
from synth import make_stage_inputs, symmetrize_lin  # noqa: E402

SCHEDULES = {"trot": lambda: trot_schedule()[2], "crawl": lambda: crawl_schedule()[2],
             "mask_walk": lambda: contact_mask_walk_schedule()[2], "jump": lambda: jump_sto_schedule()[2]}
LIN = 6


def _setup(ctrl, batch, seed):
    from robotoc_b200 import ANYMAL, DirectMultipleShooting, RiccatiRecursion, StageDims, StageLayout, anymal_constraint_table
    table = anymal_constraint_table()
    sd = StageDims(ANYMAL, nf_max=12, n_contacts=4, n_box=table.n_box)
    S = StageLayout(sd)
    lin, con, sol, dx0 = make_stage_inputs(sd, S, ctrl, batch, seed)
    rr = RiccatiRecursion(ANYMAL, len(ctrl), batch)
    rr.setTimeDiscretization(ctrl)
    dms = DirectMultipleShooting(rr, sd, table)
    return rr, dms, S, symmetrize_lin(S, lin), con, sol, dx0


def _model(name):
    return make_model_fixture.load() if name == "anymal" else R.random_model(int(name[-1]))


def _sections(S, nv=18):
    """(offset, length) of every part of the linearization record the kernel writes."""
    return {"IDC": (S.l_IDC, nv), "D": (S.l_D, S.nvf * 2 * nv), "M": (S.l_M, nv * nv), "lx": (S.l_lx, 2 * nv), "la": (S.l_la, nv)}


CASES = [(s, b, "anymal") for s in SCHEDULES for b in (1, 3)] + [("trot", 1024, "anymal")] + \
        [(s, 3, "random1") for s in ("trot", "mask_walk")] + [("jump", 3, "random2")]


@pytest.mark.gpu
@pytest.mark.parametrize("which,batch,model", CASES)
def test_kernel_matches_the_restatement(which, batch, model):
    ctrl = SCHEDULES[which]()
    rr, dms, S, lin, con, sol, dx0 = _setup(ctrl, batch, 71)
    m = _model(model)
    with pytest.raises(RuntimeError):
        dms.linearizeInverseDynamics()  # no robot model yet: RBT_ERR_STATE
    dms.setRobotModel(R.to_c(m))
    dms._up(LIN, lin, S.l_stride, None)
    dms.setSolution(sol)
    dms.linearizeInverseDynamics()
    got = dms._down(LIN, lin.shape)
    ref = R.linearize(m, S, ctrl, sol, lin)
    for name, (o, n) in _sections(S).items():
        assert rel_err(got[:, :, o:o + n], ref[:, :, o:o + n]) < 1e-12, name
    mask = np.ones(S.l_stride, bool)
    for o, n in _sections(S).values():
        mask[o:o + n] = False
    np.testing.assert_array_equal(got[:, :, mask], lin[:, :, mask])  # nothing else is touched
    term = [i for i, c in enumerate(ctrl) if c.type == 3]
    np.testing.assert_array_equal(got[:, term], lin[:, term])
    rr.close()


def _steps_of(rr, dms, dx0):
    rr.backwardRiccatiRecursion()
    rr.forwardRiccatiRecursion(dx0)
    dms.computeStepSizes()
    dms.integrateSolution()
    steps = np.stack([dms.maxPrimalStepSize(), dms.maxDualStepSize()], axis=1)
    return dict(kkt=dms.getKKT(), d=rr.getDirection(), steps=steps, sol=dms.getSolution(), con=dms.getConstraintData())


@pytest.mark.gpu
@pytest.mark.parametrize("which,batch", [("trot", 3), ("crawl", 3), ("mask_walk", 1), ("jump", 3), ("trot", 1024)])
def test_iteration_with_device_inverse_dynamics_matches_host_filled_records(which, batch):
    ctrl = SCHEDULES[which]()
    rr, dms, S, lin, con, sol, dx0 = _setup(ctrl, batch, 72)
    m = make_model_fixture.load()
    dms.setRobotModel(R.to_c(m))
    # host-filled ID sections
    dms.setSolution(sol)
    dms.condense(R.linearize(m, S, ctrl, sol, lin), con)
    a = _steps_of(rr, dms, dx0)
    # device-filled: the uploaded ID sections are ignored, the gradients lack the beta terms
    lin_raw = lin.copy()
    lin_raw[:, :, S.l_IDC:S.l_IDC + 18] = np.nan
    lin_raw[:, :, S.l_M:S.l_M + 18 * 18] = np.nan
    D = lin_raw[:, :, S.l_D:S.l_D + S.nvf * 36].reshape(batch, len(ctrl), 36, S.nvf)
    D[:, :, :, :18] = np.nan
    lin_raw[:, :, S.l_D:S.l_D + S.nvf * 36] = D.reshape(batch, len(ctrl), -1)
    term = [i for i, c in enumerate(ctrl) if c.type == 3]
    lin_raw[:, term] = lin[:, term]
    dms._up(LIN, np.ascontiguousarray(lin_raw), S.l_stride, None)
    dms.setConstraintData(con)
    dms.setSolution(sol)
    dms.linearizeInverseDynamics()
    dms.condense()
    b = _steps_of(rr, dms, dx0)
    for k in a:
        assert np.isfinite(b[k]).all(), k
        assert rel_err(b[k], a[k]) < 1e-10, k
    rr.close()


@pytest.mark.gpu
@pytest.mark.parametrize("which,batch", [("trot", 3), ("mask_walk", 3), ("crawl", 200)])
def test_resident_wire_path_with_device_inverse_dynamics(which, batch):
    ctrl = SCHEDULES[which]()
    rr, dms, S, lin, con, sol, dx0 = _setup(ctrl, batch, 73)
    m = make_model_fixture.load()
    res = np.ascontiguousarray(con[:, :, S.c_res:S.c_res + S.ncp])
    full = dms.iteration_host_bytes(resident=True)[0]
    dms.setWireCostStructure(False, device_inverse_dynamics=True)
    wire = dms.pack_wire(lin)
    with pytest.raises(RuntimeError):  # the device cannot fill the ID rows without a model
        dms.iteration_host_resident(wire, lin, res, dx0)
    dms.setRobotModel(R.to_c(m))
    assert dms.iteration_host_bytes(resident=True)[0] < 0.75 * full
    dms.setSolution(sol)
    dms.setConstraintData(con)
    sol1, sd1, steps1 = dms.iteration_host_resident(wire, lin, res, dx0)
    # step by step
    dms.setSolution(sol)
    dms.setConstraintData(con)
    dms._up(LIN, lin, S.l_stride, None)
    dms.linearizeInverseDynamics()
    dms.condense()
    b = _steps_of(rr, dms, dx0)
    used = S.s_xi + S.nsm
    np.testing.assert_array_equal(sol1[:, :, :used], b["sol"][:, :, :used])
    np.testing.assert_array_equal(steps1, b["steps"])
    np.testing.assert_array_equal(sd1[:, :, :S.nc], b["con"][:, :, S.c_slack:S.c_slack + S.nc])
    dms.setWireCostStructure(False)
    rr.close()
