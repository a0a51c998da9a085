"""rbt_linearize_contact_kinematics on the device: the kernel against the numpy restatement tests/contact_ref.py (itself pinned by
tests/test_contact_kinematics.py), the call order after the inverse-dynamics kernel, the error codes, a full iteration with the
contact rows filled on the host against one where the device fills them, and the resident wire path with
RBT_WIRE_DEVICE_CONTACT | RBT_WIRE_DEVICE_ID against the step-by-step calls."""
import ctypes
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import contact_ref as CR  # noqa: E402
import make_model_fixture  # noqa: E402
import rbd_ref as R  # noqa: E402
from helpers import contact_mask_walk_schedule, crawl_schedule, jump_sto_schedule, rel_err, trot_schedule  # noqa: E402
from synth import make_stage_inputs, symmetrize_lin  # noqa: E402

SCHEDULES = {"trot": lambda: trot_schedule()[2], "crawl": lambda: crawl_schedule()[2],
             "mask_walk": lambda: contact_mask_walk_schedule()[2], "jump": lambda: jump_sto_schedule()[2]}
LIN, CONTACT_POS = 6, 13
TERMINAL = 3


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


def _contact_inputs(ctrl, batch, seed):
    return CR.random_gains(seed, 4), CR.random_positions(seed + 1, batch, len(ctrl), 4)


def _written(S, ctrl):
    """[n_grid, l_stride] mask of what the kernel may write on each grid point: the active contact rows of J, dIDCdqv and IDC
    and the gradients lq, lv, la, lf."""
    nv, nx = S.nv, S.nx
    out = np.zeros((len(ctrl), S.l_stride), bool)
    for i, c in enumerate(ctrl):
        if c.type == TERMINAL or c.nf == 0:
            continue
        nf = c.nf
        for k in range(nv):
            out[i, S.l_J + k * S.nfm:S.l_J + k * S.nfm + nf] = True
        for k in range(nx):
            out[i, S.l_D + nv + k * S.nvf:S.l_D + nv + k * S.nvf + nf] = True
        out[i, S.l_IDC + nv:S.l_IDC + nv + nf] = True
        out[i, S.l_lx:S.l_lx + nx] = True
        out[i, S.l_la:S.l_la + nv] = True
        out[i, S.l_lf:S.l_lf + nf] = True
    return out


def _sections(S):
    nv = S.nv
    return {"J": (S.l_J, S.nfm * nv), "D": (S.l_D, S.nvf * 2 * nv), "IDC": (S.l_IDC, S.nvf), "lx": (S.l_lx, 2 * nv),
            "la": (S.l_la, nv), "lf": (S.l_lf, S.nfm)}


CASES = [(s, b, "anymal") for s in SCHEDULES for b in (1, 3)] + [("trot", 1024, "anymal")] + \
        [(s, 3, "random1") for s in ("trot", "mask_walk")] + [("jump", 3, "random2")]


@pytest.mark.gpu
@pytest.mark.parametrize("which,batch,model", CASES)
def test_kernel_matches_the_restatement(which, batch, model):
    ctrl = SCHEDULES[which]()
    rr, dms, S, lin, con, sol, dx0 = _setup(ctrl, batch, 81)
    m = _model(model)
    gains, pos = _contact_inputs(ctrl, batch, 82)
    dms.setRobotModel(R.to_c(m))
    dms.setContactGains(gains)
    dms.setContactPositions(pos)
    dms._up(LIN, lin, S.l_stride, None)
    dms.setSolution(sol)
    dms.linearizeContactKinematics()
    got = dms._down(LIN, lin.shape)
    ref = CR.linearize(m, S, ctrl, sol, lin, gains, pos)
    for name, (o, n) in _sections(S).items():
        assert rel_err(got[:, :, o:o + n], ref[:, :, o:o + n]) < 1e-12, name
    w = _written(S, ctrl)
    for i in range(len(ctrl)):  # nothing else is touched: inactive rows, terminal grid points, every other section
        np.testing.assert_array_equal(got[:, i, ~w[i]], lin[:, i, ~w[i]])
    np.testing.assert_array_equal(dms._down(CONTACT_POS, pos.shape), pos)
    rr.close()


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["trot", "jump"])
def test_inverse_dynamics_then_contact_rows_matches_the_reference_order(which):
    """linearizeContactDynamics adds the beta terms of the ID rows before the mu terms of the contact rows
    (contact_dynamics.cpp:31-51): the two kernels in that order give the restatements composed in that order."""
    ctrl = SCHEDULES[which]()
    rr, dms, S, lin, con, sol, dx0 = _setup(ctrl, 3, 83)
    m = make_model_fixture.load()
    gains, pos = _contact_inputs(ctrl, 3, 84)
    dms.setRobotModel(R.to_c(m))
    dms.setContactGains(gains)
    dms.setContactPositions(pos)
    dms._up(LIN, lin, S.l_stride, None)
    dms.setSolution(sol)
    dms.linearizeInverseDynamics()
    dms.linearizeContactKinematics()
    got = dms._down(LIN, lin.shape)
    ref = CR.linearize(m, S, ctrl, sol, R.linearize(m, S, ctrl, sol, lin), gains, pos)
    for name, (o, n) in list(_sections(S).items()) + [("M", (S.l_M, S.nv * S.nv))]:
        assert rel_err(got[:, :, o:o + n], ref[:, :, o:o + n]) < 1e-12, name
    rr.close()


@pytest.mark.gpu
def test_error_codes():
    from robotoc_b200._lib import lib
    ctrl = SCHEDULES["trot"]()
    rr, dms, S, lin, con, sol, dx0 = _setup(ctrl, 2, 85)
    gains, pos = _contact_inputs(ctrl, 2, 86)
    L = lib()
    assert L.rbt_linearize_contact_kinematics(rr._h, None) == 3           # no model, gains, positions
    assert L.rbt_download(rr._h, CONTACT_POS, pos.ctypes.data_as(ctypes.c_void_p), None) == 3  # not uploaded yet
    dms.setRobotModel(R.to_c(make_model_fixture.load()))
    assert L.rbt_linearize_contact_kinematics(rr._h, None) == 3           # no gains
    for bad in (-1.0, np.nan, np.inf):
        g = gains.copy()
        g[2, 1] = bad
        with pytest.raises(ValueError):
            dms.setContactGains(g)
    dms.setContactGains(gains)
    with pytest.raises(RuntimeError):                                      # no positions
        dms.linearizeContactKinematics()
    assert dms.iteration_host_bytes()[0] > 0
    assert L.rbt_set_wire_cost_structure(rr._h, 8) == 1                   # unknown bit
    dms.setWireCostStructure(False, device_contact_kinematics=True)       # alone: the ID rows still travel
    wire = dms.pack_wire(lin)
    res = np.ascontiguousarray(con[:, :, S.c_res:S.c_res + S.ncp])
    dms.setSolution(sol)
    dms.setConstraintData(con)
    with pytest.raises(RuntimeError):                                      # the wire path needs the positions too
        dms.iteration_host_resident(wire, lin, res, dx0)
    dms.setContactPositions(pos)
    dms.linearizeContactKinematics()
    sol1, sd1, steps1 = dms.iteration_host_resident(wire, lin, res, dx0)
    assert np.isfinite(sol1).all() and np.isfinite(steps1).all()
    dms.setWireCostStructure(False)
    rr.close()


@pytest.mark.gpu
def test_gains_before_stage_setup_are_rejected():
    from robotoc_b200 import ANYMAL, RiccatiRecursion
    from robotoc_b200._lib import lib
    rr = RiccatiRecursion(ANYMAL, 3, 1)
    g = np.ones(8)
    assert lib().rbt_set_contact_gains(rr._h, g.ctypes.data_as(ctypes.c_void_p)) == 3
    assert lib().rbt_linearize_contact_kinematics(rr._h, None) == 3
    rr.close()


def _steps_of(rr, dms, dx0):
    perf = dms.evalKKT()
    dms.condense()
    rr.backwardRiccatiRecursion()
    rr.forwardRiccatiRecursion(dx0)
    dms.computeStepSizes()
    dms.integrateSolution()
    steps = np.stack([dms.maxPrimalStepSize(), dms.maxDualStepSize()], axis=1)
    return dict(perf=perf, kkt=dms.getKKT(), d=rr.getDirection(), steps=steps, sol=dms.getSolution(),
                con=dms.getConstraintData())


def _without_device_rows(S, ctrl, lin):
    """The records a host that leaves the ID and the contact rows to the device sends: those rows NaN (never read)."""
    out = lin.copy()
    for i, c in enumerate(ctrl):
        if c.type == TERMINAL:
            continue
        r = out[:, i]
        r[:, S.l_M:S.l_M + S.nv * S.nv] = np.nan
        D = r[:, S.l_D:S.l_D + S.nvf * S.nx].reshape(-1, S.nx, S.nvf)
        D[:, :, :S.nv + c.nf] = np.nan
        r[:, S.l_D:S.l_D + S.nvf * S.nx] = D.reshape(r.shape[0], -1)
        r[:, S.l_IDC:S.l_IDC + S.nv + c.nf] = np.nan
        J = r[:, S.l_J:S.l_J + S.nfm * S.nv].reshape(-1, S.nv, S.nfm)
        J[:, :, :c.nf] = np.nan
        r[:, S.l_J:S.l_J + S.nfm * S.nv] = J.reshape(r.shape[0], -1)
        out[:, i] = r
    return np.ascontiguousarray(out)


@pytest.mark.gpu
@pytest.mark.parametrize("which,batch", [("trot", 3), ("crawl", 3), ("mask_walk", 1), ("jump", 3), ("trot", 1024)])
def test_iteration_with_device_contact_rows_matches_host_filled_records(which, batch):
    ctrl = SCHEDULES[which]()
    rr, dms, S, lin, con, sol, dx0 = _setup(ctrl, batch, 87)
    m = make_model_fixture.load()
    gains, pos = _contact_inputs(ctrl, batch, 88)
    dms.setRobotModel(R.to_c(m))
    dms.setContactGains(gains)
    dms.setContactPositions(pos)
    # host-filled ID and contact rows
    dms.setSolution(sol)
    dms._up(LIN, CR.linearize(m, S, ctrl, sol, R.linearize(m, S, ctrl, sol, lin), gains, pos), S.l_stride, None)
    dms.setConstraintData(con)
    a = _steps_of(rr, dms, dx0)
    # device-filled: the uploaded rows are ignored, the gradients lack the beta and mu terms
    dms._up(LIN, _without_device_rows(S, ctrl, lin), S.l_stride, None)
    dms.setConstraintData(con)
    dms.setSolution(sol)
    dms.linearizeInverseDynamics()
    dms.linearizeContactKinematics()
    b = _steps_of(rr, dms, dx0)
    for k in a:
        assert np.isfinite(b[k]).all(), k
        assert rel_err(b[k], a[k]) < 1e-10, k
    rr.close()


@pytest.mark.gpu
@pytest.mark.parametrize("which,batch", [("trot", 3), ("mask_walk", 3), ("crawl", 200)])
def test_resident_wire_path_with_device_contact_rows(which, batch):
    ctrl = SCHEDULES[which]()
    rr, dms, S, lin, con, sol, dx0 = _setup(ctrl, batch, 89)
    m = make_model_fixture.load()
    gains, pos = _contact_inputs(ctrl, batch, 90)
    res = np.ascontiguousarray(con[:, :, S.c_res:S.c_res + S.ncp])
    dms.setRobotModel(R.to_c(m))
    dms.setContactGains(gains)
    dms.setContactPositions(pos)
    dms.setWireCostStructure(False, device_inverse_dynamics=True)
    id_only = dms.iteration_host_bytes(resident=True)[0]
    w_id = dms.pack_wire(lin).shape[1]
    dms.setWireCostStructure(False, device_inverse_dynamics=True, device_contact_kinematics=True)
    wire = dms.pack_wire(lin)
    assert id_only - dms.iteration_host_bytes(resident=True)[0] == 8 * batch * (w_id - wire.shape[1])
    dms.setSolution(sol)
    dms.setConstraintData(con)
    sol1, sd1, steps1 = dms.iteration_host_resident(wire, lin, res, dx0)
    # step by step
    dms.setSolution(sol)
    dms.setConstraintData(con)
    dms._up(LIN, lin, S.l_stride, None)
    dms.linearizeInverseDynamics()
    dms.linearizeContactKinematics()
    dms.condense()
    rr.backwardRiccatiRecursion()
    rr.forwardRiccatiRecursion(dx0)
    dms.computeStepSizes()
    dms.integrateSolution()
    steps = np.stack([dms.maxPrimalStepSize(), dms.maxDualStepSize()], axis=1)
    used = S.s_xi + S.nsm
    np.testing.assert_array_equal(sol1[:, :, :used], dms.getSolution()[:, :, :used])
    np.testing.assert_array_equal(steps1, steps)
    np.testing.assert_array_equal(sd1[:, :, :S.nc], dms.getConstraintData()[:, :, S.c_slack:S.c_slack + S.nc])
    dms.setWireCostStructure(False)
    rr.close()
