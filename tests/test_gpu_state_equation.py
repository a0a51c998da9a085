"""rbt_linearize_state_equation on the device: the kernel against the numpy restatement tests/state_ref.py (itself pinned by
tests/test_state_equation.py) on every section it writes with every other byte of the record unchanged, Fx and the SE(3)
blocks NaN-filled before the call, the error codes, a full iteration with all three device bits against host-filled records,
and the resident wire path with RBT_WIRE_DEVICE_ID | RBT_WIRE_DEVICE_CONTACT | RBT_WIRE_DEVICE_STATE against the step-by-step
calls.  Schedules: trot N=40, the jump with switching-time optimisation N=80 (STO terms), and a receding-horizon trot whose
grid point 1 is an impact (grid point 0 takes q_prev from q0, the impact from s[0].q)."""
import ctypes
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import contact_ref as CR  # noqa: E402
import make_model_fixture  # noqa: E402
import rbd_ref as R  # noqa: E402
import state_ref as SR  # noqa: E402
from helpers import jump_sto_schedule, receding_horizon_schedules, rel_err, trot_schedule  # noqa: E402
from synth import make_stage_inputs, symmetrize_lin  # noqa: E402

LIN, Q0 = 6, 14
IMPACT, TERMINAL = 1, 3


def _impact_at_1():
    for t0, td, ev, ctrl in receding_horizon_schedules("trot", False, "edge"):
        if ctrl[1].type == IMPACT:
            return ctrl
    raise AssertionError("no receding-horizon schedule with an impact on grid point 1")


SCHEDULES = {"trot": lambda: trot_schedule(40)[2], "jump": lambda: jump_sto_schedule(80)[2], "rh_impact1": _impact_at_1}


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


def _smooth(S, sol, seed):
    """The records' configurations as a trajectory (neighbours a few degrees and centimetres apart) and q0 next to s[0].q."""
    rng = np.random.default_rng(seed)
    B, n = sol.shape[0], sol.shape[1]
    out = sol.copy()
    q = SR.random_q0(seed, B, S.nq)
    q0 = R.integrate(q, 0.02 * rng.uniform(-1, 1, (B, S.nv)))
    for i in range(n):
        out[:, i, S.s_q:S.s_q + S.nq] = q
        q = R.integrate(q, 0.05 * rng.uniform(-1, 1, (B, S.nv)))
    return np.ascontiguousarray(out), q0


def _with_sto(ctrl):
    return any(c.sto or c.sto_next for c in ctrl)


def _written(S, ctrl):
    """[n_grid, l_stride] mask of what the kernel may write on each grid point."""
    nv, nx = S.nv, S.nx
    out = np.zeros((len(ctrl), S.l_stride), bool)
    sto = _with_sto(ctrl)
    for i, c in enumerate(ctrl):
        out[i, S.l_lx:S.l_lx + nx] = True
        if c.type == TERMINAL:
            out[i, S.l_se3 + 36:S.l_se3 + 72] = True
            continue
        out[i, S.l_Fx:S.l_Fx + nx] = True
        out[i, S.l_se3:S.l_se3 + 108] = True
        out[i, S.l_la:S.l_la + nv] = True
        if sto and c.type != IMPACT:
            out[i, S.l_sc] = True
            out[i, S.l_hx + nv:S.l_hx + nx] = True
            out[i, S.l_ha:S.l_ha + nv] = True
            out[i, S.l_fx:S.l_fx + nx] = True
    return out


def _sections(S):
    nv = S.nv
    return {"Fx": (S.l_Fx, 2 * nv), "se3": (S.l_se3, 108), "lx": (S.l_lx, 2 * nv), "la": (S.l_la, nv), "h": (S.l_sc, 1),
            "hv": (S.l_hx + nv, nv), "ha": (S.l_ha, nv), "fx": (S.l_fx, 2 * nv)}


CASES = [(s, b) for s in SCHEDULES for b in (1, 3)] + [("trot", 1024)]


@pytest.mark.gpu
@pytest.mark.parametrize("which,batch", CASES)
def test_kernel_matches_the_restatement(which, batch):
    ctrl = SCHEDULES[which]()
    rr, dms, S, lin, con, sol, dx0 = _setup(ctrl, batch, 91)
    q0 = SR.random_q0(92, batch, S.nq)
    dms.setInitialConfiguration(q0)
    dms._up(LIN, lin, S.l_stride, None)
    dms.setSolution(sol)
    dms.linearizeStateEquation()
    got = dms._down(LIN, lin.shape)
    ref = SR.linearize(S, ctrl, sol, lin, q0)
    for name, (o, n) in _sections(S).items():
        assert rel_err(got[:, :, o:o + n], ref[:, :, o:o + n]) < 1e-12, name
    w = _written(S, ctrl)
    for i in range(len(ctrl)):  # every other byte of the record is what was uploaded
        np.testing.assert_array_equal(got[:, i, ~w[i]], lin[:, i, ~w[i]])
    np.testing.assert_array_equal(dms._down(Q0, q0.shape), q0)
    rr.close()


@pytest.mark.gpu
@pytest.mark.parametrize("which", list(SCHEDULES))
def test_nan_filled_blocks_give_the_same_result(which):
    """Fx, the SE(3) blocks and fx are overwritten, never read: NaN there before the call changes nothing."""
    ctrl = SCHEDULES[which]()
    rr, dms, S, lin, con, sol, dx0 = _setup(ctrl, 3, 93)
    q0 = SR.random_q0(94, 3, S.nq)
    dms.setInitialConfiguration(q0)
    dms.setSolution(sol)
    out = {}
    for fill in (False, True):
        l = lin.copy()
        if fill:
            l[:, :, S.l_Fx:S.l_Fx + S.nx] = np.nan
            l[:, :, S.l_se3:S.l_se3 + 108] = np.nan
            if _with_sto(ctrl):
                l[:, :, S.l_fx:S.l_fx + S.nx] = np.nan
            for i, c in enumerate(ctrl):
                if c.type == TERMINAL:  # only Fqq_prev is written there
                    l[:, i, S.l_Fx:S.l_Fx + S.nx] = lin[:, i, S.l_Fx:S.l_Fx + S.nx]
                    l[:, i, S.l_se3:S.l_se3 + 36] = lin[:, i, S.l_se3:S.l_se3 + 36]
                    l[:, i, S.l_se3 + 72:S.l_se3 + 108] = lin[:, i, S.l_se3 + 72:S.l_se3 + 108]
                if c.type in (TERMINAL, IMPACT) and _with_sto(ctrl):
                    l[:, i, S.l_fx:S.l_fx + S.nx] = lin[:, i, S.l_fx:S.l_fx + S.nx]
        dms._up(LIN, np.ascontiguousarray(l), S.l_stride, None)
        dms.linearizeStateEquation()
        out[fill] = dms._down(LIN, lin.shape)
    np.testing.assert_array_equal(out[True], out[False])
    rr.close()


@pytest.mark.gpu
def test_error_codes():
    from robotoc_b200 import ANYMAL, RiccatiRecursion
    from robotoc_b200._lib import lib
    L = lib()
    rr0 = RiccatiRecursion(ANYMAL, 3, 1)
    assert L.rbt_linearize_state_equation(rr0._h, None) == 3              # no stage layer
    rr0.close()
    ctrl = SCHEDULES["trot"]()
    rr, dms, S, lin, con, sol, dx0 = _setup(ctrl, 2, 95)
    q0 = SR.random_q0(96, 2, S.nq)
    assert L.rbt_linearize_state_equation(rr._h, None) == 3              # no q0
    assert L.rbt_download(rr._h, Q0, q0.ctypes.data_as(ctypes.c_void_p), None) == 3  # not uploaded yet
    with pytest.raises(ValueError):
        dms.setInitialConfiguration(q0[:, :-1])
    assert L.rbt_set_wire_cost_structure(rr._h, 32) == 1                 # unknown bit
    dms.setWireCostStructure(False, device_state_equation=True)          # alone: the ID and contact rows still travel
    wire = dms.pack_wire(lin)
    res = np.ascontiguousarray(con[:, :, S.c_res:S.c_res + S.ncp])
    dms.setSolution(sol)
    dms.setConstraintData(con)
    with pytest.raises(RuntimeError):                                      # the wire path needs q0
        dms.iteration_host_resident(wire, lin, res, dx0)
    with pytest.raises(RuntimeError):
        dms.iteration_host_wire(wire, lin, con, sol, dx0)
    dms.setInitialConfiguration(q0)
    dms.linearizeStateEquation()
    sol1, sd1, steps1 = dms.iteration_host_resident(wire, lin, res, dx0)
    assert np.isfinite(sol1).all() and np.isfinite(steps1).all()
    dms.setWireCostStructure(False)
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
    """The records a host that sets all three device bits sends: the ID, contact and state-equation rows NaN (never read)."""
    out = lin.copy()
    for i, c in enumerate(ctrl):
        r = out[:, i]
        if c.type == TERMINAL:
            r[:, S.l_se3 + 36:S.l_se3 + 72] = np.nan
            continue
        r[:, S.l_M:S.l_M + S.nv * S.nv] = np.nan
        D = r[:, S.l_D:S.l_D + S.nvf * S.nx].reshape(-1, S.nx, S.nvf)
        D[:, :, :S.nv + c.nf] = np.nan
        r[:, S.l_D:S.l_D + S.nvf * S.nx] = D.reshape(r.shape[0], -1)
        r[:, S.l_IDC:S.l_IDC + S.nv + c.nf] = np.nan
        J = r[:, S.l_J:S.l_J + S.nfm * S.nv].reshape(-1, S.nv, S.nfm)
        J[:, :, :c.nf] = np.nan
        r[:, S.l_J:S.l_J + S.nfm * S.nv] = J.reshape(r.shape[0], -1)
        r[:, S.l_Fx:S.l_Fx + S.nx] = np.nan
        r[:, S.l_se3:S.l_se3 + 108] = np.nan
        out[:, i] = r
    return np.ascontiguousarray(out)


def _device_inputs(dms, ctrl, batch, seed):
    m = make_model_fixture.load()
    gains, pos = CR.random_gains(seed, 4), CR.random_positions(seed + 1, batch, len(ctrl), 4)
    dms.setRobotModel(R.to_c(m))
    dms.setContactGains(gains)
    dms.setContactPositions(pos)
    return m, gains, pos


@pytest.mark.gpu
@pytest.mark.parametrize("which,batch", [("trot", 3), ("jump", 3), ("rh_impact1", 3), ("trot", 1024)])
def test_iteration_with_all_device_rows_matches_host_filled_records(which, batch):
    ctrl = SCHEDULES[which]()
    rr, dms, S, lin, con, sol, dx0 = _setup(ctrl, batch, 97)
    sol, q0 = _smooth(S, sol, 98)
    m, gains, pos = _device_inputs(dms, ctrl, batch, 99)
    dms.setInitialConfiguration(q0)
    # host-filled ID, contact and state-equation rows, in the reference's order
    host = SR.linearize(S, ctrl, sol, CR.linearize(m, S, ctrl, sol, R.linearize(m, S, ctrl, sol, lin), gains, pos), q0)
    dms.setSolution(sol)
    dms._up(LIN, host, S.l_stride, None)
    dms.setConstraintData(con)
    a = _steps_of(rr, dms, dx0)
    # device-filled: the uploaded rows are ignored, the gradients lack the beta, mu and costate terms
    dms._up(LIN, _without_device_rows(S, ctrl, lin), S.l_stride, None)
    dms.setConstraintData(con)
    dms.setSolution(sol)
    dms.linearizeInverseDynamics()
    dms.linearizeContactKinematics()
    dms.linearizeStateEquation()
    b = _steps_of(rr, dms, dx0)
    for k in a:
        assert np.isfinite(b[k]).all(), k
        assert rel_err(b[k], a[k]) < 1e-10, k
    rr.close()


@pytest.mark.gpu
@pytest.mark.parametrize("which,batch", [("trot", 3), ("jump", 3), ("rh_impact1", 200)])
def test_resident_wire_path_with_all_device_bits(which, batch):
    ctrl = SCHEDULES[which]()
    rr, dms, S, lin, con, sol, dx0 = _setup(ctrl, batch, 101)
    sol, q0 = _smooth(S, sol, 102)
    res = np.ascontiguousarray(con[:, :, S.c_res:S.c_res + S.ncp])
    _device_inputs(dms, ctrl, batch, 103)
    dms.setInitialConfiguration(q0)
    dms.setWireCostStructure(False, device_inverse_dynamics=True, device_contact_kinematics=True)
    two = dms.iteration_host_bytes(resident=True)[0]
    dms.setWireCostStructure(False, device_inverse_dynamics=True, device_contact_kinematics=True, device_state_equation=True)
    wire = dms.pack_wire(lin)
    assert two - dms.iteration_host_bytes(resident=True)[0] == 8 * batch * (144 * (len(ctrl) - 1) + 36)
    dms.setSolution(sol)
    dms.setConstraintData(con)
    sol1, sd1, steps1 = dms.iteration_host_resident(wire, lin, res, dx0)
    # step by step
    dms.setSolution(sol)
    dms.setConstraintData(con)
    dms._up(LIN, lin, S.l_stride, None)
    dms.linearizeInverseDynamics()
    dms.linearizeContactKinematics()
    dms.linearizeStateEquation()
    dms.condense()
    rr.backwardRiccatiRecursion()
    rr.forwardRiccatiRecursion(dx0)
    dms.computeStepSizes()
    dms.integrateSolution()
    steps = np.stack([dms.maxPrimalStepSize(), dms.maxDualStepSize()], axis=1)
    used = S.s_xi + S.nsm
    assert np.isfinite(sol1[:, :, :used]).all()
    np.testing.assert_array_equal(sol1[:, :, :used], dms.getSolution()[:, :, :used])
    np.testing.assert_array_equal(steps1, steps)
    np.testing.assert_array_equal(sd1[:, :, :S.nc], dms.getConstraintData()[:, :, S.c_slack:S.c_slack + S.nc])
    dms.setWireCostStructure(False)
    rr.close()
