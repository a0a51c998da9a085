"""Inverse dynamics of the contact-dynamics linearisation (rbt_linearize_inverse_dynamics), CPU side.

There is no Pinocchio here, so the reference's robot code cannot run: tests/rbd_ref.py restates RNEA and its derivatives, and
this file pins that restatement by central differences in the tangent space and by physical identities, on the ANYmal model
(tests/golden/anymal_model.npz, parsed from the reference's URDF) and on seeded random floating-base trees.  It also checks the
validation of rbt_robot_model and the wire segment tables with RBT_WIRE_DEVICE_ID."""
import ctypes
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_model_fixture  # noqa: E402
import rbd_ref as R  # noqa: E402

MODELS = ["anymal", "random1", "random2"]


def model_of(name):
    return make_model_fixture.load() if name == "anymal" else R.random_model(int(name[-1]))


def _state(seed, B=3, nv=18):
    return R.random_state(np.random.default_rng(seed), B, nv)


def _fext(model, seed, B, mask=0b1111):
    f = np.random.default_rng(seed).uniform(-20, 20, (B, 12))
    return R.contact_fext(model, f, mask), f


def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1.0)


@pytest.mark.parametrize("name", MODELS)
def test_derivatives_match_central_differences(name):
    m = model_of(name)
    q, v, a = _state(1)
    fx, _ = _fext(m, 2, q.shape[0], 0b1011)
    tau, dq, dv, M = R.rnea_derivatives(m, q, v, a, fx)
    h, nv = 1e-6, 18
    for k in range(nv):
        e = np.zeros((q.shape[0], nv))
        e[:, k] = h
        fd_q = (R.rnea(m, R.integrate(q, e), v, a, fx) - R.rnea(m, R.integrate(q, -e), v, a, fx)) / (2 * h)
        fd_v = (R.rnea(m, q, v + e, a, fx) - R.rnea(m, q, v - e, a, fx)) / (2 * h)
        fd_a = (R.rnea(m, q, v, a + e, fx) - R.rnea(m, q, v, a - e, fx)) / (2 * h)
        assert _rel(dq[:, :, k], fd_q) < 1e-6, k
        assert _rel(dv[:, :, k], fd_v) < 1e-6, k
        assert _rel(M[:, :, k], fd_a) < 1e-6, k


@pytest.mark.parametrize("name", MODELS)
def test_mass_matrix_is_spd_and_gives_the_kinetic_energy(name):
    m = model_of(name)
    q, v, a = _state(3)
    _, _, _, M = R.rnea_derivatives(m, q, v, a)
    assert np.array_equal(M, np.swapaxes(M, 1, 2))
    assert np.linalg.eigvalsh(M).min() > 0
    np.testing.assert_allclose(0.5 * np.einsum("bi,bij,bj->b", v, M, v), R.kinetic_energy(m, q, v), rtol=1e-12)


@pytest.mark.parametrize("name", MODELS)
def test_static_torque_is_the_gradient_of_the_potential_energy(name):
    m = model_of(name)
    q, _, _ = _state(4)
    z = np.zeros((q.shape[0], 18))
    g = R.rnea(m, q, z, z)
    h = 1e-6
    for k in range(18):
        e = np.zeros_like(z)
        e[:, k] = h
        fd = (R.potential_energy(m, R.integrate(q, e)) - R.potential_energy(m, R.integrate(q, -e))) / (2 * h)
        np.testing.assert_allclose(g[:, k], fd, rtol=1e-6, atol=1e-6 * np.abs(g).max())


@pytest.mark.parametrize("name", MODELS)
def test_inverse_dynamics_is_affine_in_a_and_f(name):
    m = model_of(name)
    q, v, a = _state(5)
    fx1, _ = _fext(m, 6, q.shape[0])
    fx2, _ = _fext(m, 7, q.shape[0])
    a2 = np.random.default_rng(8).uniform(-1, 1, a.shape)
    t = lambda aa, ff: R.rnea(m, q, v, aa, ff)  # noqa: E731
    np.testing.assert_allclose(t(a + 2.5 * a2, fx1) - t(a, fx1), 2.5 * (t(a2, fx1) - t(np.zeros_like(a), fx1)), rtol=1e-10, atol=1e-10)
    np.testing.assert_allclose(t(a, fx1 + 0.5 * fx2) - t(a, fx1), 0.5 * (t(a, fx2) - t(a, 0 * fx2)), rtol=1e-10, atol=1e-10)


@pytest.mark.parametrize("name", MODELS)
@pytest.mark.parametrize("mask", [0b0000, 0b0101, 0b1111])
def test_impact_variant_is_M_dv_minus_Jt_f(name, mask):
    m = model_of(name)
    q, _, dv = _state(9)
    fx, f = _fext(m, 10, q.shape[0], mask)
    z = np.zeros_like(dv)
    tau, _, _, M = R.rnea_derivatives(m, q, z, dv, fx, gravity=False)
    expect = np.einsum("bij,bj->bi", M, dv)
    k = 0
    for c in range(4):
        if (mask >> c) & 1:
            expect -= np.einsum("bki,bk->bi", R.contact_jacobian(m, q, c), f[:, k:k + 3])
            k += 3
    np.testing.assert_allclose(tau, expect, rtol=1e-10, atol=1e-10 * np.abs(expect).max())


# ---- rbt_robot_model validation (a handle needs a device)
def _handle_with_stage():
    from robotoc_b200 import ANYMAL, DirectMultipleShooting, RiccatiRecursion, StageDims, anymal_constraint_table
    table = anymal_constraint_table()
    sd = StageDims(ANYMAL, nf_max=12, n_contacts=4, n_box=table.n_box)
    rr = RiccatiRecursion(ANYMAL, 3, 1)
    return rr, DirectMultipleShooting(rr, sd, table)


def _malformed(case):
    m = make_model_fixture.load()
    if case == "nv":
        m["nv"] = 17
    elif case == "n_contacts":
        m["n_contacts"] = 3
    elif case == "parent_later":
        m["parent"] = m["parent"].copy(); m["parent"][4] = 5
    elif case == "parent_root":
        m["parent"] = m["parent"].copy(); m["parent"][0] = 0
    elif case == "mass":
        m["mass"] = m["mass"].copy(); m["mass"][3] = 0.0
    elif case == "inertia_asym":
        m["inertia"] = m["inertia"].copy(); m["inertia"][2][3] += 1e-3
    elif case == "inertia_indef":
        m["inertia"] = m["inertia"].copy(); m["inertia"][5][8] = -m["inertia"][5][8]
    elif case == "axis":
        m["axis"] = m["axis"].copy(); m["axis"][7] = m["axis"][7] * 1.01
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["nv", "n_contacts", "parent_later", "parent_root", "mass", "inertia_asym", "inertia_indef",
                                  "axis"])
def test_robot_model_validation_rejects(case):
    rr, dms = _handle_with_stage()
    with pytest.raises(ValueError):
        dms.setRobotModel(R.to_c(_malformed(case)))
    dms.setRobotModel(R.to_c(make_model_fixture.load()))  # the well-formed model is accepted
    rr.close()


# ---- wire segment tables with RBT_WIRE_DEVICE_ID
def _wire_numpy(S, c, cs):
    """restatement of rbt_make_wire_layout for a non-terminal grid point: (lin_off, rows, cols, ld, sym) per segment."""
    nv, nx, nf, did, dc = S.nv, S.nx, c.nf, bool(cs & 2), bool(cs & 1)
    seg = []
    if not did:
        seg += [(S.l_M, nv, nv, nv, 1)] + ([(S.l_J, nf, nv, S.nfm, 0)] if nf else []) + [(S.l_D, nv + nf, nx, S.nvf, 0),
                                                                                      (S.l_IDC, nv + nf, 1, nv + nf, 0)]
    elif nf:
        seg += [(S.l_J, nf, nv, S.nfm, 0), (S.l_D + nv, nf, nx, S.nvf, 0), (S.l_IDC + nv, nf, 1, nf, 0)]
    seg.append((S.l_Qaa, nv, 1, nv, 0))
    if nf:
        seg.append((S.l_Qff, nf, nf, S.nfm, 2 if dc else 1))
    seg += [(S.l_Qxx, nv, nv, nx, 1), (S.l_Qxx + nv * nx + nv, nv, nv, nx, 2)] if dc else [(S.l_Qxx, nx, nx, nx, 1)]
    seg.append((S.l_Quu, S.nu, S.nu, S.nu, 2 if dc else 1))
    seg.append((S.l_lx, S.l_Phix - S.l_lx, 1, S.l_Phix - S.l_lx, 0))
    for ci in range(S.ncon):
        if (c.contact_mask >> ci) & 1:
            seg += [(S.l_dgdq + ci * 5 * nv, 5 * nv, 1, 5 * nv, 0), (S.l_dgdf + ci * 15, 15, 1, 15, 0)]
    return seg


@pytest.mark.parametrize("cs", [2, 3])
def test_wire_tables_with_device_inverse_dynamics(cs):
    from helpers import trot_schedule
    from robotoc_b200 import ANYMAL, StageDims, StageLayout, anymal_constraint_table
    from robotoc_b200._lib import lib
    from robotoc_b200.grid import TERMINAL
    table = anymal_constraint_table()
    sd = StageDims(ANYMAL, nf_max=12, n_contacts=4, n_box=table.n_box)
    S = StageLayout(sd)
    _, _, ctrl = trot_schedule()
    L = lib()
    csd = sd.c()

    class seg_t(ctypes.Structure):
        _fields_ = [(f, ctypes.c_int) for f in ("lin_off", "wire_off", "rows", "cols", "ld", "sym")]

    class zero_t(ctypes.Structure):
        _fields_ = [("lin_off", ctypes.c_int), ("n", ctypes.c_int)]

    class wl_t(ctypes.Structure):
        _fields_ = [("nseg", ctypes.c_int), ("nzero", ctypes.c_int), ("w_doubles", ctypes.c_int), ("ocp_off", ctypes.c_int),
                    ("seg", seg_t * 20), ("zero", zero_t * 5)]

    n = len(ctrl)
    total = {}
    for flag in (cs & 1, cs):
        total[flag] = L.rbt_wire_doubles(ctypes.byref(csd), ctrl, n, flag)
    dropped = 0
    for i in range(n):
        w, w0 = wl_t(), wl_t()
        assert L.rbt_wire_layout_get(ctypes.byref(csd), ctrl, n, cs, i, ctypes.byref(w)) == 0
        assert L.rbt_wire_layout_get(ctypes.byref(csd), ctrl, n, cs & 1, i, ctypes.byref(w0)) == 0
        if ctrl[i].type == TERMINAL:
            assert w.w_doubles == w0.w_doubles
            continue
        got = [(w.seg[k].lin_off, w.seg[k].rows, w.seg[k].cols, w.seg[k].ld, w.seg[k].sym) for k in range(w.nseg)]
        assert got == _wire_numpy(S, ctrl[i], cs)
        nv, nf = S.nv, ctrl[i].nf
        up2 = lambda x: (x + 1) & ~1  # noqa: E731
        drop = up2(nv * (nv + 1) // 2) + up2((nv + nf) * 2 * nv) + up2(nv + nf) - (up2(nf * 2 * nv) + up2(nf) if nf else 0)
        assert w0.w_doubles - w.w_doubles == drop
        dropped += drop
    assert total[cs & 1] - total[cs] == dropped
