"""Contact rows of the contact / impact dynamics linearisation (rbt_linearize_contact_kinematics), CPU side.

There is no Pinocchio here, so the reference's contact code cannot run: tests/contact_ref.py restates the contact-frame
kinematics, the Baumgarte and impact-velocity residuals and their derivatives, and this file pins that restatement by central
differences in the tangent space, by the world-frame motion of the contact point, by rbd_ref.contact_jacobian and by the assembly
of point_contact.hxx:63-85 on Pinocchio-style LOCAL frame partials, on the ANYmal model and on seeded random floating-base trees.
It also checks the wire segment tables with RBT_WIRE_DEVICE_CONTACT."""
import ctypes
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import contact_ref as CR  # noqa: E402
import make_model_fixture  # noqa: E402
import rbd_ref as R  # noqa: E402

MODELS = ["anymal", "random1", "random2"]
GAINS = [(0.0, 0.0), (40.0, 12.0)]


def model_of(name):
    return make_model_fixture.load() if name == "anymal" else R.random_model(int(name[-1]))


def _state(seed, B=3, nv=18):
    return R.random_state(np.random.default_rng(seed), B, nv)


def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1.0)


def _unit(B, nv, k, h):
    e = np.zeros((B, nv))
    e[:, k] = h
    return e


@pytest.mark.parametrize("name", MODELS)
@pytest.mark.parametrize("kp,kv", GAINS)
def test_baumgarte_derivatives_match_central_differences(name, kp, kv):
    m = model_of(name)
    q, v, a = _state(11)
    B, nv, h = q.shape[0], 18, 1e-6
    p_des = np.random.default_rng(12).uniform(-1, 1, (B, 3))
    for c in range(int(m["n_contacts"])):
        dq, dv, da = CR.baumgarte_derivatives(m, q, v, a, c, kp, kv)
        C = lambda qq, vv, aa: CR.baumgarte_residual(m, qq, vv, aa, c, kp, kv, p_des)  # noqa: E731
        for k in range(nv):
            e = _unit(B, nv, k, h)
            assert _rel(dq[:, :, k], (C(R.integrate(q, e), v, a) - C(R.integrate(q, -e), v, a)) / (2 * h)) < 1e-6, (c, k)
            assert _rel(dv[:, :, k], (C(q, v + e, a) - C(q, v - e, a)) / (2 * h)) < 1e-6, (c, k)
            assert _rel(da[:, :, k], (C(q, v, a + e) - C(q, v, a - e)) / (2 * h)) < 1e-6, (c, k)


@pytest.mark.parametrize("name", MODELS)
def test_impact_velocity_derivatives_match_central_differences(name):
    m = model_of(name)
    q, v, _ = _state(13)
    B, nv, h = q.shape[0], 18, 1e-6
    for c in range(int(m["n_contacts"])):
        dq, dv = CR.impact_velocity_derivatives(m, q, v, c)
        C = lambda qq, vv: CR.impact_velocity_residual(m, qq, vv, c)  # noqa: E731
        for k in range(nv):
            e = _unit(B, nv, k, h)
            assert _rel(dq[:, :, k], (C(R.integrate(q, e), v) - C(R.integrate(q, -e), v)) / (2 * h)) < 1e-6, (c, k)
            assert _rel(dv[:, :, k], (C(q, v + e) - C(q, v - e)) / (2 * h)) < 1e-6, (c, k)


@pytest.mark.parametrize("name", MODELS)
def test_contact_point_motion_along_a_trajectory(name):
    """q(t) = integrate(q0, t v + t^2/2 a) passes q0 with velocity v and acceleration a: the world contact point satisfies
    p' = oRf v_f,lin and p'' = oRf a_cl -- the classical acceleration has no gravity term."""
    m = model_of(name)
    q0, v, a = _state(14)
    h = 1e-3
    path = lambda t: R.integrate(q0, t * v + 0.5 * t * t * a)  # noqa: E731
    for c in range(int(m["n_contacts"])):
        p = {t: CR.frame_placement(m, path(t), c)[1] for t in (-h, 0.0, h)}
        oRf, _ = CR.frame_placement(m, q0, c)
        vf, af, _, _ = CR.frame_motion(m, q0, v, a, c)
        pd = (p[h] - p[-h]) / (2 * h)
        pdd = (p[h] - 2 * p[0.0] + p[-h]) / (h * h)
        assert _rel(pd, np.einsum("bij,bj->bi", oRf, vf[:, :3])) < 1e-5, c
        assert _rel(pdd, np.einsum("bij,bj->bi", oRf, CR.classical_acceleration(vf, af))) < 1e-4, c


@pytest.mark.parametrize("name", MODELS)
def test_dCda_is_the_contact_jacobian(name):
    m = model_of(name)
    q, v, a = _state(15)
    for c in range(int(m["n_contacts"])):
        _, _, J = CR.baumgarte_derivatives(m, q, v, a, c, 40.0, 12.0)
        np.testing.assert_allclose(J, R.contact_jacobian(m, q, c), rtol=0, atol=1e-13 * max(1.0, np.abs(J).max()))
        _, Jimp = CR.impact_velocity_derivatives(m, q, v, c)
        np.testing.assert_array_equal(Jimp, J)


@pytest.mark.parametrize("name", MODELS)
@pytest.mark.parametrize("kp,kv", GAINS)
def test_pinocchio_assembly_equals_forward_mode(name, kp, kv):
    """point_contact.hxx:63-85 builds dC/dq, dC/dv from the LOCAL frame partials of getFrameAccelerationDerivatives and the
    LOCAL frame Jacobian with skew terms; here those partials come from central differences."""
    m = model_of(name)
    q, v, a = _state(16)
    B, nv, h = q.shape[0], 18, 1e-6
    skew = R.skew
    for c in range(int(m["n_contacts"])):
        vf, _, _, _ = CR.frame_motion(m, q, v, a, c)
        oRf, _ = CR.frame_placement(m, q, c)
        vdq, adq, adv, Jf = (np.zeros((B, 6, nv)) for _ in range(4))
        for k in range(nv):
            e = _unit(B, nv, k, h)
            vp, ap, _, _ = CR.frame_motion(m, R.integrate(q, e), v, a, c)
            vm, am, _, _ = CR.frame_motion(m, R.integrate(q, -e), v, a, c)
            vdq[:, :, k], adq[:, :, k] = (vp - vm) / (2 * h), (ap - am) / (2 * h)
            vp, ap, _, _ = CR.frame_motion(m, q, v + e, a, c)
            vm, am, _, _ = CR.frame_motion(m, q, v - e, a, c)
            Jf[:, :, k], adv[:, :, k] = (vp - vm) / (2 * h), (ap - am) / (2 * h)
        Wk, Vk = skew(vf[:, 3:]), skew(vf[:, :3])
        dq = adq[:, :3] + Wk @ vdq[:, :3] - Vk @ vdq[:, 3:] + kv * vdq[:, :3] + kp * oRf @ Jf[:, :3]
        dv = adv[:, :3] + Wk @ Jf[:, :3] - Vk @ Jf[:, 3:] + kv * Jf[:, :3]
        fq, fv, _ = CR.baumgarte_derivatives(m, q, v, a, c, kp, kv)
        assert _rel(fq, dq) < 1e-6, c
        assert _rel(fv, dv) < 1e-6, c


# ---- wire segment tables with RBT_WIRE_DEVICE_CONTACT
class _seg(ctypes.Structure):
    _fields_ = [(f, ctypes.c_int) for f in ("lin_off", "wire_off", "rows", "cols", "ld", "sym")]


class _zero(ctypes.Structure):
    _fields_ = [("lin_off", ctypes.c_int), ("n", ctypes.c_int)]


class _wl(ctypes.Structure):
    _fields_ = [("nseg", ctypes.c_int), ("nzero", ctypes.c_int), ("w_doubles", ctypes.c_int), ("ocp_off", ctypes.c_int),
                ("seg", _seg * 20), ("zero", _zero * 5)]


def _schedule(which):
    import helpers
    return {"trot": helpers.trot_schedule, "crawl": helpers.crawl_schedule, "mask_walk": helpers.contact_mask_walk_schedule,
            "jump": helpers.jump_sto_schedule}[which]()[2]


def _contact_segs(S, c, cs):
    """(lin_off, rows, cols, ld, sym) of the ID / contact-row segments of a non-terminal grid point: what rbt_make_wire_layout
    puts before Qaa."""
    nv, nx, nf = S.nv, S.nx, c.nf
    did, dcon = bool(cs & 2), bool(cs & 4)
    seg = []
    if not did:
        seg.append((S.l_M, nv, nv, nv, 1))
    if nf and not dcon:
        seg.append((S.l_J, nf, nv, S.nfm, 0))
    rows = (0 if did else nv) + (0 if dcon else nf)
    if rows:
        off = 0 if not did else nv
        seg += [(S.l_D + off, rows, nx, S.nvf, 0), (S.l_IDC + off, rows, 1, rows, 0)]
    return seg


def _unpack(W, wire, lin):
    """rbt_unpack_wire_record restated."""
    for k in range(W.nzero):
        z = W.zero[k]
        lin[z.lin_off:z.lin_off + z.n] = 0.0
    for k in range(W.nseg):
        g = W.seg[k]
        src = wire[g.wire_off:]
        for j in range(g.cols if g.sym == 0 else g.rows):
            for i in range(g.rows):
                if g.sym == 0:
                    lin[g.lin_off + i + j * g.ld] = src[i + j * g.rows]
                elif g.sym == 2:
                    if i == j:
                        lin[g.lin_off + i * (g.ld + 1)] = src[i]
                else:
                    lin[g.lin_off + i + j * g.ld] = src[j * (j + 1) // 2 + i] if i <= j else src[i * (i + 1) // 2 + j]


def _contact_sections(S, nf):
    """flat offsets of J's nf rows, the contact rows of dIDCdqv and IDC in a linearization record"""
    out = [S.l_J + r + k * S.nfm for k in range(S.nv) for r in range(nf)]
    out += [S.l_D + S.nv + r + k * S.nvf for k in range(S.nx) for r in range(nf)]
    return out + [S.l_IDC + S.nv + r for r in range(nf)]


def _id_sections(S):
    out = list(range(S.l_M, S.l_M + S.nv * S.nv))
    out += [S.l_D + r + k * S.nvf for k in range(S.nx) for r in range(S.nv)]
    return out + list(range(S.l_IDC, S.l_IDC + S.nv))


@pytest.mark.parametrize("which", ["trot", "crawl", "mask_walk", "jump"])
@pytest.mark.parametrize("cs", [4, 5, 6, 7])
def test_wire_tables_with_device_contact_kinematics(which, cs):
    from robotoc_b200 import ANYMAL, StageDims, StageLayout, anymal_constraint_table
    from robotoc_b200._lib import lib
    from robotoc_b200.grid import TERMINAL
    from synth import make_stage_inputs, symmetrize_lin
    table = anymal_constraint_table()
    sd = StageDims(ANYMAL, nf_max=12, n_contacts=4, n_box=table.n_box)
    S = StageLayout(sd)
    ctrl = _schedule(which)
    L = lib()
    csd = sd.c()
    n = len(ctrl)
    base = cs & ~4  # the same records with the contact rows on the wire
    total = {f: L.rbt_wire_doubles(ctypes.byref(csd), ctrl, n, f) for f in (base, cs)}
    lin = symmetrize_lin(S, make_stage_inputs(sd, S, ctrl, 1, 5)[0])[0]
    wire_b = np.zeros(total[base])
    wire_c = np.zeros(total[cs])
    assert L.rbt_pack_wire(ctypes.byref(csd), ctrl, n, base, lin.ctypes.data_as(ctypes.c_void_p),
                           wire_b.ctypes.data_as(ctypes.c_void_p), 1) == 0
    assert L.rbt_pack_wire(ctypes.byref(csd), ctrl, n, cs, lin.ctypes.data_as(ctypes.c_void_p),
                           wire_c.ctypes.data_as(ctypes.c_void_p), 1) == 0
    up2 = lambda x: (x + 1) & ~1  # noqa: E731
    dropped = 0
    for i in range(n):
        w, w0 = _wl(), _wl()
        assert L.rbt_wire_layout_get(ctypes.byref(csd), ctrl, n, cs, i, ctypes.byref(w)) == 0
        assert L.rbt_wire_layout_get(ctypes.byref(csd), ctrl, n, base, i, ctypes.byref(w0)) == 0
        got = [(w.seg[k].lin_off, w.seg[k].rows, w.seg[k].cols, w.seg[k].ld, w.seg[k].sym) for k in range(w.nseg)]
        ref = [(w0.seg[k].lin_off, w0.seg[k].rows, w0.seg[k].cols, w0.seg[k].ld, w0.seg[k].sym) for k in range(w0.nseg)]
        if ctrl[i].type == TERMINAL:
            assert got == ref
            continue
        nv, nf = S.nv, ctrl[i].nf
        # exactly the contact-row segments disappear: the tail (Qaa onwards) is the same
        k0, k1 = len(_contact_segs(S, ctrl[i], base)), len(_contact_segs(S, ctrl[i], cs))
        assert ref[:k0] == _contact_segs(S, ctrl[i], base)
        assert got[:k1] == _contact_segs(S, ctrl[i], cs)
        assert got[k1:] == ref[k0:]
        did = bool(cs & 2)
        if did:
            drop = (up2(nf * nv) + up2(nf * 2 * nv) + up2(nf)) if nf else 0
        else:
            drop = (up2(nf * nv) if nf else 0) + up2((nv + nf) * 2 * nv) + up2(nv + nf) - up2(nv * 2 * nv) - up2(nv)
        assert w0.w_doubles - w.w_doubles == drop
        dropped += drop
        # round trip: the dropped rows stay as the device left them, everything else is what the full wire record gives
        full = np.full(S.l_stride, np.nan)
        mine = np.full(S.l_stride, np.nan)
        _unpack(w0, wire_b[w0.ocp_off:], full)
        _unpack(w, wire_c[w.ocp_off:], mine)
        contact = _contact_sections(S, nf)
        assert np.isnan(mine[contact]).all()
        if nf:
            assert not np.isnan(full[contact]).any()
        keep = np.ones(S.l_stride, bool)
        keep[contact] = False
        if did:
            keep[_id_sections(S)] = False
        np.testing.assert_array_equal(mine[keep], full[keep])
    assert total[base] - total[cs] == dropped

