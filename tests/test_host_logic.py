"""CPU-only tests: C-ABI surface, layouts, schedule producer, sharding (no compute calls without a GPU)."""
import ctypes
import os
import re

import numpy as np
import pytest

import oracle_lib
from helpers import jump_sto_schedule, small_event_schedule, trot_schedule
from robotoc_b200 import ANYMAL, Layout, ULayout, _lib
from robotoc_b200.grid import IMPACT, INTERMEDIATE, LIFT, TERMINAL
from robotoc_b200.shard import shard_range

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "robotoc_b200.h")).read()
    declared = set(re.findall(r"\b(rbt_[a-z_0-9]+)\s*\(", hdr))
    declared -= {"rbt_make_layout", "rbt_make_ulayout"}
    assert declared == set(_lib.EXPORTS), declared ^ set(_lib.EXPORTS)
    L = _lib.lib()
    for name in declared:
        assert hasattr(L, name), name
    assert b"sm_90a" in L.rbt_version()


def test_no_cpu_fallback_without_device():
    """On a box without a GPU the compute entry points must fail loudly, never fall back."""
    L = _lib.lib()
    sm, nsm = ctypes.c_int(), ctypes.c_int()
    if L.rbt_device_info(0, ctypes.byref(sm), ctypes.byref(nsm), None, 0) == 0:
        pytest.skip("a CUDA device is present")
    from robotoc_b200 import RiccatiRecursion
    with pytest.raises(RuntimeError):
        RiccatiRecursion(ANYMAL, 10, 2)


def test_unsupported_dims_are_argument_errors():
    L = _lib.lib()
    h = ctypes.c_void_p()
    d = _lib.rbt_dims(5, 3, 3, 0)
    assert L.rbt_create(ctypes.byref(d), 10, 2, 0, ctypes.byref(h)) == 1  # RBT_ERR_ARG before touching CUDA
    assert L.rbt_unconstr_create(0, 10, 0.1, 1, 0, ctypes.byref(h)) == 1
    assert L.rbt_unconstr_create(7, 10, -0.1, 1, 0, ctypes.byref(h)) == 1


def test_layouts_match_between_product_and_oracle():
    lib = oracle_lib.load()
    La = Layout(ANYMAL)
    Lb = Layout(ANYMAL, getter=lib.orc_layout_get)
    for k, v in vars(La).items():
        if isinstance(v, int):
            assert getattr(Lb, k) == v, k
    Ua, Ub = ULayout(7), ULayout(7, getter=lib.orc_ulayout_get)
    for k, v in vars(Ua).items():
        if isinstance(v, int):
            assert getattr(Ub, k) == v, k
    # SURVEY.md 8(d) per-stage figures
    nx, nu, nv = 36, 12, 18
    assert La.k_core_size == nx * nx + nv * nu + nx * nx + nx * nu + nu * nu + nx + nx + nu == 3468
    assert La.r_core_size == nx * nx + nx + nu * nx + nu == 1776
    assert La.k_stride % 16 == 0 and La.r_stride % 16 == 0 and La.d_stride % 16 == 0
    for f in ("k_Fxx", "k_Fvu", "k_Qxx", "k_Phix", "k_fx", "r_P", "r_K", "r_M", "r_Psi", "r_dtsdx", "d_dx", "d_du"):
        assert getattr(La, f) % 2 == 0, f  # 16-byte granule of cp.async.bulk


def test_trot_schedule_config3():
    """examples/anymal/trot.cpp:41-47,172-190 with N=40: 47 grid points, 2 Lift, 2 Impact, 2 switching stages (ns=6)."""
    td, ev, ctrl = trot_schedule(40)
    types = [c.type for c in ctrl]
    assert len(ctrl) == 47 and types[-1] == TERMINAL
    assert types.count(LIFT) == 2 and types.count(IMPACT) == 2
    sw = [i for i, c in enumerate(ctrl) if c.ns > 0]
    assert len(sw) == 2 and all(ctrl[i].ns == 6 and ctrl[i + 2].type == IMPACT for i in sw)
    assert all(c.dt == 0.0 for c in ctrl if c.type in (IMPACT, TERMINAL))
    assert abs(sum(c.dt for c in ctrl) - 1.12) < 1e-12
    assert not any(c.sto or c.sto_next for c in ctrl)
    # contact dimension per phase: 12 -> 6 -> 12 -> 6 -> 12
    assert [ctrl[0].nf, ctrl[3].nf, ctrl[23].nf, ctrl[30].nf, ctrl[45].nf] == [12, 6, 12, 6, 12]


def test_jump_sto_schedule_config4():
    """examples/anymal/jump_sto.cpp:42-48,131-140 with N=80: 84 grid points, all three phases STO-enabled."""
    td, ev, ctrl = jump_sto_schedule(80)
    assert len(ctrl) == 84
    types = [c.type for c in ctrl]
    assert types.count(LIFT) == 1 and types.count(IMPACT) == 1
    imp = types.index(IMPACT)
    assert ctrl[imp - 2].ns == 12 and ctrl[imp].sto and not ctrl[imp].sto_next
    assert all(c.sto for c in ctrl[:-1])
    assert ctrl[0].sto_next and ctrl[types.index(LIFT)].sto_next
    # num_grids_in_phase is what expandDual divides by (intermediate_stage.cpp:167-172)
    assert ctrl[0].ngrids_in_phase == types.index(LIFT)


def test_small_event_schedule_shapes():
    td, ev, ctrl = small_event_schedule(sto=False)
    assert [c.type for c in ctrl].count(INTERMEDIATE) == len(ctrl) - 3


@pytest.mark.parametrize("batch,world", [(1024, 8), (1000, 8), (7, 3), (0, 2), (5, 8)])
def test_shard_range_partitions(batch, world):
    spans = [shard_range(batch, world, r) for r in range(world)]
    assert spans[0][0] == 0 and spans[-1][1] == batch
    for (a, b), (c, d) in zip(spans, spans[1:]):
        assert b == c and a <= b
    sizes = [b - a for a, b in spans]
    assert max(sizes) - min(sizes) <= 1
    with pytest.raises(ValueError):
        shard_range(batch, world, world)


def test_wire_format_pack_is_documented_packed_upper_storage():
    """rbt_pack_wire (host helper of the C ABI) against an independent numpy restatement of the format in
    include/rbt_stage_layout.h: per grid point M / Qff / Qxx / Quu as column-major packed upper triangles, contact blocks sized
    by the active contact dimension, cone Jacobians of the active contacts only, no Qqf, the STO section only on schedules with
    a switching-time stage, three blocks on the terminal grid point."""
    import ctypes
    from robotoc_b200 import ANYMAL, StageDims, StageLayout, anymal_constraint_table
    from robotoc_b200._lib import lib
    from robotoc_b200.grid import TERMINAL
    from synth import make_stage_inputs
    from helpers import small_event_schedule
    L = lib()
    tab = anymal_constraint_table()
    sd = StageDims(ANYMAL, nf_max=12, n_contacts=tab.n_contacts, n_box=tab.n_box)
    S = StageLayout(sd)
    csd = sd.c()
    nv, nx, nu, nfm, nvfm = 18, 36, 12, 12, 30
    up2 = lambda n: n + (n & 1)  # noqa: E731
    for sto in (False, True):
        td, ev, ctrl = small_event_schedule(sto)
        n_grid = len(ctrl)
        lin, con, sol, dx0 = make_stage_inputs(sd, S, ctrl, 2, seed=4)
        with_sto = any(c.sto or c.sto_next for c in ctrl)
        assert with_sto == sto
        w = L.rbt_wire_doubles(ctypes.byref(csd), ctrl, n_grid, 0)
        wire = np.zeros((2, w))
        assert L.rbt_pack_wire(ctypes.byref(csd), ctrl, n_grid, 0, lin.ctypes.data_as(ctypes.c_void_p),
                               wire.ctypes.data_as(ctypes.c_void_p), 2) == 0
        o = 0
        for i, c in enumerate(ctrl):
            rec, back = lin[1, i], np.zeros(S.l_stride)
            nf = c.nf
            if c.type == TERMINAL:
                segs = [("sym", S.l_Qxx, nx, nx), ("d", S.l_lx, nx, 1, nx), ("d", S.l_se3 + 36, 36, 1, 36)]
            else:
                segs = [("sym", S.l_M, nv, nv)]
                if nf:
                    segs.append(("d", S.l_J, nf, nv, nfm))
                segs += [("d", S.l_D, nv + nf, nx, nvfm), ("d", S.l_IDC, nv + nf, 1, nv + nf), ("d", S.l_Qaa, nv, 1, nv)]
                if nf:
                    segs.append(("sym", S.l_Qff, nf, nfm))
                segs += [("sym", S.l_Qxx, nx, nx), ("sym", S.l_Quu, nu, nu), ("d", S.l_lx, S.l_Phix - S.l_lx, 1, S.l_Phix - S.l_lx)]
                for ci in range(4):
                    if (c.contact_mask >> ci) & 1:
                        segs += [("d", S.l_dgdq + ci * 90, 90, 1, 90), ("d", S.l_dgdf + ci * 15, 15, 1, 15)]
                if with_sto:
                    segs.append(("d", S.l_ha, S.l_dgdq - S.l_ha, 1, S.l_dgdq - S.l_ha))
            keep = np.zeros(S.l_stride, bool)
            want = rec.copy()
            for sg in segs:
                if sg[0] == "d":
                    _, off, rows, cols, ld = sg
                    blk = wire[1, o:o + rows * cols].reshape(cols, rows)
                    for j in range(cols):
                        back[off + j * ld:off + j * ld + rows] = blk[j]
                        keep[off + j * ld:off + j * ld + rows] = True
                    o += up2(rows * cols)
                else:
                    _, off, n, ld = sg
                    a = np.zeros((n, n))
                    for j in range(n):
                        for r in range(j + 1):
                            a[r, j] = a[j, r] = wire[1, o + j * (j + 1) // 2 + r]
                    for j in range(n):
                        back[off + j * ld:off + j * ld + n] = a[:, j]
                        keep[off + j * ld:off + j * ld + n] = True
                        col = want[off + j * ld:off + j * ld + n]
                        for r in range(j + 1, n):           # upper triangle authoritative
                            col[r] = rec[off + r * ld + j]
                    o += up2(n * (n + 1) // 2)
            np.testing.assert_array_equal(back[keep], want[keep])
            assert not keep[S.l_Qqf:S.l_Qxx].any() and not keep[S.l_Phix:S.l_ha].any()
        assert o == w
        if not sto:
            full = 3104 - 118  # the record of a 4-contact intermediate grid point without the STO section
            n4 = sum(1 for c in ctrl if c.type != TERMINAL and c.nf == 12)
            assert w < full * n_grid and (n4 == 0 or w > 0)


def test_wire_format_robotoc_cost_structure():
    """RBT_COST_ROBOTOC wire records: Qqq packed + diag(Qvv), diag(Quu), diag(Qff) instead of the full packed triangles; the
    segment table says where each piece sits, and the packed values are the diagonals / the Qqq triangle of the dense record."""
    import ctypes
    from robotoc_b200 import ANYMAL, StageDims, StageLayout, anymal_constraint_table
    from robotoc_b200._lib import lib
    from robotoc_b200.grid import TERMINAL
    from synth import make_stage_inputs, robotoc_cost_structure
    from helpers import small_event_schedule
    L = lib()
    tab = anymal_constraint_table()
    sd = StageDims(ANYMAL, nf_max=12, n_contacts=tab.n_contacts, n_box=tab.n_box)
    S = StageLayout(sd)
    csd = sd.c()
    td, ev, ctrl = small_event_schedule(False)
    n_grid = len(ctrl)
    lin, con, sol, dx0 = make_stage_inputs(sd, S, ctrl, 2, seed=5)
    lin = robotoc_cost_structure(S, lin)
    up2 = lambda n: n + (n & 1)  # noqa: E731
    w0 = L.rbt_wire_doubles(ctypes.byref(csd), ctrl, n_grid, 0)
    w1 = L.rbt_wire_doubles(ctypes.byref(csd), ctrl, n_grid, 1)
    save = sum((666 - 172 - 18) + (0 if c.type == TERMINAL else (78 - 12) + up2(c.nf * (c.nf + 1) // 2) - up2(c.nf)) for c in ctrl)
    assert w0 - w1 == save
    wire = np.zeros((2, w1))
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    assert L.rbt_pack_wire(ctypes.byref(csd), ctrl, n_grid, 1, P(lin), P(wire), 2) == 0

    class Seg(ctypes.Structure):
        _fields_ = [(k, ctypes.c_int) for k in ("lin_off", "wire_off", "rows", "cols", "ld", "sym")]

    class Zero(ctypes.Structure):
        _fields_ = [("lin_off", ctypes.c_int), ("n", ctypes.c_int)]

    class WL(ctypes.Structure):
        _fields_ = [(k, ctypes.c_int) for k in ("nseg", "nzero", "w_doubles", "ocp_off")] + [("seg", Seg * 20), ("zero", Zero * 5)]

    for i, c in enumerate(ctrl):
        W = WL()
        assert L.rbt_wire_layout_get(ctypes.byref(csd), ctrl, n_grid, 1, i, ctypes.byref(W)) == 0
        rec = lin[1, i]
        back = rec.copy()
        for k in range(W.nzero):
            back[W.zero[k].lin_off:W.zero[k].lin_off + W.zero[k].n] = 0.0
        kinds = set()
        for k in range(W.nseg):
            g = W.seg[k]
            src = wire[1, W.ocp_off + g.wire_off:]
            kinds.add(g.sym)
            if g.sym == 0:
                for j in range(g.cols):
                    back[g.lin_off + j * g.ld:g.lin_off + j * g.ld + g.rows] = src[j * g.rows:(j + 1) * g.rows]
            elif g.sym == 2:
                for q in range(g.rows):
                    back[g.lin_off + q * (g.ld + 1)] = src[q]
            else:
                for j in range(g.rows):
                    for r in range(g.rows):
                        back[g.lin_off + r + j * g.ld] = src[j * (j + 1) // 2 + r] if r <= j else src[r * (r + 1) // 2 + j]
        assert 2 in kinds
        # everything the kernels read of this grid point's record is reproduced exactly
        if c.type == TERMINAL:
            for off, n in ((S.l_Qxx, 36 * 36), (S.l_lx, 36), (S.l_se3 + 36, 36)):
                np.testing.assert_array_equal(back[off:off + n], rec[off:off + n])
        else:
            keep = np.ones(S.l_stride, bool)
            keep[S.l_Phix:S.l_ha] = False
            keep[S.l_ha:S.l_dgdq] = False      # no switching-time stage in this schedule
            keep[S.l_dgdf + 60:] = False
            np.testing.assert_array_equal(back[keep], rec[keep])
