"""The MJtJinv kernel (K1) and the free-flyer part of the update kernel against the extended-precision reference
tests/stage_mp.py (tests/golden/stage_mp_cases.npz), row by row, on ANYmal's own M and J and on SE(3) steps around the
branches of the exponential.

Comparison rule, per kernel, grid point and row r: with e = max over the row of |x - mp| and C(r) the row's scale
(stage_mp.py), the kernel passes iff e_dev(r) <= max(A e_orc(r), B 2^-53 C(r)), e_orc the error of the oracle
(oracle/condense_oracle.c) fed the same fp64 inputs.  A = 4, B = 16: the kernel may be a small factor less accurate than the
fp64 implementation of the same algorithm, entry for entry, or within a few roundings of what its row is made of.

Also: the entries of Z beyond nv + nf are exactly zero, and the condensing (K1 + K2) reads nothing of J beyond the active
contact rows -- NaN there gives the bits of zeros there, in every record rbt_condense writes."""
import ctypes
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_stage_mp as G  # noqa: E402
import stage_mp  # noqa: E402
from synth import make_stage_inputs, symmetrize_lin  # noqa: E402
from test_stage_mp import _oracle_z, oracle_update_q  # noqa: E402

pytestmark = pytest.mark.gpu
A_, B_ = 4.0, 16.0
DIR, LIN, SOL, STEPS = 3, 6, 9, 11   # RBT_BUF_*
TYPES = (0, 2, 1)   # Intermediate, Lift, Impact
DATA = G.load()


def _setup(ctrl, batch):
    from robotoc_b200 import ANYMAL, DirectMultipleShooting, Layout, RiccatiRecursion, StageDims, StageLayout, anymal_constraint_table
    table = anymal_constraint_table()
    sd = StageDims(ANYMAL, nf_max=12, n_contacts=4, n_box=table.n_box)
    rr = RiccatiRecursion(ANYMAL, len(ctrl), batch)
    rr.setTimeDiscretization(ctrl)
    return rr, DirectMultipleShooting(rr, sd, table), sd, StageLayout(sd), Layout(ANYMAL)


def _kkt_schedule():
    """Grid point 3 m + t: mask MASKS[m] on grid-point type TYPES[t]; then Terminal."""
    from robotoc_b200.grid import plain_schedule
    n = len(G.MASKS) * len(TYPES)
    ctrl = plain_schedule(n, 0.02, 0)
    for i in range(n):
        mask = int(G.MASKS[i // len(TYPES)])
        ctrl[i].type, ctrl[i].contact_mask, ctrl[i].nf = TYPES[i % len(TYPES)], mask, G.nf_of(mask)
    return ctrl


def _kkt_lin(sd, S, ctrl, pad):
    """Linearization records with batch entry s holding state s's M and J; `pad` fills J beyond the active contact rows."""
    B = len(G.STATES)
    lin1, con1, _, _ = make_stage_inputs(sd, S, ctrl, 1, 97)
    lin, con = np.repeat(symmetrize_lin(S, lin1), B, 0), np.repeat(con1, B, 0)
    for s in range(B):
        for i in range(len(ctrl) - 1):
            m = i // len(TYPES)
            nf = G.nf_of(int(G.MASKS[m]))
            r = lin[s, i]
            r[S.l_M:S.l_M + 324] = DATA["M"][s].T.reshape(-1)
            J = DATA["J"][s, m].copy()
            J[nf:] = pad
            r[S.l_J:S.l_J + 12 * 18] = J.T.reshape(-1)
    return np.ascontiguousarray(lin), np.ascontiguousarray(con)


def _condense(pad):
    ctrl = _kkt_schedule()
    rr, dms, sd, S, K = _setup(ctrl, len(G.STATES))
    try:
        lin, con = _kkt_lin(sd, S, ctrl, pad)
        dms.condense(lin, con)
        out = {"lin": dms._down(LIN, lin.shape), "ex": dms.getExpansionData(), "kkt": dms.getKKT(),
               "con": dms.getConstraintData()}
        assert int(rr.info().max()) == 0
    finally:
        rr.close()
    return ctrl, S, out


def test_mjtjinv_matches_the_extended_precision_reference():
    ctrl, S, out = _condense(0.0)
    n_all = 30
    worst = {}
    for s, name in enumerate(G.STATES):
        fam = name
        for i in range(len(ctrl) - 1):
            m = i // len(TYPES)
            n = G.NV + G.nf_of(int(G.MASKS[m]))
            Z = out["ex"][s, i, S.e_Z:S.e_Z + n_all * n_all].reshape(n_all, n_all).T
            assert not np.any(Z[n:]) and not np.any(Z[:, n:]), f"{name} grid {i}: Z beyond nv + nf is not zero"
            r = stage_mp.row_errors(Z[:n, :n], DATA["Z"][s, m, :n, :n], DATA["Z_scale"][s, m, :n], _oracle_z(s, m), A_, B_)
            worst[fam] = max(worst.get(fam, 0.0), r.max())
            assert np.all(r <= 1.0), f"{name} grid {i} (mask {G.MASKS[m]:04b}): rows {np.argwhere(~(r <= 1.0)).ravel()} ratio {r.max():.2f}"
    print("K1 worst e_dev / max(A e_orc, B u C): " + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))


def test_condensing_reads_no_inactive_contact_row_of_j():
    """NaN in the rows of J beyond nf (the kernels' contract: only the active contact rows are read) gives, bit for bit, the
    expansion, KKT and PDIPM records of zeros there."""
    _, S, zero = _condense(0.0)
    ctrl, _, nan = _condense(np.nan)
    poisoned = sum(int(np.isnan(nan["lin"][:, i, S.l_J:S.l_J + 216]).sum()) for i in range(len(ctrl) - 1))
    assert poisoned == len(G.STATES) * sum((12 - G.nf_of(int(m))) * 18 * len(TYPES) for m in G.MASKS), "the NaNs did not land"
    for key in ("ex", "kkt", "con"):
        np.testing.assert_array_equal(nan[key].view(np.uint64), zero[key].view(np.uint64), err_msg=key)


class _DeviceView:
    """The handle's buffer `which` as a CUDA array (rbt_dev_ptr), so that torch can write into it in place."""

    def __init__(self, rr, which):
        n = rr.buf_doubles(which)
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f8", "data": (rr.dev_ptr(which), False), "version": 2}


def _write_steps(rr, a):
    """RBT_BUF_STEPS cannot be bound or uploaded: write it in place through rbt_dev_ptr."""
    import torch
    view = torch.as_tensor(_DeviceView(rr, STEPS), device="cuda")
    assert view.numel() == a.size
    torch.cuda.synchronize()
    view.copy_(torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64).reshape(-1)))
    torch.cuda.synchronize()


def test_update_free_flyer_matches_the_extended_precision_reference():
    """OCP b steps by STEPS[b]; grid point g holds configuration g // 10 and turns by ANGLES[g % 10]."""
    import torch
    from robotoc_b200.grid import plain_schedule
    q, dq, steps = DATA["q"], DATA["dq"], DATA["steps"]
    B, Gn = dq.shape[0], dq.shape[1]
    ctrl = plain_schedule(Gn, 0.02, 0)
    rr, dms, sd, S, K = _setup(ctrl, B)
    try:
        lin, con, sol, _ = make_stage_inputs(sd, S, ctrl, B, 98)
        sol[:, :Gn, S.s_q:S.s_q + S.nq] = q[None]
        sol[:, Gn, S.s_q:S.s_q + S.nq] = q[0]
        d = np.zeros((B, Gn + 1, K.d_stride))
        d[:, :Gn, K.d_dx:K.d_dx + S.nv] = dq
        d[:, Gn, K.d_dx:K.d_dx + S.nv] = dq[:, 0]
        dms.condense(symmetrize_lin(S, lin), con)
        dms.setSolution(sol)
        dir_t = torch.from_numpy(d).cuda()   # the direction records, bound as RBT_BUF_DIR (as bench.py binds them)
        rr.bind_buffer(DIR, ctypes.c_void_p(dir_t.data_ptr()))
        torch.cuda.synchronize()
        dms.computeStepSizes()
        _write_steps(rr, np.stack([steps, np.full(B, 0.5)], 1))
        before = {w: dms._down(w, (B, Gn + 1, st)) for w, st in ((SOL, S.s_stride), (DIR, K.d_stride))}
        dms.integrateSolution()
        got = dms._down(SOL, (B, Gn + 1, S.s_stride))
    finally:
        rr.close()
    np.testing.assert_array_equal(before[SOL][:, :Gn, S.s_q:S.s_q + S.nq], np.broadcast_to(q, (B, Gn, S.nq)))
    np.testing.assert_array_equal(before[DIR][:, :Gn, K.d_dx:K.d_dx + S.nv], dq)
    qd = got[:, :Gn, S.s_q:S.s_q + S.nq]
    qo = oracle_update_q(q, dq, steps)
    r = stage_mp.row_errors(qd, DATA["q_new"], DATA["q_scale"], qo, A_, B_)
    worst = {}
    for k, th in enumerate(G.ANGLES):
        worst[f"{th:.17g}"] = r[:, k::len(G.ANGLES)].max()
    print("update worst e_dev / max(A e_orc, B u C) per angle: " + ", ".join(f"{k}: {v:.3f}" for k, v in worst.items()))
    bad = np.argwhere(~(r <= 1.0))
    assert bad.size == 0, f"(OCP, grid point, q row) {bad[:8].tolist()}: ratio {r.max():.2f}"
    assert np.all(np.isfinite(got[:, :, S.s_q:S.s_q + S.nq]))
    np.testing.assert_array_equal(got[:, Gn, S.s_q:S.s_q + S.nq], qd[:, 0])  # the Terminal grid point runs the same code
