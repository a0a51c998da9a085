"""The extended-precision stage-layer reference tests/stage_mp.py and its cases tests/golden/stage_mp_cases.npz (CPU):
identities of the reference at 1e-40, the oracle (oracle/condense_oracle.c) held to the npz row by row, and the npz
recomputed live.  The kernels are held to the same npz by tests/test_gpu_stage_mp.py."""
import ctypes
import os
import sys

import numpy as np
import pytest
from mpmath import mp

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_stage_mp as G  # noqa: E402
import oracle_lib  # noqa: E402
import stage_mp  # noqa: E402

DATA = G.load()


def test_case_file_holds_the_current_inputs():
    M, J = G.kkt_inputs()
    q, dq = G.se3_inputs()
    assert G.inputs_sha256(M, J, q, dq) == str(DATA["sha256"]), "the input builders changed: rerun make_stage_mp.py"
    assert G.inputs_sha256(DATA["M"], DATA["J"], DATA["q"], DATA["dq"]) == str(DATA["sha256"])
    assert os.path.getsize(G.PATH) < 1 << 20


def test_case_file_covers_the_edges():
    assert sorted({G.nf_of(m) for m in DATA["masks"]}) == [0, 3, 6, 9, 12]
    assert 0b0101 in DATA["masks"]                                      # feet 0 and 2: not contiguous
    assert DATA["cond"].max() > 1e6                                     # an ill-conditioned J M^-1 J^T
    th = np.linalg.norm(DATA["steps"][:, None, None] * DATA["dq"][:, :, 3:6], axis=-1)
    for k in (2, 3, 4):                                                 # the kernels' own th, on the fp64 neighbours of 1e-6
        for b, step in enumerate(DATA["steps"]):
            g = k + np.arange(len(G.CONFIGS)) * len(G.ANGLES)
            w = step * DATA["dq"][b, g, 5]
            assert np.all(np.sqrt(w * w) == G.ANGLES[k])
    assert np.allclose(th[:, :len(G.ANGLES)], G.ANGLES[None], rtol=1e-14, atol=0)
    assert DATA["q"][:, 6].min() < 0 and np.abs(DATA["q"][:, 6]).min() < 1e-8 and np.linalg.norm(DATA["q"][:, :3], axis=1).max() >= 1e3


@pytest.mark.parametrize("s,m", [(4, 5), (1, 2)])
def test_reference_inverse_is_exact(s, m):
    nf = G.nf_of(int(DATA["masks"][m]))
    M, J = DATA["M"][s], DATA["J"][s, m, :nf]
    with mp.workdps(stage_mp.DPS):
        A = stage_mp.kkt(M, J)
        Z = mp.inverse(A)
        E = Z * A - mp.eye(A.rows)
        assert max(abs(x) for x in E) < mp.mpf(10) ** -40


def test_reference_quaternion_is_the_expm_rotation():
    """The quaternion of the reference is a unit quaternion whose rotation is R(q) expm([w]x), for every angle (incl. th > pi)."""
    for b in (0, 3):
        for g in range(DATA["q"].shape[0]):
            q, dq, step = DATA["q"][g], DATA["dq"][b, g], DATA["steps"][b]
            with mp.workdps(stage_mp.DPS):
                _, n, Re, _, _, _, _, _, _ = stage_mp._integrate(q, dq, step)
                qq = [mp.mpf(float(x)) for x in q[3:7]]
                nq = mp.sqrt(sum(x * x for x in qq))
                R0 = stage_mp.quat_rot([x / nq for x in qq])
                assert abs(sum(x * x for x in n) - 1) < mp.mpf(10) ** -40
                D = stage_mp.quat_rot(n) - R0 * Re
                assert max(abs(x) for x in D) < mp.mpf(10) ** -40


def test_npz_is_what_the_reference_computes():
    """Two cases recomputed live, bit for bit: the stretched knee on all four feet, and the update at step 0.75^8."""
    z, sc = G.kkt_case(DATA["M"], DATA["J"], 4, 5)
    np.testing.assert_array_equal(z, DATA["Z"][4, 5])
    np.testing.assert_array_equal(sc, DATA["Z_scale"][4, 5])
    for g in range(DATA["q"].shape[0]):
        qn, qs = stage_mp.integrate_free_flyer(DATA["q"][g], DATA["dq"][2, g], DATA["steps"][2])
        np.testing.assert_array_equal(qn, DATA["q_new"][2, g])
        np.testing.assert_array_equal(qs, DATA["q_scale"][2, g])


def _oracle_z(s, m):
    nf = G.nf_of(int(DATA["masks"][m]))
    n = G.NV + nf
    Zt = np.zeros((n, n))                                  # column-major: Zt[j, i] = Z[i, j]
    Jt = np.ascontiguousarray(DATA["J"][s, m, :max(nf, 1)].T)
    Mt = np.ascontiguousarray(DATA["M"][s].T)
    assert oracle_lib.load().orc_mjtjinv(G.NV, nf, oracle_lib.ptr(Mt), oracle_lib.ptr(Jt), Jt.shape[1], oracle_lib.ptr(Zt),
                                         n) == 0
    return Zt.T


def test_oracle_mjtjinv_against_the_reference():
    """The oracle (Cholesky of M and of J M^-1 J^T, as Robot::computeMJtJinv) against the exact inverse, row by row.  It is
    the witness e_orc of the kernel's comparison, so a loss of accuracy in the witness itself must show.  Where J M^-1 J^T is
    well conditioned it is held to 32 u of each row's |Z||A||Z| (measured: 16.8 u, trot with all four feet).  The
    Cholesky-plus-Schur-complement route is not componentwise stable: its error grows with the condition number of
    J M^-1 J^T, which the row scale |Z||A||Z| does not see.  So on the heavy-base, straight-knee case (condition number
    1e7) it is held to u C cond(J M^-1 J^T) instead (measured: 1.0e4 u C)."""
    worst = {}
    for s, name in enumerate(G.STATES):
        for m, mask in enumerate(DATA["masks"]):
            n = G.NV + G.nf_of(int(mask))
            r = stage_mp.row_errors(_oracle_z(s, m), DATA["Z"][s, m, :n, :n], DATA["Z_scale"][s, m, :n], b=1.0)
            bound = 32.0 if DATA["cond"][s, m] < 1e3 else DATA["cond"][s, m]
            assert np.all(r <= bound), f"{name} mask {mask:04b}: e / (u C) = {r.max():.3g}"
            worst[name] = max(worst.get(name, 0.0), r.max())
    print("oracle MJtJinv: worst e / (u C): " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))


def oracle_update_q(q, dq, steps):
    """orc_update_batch on Terminal-free records that hold only q and dx: the configuration it returns per (OCP, grid point)."""
    from robotoc_b200 import ANYMAL, Layout, StageDims, StageLayout, anymal_constraint_table
    from robotoc_b200.grid import plain_schedule
    lib = oracle_lib.load()
    table = anymal_constraint_table()
    sd = StageDims(ANYMAL, nf_max=12, n_contacts=4, n_box=table.n_box)
    S, K = StageLayout(sd), Layout(ANYMAL)
    B, Gn = dq.shape[0], dq.shape[1]
    ctrl = plain_schedule(Gn, 0.02, 0)
    ex, d = np.zeros((B, Gn + 1, S.e_stride)), np.zeros((B, Gn + 1, K.d_stride))
    xd, con, sol = np.zeros((B, Gn + 1, S.x_stride)), np.zeros((B, Gn + 1, S.c_stride)), np.zeros((B, Gn + 1, S.s_stride))
    sol[:, :Gn, S.s_q:S.s_q + S.nq] = q[None]
    sol[:, Gn, S.s_q:S.s_q + S.nq] = q[0]
    d[:, :Gn, K.d_dx:K.d_dx + S.nv] = dq
    st = np.stack([steps, np.ones_like(steps)], 1)
    lib.orc_update_batch(ctypes.byref(sd.c()), ctypes.byref(table), ctrl, Gn + 1, B, oracle_lib.ptr(ex), oracle_lib.ptr(d),
                         oracle_lib.ptr(xd), oracle_lib.ptr(con), oracle_lib.ptr(sol), oracle_lib.ptr(st), 0)
    return sol[:, :Gn, S.s_q:S.s_q + S.nq]


def test_oracle_update_against_the_reference():
    """The oracle's SE(3) exponential within 16 u of each configuration row's scale at every angle and step size."""
    got = oracle_update_q(DATA["q"], DATA["dq"], DATA["steps"])
    r = stage_mp.row_errors(got, DATA["q_new"], DATA["q_scale"], b=1.0)
    print(f"oracle update: worst e / (u C) = {r.max():.2f}")
    assert r.max() <= 16.0, np.argwhere(r > 16.0)
