"""Time-parallel (segmented) Riccati sweeps.

CPU part: a numpy restatement of the algebra the CUDA path uses -- the per-stage conditional value-function elements
(A, b, C, eta, J) of Saerkkae & Garcia-Fernandez, "Temporal parallelization of dynamic programming and linear quadratic
control" (IEEE TAC 68(2), 2023), in robotoc's convention V(dx) = 1/2 dx^T P dx - s^T dx, their associative combine, the
segmented backward sweep and the composed closed-loop maps of the forward sweep -- pinned against the oracle's P, s, dx and
a dense KKT solve.  GPU part: the device path with forced and automatic segment counts against the oracle and against the
serial device path."""
import ctypes
import copy

import numpy as np
import pytest

import oracle_lib
from helpers import (contact_mask_walk_schedule, crawl_schedule, dense_kkt_solve, jump_sto_schedule, rel_err,
                     small_event_schedule, trot_schedule)
from robotoc_b200 import ANYMAL, Layout
from robotoc_b200.grid import IMPACT, TERMINAL
from synth import make_kkt, mat


def _no_sto(ctrl):
    out = copy.deepcopy(ctrl)
    for c in out:
        c.sto = 0
        c.sto_next = 0
    return out


SCHEDULES = {
    "small_event": lambda: small_event_schedule(sto=False)[2],
    "trot": lambda: trot_schedule(40)[2],
    "crawl": lambda: crawl_schedule(54)[2],
    "mask_walk": lambda: contact_mask_walk_schedule()[2],
    "jump_no_sto": lambda: _no_sto(jump_sto_schedule(80)[2]),
}


# ---------------------------------------------------------------------------------------------------- numpy prototype
def element(dims, L, c, rec):
    """(A, b, C, eta, J) of one grid point: V_i(dx) = min over du of stage cost + V_{i+1}(A dx + B du + Fx), as a function
    of the value function after it."""
    nx, nu, nv = dims.nx, dims.nu, dims.nv
    Qxx = mat(rec, L.k_Qxx, nx, nx)
    lx = rec[L.k_lx:L.k_lx + nx]
    Z = np.zeros((nx, nx))
    if c.type == TERMINAL:
        return Z, np.zeros(nx), Z.copy(), -lx, Qxx
    A = mat(rec, L.k_Fxx, nx, nx)
    Fx = rec[L.k_Fx:L.k_Fx + nx]
    if c.type == IMPACT:
        return A, Fx, Z, -lx, Qxx
    B = np.zeros((nx, nu))
    B[nv:] = mat(rec, L.k_Fvu, nv, nu)
    S = mat(rec, L.k_Qxu, nx, nu)
    R = mat(rec, L.k_Quu, nu, nu)
    lu = rec[L.k_lu:L.k_lu + nu]
    Ri = np.linalg.inv(np.linalg.cholesky(R))
    Ri = Ri.T @ Ri
    X, x = Ri @ S.T, Ri @ lu
    J, eta = Qxx - S @ X, -(lx - S @ x)
    Rt = Ri
    ns = c.ns
    if ns > 0:
        Phx, Phu, p = mat(rec, L.k_Phix, ns, nx), mat(rec, L.k_Phiu, ns, nu), rec[L.k_p:L.k_p + ns]
        Y = Ri @ Phu.T
        W = Phu @ Y
        D, e = Phx - Phu @ X, p - Phu @ x
        Wi = np.linalg.inv(W)
        J, eta = J + D.T @ Wi @ D, eta - D.T @ Wi @ e
        X, x = X + Y @ Wi @ D, x + Y @ Wi @ e
        Rt = Ri - Y @ Wi @ Y.T
    return A - B @ X, Fx - B @ x, B @ Rt @ B.T, eta, J


def combine(ei, ej):
    """Element i followed by element j."""
    Ai, bi, Ci, ei_, Ji = ei
    Aj, bj, Cj, ej_, Jj = ej
    I = np.eye(Ai.shape[0])
    Minv = np.linalg.inv(I + Ci @ Jj)
    T1 = Minv @ Ai
    return (Aj @ T1, Aj @ Minv @ (bi + Ci @ ej_) + bj, Aj @ Minv @ Ci @ Aj.T + Cj, T1.T @ (ej_ - Jj @ bi) + ei_,
            T1.T @ Jj @ Ai + Ji)


def seg_bounds(N, S):
    return [(j * N) // S for j in range(S + 1)]


def segmented_backward(dims, L, ctrl, rec1, S):
    """(P, s) at every grid point: segment aggregates combined from the terminal give the value at every segment end; each
    segment then walks its stages from that seed."""
    N = len(ctrl) - 1
    E = [element(dims, L, c, rec1[i]) for i, c in enumerate(ctrl)]
    bnd = seg_bounds(N, S)
    agg = []
    for j in range(S):
        a = E[bnd[j]]
        for i in range(bnd[j] + 1, bnd[j + 1]):
            a = combine(a, E[i])
        agg.append(a)
    seeds = [None] * S
    v = E[N]
    for j in range(S - 1, -1, -1):
        seeds[j] = v
        v = combine(agg[j], v)
    P, s = [None] * (N + 1), [None] * (N + 1)
    P[N], s[N] = E[N][4], E[N][3]
    for j in range(S):
        v = seeds[j]
        P[bnd[j + 1]], s[bnd[j + 1]] = v[4], v[3]
        for i in range(bnd[j + 1] - 1, bnd[j] - 1, -1):
            v = combine(E[i], v)
            P[i], s[i] = v[4], v[3]
    return P, s


def segmented_forward(dims, L, ctrl, rec1, ric1, dx0, S):
    """dx at every grid point from the closed-loop maps dx+ = T dx + t, composed per segment and applied from dx0."""
    nx, nu, nv = dims.nx, dims.nu, dims.nv
    N = len(ctrl) - 1
    maps = []
    for i in range(N):
        A, Fx = mat(rec1[i], L.k_Fxx, nx, nx), rec1[i][L.k_Fx:L.k_Fx + nx]
        if ctrl[i].type == IMPACT:
            maps.append((A, Fx))
            continue
        B = np.zeros((nx, nu))
        B[nv:] = mat(rec1[i], L.k_Fvu, nv, nu)
        K = ric1[i][L.r_K:L.r_K + nu * nx].reshape(nu, nx)
        k = ric1[i][L.r_k:L.r_k + nu]
        maps.append((A + B @ K, B @ k + Fx))
    bnd = seg_bounds(N, S)
    starts = [dx0]
    for j in range(S - 1):
        T, t = np.eye(nx), np.zeros(nx)
        for i in range(bnd[j], bnd[j + 1]):
            T, t = maps[i][0] @ T, maps[i][0] @ t + maps[i][1]
        starts.append(T @ starts[-1] + t)
    dx = [None] * (N + 1)
    for j in range(S):
        x = starts[j]
        last = N if j == S - 1 else bnd[j + 1] - 1
        for i in range(bnd[j], last + 1):
            dx[i] = x
            if i < N:
                x = maps[i][0] @ x + maps[i][1]
    return dx


@pytest.mark.parametrize("which", sorted(SCHEDULES))
def test_prototype_against_oracle(which):
    ctrl = SCHEDULES[which]()
    assert not any(c.sto or c.sto_next for c in ctrl)
    dims, L = ANYMAL, Layout(ANYMAL)
    nx = dims.nx
    N = len(ctrl) - 1
    kkt, dx0 = make_kkt(dims, L, ctrl, batch=1, seed=20261015)
    _, ric_o, d_o, info = oracle_lib.riccati_batch(dims, L, ctrl, kkt, dx0)
    assert info == 0
    ref = dense_kkt_solve(dims, L, ctrl, kkt[0], dx0[0])
    for S in sorted({2, 3, 7, N}):
        P, s = segmented_backward(dims, L, ctrl, kkt[0], S)
        for i in range(N + 1):
            assert rel_err(P[i], mat(ric_o[0, i], L.r_P, nx, nx)) < 1e-9, f"S={S} grid {i} P"
            assert rel_err(s[i], ric_o[0, i, L.r_s:L.r_s + nx]) < 1e-9, f"S={S} grid {i} s"
        dx = segmented_forward(dims, L, ctrl, kkt[0], ric_o[0], dx0[0], S)
        for i in range(N + 1):
            assert rel_err(dx[i], d_o[0, i, L.d_dx:L.d_dx + nx]) < 1e-9, f"S={S} grid {i} dx"
            assert rel_err(dx[i], ref[("dx", i)]) < 1e-7, f"S={S} grid {i} dx (dense KKT)"
            # costate: lmd = P dx - s
            assert rel_err(P[i] @ dx[i] - s[i], ref[("lmd", i)]) < 1e-7, f"S={S} grid {i} lmd (dense KKT)"


def test_combine_is_associative():
    ctrl = SCHEDULES["small_event"]()
    dims, L = ANYMAL, Layout(ANYMAL)
    kkt, _ = make_kkt(dims, L, ctrl, batch=1, seed=7)
    E = [element(dims, L, c, kkt[0, i]) for i, c in enumerate(ctrl)]
    left = combine(combine(E[1], E[2]), E[3])
    right = combine(E[1], combine(E[2], E[3]))
    for a, b in zip(left, right):
        assert rel_err(a, b) < 1e-11


# ---------------------------------------------------------------------------------------------------------- C ABI, no GPU
RBT_ERR_ARG = 1  # include/robotoc_b200.h


def test_set_time_segments_rejects_bad_arguments_without_a_device():
    from robotoc_b200 import _lib
    L = _lib.lib()
    assert "rbt_set_time_segments" in _lib.EXPORTS
    for k in (-1, 0, 1, 2):
        assert L.rbt_set_time_segments(None, k) == RBT_ERR_ARG


# ---------------------------------------------------------------------------------------------------------- device path
BATCHES = (1, 3, 17)


def _solve(rr, kkt, dx0, segments, write_fact=True):
    rr.setTimeSegments(segments)
    rr.backwardRiccatiRecursion(kkt, write_fact=write_fact)
    rr.forwardRiccatiRecursion(dx0)
    return rr.getRiccatiFactorization(), rr.getDirection(), rr.getFactorizedKKT(), rr.info()


@pytest.mark.gpu
@pytest.mark.parametrize("batch", BATCHES)
@pytest.mark.parametrize("which", sorted(SCHEDULES))
def test_segmented_parity(which, batch):
    """Every block of RIC, FACT and DIR against the oracle, at 2, 3, 7, n_grid - 1 segments and the automatic choice."""
    from robotoc_b200 import RiccatiRecursion
    from test_gpu_parity import _compare
    ctrl = SCHEDULES[which]()
    dims, L = ANYMAL, Layout(ANYMAL)
    N = len(ctrl) - 1
    kkt, dx0 = make_kkt(dims, L, ctrl, batch=batch, seed=20261016 + batch)
    kk, ric_o, d_o, info = oracle_lib.riccati_batch(dims, L, ctrl, kkt, dx0)
    assert info == 0
    rr = RiccatiRecursion(dims, len(ctrl), batch)
    rr.setTimeDiscretization(ctrl)
    ser = _solve(rr, kkt, dx0, 1)
    worst_ser = 0.0
    for S in (2, 3, 7, N, 0):
        ric, d, f, inf = _solve(rr, kkt, dx0, S)
        assert int(inf.max()) == 0
        w = _compare(dims, L, ctrl, ric, ric_o, d, d_o, f, kk)
        worst_ser = max(worst_ser, rel_err(ric, ser[0]), rel_err(d, ser[1]), rel_err(f, ser[2]))
        print(f"{which} batch {batch} S={S}: worst rel err vs oracle {w:.2e}")
        ric2, d2 = rr.solve_host(kkt, dx0)
        assert np.array_equal(ric2, ric) and np.array_equal(d2, d)
    print(f"{which} batch {batch}: worst rel err vs the serial device path {worst_ser:.2e}")
    rr.close()


@pytest.mark.gpu
def test_batch1024_auto_is_serial_bits():
    from robotoc_b200 import RiccatiRecursion
    ctrl = trot_schedule(40)[2]
    dims, L = ANYMAL, Layout(ANYMAL)
    kkt, dx0 = make_kkt(dims, L, ctrl, batch=1024, seed=20261017)
    rr = RiccatiRecursion(dims, len(ctrl), 1024)
    rr.setTimeDiscretization(ctrl)
    a = _solve(rr, kkt, dx0, 0)
    s = _solve(rr, kkt, dx0, 1)
    for x, y in zip(a, s):
        np.testing.assert_array_equal(x, y)
    rr.close()


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["small_event_sto", "jump_sto"])
def test_sto_schedules_stay_serial(which):
    from robotoc_b200 import RiccatiRecursion
    ctrl = {"small_event_sto": lambda: small_event_schedule(sto=True)[2], "jump_sto": lambda: jump_sto_schedule(80)[2]}[which]()
    dims, L = ANYMAL, Layout(ANYMAL)
    kkt, dx0 = make_kkt(dims, L, ctrl, batch=3, seed=20261018)
    for batch in (3,):
        rr = RiccatiRecursion(dims, len(ctrl), batch)
        rr.setTimeDiscretization(ctrl)
        a = _solve(rr, kkt, dx0, 0)
        s = _solve(rr, kkt, dx0, 1)
        for x, y in zip(a, s):
            np.testing.assert_array_equal(x, y)
        with pytest.raises(ValueError):
            rr.setTimeSegments(2)
        with pytest.raises(ValueError):
            rr.setTimeSegments(-1)
        rr.close()


@pytest.mark.gpu
def test_set_time_segments_bounds():
    from robotoc_b200 import RiccatiRecursion
    ctrl = trot_schedule(40)[2]
    rr = RiccatiRecursion(ANYMAL, len(ctrl), 1)
    with pytest.raises(ValueError):  # no schedule yet
        rr.setTimeSegments(2)
    rr.setTimeDiscretization(ctrl)
    rr.setTimeSegments(len(ctrl) - 1)
    with pytest.raises(ValueError):
        rr.setTimeSegments(len(ctrl))
    rr.close()


@pytest.mark.gpu
def test_element_factorisation_fallback():
    """OCP 1 has an indefinite Quu at one stage but a positive definite Quu + B^T P B: the elements cannot be built, so its
    segments fall back to one serial sweep with the serial path's bits.  OCP 3 has a G that is not positive definite either:
    rbt_check_info reports flag 1 for it, as on the serial path.  The other OCPs match the oracle."""
    from robotoc_b200 import RiccatiRecursion
    from test_gpu_parity import _compare
    ctrl = trot_schedule(40)[2]
    dims, L = ANYMAL, Layout(ANYMAL)
    nu = dims.nu
    kkt, dx0 = make_kkt(dims, L, ctrl, batch=5, seed=20261019)
    rr = RiccatiRecursion(dims, len(ctrl), 5)
    rr.setTimeDiscretization(ctrl)
    f0 = _solve(rr, kkt, dx0, 1)[2]
    i = next(i for i in range(len(ctrl) // 2, len(ctrl)) if ctrl[i].type == 0 and ctrl[i].ns == 0)
    bad = kkt.copy()
    for ob, between in ((1, True), (3, False)):
        Quu = mat(kkt[ob, i], L.k_Quu, nu, nu)
        G = mat(f0[ob, i], L.f_G, nu, nu)
        lq, lg = np.linalg.eigvalsh(Quu)[0], np.linalg.eigvalsh(G)[0]
        assert lg > lq + 1e-6
        t = 0.5 * (lq + lg) if between else lg + 1.0
        bad[ob, i, L.k_Quu:L.k_Quu + nu * nu] = (Quu - t * np.eye(nu)).T.reshape(-1)
    ser = _solve(rr, bad, dx0, 1)
    assert list(np.nonzero(ser[3])[0]) == [3] and ser[3][3] & 1
    seg = _solve(rr, bad, dx0, 4)
    np.testing.assert_array_equal(seg[3], ser[3])
    for ob in (1, 3):
        for x, y in zip(seg[:3], ser[:3]):
            np.testing.assert_array_equal(x[ob], y[ob])
    first = ctypes.c_int(-1)
    assert rr._lib.rbt_check_info(rr._h, ctypes.byref(first), None) != 0 and first.value == 3
    keep = [0, 1, 2, 4]
    kk, ric_o, d_o, info = oracle_lib.riccati_batch(dims, L, ctrl, np.ascontiguousarray(bad[keep]), np.ascontiguousarray(dx0[keep]))
    assert info == 0
    w = _compare(dims, L, ctrl, seg[0][keep], ric_o, seg[1][keep], d_o, seg[2][keep], kk)
    print("worst rel err vs oracle (fallback batch)", w)
    rr.close()


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["trot", "crawl"])
def test_full_iteration_batch1(which):
    """condense -> backward -> forward -> expand -> update at batch 1 with the automatic choice and with forced segments, on
    the step-by-step path and through iteration_host_resident."""
    from iteration_check import compare_final, oracle_iteration, run_device_iteration
    from robotoc_b200 import DirectMultipleShooting, RiccatiRecursion, StageDims, StageLayout, anymal_constraint_table
    from synth import make_stage_inputs, symmetrize_lin
    ctrl = {"trot": lambda: trot_schedule(40)[2], "crawl": lambda: crawl_schedule(54)[2]}[which]()
    table = anymal_constraint_table()
    sd = StageDims(ANYMAL, nf_max=12, n_contacts=table.n_contacts, n_box=table.n_box)
    S, K = StageLayout(sd), Layout(ANYMAL)
    lin, con, sol, dx0 = make_stage_inputs(sd, S, ctrl, 1, 20261020)
    lin = symmetrize_lin(S, lin)
    ref = oracle_iteration(sd, S, K, table, ctrl, lin, con, sol, dx0)
    used = S.s_xi + S.nsm
    for segs in (0, 4):
        rr = RiccatiRecursion(ANYMAL, len(ctrl), 1)
        rr.setTimeDiscretization(ctrl)
        rr.setTimeSegments(segs)
        dms = DirectMultipleShooting(rr, sd, table)
        got = run_device_iteration(rr, dms, lin, con, sol, dx0)
        assert int(got["info"].max()) == 0
        w = compare_final(S, K, ctrl, ref, got["ric"], got["d"], got["steps"], got["sol"], got["cc"], 1e-8)
        print(f"{which} segments={segs}: worst rel err {w:.2e}")
        dms.setSolution(sol)
        dms.setConstraintData(con)
        res = np.ascontiguousarray(con[:, :, S.c_res:S.c_res + S.ncp])
        sol5, sd5, steps5 = dms.iteration_host_resident(dms.pack_wire(lin), lin, res, dx0)
        assert rel_err(sol5[:, :, :used], got["sol"][:, :, :used]) < 1e-12
        assert rel_err(steps5, got["steps"]) < 1e-12
        rr.close()
