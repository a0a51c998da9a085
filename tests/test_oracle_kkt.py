"""Pins the CPU oracle (oracle/riccati_oracle.c) independently of the Riccati algebra:
the Newton direction it returns must solve the full block-tridiagonal KKT system (numpy dense solve).
This covers Intermediate, Lift, Impact stages and the switching-constraint (Schur) path."""
import numpy as np
import pytest

import oracle_lib
from helpers import crawl_schedule, dense_kkt_solve, dense_kkt_solve_sto, small_event_schedule, rel_err
from robotoc_b200 import ANYMAL, Layout
from robotoc_b200.grid import IMPACT, LIFT
from synth import make_kkt


def _direction_solves_full_kkt(ctrl, batch, seed):
    dims = ANYMAL
    L = Layout(dims)
    types = [c.type for c in ctrl]
    assert IMPACT in types and LIFT in types and any(c.ns > 0 for c in ctrl)
    kkt, dx0 = make_kkt(dims, L, ctrl, batch=batch, seed=seed)
    kk, ric, d, info = oracle_lib.riccati_batch(dims, L, ctrl, kkt, dx0)
    assert info == 0
    for b in range(batch):
        ref = dense_kkt_solve(dims, L, ctrl, kkt[b], dx0[b])
        for i in range(len(ctrl)):
            di = d[b, i]
            assert rel_err(di[L.d_dx:L.d_dx + dims.nx], ref[("dx", i)]) < 1e-9
            assert rel_err(di[L.d_dlmdgmm:L.d_dlmdgmm + dims.nx], ref[("lmd", i)]) < 1e-8
            if ("du", i) in ref:
                assert rel_err(di[L.d_du:L.d_du + dims.nu], ref[("du", i)]) < 1e-9
            if ("xi", i) in ref:
                ns = ctrl[i].ns
                assert rel_err(di[L.d_dxi:L.d_dxi + ns], ref[("xi", i)]) < 1e-8


@pytest.mark.parametrize("seed", [20260924, 7])
def test_oracle_direction_solves_full_kkt(seed):
    td, ev, ctrl = small_event_schedule(sto=False)
    _direction_solves_full_kkt(ctrl, 2, seed)


def test_oracle_direction_solves_full_kkt_crawl():
    """The crawl schedule (the Riccati case of golden_ref_gaits.npz): three-dimensional switching constraints (ns = 3) two grid
    points before each single-foot impact, and impacts at which another foot lifts."""
    td, ev, ctrl = crawl_schedule(54)
    assert {c.ns for c in ctrl} == {0, 3}
    _direction_solves_full_kkt(ctrl, 1, 35)


def test_oracle_riccati_symmetry_and_mutation():
    """reference identities: P symmetric (backward_..factorizer.cpp:85); K = -G^-1 H^T on plain stages
    (riccati_factorizer.cpp:55); the mutated Qxx equals F - K^T G K (test/riccati/riccati_factorizer_test.cpp:36-71)."""
    dims = ANYMAL
    L = Layout(dims)
    td, ev, ctrl = small_event_schedule(sto=False)
    kkt, dx0 = make_kkt(dims, L, ctrl, batch=1, seed=3)
    kk, ric, d, info = oracle_lib.riccati_batch(dims, L, ctrl, kkt, dx0)
    nx, nu = dims.nx, dims.nu
    from synth import mat
    for i in range(len(ctrl) - 1):
        P = mat(ric[0, i], L.r_P, nx, nx)
        assert np.allclose(P, P.T, rtol=0, atol=1e-12 * np.abs(P).max())
        if ctrl[i].type != IMPACT and ctrl[i].ns == 0:
            G = mat(kk[0, i], L.k_Quu, nu, nu)
            H = mat(kk[0, i], L.k_Qxu, nx, nu)
            Kt = mat(ric[0, i], L.r_K, nx, nu)
            assert rel_err(Kt.T, -np.linalg.solve(G, H.T)) < 1e-10


@pytest.mark.parametrize("with_phit", [False, True])
def test_oracle_sto_direction_solves_full_kkt_single_impact(with_phit):
    """Switching-time optimisation, pinned independently of the Riccati algebra where the reference's recursion IS an exact
    elimination: one STO-enabled impact event (phase transition without elimination of a later switching time).  Checks
    dx, du, the costate, the switching-constraint multiplier and the switching-time increment itself.
    with_phit: the switching constraint depends on the switching time (Phit != 0).  There the reference counts
    Phit^T mt_next twice in chi (riccati_factorizer.cpp:139 on top of T.phi_u, backward_..._factorizer.cpp:118); the oracle
    restates that, and its step then differs from the KKT solution at the 1e-5 level -- asserted -- while with the second
    count left out (orc_debug_exact_chi, tests only) it IS the KKT solution to 1e-9, which pins every other Phit term.
    (Phase transitions that eliminate a later switching time: next test.)"""
    import ctypes
    from schedule_fixture import ContactEvents, TimeDiscretization, stage_ctrl_array
    dims = ANYMAL
    L = Layout(dims)
    ev = ContactEvents(phase_dimf=[6], phase_mask=[0b1001])
    ev.push_back(True, 0.23, 12, impact_dimf=6, sto=True, post_mask=0b1111, impact_mask=0b0110)
    td = TimeDiscretization(0.4, 8).discretize(ev, 0.0, sto=True)
    ctrl = stage_ctrl_array(td, ev)
    assert any(c.type == IMPACT for c in ctrl) and all(c.sto for c in ctrl[:-1])
    for seed in (5, 11):
        kkt, dx0 = make_kkt(dims, L, ctrl, batch=1, seed=seed)
        kkt[:, :, L.k_sc + 0] *= 50.0   # convex in the switching time: the unregularised branch of the phase transition
        kkt[:, :, L.k_sc + 1] *= 50.0
        if not with_phit:
            kkt[:, :, L.k_Phit:L.k_Phit + dims.ns_max] = 0.0
        ref, phase, n_events = dense_kkt_solve_sto(dims, L, ctrl, kkt[0], dx0[0])
        flag = ctypes.c_int.in_dll(oracle_lib.load(), "orc_debug_exact_chi")
        if with_phit:  # the restated reference formula: close to, but not, the KKT solution
            kk, ric, d, info = oracle_lib.riccati_batch(dims, L, ctrl, kkt, dx0, max_dts0=1e9)
            dev = max(rel_err(d[0, i, L.d_dx:L.d_dx + dims.nx], ref[("dx", i)]) for i in range(len(ctrl)))
            assert 1e-8 < dev < 1e-3
            flag.value = 1
        try:
            kk, ric, d, info = oracle_lib.riccati_batch(dims, L, ctrl, kkt, dx0, max_dts0=1e9)
        finally:
            flag.value = 0
        assert info == 0
        assert n_events == 1
        ts = float(ref[("ts", 1)][0])
        assert abs(ts) > 1e-3
        for i in range(len(ctrl)):
            di = d[0, i]
            assert rel_err(di[L.d_dx:L.d_dx + dims.nx], ref[("dx", i)]) < 1e-9
            if ctrl[i].type != IMPACT:
                # (at the impact grid itself the reference evaluates the costate with dts_next = 0,
                #  riccati_recursion.cpp:96-107 + riccati_factorizer.cpp:248-256, i.e. without the -Phi*ts term of the KKT)
                assert rel_err(di[L.d_dlmdgmm:L.d_dlmdgmm + dims.nx], ref[("lmd", i)]) < 1e-8
            if ("du", i) in ref:
                assert rel_err(di[L.d_du:L.d_du + dims.nu], ref[("du", i)]) < 1e-9
            if ("xi", i) in ref:
                assert rel_err(di[L.d_dxi:L.d_dxi + ctrl[i].ns], ref[("xi", i)]) < 1e-7
            if i < len(ctrl) - 1:  # phase 0: (dts, dts_next) = (0, ts) ; phase 1 (from the impact on): (ts, 0)
                want = (0.0, ts) if phase[i] == 0 and ctrl[i].type != IMPACT else (ts, 0.0)
                assert abs(di[L.d_dts] - want[0]) < 1e-9 * max(1.0, abs(ts)) and abs(di[L.d_dts + 1] - want[1]) < 1e-9 * max(1.0, abs(ts))


@pytest.mark.parametrize("seed", [5, 7])
def test_oracle_sto_lift_impact_is_exact_kkt_up_to_three_documented_terms(seed):
    """Lift -> impact with both events STO-enabled, a switching-constraint stage and Phit != 0: the phase transition at the
    lift ELIMINATES the impact's switching time.  The reference's recursion differs from the exact Newton step of the LQ
    sub-problem in exactly three places -- it keeps riccati_m.P = riccati.P where minimising over the switching time gives
    P - (Psi-Phi)(Psi-Phi)^T/sgm (riccati_factorizer.cpp:149), it counts Phit^T mt_next twice in chi (:139), and at an impact
    grid it multiplies Phi by dts_next instead of the event's own dts in the costate (:262-264) -- and the oracle restates
    all three.  With these put right (orc_debug_exact_* switches, tests only) the oracle's direction, costate included,
    both switching-time increments included, IS the dense KKT solution to 1e-9: every other STO term (stage terms,
    Hamiltonian factorisation, T / W / mt / mt_next, phase transition, STO policy, forward dts propagation, Lagrange
    multipliers) is thereby pinned independently of the Riccati algebra.  As restated (default) the step is within 5e-2."""
    import ctypes
    dims = ANYMAL
    L = Layout(dims)
    td, ev, ctrl = small_event_schedule(sto=True)
    assert [c.type for c in ctrl].count(LIFT) == 1 and [c.type for c in ctrl].count(IMPACT) == 1
    kkt, dx0 = make_kkt(dims, L, ctrl, batch=1, seed=seed)
    kkt[:, :, L.k_sc + 0] *= 50.0   # convex in the switching times: the unregularised branch of the phase transitions
    kkt[:, :, L.k_sc + 1] *= 50.0
    ref, phase, n_events = dense_kkt_solve_sto(dims, L, ctrl, kkt[0], dx0[0])
    assert n_events == 2
    ts = [float(ref[("ts", k)][0]) for k in (1, 2)]
    lib = oracle_lib.load()
    kk, ric, d, info = oracle_lib.riccati_batch(dims, L, ctrl, kkt, dx0, max_dts0=1e9)  # as the reference
    dev = max(rel_err(d[0, i, L.d_dx:L.d_dx + dims.nx], ref[("dx", i)]) for i in range(len(ctrl)))
    assert info == 0 and 1e-6 < dev < 5e-2
    flags = [ctypes.c_int.in_dll(lib, n) for n in ("orc_debug_exact_chi", "orc_debug_exact_transition", "orc_debug_exact_impact_costate")]
    try:
        for f in flags:
            f.value = 1
        kk, ric, d, info = oracle_lib.riccati_batch(dims, L, ctrl, kkt, dx0, max_dts0=1e9)
    finally:
        for f in flags:
            f.value = 0
    assert info == 0
    for i in range(len(ctrl)):
        di = d[0, i]
        assert rel_err(di[L.d_dx:L.d_dx + dims.nx], ref[("dx", i)]) < 1e-9
        if ("du", i) in ref:
            assert rel_err(di[L.d_du:L.d_du + dims.nu], ref[("du", i)]) < 1e-9
        if ("xi", i) in ref:
            assert rel_err(di[L.d_dxi:L.d_dxi + ctrl[i].ns], ref[("xi", i)]) < 1e-7
        assert rel_err(di[L.d_dlmdgmm:L.d_dlmdgmm + dims.nx], ref[("lmd", i)]) < 1e-8  # (impact grid: third switch)
        if ctrl[i].type != IMPACT and i < len(ctrl) - 1:
            a = ts[phase[i] - 1] if phase[i] >= 1 else 0.0
            b = ts[phase[i]] if phase[i] < n_events else 0.0
            assert abs(di[L.d_dts] - a) < 1e-9 and abs(di[L.d_dts + 1] - b) < 1e-9


def test_unconstr_oracle_direction_solves_full_kkt():
    """Unconstrained (iiwa14) Riccati oracle (unconstr_riccati_recursion.cpp:26-48 and factorizers) against a dense solve of
    the LQ KKT system with the implicit dynamics  x+ = [[I, dt I],[0, I]] x + [0; dt I] a + Fx."""
    from robotoc_b200.layout import ULayout
    from synth import make_unconstr_kkt, mat
    nv, N, dt = 7, 12, 0.05
    nx = 2 * nv
    lib = oracle_lib.load()
    UL = ULayout(nv, getter=lib.orc_ulayout_get)
    kkt, dx0 = make_unconstr_kkt(nv, UL, N, 2, 31)
    kk, ric, d, info = oracle_lib.unconstr_batch(nv, UL, N, dt, kkt, dx0)
    assert info == 0
    A = np.block([[np.eye(nv), dt * np.eye(nv)], [np.zeros((nv, nv)), np.eye(nv)]])
    B = np.vstack([np.zeros((nv, nv)), dt * np.eye(nv)])
    for b in range(2):
        idx, n = {}, 0
        for i in range(N + 1):
            for name, size in (("dx", nx), ("lmd", nx)) + ((("da", nv),) if i < N else ()):
                idx[(name, i)] = slice(n, n + size)
                n += size
        Kmat, rhs, I = np.zeros((n, n)), np.zeros(n), np.eye(nx)
        for i in range(N + 1):
            rec = kkt[b, i]
            sx, sl = idx[("dx", i)], idx[("lmd", i)]
            Kmat[sx, sx] += mat(rec, UL.k_Qxx, nx, nx)
            Kmat[sx, sl] += -I
            rhs[sx] += -rec[UL.k_lx:UL.k_lx + nx]
            if i == 0:
                Kmat[sl, sx] += I
                rhs[sl] += dx0[b]
            if i < N:
                sa, sxn, sln = idx[("da", i)], idx[("dx", i + 1)], idx[("lmd", i + 1)]
                Qxa = mat(rec, UL.k_Qxu, nx, nv)
                Kmat[sx, sa] += Qxa
                Kmat[sa, sx] += Qxa.T
                Kmat[sa, sa] += mat(rec, UL.k_Qaa, nv, nv)
                rhs[sa] += -rec[UL.k_la:UL.k_la + nv]
                Kmat[sx, sln] += A.T
                Kmat[sln, sx] += A
                Kmat[sa, sln] += B.T
                Kmat[sln, sa] += B
                Kmat[sln, sxn] += -I
                rhs[sln] += -rec[UL.k_Fx:UL.k_Fx + nx]
        sol = np.linalg.solve(Kmat, rhs)
        for i in range(N + 1):
            assert rel_err(d[b, i, UL.d_dx:UL.d_dx + nx], sol[idx[("dx", i)]]) < 1e-9
            assert rel_err(d[b, i, UL.d_dlmdgmm:UL.d_dlmdgmm + nx], sol[idx[("lmd", i)]]) < 1e-8
            if i < N:
                assert rel_err(d[b, i, UL.d_da:UL.d_da + nv], sol[idx[("da", i)]]) < 1e-9
