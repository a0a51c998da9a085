"""GPU parity: the CUDA path (through the C ABI / host mirror) against the CPU oracle on identical seeded inputs.
Tolerance: BASELINE.json north_star -- 1e-6 relative on P, K and the Newton direction (we assert 1e-8)."""
import numpy as np
import pytest

import oracle_lib
from helpers import contact_mask_walk_schedule, crawl_schedule, jump_sto_schedule, rel_err, small_event_schedule, trot_schedule
from robotoc_b200 import ANYMAL, Layout, RiccatiRecursion, ULayout, UnconstrRiccatiRecursion
from robotoc_b200 import _lib
from robotoc_b200.grid import IMPACT, INTERMEDIATE
from iteration_check import compare_riccati as _compare
from synth import make_kkt, make_unconstr_kkt

pytestmark = pytest.mark.gpu
TOL = 1e-8


def _run_case(ctrl, batch, seed, max_dts0=0.1):
    dims = ANYMAL
    L = Layout(dims)
    kkt, dx0 = make_kkt(dims, L, ctrl, batch=batch, seed=seed)
    rr = RiccatiRecursion(dims, len(ctrl), batch, max_dts0=max_dts0)
    rr.setTimeDiscretization(ctrl)
    rr.backwardRiccatiRecursion(kkt, write_fact=True)
    rr.forwardRiccatiRecursion(dx0)
    ric, d, f = rr.getRiccatiFactorization(), rr.getDirection(), rr.getFactorizedKKT()
    assert int(rr.info().max()) == 0
    kk, ric_o, d_o, info = oracle_lib.riccati_batch(dims, L, ctrl, kkt, dx0, max_dts0=max_dts0)
    assert info == 0
    worst = _compare(dims, L, ctrl, ric, ric_o, d, d_o, f, kk)
    # one-call host API gives the same answer
    ric2, d2 = rr.solve_host(kkt, dx0)
    assert np.array_equal(ric2, ric) and np.array_equal(d2, d)
    rr.close()
    return worst


def test_small_event_schedule():
    td, ev, ctrl = small_event_schedule(sto=False)
    w = _run_case(ctrl, batch=5, seed=11)
    print("worst rel err", w)


def test_trot_n40_config3_small_batch():
    """BASELINE config 3 schedule (47 grid points: 2 Lift, 2 Impact, 2 switching stages), small batch."""
    td, ev, ctrl = trot_schedule(40)
    assert len(ctrl) == 47
    w = _run_case(ctrl, batch=6, seed=20260927)
    print("worst rel err", w)


def test_small_event_schedule_sto():
    td, ev, ctrl = small_event_schedule(sto=True)
    assert any(c.sto for c in ctrl)
    w = _run_case(ctrl, batch=4, seed=5)
    print("worst rel err", w)


def test_jump_sto_n80_config4_small_batch():
    """BASELINE config 4 schedule (84 grid points, all phases STO, ns=12 switching stage)."""
    td, ev, ctrl = jump_sto_schedule(80)
    assert len(ctrl) == 84
    w = _run_case(ctrl, batch=3, seed=20260928)
    print("worst rel err", w)


@pytest.mark.parametrize("which,batch,seed", [("crawl", 5, 20260940), ("crawl_sto", 4, 20260941), ("mask_walk", 3, 20260942)])
def test_gait_schedules(which, batch, seed):
    """Crawl (nf = 3 / 9, ns = 3 switching constraints, impacts that also lift a foot), with and without switching-time
    optimisation, and the walk through all 16 contact masks (ns = 3, 6, 9, 12 through the NS = 12 Schur path)."""
    td, ev, ctrl = {"crawl": lambda: crawl_schedule(54), "crawl_sto": lambda: crawl_schedule(54, sto=True),
                    "mask_walk": contact_mask_walk_schedule}[which]()
    w = _run_case(ctrl, batch=batch, seed=seed)
    print("worst rel err", w)


RBT_FXX_AUTO, RBT_FXX_MECHANICAL, RBT_FXX_GENERAL = 0, 1, 2  # include/robotoc_b200.h


def test_backward_instance_selection_on_a_mixed_batch():
    """The backward sweep has an instance for Fxx with the mechanical structure (Fqq = I, Fqv = dt I outside the floating-base
    blocks) and a general one; with RBT_FXX_AUTO the uploaded records are inspected on the device.  One entry of ONE OCP in the
    middle of the batch breaks the structure: every OCP must still match the oracle.  On conforming records the forced general
    instance agrees with AUTO to rounding, and the declared structure gives AUTO's bits."""
    td, ev, ctrl = crawl_schedule(54)
    dims, L = ANYMAL, Layout(ANYMAL)
    nx, batch = dims.nx, 7
    kkt, dx0 = make_kkt(dims, L, ctrl, batch=batch, seed=20260943)
    lib = _lib.lib()
    rr = RiccatiRecursion(dims, len(ctrl), batch)
    rr.setTimeDiscretization(ctrl)

    def solve(mode, k):
        assert lib.rbt_set_fxx_structure(rr._h, mode) == 0
        rr.backwardRiccatiRecursion(k, write_fact=True)
        rr.forwardRiccatiRecursion(dx0)
        assert int(rr.info().max()) == 0
        return rr.getRiccatiFactorization(), rr.getDirection(), rr.getFactorizedKKT()

    auto = solve(RBT_FXX_AUTO, kkt)
    for a, b in zip(solve(RBT_FXX_MECHANICAL, kkt), auto):
        np.testing.assert_array_equal(a, b)
    gen = solve(RBT_FXX_GENERAL, kkt)
    assert rel_err(gen[0], auto[0]) < 1e-12 and rel_err(gen[1], auto[1]) < 1e-12
    for i, c in enumerate(ctrl[:-1]):  # the factorized KKT blocks the sweep writes
        for fo, n in ((L.f_F, nx * nx),) + (((L.f_H, nx * dims.nu), (L.f_G, dims.nu ** 2), (L.f_lu, dims.nu)) if c.type != IMPACT else ()):
            assert rel_err(gen[2][:, i, fo:fo + n], auto[2][:, i, fo:fo + n]) < 1e-12, f"stage {i}"
    # one Fqq entry of a leg joint row (rows NP..NV-1) of OCP 4, at a middle Intermediate stage
    ob, i = 4, next(i for i in range(len(ctrl) // 2, len(ctrl)) if ctrl[i].type == INTERMEDIATE)
    bad = kkt.copy()
    bad[ob, i, L.k_Fxx + 10 + 3 * nx] = 0.05
    kk, ric_o, d_o, info = oracle_lib.riccati_batch(dims, L, ctrl, bad, dx0)
    assert info == 0
    ric, d, f = solve(RBT_FXX_AUTO, bad)
    w = _compare(dims, L, ctrl, ric, ric_o, d, d_o, f, kk)
    print("worst rel err", w)
    # the entry matters: the structured instance, wrongly declared, misses it on that OCP only
    ric_m = solve(RBT_FXX_MECHANICAL, bad)[0]
    assert rel_err(ric_m[ob, :i + 1], ric_o[ob, :i + 1]) > 1e-6
    assert rel_err(np.delete(ric_m, ob, 0), np.delete(ric, ob, 0)) < 1e-12
    assert lib.rbt_set_fxx_structure(rr._h, RBT_FXX_AUTO) == 0
    rr.close()


@pytest.mark.parametrize("N,batch,dt", [(20, 1, 0.05), (50, 16, 0.02)])
def test_unconstr_iiwa14(N, batch, dt):
    """BASELINE configs 1 and 2 (iiwa14, nv=7)."""
    nv = 7
    UL = ULayout(nv)
    kkt, dx0 = make_unconstr_kkt(nv, UL, N, batch, seed=20260925)
    ur = UnconstrRiccatiRecursion(nv, N, dt, batch)
    ur.backwardRiccatiRecursion(kkt, write_fact=True)
    ur.forwardRiccatiRecursion(dx0)
    ric, d, f = ur.getRiccatiFactorization(), ur.getDirection(), ur.getFactorizedKKT()
    assert int(ur.info().max()) == 0
    kk, ric_o, d_o, info = oracle_lib.unconstr_batch(nv, UL, N, dt, kkt, dx0)
    assert info == 0
    nx = 2 * nv
    for i in range(N + 1):
        blocks = {"P": (UL.r_P, nx * nx), "s": (UL.r_s, nx)}
        if i < N:
            blocks.update({"K": (UL.r_K, nx * nv), "k": (UL.r_k, nv)})
        for name, (off, n) in blocks.items():
            e = rel_err(ric[:, i, off:off + n], ric_o[:, i, off:off + n])
            assert e < TOL, f"stage {i} {name}: {e:.3e}"
        dbl = {"dx": (UL.d_dx, nx), "dlmdgmm": (UL.d_dlmdgmm, nx)}
        if i < N:
            dbl["da"] = (UL.d_da, nv)
        for name, (off, n) in dbl.items():
            e = rel_err(d[:, i, off:off + n], d_o[:, i, off:off + n])
            assert e < TOL, f"dir stage {i} {name}: {e:.3e}"
        if i < N:
            for name, fo, ko, n in [("F", UL.f_F, UL.k_Qxx, nx * nx), ("H", UL.f_H, UL.k_Qxu, nx * nv),
                                    ("G", UL.f_G, UL.k_Qaa, nv * nv), ("la", UL.f_la, UL.k_la, nv)]:
                e = rel_err(f[:, i, fo:fo + n], kk[:, i, ko:ko + n])
                assert e < TOL, f"fact stage {i} {name}: {e:.3e}"
    ric2, d2 = ur.solve_host(kkt, dx0)
    assert np.array_equal(ric2, ric) and np.array_equal(d2, d)
    ur.close()
