"""GPU parity at the BASELINE.json batch sizes: every OCP of the batch against the CPU oracle, through the C ABI.

  configs[2]  ANYmal trot N=40, batch 1024   full iteration + Riccati-only API
  configs[3]  ANYmal jump STO N=80, batch 512  full iteration
  configs[1]  iiwa14 N=50, batch 256          Riccati-only API (the full unconstrained iteration at 256 is in
                                              test_gpu_unconstr_stage.py)
48,128-CTA grids of the stage kernels, the >1-wave backward sweep and the 8-chunk host pipeline only exist at these sizes.
Tolerance 1e-8 relative per block (north_star: 1e-6 on P, K and the Newton direction)."""
import numpy as np
import pytest

import oracle_lib
from helpers import crawl_schedule, jump_sto_schedule, rel_err, trot_schedule
from iteration_check import compare_final, oracle_iteration, oracle_sensitivity, run_device_iteration
from robotoc_b200 import (ANYMAL, DirectMultipleShooting, Layout, RiccatiRecursion, StageDims, StageLayout, ULayout,
                          UnconstrRiccatiRecursion, anymal_constraint_table)
from synth import make_kkt, make_stage_inputs, make_unconstr_kkt, symmetrize_lin
from test_gpu_parity import _compare

pytestmark = pytest.mark.gpu
TOL = 1e-8


def _full_iteration(ctrl, batch, seed):
    table = anymal_constraint_table()
    sd = StageDims(ANYMAL, nf_max=12, n_contacts=table.n_contacts, n_box=table.n_box)
    S, K = StageLayout(sd), Layout(ANYMAL)
    lin, con, sol, dx0 = make_stage_inputs(sd, S, ctrl, batch, seed)
    lin = symmetrize_lin(S, lin)
    ref = oracle_iteration(sd, S, K, table, ctrl, lin, con, sol, dx0)
    sens = oracle_sensitivity(sd, S, K, table, ctrl, lin, con, sol, dx0, ref)
    print(f"oracle sensitivity to a 1e-15 input perturbation: median {np.median(sens):.1e}, max {sens.max():.1e}, "
          f"{int((sens > 1e-11).sum())} of {batch} OCPs above 1e-11")
    rr = RiccatiRecursion(ANYMAL, len(ctrl), batch)
    rr.setTimeDiscretization(ctrl)
    dms = DirectMultipleShooting(rr, sd, table)
    got = run_device_iteration(rr, dms, lin, con, sol, dx0)
    assert int(got["info"].max()) == 0
    worst = compare_final(S, K, ctrl, ref, got["ric"], got["d"], got["steps"], got["sol"], got["cc"], TOL, sensitivity=sens)
    # the one-call host path (8 chunks at this batch size, wire records) returns the same bits
    sol2, con2, steps2 = dms.iteration_host_wire(dms.pack_wire(lin), lin, con, sol, dx0)
    used = S.s_xi + S.nsm
    np.testing.assert_array_equal(sol2[:, :, :used], got["sol"][:, :, :used])
    np.testing.assert_array_equal(steps2, got["steps"])
    for f in ("c_slack", "c_dual"):
        o = getattr(S, f)
        np.testing.assert_array_equal(con2[:, :, o:o + S.nc], got["cc"][:, :, o:o + S.nc])
    rr.close()
    return worst


def test_config3_trot_n40_batch1024_full_iteration():
    td, ev, ctrl = trot_schedule(40)
    assert len(ctrl) == 47
    print("worst rel err", _full_iteration(ctrl, 1024, 20260930))


def test_config4_jump_sto_n80_batch512_full_iteration():
    td, ev, ctrl = jump_sto_schedule(80)
    assert len(ctrl) == 84 and any(c.sto for c in ctrl)
    print("worst rel err", _full_iteration(ctrl, 512, 20260931))


def test_crawl_n54_batch1024_full_iteration():
    """The crawl schedule (three-foot stances, single-foot impacts, ns = 3) at the trot config's batch size."""
    td, ev, ctrl = crawl_schedule(54)
    assert len(ctrl) == 61
    print("worst rel err", _full_iteration(ctrl, 1024, 20260935))


def test_config3_trot_n40_batch1024_riccati_api():
    """Riccati-only API on factory-style KKT blocks (kkt_factory.cpp recipe), every block of every record of every OCP."""
    td, ev, ctrl = trot_schedule(40)
    dims, L = ANYMAL, Layout(ANYMAL)
    kkt, dx0 = make_kkt(dims, L, ctrl, batch=1024, seed=20260932)
    rr = RiccatiRecursion(dims, len(ctrl), 1024)
    rr.setTimeDiscretization(ctrl)
    rr.backwardRiccatiRecursion(kkt, write_fact=True)
    rr.forwardRiccatiRecursion(dx0)
    assert int(rr.info().max()) == 0
    kk, ric_o, d_o, info = oracle_lib.riccati_batch(dims, L, ctrl, kkt, dx0)
    assert info == 0
    w = _compare(dims, L, ctrl, rr.getRiccatiFactorization(), ric_o, rr.getDirection(), d_o, rr.getFactorizedKKT(), kk)
    print("worst rel err", w)
    rr.close()


def test_config4_jump_sto_n80_batch512_riccati_api():
    td, ev, ctrl = jump_sto_schedule(80)
    dims, L = ANYMAL, Layout(ANYMAL)
    kkt, dx0 = make_kkt(dims, L, ctrl, batch=512, seed=20260933)
    rr = RiccatiRecursion(dims, len(ctrl), 512)
    rr.setTimeDiscretization(ctrl)
    rr.backwardRiccatiRecursion(kkt, write_fact=True)
    rr.forwardRiccatiRecursion(dx0)
    assert int(rr.info().max()) == 0
    kk, ric_o, d_o, info = oracle_lib.riccati_batch(dims, L, ctrl, kkt, dx0)
    assert info == 0
    w = _compare(dims, L, ctrl, rr.getRiccatiFactorization(), ric_o, rr.getDirection(), d_o, rr.getFactorizedKKT(), kk)
    print("worst rel err", w)
    rr.close()


def test_config2_iiwa14_n50_batch256_riccati_api():
    nv, N, batch, dt = 7, 50, 256, 0.02
    UL = ULayout(nv)
    kkt, dx0 = make_unconstr_kkt(nv, UL, N, batch, seed=20260934)
    ur = UnconstrRiccatiRecursion(nv, N, dt, batch)
    ur.backwardRiccatiRecursion(kkt)
    ur.forwardRiccatiRecursion(dx0)
    assert int(ur.info().max()) == 0
    kk, ric_o, d_o, info = oracle_lib.unconstr_batch(nv, UL, N, dt, kkt, dx0)
    assert info == 0
    ric, d = ur.getRiccatiFactorization(), ur.getDirection()
    nx = 2 * nv
    for i in range(N + 1):
        for name, off, n in (("P", UL.r_P, nx * nx), ("s", UL.r_s, nx)) + ((("K", UL.r_K, nx * nv), ("k", UL.r_k, nv)) if i < N else ()):
            assert rel_err(ric[:, i, off:off + n], ric_o[:, i, off:off + n]) < TOL, f"stage {i} {name}"
        for name, off, n in (("dx", UL.d_dx, nx), ("dlmdgmm", UL.d_dlmdgmm, nx)) + ((("da", UL.d_da, nv),) if i < N else ()):
            assert rel_err(d[:, i, off:off + n], d_o[:, i, off:off + n]) < TOL, f"dir stage {i} {name}"
    ur.close()
