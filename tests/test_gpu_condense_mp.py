"""The condensing kernel K2 and the expansion kernel against the extended-precision reference tests/condense_mp.py, row by
row, on the cases of tests/golden/condense_mp_cases.npz: ANYmal's own dynamics, cost scales from 1e-8 to 1e6, near-converged
and far barrier rows, gated rows, switching-constraint and STO grid points, SE(3) blocks around the branches of Jlog6.

Each kernel is isolated from the kernels before it: K2 is compared with the reference evaluated on the Z that K1 wrote, the
expansion with the reference on the R, r, Z and cmpl that K2 wrote.  Comparison rule per record, grid point and row r (as
for K1, tests/test_gpu_stage_mp.py): e_dev(r) <= max(4 e_orc(r), 16 u C(r)), with e_orc the oracle's error against the
reference on the oracle's own records (stored in the npz) and C(r) the row's scale.

Also: the Terminal copy is bit-exact, and the primal and dual step sizes are the minimum over exactly robotoc's candidate
rows (0 < -tau v / dv < 1, acting rows only) of the device's own slack and dual directions, within 4 u of its exact value."""
import ctypes
import os
import sys
import time

import numpy as np
import pytest
from mpmath import mp

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import condense_mp as C  # noqa: E402
import make_condense_mp as G  # noqa: E402

pytestmark = pytest.mark.gpu
A_, B_ = 4.0, 16.0
DIR = 3   # RBT_BUF_DIR
U = 2.0 ** -53


def _bind_direction(rr, d):
    """The direction records as RBT_BUF_DIR (a torch tensor kept alive by the caller)."""
    import torch
    t = torch.from_numpy(np.ascontiguousarray(d)).cuda()
    rr.bind_buffer(DIR, ctypes.c_void_p(t.data_ptr()))
    torch.cuda.synchronize()
    return t


def _device(run, ctrl, table, lin, con, d):
    from robotoc_b200 import ANYMAL, DirectMultipleShooting, RiccatiRecursion
    _, sd, S, K = G.setup(run)
    rr = RiccatiRecursion(ANYMAL, len(ctrl), lin.shape[0])
    rr.setTimeDiscretization(ctrl)
    try:
        dms = DirectMultipleShooting(rr, sd, table)
        dms.condense(lin, con)
        out = {"kkt": dms.getKKT(), "ex": dms.getExpansionData(), "cc": dms.getConstraintData()}
        assert int(rr.info().max()) == 0
        keep = _bind_direction(rr, d)
        dms.computeStepSizes()
        out.update(xd=dms.getExpandedDirection(), ce=dms.getConstraintData(),
                   steps=np.stack([dms.maxPrimalStepSize(), dms.maxDualStepSize()], 1))
        del keep
    finally:
        rr.close()
    return out


_DEV = {}


def _case(args):
    run, b, i = args
    _, sd, S, K = G.setup(run)
    _, _, lin, con = G.inputs_cached(run)
    dev, d = _DEV[run]
    g = G.grid_point(run, lin, con, b, i)
    return G.errors(S, K, g, dev["kkt"][b, i], dev["ex"][b, i], dev["cc"][b, i], dev["xd"][b, i], dev["ce"][b, i], d[b, i])


def test_condense_and_expansion_match_the_extended_precision_reference():
    t0 = time.time()
    data = G.load()
    for run in range(len(G.RUNS)):
        ctrl, table, lin, con = G.inputs_cached(run)
        _, sd, S, K = G.setup(run)
        d = G.direction(S, K, run)
        assert G.sha256(lin, con, d) == str(data[f"sha_inputs_{run}"]), "the case builders changed: rerun make_condense_mp.py"
        _DEV[run] = (_device(run, ctrl, table, lin, con, d), d)
        dev = _DEV[run][0]
        n = G.N_GRID - 1   # the Terminal copy is bit-exact                                     terminal_stage.cpp:94-106
        np.testing.assert_array_equal(dev["kkt"][:, n, K.k_Qxx:K.k_Qxx + S.nx * S.nx], lin[:, n, S.l_Qxx:S.l_Qxx + S.nx * S.nx])
        np.testing.assert_array_equal(dev["kkt"][:, n, K.k_lx:K.k_lx + S.nx], lin[:, n, S.l_lx:S.l_lx + S.nx])
    res = dict(zip(G.keys(), G.pool_map(_case, G.keys())))
    worst_blk, worst_fam, bad = {}, {}, []
    for (run, b, i), errs in res.items():
        for k, (e, sc) in errs.items():
            w = G.witness(data, run, k, b, i)
            e_orc = w[0] if w is not None and len(w[0]) == len(e) else np.zeros_like(e)
            bound = np.maximum(A_ * e_orc, B_ * U * sc)
            r = np.where(e == 0, 0.0, e / np.where(bound > 0, bound, 1e-300))
            r = np.where(np.isfinite(e) & np.isfinite(bound), r, np.inf)
            if r.size == 0:
                continue
            worst_blk[k] = max(worst_blk.get(k, 0.0), r.max())
            fam = f"{G.STATES[b]}/mu={G.RUNS[run][0]:g}"
            worst_fam[fam] = max(worst_fam.get(fam, 0.0), r.max())
            if not np.all(r <= 1.0):
                bad.append(f"run {run} {G.STATES[b]} grid {i} {k}: rows {np.argwhere(~(r <= 1.0)).ravel()[:6]} ratio {r.max():.3g}")
    print("worst e_dev / max(A e_orc, B u C) per block: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(worst_blk.items())))
    print("per input family: " + ", ".join(f"{k} {v:.3f}" for k, v in worst_fam.items()))
    print(f"({time.time() - t0:.1f} s)")
    assert not bad, "\n".join(bad[:20])
    for run in range(len(G.RUNS)):
        ctrl, table, lin, con = G.inputs_cached(run)
        dev, _ = _DEV[run]
        _check_steps(run, ctrl, table, lin, con, dev)


def _steps_of(S, table, ctrl, lin, con, ce, levels):
    """robotoc's step sizes over the device's own dslack / ddual: (primal, dual) per OCP, and the exact -tau v / dv (mp) of
    the two binding rows.  Candidate rows: acting rows with 0 < -tau v / dv < 1 in fp64 (pdipm.hxx:121-142); min over the
    horizon (direct_multiple_shooting.cpp:202-209)."""
    tau = table.fraction_to_boundary
    B = ce.shape[0]
    out = np.ones((B, 2))
    exact = np.ones((B, 2))
    for b in range(B):
        for i, c in enumerate(ctrl):
            if c.type == C.TERMINAL:
                continue
            g = C.unpack(S, table, c, levels, lin[b, i], con[b, i])
            for r in C.acting_rows(g)[0]:
                for k, (v, dv) in enumerate(((con[b, i, S.c_slack + r], ce[b, i, S.c_dslack + r]),
                                             (con[b, i, S.c_dual + r], ce[b, i, S.c_ddual + r]))):
                    with np.errstate(divide="ignore", invalid="ignore"):
                        f = -tau * (v / dv)
                    if 0.0 < f < 1.0 and f < out[b, k]:
                        out[b, k] = f
                        with mp.workdps(50):
                            exact[b, k] = float(-mp.mpf(tau) * mp.mpf(float(v)) / mp.mpf(float(dv)))
    return out, exact


def _check_steps(run, ctrl, table, lin, con, dev):
    _, sd, S, K = G.setup(run)
    want, exact = _steps_of(S, table, ctrl, lin, con, dev["ce"], G.row_levels(table))
    got = dev["steps"]
    assert np.all(np.abs(got - exact) <= 4 * U * exact), f"step sizes {got} != {exact}"
    np.testing.assert_array_equal(got, want)


# ---- the step sizes on rows chosen to bind -------------------------------------------------------------------------------
def test_step_sizes_bind_on_every_row():
    """OCP b < nc binds its primal step on row b and its dual step on row (b + 37) mod nc, on grid point 2 (every row acts),
    or on the first non-terminal grid point (b = 1 mod 3, if row b acts there) or the last one (b = 2 mod 3); gated rows
    (grid points 0 and 1, the Impact grid point) and inactive contacts' cone rows hold values that would bind at 0.1.  Then:
    no binding row (alpha = 1 exactly), a row at -tau s / ds == 1 exactly (not a candidate) and one at 1 - 2^-53 (a
    candidate), and ds = 0 | -0.0.  Directions dx = du = 0 and zero cone Jacobians make dslack = -residual exactly."""
    import torch
    from robotoc_b200 import ANYMAL, DirectMultipleShooting, Layout, RiccatiRecursion, StageDims, StageLayout, anymal_constraint_table
    from robotoc_b200.grid import plain_schedule
    from synth import make_stage_inputs, symmetrize_lin
    table = anymal_constraint_table(fraction_to_boundary=0.5)   # -tau s / ds can land on 1 exactly (not with tau = 0.995)
    sd = StageDims(ANYMAL, nf_max=12, n_contacts=4, n_box=table.n_box)
    S, K = StageLayout(sd), Layout(ANYMAL)
    tau, mu, nc, nbox = table.fraction_to_boundary, table.barrier, S.nc, table.n_box
    ctrl = plain_schedule(5, 0.02, 12, 0b1111)
    ctrl[1].contact_mask, ctrl[1].nf = 0b0101, 6
    ctrl[3].type = C.IMPACT
    levels = G.row_levels(table)
    B = nc + 4
    lin, con, _, _ = make_stage_inputs(sd, S, ctrl, B, 61)
    lin = symmetrize_lin(S, lin)
    lin[:, :, S.l_dgdq:S.l_dgdq + 4 * 5 * S.nv + 60] = 0.0
    sl, du, res = (con[:, :, getattr(S, f):getattr(S, f) + nc] for f in ("c_slack", "c_dual", "c_res"))
    sl[:], du[:], res[:] = 1.0, 1e-6, -1.0        # dslack = 1, ddual > 0: no candidate
    cm = 1e-6 - mu

    def bind(b, i, r, alpha, dual=False):
        if dual:   # dslack = X > 0, ddual = -(1e-6 X + cm) < 0, -tau du / ddual = alpha
            res[b, i, r] = -(tau * 1e-6 / alpha - cm) / 1e-6
        else:      # dslack = -tau / alpha, -tau s / dslack = alpha
            res[b, i, r] = tau / alpha

    for b in range(B):
        for r in range(nc):
            bind(b, 0, r, 0.1) if not (r >= nbox or levels[r] == 0) else None
            bind(b, 1, r, 0.1) if (r < nbox and levels[r] == 2) or (r >= nbox and not (0b0101 >> ((r - nbox) // 5)) & 1) else None
            bind(b, 3, r, 0.1)
    want = np.ones((B, 2))
    for b in range(nc):
        ip = 0 if (b % 3 == 1 and (b >= nbox or levels[b] == 0)) else 4 if b % 3 == 2 else 2
        want[b] = 0.5 + b / 1000, 0.6 + b / 1000
        bind(b, ip, b, want[b, 0])
        bind(b, 2, (b + 37) % nc, want[b, 1], dual=True)
    b1, b2, b3 = nc + 1, nc + 2, nc + 3
    res[b1, 2, 60], sl[b1, 2, 60] = 0.5, 1.0                      # -0.5 (1 / -0.5) = 1 exactly: not a candidate
    res[b2, 2, 61], sl[b2, 2, 61] = 1.0, np.nextafter(2.0, 0.0)   # -0.5 ((2 - 2^-51) / -1) = 1 - 2^-53: a candidate
    res[b3, 2, 62], res[b3, 2, 63] = 0.0, -0.0                                   # dslack = -0.0 | 0.0
    want[b2, 0] = np.nextafter(1.0, 0.0)
    rr = RiccatiRecursion(ANYMAL, len(ctrl), B)
    rr.setTimeDiscretization(ctrl)
    try:
        dms = DirectMultipleShooting(rr, sd, table)
        dms.condense(lin, np.ascontiguousarray(con))
        keep = _bind_direction(rr, np.zeros((B, len(ctrl), K.d_stride)))
        dms.computeStepSizes()
        torch.cuda.synchronize()
        ce = dms.getConstraintData()
        got = np.stack([dms.maxPrimalStepSize(), dms.maxDualStepSize()], 1)
        del keep
    finally:
        rr.close()
    robotoc, exact = _steps_of(S, table, ctrl, lin, con, ce, levels)
    np.testing.assert_array_equal(got, robotoc)
    assert np.all(np.abs(got - exact) <= 4 * U * exact)
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=0)
    assert got[b2, 0] == np.nextafter(1.0, 0.0) and np.all(got[[nc, b1, b3]] == 1.0)
