"""TEST INFRASTRUCTURE: one full hot-path iteration on the CPU oracle and the block-by-block comparison of a CUDA result
with it.  Shared by the -m gpu parity tests, __graft_entry__.smoke() and the pre-timing check of bench.py.

  condense -> backward Riccati -> forward Riccati -> expand + step sizes -> update
  (the linear-algebra body of OCPSolver::updateSolution, robotoc/src/solver/ocp_solver.cpp:118-144)
"""
import ctypes

import numpy as np

import oracle_lib
from robotoc_b200 import ANYMAL
from robotoc_b200.grid import IMPACT, TERMINAL


def oracle_iteration(sd, S, K, table, ctrl, lin, con, sol, dx0, nthreads=0):
    """Returns every intermediate record of the iteration as the oracle computes it (inputs are not modified)."""
    lib = oracle_lib.load()
    P = oracle_lib.ptr
    batch, n_grid = lin.shape[0], lin.shape[1]
    csd = sd.c()
    kkt = np.zeros((batch, n_grid, K.k_stride))
    ex = np.zeros((batch, n_grid, S.e_stride))
    cc, ss = con.copy(), sol.copy()
    rc = lib.orc_condense_batch(ctypes.byref(csd), ctypes.byref(table), ctrl, n_grid, batch, P(lin), P(cc), P(kkt), P(ex), nthreads)
    assert rc == 0, "oracle: condensing failed (non-SPD M / J M^-1 J^T)"
    cc_cond = cc.copy()
    kk, ric, d, info = oracle_lib.riccati_batch(ANYMAL, K, ctrl, kkt, dx0, nthreads=nthreads)
    assert info == 0, "oracle: Cholesky failure in the Riccati recursion"
    xd = np.zeros((batch, n_grid, S.x_stride))
    steps = np.zeros((batch, 2))
    lib.orc_expand_batch(ctypes.byref(csd), ctypes.byref(table), ctrl, n_grid, batch, P(lin), P(ex), P(d), P(cc), P(xd), P(steps), nthreads)
    d_exp, cc_exp, xd_exp = d.copy(), cc.copy(), xd.copy()
    lib.orc_update_batch(ctypes.byref(csd), ctypes.byref(table), ctrl, n_grid, batch, P(ex), P(d), P(xd), P(cc), P(ss), P(steps), nthreads)
    return dict(kkt=kkt, cc_cond=cc_cond, ric=ric, d=d_exp, cc_exp=cc_exp, xd_exp=xd_exp, steps=steps, d_upd=d, xd_upd=xd,
                cc_upd=cc, sol=ss, ex_upd=ex)


def oracle_sensitivity(sd, S, K, table, ctrl, lin, con, sol, dx0, ref, eps=1e-15, seed=0):
    """Per-OCP conditioning of the iteration, measured with the oracle itself: the largest relative change of its Riccati
    factorization, Newton direction and updated solution when the linearisation records are perturbed by `eps` relative
    (one rounding error).  No implementation can agree with another one more closely than a small multiple of this."""
    rng = np.random.default_rng(seed)
    ref2 = oracle_iteration(sd, S, K, table, ctrl, lin * (1.0 + eps * rng.standard_normal(lin.shape)), con, sol, dx0)
    nx, nu = K.nx, K.nu
    delta = np.zeros(lin.shape[0])
    for key, secs in (("ric", ((K.r_P, nx * nx), (K.r_s, nx), (K.r_K, nx * nu), (K.r_k, nu))),
                      ("d_upd", ((K.d_dx, nx), (K.d_du, nu), (K.d_dlmdgmm, nx))), ("sol", ((0, S.s_stride),))):
        for off, n in secs:
            a, b = ref[key][:, :, off:off + n], ref2[key][:, :, off:off + n]
            scale = np.max(np.abs(a), axis=(0, 2))
            scale[scale == 0.0] = 1.0
            delta = np.maximum(delta, np.max(np.max(np.abs(a - b), axis=2) / scale[None, :], axis=1))
    return delta


def _cmp(name, got, ref, tol, worst):
    """Block `name` of every OCP: max |got - ref| per OCP, relative to the block's scale over the batch (like Eigen's
    isApprox, but per instance); `tol` is a scalar or a per-OCP array."""
    scale = float(np.max(np.abs(ref)))
    if scale == 0.0:
        assert float(np.max(np.abs(got))) == 0.0, f"{name}: expected zeros"
        return
    e = np.max(np.abs(got - ref).reshape(got.shape[0], -1), axis=1) / scale
    if np.ndim(tol) == 0:
        worst[0] = max(worst[0], float(e.max()))
    else:
        strict = tol <= worst[1]
        if strict.any():
            worst[0] = max(worst[0], float(e[strict].max()))
    bad = np.nonzero(~(e < tol))[0]
    assert bad.size == 0, f"{name}: OCP {bad[0]}: rel err {e[bad[0]]:.3e} (tol {np.broadcast_to(tol, e.shape)[bad[0]]:g})"


def compare_final(S, K, ctrl, ref, ric, d, steps, sol, cc, tol=1e-8, sensitivity=None):
    """What a caller of the iteration sees at its end, EVERY OCP of the batch, block by block and stage by stage:
    P, s, K, k (north_star: 1e-6 relative; asserted at `tol`), the Newton direction dx, du, dlmd|dgmm (after the costate
    correction of the update), the horizon-wide step sizes, the updated solution and slack / dual.
    `sensitivity` (oracle_sensitivity): OCPs whose own oracle result moves by more than 1e-3 * tol under a one-rounding-error
    input perturbation are ill-conditioned instances; they are held to max(tol, 1e3 * sensitivity) instead, and may be at most
    2 % of the batch.  Returns the worst error over the strictly compared OCPs."""
    nx, nu = K.nx, K.nu
    worst = [0.0, tol]
    steps_tol = 1e-10
    if sensitivity is not None:
        loose = sensitivity > 1e-3 * tol
        assert loose.sum() <= max(1, len(sensitivity) // 50), f"{loose.sum()} ill-conditioned OCPs: the synthetic inputs are unfit"
        tol = np.where(loose, np.maximum(tol, 1e3 * sensitivity), tol)
        steps_tol = np.where(loose, np.maximum(steps_tol, 1e3 * sensitivity), steps_tol)
    for i, c in enumerate(ctrl):
        _cmp(f"P[{i}]", ric[:, i, K.r_P:K.r_P + nx * nx], ref["ric"][:, i, K.r_P:K.r_P + nx * nx], tol, worst)
        _cmp(f"s[{i}]", ric[:, i, K.r_s:K.r_s + nx], ref["ric"][:, i, K.r_s:K.r_s + nx], tol, worst)
        _cmp(f"dx[{i}]", d[:, i, K.d_dx:K.d_dx + nx], ref["d_upd"][:, i, K.d_dx:K.d_dx + nx], tol, worst)
        _cmp(f"dlmdgmm[{i}]", d[:, i, K.d_dlmdgmm:K.d_dlmdgmm + nx], ref["d_upd"][:, i, K.d_dlmdgmm:K.d_dlmdgmm + nx], tol, worst)
        _cmp(f"sol[{i}]", sol[:, i], ref["sol"][:, i], tol, worst)
        if c.type in (IMPACT, TERMINAL):
            continue
        _cmp(f"K[{i}]", ric[:, i, K.r_K:K.r_K + nx * nu], ref["ric"][:, i, K.r_K:K.r_K + nx * nu], tol, worst)
        _cmp(f"k[{i}]", ric[:, i, K.r_k:K.r_k + nu], ref["ric"][:, i, K.r_k:K.r_k + nu], tol, worst)
        _cmp(f"du[{i}]", d[:, i, K.d_du:K.d_du + nu], ref["d_upd"][:, i, K.d_du:K.d_du + nu], tol, worst)
        if c.ns > 0:
            _cmp(f"dxi[{i}]", d[:, i, K.d_dxi:K.d_dxi + c.ns], ref["d_upd"][:, i, K.d_dxi:K.d_dxi + c.ns], tol, worst)
        for f in ("c_slack", "c_dual"):
            o = getattr(S, f)
            _cmp(f"{f}[{i}]", cc[:, i, o:o + S.nc], ref["cc_upd"][:, i, o:o + S.nc], tol, worst)
    _cmp("steps", steps, ref["steps"], steps_tol, worst)
    return worst[0]


def mask_unread_sto(K, S, ctrl, kkt=None, ex=None):
    """The CUDA condensing computes the switching-time sensitivities hx, hu, {Qtt, Qtt_prev, h} (KKT record) and haf (expansion
    record) only on grid points whose phase duration is optimised (sto or sto_next) -- nothing reads them elsewhere; the
    reference / oracle compute them everywhere.  Zeroes those sections on the other grid points (in place) so that whole
    records can be compared."""
    for i, c in enumerate(ctrl):
        if c.sto or c.sto_next:
            continue
        if kkt is not None:
            for off, n in ((K.k_hx, K.nx), (K.k_hu, K.nu), (K.k_sc, 4)):
                kkt[:, i, off:off + n] = 0.0
        if ex is not None:
            ex[:, i, S.e_haf:S.e_haf + S.nvf] = 0.0
    return kkt if kkt is not None else ex


def reference_view_of_expansion(S, ex):
    """The CUDA path keeps only the contact rows [Qaf | Quf] of Qafqv / Qafu_full plus diag(Qaa) (rbt_stage_layout.h); this
    fills the full matrices the reference / oracle hold (contact_dynamics.cpp:68-86: acceleration rows -diag(Qaa) R_a and
    diag(Qaa) Z_aa) into a copy of the expansion records, so that the same comparisons apply to both."""
    out = ex.copy()
    nv, nx, nfm, nvf = S.nv, S.nx, S.nfm, S.nvf
    sh = ex.shape[:2]
    Qaa = ex[..., S.e_Qaa:S.e_Qaa + nv]
    R = ex[..., S.e_R:S.e_R + nvf * nx].reshape(sh + (nx, nvf))        # [.., col, row]
    Z = ex[..., S.e_Z:S.e_Z + nvf * nvf].reshape(sh + (nvf, nvf))
    Qaf = ex[..., S.e_Qaf:S.e_Qaf + nfm * nx].reshape(sh + (nx, nfm))
    Quf = ex[..., S.e_Quf:S.e_Quf + nfm * nv].reshape(sh + (nv, nfm))
    full = np.zeros(sh + (nx, nvf))
    full[..., :nv] = -R[..., :nv] * Qaa[..., None, :]
    full[..., nv:] = Qaf
    out[..., S.e_Qafqv:S.e_Qafqv + nvf * nx] = full.reshape(sh + (-1,))
    fullu = np.zeros(sh + (nv, nvf))
    fullu[..., :nv] = Z[..., :nv, :nv] * Qaa[..., None, :]
    fullu[..., nv:] = Quf
    out[..., S.e_Qafu:S.e_Qafu + nvf * nv] = fullu.reshape(sh + (-1,))
    return out


def run_device_iteration(rr, dms, lin, con, sol, dx0, stream=None):
    """The five C-ABI calls of one iteration on device-resident records; returns what compare_final needs."""
    dms.condense(lin, con, stream=stream)
    rr.backwardRiccatiRecursion(stream=stream)
    rr.forwardRiccatiRecursion(dx0, stream=stream)
    dms.computeStepSizes(stream=stream)
    dms.integrateSolution(sol, stream=stream)
    steps = np.stack([dms.maxPrimalStepSize(stream), dms.maxDualStepSize(stream)], axis=1)
    return dict(ric=rr.getRiccatiFactorization(stream), d=rr.getDirection(stream), steps=steps, sol=dms.getSolution(stream),
                cc=dms.getConstraintData(stream), info=rr.info(stream))
