"""TEST INFRASTRUCTURE: one full hot-path iteration on the CPU oracle and the block-by-block comparison of a CUDA result
with it.  Shared by the -m gpu parity tests, __graft_entry__.smoke() and the pre-timing check of bench.py.

  condense -> backward Riccati -> forward Riccati -> expand + step sizes -> update
  (the linear-algebra body of OCPSolver::updateSolution, robotoc/src/solver/ocp_solver.cpp:118-144)
"""
import ctypes

import numpy as np

import oracle_lib
from helpers import rel_err
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


def compare_reference_records(S, K, ctrl, got, ref, tol, skip_sol=True, impact_cones=False):
    """Every section the reference's code produces, stage by stage (sections it leaves untouched are not compared)."""
    def rel(name, a, b):
        s = float(np.max(np.abs(b)))
        if s == 0.0:
            assert float(np.max(np.abs(a))) == 0.0, name
            return
        e = float(np.max(np.abs(a - b))) / s
        assert e < tol, f"{name}: {e:.2e}"
    nx, nu, nv = K.nx, K.nu, K.nv
    got, ref = dict(got), dict(ref)
    for dct in (got, ref):  # sections nothing reads on grid points without switching-time optimisation
        dct["kkt"] = mask_unread_sto(K, S, ctrl, kkt=np.array(dct["kkt"]))
        dct["ex_upd"] = mask_unread_sto(K, S, ctrl, ex=np.array(dct["ex_upd"]))
    for i, c in enumerate(ctrl):
        rel(f"Qxx[{i}]", got["kkt"][:, i, K.k_Qxx:K.k_Qxx + nx * nx], ref["kkt"][:, i, K.k_Qxx:K.k_Qxx + nx * nx])
        rel(f"lx[{i}]", got["kkt"][:, i, K.k_lx:K.k_lx + nx], ref["kkt"][:, i, K.k_lx:K.k_lx + nx])
        rel(f"P[{i}]", got["ric"][:, i, K.r_P:K.r_P + nx * nx], ref["ric"][:, i, K.r_P:K.r_P + nx * nx])
        rel(f"dx[{i}]", got["d_upd"][:, i, K.d_dx:K.d_dx + nx], ref["d_upd"][:, i, K.d_dx:K.d_dx + nx])
        rel(f"dlmdgmm[{i}]", got["d_upd"][:, i, K.d_dlmdgmm:K.d_dlmdgmm + nx], ref["d_upd"][:, i, K.d_dlmdgmm:K.d_dlmdgmm + nx])
        if c.type == TERMINAL:
            continue
        nvf = nv + c.nf
        rel(f"kkt[{i}]", got["kkt"][:, i], ref["kkt"][:, i])
        for f, n in (("e_Z", S.nvf * S.nvf), ("e_R", S.nvf * nx), ("e_r", nvf), ("e_Qafqv", S.nvf * nx), ("e_laf", nvf), ("e_Fqqpi", 36)):
            o = getattr(S, f)
            rel(f"{f}[{i}]", got["ex_upd"][:, i, o:o + n], ref["ex_upd"][:, i, o:o + n])
        rel(f"daf[{i}]", got["xd_exp"][:, i, S.x_daf:S.x_daf + nvf], ref["xd_exp"][:, i, S.x_daf:S.x_daf + nvf])
        rel(f"dbetamu[{i}]", got["xd_upd"][:, i, S.x_dbetamu:S.x_dbetamu + nvf], ref["xd_upd"][:, i, S.x_dbetamu:S.x_dbetamu + nvf])
        if c.type == IMPACT:
            if impact_cones:  # the ImpactFrictionCone rows (the box rows do not exist on an impact stage)
                for key, fields in (("cc_cond", ("c_cmpl", "c_cond")), ("cc_exp", ("c_dslack", "c_ddual")), ("cc_upd", ("c_slack", "c_dual"))):
                    for f in fields:
                        o = getattr(S, f)
                        rel(f"impact {f}[{i}]", got[key][:, i, o + S.nbox:o + S.nc], ref[key][:, i, o + S.nbox:o + S.nc])
            continue
        for f, n in (("e_Qafu", S.nvf * nv), ("e_Qxup", nx * S.np), ("e_Quup", S.np * nu), ("e_lup", S.np), ("e_haf", nvf)):
            o = getattr(S, f)
            rel(f"{f}[{i}]", got["ex_upd"][:, i, o:o + n], ref["ex_upd"][:, i, o:o + n])
        rel(f"dnup[{i}]", got["xd_upd"][:, i, S.x_dnup:S.x_dnup + S.np], ref["xd_upd"][:, i, S.x_dnup:S.x_dnup + S.np])
        rel(f"K[{i}]", got["ric"][:, i, K.r_K:K.r_K + nx * nu], ref["ric"][:, i, K.r_K:K.r_K + nx * nu])
        rel(f"du[{i}]", got["d_upd"][:, i, K.d_du:K.d_du + nu], ref["d_upd"][:, i, K.d_du:K.d_du + nu])
        for key, fields in (("cc_cond", ("c_cmpl", "c_cond")), ("cc_exp", ("c_dslack", "c_ddual")), ("cc_upd", ("c_slack", "c_dual"))):
            for f in fields:
                o = getattr(S, f)
                rel(f"{f}[{i}]", got[key][:, i, o:o + S.nc], ref[key][:, i, o:o + S.nc])
    rel("steps", got["steps"], ref["steps"])


def cuda_iteration_records(rr, dms, S, lin, con, sol, dx0):
    """One iteration through the C ABI, every record the reference iteration stores."""
    dms.condense(lin, con)
    got = dict(kkt=dms.getKKT(), cc_cond=dms.getConstraintData())
    rr.backwardRiccatiRecursion()
    rr.forwardRiccatiRecursion(dx0)
    assert int(rr.info().max()) == 0
    got["ric"] = rr.getRiccatiFactorization()
    dms.computeStepSizes()
    got["steps"] = np.stack([dms.maxPrimalStepSize(), dms.maxDualStepSize()], axis=1)
    got["cc_exp"], got["xd_exp"] = dms.getConstraintData(), dms.getExpandedDirection()
    dms.integrateSolution(sol)
    got["d_upd"], got["xd_upd"], got["cc_upd"], got["ex_upd"] = (rr.getDirection(), dms.getExpandedDirection(), dms.getConstraintData(),
                                                                 reference_view_of_expansion(S, dms.getExpansionData()))
    return got


def riccati_blocks(L, d, c):
    nx, nu, ns = d.nx, d.nu, c.ns
    b = {"P": (L.r_P, nx * nx), "s": (L.r_s, nx)}
    if c.type != IMPACT and c.type != 3:
        b.update({"K": (L.r_K, nx * nu), "k": (L.r_k, nu)})
        if ns > 0:
            b.update({"M": (L.r_M, ns * nx), "m": (L.r_m, ns)})
    if c.sto:
        b.update({"Psi": (L.r_Psi, nx), "Phi": (L.r_Phi, nx), "sc": (L.r_sc, 5)})
        if c.type != IMPACT:
            b.update({"T": (L.r_T, nu), "W": (L.r_W, nu), "psix": (L.r_psix, nx), "psiu": (L.r_psiu, nu),
                      "phix": (L.r_phix, nx), "phiu": (L.r_phiu, nu)})
            if ns > 0:
                b.update({"mt": (L.r_mt, ns), "mtn": (L.r_mtn, ns)})
    b.update({"dtsdx": (L.r_dtsdx, nx), "stosc": (L.r_stosc, 2)})
    return b


def compare_riccati(dims, L, ctrl, got_ric, ref_ric, got_d, ref_d, got_f=None, ref_kkt=None, tol=1e-8):
    """Every block of the Riccati factorization, the direction and (if given) the factorized KKT records against the oracle's,
    stage by stage, relative to each block's scale.  Returns the worst error."""
    worst = 0.0
    for i, c in enumerate(ctrl):
        for name, (off, n) in riccati_blocks(L, dims, c).items():
            a, b = got_ric[:, i, off:off + n], ref_ric[:, i, off:off + n]
            if np.max(np.abs(b)) == 0.0:
                assert np.max(np.abs(a)) == 0.0, f"stage {i} block {name}: expected zeros"
                continue
            if name == "W" and c.ns == dims.nu:
                # ns == nu: the projected inverse Ginv - SDG^T DG is analytically zero, so W = -Ginv phi_u is pure
                # cancellation noise (~1e-14); compare on the scale of its sibling T instead of its own.
                scale = np.max(np.abs(ref_ric[:, i, L.r_T:L.r_T + dims.nu]))
                assert np.max(np.abs(a - b)) < 1e-9 * scale, f"riccati stage {i} block W (ns==nu)"
                continue
            e = rel_err(a, b)
            worst = max(worst, e)
            assert e < tol, f"riccati stage {i} block {name}: rel err {e:.3e}"
        dblocks = {"dx": (L.d_dx, dims.nx), "dlmdgmm": (L.d_dlmdgmm, dims.nx), "dts": (L.d_dts, 2)}
        if c.type not in (IMPACT, 3):
            dblocks["du"] = (L.d_du, dims.nu)
            if c.ns > 0:
                dblocks["dxi"] = (L.d_dxi, c.ns)
        for name, (off, n) in dblocks.items():
            a, b = got_d[:, i, off:off + n], ref_d[:, i, off:off + n]
            if np.max(np.abs(b)) == 0.0:
                assert np.max(np.abs(a)) < 1e-300, f"stage {i} dir {name}: expected zeros"
                continue
            e = rel_err(a, b)
            worst = max(worst, e)
            assert e < tol, f"direction stage {i} block {name}: rel err {e:.3e}"
        if got_f is not None and c.type != 3:
            fb = {"F": (L.f_F, L.k_Qxx, dims.nx ** 2)}
            if c.type != IMPACT:
                fb.update({"H": (L.f_H, L.k_Qxu, dims.nx * dims.nu), "G": (L.f_G, L.k_Quu, dims.nu ** 2),
                           "lu": (L.f_lu, L.k_lu, dims.nu)})
            for name, (fo, ko, n) in fb.items():
                e = rel_err(got_f[:, i, fo:fo + n], ref_kkt[:, i, ko:ko + n])
                worst = max(worst, e)
                assert e < tol, f"factorized KKT stage {i} block {name}: rel err {e:.3e}"
    return worst


def oracle_perf_index(lib, sd, table, ctrl, lin, con):
    """The oracle's PerformanceIndex of evalKKT per OCP: the eight values rbt_eval_kkt returns."""
    lib.orc_perf_index_batch.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 3
    perf = np.zeros((lin.shape[0], 8))
    csd = sd.c()
    lib.orc_perf_index_batch(ctypes.byref(csd), ctypes.byref(table), ctrl, len(ctrl), lin.shape[0], oracle_lib.ptr(lin),
                             oracle_lib.ptr(con), oracle_lib.ptr(perf))
    return perf


TRIAL_STRIDE = 80  # doubles per grid point of a line-search trial record: q | v | a (dv) | u | f


def oracle_trials(lib, sd, table, ctrl, sol, ref, n_trials, rate=0.75):
    """The oracle's line-search trials from the iterate `sol` along the direction of `ref` (oracle_iteration): step sizes,
    log barrier and trial records [n_trials, batch, n_grid, TRIAL_STRIDE]."""
    vp, ci, cd = ctypes.c_void_p, ctypes.c_int, ctypes.c_double
    lib.orc_trial_batch.argtypes = [vp, vp, vp, ci, ci, ci, cd] + [vp] * 8
    batch, n_grid = sol.shape[0], sol.shape[1]
    alphas, barrier = np.zeros((n_trials, batch)), np.zeros((n_trials, batch))
    trial = np.zeros((n_trials, batch, n_grid, TRIAL_STRIDE))
    csd = sd.c()
    P = oracle_lib.ptr
    lib.orc_trial_batch(ctypes.byref(csd), ctypes.byref(table), ctrl, n_grid, batch, n_trials, rate, P(sol), P(ref["d"]), P(ref["xd_exp"]),
                        P(ref["cc_exp"]), P(ref["steps"]), P(alphas), P(trial), P(barrier))
    return alphas, barrier, trial

