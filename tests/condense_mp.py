"""Extended-precision (mpmath, 100 digits) reference of the condensing kernel K2 and of the expansion kernel, written from
robotoc's source and independent of oracle/condense_oracle.c:

  condense(g, Z): one grid point's "Forms linear system" (intermediate_stage.cpp:133-148 / impact_stage.cpp:116-121)
    - PDIPM condensing of the box rows (joint_*_limit.cpp:68-75 -> pdipm.hxx computeComplementarySlackness /
      computeCondensingCoeffcient) and of the friction cones (friction_cone.cpp:194-235, impact_friction_cone.cpp:196-235),
      gated as Constraints::condenseSlackAndDual gates them: box rows never on Impact grid points, position- / velocity-level
      rows not on grid points 0 / 1 (constraints_data.cpp:20-45), cone rows of active contacts only (cond = 0 otherwise);
    - condenseContactDynamics (contact_dynamics.cpp:55-163) and condenseImpactDynamics (impact_dynamics.cpp:38-80).  Z is
      an INPUT: the MJtJinv the condensing kernel actually read, so that K1's error (tests/stage_mp.py holds K1) is not charged
      to K2.  R = Z D with the record's dIDCdqv D (on Impact grid points D holds [dIDdq 0 ; dCdq dCdv], which makes Z D the
      three products of impact_dynamics.cpp:44-49);
    - correctLinearizeStateEquation (state_equation.cpp:68-85) with the SE(3) Jacobian inverse
      [[A, X], [0, A]]^-1 = [[A^-1, -A^-1 X A^-1], [0, A^-1]] (se3_jacobian_inverse.hxx) taken from mp.inverse of A;
    - the STO scaling by 1 / num_grids_in_phase (intermediate_stage.cpp:140-148); the Terminal copy (terminal_stage.cpp:94-106).
  expand(g, rec, d): expandContactDynamicsPrimal (contact_dynamics.cpp:167-174), the slack and dual directions
    (joint_*_limit.cpp:78-82, friction_cone.cpp:238-268, pdipm.hxx:159-164) on the records the expansion reads (R, r, Z,
    cmpl as the condensing wrote them), and the fraction-to-boundary candidates (pdipm.hxx:121-142).

Every output row comes with a scale C: the same expression tree evaluated on absolute values (|Z||D| for R, sl du + mu for
cmpl, ...), so tests/stage_mp.row_errors applies unchanged: a row is held to the roundings of what it is made of, however
small it is next to its block's largest entry.

A grid point `g` is a dict of fp64 numpy arrays in mathematical (row, column) layout -- `unpack` builds it from the records.
Every function works under mp.workdps(DPS) and leaves the process's precision alone."""
import numpy as np
from mpmath import mp

DPS = 100
INTERMEDIATE, IMPACT, LIFT, TERMINAL = 0, 1, 2, 3
VAR_Q, VAR_V, VAR_A, VAR_U = 0, 1, 2, 3
NP = 6  # floating base: dim_passive


def _mpv(a):
    """fp64 values as mpf (exact); an object array of mpf passes through."""
    if isinstance(a, np.ndarray) and a.dtype == object:
        return a.copy()
    a = np.asarray(a, float)
    out = np.empty(a.shape, dtype=object)
    for idx in np.ndindex(a.shape):
        out[idx] = mp.mpf(float(a[idx]))
    return out


def _zeros(*shape):
    out = np.empty(shape, dtype=object)
    out[...] = mp.mpf(0)
    return out


def mm(A, B):
    """A @ B of object arrays of mpf, every entry one fsum at the working precision (mp.fdot)."""
    A2, B2 = np.atleast_2d(A), B if B.ndim == 2 else B[:, None]
    out = _zeros(A2.shape[0], B2.shape[1])
    if A2.shape[1] == 0:
        return out if B.ndim == 2 else out[:, 0]
    cols = [list(B2[:, j]) for j in range(B2.shape[1])]
    for i in range(A2.shape[0]):
        row = list(A2[i])
        for j, col in enumerate(cols):
            out[i, j] = mp.fdot(row, col)
    return out if B.ndim == 2 else out[:, 0]


def _f64(X):
    X = np.asarray(X, dtype=object)
    out = np.empty(X.shape)
    for idx in np.ndindex(X.shape):
        out[idx] = float(X[idx])
    return out


def _rowscale(C):
    """Scale per row: a matrix's row max, a vector's entry."""
    C = _f64(C)
    return C if C.ndim == 1 else (C.max(axis=1) if C.shape[1] else np.zeros(C.shape[0]))


def se3_inverse(blk, absolute=False):
    """[[A, X], [0, A]]^-1 (se3_jacobian_inverse.hxx:17-32) of a 6 x 6 block in mp; absolute: the |.| tree of that formula."""
    A, X = _mpv(blk[:3, :3]), _mpv(blk[:3, 3:])
    Ai = np.array(mp.inverse(mp.matrix(A.tolist())).tolist(), dtype=object)
    out = _zeros(6, 6)
    if absolute:
        Ai, X = np.abs(Ai), np.abs(X)
        out[:3, 3:] = mm(Ai, mm(X, Ai))
    else:
        out[:3, 3:] = -mm(Ai, mm(X, Ai))
    out[:3, :3], out[3:, 3:] = Ai, Ai
    return out


def _gated(g, r):
    """Does inequality row r act on this grid point (Constraints::condenseSlackAndDual / expandSlackAndDual)?"""
    nbox = len(g["box"])
    if r < nbox:
        return g["type"] != IMPACT and g["row_level"][r] + g["ineq_gate"] <= 2
    if g["type"] == IMPACT and not g["icone"]:
        return False
    return bool((g["mask"] >> ((r - nbox) // 5)) & 1)


def condense(g, Z):
    """The records the condensing writes on grid point g, from the fp64 inputs g and the fp64 MJtJinv Z [nv+nf, nv+nf]
    (None on the Terminal grid point).  Returns {name: (value [rows(, cols)], scale [rows])}."""
    with mp.workdps(DPS):
        return _condense(g, Z)


def _condense(g, Zf):
    vals, abss = _tree(g, Zf, False), _tree(g, Zf, True)
    return {k: (_f64(vals[k]), _rowscale(abss[k])) for k in vals if not k.startswith("_")}


def condense_exact(g, Z):
    """The mp values of condense(), and under "_qp" the stage QP the contact dynamics are eliminated from: the cost blocks
    after the PDIPM condensing (Qxx, Quu, Qaa, Qff, Qqf, lx, la, lf, lu).  Call under mp.workdps(DPS)."""
    return _tree(g, Z, False)


def _tree(g, Zf, A):
    """One evaluation of the whole tree: exact values (A = False) or the same tree on absolute values (A = True)."""
    I = (lambda x: np.abs(_mpv(x))) if A else _mpv           # an input
    neg = (lambda x: x) if A else (lambda x: -x)
    sub = (lambda x, y: x + y) if A else (lambda x, y: x - y)
    typ, nv, nu, nx = g["type"], g["nv"], g["nu"], 2 * g["nv"]
    if typ == TERMINAL:                                       # terminal_stage.cpp:94-106
        return {"Qxx": I(g["Qxx"]), "lx": I(g["lx"]), "Fqqpi": se3_inverse(g["se3"][1], A)}
    impact = typ == IMPACT
    nf, mu = g["nf"], mp.mpf(float(g["mu"]))
    nvf, ng, dt = nv + nf, mp.mpf(int(g["ng"])), mp.mpf(float(g["dt"]))
    Qxx, Quu, Qaa, Qff, Qqf = I(g["Qxx"]), I(g["Quu"]), I(g["Qaa"]), I(g["Qff"]), I(g["Qqf"])
    lx, la, lf, lu = I(g["lx"]), I(g["la"]), I(g["lf"]), I(g["lu"])
    out = {}
    # ---- PDIPM condensing                                   pdipm.hxx:27-100, joint_*_limit.cpp:68-75, friction_cone.cpp:194-235
    nbox, nc = len(g["box"]), len(g["slack"])
    cmpl, cond = _zeros(nc), _zeros(nc)
    sl, du, res = I(g["slack"]), I(g["dual"]), I(g["res"])
    acts = np.array([_gated(g, r) for r in range(nc)])
    for r in range(nc):
        if acts[r]:
            cmpl[r] = sub(sl[r] * du[r], mu)
            cond[r] = sub(du[r] * res[r], cmpl[r]) / sl[r]
    for r in range(nbox):
        if not acts[r]:
            continue
        var, idx, sign = g["box"][r]
        w, gs = du[r] / sl[r], (cond[r] if sign > 0 or A else -cond[r])
        if var == VAR_Q:
            Qxx[idx, idx] += w
            lx[idx] += gs
        elif var == VAR_V:
            Qxx[nv + idx, nv + idx] += w
            lx[nv + idx] += gs
        elif var == VAR_A:
            Qaa[idx] += w
            la[idx] += gs
        else:
            Quu[idx, idx] += w
            lu[idx] += gs
    stack = 0
    for ci in range(g["ncon"]):
        if not (g["mask"] >> ci) & 1:
            continue
        rows = slice(nbox + 5 * ci, nbox + 5 * ci + 5)
        if acts[nbox + 5 * ci]:
            dq, df, w = I(g["dgdq"][ci]), I(g["dgdf"][ci]), du[rows] / sl[rows]
            lx[:nv] += mm(dq.T, cond[rows])
            lf[stack:stack + 3] += mm(df.T, cond[rows])
            Qxx[:nv, :nv] += mm(dq.T, w[:, None] * dq)
            Qqf[:, stack:stack + 3] += mm(dq.T, w[:, None] * df)
            Qff[stack:stack + 3, stack:stack + 3] += mm(df.T, w[:, None] * df)
        stack += 3
    pd = [r for r in range(nc) if acts[r] or (r >= nbox and (typ != IMPACT or g["icone"]))]
    out["cmpl"] = cmpl[[r for r in range(nc) if acts[r]]]
    out["cond"] = cond[pd]                                    # data.cond.setZero() for inactive contacts   friction_cone.cpp:198
    # ---- contact / impact dynamics                          contact_dynamics.cpp:55-135, impact_dynamics.cpp:38-74
    Z, D, IDC = I(Zf), I(g["D"]), I(g["IDC"])
    R, rr = mm(Z, D), mm(Z, IDC)
    Ra, Rf, ra, rf = R[:nv], R[nv:], rr[:nv], rr[nv:]
    Qafqv = np.concatenate([neg(Qaa[:, None] * Ra), neg(mm(Qff, Rf))])
    Qafqv[nv:, :nv] = sub(Qafqv[nv:, :nv], Qqf.T)
    Qafu = np.concatenate([Qaa[:, None] * Z[:nv, :nv], mm(Qff, Z[nv:, :nv])])
    laf = np.concatenate([sub(la, Qaa * ra), sub(neg(lf), mm(Qff, rf))])
    Qxx_c = sub(Qxx, mm(R.T, Qafqv))
    Qxx_c[:nv] += mm(Qqf, Rf)
    lx_c = sub(lx, mm(R.T, laf))
    lx_c[:nv] += mm(Qqf, rf)
    out.update(R=R, r=rr, Qaf=Qafqv[nv:], laf=laf, Qaa=Qaa, Qxx=Qxx_c, lx=lx_c,
               _qp=dict(Qxx=Qxx, Quu=Quu, Qaa=Qaa, Qff=Qff, Qqf=Qqf, lx=lx, la=la, lf=lf, lu=lu))
    sdt = mp.mpf(1) if impact else dt
    F = _zeros(nx, nx)
    F[nv:, :] = neg(sdt * R[:nv])
    for k in range(nv):
        F[nv + k, nv + k] += 1
        F[k, k] = mp.mpf(1)
        if not impact:
            F[k, nv + k] = dt
    Fx = I(g["Fx"])
    Fx[nv:] = sub(Fx[nv:], sdt * ra)
    Fi = se3_inverse(g["se3"][2], A)                          # Fqq_inv          state_equation.cpp:77-78
    S0 = I(g["se3"][0])
    F[:NP, :NP] = neg(mm(Fi, S0))                             # :79-80
    if not impact:
        F[:NP, nv:nv + NP] = neg(dt * Fi)                     # :81
    Fx[:NP] = neg(mm(Fi, I(g["Fx"])[:NP]))                    # :82-83
    out.update(Fxx=F, Fx=Fx, Fqqpi=se3_inverse(g["se3"][1], A))
    if not impact:
        Qxu_full = neg(mm(R.T, Qafu))
        Qxu_full[:nv] = sub(Qxu_full[:nv], mm(Qqf, Z[nv:, :nv]))
        Quu_full = mm(Z[:nv], Qafu[:, NP:])
        Quu_full[NP:] += Quu
        lu_full = mm(Z[:nv], laf)
        lu_full[:NP] += I(g["lup"])
        lu_full[NP:] += lu
        fx = I(g["fx"])
        fx[:NP] = neg(mm(Fi, I(g["fx"])[:NP]))               # :84-85
        out.update(Quf=Qafu[nv:], Qxup=Qxu_full[:, :NP], Qxu=Qxu_full[:, NP:], Quup=Quu_full[:NP], Quu=Quu_full[NP:],
                   lup=lu_full[:NP], lu=lu_full[NP:], Fvu=dt * Z[:nv, NP:nv], fx=fx / ng)
        ns = g["ns"]
        if ns > 0:                                            # contact_dynamics.cpp:138-153
            Phia = I(g["Phia"])
            Pr = mm(Phia, ra)
            out.update(Phia=Phia, Phix=sub(I(g["Phix"]), mm(Phia, Ra)), Phiu=mm(Phia, Z[:nv, NP:nv]), p=sub(I(g["p"]), Pr),
                       Phit=sub(I(g["Phit"]), Pr) / ng)
        if g["sto"] or g["sto_next"]:                         # :156-163, intermediate_stage.cpp:140-148
            haf = np.concatenate([I(g["ha"]), neg(I(g["hf"]))])
            hx = sub(I(g["hx"]), mm(R.T, haf))
            hx[:nv] += mm(Qqf, rf) / dt
            out.update(haf=haf, hx=hx / ng, hu=(I(g["hu"]) + mm(Z[NP:nv], haf)) / ng,
                       h=np.array([sub(mp.mpf(float(abs(g["sc"][0]) if A else g["sc"][0])), mm(rr[None], haf)[0]) / ng],
                                  dtype=object),
                       Qtt=np.array([I(g["sc"][1:2])[0] / (ng * ng)], dtype=object))
    return out


def expand(g, R, r, Z, cmpl, dx, du):
    """expandContactDynamicsPrimal and the slack / dual directions on one grid point, from the fp64 records the expansion
    reads (R [nv+nf, nx], r, Z [nv+nf, nv+nf], cmpl [nc]) and the direction (dx, du).  Returns
    {"daf" | "dslack" | "ddual": (value, scale)} and the exact dslack, ddual of the acting rows (for the step sizes)."""
    with mp.workdps(DPS):
        v, a = _expand(g, R, r, Z, cmpl, dx, du, False), _expand(g, R, r, Z, cmpl, dx, du, True)
        return {k: (_f64(v[k]), _rowscale(a[k])) for k in ("daf", "dslack", "ddual")}, v


def _expand(g, Rf, rf, Zf, cmf, dxf, duf, A):
    I = (lambda x: np.abs(_mpv(x))) if A else _mpv
    neg = (lambda x: x) if A else (lambda x: -x)
    sub = (lambda x, y: x + y) if A else (lambda x, y: x - y)
    nv, impact = g["nv"], g["type"] == IMPACT
    R, rr, Z, dx = I(Rf), I(rf), I(Zf), I(dxf)
    daf = neg(mm(R, dx))                                      # contact_dynamics.cpp:167-174
    if not impact:
        daf = daf + mm(Z[:, NP:nv], I(duf))
    daf = sub(daf, rr)
    daf[nv:] = neg(daf[nv:])
    nbox, nc = len(g["box"]), len(g["slack"])
    sl, dl, res, cm = I(g["slack"]), I(g["dual"]), I(g["res"]), I(cmf)
    rows = [r for r in range(nc) if _gated(g, r)]
    dsl, ddu = _zeros(len(rows)), _zeros(len(rows))
    for k, r in enumerate(rows):
        if r < nbox:                                          # joint_*_limit.cpp:78-82: dslack = -sign dvar - residual
            var, idx, sign = g["box"][r]
            x = dx[idx] if var == VAR_Q else dx[nv + idx] if var == VAR_V else daf[idx] if var == VAR_A else I(duf)[idx]
            dsl[k] = sub(x if (sign < 0 or A) else -x, res[r])
        else:                                                 # friction_cone.cpp:253-256
            ci = (r - nbox) // 5
            stack = 3 * bin(g["mask"] & ((1 << ci) - 1)).count("1")
            dq, df = I(g["dgdq"][ci])[(r - nbox) % 5], I(g["dgdf"][ci])[(r - nbox) % 5]
            dsl[k] = sub(neg(mp.fdot(list(dq), list(dx[:nv])) + mp.fdot(list(df), list(daf[nv + stack:nv + stack + 3]))),
                         res[r])
        ddu[k] = neg(dl[r] * dsl[k] + cm[r]) / sl[r]          # pdipm.hxx:159-164
    return {"daf": daf, "dslack": dsl, "ddual": ddu, "rows": rows}


# ---- the records <-> a grid point ----------------------------------------------------------------------------------------
def _blk(rec, off, rows, cols, ld):
    return rec[off:off + ld * cols].reshape(cols, ld)[:, :rows].T.copy()


def unpack(S, tab, c, row_level, lin, con):
    """Grid point dict from one linearization record `lin`, one PDIPM record `con`, its control word c and the table."""
    nv, nu, nx, nfm = S.nv, S.nu, S.nx, S.nfm
    nf = c.nf
    g = dict(type=int(c.type), nv=nv, nu=nu, nf=nf, mask=int(c.contact_mask), ineq_gate=int(c.ineq_gate), ns=int(c.ns),
             sto=bool(c.sto), sto_next=bool(c.sto_next), ng=int(c.ngrids_in_phase), dt=float(c.dt), mu=float(tab.barrier),
             icone=bool(tab.impact_friction_cone), ncon=int(tab.n_contacts),
             box=[(tab.box[r].var, tab.box[r].idx, tab.box[r].sign) for r in range(tab.n_box)], row_level=list(row_level))
    g["Qxx"], g["lx"] = _blk(lin, S.l_Qxx, nx, nx, nx), lin[S.l_lx:S.l_lx + nx].copy()
    g["se3"] = [_blk(lin, S.l_se3 + 36 * k, 6, 6, 6) for k in range(3)]
    if c.type == TERMINAL:
        return g
    nc = S.nc
    g.update(D=_blk(lin, S.l_D, nv + nf, nx, S.nvf), IDC=lin[S.l_IDC:S.l_IDC + nv + nf].copy(),
             Qaa=lin[S.l_Qaa:S.l_Qaa + nv].copy(), Qff=_blk(lin, S.l_Qff, nf, nf, nfm), Qqf=_blk(lin, S.l_Qqf, nv, nf, nv),
             Quu=_blk(lin, S.l_Quu, nu, nu, nu), la=lin[S.l_la:S.l_la + nv].copy(), lf=lin[S.l_lf:S.l_lf + nf].copy(),
             lu=lin[S.l_lu:S.l_lu + nu].copy(), Fx=lin[S.l_Fx:S.l_Fx + nx].copy(), lup=lin[S.l_lup:S.l_lup + NP].copy(),
             Phix=_blk(lin, S.l_Phix, c.ns, nx, max(c.ns, 1)), Phia=_blk(lin, S.l_Phia, c.ns, nv, max(c.ns, 1)),
             p=lin[S.l_p:S.l_p + c.ns].copy(), Phit=lin[S.l_Phit:S.l_Phit + c.ns].copy(), ha=lin[S.l_ha:S.l_ha + nv].copy(),
             hf=lin[S.l_hf:S.l_hf + nf].copy(), hx=lin[S.l_hx:S.l_hx + nx].copy(), hu=lin[S.l_hu:S.l_hu + nu].copy(),
             fx=lin[S.l_fx:S.l_fx + nx].copy(), sc=lin[S.l_sc:S.l_sc + 2].copy(),
             dgdq=[_blk(lin, S.l_dgdq + ci * 5 * nv, 5, nv, 5) for ci in range(S.ncon)],
             dgdf=[_blk(lin, S.l_dgdf + ci * 15, 5, 3, 5) for ci in range(S.ncon)],
             slack=con[S.c_slack:S.c_slack + nc].copy(), dual=con[S.c_dual:S.c_dual + nc].copy(),
             res=con[S.c_res:S.c_res + nc].copy())
    return g


def acting_rows(g):
    """Inequality rows whose cmpl the condensing writes, and rows whose cond it writes (inactive contacts' cones: zero)."""
    nbox, nc = len(g["box"]), len(g["slack"])
    acts = [r for r in range(nc) if _gated(g, r)]
    pd = [r for r in range(nc) if _gated(g, r) or (r >= nbox and (g["type"] != IMPACT or g["icone"]))]
    return acts, pd


def written(S, K, g, kkt, ex, con, oracle=False):
    """What the kernels wrote on grid point g, in the shapes and names of condense(): {name: array}.  oracle: the records of
    oracle/condense_oracle.c, which holds the full Qafqv | Qafu instead of their contact rows Qaf | Quf and diag(Qaa)."""
    nv, nu, nx, nfm, nvf = S.nv, S.nu, S.nx, S.nfm, S.nv + g["nf"]
    out = {"Qxx": _blk(kkt, K.k_Qxx, nx, nx, nx), "lx": kkt[K.k_lx:K.k_lx + nx].copy(),
           "Fqqpi": _blk(ex, S.e_Fqqpi, 6, 6, 6)}
    if g["type"] == TERMINAL:
        return out
    nf, ns = g["nf"], g["ns"]
    acts, pd = acting_rows(g)
    out.update(R=_blk(ex, S.e_R, nvf, nx, S.nvf), r=ex[S.e_r:S.e_r + nvf].copy(), Qaf=_blk(ex, S.e_Qaf, nf, nx, nfm),
               laf=ex[S.e_laf:S.e_laf + nvf].copy(), Qaa=ex[S.e_Qaa:S.e_Qaa + nv].copy(), Fxx=_blk(kkt, K.k_Fxx, nx, nx, nx),
               Fx=kkt[K.k_Fx:K.k_Fx + nx].copy(), cmpl=con[S.c_cmpl + np.array(acts, int)],
               cond=con[S.c_cond + np.array(pd, int)])
    if oracle:
        out["Qaf"] = _blk(ex, S.e_Qafqv, nv + nf, nx, S.nvf)[nv:]
        del out["Qaa"]
    if g["type"] != IMPACT:
        out.update(Quf=_blk(ex, S.e_Qafu, nv + nf, nv, S.nvf)[nv:] if oracle else _blk(ex, S.e_Quf, nf, nv, nfm), Qxup=_blk(ex, S.e_Qxup, nx, NP, nx), Qxu=_blk(kkt, K.k_Qxu, nx, nu, nx),
                   Quup=_blk(ex, S.e_Quup, NP, nu, NP), Quu=_blk(kkt, K.k_Quu, nu, nu, nu),
                   lup=ex[S.e_lup:S.e_lup + NP].copy(), lu=kkt[K.k_lu:K.k_lu + nu].copy(), Fvu=_blk(kkt, K.k_Fvu, nv, nu, nv),
                   fx=kkt[K.k_fx:K.k_fx + nx].copy())
        if ns > 0:
            out.update(Phia=_blk(ex, S.e_Phia, ns, nv, ns), Phix=_blk(kkt, K.k_Phix, ns, nx, ns),
                       Phiu=_blk(kkt, K.k_Phiu, ns, nu, ns), p=kkt[K.k_p:K.k_p + ns].copy(),
                       Phit=kkt[K.k_Phit:K.k_Phit + ns].copy())
        if g["sto"] or g["sto_next"]:
            out.update(haf=ex[S.e_haf:S.e_haf + nvf].copy(), hx=kkt[K.k_hx:K.k_hx + nx].copy(),
                       hu=kkt[K.k_hu:K.k_hu + nu].copy(), h=kkt[K.k_sc + 2:K.k_sc + 3].copy(),
                       Qtt=kkt[K.k_sc:K.k_sc + 1].copy())
    return out
