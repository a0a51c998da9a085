"""Extended-precision, definition-level reference of the rigid-body rows of the contact-dynamics linearisation (mpmath).

A different formulation from tests/rbd_ref.py and tests/contact_ref.py, on purpose: nothing is propagated forward-mode, and
every quantity is derived from world poses.
  - World poses chain the placements: oMi = oMparent * placement * M_J(q), M_J by mp.sin / mp.cos for a revolute joint and by
    the unit quaternion for the free flyer.  integrate(q, xi) right-multiplies the free flyer's M_J by mp.expm of the 4x4 twist
    matrix of xi and adds xi to the joint angles.
  - LOCAL body twist and acceleration (Pinocchio's convention, motion = [linear | angular]) along q(t) = integrate(q, t v +
    t^2/2 a): V = (R^T p', (R^T R')v), A = dV/dt = (R'^T p' + R^T p'', (R^T R'')v), with p', R', p'', R'' by central
    differences of the poses at t = -h, 0, h.
  - Column k of a Jacobian is the twist along integrate(q, t e_k).
  - tau = sum_b J_b^T (I_b (A_b - g_b) + V_b x* I_b V_b - fext_b) by virtual work, g_b the gravity in body b's frame;
    M = sum_b J_b^T I_b J_b.  fext follows Robot::setContactForces: per contact in order, fext[parent] = jXf (f, 0), zero for an
    inactive contact, so a later contact on the same parent replaces an earlier one.
  - Contact rows: C = a_f,lin + w_f x v_f,lin + kv v_f,lin + kp (oMf.p - p_des) from the contact frame's own poses (the
    classical acceleration), C = v_f,lin at v + dv on Impact grid points.
  - d/dv by a central difference with a unit step: every row is at most quadratic in v, so this is exact.  d/dq by central
    differences q (+) (+-h e_k).  Impact grid points use v = 0, dv in place of a and no gravity in the ID rows.
Every row comes with the size of its largest additive contribution (tau: inertial, bias, gravity, contact, each measured as
sum_b |J_b|^T |f_b|, the size of the terms the sum adds; C: a_cl, kv v, kp oMf.p, kp p_des), and every derivative row with the
largest entry of the same split, so a comparison can scale each row by what it is made of.

Precision: 100 digits and h = 2^-66 ~ 1.4e-20.  The nested differences (a second difference in t inside a first difference in q) lose
at most 60 digits to cancellation and have truncation errors of order h^2 = 1e-40, far below the 1e-25 the comparisons need."""
from mpmath import mp

DPS = 100                  # evaluate() works at this precision (mp.workdps); the process's mp.dps is left alone
H = mp.mpf(2) ** -66       # ~1.4e-20, exact at any precision
NV, NB, NCON = 18, 13, 4
ZERO, FLOOR = 1e-30, 1e-3  # see row_scale
DQ_FLOOR = 1e-4            # see row_scale


# ---- 3-vectors and row-major 3x3 matrices as lists of mpf
def mm(A, B):
    return [A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j] for i in range(3) for j in range(3)]


def mv(A, x):
    return [A[3 * i] * x[0] + A[3 * i + 1] * x[1] + A[3 * i + 2] * x[2] for i in range(3)]


def mtv(A, x):
    return [A[i] * x[0] + A[3 + i] * x[1] + A[6 + i] * x[2] for i in range(3)]


def mtm(A, B):  # A^T B
    return [A[i] * B[j] + A[3 + i] * B[3 + j] + A[6 + i] * B[6 + j] for i in range(3) for j in range(3)]


def cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def vee(X):  # of the skew-symmetric part
    return [(X[7] - X[5]) / 2, (X[2] - X[6]) / 2, (X[3] - X[1]) / 2]


def add(a, b):
    return [x + y for x, y in zip(a, b)]


def sub(a, b):
    return [x - y for x, y in zip(a, b)]


def scale(s, a):
    return [s * x for x in a]


class Model:
    """A model dict (fields of rbt_robot_model) in mpf: rotations row-major."""

    def __init__(self, model):
        f = lambda x: mp.mpf(float(x))  # noqa: E731
        col = lambda r: [f(r[3 * j + i]) for i in range(3) for j in range(3)]  # noqa: E731  (stored column-major)
        self.parent = [int(x) for x in model["parent"]]
        self.axis = [[f(x) for x in u] for u in model["axis"]]
        self.RP = [col(pl[:9]) for pl in model["placement"]]
        self.pP = [[f(x) for x in pl[9:12]] for pl in model["placement"]]
        self.mass = [f(x) for x in model["mass"]]
        self.com = [[f(x) for x in c] for c in model["com"]]
        self.Ic = [col(i) for i in model["inertia"]]
        self.cparent = [int(x) for x in model["contact_parent"]]
        self.cR = [col(pl[:9]) for pl in model["contact_placement"]]
        self.cp = [[f(x) for x in pl[9:12]] for pl in model["contact_placement"]]
        self.gravity = [f(x) for x in model["gravity"]]


# ---- configurations: (R, p) of the free flyer's joint transform and the joint angles
def config(q):
    x, y, z, w = (mp.mpf(float(t)) for t in q[3:7])
    n = mp.sqrt(x * x + y * y + z * z + w * w)
    x, y, z, w = x / n, y / n, z / n, w / n
    R = [1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
         2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
         2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]
    return R, [mp.mpf(float(t)) for t in q[:3]], [mp.mpf(float(t)) for t in q[7:]]


def integrate(cfg, xi):
    """cfg (+) xi: the free flyer's M_J times expm of the twist [v | w] of xi[:6], the joint angles plus xi[6:]."""
    R, p, th = cfg
    if any(xi[:6]):
        v, w = xi[:3], xi[3:6]
        T = mp.expm(mp.matrix([[0, -w[2], w[1], v[0]], [w[2], 0, -w[0], v[1]], [-w[1], w[0], 0, v[2]], [0, 0, 0, 0]]))
        Re = [T[i, j] for i in range(3) for j in range(3)]
        p = add(p, mv(R, [T[0, 3], T[1, 3], T[2, 3]]))
        R = mm(R, Re)
    return R, p, [t + d for t, d in zip(th, xi[6:])]


def poses(M, cfg):
    """World (R, p) of every body, then of every contact frame."""
    R0, p0, th = cfg
    out = []
    for b in range(len(M.parent)):
        if b == 0:
            RJ, pJ = R0, p0
        else:
            s, c = mp.sin(th[b - 1]), mp.cos(th[b - 1])
            u = M.axis[b]
            t = 1 - c
            RJ = [c + u[0] * u[0] * t, u[0] * u[1] * t - u[2] * s, u[0] * u[2] * t + u[1] * s,
                  u[1] * u[0] * t + u[2] * s, c + u[1] * u[1] * t, u[1] * u[2] * t - u[0] * s,
                  u[2] * u[0] * t - u[1] * s, u[2] * u[1] * t + u[0] * s, c + u[2] * u[2] * t]
            pJ = None
        R = mm(M.RP[b], RJ)
        p = M.pP[b] if pJ is None else add(M.pP[b], mv(M.RP[b], pJ))
        pa = M.parent[b]
        if pa >= 0:
            Rp, pp = out[pa]
            R, p = mm(Rp, R), add(pp, mv(Rp, p))
        out.append((R, p))
    for c in range(len(M.cparent)):
        Rp, pp = out[M.cparent[c]]
        out.append((mm(Rp, M.cR[c]), add(pp, mv(Rp, M.cp[c]))))
    return out


def motion(M, cfg, v, a):
    """(poses, V, A) of every body and contact frame along integrate(cfg, t v + t^2/2 a) at t = 0, without gravity."""
    Pm, P0, Pp = (poses(M, integrate(cfg, [s * H * x + (s * H) ** 2 / 2 * y for x, y in zip(v, a)])) for s in (-1, 0, 1))
    V, A = [], []
    for (Rm, pm), (R, p), (Rp, pp) in zip(Pm, P0, Pp):
        Rd, pd = scale(1 / (2 * H), sub(Rp, Rm)), scale(1 / (2 * H), sub(pp, pm))
        Rdd = scale(1 / (H * H), add(sub(Rp, scale(2, R)), Rm))
        pdd = scale(1 / (H * H), add(sub(pp, scale(2, p)), pm))
        V.append(mtv(R, pd) + vee(mtm(R, Rd)))
        A.append(add(mtv(Rd, pd), mtv(R, pdd)) + vee(mtm(R, Rdd)))
    return P0, V, A


def jacobians(M, cfg):
    """J[o][k]: the LOCAL twist of body / contact frame o per unit velocity in direction k."""
    P0 = poses(M, cfg)
    cols = []
    for k in range(NV):
        e = [mp.zero] * NV
        e[k] = H
        Pp, Pm = poses(M, integrate(cfg, e)), poses(M, integrate(cfg, [-x for x in e]))
        cols.append([mtv(R, scale(1 / (2 * H), sub(p1, p0))) + vee(mtm(R, scale(1 / (2 * H), sub(R1, R0))))
                     for (R, _), (R1, p1), (R0, p0) in zip(P0, Pp, Pm)])
    return [[cols[k][o] for k in range(NV)] for o in range(len(P0))]


# ---- spatial algebra on 6-vectors [lin | ang]
def inertia_mul(M, b, m):
    c = M.com[b]
    f = scale(M.mass[b], sub(m[:3], cross(c, m[3:])))
    return f + add(mv(M.Ic[b], m[3:]), cross(c, f))


def cross_force(m, f):  # m x* f
    return cross(m[3:], f[:3]) + add(cross(m[3:], f[3:]), cross(m[:3], f[:3]))


def jt(Jo, f):  # J^T f [NV]
    return [sum(x * y for x, y in zip(col, f)) for col in Jo]


def fext(M, f, mask):
    """Body-frame external forces by Robot::setContactForces' assignment semantics; f stacks the active contacts' forces."""
    out, k = {}, 0
    for c in range(len(M.cparent)):
        if (mask >> c) & 1:
            lin = mv(M.cR[c], [mp.mpf(float(x)) for x in f[k:k + 3]])
            out[M.cparent[c]] = lin + cross(M.cp[c], lin)
            k += 3
        else:
            out[M.cparent[c]] = [mp.zero] * 6
    return out


def jt_abs(Jo, f):  # |J|^T |f| [NV]: the size of the terms J^T f sums
    return [sum(abs(x * y) for x, y in zip(col, f)) for col in Jo]


def tau_terms(M, kin, gravity):
    """[inertial, bias, gravity] [3] of {body: its body-frame force} whose J_b^T sum to tau = RNEA without external forces."""
    P, V, A = kin
    out = [{}, {}, {}]
    for b in range(len(M.parent)):
        g = mtv(P[b][0], M.gravity) + [mp.zero] * 3 if gravity else [mp.zero] * 6
        out[0][b] = inertia_mul(M, b, A[b])
        out[1][b] = cross_force(V[b], inertia_mul(M, b, V[b]))
        out[2][b] = scale(-1, inertia_mul(M, b, g))
    return out


def contact_terms(fx):
    """The contact part of tau as {body: -fext_b}."""
    return {b: scale(-1, f) for b, f in fx.items()}


def sum_terms(J, terms):
    """(sum_b J_b^T t_b, sum_b |J_b|^T |t_b|) [NV] each: a row and the size of the terms it sums."""
    out, mag = [mp.zero] * NV, [mp.zero] * NV
    for b, t in terms.items():
        out = add(out, jt(J[b], t))
        mag = add(mag, jt_abs(J[b], t))
    return out, mag


def dsum_terms_size(J, Jp, Jm, terms, tp, tm, step):
    """Size of the central difference of sum_b J_b^T t_b in one direction: sum_b |dJ_b|^T |t_b| + |J_b|^T |dt_b| [NV]."""
    mag = [mp.zero] * NV
    for b, t in terms.items():
        dt = scale(1 / (2 * step), sub(tp[b], tm[b]))
        if Jp is J:
            mag = add(mag, jt_abs(J[b], dt))
        else:
            dJ = [scale(1 / (2 * step), sub(x, y)) for x, y in zip(Jp[b], Jm[b])]
            mag = add(mag, add(jt_abs(dJ, t), jt_abs(J[b], dt)))
    return mag


def contact_parts(M, c, kin, impact, kp, kv, pdes):
    """[a_cl, kv v, kp oMf.p, -kp p_des] [4][3] of C_c (Impact: [v_f,lin, 0, 0, 0])."""
    P, V, A = kin
    o = len(M.parent) + c
    vf, af = V[o], A[o]
    z = [mp.zero] * 3
    if impact:
        return [vf[:3], z, z, z]
    kp, kv = mp.mpf(float(kp)), mp.mpf(float(kv))
    return [add(af[:3], cross(vf[3:], vf[:3])), scale(kv, vf[:3]), scale(kp, P[o][1]),
            [-kp * mp.mpf(float(x)) for x in pdes]]


def mass_matrix(M, J):
    """(M [NV][NV], row scale: the largest entry of any body's J^T I J in the row)."""
    out = [[mp.zero] * NV for _ in range(NV)]
    rs = [mp.zero] * NV
    for b in range(len(M.parent)):
        IJ = [inertia_mul(M, b, J[b][k]) for k in range(NV)]
        for i in range(NV):
            row = jt(J[b], IJ[i])
            out[i] = add(out[i], row)
            rs[i] = max(rs[i], max(abs(x) for x in row))
    return out, rs


def evaluate(model, q, v, a, dv, masks, forces, gains, pdes):
    """Every row of one state as float arrays (a dict of numpy arrays), computed at DPS digits.

    masks [n_mask] contact masks, forces [n_mask, 12] (the active contacts' forces stacked), gains [NCON, 2] (kp, kv),
    pdes [NCON, 3].  Index g: 0 = Intermediate / Lift (q, v, a, gravity), 1 = Impact (ID rows at v = 0, a = dv, no gravity;
    contact rows at v + dv).  tau* [2, n_mask, NV], dtau_dq*, dtau_dv* [2, n_mask, NV, NV] (dtau_dv[1] = 0: the ID kernel
    writes that block as zero), M [NV, NV], C* [2, NCON, 3], dC_dq*, dC_dv* [2, NCON, 3, NV], J [NCON, 3, NV]; each *_scale
    the row's largest contribution.  The contributions of tau and of its derivatives are measured by the size of the terms
    they sum (sum_b |J_b|^T |f_b|, and for a derivative in direction k sum_b |dJ_b|^T |f_b| + |J_b|^T |df_b|, largest over
    k), so a row that cancels between bodies (the yaw torque of a vertical gravity) keeps the size of what it cancels."""
    with mp.workdps(DPS):
        return _evaluate(model, q, v, a, dv, masks, forces, gains, pdes)


def _evaluate(model, q, v, a, dv, masks, forces, gains, pdes):
    import numpy as np
    M = Model(model)
    mpf = lambda x: [mp.mpf(float(t)) for t in x]  # noqa: E731
    v, a, dv = mpf(v), mpf(a), mpf(dv)
    z = [mp.zero] * NV
    vdv = add(v, dv)
    cfg = config(q)
    fxs = [fext(M, f, m) for m, f in zip(masks, forces)]
    kin_args = [(v, a), (z, dv), (vdv, z)]   # ID / contact rows (0), ID rows at Impact (1), contact rows at Impact (2)

    cterms = [contact_terms(fx) for fx in fxs]

    def rows(cfg, J, kins):
        """At one configuration: tau parts [2][n_mask] of ([4][NV] rows, [4][NV] sizes), contact parts [2][NCON][4][3], the
        Jacobians and the tau terms [2] of ([3] common {body: force}) -- what the differences below need."""
        terms = [tau_terms(M, kins[g], g == 0) for g in (0, 1)]
        common = [[sum_terms(J, t) for t in terms[g]] for g in (0, 1)]
        tp = []
        for g in (0, 1):
            tp.append([])
            for ct in cterms:
                parts = common[g] + [sum_terms(J, ct)]
                tp[g].append(([p[0] for p in parts], [p[1] for p in parts]))
        cp = [[contact_parts(M, c, kins[0 if g == 0 else 2], g == 1, gains[c][0], gains[c][1], pdes[c]) for c in range(NCON)]
              for g in (0, 1)]
        return tp, cp, J, terms

    J = jacobians(M, cfg)
    kin0 = [motion(M, cfg, *x) for x in kin_args]
    base = rows(cfg, J, kin0)
    dq_cols = []
    for k in range(NV):
        e = [mp.zero] * NV
        e[k] = H
        pm = []
        for s in (1, -1):
            c2 = integrate(cfg, scale(s, e))
            pm.append(rows(c2, jacobians(M, c2), [motion(M, c2, *x) for x in kin_args]))
        dq_cols.append(pm)
    dv_cols = []
    for k in range(NV):
        e = [mp.zero] * NV
        e[k] = mp.one
        pm = []
        for s in (1, -1):
            ek = scale(s, e)
            kins = [motion(M, cfg, add(v, ek), a), kin0[1], motion(M, cfg, add(vdv, ek), z)]
            pm.append(rows(cfg, J, kins))
        dv_cols.append(pm)

    def diff(cols, step, sel):
        """[parts][rows][NV] central differences of the part array selected by sel from rows()."""
        plus = [sel(c[0]) for c in cols]
        minus = [sel(c[1]) for c in cols]
        return [[[(plus[k][i][r] - minus[k][i][r]) / (2 * step) for k in range(NV)] for r in range(len(plus[0][i]))]
                for i in range(4)]

    f64 = lambda x: np.array(x, dtype=object).astype(float)  # noqa: E731  (mpf -> nearest double)
    tot = lambda parts: [sum(p[r] for p in parts) for r in range(len(parts[0]))]  # noqa: E731
    rsc = lambda parts: [max(abs(p[r]) for p in parts) for r in range(len(parts[0]))]  # noqa: E731
    msc = lambda parts: [max(max(abs(x) for x in p[r]) for p in parts) for r in range(len(parts[0]))]  # noqa: E731

    def dsize(cols, step, g, j):
        """[NV] row sizes of the derivative of tau (grid kind g, mask j) along cols: the largest over directions and parts."""
        rs = [mp.zero] * NV
        for (pp, pm) in cols:
            Jp, Jm = pp[2], pm[2]
            parts = [(base[3][g][i], pp[3][g][i], pm[3][g][i]) for i in range(3)] + [(cterms[j], cterms[j], cterms[j])]
            for t0, tp_, tm_ in parts:
                rs = [max(x, y) for x, y in zip(rs, dsum_terms_size(J, Jp, Jm, t0, tp_, tm_, step))]
        return rs

    mtot = lambda parts: [[sum(p[r][k] for p in parts) for k in range(NV)] for r in range(len(parts[0]))]  # noqa: E731
    out = {k: [] for k in ("tau", "tau_scale", "dtau_dq", "dtau_dq_scale", "dtau_dv", "dtau_dv_scale", "C", "C_scale",
                           "dC_dq", "dC_dq_scale", "dC_dv", "dC_dv_scale")}
    for g in (0, 1):
        for key in out:
            out[key].append([])
        for i in range(len(masks)):
            tp, tm = base[0][g][i]
            dq = diff(dq_cols, H, lambda r: r[0][g][i][0])
            dvv = diff(dv_cols, mp.one, lambda r: r[0][g][i][0])
            out["tau"][g].append(tot(tp))
            out["tau_scale"][g].append(rsc(tm))
            out["dtau_dq"][g].append(mtot(dq))
            out["dtau_dq_scale"][g].append(dsize(dq_cols, H, g, i))
            out["dtau_dv"][g].append(mtot(dvv) if g == 0 else [z] * NV)
            out["dtau_dv_scale"][g].append(dsize(dv_cols, mp.one, g, i) if g == 0 else z)
        for c in range(NCON):
            cp = base[1][g][c]
            dq = diff(dq_cols, H, lambda r: r[1][g][c])
            dvv = diff(dv_cols, mp.one, lambda r: r[1][g][c])
            out["C"][g].append(tot(cp))
            out["C_scale"][g].append(rsc(cp))
            out["dC_dq"][g].append(mtot(dq))
            out["dC_dq_scale"][g].append(msc(dq))
            out["dC_dv"][g].append(mtot(dvv))
            out["dC_dv_scale"][g].append(msc(dvv))
    Mm, Ms = mass_matrix(M, J)
    out = {k: f64(x) for k, x in out.items()}
    out["M"], out["M_scale"] = f64(Mm), f64(Ms)
    Jc = [[[J[len(M.parent) + c][k][r] for k in range(NV)] for r in range(3)] for c in range(NCON)]
    out["J"] = f64(Jc)
    out["J_scale"] = f64([[max(abs(x) for x in row) for row in Jr] for Jr in Jc])
    return out



def row_scale(scale, floor=0.0):
    """The scale each row of a block is held to: its own, with two exceptions.
    - A row that vanishes analytically (its reference size is below ZERO of the block's largest, the differences' noise at
      DPS digits: the q-derivative of a base contact's velocity) still carries the rounding of the block's intermediates, so
      it is held to FLOOR of the block's largest.
    - floor > 0 raises every row to floor x the block's largest.  dtau/dq takes DQ_FLOOR: its rows for a 1e-3 kg link at the
      end of a 12-joint chain are ~1e-6 of the block's largest but carry the rounding of the chain's accelerations, which the
      contributions of the row do not show (fp64 restatements miss them by 3e-17 of the block's largest); DQ_FLOOR holds
      such a row to 1e-16 of the block's largest, one rounding of its largest entry."""
    import numpy as np
    scale = np.asarray(scale, float)
    mx = scale.max() if scale.size else 0.0
    return np.maximum(np.where(scale < ZERO * mx, FLOOR * mx, scale), floor * mx)


def row_err(got, ref, scale, floor=0.0):
    """max over a block of |got - ref| / its row's row_scale; got, ref [rows] or [rows, cols], scale [rows]."""
    import numpy as np
    got, ref = np.asarray(got, float), np.asarray(ref, float)
    sc = row_scale(scale, floor)
    if got.ndim > sc.ndim:
        sc = sc[..., None]
    d = np.abs(got - ref)
    return float(np.max(np.where(d == 0, 0.0, d / np.where(sc > 0, sc, 1e-300)))) if d.size else 0.0
