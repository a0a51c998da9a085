"""Writes tests/golden/condense_mp_cases.npz: the inputs of the condensing kernel K2 and of the expansion on the grid points
where they could go wrong, and the oracle's (oracle/condense_oracle.c) row errors against tests/condense_mp.py evaluated on
the oracle's own MJtJinv Z -- the witness e_orc of the kernels' comparison.

Cases (one schedule, OCP b = dynamics state b, two runs):
  - dynamics: ANYmal's M, J, dIDCdqv and IDC (tests/rbd_ref.py, tests/contact_ref.py) at the six K1 states of
    make_stage_mp.py (standing, trot, touch-down, base 1e3 m away, LF knee 1e-3 rad from straight, and the same with the
    heavy base), with the v, a, dv of make_rbd_mp.anymal_states;
  - grid point 3 m + t: contact mask MASKS[m] (nf = 0, 3, 6 non-contiguous, 6, 9, 12) on grid type TYPES[t] (Intermediate,
    Lift, Impact); then Terminal.  Grid points 0 and 1 gate the position- / velocity-level box rows off;
  - switching constraints (ns = 3, 6, 12, Phia = rows of the contact Jacobian), STO grid points (sto and sto_next,
    num_grids_in_phase 1, 3, 17, dt 1e-4 ... 0.05): GRID below;
  - cost scales: diag(Qxx) 1e-4 ... 1e6 (base rows 1e6, a joint row at 1e-4), Qaa 1e-6 ... 1e1, Qff 1e-8 ... 1e-1,
    Quu 1e-6 ... 1e2, gradients scaled to match;
  - barrier rows: near-converged (slack 1e-10 ... 1e-6, dual = mu / slack (1 + delta), delta in {0, +-1e-8}, residual
    ~1e-12) and far (slack 1e1 ... 1e3, dual 1e-9 ... 1e-6) mixed inside every contact's five cone rows and on the lower /
    upper limit of the same joint; run 0: mu = 1e-3 without ImpactFrictionCone, run 1: mu = 1e-8 with it;
  - unread inputs (gated box rows, inactive contacts' cone rows and Jacobians, J beyond nf) hold garbage that would change
    every record if it were read;
  - SE(3) blocks [[Jlog3, X], [0, Jlog3]]: the inverse of the right Jacobian of exp on SE(3), sum_k (-ad xi)^k / (k+1)!
    summed in mp, at rotation angles 0, 1e-6, 1, 3, pi - 1e-6 (translation 1e3 m for the far base).
The npz holds the SHA-256 of the inputs (rebuilt by the functions below) and of the oracle's outputs, and per record and row
e_orc and the scale C (in fp32: it only sets a bound).  Deterministic bit for bit: python tests/golden/make_condense_mp.py"""
import ctypes
import hashlib
import io
import os
import sys
import zipfile

import numpy as np
from mpmath import mp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import condense_mp as C  # noqa: E402
import contact_ref  # noqa: E402
import make_rbd_mp  # noqa: E402
import make_stage_mp  # noqa: E402
import rbd_ref  # noqa: E402

PATH = os.path.join(HERE, "condense_mp_cases.npz")
STATES = make_stage_mp.STATES
MASKS = make_stage_mp.MASKS
TYPES = (0, 2, 1)   # Intermediate, Lift, Impact
RUNS = ((1e-3, False), (1e-8, True))   # (barrier mu, ImpactFrictionCone)
ANGLES = (0.0, 1e-6, 1.0, 3.0, np.pi - 1e-6)
# grid point -> (ns, sto, sto_next, num_grids_in_phase, dt) on Intermediate / Lift grid points
GRID = {0: (0, 1, 0, 17, 0.05), 3: (3, 0, 0, 3, 0.02), 4: (0, 1, 0, 1, 1e-4), 6: (6, 0, 1, 3, 1e-4), 9: (0, 0, 0, 17, 0.01),
        10: (0, 0, 1, 17, 1e-3), 12: (12, 1, 0, 3, 0.02), 13: (0, 0, 1, 1, 0.05), 15: (6, 0, 0, 17, 1e-3)}
N_GRID = len(MASKS) * len(TYPES) + 1


def schedule():
    from robotoc_b200.grid import plain_schedule
    ctrl = plain_schedule(N_GRID - 1, 0.02, 0)
    for i in range(N_GRID - 1):
        mask = int(MASKS[i // len(TYPES)])
        c = ctrl[i]
        c.type, c.contact_mask, c.nf = TYPES[i % len(TYPES)], mask, make_stage_mp.nf_of(mask)
        ns, sto, sto_next, ng, dt = GRID.get(i, (0, 0, 0, 5, 0.02))
        if c.type == 1:
            ns, sto, sto_next, dt = 0, 0, 0, 0.0
        c.ns, c.sto, c.sto_next, c.ngrids_in_phase, c.dt = ns, sto, sto_next, ng, dt
    return ctrl


def setup(run):
    from robotoc_b200 import ANYMAL, Layout, StageDims, StageLayout, anymal_constraint_table
    mu, icone = RUNS[run]
    table = anymal_constraint_table(barrier=mu, impact_friction_cone=icone)
    sd = StageDims(ANYMAL, nf_max=12, n_contacts=4, n_box=table.n_box)
    return table, sd, StageLayout(sd), Layout(ANYMAL)


def row_levels(table):
    """2 = position-, 1 = velocity-, 0 = acceleration-level row (the torque limits; JointPosition / Velocity / Torques*Limit)."""
    return [2 if table.box[r].var == C.VAR_Q else 1 if table.box[r].var == C.VAR_V else 0 for r in range(table.n_box)]


_JLOG = {}


def jlog6(rho, phi):
    key = tuple(rho) + tuple(phi)
    if key not in _JLOG:
        _JLOG[key] = _jlog6(rho, phi)
    return _JLOG[key]


def _jlog6(rho, phi):
    """[[Jlog3, X], [0, Jlog3]] = Jr(xi)^-1, Jr the right Jacobian of exp on SE(3) (motion = [linear | angular]), in mp."""
    with mp.workdps(120):
        xi = [mp.mpf(float(x)) for x in list(rho) + list(phi)]
        sk = lambda w: mp.matrix([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])  # noqa: E731
        ad = mp.zeros(6, 6)
        W, V = sk(xi[3:]), sk(xi[:3])
        for i in range(3):
            for j in range(3):
                ad[i, j], ad[i, 3 + j], ad[3 + i, 3 + j] = W[i, j], V[i, j], W[i, j]
        Jr, term, k = mp.eye(6), mp.eye(6), 1
        while True:
            term = -term * ad / (k + 1)
            Jr += term
            k += 1
            if mp.mnorm(term, 1) < mp.mpf(10) ** -110 and k > 8:
                break
        Ji = mp.inverse(Jr)
        return np.array([[float(Ji[i, j]) for j in range(6)] for i in range(6)])


def _logu(rng, lo, hi, n):
    return 10.0 ** rng.uniform(lo, hi, n)


def inputs(run):
    """(ctrl, table, lin [B, N_GRID, l_stride], con [B, N_GRID, c_stride]) of run `run`."""
    table, sd, S, K = setup(run)
    ctrl = schedule()
    B, nv, nu, nx, nfm = len(STATES), S.nv, S.nu, S.nx, S.nfm
    rng = np.random.default_rng(1234 + run)
    anymal, qs = make_stage_mp.anymal_states()
    dyn = {s["name"]: s for s in make_rbd_mp.anymal_states(anymal)}
    lin = np.zeros((B, N_GRID, S.l_stride))
    con = np.zeros((B, N_GRID, S.c_stride))
    sol = np.zeros((B, N_GRID, S.s_stride))
    for b, name in enumerate(STATES):
        st = dyn.get(name, dyn["standing"])
        sol[b, :, S.s_q:S.s_q + S.nq] = qs[name]
        sol[b, :, S.s_v:S.s_v + nv], sol[b, :, S.s_a:S.s_a + nv], sol[b, :, S.s_dv:S.s_dv + nv] = st["v"], st["a"], st["dv"]
        sol[b, :, S.s_f:S.s_f + nfm] = rng.uniform(-50, 50, (N_GRID, nfm)) + np.tile([0.0, 0.0, 75.0], 4)
        sol[b, :, S.s_u:S.s_u + nu] = rng.uniform(-20, 20, (N_GRID, nu))
    gains, pos = contact_ref.random_gains(5, 4), contact_ref.random_positions(6, 1, N_GRID, 4)
    for b, name in enumerate(STATES):
        model = make_stage_mp.heavy_base_model(anymal) if name.startswith("heavy_base") else anymal
        one = rbd_ref.linearize(model, S, ctrl, sol[b:b + 1], lin[b:b + 1])
        lin[b:b + 1] = contact_ref.linearize(model, S, ctrl, sol[b:b + 1], one, gains, pos)
    Jall = {b: [rbd_ref.contact_jacobian(make_stage_mp.heavy_base_model(anymal) if n.startswith("heavy") else anymal,
                                         qs[n][None], c)[0] for c in range(4)] for b, n in enumerate(STATES)}
    for b in range(B):
        for i, c in enumerate(ctrl):
            r = lin[b, i]
            ang = ANGLES[(b + i) % len(ANGLES)]
            for k in range(3):   # one axis and translation per (angle, block): the series is slow in mp
                a = (b + i) % len(ANGLES)
                axis = np.array([np.sin(a + k), np.cos(a + k), 0.5 * k - 0.5])
                axis /= np.linalg.norm(axis)
                rho = np.array([800.0, -600.0, 0.5]) if STATES[b] == "far_base" else np.array([0.3, -0.2, 0.1 * k])
                blk = jlog6(tuple(rho), tuple(axis * ang))
                r[S.l_se3 + 36 * k:S.l_se3 + 36 * (k + 1)] = (blk if k == 0 else -blk).T.reshape(-1)
            d = np.concatenate([np.full(6, 1e6), _logu(rng, -4, 2, 12), np.full(6, 1e6), _logu(rng, -4, 2, 12)])
            d[6 + (b + i) % 12] = 1e-4
            U = rng.uniform(-1, 1, (nx, nx))
            h = np.sqrt(d)
            Q = h[:, None] * (np.eye(nx) + 0.1 * (U + U.T)) * h[None]
            Q = 0.5 * (Q + Q.T)   # exactly symmetric, as the Hessians robotoc holds
            r[S.l_Qxx:S.l_Qxx + nx * nx] = Q.T.reshape(-1)
            r[S.l_lx:S.l_lx + nx] = h * rng.uniform(-1, 1, nx)
            if c.type == 3:
                continue
            nf = c.nf
            qaa = _logu(rng, -6, 1, nv)
            r[S.l_Qaa:S.l_Qaa + nv] = qaa
            r[S.l_la:S.l_la + nv] = np.sqrt(qaa) * rng.uniform(-1, 1, nv)
            qff = _logu(rng, -8, -1, nf)
            Qff = np.zeros((nfm, nfm))
            Qff[np.arange(nf), np.arange(nf)] = qff
            r[S.l_Qff:S.l_Qff + nfm * nfm] = Qff.T.reshape(-1)
            r[S.l_lf:S.l_lf + nfm] = 0.0
            r[S.l_lf:S.l_lf + nf] = np.sqrt(qff) * rng.uniform(-1, 1, nf)
            quu = _logu(rng, -6, 2, nu)
            hu = np.sqrt(quu)
            Uu = rng.uniform(-1, 1, (nu, nu))
            Qu = hu[:, None] * (np.eye(nu) + 0.1 * (Uu + Uu.T)) * hu[None]
            r[S.l_Quu:S.l_Quu + nu * nu] = (0.5 * (Qu + Qu.T)).T.reshape(-1)
            r[S.l_lu:S.l_lu + nu] = hu * rng.uniform(-1, 1, nu)
            r[S.l_lup:S.l_lup + 6] = 1e3 * rng.uniform(-1, 1, 6)
            r[S.l_Fx:S.l_Fx + nx] = 0.1 * rng.uniform(-1, 1, nx)
            r[S.l_fx:S.l_fx + nx] = rng.uniform(-1, 1, nx)
            r[S.l_ha:S.l_ha + nv], r[S.l_hx:S.l_hx + nx] = rng.uniform(-1, 1, nv), rng.uniform(-1, 1, nx)
            r[S.l_hf:S.l_hf + nf], r[S.l_hu:S.l_hu + nu] = rng.uniform(-1, 1, nf), rng.uniform(-1, 1, nu)
            r[S.l_sc:S.l_sc + 2] = [rng.uniform(-1, 1), rng.uniform(0.5, 1.5)]
            J4 = np.concatenate(Jall[b])
            if c.ns:
                r[S.l_Phix:S.l_Phix + c.ns * nx] = rng.uniform(-1, 1, (c.ns, nx)).T.reshape(-1)
                r[S.l_Phia:S.l_Phia + c.ns * nv] = J4[:c.ns].T.reshape(-1)
                r[S.l_p:S.l_p + c.ns], r[S.l_Phit:S.l_Phit + c.ns] = rng.uniform(-1, 1, c.ns), rng.uniform(-1, 1, c.ns)
            for ci in range(4):   # inactive contacts hold garbage: nothing may read it
                r[S.l_dgdq + ci * 5 * nv:S.l_dgdq + (ci + 1) * 5 * nv] = rng.uniform(-1, 1, (5, nv)).T.reshape(-1)
                r[S.l_dgdf + ci * 15:S.l_dgdf + (ci + 1) * 15] = rng.uniform(-1, 1, (5, 3)).T.reshape(-1)
            Jb = r[S.l_J:S.l_J + nfm * nv].reshape(nv, nfm)
            Jb[:, nf:] = rng.uniform(-1, 1, (nv, nfm - nf))
            mu = table.barrier
            ncr = S.nc
            near = rng.random(ncr) < 0.5
            sl = np.where(near, _logu(rng, -10, -6, ncr), _logu(rng, 1, 3, ncr))
            delta = rng.choice([0.0, 1e-8, -1e-8], ncr)
            du = np.where(near, mu / sl * (1.0 + delta), _logu(rng, -9, -6, ncr))
            res = np.where(near, 1e-12 * rng.uniform(-1, 1, ncr), rng.uniform(-1, 1, ncr))
            con[b, i, S.c_slack:S.c_slack + ncr], con[b, i, S.c_dual:S.c_dual + ncr] = sl, du
            con[b, i, S.c_res:S.c_res + ncr] = res
    return ctrl, table, np.ascontiguousarray(lin), np.ascontiguousarray(con)


def direction(S, K, run):
    """The direction records of the expansion: dx and du with entries from 1e-8 to 1e2 in magnitude."""
    rng = np.random.default_rng(77 + run)
    d = np.zeros((len(STATES), N_GRID, K.d_stride))
    n = S.nx + S.nu
    v = rng.choice([-1.0, 1.0], (len(STATES), N_GRID, n)) * _logu(rng, -8, 2, len(STATES) * N_GRID * n).reshape(-1, N_GRID, n)
    d[:, :, K.d_dx:K.d_dx + S.nx], d[:, :, K.d_du:K.d_du + S.nu] = v[..., :S.nx], v[..., S.nx:]
    return d


def oracle(run, lin, con, d):
    """The oracle's condensing and expansion: (kkt, ex, con after condense, xd, con after expansion, steps)."""
    import oracle_lib
    lib = oracle_lib.load()
    table, sd, S, K = setup(run)
    ctrl = schedule()
    B = lin.shape[0]
    kkt, ex = np.zeros((B, N_GRID, K.k_stride)), np.zeros((B, N_GRID, S.e_stride))
    cc = con.copy()
    assert lib.orc_condense_batch(ctypes.byref(sd.c()), ctypes.byref(table), ctrl, N_GRID, B, oracle_lib.ptr(lin),
                                  oracle_lib.ptr(cc), oracle_lib.ptr(kkt), oracle_lib.ptr(ex), 1) == 0
    ce, xd, steps = cc.copy(), np.zeros((B, N_GRID, S.x_stride)), np.ones((B, 2))
    lib.orc_expand_batch(ctypes.byref(sd.c()), ctypes.byref(table), ctrl, N_GRID, B, oracle_lib.ptr(lin), oracle_lib.ptr(ex),
                         oracle_lib.ptr(d), oracle_lib.ptr(ce), oracle_lib.ptr(xd), oracle_lib.ptr(steps), 1)
    return kkt, ex, cc, xd, ce, steps


def grid_point(run, lin, con, b, i):
    table, sd, S, K = setup(run)
    return C.unpack(S, table, schedule()[i], row_levels(table), lin[b, i], con[b, i])


def z_of(S, g, ex):
    n = S.nv + g["nf"]
    return ex[S.e_Z:S.e_Z + S.nvf * S.nvf].reshape(S.nvf, S.nvf).T[:n, :n].copy()


def errors(S, K, g, kkt, ex, cc, xd, ce, d, oracle=False):
    """{record: (e [rows], C [rows])} of the kernels' outputs (kkt, ex, cc after condense, xd, ce after expansion) on grid
    point g, against the reference evaluated on the records they themselves read (their own Z, R, r, cmpl)."""
    out = {}
    if g["type"] == 3:
        ref = C.condense(g, None)
    else:
        ref = C.condense(g, z_of(S, g, ex))
    got = C.written(S, K, g, kkt, ex, cc, oracle)
    for k, (v, sc) in ref.items():
        if k not in got:
            continue
        e = np.abs(got[k] - v)
        out[k] = (e if e.ndim == 1 else e.max(axis=1) if e.shape[1] else np.zeros(e.shape[0]), sc)
    if g["type"] == 3:
        return out
    nv, nf, nx = S.nv, g["nf"], S.nx
    rec = {"R": C._blk(ex, S.e_R, nv + nf, nx, S.nvf), "r": ex[S.e_r:S.e_r + nv + nf], "Z": z_of(S, g, ex),
           "cmpl": cc[S.c_cmpl:S.c_cmpl + S.nc]}
    xr, v = C.expand(g, rec["R"], rec["r"], rec["Z"], rec["cmpl"], d[K.d_dx:K.d_dx + nx], d[K.d_du:K.d_du + S.nu])
    rows = np.array(v["rows"], int)
    got = {"daf": xd[S.x_daf:S.x_daf + nv + nf], "dslack": ce[S.c_dslack + rows], "ddual": ce[S.c_ddual + rows]}
    for k, (val, sc) in xr.items():
        out[k] = (np.abs(got[k] - val), sc)
    return out


def _case(args):
    run, b, i = args
    table, sd, S, K = setup(run)
    ctrl, _, lin, con = inputs_cached(run)
    d = direction(S, K, run)
    kkt, ex, cc, xd, ce, _ = oracle_cached(run)
    g = grid_point(run, lin, con, b, i)
    return errors(S, K, g, kkt[b, i], ex[b, i], cc[b, i], xd[b, i], ce[b, i], d[b, i], oracle=True)


_CACHE = {}


def inputs_cached(run):
    if ("in", run) not in _CACHE:
        _CACHE[("in", run)] = inputs(run)
    return _CACHE[("in", run)]


def oracle_cached(run):
    if ("orc", run) not in _CACHE:
        table, sd, S, K = setup(run)
        _, _, lin, con = inputs_cached(run)
        _CACHE[("orc", run)] = oracle(run, lin, con, direction(S, K, run))
    return _CACHE[("orc", run)]


def sha256(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a, dtype="<f8").tobytes())
    return h.hexdigest()


def pool_map(fn, args):
    import multiprocessing as mpr
    with mpr.get_context("fork").Pool(min(len(args), os.cpu_count() or 1)) as p:
        return p.map(fn, args, chunksize=1)


def keys():
    return [(run, b, i) for run in range(len(RUNS)) for b in range(len(STATES)) for i in range(N_GRID)]


def build():
    data = {"states": np.array(STATES), "masks": np.array(MASKS)}
    for run in range(len(RUNS)):
        ctrl, table, lin, con = inputs_cached(run)
        table_, sd, S, K = setup(run)
        orc = oracle_cached(run)
        data[f"sha_inputs_{run}"] = np.array(sha256(lin, con, direction(S, K, run)))
        data[f"sha_oracle_{run}"] = np.array(sha256(*orc))
    res = dict(zip(keys(), pool_map(_case, keys())))
    for run in range(len(RUNS)):
        names = sorted({k for (r, _, _), errs in res.items() if r == run for k in errs})
        for k in names:
            parts = [res[(run, b, i)].get(k, (np.zeros(0), np.zeros(0))) for b in range(len(STATES)) for i in range(N_GRID)]
            data[f"rows/{run}/{k}"] = np.array([len(e) for e, _ in parts], dtype=np.int32)
            data[f"e_orc/{run}/{k}"] = np.concatenate([e for e, _ in parts])
            sc = np.concatenate([sc for _, sc in parts]).astype(np.float32)   # a bound: 24 bits are plenty, and the file
            data[f"scale/{run}/{k}"] = sc                                     # stays under 1 MB
    return data


def witness(data, run, k, b, i):
    """(e_orc [rows], C [rows]) of record k on OCP b, grid point i of run `run` (None if the grid point has no such record)."""
    if f"rows/{run}/{k}" not in data:   # diag(Qaa) after the PDIPM terms: the oracle keeps the full Qafqv instead
        return None
    n = data[f"rows/{run}/{k}"]
    j = b * N_GRID + i
    if n[j] == 0:
        return None
    o = int(n[:j].sum())
    return data[f"e_orc/{run}/{k}"][o:o + n[j]], data[f"scale/{run}/{k}"][o:o + n[j]].astype(float)


def save(data, path=PATH):
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as zf:
        for key in sorted(data):
            buf = io.BytesIO()
            np.save(buf, np.asarray(data[key]), allow_pickle=False)
            info = zipfile.ZipInfo(key + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(info, buf.getvalue())


def load():
    with np.load(PATH) as z:
        return {k: z[k] for k in z.files}


if __name__ == "__main__":
    data = build()
    save(data)
    print(f"wrote {PATH}: {os.path.getsize(PATH)} bytes")
