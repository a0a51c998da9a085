"""The extended-precision reference of the condensing and expansion kernels, tests/condense_mp.py, and its cases
tests/golden/condense_mp_cases.npz (CPU): identities of the reference at 1e-40, the npz recomputed live, and the oracle
(oracle/condense_oracle.c) held to the reference row by row on its own records.  The kernels are held to the same cases by
tests/test_gpu_condense_mp.py."""
import os
import sys

import numpy as np
import pytest
from mpmath import mp

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import condense_mp as C  # noqa: E402
import make_condense_mp as G  # noqa: E402

DATA = G.load()
EPS = mp.mpf(10) ** -40


def test_case_file_holds_the_current_inputs_and_oracle():
    """A changed case builder or a changed oracle fails here instead of comparing against a stale witness."""
    for run in range(len(G.RUNS)):
        _, _, lin, con = G.inputs_cached(run)
        _, _, S, K = G.setup(run)
        assert G.sha256(lin, con, G.direction(S, K, run)) == str(DATA[f"sha_inputs_{run}"]), "rerun make_condense_mp.py"
        assert G.sha256(*G.oracle_cached(run)) == str(DATA[f"sha_oracle_{run}"]), "the oracle changed: rerun make_condense_mp.py"
    assert os.path.getsize(G.PATH) < 1 << 20


def test_case_file_covers_the_edges():
    ctrl = G.schedule()
    cs = [ctrl[i] for i in range(G.N_GRID - 1)]
    for t in G.TYPES:
        assert sorted(c.nf for c in cs if c.type == t) == [0, 3, 6, 6, 9, 12]
    assert {c.ns for c in cs} == {0, 3, 6, 12}
    assert any(c.sto for c in cs) and any(c.sto_next for c in cs) and {1, 3, 17} <= {c.ngrids_in_phase for c in cs if c.sto or c.sto_next}
    dts = [c.dt for c in cs if c.type != C.IMPACT]
    assert min(dts) == 1e-4 and max(dts) == 0.05
    assert [ctrl[0].ineq_gate, ctrl[1].ineq_gate] == [2, 1] and ctrl[G.N_GRID - 1].type == C.TERMINAL
    for run in range(len(G.RUNS)):
        table, _, S, _ = G.setup(run)
        _, _, lin, con = G.inputs_cached(run)
        mu = table.barrier
        sl, du = con[:, :-1, S.c_slack:S.c_slack + S.nc], con[:, :-1, S.c_dual:S.c_dual + S.nc]
        near, far = (sl <= 1e-6) & (np.abs(sl * du - mu) <= 2e-8 * mu), (sl >= 10) & (du <= 1e-6)
        assert np.all(near | far)
        assert np.any(sl * du == mu) and np.any(sl * du > mu) and np.any(sl * du < mu)
        cones = near[..., S.nbox:].reshape(near.shape[:2] + (4, 5))
        assert np.any(cones.any(-1) & ~cones.all(-1))                              # both kinds inside one contact's cone
        box = near[..., :S.nbox].reshape(near.shape[:2] + (3, 2, 12))
        assert np.any(box[..., 0, :] != box[..., 1, :])                             # lower and upper limit of one joint
        d = np.einsum("bgii->bgi", lin[:, :-1, S.l_Qxx:S.l_Qxx + S.nx * S.nx].reshape(lin.shape[0], -1, S.nx, S.nx))
        assert d.min() < 2e-4 and d.max() > 5e5                                     # 1e-4 ... 1e6 before the coupling
        qaa = lin[:, :-1, S.l_Qaa:S.l_Qaa + S.nv]
        assert qaa.min() < 1e-5 and qaa.max() > 1.0
    angles = {float(np.linalg.norm(k[3:])) for k in G._JLOG}                      # the SE(3) blocks' rotation angles
    for a in G.ANGLES:
        assert any(abs(x - a) <= 1e-15 * max(a, 1e-6) for x in angles), a
    assert any(k[0] == 800.0 for k in G._JLOG)                                     # the far base's translation


def _kkt_inverse(Z):
    return mp.inverse(mp.matrix(np.asarray(C._mpv(Z)).tolist()))


@pytest.mark.parametrize("run,b,i", [(0, 1, 15), (1, 4, 4), (1, 5, 9)])
def test_reference_condensing_is_the_reduced_stage_qp(run, b, i):
    """Eliminating (a, f) from the stage QP -- the cost after the PDIPM condensing, subject to the linearised contact
    dynamics K [a; -f] + D dx - [0 ; I_nu ; 0] du + IDC = 0 with K = Z^-1 (Z the oracle's, made exactly symmetric) -- gives a reduced gradient equal to
    [Qxx Qxu; Qxu^T Quu] [dx; du] + [lx; lu] of the reference, at two random (dx, du)."""
    _, _, S, _ = G.setup(run)
    _, _, lin, con = G.inputs_cached(run)
    kkt, ex, *_ = G.oracle_cached(run)
    g = G.grid_point(run, lin, con, b, i)
    Zf = G.z_of(S, g, ex[b, i])
    nv, nu, nx, nf = S.nv, S.nu, S.nx, g["nf"]
    rng = np.random.default_rng(3)
    with mp.workdps(C.DPS):
        Zm = C._mpv(Zf)
        Zs = (Zm + Zm.T) / 2   # the identity needs K = Z^-1 symmetric; the fp64 Z of the oracle is so only to rounding
        out = C.condense_exact(g, Zs)
        qp = out["_qp"]
        Kinv = mp.inverse(mp.matrix(Zs.tolist()))
        D, IDC = C._mpv(g["D"]), C._mpv(g["IDC"])
        for _ in range(2):
            x, u = C._mpv(rng.uniform(-1, 1, nx)), C._mpv(rng.uniform(-1, 1, nu))

            def solve(x, u, aff):
                rhs = C.mm(D, x)
                rhs[6:nv] -= u
                if aff:
                    rhs = rhs + IDC
                w = mp.lu_solve(Kinv, mp.matrix(list(-rhs)))
                return np.array([w[k] for k in range(nv)], dtype=object), np.array([-w[nv + k] for k in range(nf)], dtype=object)

            a, f = solve(x, u, True)
            ga = qp["Qaa"] * a + qp["la"]                          # dPhi/da, dPhi/df, dPhi/dx, dPhi/du at (x, u, a, f)
            gf = C.mm(qp["Qff"], f) + qp["lf"] + C.mm(qp["Qqf"].T, x[:nv])
            gx = C.mm(qp["Qxx"], x) + qp["lx"]
            gx[:nv] += C.mm(qp["Qqf"], f)
            gu = C.mm(qp["Quu"], u) + qp["lu"]
            red = np.concatenate([gx, gu])
            for k in range(nx + nu):                               # chain rule through the linear part of (a, f)
                e = C._zeros(nx + nu)
                e[k] = mp.mpf(1)
                da, df = solve(e[:nx], e[nx:], False)
                red[k] += mp.fdot(list(ga), list(da)) + mp.fdot(list(gf), list(df))
            cond = np.concatenate([C.mm(out["Qxx"], x) + C.mm(out["Qxu"], u) + out["lx"],
                                   C.mm(out["Qxu"].T, x) + C.mm(out["Quu"], u) + out["lu"]])
            err = max(abs(p - q) for p, q in zip(red, cond))
            assert err < EPS * max(1, max(abs(q) for q in cond)), f"reduced gradient off by {err}"


def test_reference_se3_inverse_and_expansion_identities():
    """Fqq_inv * block = I for every SE(3) block of the cases, and daf of the reference satisfies the eliminated contact
    dynamics K [da; -df] + D dx - [0 ; I_nu ; 0] du + IDC = 0 (K = Z^-1)."""
    with mp.workdps(C.DPS):
        for blk in list(G._JLOG.values()) + [-v for v in G._JLOG.values()]:
            E = C.mm(C.se3_inverse(blk), C._mpv(blk))
            assert max(abs(E[i, j] - (1 if i == j else 0)) for i in range(6) for j in range(6)) < EPS
    for run, b, i in ((0, 2, 12), (1, 3, 7), (1, 0, 14)):
        _, _, S, K = G.setup(run)
        _, _, lin, con = G.inputs_cached(run)
        _, ex, cc, *_ = G.oracle_cached(run)
        g = G.grid_point(run, lin, con, b, i)
        Zf = G.z_of(S, g, ex[b, i])
        nv, nf = S.nv, g["nf"]
        d = G.direction(S, K, run)[b, i]
        with mp.workdps(C.DPS):
            Z, D, IDC = C._mpv(Zf), C._mpv(g["D"]), C._mpv(g["IDC"])
            dx, du = C._mpv(d[K.d_dx:K.d_dx + S.nx]), C._mpv(d[K.d_du:K.d_du + S.nu])
            _, v = C.expand(g, C.mm(Z, D), C.mm(Z, IDC), Z, cc[b, i][S.c_cmpl:S.c_cmpl + S.nc], dx, du)
            w = np.concatenate([v["daf"][:nv], -v["daf"][nv:]])
            res = C.mm(np.array(_kkt_inverse(Zf).tolist(), dtype=object), w) + C.mm(D, dx) + IDC
            if g["type"] != C.IMPACT:
                res[6:nv] -= du
            scale = max(1, max(abs(x) for x in C.mm(D, dx) + IDC))
            assert max(abs(x) for x in res) < EPS * scale


@pytest.mark.parametrize("run,b,i", [(0, 4, 9), (1, 5, 13)])
def test_npz_is_what_the_reference_computes(run, b, i):
    """Two grid points recomputed live, bit for bit: the oracle's row errors and the row scales."""
    for k, (e, sc) in G._case((run, b, i)).items():
        w = G.witness(DATA, run, k, b, i)
        assert w is not None, k
        np.testing.assert_array_equal(e, w[0], err_msg=k)
        np.testing.assert_array_equal(sc.astype(np.float32).astype(float), w[1], err_msg=k)


def test_oracle_against_the_reference():
    """The oracle, the witness of the GPU comparison, within 16 u of each row's scale on every record it writes (measured:
    at most 6.9 u C, on daf)."""
    U = 2.0 ** -53
    worst = {}
    for key in DATA:
        if not key.startswith("e_orc/"):
            continue
        _, run, k = key.split("/")
        e, sc = DATA[key], DATA[f"scale/{run}/{k}"].astype(float)
        r = np.where(e == 0, 0.0, e / np.where(sc > 0, U * sc, 1e-300))
        worst[k] = max(worst.get(k, 0.0), float(r.max()) if r.size else 0.0)
        assert np.all(r <= 16.0), f"run {run} {k}: e / (u C) = {r.max():.3g}"
    print("oracle worst e / (u C) per block: " + ", ".join(f"{k} {v:.2f}" for k, v in sorted(worst.items())))
