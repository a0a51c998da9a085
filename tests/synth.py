"""TEST FIXTURE (not product code): synthetic, structure-faithful KKT / linearization inputs (there is no Pinocchio here to linearise a real robot).

Recipes follow the reference's own test factories with FIXED seeds:
  robotoc/test/test_helper/kkt_factory.cpp:7-64        (CreateSplitKKTMatrix / Residual)
  robotoc/test/riccati/riccati_factorizer_test.cpp:131-140 (switching-constraint blocks)
  robotoc/test/riccati/unconstr_riccati_recursion_test.cpp:33-46 (unconstrained horizon)
"Random" is U(-1,1) like Eigen::Random.  Documented deviation (SURVEY.md 8d): the velocity rows of Fxx are
`Fvq = dt*R, Fvv = I + dt*R, Fvu = dt*R` and the floating-base 6x6 blocks are `I + dt*R` / `dt*(I+R)`, which is the
structure condensing produces (contact_dynamics.cpp:130-134, state_equation.cpp:80-82) and keeps a 40-90 step
recursion well conditioned; `contractive=False` gives the raw unit-scale factory blocks.
"""
import numpy as np

from robotoc_b200.grid import IMPACT, TERMINAL
from robotoc_b200.layout import Dims, Layout, ULayout
from robotoc_b200.stage import StageDims, StageLayout


def _u(rng, *shape):
    return rng.uniform(-1.0, 1.0, size=shape)


def _sel(ns, nu):
    """[I_ns | 0] (ns x nu).  The switching-constraint Jacobian w.r.t. the controls is `selection + 0.3 * U(-1,1)` instead of
    the plain U(-1,1) block of riccati_factorizer_test.cpp:131-140: a random square 12 x 12 block has cond ~ 1e3..1e4, so the
    Schur complement Phiu G^-1 Phiu^T loses ~8 digits on a few instances of a 512-OCP batch (measured with the oracle itself:
    a 1e-15 relative input perturbation moved its s by 1e-4 there) and no implementation-independent comparison is possible;
    a contact Jacobian's actuated block is made of well-conditioned 3 x 3 leg Jacobians."""
    return np.eye(ns, nu)[None]


def _put(rec, off, block):
    """Store a batch of column-major blocks: block[b, i, j] -> rec[b, off + i + j*rows]."""
    b = block.shape[0]
    if block.ndim == 2:
        rec[:, off:off + block.shape[1]] = block
    else:
        rec[:, off:off + block.shape[1] * block.shape[2]] = np.transpose(block, (0, 2, 1)).reshape(b, -1)


def make_kkt(dims: Dims, L: Layout, ctrl, batch: int, seed: int, contractive: bool = True):
    """Returns kkt[batch, n_grid, k_stride] (float64, C-contiguous) and dx0[batch, nx]."""
    rng = np.random.default_rng(seed)
    n_grid = len(ctrl)
    nv, nu, nx = dims.nv, dims.nu, dims.nx
    kkt = np.zeros((batch, n_grid, L.k_stride))
    fb = dims.n_passive == 6
    eye = np.eye(nv)[None]
    for i in range(n_grid):
        c = ctrl[i]
        rec = kkt[:, i, :]
        if c.type == TERMINAL:
            S = _u(rng, batch, nx, nx)
            _put(rec, L.k_Qxx, S @ np.transpose(S, (0, 2, 1)))
            _put(rec, L.k_lx, _u(rng, batch, nx))
            continue
        dt = c.dt if c.dt > 0 else 0.0
        sc = dt if contractive else 1.0
        Fxx = np.zeros((batch, nx, nx))
        Fqq = np.repeat(eye, batch, 0).copy()
        if c.type == IMPACT:
            Fqv = np.zeros((batch, nv, nv))
            if fb:
                R = _u(rng, batch, 6, 6)
                Fqq[:, :6, :6] = (np.eye(6)[None] + 0.02 * R) if contractive else R
            Fvq = _u(rng, batch, nv, nv) * (0.05 if contractive else 1.0)
            Fvv = _u(rng, batch, nv, nv) * (0.05 if contractive else 1.0) + (eye if contractive else 0.0)
        else:
            Fqv = np.repeat(dt * eye, batch, 0).copy()
            if fb:
                R1, R2 = _u(rng, batch, 6, 6), _u(rng, batch, 6, 6)
                Fqq[:, :6, :6] = (np.eye(6)[None] + dt * R1) if contractive else R1
                Fqv[:, :6, :6] = (dt * (np.eye(6)[None] + 0.5 * R2)) if contractive else R2
            Fvq = sc * _u(rng, batch, nv, nv)
            Fvv = sc * _u(rng, batch, nv, nv) + (eye if contractive else 0.0)
        Fxx[:, :nv, :nv], Fxx[:, :nv, nv:], Fxx[:, nv:, :nv], Fxx[:, nv:, nv:] = Fqq, Fqv, Fvq, Fvv
        _put(rec, L.k_Fxx, Fxx)
        _put(rec, L.k_Fx, _u(rng, batch, nx))
        _put(rec, L.k_lx, _u(rng, batch, nx))
        if c.type == IMPACT:
            S = _u(rng, batch, nx, nx)
            _put(rec, L.k_Qxx, S @ np.transpose(S, (0, 2, 1)))
        else:
            _put(rec, L.k_Fvu, sc * _u(rng, batch, nv, nu))
            Hs = _u(rng, batch, nx + nu, nx + nu)
            H = Hs @ np.transpose(Hs, (0, 2, 1))
            _put(rec, L.k_Qxx, H[:, :nx, :nx])
            _put(rec, L.k_Qxu, H[:, :nx, nx:])
            _put(rec, L.k_Quu, H[:, nx:, nx:])
            _put(rec, L.k_lu, _u(rng, batch, nu))
            if c.ns > 0:
                _put(rec, L.k_Phix, _u(rng, batch, c.ns, nx))
                _put(rec, L.k_Phiu, _sel(c.ns, nu) + 0.3 * _u(rng, batch, c.ns, nu))
                _put(rec, L.k_p, _u(rng, batch, c.ns))
            if c.sto:
                ng = max(c.ngrids_in_phase, 1)
                _put(rec, L.k_fx, _u(rng, batch, nx) / ng)
                _put(rec, L.k_hx, _u(rng, batch, nx) / ng)
                _put(rec, L.k_hu, _u(rng, batch, nu) / ng)
                if c.ns > 0:
                    _put(rec, L.k_Phit, _u(rng, batch, c.ns) / ng)
                qtt = rng.uniform(0.5, 1.5, size=batch) / (ng * ng) + 1.0
                rec[:, L.k_sc + 0] = qtt
                rec[:, L.k_sc + 1] = -qtt          # intermediate_stage.cpp:145
                rec[:, L.k_sc + 2] = _u(rng, batch) / ng
    dx0 = _u(rng, batch, nx)
    return np.ascontiguousarray(kkt), np.ascontiguousarray(dx0)


def make_unconstr_kkt(nv: int, UL: ULayout, N: int, batch: int, seed: int):
    """unconstr_riccati_recursion_test.cpp:33-46: [Qxx Qxu; . Qaa] = G G^T, G in U(-1,1)^{3nv x 3nv}; Fx,lx,la random."""
    rng = np.random.default_rng(seed)
    nx = 2 * nv
    kkt = np.zeros((batch, N + 1, UL.k_stride))
    for i in range(N + 1):
        rec = kkt[:, i, :]
        Gs = _u(rng, batch, 3 * nv, 3 * nv)
        H = Gs @ np.transpose(Gs, (0, 2, 1))
        _put(rec, UL.k_Qxx, H[:, :nx, :nx])
        _put(rec, UL.k_lx, _u(rng, batch, nx))
        if i < N:
            _put(rec, UL.k_Qxu, H[:, :nx, nx:])
            _put(rec, UL.k_Qaa, H[:, nx:, nx:])
            _put(rec, UL.k_Fx, _u(rng, batch, nx))
            _put(rec, UL.k_la, _u(rng, batch, nv))
    dx0 = _u(rng, batch, nx)
    return np.ascontiguousarray(kkt), np.ascontiguousarray(dx0)


def mat(rec, off, rows, cols):
    """View helper: column-major block at `off` of a single record -> (rows, cols) array."""
    return rec[off:off + rows * cols].reshape(cols, rows).T


# ---- stage layer (linearization / PDIPM / solution records) -------------------------------------------------------
def _putm(rec, off, block, ld):
    """block[b, i, j] -> rec[b, off + i + j*ld] (column-major with leading dimension ld)."""
    b, m, n = block.shape
    view = rec[:, off:off + ld * n].reshape(b, n, ld)
    view[:, :, :m] = np.transpose(block, (0, 2, 1))


def make_stage_inputs(sd: StageDims, S: StageLayout, ctrl, batch: int, seed: int, impact_cones: bool = False):
    """Synthetic linearization / PDIPM / solution records (there is no Pinocchio here).  Structure follows what the
    reference's linearize* halves produce: M SPD (joint-space inertia), J a contact Jacobian, diagonal Qaa, friction-cone
    Jacobians per active contact, SE(3) blocks [[A,B],[0,D]] (se3_jacobian_inverse.hxx), slack/dual > 0.
    impact_cones: also the ImpactFrictionCone rows of Impact stages (drawn from a second generator, so the other records do
    not depend on the switch)."""
    rng = np.random.default_rng(seed)
    d = sd.dims
    nv, nu, nx, np_, nfm, nvfm = d.nv, d.nu, d.nx, d.n_passive, sd.nf_max, d.nv + sd.nf_max
    n_grid = len(ctrl)
    lin = np.zeros((batch, n_grid, S.l_stride))
    con = np.zeros((batch, n_grid, S.c_stride))
    sol = np.zeros((batch, n_grid, S.s_stride))
    for i in range(n_grid):
        c = ctrl[i]
        rec = lin[:, i, :]
        Ss = _u(rng, batch, nx, nx)
        _putm(rec, S.l_Qxx, Ss @ np.transpose(Ss, (0, 2, 1)) / nx + np.eye(nx)[None], nx)
        rec[:, S.l_lx:S.l_lx + nx] = _u(rng, batch, nx)
        if np_ == 6:
            for k in range(3):
                blk = np.zeros((batch, 6, 6))
                blk[:, :3, :3] = np.eye(3) + 0.1 * _u(rng, batch, 3, 3)
                blk[:, 3:, 3:] = np.eye(3) + 0.1 * _u(rng, batch, 3, 3)
                blk[:, :3, 3:] = 0.1 * _u(rng, batch, 3, 3)
                if k == 0:
                    blk = -blk  # dSubtract/dqf ~ -I near q_next ~ q
                _putm(rec, S.l_se3 + 36 * k, blk, 6)
        # solution (all stages)
        q = _u(rng, batch, S.nq)
        if np_ == 6:
            quat = _u(rng, batch, 4)
            q[:, 3:7] = quat / np.linalg.norm(quat, axis=1, keepdims=True)
        sol[:, i, S.s_q:S.s_q + S.nq] = q
        for off, n in ((S.s_v, nv), (S.s_a, nv), (S.s_dv, nv), (S.s_u, nu), (S.s_f, nfm), (S.s_lmd, nv), (S.s_gmm, nv),
                       (S.s_beta, nv), (S.s_mu, nfm), (S.s_nup, np_), (S.s_xi, S.nsm)):
            sol[:, i, off:off + n] = _u(rng, batch, n)
        if c.type == TERMINAL:
            continue
        impact = c.type == IMPACT
        nf = c.nf
        Sm = _u(rng, batch, nv, nv)
        _putm(rec, S.l_M, np.eye(nv)[None] + 0.1 * Sm @ np.transpose(Sm, (0, 2, 1)), nv)
        if nf > 0:
            Jimp = _u(rng, batch, nf, nv)
            _putm(rec, S.l_J, Jimp, nfm)
        D = 0.5 * _u(rng, batch, nv + nf, nx)
        if impact:
            D[:, :nv, nv:] = 0.0  # dIDdv does not exist on an impact stage (impact_dynamics.cpp:44-52)
            if nf > 0:            # ... and the Jacobian of MJtJinv IS the dCdv block of dIDCdqv there (impact_dynamics.cpp:40)
                D[:, nv:nv + nf, nv:] = Jimp
        _putm(rec, S.l_D, D, nvfm)
        rec[:, S.l_IDC:S.l_IDC + nv + nf] = 0.5 * _u(rng, batch, nv + nf)
        rec[:, S.l_Qaa:S.l_Qaa + nv] = rng.uniform(0.01, 1.0, size=(batch, nv))
        if nf > 0:
            _putm(rec, S.l_Qff, np.repeat(1e-3 * np.eye(nf)[None], batch, 0), nfm)
        rec[:, S.l_la:S.l_la + nv] = _u(rng, batch, nv)
        rec[:, S.l_lf:S.l_lf + nf] = _u(rng, batch, nf)
        rec[:, S.l_Fx:S.l_Fx + nx] = 0.1 * _u(rng, batch, nx)
        if not impact:
            Su = _u(rng, batch, nu, nu)
            _putm(rec, S.l_Quu, Su @ np.transpose(Su, (0, 2, 1)) / nu + 0.1 * np.eye(nu)[None], nu)
            rec[:, S.l_lu:S.l_lu + nu] = _u(rng, batch, nu)
            rec[:, S.l_lup:S.l_lup + np_] = _u(rng, batch, np_)
            if c.ns > 0:
                _putm(rec, S.l_Phix, _u(rng, batch, c.ns, nx), c.ns)
                Phia = _u(rng, batch, c.ns, nv)
                Phia[:, :, nv - nu:] = _sel(c.ns, nu) + 0.3 * Phia[:, :, nv - nu:]   # leg-Jacobian-like actuated block
                _putm(rec, S.l_Phia, Phia, c.ns)
                rec[:, S.l_p:S.l_p + c.ns] = _u(rng, batch, c.ns)
                rec[:, S.l_Phit:S.l_Phit + c.ns] = _u(rng, batch, c.ns)
            rec[:, S.l_ha:S.l_ha + nv] = _u(rng, batch, nv)
            rec[:, S.l_hf:S.l_hf + nf] = _u(rng, batch, nf)
            rec[:, S.l_hx:S.l_hx + nx] = _u(rng, batch, nx)
            rec[:, S.l_hu:S.l_hu + nu] = _u(rng, batch, nu)
            rec[:, S.l_fx:S.l_fx + nx] = _u(rng, batch, nx)
            rec[:, S.l_sc + 0] = _u(rng, batch)
            rec[:, S.l_sc + 1] = rng.uniform(0.5, 1.5, size=batch)
            for ci in range(sd.n_contacts):
                if (c.contact_mask >> ci) & 1:
                    _putm(rec, S.l_dgdq + ci * 5 * nv, 0.3 * _u(rng, batch, 5, nv), 5)
                    _putm(rec, S.l_dgdf + ci * 15, _u(rng, batch, 5, 3), 5)
            nc = S.nc
            con[:, i, S.c_slack:S.c_slack + nc] = rng.uniform(0.01, 1.0, size=(batch, nc))
            con[:, i, S.c_dual:S.c_dual + nc] = rng.uniform(0.01, 1.0, size=(batch, nc))
            con[:, i, S.c_res:S.c_res + nc] = 0.1 * _u(rng, batch, nc)
    dx0 = 0.1 * _u(rng, batch, nx)
    if impact_cones:
        rng2 = np.random.default_rng(seed + 7919)
        for i in range(n_grid):
            c = ctrl[i]
            if c.type != IMPACT:
                continue
            rec = lin[:, i]
            for ci in range(sd.n_contacts):
                if (c.contact_mask >> ci) & 1:
                    _putm(rec, S.l_dgdq + ci * 5 * nv, 0.3 * _u(rng2, batch, 5, nv), 5)
                    _putm(rec, S.l_dgdf + ci * 15, _u(rng2, batch, 5, 3), 5)
            o0, o1 = S.nbox, S.nc
            con[:, i, S.c_slack + o0:S.c_slack + o1] = rng2.uniform(0.01, 1.0, size=(batch, o1 - o0))
            con[:, i, S.c_dual + o0:S.c_dual + o1] = rng2.uniform(0.01, 1.0, size=(batch, o1 - o0))
            con[:, i, S.c_res + o0:S.c_res + o1] = 0.1 * _u(rng2, batch, o1 - o0)
    return np.ascontiguousarray(lin), np.ascontiguousarray(con), np.ascontiguousarray(sol), np.ascontiguousarray(dx0)


def symmetrize_lin(S: StageLayout, lin):
    """Brings linearization records to what the reference's containers hold when the hot path starts, which is what the host
    wire format assumes: the symmetric blocks exactly symmetric (upper triangle authoritative; cost Hessians, joint-space
    inertia) and Qqf = 0 (no cost writes it: it is filled by the friction-cone condensing, friction_cone.cpp:219)."""
    out = lin.copy()
    flat = out.reshape(-1, out.shape[-1])
    flat[:, S.l_Qqf:S.l_Qxx] = 0.0
    for off, n in ((S.l_M, S.nv), (S.l_Qff, S.nfm), (S.l_Qxx, S.nx), (S.l_Quu, S.nu)):
        blk = flat[:, off:off + n * n].reshape(-1, n, n)  # [rec, col, row] (column-major)
        a = np.transpose(blk, (0, 2, 1))                  # a[rec, row, col]
        up = np.triu(a)
        sym = up + np.transpose(np.triu(a, 1), (0, 2, 1))
        flat[:, off:off + n * n] = np.transpose(sym, (0, 2, 1)).reshape(-1, n * n)
    return out


def robotoc_cost_structure(S: StageLayout, lin):
    """Cost Hessians as every cost component robotoc ships produces them (configuration_space_cost.cpp:308-322,
    task_space_*_cost.cpp, com_cost.cpp, local_contact_force_cost.cpp:130): Qqq dense, Qvv / Quu / Qff diagonal, Qqv = 0 (and
    Qqf = 0, symmetric blocks exactly symmetric, like symmetrize_lin)."""
    out = symmetrize_lin(S, lin)
    flat = out.reshape(-1, out.shape[-1])
    nv, nx = S.nv, S.nx
    Q = flat[:, S.l_Qxx:S.l_Qxx + nx * nx].reshape(-1, nx, nx)   # [rec, col, row]
    dv = np.einsum("rii->ri", Q[:, nv:, nv:]).copy()
    Q[:, nv:, :] = 0.0
    Q[:, :, nv:] = 0.0
    for k in range(nv):
        Q[:, nv + k, nv + k] = dv[:, k]
    for off, n in ((S.l_Quu, S.nu), (S.l_Qff, S.nfm)):
        B = flat[:, off:off + n * n].reshape(-1, n, n)
        d = np.einsum("rii->ri", B).copy()
        B[:] = 0.0
        for k in range(n):
            B[:, k, k] = d[:, k]
    return out


def make_unconstr_stage_inputs(S, N: int, batch: int, seed: int):
    """Synthetic linearization / PDIPM / solution records (no Pinocchio here): dID_da = M SPD, dense dID_dq / dID_dv,
    diagonal cost Hessians as ConfigurationSpaceCost produces them, slack / dual > 0."""
    rng = np.random.default_rng(seed)
    nv, nx = S.nv, S.nx
    u = lambda *shape: rng.uniform(-1.0, 1.0, size=shape)  # noqa: E731
    lin = np.zeros((batch, N + 1, S.l_stride))
    con = np.zeros((batch, N + 1, S.c_stride))
    sol = np.zeros((batch, N + 1, S.s_stride))

    def putm(rec, off, block):  # block[b, i, j] -> column-major
        b, m, n = block.shape
        rec[:, off:off + m * n] = np.transpose(block, (0, 2, 1)).reshape(b, m * n)

    for i in range(N + 1):
        rec = lin[:, i, :]
        Qxx = np.zeros((batch, nx, nx))
        Qxx[:, np.arange(nx), np.arange(nx)] = rng.uniform(0.01, 10.0, size=(batch, nx))
        if i % 3 == 0:  # a dense symmetric part (task-space costs)
            T = u(batch, nx, nx)
            Qxx += 0.05 * T @ np.transpose(T, (0, 2, 1))
        putm(rec, S.l_Qxx, Qxx)
        rec[:, S.l_lx:S.l_lx + nx] = u(batch, nx)
        for off in (S.s_q, S.s_v, S.s_a, S.s_u, S.s_beta, S.s_lmd, S.s_gmm):
            sol[:, i, off:off + nv] = u(batch, nv)
        if i == N:
            continue
        Sm = u(batch, nv, nv)
        putm(rec, S.l_dIDda, np.eye(nv)[None] + 0.2 * Sm @ np.transpose(Sm, (0, 2, 1)))
        putm(rec, S.l_dIDdq, u(batch, nv, nv))
        putm(rec, S.l_dIDdv, 0.3 * u(batch, nv, nv))
        rec[:, S.l_ID:S.l_ID + nv] = 0.5 * u(batch, nv)
        Qaa = np.zeros((batch, nv, nv))
        Qaa[:, np.arange(nv), np.arange(nv)] = rng.uniform(0.01, 1.0, size=(batch, nv))
        putm(rec, S.l_Qaa, Qaa)
        Quu = np.zeros((batch, nv, nv))
        Quu[:, np.arange(nv), np.arange(nv)] = rng.uniform(0.01, 1.0, size=(batch, nv))
        putm(rec, S.l_Quu, Quu)
        rec[:, S.l_la:S.l_la + nv] = u(batch, nv)
        rec[:, S.l_lu:S.l_lu + nv] = u(batch, nv)
        rec[:, S.l_Fx:S.l_Fx + nx] = 0.1 * u(batch, nx)
        nb = S.nbox
        con[:, i, S.c_slack:S.c_slack + nb] = rng.uniform(0.01, 1.0, size=(batch, nb))
        con[:, i, S.c_dual:S.c_dual + nb] = rng.uniform(0.01, 1.0, size=(batch, nb))
        con[:, i, S.c_res:S.c_res + nb] = 0.1 * u(batch, nb)
    dx0 = 0.1 * u(batch, nx)
    return np.ascontiguousarray(lin), np.ascontiguousarray(con), np.ascontiguousarray(sol), np.ascontiguousarray(dx0)


def unconstr_table(rows, barrier=1.0e-3, fraction_to_boundary=0.995):
    """rbt_constraint_table for the unconstrained path (n_contacts = 0) with the box rows `rows` = [(var, idx, sign), ...], in
    that order."""
    from robotoc_b200.stage import rbt_constraint_table
    t = rbt_constraint_table()
    t.n_contacts = 0
    t.barrier, t.fraction_to_boundary = barrier, fraction_to_boundary
    for r, (var, idx, sign) in enumerate(rows):
        t.box[r].var, t.box[r].idx, t.box[r].sign = var, idx, sign
    t.n_box = len(rows)
    return t


def table_rows(tab):
    return [(tab.box[r].var, tab.box[r].idx, tab.box[r].sign) for r in range(tab.n_box)]


def iiwa14_rows(nv=7, acceleration_limits=False):
    """Box rows of examples/iiwa14/unconstr_ocp_benchmark.cpp:45-60 in component order (joint position, velocity, torque
    lower / upper limits), optionally followed by JointAccelerationLowerLimit / UpperLimit: what the reference can express."""
    from robotoc_b200.stage import VAR_A, VAR_Q, VAR_U, VAR_V
    vs = (VAR_Q, VAR_V, VAR_U) + ((VAR_A,) if acceleration_limits else ())
    return [(var, j, sign) for var in vs for sign in (-1, +1) for j in range(nv)]


def bind_unconstr_rows(S, con, binds, R=(100.0, 50.0)):
    """Makes chosen rows the binding rows of the fraction-to-boundary rule.  binds: [(b, i, r, kind)], kind "p" (primal: the
    Newton step drives the slack of row r on grid point i of OCP b far below zero) or "d" (dual: the slack grows by far more
    than it is, which drives the dual below zero).  slack = dual = 1e-4 keeps the row's barrier weight near the cost
    curvature, so the condensed step cannot satisfy the linearised row; the residual R sets how far it misses."""
    con = con.copy()
    for b, i, r, kind in binds:
        con[b, i, S.c_slack + r] = 1.0e-4
        con[b, i, S.c_dual + r] = 1.0e-4
        con[b, i, S.c_res + r] = R[0] if kind == "p" else -R[1]
    return con
