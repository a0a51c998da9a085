"""numpy restatement of Pinocchio's RNEA (pinocchio::rnea with external forces) and of its derivatives, in spatial algebra with
Pinocchio's conventions: motion = [linear | angular], force = [linear | angular], body quantities in the joint frames,
liMi = jointPlacement * M_J(q), free flyer q = [p | quaternion xyzw] with integrate(q, dq) = M exp6(dq).

The model is the dict of tests/golden/anymal_model.npz (fields of rbt_robot_model).  Everything is vectorised over a leading
batch axis.  The derivatives are forward-mode: one tangent per direction (nv in q, nv in v, nv in a), propagated through the
same recursion with 6x6 matrices; tests/test_rnea.py checks them against central differences and physical identities."""
import numpy as np


def skew(x):
    x = np.asarray(x)
    z = np.zeros(x.shape[:-1])
    return np.stack([np.stack([z, -x[..., 2], x[..., 1]], -1), np.stack([x[..., 2], z, -x[..., 0]], -1),
                     np.stack([-x[..., 1], x[..., 0], z], -1)], -2)


def crm(v):  # v x m  as a 6x6 matrix
    out = np.zeros(v.shape[:-1] + (6, 6))
    W, V = skew(v[..., 3:]), skew(v[..., :3])
    out[..., :3, :3] = W
    out[..., :3, 3:] = V
    out[..., 3:, 3:] = W
    return out


def crf(v):  # v x* f  as a 6x6 matrix
    return -np.swapaxes(crm(v), -1, -2)


def quat_to_rot(x, y, z, w):
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], -1),
                     np.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], -1),
                     np.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1)], -2)


def axis_rot(u, th):  # Rodrigues, batch of angles th [B]
    K = skew(np.asarray(u, dtype=float))
    th = th[..., None, None]
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * (K @ K)


def xinv_motion(R, p):  # 6x6 of SE3::actInv on a motion
    Rt = np.swapaxes(R, -1, -2)
    out = np.zeros(R.shape[:-2] + (6, 6))
    out[..., :3, :3] = Rt
    out[..., :3, 3:] = -Rt @ skew(p)
    out[..., 3:, 3:] = Rt
    return out


def inertia6(mass, com, Ic):
    C = skew(np.asarray(com, dtype=float))
    out = np.zeros((6, 6))
    out[:3, :3] = mass * np.eye(3)
    out[:3, 3:] = -mass * C
    out[3:, :3] = mass * C
    out[3:, 3:] = Ic - mass * C @ C
    return out


def n_bodies(model):
    return int(model["n_bodies"])


def _R(pl):
    return np.asarray(pl[:9], dtype=float).reshape(3, 3).T  # column-major storage


def joint_transforms(model, q):
    """liMi of every body: lists of R [B,3,3], p [B,3]."""
    B = q.shape[0]
    Rs, ps = [], []
    for b in range(n_bodies(model)):
        RP, pP = _R(model["placement"][b]), np.asarray(model["placement"][b][9:12], dtype=float)
        if b == 0:
            RJ, pJ = quat_to_rot(q[:, 3], q[:, 4], q[:, 5], q[:, 6]), q[:, :3]
        else:
            RJ, pJ = axis_rot(model["axis"][b], q[:, b + 6]), np.zeros((B, 3))
        Rs.append(RP @ RJ)
        ps.append(pP + pJ @ RP.T)
    return Rs, ps


def subspace(model, b):
    if b == 0:
        return np.eye(6)
    S = np.zeros((6, 1))
    S[3:, 0] = model["axis"][b]
    return S


def dofs(b):
    return slice(0, 6) if b == 0 else slice(b + 5, b + 6)


def contact_fext(model, f, mask):
    """Robot::setContactForces: fext[parent] = jXf.act(Force(f_c, 0)) per contact in order (zero if inactive)."""
    B = f.shape[0]
    fx = np.zeros((n_bodies(model), B, 6))
    k = 0
    for c in range(int(model["n_contacts"])):
        par = int(model["contact_parent"][c])
        if (mask >> c) & 1:
            R, p = _R(model["contact_placement"][c]), np.asarray(model["contact_placement"][c][9:12], dtype=float)
            lin = f[:, k:k + 3] @ R.T
            fx[par] = np.concatenate([lin, np.cross(p, lin)], -1)
            k += 3
        else:
            fx[par] = 0.0
    return fx


def rnea(model, q, v, a, fext=None, gravity=True, tangents=None):
    """tau = RNEA(q, v, a, fext) [B, nv]; with tangents = (Tq, Tv, Ta) [D, nv] each, also the directional derivatives
    dtau [B, D, nv]."""
    B, nv = q.shape[0], v.shape[1]
    nb = n_bodies(model)
    Rs, ps = joint_transforms(model, q)
    Xi = [xinv_motion(Rs[b], ps[b]) for b in range(nb)]
    I6 = [inertia6(model["mass"][b], model["com"][b], np.asarray(model["inertia"][b], dtype=float).reshape(3, 3).T) for b in range(nb)]
    ag = np.zeros((B, 6))
    if gravity:
        ag[:, :3] = -np.asarray(model["gravity"], dtype=float)
    D = 0 if tangents is None else tangents[0].shape[0]
    Tq, Tv, Ta = tangents if tangents is not None else (np.zeros((0, nv)),) * 3
    V, A, F = [None] * nb, [None] * nb, [None] * nb
    dV, dA, dF = [None] * nb, [None] * nb, [None] * nb
    delta = [None] * nb
    for b in range(nb):
        pa = int(model["parent"][b])
        S, sl = subspace(model, b), dofs(b)
        vJ = v[:, sl] @ S.T
        dvJ = Tv[:, sl] @ S.T                      # [D, 6]
        delta[b] = Tq[:, sl] @ S.T                 # perturbation twist of this joint per direction
        vp = np.zeros((B, 6)) if pa < 0 else V[pa]
        ap = ag if pa < 0 else A[pa]
        wv = np.einsum("bij,bj->bi", Xi[b], vp)
        wa = np.einsum("bij,bj->bi", Xi[b], ap)
        V[b] = wv + vJ
        A[b] = wa + a[:, sl] @ S.T + np.einsum("bij,bj->bi", crm(V[b]), vJ)
        F[b] = A[b] @ I6[b].T + np.einsum("bij,bj->bi", crf(V[b]), V[b] @ I6[b].T)
        if fext is not None:
            F[b] = F[b] - fext[b]
        if D:
            dvp = np.zeros((B, D, 6)) if pa < 0 else dV[pa]
            dap = np.zeros((B, D, 6)) if pa < 0 else dA[pa]
            dV[b] = (np.einsum("bij,bdj->bdi", Xi[b], dvp) + np.einsum("bij,dj->bdi", crm(wv), delta[b]) + dvJ[None])
            dA[b] = (np.einsum("bij,bdj->bdi", Xi[b], dap) + np.einsum("bij,dj->bdi", crm(wa), delta[b]) + (Ta[:, sl] @ S.T)[None]
                     + np.einsum("bdij,bj->bdi", crm(dV[b]), vJ) + np.einsum("bij,dj->bdi", crm(V[b]), dvJ))
            dF[b] = (dA[b] @ I6[b].T + np.einsum("bdij,bj->bdi", crf(dV[b]), V[b] @ I6[b].T)
                     + np.einsum("bij,bdj->bdi", crf(V[b]), dV[b] @ I6[b].T))
    tau = np.zeros((B, nv))
    dtau = np.zeros((B, D, nv))
    for b in range(nb - 1, -1, -1):
        pa = int(model["parent"][b])
        S, sl = subspace(model, b), dofs(b)
        tau[:, sl] = F[b] @ S
        if D:
            dtau[:, :, sl] = dF[b] @ S
        if pa >= 0:
            Xf = np.swapaxes(Xi[b], -1, -2)  # SE3::act on a force = (actInv on a motion)^T
            F[pa] = F[pa] + np.einsum("bij,bj->bi", Xf, F[b])
            if D:
                dF[pa] = dF[pa] + np.einsum("bij,bdj->bdi", Xf, dF[b] + np.einsum("dij,bj->bdi", crf(delta[b]), F[b]))
    return (tau, dtau) if tangents is not None else tau


def rnea_derivatives(model, q, v, a, fext=None, gravity=True):
    """(tau, dtau/dq, dtau/dv, dtau/da) with dtau/da symmetrised from its upper triangle (Robot::RNEADerivatives)."""
    nv = v.shape[1]
    E, Z = np.eye(nv), np.zeros((nv, nv))
    T = (np.concatenate([E, Z, Z]), np.concatenate([Z, E, Z]), np.concatenate([Z, Z, E]))
    tau, dt = rnea(model, q, v, a, fext, gravity, T)
    dq, dv, M = [np.swapaxes(dt[:, k * nv:(k + 1) * nv], 1, 2) for k in range(3)]
    M = np.triu(M) + np.swapaxes(np.triu(M, 1), 1, 2)
    return tau, dq, dv, M


def integrate(q, dq):
    """Robot::integrateConfiguration for the free flyer + revolute joints: q (+) dq (pinocchio::integrate)."""
    q = q.copy()
    v, w = dq[:, :3], dq[:, 3:6]
    th = np.linalg.norm(w, axis=1)
    Rw = np.stack([axis_rot(w[i] / th[i] if th[i] > 0 else np.array([1.0, 0, 0]), th[i:i + 1])[0] for i in range(q.shape[0])])
    K = skew(w)
    th2 = np.where(th > 1e-12, th, 1.0)[:, None, None]
    Vm = (np.eye(3) + ((1 - np.cos(th2)) / th2 ** 2) * K + ((th2 - np.sin(th2)) / th2 ** 3) * (K @ K))
    Vm = np.where(th[:, None, None] > 1e-12, Vm, np.eye(3) + 0.5 * K)
    R0 = quat_to_rot(q[:, 3], q[:, 4], q[:, 5], q[:, 6])
    q[:, :3] += np.einsum("bij,bj->bi", R0, np.einsum("bij,bj->bi", Vm, v))
    R1 = R0 @ Rw
    q[:, 3:7] = rot_to_quat(R1, q[:, 3:7])
    q[:, 7:] += dq[:, 6:]
    return q


def rot_to_quat(R, ref):
    """Rotation matrices -> quaternions xyzw, sign chosen to agree with ref."""
    out = np.zeros((R.shape[0], 4))
    for i in range(R.shape[0]):
        m = R[i]
        tr = np.trace(m)
        if tr > 0:
            s = 2 * np.sqrt(tr + 1)
            out[i] = [(m[2, 1] - m[1, 2]) / s, (m[0, 2] - m[2, 0]) / s, (m[1, 0] - m[0, 1]) / s, s / 4]
        else:
            k = int(np.argmax(np.diag(m)))
            i1, i2 = (k + 1) % 3, (k + 2) % 3
            s = 2 * np.sqrt(1 + m[k, k] - m[i1, i1] - m[i2, i2])
            qv = np.zeros(4)
            qv[k] = s / 4
            qv[i1] = (m[i1, k] + m[k, i1]) / s
            qv[i2] = (m[i2, k] + m[k, i2]) / s
            qv[3] = (m[i2, i1] - m[i1, i2]) / s
            out[i] = qv
        if np.dot(out[i], ref[i]) < 0:
            out[i] = -out[i]
    return out


def world_poses(model, q):
    Rs, ps = joint_transforms(model, q)
    oR, op = [None] * len(Rs), [None] * len(Rs)
    for b in range(len(Rs)):
        pa = int(model["parent"][b])
        if pa < 0:
            oR[b], op[b] = Rs[b], ps[b]
        else:
            oR[b] = oR[pa] @ Rs[b]
            op[b] = op[pa] + np.einsum("bij,bj->bi", oR[pa], ps[b])
    return oR, op


def body_velocities(model, q, v):
    Rs, ps = joint_transforms(model, q)
    V = []
    for b in range(n_bodies(model)):
        pa = int(model["parent"][b])
        vJ = v[:, dofs(b)] @ subspace(model, b).T
        V.append(vJ if pa < 0 else np.einsum("bij,bj->bi", xinv_motion(Rs[b], ps[b]), V[pa]) + vJ)
    return V


def kinetic_energy(model, q, v):
    V = body_velocities(model, q, v)
    I6 = [inertia6(model["mass"][b], model["com"][b], np.asarray(model["inertia"][b]).reshape(3, 3).T) for b in range(n_bodies(model))]
    return sum(0.5 * np.einsum("bi,ij,bj->b", V[b], I6[b], V[b]) for b in range(n_bodies(model)))


def potential_energy(model, q):
    oR, op = world_poses(model, q)
    g = np.asarray(model["gravity"], dtype=float)
    return sum(-model["mass"][b] * ((op[b] + np.einsum("bij,j->bi", oR[b], np.asarray(model["com"][b]))) @ g) for b in range(n_bodies(model)))


def contact_jacobian(model, q, c):
    """Linear velocity of contact frame c in its own frame per unit generalized velocity: [B, 3, nv]."""
    nv = int(model["nv"])
    B = q.shape[0]
    R, p = _R(model["contact_placement"][c]), np.asarray(model["contact_placement"][c][9:12], dtype=float)
    X = xinv_motion(R[None], p[None])[0]
    J = np.zeros((B, 3, nv))
    for k in range(nv):
        e = np.zeros((B, nv))
        e[:, k] = 1.0
        vb = body_velocities(model, q, e)[int(model["contact_parent"][c])]
        J[:, :, k] = (vb @ X.T)[:, :3]
    return J


def random_rotation(rng):
    Q, R = np.linalg.qr(rng.standard_normal((3, 3)))
    Q = Q * np.sign(np.diag(R))
    return Q if np.linalg.det(Q) > 0 else -Q


def random_model(seed, nv=18, n_contacts=4):
    """Seeded random floating-base tree of revolute joints with the field layout of rbt_robot_model."""
    rng = np.random.default_rng(seed)
    nb = nv - 5
    m = {"nv": nv, "n_bodies": nb, "n_contacts": n_contacts}
    m["parent"] = np.array([-1] + [int(rng.integers(0, b)) for b in range(1, nb)])
    ax = rng.standard_normal((nb, 3))
    m["axis"] = ax / np.linalg.norm(ax, axis=1, keepdims=True)
    pl = np.zeros((nb, 12))
    for b in range(nb):
        R = np.eye(3) if b == 0 else random_rotation(rng)
        pl[b, :9] = R.T.reshape(-1)
        pl[b, 9:] = 0.0 if b == 0 else rng.uniform(-0.4, 0.4, 3)
    m["placement"] = pl
    m["mass"] = rng.uniform(0.5, 5.0, nb)
    m["com"] = rng.uniform(-0.2, 0.2, (nb, 3))
    I = np.zeros((nb, 9))
    for b in range(nb):
        A = rng.standard_normal((3, 3)) * 0.1
        I[b] = (A @ A.T + 0.02 * np.eye(3)).T.reshape(-1)
    m["inertia"] = I
    m["contact_parent"] = rng.choice(np.arange(1, nb), n_contacts, replace=False)
    cp = np.zeros((n_contacts, 12))
    for c in range(n_contacts):
        cp[c, :9] = random_rotation(rng).T.reshape(-1)
        cp[c, 9:] = rng.uniform(-0.3, 0.3, 3)
    m["contact_placement"] = cp
    m["gravity"] = np.array([0.0, 0.0, -9.81])
    return m


def random_state(rng, B, nv):
    q = rng.uniform(-1, 1, (B, nv + 1))
    qu = rng.standard_normal((B, 4))
    q[:, 3:7] = qu / np.linalg.norm(qu, axis=1, keepdims=True)
    return q, rng.uniform(-1, 1, (B, nv)), rng.uniform(-1, 1, (B, nv))


def to_c(model):
    """dict -> rbt_robot_model (ctypes)."""
    from robotoc_b200.dms import rbt_robot_model
    m = rbt_robot_model()
    m.nv, m.n_bodies, m.n_contacts = int(model["nv"]), int(model["n_bodies"]), int(model["n_contacts"])
    for b in range(m.n_bodies):
        m.parent[b] = int(model["parent"][b])
        m.mass[b] = float(model["mass"][b])
        for e in range(3):
            m.axis[b][e] = float(model["axis"][b][e])
            m.com[b][e] = float(model["com"][b][e])
        for e in range(12):
            m.placement[b][e] = float(model["placement"][b][e])
        for e in range(9):
            m.inertia[b][e] = float(model["inertia"][b][e])
    for c in range(m.n_contacts):
        m.contact_parent[c] = int(model["contact_parent"][c])
        for e in range(12):
            m.contact_placement[c][e] = float(model["contact_placement"][c][e])
    for e in range(3):
        m.gravity[e] = float(model["gravity"][e])
    return m


def linearize(model, S, ctrl, sol, lin):
    """What rbt_linearize_inverse_dynamics writes, for records [batch, n_grid, ...]: returns the updated linearization records."""
    from robotoc_b200.grid import IMPACT, TERMINAL
    l = lin.copy()
    nv, nvf = S.nv, S.nvf
    for i, c in enumerate(ctrl):
        if c.type == TERMINAL:
            continue
        impact = c.type == IMPACT
        s = sol[:, i]
        q, beta = s[:, S.s_q:S.s_q + S.nq], s[:, S.s_beta:S.s_beta + nv]
        v = np.zeros((s.shape[0], nv)) if impact else s[:, S.s_v:S.s_v + nv]
        a = s[:, (S.s_dv if impact else S.s_a):][:, :nv]
        fx = contact_fext(model, s[:, S.s_f:S.s_f + S.nfm], c.contact_mask)
        tau, dq, dv, M = rnea_derivatives(model, q, v, a, fx, gravity=not impact)
        if impact:
            dv = np.zeros_like(dv)
        else:
            tau[:, 6:] -= s[:, S.s_u:S.s_u + S.nu]
        r = l[:, i]
        r[:, S.l_IDC:S.l_IDC + nv] = tau
        D = r[:, S.l_D:S.l_D + nvf * 2 * nv].reshape(-1, 2 * nv, nvf).copy()   # column-major (ld nvf) -> [col][row]
        D[:, :nv, :nv] = np.swapaxes(dq, 1, 2)
        D[:, nv:, :nv] = np.swapaxes(dv, 1, 2)
        r[:, S.l_D:S.l_D + nvf * 2 * nv] = D.reshape(-1, 2 * nv * nvf)
        r[:, S.l_M:S.l_M + nv * nv] = np.swapaxes(M, 1, 2).reshape(-1, nv * nv)
        r[:, S.l_lx:S.l_lx + nv] += np.einsum("brk,br->bk", dq, beta)
        if not impact:
            r[:, S.l_lx + nv:S.l_lx + 2 * nv] += np.einsum("brk,br->bk", dv, beta)
        r[:, S.l_la:S.l_la + nv] += np.einsum("brk,br->bk", M, beta)
    return l
