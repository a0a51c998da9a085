"""numpy restatement of the contact rows of the contact / impact dynamics linearisation: Pinocchio's forwardKinematics (no
gravity) and the LOCAL velocity / classical acceleration of the point-contact frames, the Baumgarte residual and the impact
velocity residual of robotoc's PointContact (point_contact.hxx:16-117), and their derivatives.

Conventions as tests/rbd_ref.py: motion = [linear | angular], body quantities in the joint frames, q-derivatives in the tangent
space (q (+) dq = rbd_ref.integrate).  The derivatives are forward-mode: one tangent per direction (nv in q, nv in v) through the
same recursion with 6x6 matrices; tests/test_contact_kinematics.py checks them against central differences, against the
world-frame motion of the contact point and against the assembly Pinocchio's frame derivatives give."""
import numpy as np

import rbd_ref as R


def kinematics(model, q, v, a, tangents=None):
    """Body velocities V[b] and (spatial) accelerations A[b] [B, 6] without gravity; with tangents = (Tq, Tv) [D, nv], also
    their directional derivatives dV[b], dA[b] [B, D, 6]."""
    B, nv = q.shape[0], v.shape[1]
    nb = R.n_bodies(model)
    Rs, ps = R.joint_transforms(model, q)
    Tq, Tv = tangents if tangents is not None else (np.zeros((0, nv)), np.zeros((0, nv)))
    D = Tq.shape[0]
    V, A, dV, dA = [None] * nb, [None] * nb, [None] * nb, [None] * nb
    for b in range(nb):
        pa = int(model["parent"][b])
        S, sl = R.subspace(model, b), R.dofs(b)
        Xi = R.xinv_motion(Rs[b], ps[b])
        vJ, aJ = v[:, sl] @ S.T, a[:, sl] @ S.T
        dvJ, delta = Tv[:, sl] @ S.T, Tq[:, sl] @ S.T
        vp = np.zeros((B, 6)) if pa < 0 else V[pa]
        ap = np.zeros((B, 6)) if pa < 0 else A[pa]
        wv, wa = np.einsum("bij,bj->bi", Xi, vp), np.einsum("bij,bj->bi", Xi, ap)
        V[b] = wv + vJ
        A[b] = wa + aJ + np.einsum("bij,bj->bi", R.crm(V[b]), vJ)
        dvp = np.zeros((B, D, 6)) if pa < 0 else dV[pa]
        dap = np.zeros((B, D, 6)) if pa < 0 else dA[pa]
        dV[b] = np.einsum("bij,bdj->bdi", Xi, dvp) + np.einsum("bij,dj->bdi", R.crm(wv), delta) + dvJ[None]
        dA[b] = (np.einsum("bij,bdj->bdi", Xi, dap) + np.einsum("bij,dj->bdi", R.crm(wa), delta)
                 + np.einsum("bdij,bj->bdi", R.crm(dV[b]), vJ) + np.einsum("bij,dj->bdi", R.crm(V[b]), dvJ))
    return V, A, dV, dA


def _frame(model, c):
    Rf = R._R(model["contact_placement"][c])
    pf = np.asarray(model["contact_placement"][c][9:12], dtype=float)
    return Rf, pf, R.xinv_motion(Rf[None], pf[None])[0]


def frame_placement(model, q, c):
    """oMf of contact c: (oRf [B, 3, 3], o p_f [B, 3])."""
    oR, op = R.world_poses(model, q)
    par = int(model["contact_parent"][c])
    Rf, pf, _ = _frame(model, c)
    return oR[par] @ Rf, op[par] + np.einsum("bij,j->bi", oR[par], pf)


def frame_motion(model, q, v, a, c, tangents=None):
    """LOCAL spatial velocity and acceleration of contact frame c [B, 6] (and their tangents [B, D, 6])."""
    V, A, dV, dA = kinematics(model, q, v, a, tangents)
    par = int(model["contact_parent"][c])
    _, _, X = _frame(model, c)
    return V[par] @ X.T, A[par] @ X.T, dV[par] @ X.T, dA[par] @ X.T


def classical_acceleration(vf, af):
    """a_f,lin + w_f x v_f,lin (pinocchio::getFrameClassicalAcceleration, LOCAL)."""
    return af[..., :3] + np.cross(vf[..., 3:], vf[..., :3])


def baumgarte_residual(model, q, v, a, c, kp, kv, p_des):
    vf, af, _, _ = frame_motion(model, q, v, a, c)
    _, opf = frame_placement(model, q, c)
    return classical_acceleration(vf, af) + kv * vf[:, :3] + kp * (opf - p_des)


def impact_velocity_residual(model, q, v, c):
    vf, _, _, _ = frame_motion(model, q, v, np.zeros_like(v), c)
    return vf[:, :3]


def _tangents(nv):
    E, Z = np.eye(nv), np.zeros((nv, nv))
    return np.concatenate([E, Z]), np.concatenate([Z, E])


def baumgarte_derivatives(model, q, v, a, c, kp, kv):
    """(dC/dq, dC/dv, dC/da) [B, 3, nv] of the Baumgarte residual, forward mode."""
    nv = v.shape[1]
    vf, af, dvf, daf = frame_motion(model, q, v, a, c, _tangents(nv))
    oRf, _ = frame_placement(model, q, c)
    w, vl = vf[:, None, 3:], vf[:, None, :3]
    dC = daf[..., :3] + np.cross(w, dvf[..., :3]) + np.cross(dvf[..., 3:], vl) + kv * dvf[..., :3]   # [B, 2 nv, 3]
    J = np.swapaxes(dvf[:, nv:, :3], 1, 2)
    dCdq = np.swapaxes(dC[:, :nv], 1, 2) + kp * oRf @ J
    return dCdq, np.swapaxes(dC[:, nv:], 1, 2), J


def impact_velocity_derivatives(model, q, v, c):
    """(dC/dq, dC/dv) [B, 3, nv] of the impact velocity residual."""
    nv = v.shape[1]
    _, _, dvf, _ = frame_motion(model, q, v, np.zeros_like(v), c, _tangents(nv))
    return np.swapaxes(dvf[:, :nv, :3], 1, 2), np.swapaxes(dvf[:, nv:, :3], 1, 2)


def linearize(model, S, ctrl, sol, lin, gains, pos):
    """What rbt_linearize_contact_kinematics writes, for records [batch, n_grid, ...]; gains [n_contacts, 2], pos
    [batch, n_grid, n_contacts, 3]: returns the updated linearization records."""
    from robotoc_b200.grid import IMPACT, TERMINAL
    l = lin.copy()
    nv, nvf, nfm = S.nv, S.nvf, S.nfm
    for i, c in enumerate(ctrl):
        if c.type == TERMINAL or c.nf == 0:
            continue
        impact = c.type == IMPACT
        s = sol[:, i]
        q, beta, mu = s[:, S.s_q:S.s_q + S.nq], s[:, S.s_beta:S.s_beta + nv], s[:, S.s_mu:S.s_mu + c.nf]
        v, a = s[:, S.s_v:S.s_v + nv], s[:, S.s_a:S.s_a + nv]
        rows_C, rows_q, rows_v, rows_J = [], [], [], []
        for ci in range(S.ncon):
            if not (c.contact_mask >> ci) & 1:
                continue
            if impact:
                vv = v + s[:, S.s_dv:S.s_dv + nv]
                rows_C.append(impact_velocity_residual(model, q, vv, ci))
                dq, J = impact_velocity_derivatives(model, q, vv, ci)
                dv = J
            else:
                kp, kv = gains[ci]
                rows_C.append(baumgarte_residual(model, q, v, a, ci, kp, kv, pos[:, i, ci]))
                dq, dv, J = baumgarte_derivatives(model, q, v, a, ci, kp, kv)
            rows_q.append(dq)
            rows_v.append(dv)
            rows_J.append(J)
        Cc, Dq, Dv, J = (np.concatenate(x, axis=1) for x in (rows_C, rows_q, rows_v, rows_J))
        nf = c.nf
        r = l[:, i]
        Jb = r[:, S.l_J:S.l_J + nfm * nv].reshape(-1, nv, nfm).copy()   # column-major (ld nfm) -> [col][row]
        Jb[:, :, :nf] = np.swapaxes(J, 1, 2)
        r[:, S.l_J:S.l_J + nfm * nv] = Jb.reshape(-1, nfm * nv)
        D = r[:, S.l_D:S.l_D + nvf * 2 * nv].reshape(-1, 2 * nv, nvf).copy()
        D[:, :nv, nv:nv + nf] = np.swapaxes(Dq, 1, 2)
        D[:, nv:, nv:nv + nf] = np.swapaxes(Dv, 1, 2)
        r[:, S.l_D:S.l_D + nvf * 2 * nv] = D.reshape(-1, 2 * nv * nvf)
        r[:, S.l_IDC + nv:S.l_IDC + nv + nf] = Cc
        r[:, S.l_lf:S.l_lf + nf] -= np.einsum("brk,bk->br", J, beta)
        r[:, S.l_lx:S.l_lx + nv] += np.einsum("brk,br->bk", Dq, mu)
        r[:, S.l_lx + nv:S.l_lx + 2 * nv] += np.einsum("brk,br->bk", Dv, mu)
        r[:, S.l_la:S.l_la + nv] += np.einsum("brk,br->bk", J, mu)
    return l


def random_gains(seed, n_contacts):
    rng = np.random.default_rng(seed)
    return np.stack([rng.uniform(0.0, 50.0, n_contacts), rng.uniform(0.0, 20.0, n_contacts)], axis=1)


def random_positions(seed, batch, n_grid, n_contacts):
    return np.random.default_rng(seed).uniform(-1.0, 1.0, (batch, n_grid, n_contacts, 3))
