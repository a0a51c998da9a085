"""Writes tests/golden/stage_mp_cases.npz: fp64 inputs and tests/stage_mp.py reference outputs of the MJtJinv kernel and of
the free-flyer update, on the inputs where those kernels could go wrong.

MJtJinv (K1) on ANYmal's own M and J (tests/rbd_ref.py on the fixture tests/golden/anymal_model.npz), at the states of
make_rbd_mp.py -- standing, trot, touch-down, the base 1e3 m from the origin -- a stance with the LF knee 1e-3 rad from
straight, and the same stance with a base 1e6 times heavier, where J M^-1 J^T is ill-conditioned ("cond" records the 2-norm
condition number of J M^-1 J^T per case: up to 77 without the payload, 1.0e7 with it).  Contact masks: none, LF, LF + RF (feet 0 and 2, not contiguous), LH + RH, three feet, all four (nf = 0, 3, 6, 6, 9, 12).

Free-flyer update: step sizes 1, 0.5, 0.75^8 and 1e-8 (one per OCP) times directions whose rotation th = step |w| is 0, 1e-12,
1e-6 (1 - 2^-52), 1e-6, 1e-6 (1 + 2^-52), 1e-4, 1, pi, 3 pi / 2 and 10 (rounded as the kernels round step * dq: the three
angles around the 1e-6 branch of the exponential land on the fp64 neighbours of 1e-6 exactly), each from three
configurations: the base 1e3 m from the origin, a quaternion with w < 0, and one with w = 1e-9.

The inputs are rebuilt by the functions below (shared with the tests); the npz stores them and their SHA-256, so a change of
the builders fails loudly instead of comparing against stale references.  Runs in a few seconds; the output is the same bit
for bit on every run: python tests/golden/make_stage_mp.py"""
import hashlib
import io
import os
import sys
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_model_fixture  # noqa: E402
import make_rbd_mp  # noqa: E402
import rbd_ref as R  # noqa: E402
import stage_mp  # noqa: E402

PATH = os.path.join(HERE, "stage_mp_cases.npz")
MASKS = [0b0000, 0b0001, 0b0101, 0b1010, 0b0111, 0b1111]
STATES = ("standing", "trot", "touchdown", "far_base", "stretched_knee", "heavy_base_stretched_knee")
STEPS = np.array([1.0, 0.5, 0.75 ** 8, 1e-8])
ANGLES = np.array([0.0, 1e-12, np.nextafter(1e-6, 0.0), 1e-6, np.nextafter(1e-6, 1.0), 1e-4, 1.0, np.pi, 1.5 * np.pi, 10.0])
CONFIGS = ("far_base", "quat_wneg", "quat_w1e-9")
NV, NQ = 18, 19
# The LF knee angle (KFE) at which the LF leg is straight: the foot sits off the shank's axis, so this is not 0.  It is where
# the smallest singular value of the foot's 3 x 3 leg Jacobian vanishes (1e-10 here, from 0.036 at KFE = 0), with the hip
# flexion at 0.
LF_KNEE_STRAIGHT = 0.3017767139321471


def anymal_states():
    """name -> q of the K1 cases."""
    model = make_model_fixture.load()
    out = {s["name"]: s["q"] for s in make_rbd_mp.anymal_states(model) if s["name"] in STATES}
    q = make_rbd_mp.Q_STANDING.copy()
    q[7 + 1] = 0.0                          # LF hip flexion
    q[7 + 2] = LF_KNEE_STRAIGHT + 1e-3      # LF knee 1e-3 rad from straight
    out["stretched_knee"] = q
    out["heavy_base_stretched_knee"] = q.copy()
    return model, out


def heavy_base_model(model):
    """ANYmal carrying a payload that makes the base 1e6 times heavier (mass and rotational inertia).  With the LF knee
    nearly straight, the foot can then move along the leg only by moving the heavy base, so J M^-1 J^T becomes
    ill-conditioned (its condition number is recorded in "cond")."""
    m = {k: np.array(v, copy=True) for k, v in model.items()}
    m["mass"][0] *= 1e6
    m["inertia"][0] *= 1e6
    return m


def kkt_inputs():
    """M [S, nv, nv] and J [S, n_masks, 12, nv] (rows >= nf zero) for the states in STATES order."""
    anymal, qs = anymal_states()
    M = np.zeros((len(STATES), NV, NV))
    J = np.zeros((len(STATES), len(MASKS), 12, NV))
    for s, name in enumerate(STATES):
        model = heavy_base_model(anymal) if name.startswith("heavy_base") else anymal
        q = qs[name][None]
        z = np.zeros((1, NV))
        M[s] = R.rnea_derivatives(model, q, z, z)[3][0]
        Jc = [R.contact_jacobian(model, q, c)[0] for c in range(4)]
        for m, mask in enumerate(MASKS):
            act = [c for c in range(4) if (mask >> c) & 1]
            if act:
                J[s, m, :3 * len(act)] = np.concatenate([Jc[c] for c in act])
    return M, J


def nf_of(mask):
    return 3 * bin(mask).count("1")


def se3_inputs():
    """q [n_cfg * n_angles, nq], dq [n_steps, n_cfg * n_angles, nv]: grid point g = cfg * len(ANGLES) + angle index; OCP b uses
    STEPS[b].  The rotation axis is random except for the three angles around 1e-6, which turn about z so that the kernels'
    th = sqrt((step dq)^2) is exactly the angle."""
    rng = np.random.default_rng(71)
    base = make_rbd_mp.Q_STANDING.copy()
    base[7:] += rng.uniform(-0.3, 0.3, 12)
    cfgs = []
    for name in CONFIGS:
        q = base.copy()
        if name == "far_base":
            q[:3] = [800.0, -600.0, 0.4792]
            q[3:7] = make_rbd_mp._yaw(0.7)
        elif name == "quat_wneg":
            q[3:7] = make_rbd_mp._quat(0.1, -0.2, 0.3, -0.9)
        else:
            q[3:7] = np.array([0.28, -0.96, 0.0, 1e-9])
        cfgs.append(q)
    G = len(CONFIGS) * len(ANGLES)
    q = np.stack([cfgs[g // len(ANGLES)] for g in range(G)])
    dq = np.zeros((len(STEPS), G, NV))
    for g in range(G):
        k = g % len(ANGLES)
        th = ANGLES[k]
        axis = np.array([0.0, 0.0, 1.0]) if k in (2, 3, 4) else rng.standard_normal(3)
        axis /= np.linalg.norm(axis)
        v = rng.uniform(-1.0, 1.0, 3)
        joints = rng.uniform(-1.0, 1.0, 12)
        for b, step in enumerate(STEPS):
            w = axis * th / step
            if k in (2, 3, 4):
                w[2] = _exact_multiple(th, step)
            dq[b, g, :3], dq[b, g, 3:6], dq[b, g, 6:] = v / step, w, joints / step
    return q, dq


def _exact_multiple(th, step):
    """x with fl(step * x) == th (the kernels form step * dq before the norm)."""
    x = th / step
    for _ in range(64):
        y = step * x
        if y == th:
            return x
        x = np.nextafter(x, np.inf if y < th else -np.inf)
    raise AssertionError(f"no fp64 x with step * x == {th!r} for step {step!r}")


def inputs_sha256(M, J, q, dq):
    h = hashlib.sha256()
    for a in (M, J, q, dq, STEPS):
        h.update(np.ascontiguousarray(a, dtype="<f8").tobytes())
    return h.hexdigest()


def kkt_case(M, J, s, m):
    nf = nf_of(MASKS[m])
    return stage_mp.mjtjinv(M[s], J[s, m, :nf])


def build():
    M, J = kkt_inputs()
    q, dq = se3_inputs()
    n = NV + 12
    Z = np.zeros((len(STATES), len(MASKS), n, n))
    Zs = np.zeros((len(STATES), len(MASKS), n))
    cond = np.zeros((len(STATES), len(MASKS)))
    for s in range(len(STATES)):
        Mi = np.linalg.inv(M[s])
        for m, mask in enumerate(MASKS):
            nf = nf_of(mask)
            z, sc = kkt_case(M, J, s, m)
            Z[s, m, :NV + nf, :NV + nf], Zs[s, m, :NV + nf] = z, sc
            if nf:
                Jm = J[s, m, :nf]
                cond[s, m] = np.linalg.cond(Jm @ Mi @ Jm.T)
    qn = np.zeros((len(STEPS),) + q.shape)
    qs = np.zeros_like(qn)
    for b, step in enumerate(STEPS):
        for g in range(q.shape[0]):
            qn[b, g], qs[b, g] = stage_mp.integrate_free_flyer(q[g], dq[b, g], step)
    return {"states": np.array(STATES), "masks": np.array(MASKS), "M": M, "J": J, "Z": Z, "Z_scale": Zs, "cond": cond,
            "steps": STEPS, "angles": ANGLES, "configs": np.array(CONFIGS), "q": q, "dq": dq, "q_new": qn, "q_scale": qs,
            "sha256": np.array(inputs_sha256(M, J, q, dq))}


def save(data, path=PATH):
    """A zip with fixed member dates, so that the file is the same bit for bit on every run."""
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
    print(f"wrote {PATH}: {os.path.getsize(PATH)} bytes; cond(J M^-1 J^T) up to {data['cond'].max():.2e}")
