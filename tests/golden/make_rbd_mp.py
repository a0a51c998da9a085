"""Writes tests/golden/rbd_mp_cases.npz: inputs and tests/rbd_mp.py reference rows of the rigid-body linearisation on the
states where the device kernels and the numpy restatements could go wrong.

Models: ANYmal (tests/golden/anymal_model.npz, Pinocchio's joint order) and two tree edges built here, each with 13 bodies (the
most the kernels allow): a serial chain and a star (every joint on the base).  Both edge trees carry gravity off the z axis,
link masses from 50 kg (base) down to 1e-3 kg (the last body, a leaf), a contact on the leaf, one on the base body, and two on
one body, the last of them at the joint origin with the identity rotation.

States per model (key "state" names them):
  - ANYmal: standing at q_standing with foot forces that carry the weight; trot states (joint rates up to 8 rad/s, the base at
    1 m/s with a yaw rate, and a touch-down at 0.5 m/s); the base 1e3 m from the origin with p_des within 1 mm of the feet;
    joint angles theta + 2 pi k (k up to 1e5); angles on a decade sweep from 1 to 1e12 rad (every decade on some joint);
    quaternions with w = 0, w = 1e-9, w < 0, and the sign-flipped quaternion of a trot state.
  - chain and star: a slow and a fast state.
Every state is evaluated for four contact masks (one, two and all four contacts; on the edge trees the masks put the base
contact alone, the earlier of the shared-body pair alone, the pair, and all four) on Intermediate / Lift and Impact grid points.

Runs in about a minute on 8 cores; the output is the same bit for bit on every run: python tests/golden/make_rbd_mp.py"""
import multiprocessing
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import contact_ref as CR  # noqa: E402
import make_model_fixture  # noqa: E402
import rbd_mp  # noqa: E402
import rbd_ref as R  # noqa: E402

PATH = os.path.join(HERE, "rbd_mp_cases.npz")
# examples/anymal/trot.cpp:52-56 (LF, LH, RF, RH)
Q_STANDING = np.array([0, 0, 0.4792, 0, 0, 0, 1, -0.1, 0.7, -1.0, -0.1, -0.7, 1.0, 0.1, 0.7, -1.0, 0.1, -0.7, 1.0])
# Baumgarte gains of baumgarte_time_step = 0.04 (examples/anymal/trot.cpp:33): kp = 1 / dt^2, kv = 2 / dt
ANYMAL_GAINS = np.array([[625.0, 50.0]] * 4)
ANYMAL_MASKS = [0b0001, 0b0110, 0b1001, 0b1111]
EDGE_MASKS = [0b0010, 0b0100, 0b1100, 0b1111]
MODEL_KEYS = ("nv", "n_bodies", "n_contacts", "parent", "axis", "placement", "mass", "com", "inertia", "contact_parent",
              "contact_placement", "gravity")


def edge_model(kind):
    """13-body floating-base tree: "chain" (parent b - 1) or "star" (every joint on the base)."""
    rng = np.random.default_rng({"chain": 31, "star": 32}[kind])
    nb = 13
    m = {"nv": 18, "n_bodies": nb, "n_contacts": 4}
    m["parent"] = np.array([-1] + [b - 1 if kind == "chain" else 0 for b in range(1, nb)])
    ax = rng.standard_normal((nb, 3))
    m["axis"] = ax / np.linalg.norm(ax, axis=1, keepdims=True)
    pl = np.zeros((nb, 12))
    pl[0, :9] = np.eye(3).reshape(-1)
    for b in range(1, nb):
        pl[b, :9] = R.random_rotation(rng).T.reshape(-1)
        pl[b, 9:] = rng.uniform(-0.3, 0.3, 3)
    m["placement"] = pl
    m["mass"] = np.geomspace(50.0, 1e-3, nb)
    m["com"] = rng.uniform(-0.1, 0.1, (nb, 3))
    inertia = np.zeros((nb, 9))
    for b in range(nb):
        A = rng.standard_normal((3, 3)) * 0.1
        inertia[b] = (m["mass"][b] * (A @ A.T + 0.01 * np.eye(3))).T.reshape(-1)
    m["inertia"] = inertia
    shared = 6 if kind == "chain" else 5
    m["contact_parent"] = np.array([nb - 1, 0, shared, shared])
    cp = np.zeros((4, 12))
    for c in range(3):
        cp[c, :9] = R.random_rotation(rng).T.reshape(-1)
        cp[c, 9:] = rng.uniform(-0.2, 0.2, 3)
    cp[3, :9] = np.eye(3).reshape(-1)
    m["contact_placement"] = cp
    m["gravity"] = np.array([1.2, -0.7, -9.7])
    return m


def _quat(x, y, z, w):
    q = np.array([x, y, z, w], dtype=float)
    return q / np.linalg.norm(q)


def _yaw(psi):
    return np.array([0.0, 0.0, np.sin(psi / 2), np.cos(psi / 2)])


def _feet(model, q):
    return np.stack([CR.frame_placement(model, q[None], c)[1][0] for c in range(4)])


def _weight_forces(model, q, masks):
    """Per mask: the active feet share the weight, forces in the contact frames."""
    w = model["mass"].sum() * 9.81
    out = np.zeros((len(masks), 12))
    for i, mask in enumerate(masks):
        act = [c for c in range(4) if (mask >> c) & 1]
        for k, c in enumerate(act):
            oRf, _ = CR.frame_placement(model, q[None], c)
            out[i, 3 * k:3 * k + 3] = oRf[0].T @ np.array([0.0, 0.0, w / len(act)])
    return out


def anymal_states(model):
    rng = np.random.default_rng(41)
    S = []

    def state(name, q, v, a, dv, forces=None, pdes=None):
        if forces is None:
            forces = rng.uniform(-50, 50, (4, 12)) + np.tile([0.0, 0.0, 75.0], 4)
        if pdes is None:
            pdes = _feet(model, q) + rng.uniform(-0.05, 0.05, (4, 3))
        S.append(dict(name=name, q=q, v=v, a=a, dv=dv, forces=forces, pdes=pdes))

    z = np.zeros(18)
    state("standing", Q_STANDING.copy(), z, z, rng.uniform(-0.5, 0.5, 18), _weight_forces(model, Q_STANDING, ANYMAL_MASKS))
    trot_q = Q_STANDING.copy()
    trot_q[3:7] = _yaw(0.7)
    trot_q[7:] += rng.uniform(-0.3, 0.3, 12)
    trot_v = np.concatenate([[1.0, 0.1, 0.05, 0.1, -0.05, 0.6], rng.uniform(-8, 8, 12)])
    trot_a = np.concatenate([rng.uniform(-3, 3, 6), rng.uniform(-30, 30, 12)])
    state("trot", trot_q, trot_v, trot_a, rng.uniform(-1, 1, 18))
    td_q = Q_STANDING.copy()
    td_q[7:] += rng.uniform(-0.2, 0.2, 12)
    td_v = np.concatenate([[0.8, 0.0, -0.5, 0.05, 0.1, -0.2], rng.uniform(-8, 8, 12)])
    state("touchdown", td_q, td_v, rng.uniform(-5, 5, 18), -td_v * rng.uniform(0.5, 1.0, 18))
    far_q = trot_q.copy()
    far_q[:3] = [800.0, -600.0, 0.4792]
    state("far_base", far_q, trot_v, trot_a, rng.uniform(-1, 1, 18),
          pdes=_feet(model, far_q) + rng.uniform(-1e-3, 1e-3, (4, 3)))
    k = np.array([1e5, -99999, 31416, 1, -1, 12345, 77777, -50000, 2, 100000, -3, 4321])
    wrap_q = trot_q.copy()
    wrap_q[7:] += 2 * np.pi * k
    state("two_pi_k", wrap_q, trot_v, trot_a, rng.uniform(-1, 1, 18), pdes=S[1]["pdes"])
    sweep = 10.0 ** np.arange(12) * np.tile([1, -1], 6)
    for name, th in (("decades_1_1e11", sweep), ("decades_10_1e12", -10.0 * sweep[::-1])):
        q = trot_q.copy()
        q[7:] = th
        state(name, q, trot_v, trot_a, rng.uniform(-1, 1, 18))
    for name, quat in (("quat_w0", _quat(0.6, 0.0, 0.8, 0.0)), ("quat_w1e-9", np.array([0.28, -0.96, 0.0, 1e-9])),
                       ("quat_wneg", _quat(0.1, -0.2, 0.3, -0.9))):
        q = trot_q.copy()
        q[3:7] = quat
        state(name, q, trot_v, trot_a, rng.uniform(-1, 1, 18))
    neg_q = trot_q.copy()
    neg_q[3:7] = -neg_q[3:7]
    state("trot_minus_q", neg_q, trot_v, trot_a, S[1]["dv"], forces=S[1]["forces"], pdes=S[1]["pdes"])
    return S


def edge_states(kind, model):
    rng = np.random.default_rng({"chain": 51, "star": 52}[kind])
    S = []
    for name, rate in (("slow", 1.0), ("fast", 6.0)):
        q, _, _ = R.random_state(rng, 1, 18)
        q = q[0]
        q[:3] = rng.uniform(-2, 2, 3)
        v = rng.uniform(-rate, rate, 18)
        S.append(dict(name=f"{kind}_{name}", q=q, v=v, a=rng.uniform(-3 * rate, 3 * rate, 18), dv=rng.uniform(-1, 1, 18),
                      forces=rng.uniform(-20, 20, (4, 12)), pdes=_feet(model, q) + rng.uniform(-0.1, 0.1, (4, 3))))
    return S


def models():
    return {"anymal": make_model_fixture.load(), "chain": edge_model("chain"), "star": edge_model("star")}


def cases():
    """(model name, masks, gains, state dict) per state, in the npz's order."""
    ms = models()
    out = [("anymal", ANYMAL_MASKS, ANYMAL_GAINS, s) for s in anymal_states(ms["anymal"])]
    for kind in ("chain", "star"):
        gains = np.stack([np.random.default_rng(61).uniform(0.0, 400.0, 4), np.random.default_rng(62).uniform(0.0, 40.0, 4)], 1)
        out += [(kind, EDGE_MASKS, gains, s) for s in edge_states(kind, ms[kind])]
    return out


def evaluate_case(case):
    name, masks, gains, s = case
    return rbd_mp.evaluate(models()[name], s["q"], s["v"], s["a"], s["dv"], masks, s["forces"], gains, s["pdes"])


def build():
    cs = cases()
    with multiprocessing.Pool(min(len(cs), os.cpu_count() or 1)) as pool:
        res = pool.map(evaluate_case, cs, chunksize=1)
    out = {"model": np.array([c[0] for c in cs]), "state": np.array([c[3]["name"] for c in cs]),
           "masks": np.array([c[1] for c in cs]), "gains": np.stack([c[2] for c in cs])}
    for key in ("q", "v", "a", "dv", "forces", "pdes"):
        out[key] = np.stack([c[3][key] for c in cs])
    for key in res[0]:
        out[key] = np.stack([r[key] for r in res])
    for name, m in models().items():
        for key in MODEL_KEYS:
            out[f"{name}.{key}"] = np.asarray(m[key])
    return out


def load():
    with np.load(PATH) as z:
        return {k: z[k] for k in z.files}


def model_of(data, name):
    return {key: data[f"{name}.{key}"] for key in MODEL_KEYS}


if __name__ == "__main__":
    data = build()
    np.savez_compressed(PATH, **data)
    print(f"wrote {PATH}: {len(data['state'])} states, {os.path.getsize(PATH)} bytes")
