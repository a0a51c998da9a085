"""The numpy restatements tests/rbd_ref.py and tests/contact_ref.py against the extended-precision, definition-level reference
tests/rbd_mp.py, row by row, on the states of tests/golden/rbd_mp_cases.npz (ANYmal at physical states, far from the origin, at
huge joint angles and odd quaternions; a 13-body chain and star with off-axis gravity, light links, a contact on the base and
two contacts on one body).  Also pins the ANYmal fixture to Pinocchio's joint order with facts from the reference's examples,
and recomputes a case of the npz live.

A row passes when |restatement - reference| <= 1e-12 x the row's largest additive contribution (tau: inertial, bias, gravity,
contact; C: a_cl, kv v, kp oMf.p, kp p_des; derivatives: the same split), so a small row next to a large one is held to its own
size (rbd_mp.row_err; the only exceptions, a row that vanishes analytically and the dtau/dq rows of a link far smaller than
its block, are described at rbd_mp.row_scale)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import contact_ref as CR  # noqa: E402
import make_model_fixture  # noqa: E402
import make_rbd_mp  # noqa: E402
import rbd_mp  # noqa: E402
import rbd_ref as R  # noqa: E402

TOL = 1e-12
DATA = make_rbd_mp.load()
STATES = [str(s) for s in DATA["state"]]


# ---- the ANYmal fixture in Pinocchio's joint order
def test_fixture_joint_order_is_pinocchios():
    """urdfdom lists a link's child joints by name, so Pinocchio numbers the legs LF, LH, RF, RH -- the order the examples
    write q in (examples/anymal/trot.cpp:52-56, contact frames at trot.cpp:34-37)."""
    m = make_model_fixture.load()
    legs = ["LF", "LH", "RF", "RH"]
    assert list(m["joint_names"]) == [f"{leg}_{j}" for leg in legs for j in ("HAA", "HFE", "KFE")]
    assert list(m["contact_names"]) == [f"{leg}_FOOT" for leg in legs]
    assert list(m["contact_parent"]) == [3, 6, 9, 12]
    assert list(m["parent"]) == [-1, 0, 1, 2, 0, 4, 5, 0, 7, 8, 0, 10, 11]


def test_fixture_standing_pose_is_symmetric_on_the_ground():
    """At the examples' q_standing (examples/anymal/jump.cpp:52-56, trot.cpp:52-56) the four feet are mirror images and touch
    the ground."""
    m = make_model_fixture.load()
    q = make_rbd_mp.Q_STANDING[None]
    feet = np.stack([CR.frame_placement(m, q, c)[1][0] for c in range(4)])
    signs = {0: (1, 1), 1: (-1, 1), 2: (1, -1), 3: (-1, -1)}   # LF, LH, RF, RH
    for c, (sx, sy) in signs.items():
        assert np.sign(feet[c, 0]) == sx and np.sign(feet[c, 1]) == sy, c
    np.testing.assert_allclose(np.abs(feet), np.abs(feet[:1]).repeat(4, 0), rtol=0, atol=1e-12)
    assert np.abs(feet[:, 2]).max() < 1e-5


def test_fixture_total_mass_is_the_urdf_links():
    """Sum of the 23 <mass> entries of examples/anymal/anymal_b_simple_description/urdf/anymal.urdf (base 1e-6, base_inertia
    16.793507758, per leg 1.42462064 + 1.634976467 + 0.207204302 + 0.140170767 + 0.001, imu_link 0.05)."""
    urdf = 1e-6 + 16.793507758 + 4 * (1.42462064 + 1.634976467 + 0.207204302 + 0.140170767 + 0.001) + 0.05
    assert abs(make_model_fixture.load()["mass"].sum() - urdf) < 1e-12


def test_case_file_holds_the_current_fixture():
    m, stored = make_model_fixture.load(), make_rbd_mp.model_of(DATA, "anymal")
    for k in make_rbd_mp.MODEL_KEYS:
        np.testing.assert_array_equal(stored[k], m[k], err_msg=k)


# ---- the restatements against the reference
def _restated(model, s, masks, gains, pdes):
    """The rows of one state by rbd_ref / contact_ref, in the layout of rbd_mp.evaluate."""
    q, v, a, dv = (DATA[k][s][None] for k in ("q", "v", "a", "dv"))
    z = np.zeros_like(v)
    out = {k: np.zeros_like(DATA[k][s]) for k in ("tau", "dtau_dq", "dtau_dv", "C", "dC_dq", "dC_dv", "J")}
    for j, mask in enumerate(masks):
        fx = R.contact_fext(model, DATA["forces"][s][j][None], int(mask))
        tau, dq, dvv, M = R.rnea_derivatives(model, q, v, a, fx)
        out["tau"][0, j], out["dtau_dq"][0, j], out["dtau_dv"][0, j] = tau[0], dq[0], dvv[0]
        tau, dq, _, _ = R.rnea_derivatives(model, q, z, dv, fx, gravity=False)
        out["tau"][1, j], out["dtau_dq"][1, j] = tau[0], dq[0]
    out["M"] = M[0]
    for c in range(4):
        kp, kv = gains[c]
        out["C"][0, c] = CR.baumgarte_residual(model, q, v, a, c, kp, kv, pdes[c][None])[0]
        dq, dvv, J = CR.baumgarte_derivatives(model, q, v, a, c, kp, kv)
        out["dC_dq"][0, c], out["dC_dv"][0, c], out["J"][c] = dq[0], dvv[0], J[0]
        out["C"][1, c] = CR.impact_velocity_residual(model, q, v + dv, c)[0]
        dq, dvv = CR.impact_velocity_derivatives(model, q, v + dv, c)
        out["dC_dq"][1, c], out["dC_dv"][1, c] = dq[0], dvv[0]
    return out


def _blocks(key, got, ref, scale):
    """(got, ref, scale) per block of rows one grid point holds: tau rows per grid kind and mask, the contact rows of the four
    contacts per grid kind, M and J whole."""
    if key in ("M", "J"):
        return [(got.reshape(scale.size, -1), ref.reshape(scale.size, -1), scale.reshape(-1))]
    if key.startswith("C") or key.startswith("dC"):
        return [(got[g].reshape(scale[g].size, -1), ref[g].reshape(scale[g].size, -1), scale[g].reshape(-1)) for g in (0, 1)]
    return [(got[i], ref[i], scale[i]) for i in np.ndindex(scale.shape[:-1])]


SECTIONS = ("tau", "dtau_dq", "dtau_dv", "M", "C", "dC_dq", "dC_dv", "J")


@pytest.mark.parametrize("state", STATES)
def test_restatements_match_the_extended_precision_reference(state):
    s = STATES.index(state)
    model = make_rbd_mp.model_of(DATA, str(DATA["model"][s]))
    got = _restated(model, s, DATA["masks"][s], DATA["gains"][s], DATA["pdes"][s])
    worst = {k: max(rbd_mp.row_err(g, r, sc, rbd_mp.DQ_FLOOR if k == "dtau_dq" else 0.0)
                    for g, r, sc in _blocks(k, got[k], DATA[k][s], DATA[k + "_scale"][s])) for k in SECTIONS}
    print(state, " ".join(f"{k} {e:.1e}" for k, e in worst.items()))
    for k, e in worst.items():
        assert e <= TOL, (k, e)


def test_the_reference_sees_what_the_rows_are_made_of():
    """The cases reach what they are there for: the standing base rows are a near-cancellation of the weight and the contact
    forces, the far base puts kp |oMf.p| ~ 1e3 kp next to a C of a few kp mm, and the light links' rows are their own size."""
    s = STATES.index("standing")
    tau, sc = DATA["tau"][s, 0, 3, :6], DATA["tau_scale"][s, 0, 3, :6]
    assert sc[2] > 250 and abs(tau[2]) < 1e-9 * sc[2]
    s = STATES.index("far_base")
    C, sc = DATA["C"][s, 0], DATA["C_scale"][s, 0]
    assert (sc[:, :2] > 400 * DATA["gains"][s][:, :1]).all() and (np.abs(C[:, :2]) < 1e-2 * sc[:, :2]).all()
    for s in (STATES.index("chain_fast"), STATES.index("star_fast")):
        assert DATA["tau_scale"][s, 0, 0, 17] < 1e-2 * DATA["tau_scale"][s, 0, 0, :6].max()


def test_npz_is_what_the_reference_computes():
    """One state recomputed live (about 30 s): the star tree, with the base contact, the shared-body pair and off-axis
    gravity.  The generator reproduces the whole file bit for bit."""
    s = STATES.index("star_fast")
    name = str(DATA["model"][s])
    model = make_model_fixture.load() if name == "anymal" else make_rbd_mp.edge_model(name)
    d = {k: DATA[k][s] for k in ("q", "v", "a", "dv", "forces", "pdes")}
    out = rbd_mp.evaluate(model, d["q"], d["v"], d["a"], d["dv"], list(DATA["masks"][s]), d["forces"], DATA["gains"][s],
                          d["pdes"])
    for k, x in out.items():
        np.testing.assert_array_equal(x, DATA[k][s], err_msg=k)
