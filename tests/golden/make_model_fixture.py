"""Writes tests/golden/anymal_model.npz: the robot model (fields of rbt_robot_model) of the reference's ANYmal example, parsed
from examples/anymal/anymal_b_simple_description/urdf/anymal.urdf with the standard-library XML parser the way Pinocchio's URDF
parser builds a pinocchio::Model with a JointModelFreeFlyer root:
  - joints in depth-first order of the kinematic tree, the root link on the free flyer; each link's child joints are visited in
    the order of their names, because urdfdom builds a link's child list by walking its std::map of joints keyed by name (this
    gives the legs LF, LH, RF, RH, the order the reference's examples write q in);
  - a fixed joint merges its child link into the parent body: the link's inertia is added in the body's joint frame, and its frame
    (e.g. LF_FOOT) is placed in the parent joint's frame;
  - a revolute joint's placement = (fixed-joint chain from its parent body to its parent link) * its URDF origin;
  - contacts LF_FOOT, LH_FOOT, RF_FOOT, RH_FOOT (examples/anymal/trot.cpp:34-37), gravity (0, 0, -9.81).
The npz also holds the revolute joint names in q order ("joint_names") and the contact frame names ("contact_names").
Runs only where a reference tree exists: ROBOTOC_REFERENCE=/path/to/robotoc python tests/golden/make_model_fixture.py"""
import os
import sys
import xml.etree.ElementTree as ET

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "anymal_model.npz")
CONTACTS = ["LF_FOOT", "LH_FOOT", "RF_FOOT", "RH_FOOT"]


def rpy_to_rot(r, p, y):
    cr, sr, cp, sp, cy, sy = np.cos(r), np.sin(r), np.cos(p), np.sin(p), np.cos(y), np.sin(y)
    Rx = np.array([[1, 0, 0], [0, cr, -sr], [0, sr, cr]])
    Ry = np.array([[cp, 0, sp], [0, 1, 0], [-sp, 0, cp]])
    Rz = np.array([[cy, -sy, 0], [sy, cy, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def origin(el):
    o = el.find("origin") if el is not None else None
    if o is None:
        return np.eye(3), np.zeros(3)
    xyz = np.array([float(x) for x in o.get("xyz", "0 0 0").split()])
    rpy = [float(x) for x in o.get("rpy", "0 0 0").split()]
    return rpy_to_rot(*rpy), xyz


def compose(A, B):
    return A[0] @ B[0], A[0] @ B[1] + A[1]


def link_inertia(link):
    """(mass, com, rotational inertia about the com) of a URDF link, in the link frame."""
    inn = link.find("inertial")
    if inn is None:
        return 0.0, np.zeros(3), np.zeros((3, 3))
    R, c = origin(inn)
    m = float(inn.find("mass").get("value"))
    i = inn.find("inertia")
    g = {k: float(i.get(k)) for k in ("ixx", "ixy", "ixz", "iyy", "iyz", "izz")}
    Ic = np.array([[g["ixx"], g["ixy"], g["ixz"]], [g["ixy"], g["iyy"], g["iyz"]], [g["ixz"], g["iyz"], g["izz"]]])
    return m, c, R @ Ic @ R.T


def add_inertia(a, b):
    """pinocchio::Inertia::operator+ of two inertias expressed in the same frame."""
    (m1, c1, I1), (m2, c2, I2) = a, b
    m = m1 + m2
    if m == 0.0:
        return a
    c = (m1 * c1 + m2 * c2) / m
    def shift(mi, ci):
        d = ci - c
        return mi * (d @ d * np.eye(3) - np.outer(d, d))
    return m, c, I1 + shift(m1, c1) + I2 + shift(m2, c2)


def parse(urdf):
    root = ET.parse(urdf).getroot()
    links = {l.get("name"): l for l in root.findall("link")}
    joints = root.findall("joint")
    children = {}
    for j in sorted(joints, key=lambda j: j.get("name")):
        children.setdefault(j.find("parent").get("link"), []).append(j)
    root_link = (set(links) - {j.find("child").get("link") for j in joints}).pop()
    parent, axis, placement, inertias, frames, names = [-1], [np.zeros(3)], [(np.eye(3), np.zeros(3))], [], {}, []
    inertias.append((0.0, np.zeros(3), np.zeros((3, 3))))

    def visit(link, body, T):
        m, c, Ic = link_inertia(links[link])
        inertias[body] = add_inertia(inertias[body], (m, T[0] @ c + T[1], T[0] @ Ic @ T[0].T))
        frames[link] = (body, T)
        for j in children.get(link, []):
            child = j.find("child").get("link")
            O = origin(j)
            if j.get("type") == "fixed":
                visit(child, body, compose(T, O))
            elif j.get("type") in ("revolute", "continuous"):
                ax = j.find("axis")
                u = np.array([float(x) for x in (ax.get("xyz") if ax is not None else "1 0 0").split()])
                parent.append(body)
                names.append(j.get("name"))
                axis.append(u / np.linalg.norm(u))
                placement.append(compose(T, O))
                inertias.append((0.0, np.zeros(3), np.zeros((3, 3))))
                visit(child, len(parent) - 1, (np.eye(3), np.zeros(3)))
            else:
                raise ValueError(f"joint type {j.get('type')} not supported")

    visit(root_link, 0, (np.eye(3), np.zeros(3)))
    nb = len(parent)
    pack = lambda T: np.concatenate([T[0].T.reshape(-1), T[1]])  # noqa: E731  (R column-major | p)
    return {
        "nv": nb + 5, "n_bodies": nb, "n_contacts": len(CONTACTS),
        "parent": np.array(parent), "axis": np.array(axis), "placement": np.array([pack(T) for T in placement]),
        "mass": np.array([x[0] for x in inertias]), "com": np.array([x[1] for x in inertias]),
        "inertia": np.array([x[2].T.reshape(-1) for x in inertias]),
        "contact_parent": np.array([frames[c][0] for c in CONTACTS]),
        "contact_placement": np.array([pack(frames[c][1]) for c in CONTACTS]),
        "gravity": np.array([0.0, 0.0, -9.81]),
        "joint_names": np.array(names), "contact_names": np.array(CONTACTS),
    }


def load():
    with np.load(PATH) as z:
        return {k: z[k] for k in z.files}


if __name__ == "__main__":
    ref = os.environ.get("ROBOTOC_REFERENCE", "")
    urdf = os.path.join(ref, "examples", "anymal", "anymal_b_simple_description", "urdf", "anymal.urdf")
    if not ref or not os.path.exists(urdf):
        sys.exit("set ROBOTOC_REFERENCE to a robotoc source tree")
    model = parse(urdf)
    np.savez(PATH, **model)
    print(f"wrote {PATH}: {model['n_bodies']} bodies, total mass {model['mass'].sum():.4f} kg")
