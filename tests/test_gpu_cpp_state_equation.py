"""Builds and runs tests/cpp/test_state_equation.cpp: the C++ adaptor's setInitialConfiguration / linearizeStateEquation and the
resident wire path with the inverse dynamics, the contact rows and the state equation left to the device.  The records the C++
side writes are checked here against the numpy restatement tests/state_ref.py."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_model_fixture  # noqa: E402
import rbd_ref as R  # noqa: E402
import state_ref as SR  # noqa: E402
from helpers import rel_err  # noqa: E402


def _build(tmp):
    exe = os.path.join(tmp, "test_state_equation")
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    cmd = [gxx, "-std=c++14", "-O1", "-I", os.path.join(ROOT, "include"), os.path.join(HERE, "cpp", "test_state_equation.cpp"),
           "-L", os.path.join(ROOT, "robotoc_b200"), "-lrobotoc_b200", "-Wl,-rpath," + os.path.join(ROOT, "robotoc_b200"), "-o", exe]
    subprocess.run(cmd, check=True)
    return exe


def test_cpp_state_equation_test_compiles_and_links(tmp_path):
    """CPU: the adaptor's new methods compile as C++14 and link against the C ABI."""
    assert os.path.exists(_build(str(tmp_path)))


@pytest.mark.gpu
def test_cpp_state_equation(tmp_path):
    from robotoc_b200 import ANYMAL, StageDims, StageLayout, anymal_constraint_table
    from robotoc_b200._lib import rbt_stage_ctrl
    exe = _build(str(tmp_path))
    mpath = os.path.join(str(tmp_path), "model.bin")
    with open(mpath, "wb") as f:
        f.write(bytes(R.to_c(make_model_fixture.load())))
    out = subprocess.run([exe, mpath, str(tmp_path)], capture_output=True, text=True, timeout=120)
    print(out.stdout, out.stderr)
    assert out.returncode == 0, out.stdout + out.stderr
    table = anymal_constraint_table()
    S = StageLayout(StageDims(ANYMAL, nf_max=12, n_contacts=4, n_box=table.n_box))
    raw = open(os.path.join(str(tmp_path), "ctrl.bin"), "rb").read()
    n_grid = len(raw) // ctypes.sizeof(rbt_stage_ctrl)
    ctrl = (rbt_stage_ctrl * n_grid).from_buffer_copy(raw)
    load = lambda name, stride: np.fromfile(os.path.join(str(tmp_path), name)).reshape(-1, n_grid, stride)  # noqa: E731
    sol, lin_in, lin_out = load("sol.bin", S.s_stride), load("lin_in.bin", S.l_stride), load("lin_out.bin", S.l_stride)
    q0 = np.fromfile(os.path.join(str(tmp_path), "q0.bin")).reshape(-1, S.nq)
    assert rel_err(lin_out, SR.linearize(S, ctrl, sol, lin_in, q0)) < 1e-12
