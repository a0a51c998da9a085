"""Builds and runs the C++ drop-in test (reference class/method names over the C ABI) on the GPU box."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(tmp, name="test_riccati_recursion"):
    exe = os.path.join(tmp, name)
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "oracle")], check=True)
    cmd = [gxx, "-std=c++14", "-O1", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", name + ".cpp"),
           "-L", os.path.join(ROOT, "robotoc_b200"), "-lrobotoc_b200", "-L", os.path.join(ROOT, "oracle"), "-loracle",
           "-Wl,-rpath," + os.path.join(ROOT, "robotoc_b200"), "-Wl,-rpath," + os.path.join(ROOT, "oracle"), "-o", exe]
    subprocess.run(cmd, check=True)
    return exe


def test_cpp_adaptor_compiles_and_links(tmp_path):
    """CPU: the header compiles as C++14 and links against the C ABI (no compute call)."""
    assert os.path.exists(_build(str(tmp_path)))
    assert os.path.exists(_build(str(tmp_path), "test_direct_multiple_shooting"))
    assert os.path.exists(_build(str(tmp_path), "test_unconstr_riccati_recursion"))


@pytest.mark.gpu
def test_cpp_adaptor_matches_oracle(tmp_path):
    exe = _build(str(tmp_path))
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    print(out.stdout, out.stderr)
    assert out.returncode == 0, out.stdout + out.stderr


@pytest.mark.gpu
def test_cpp_direct_multiple_shooting_matches_oracle(tmp_path):
    exe = _build(str(tmp_path), "test_direct_multiple_shooting")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    print(out.stdout, out.stderr)
    assert out.returncode == 0, out.stdout + out.stderr


@pytest.mark.gpu
def test_cpp_unconstr_adaptor_matches_oracle(tmp_path):
    exe = _build(str(tmp_path), "test_unconstr_riccati_recursion")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    print(out.stdout, out.stderr)
    assert out.returncode == 0, out.stdout + out.stderr


def _build_allgather(tmp):
    exe = os.path.join(tmp, "test_allgather_two_ranks")
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    cmd = [gxx, "-std=c++14", "-O1", "-I", os.path.join(ROOT, "include"), "-I", "/usr/local/cuda/include",
           os.path.join(ROOT, "tests", "cpp", "test_allgather_two_ranks.cpp"), "-L", os.path.join(ROOT, "robotoc_b200"),
           "-lrobotoc_b200", "-L", "/usr/local/cuda/lib64", "-lcudart", "-lnccl", "-Wl,-rpath," + os.path.join(ROOT, "robotoc_b200"),
           "-o", exe]
    subprocess.run(cmd, check=True)
    return exe


def test_cpp_allgather_test_compiles_and_links(tmp_path):
    """CPU: the two-rank C-ABI test (rbt_allgather_step + the host's NCCL) compiles and links."""
    assert os.path.exists(_build_allgather(str(tmp_path)))


@pytest.mark.gpu
def test_cpp_allgather_step_two_ranks(tmp_path):
    """Two ranks in one process (ncclCommInitAll) gather the packed Newton step through rbt_allgather_step.
    Needs two GPUs: skipped (exit code 77) on a single-GPU machine."""
    exe = _build_allgather(str(tmp_path))
    out = subprocess.run([exe], capture_output=True, text=True, timeout=180)
    print(out.stdout, out.stderr)
    if out.returncode == 77:
        pytest.skip(out.stdout.strip())
    assert out.returncode == 0, out.stdout + out.stderr
