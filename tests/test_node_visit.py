"""CPU tests of the box test's integer reduction (trace.cuh, INTEGER BOX TEST): for every ray ray_setup flags B2_RAY_INTBOX, the hit bits of
node_test<true> equal the float reduction's, on special values (-0, +-inf, NaN, denormals, huge coordinates, tfar of -0 / NaN) and on
random rays, nodes and tbest; rays outside the integer domain take node_test<false>, which must equal the float reduction too."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "node_visit", "node_visit.cu")


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("node_visit") / "node_visit")
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    subprocess.run([nvcc if os.path.exists(nvcc) else "nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-fmad=false", "-Xcompiler", "-ffp-contract=off,-mfma",
                    "-o", exe, SRC], check=True, timeout=600)
    return exe


def run(exe, *args):
    out = subprocess.run([exe, *args], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    m = re.search(r"cases (\d+) intbox (\d+) mismatch (\d+) premise (\d+)", out.stdout)
    assert m, out.stdout
    return tuple(int(x) for x in m.groups()), out.stderr


def test_corner_values(harness):
    (cases, intbox, mismatch, premise), err = run(harness, "corner")
    assert mismatch == 0, err
    assert premise == 0
    assert cases > 50000 and 0 < intbox < cases          # both paths are exercised


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_rays_and_nodes(harness, seed):
    (cases, intbox, mismatch, premise), err = run(harness, "random", "200000", str(seed))
    assert mismatch == 0, err
    assert premise == 0
    assert cases == 200000 and intbox > 0.8 * cases      # unit-scale rays from finite origins take the integer path
