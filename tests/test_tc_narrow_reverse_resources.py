"""Compile-time resources of the narrow tensor-core kernel's reverse sweep (csrc/tc_kernel.cu), from ptxas -v.

The reverse sweep of a tensor layer (recompute, dgrad, wgrad) keeps its wgmma accumulators in registers and issues each
product as one straight-line sequence on all four warpgroups.  ptxas serializes wgmmas whose accumulators are carried
around a loop or a divergent branch (warning C7520, naming the function that holds them); that costs speed without
failing any numerical test, so it is checked here for every net_backward instantiation.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "neuralpde.jl_b200", "csrc")


def _nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return None


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("tc_narrow_reverse") / "tc_kernel.o"
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"),
           "--split-compile=0", "-c", os.path.join(CSRC, "tc_kernel.cu"), "-o", str(out), "-Xptxas", "-v"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stderr


def test_backward_wgmma_not_serialized(ptxas_log):
    # one instantiation per channel structure and activation kind of PINN_TC_DISPATCH (24 with five channels)
    names = set(re.findall(r"_ZN4pinn12net_backwardI\w+", ptxas_log))
    assert len(names) == 24, sorted(names)
    bad = [l for l in ptxas_log.splitlines() if "C7520" in l and "net_backward" in l]
    assert not bad, "\n".join(bad)
