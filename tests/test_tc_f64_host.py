"""PINN_MODE_TC_F64 without a GPU: the DMMA instantiations of the FFMA kernel (csrc/ffma_inst.cu with
-DPINN_INST_DMMA=1) compile to DMMA.16x8x16 for sm_90a without serialisation warnings, with products that use no stack,
and the Python mode table refuses float32 before any engine exists."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import neuralpde_jl_b200 as npde
from neuralpde_jl_b200 import configs
from neuralpde_jl_b200 import engine as E
from neuralpde_jl_b200 import pinn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "neuralpde.jl_b200", "csrc")


def _nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return None


def _compile(tmp, name, defs):
    nvcc = _nvcc()
    out = os.path.join(tmp, name + ".o")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"),
           "-DPINN_INST_REAL=double", *defs, "-c", os.path.join(CSRC, "ffma_inst.cu"), "-o", out, "-Xptxas", "-v"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    sass = subprocess.run([os.path.join(os.path.dirname(nvcc), "cuobjdump"), "-sass", out], capture_output=True,
                          text=True, check=True).stdout
    return r.stderr, sass


def _kernel_stack(log):
    """stack frame bytes of ffma_loss_grad_kernel from ptxas -v"""
    m = re.search(r"Function properties for _ZN4pinn21ffma_loss_grad_kernel\S*\n\s*(\d+) bytes stack frame", log)
    assert m, log[-2000:]
    return int(m.group(1))


VARIANTS = {"plain": ["-DPINN_INST_BUFS=1"],
            "func_gmem": ["-DPINN_INST_BUFS=0", "-DPINN_INST_INTEG=1", "-DPINN_INST_FIXED=1", "-DPINN_INST_FUNC=1"]}


@pytest.fixture(scope="module", params=sorted(VARIANTS))
def compiled(request, tmp_path_factory):
    if _nvcc() is None:
        pytest.skip("nvcc not found")
    tmp = str(tmp_path_factory.mktemp("tc_f64"))
    defs = VARIANTS[request.param]
    return _compile(tmp, "fma", defs), _compile(tmp, "dmma", defs + ["-DPINN_INST_DMMA=1"])


def test_dmma_in_sass(compiled):
    (_, fma_sass), (_, dmma_sass) = compiled
    assert "DMMA.16x8x16" in dmma_sass
    assert "DMMA" not in fma_sass


def test_no_serialisation_warnings_and_no_stack_in_the_products(compiled):
    (fma_log, _), (dmma_log, _) = compiled
    bad = [l for l in dmma_log.splitlines() if re.search(r"C75\d\d", l)]
    assert not bad, "\n".join(bad)
    # the DMMA products (one function per channel count) keep their accumulators and fragments in registers: no stack
    # frame (ptxas reports a few spilled registers at C = 5 and 6 in the global-buffer instantiations)
    props = re.findall(r"Function properties for (_ZN4pinn\d+gemm_\w+_dmma\w*)\n\s*(\d+) bytes stack frame", dmma_log)
    assert len(props) == 30, props
    assert all(p[1] == "0" for p in props), props
    # the residual program's per-point arrays give both kernel instantiations a frame; the calls add a few saves
    assert _kernel_stack(dmma_log) <= _kernel_stack(fma_log) + 256


def test_mode_table():
    assert pinn.MODES == {"ffma": 0, "tc_bf16": 1, "tc_split": 2, "tc_f64": 3}
    assert E.MODE_TC_F64 == npde.MODE_TC_F64 == 3
    assert pinn.FFMA_KERNEL_MODES == (E.MODE_FFMA, E.MODE_TC_F64)


def test_float32_refused_before_an_engine_exists(monkeypatch):
    def no_engine(*a, **k):
        raise AssertionError("an engine was created")
    monkeypatch.setattr(pinn, "Engine", no_engine)
    cfg = configs.config2(n=8, width=16, hidden=2)
    with pytest.raises(ValueError, match=r'mode="tc_f64" .* needs float64'):
        npde.symbolic_discretize(cfg.pde_system, cfg.discretization(dtype=np.float32, mode="tc_f64"))
