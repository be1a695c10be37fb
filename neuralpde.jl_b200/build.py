"""Build libpinn_b200.so (sm_90a) in-tree with nvcc.

The library is the C-ABI product (include/pinn_b200.h).  Objects are rebuilt only when a
source or header is newer, and translation units compile in parallel.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(HERE, "build")
LIB = os.path.join(LIBDIR, "libpinn_b200.so")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "-I", INCLUDE,
]

# (object name, source, extra defines)
UNITS = [
    ("pinn_abi.o", "pinn_abi.cu", []),
    ("plan.o", "plan.cu", []),
    ("qn.o", "qn.cu", []),
    ("hmc.o", "hmc.cu", []),
    ("ffma_launch.o", "ffma_launch.cu", []),
    ("ffma_f32_smem.o", "ffma_inst.cu", ["-DPINN_INST_REAL=float", "-DPINN_INST_BUFS=1"]),
    ("ffma_f32_gmem.o", "ffma_inst.cu", ["-DPINN_INST_REAL=float", "-DPINN_INST_BUFS=0"]),
    ("ffma_f64_smem.o", "ffma_inst.cu", ["-DPINN_INST_REAL=double", "-DPINN_INST_BUFS=1"]),
    ("ffma_f64_gmem.o", "ffma_inst.cu", ["-DPINN_INST_REAL=double", "-DPINN_INST_BUFS=0"]),
    # the same four with integral terms (node tiles, PINN_OP_INTEGRAL)
    ("ffma_f32_smem_integ.o", "ffma_inst.cu", ["-DPINN_INST_REAL=float", "-DPINN_INST_BUFS=1", "-DPINN_INST_INTEG=1"]),
    ("ffma_f32_gmem_integ.o", "ffma_inst.cu", ["-DPINN_INST_REAL=float", "-DPINN_INST_BUFS=0", "-DPINN_INST_INTEG=1"]),
    ("ffma_f64_smem_integ.o", "ffma_inst.cu", ["-DPINN_INST_REAL=double", "-DPINN_INST_BUFS=1", "-DPINN_INST_INTEG=1"]),
    ("ffma_f64_gmem_integ.o", "ffma_inst.cu", ["-DPINN_INST_REAL=double", "-DPINN_INST_BUFS=0", "-DPINN_INST_INTEG=1"]),
    # and with fixed networks (neural adapters, registered network functions), with or without integral terms
    ("ffma_f32_smem_fixed.o", "ffma_inst.cu", ["-DPINN_INST_REAL=float", "-DPINN_INST_BUFS=1", "-DPINN_INST_INTEG=1",
                                              "-DPINN_INST_FIXED=1"]),
    ("ffma_f32_gmem_fixed.o", "ffma_inst.cu", ["-DPINN_INST_REAL=float", "-DPINN_INST_BUFS=0", "-DPINN_INST_INTEG=1",
                                              "-DPINN_INST_FIXED=1"]),
    ("ffma_f64_smem_fixed.o", "ffma_inst.cu", ["-DPINN_INST_REAL=double", "-DPINN_INST_BUFS=1", "-DPINN_INST_INTEG=1",
                                              "-DPINN_INST_FIXED=1"]),
    ("ffma_f64_gmem_fixed.o", "ffma_inst.cu", ["-DPINN_INST_REAL=double", "-DPINN_INST_BUFS=0", "-DPINN_INST_INTEG=1",
                                              "-DPINN_INST_FIXED=1"]),
    # and with a functional term (integral constraints), with integral terms and fixed networks
    ("ffma_f32_smem_func.o", "ffma_inst.cu", ["-DPINN_INST_REAL=float", "-DPINN_INST_BUFS=1", "-DPINN_INST_INTEG=1",
                                             "-DPINN_INST_FIXED=1", "-DPINN_INST_FUNC=1"]),
    ("ffma_f32_gmem_func.o", "ffma_inst.cu", ["-DPINN_INST_REAL=float", "-DPINN_INST_BUFS=0", "-DPINN_INST_INTEG=1",
                                             "-DPINN_INST_FIXED=1", "-DPINN_INST_FUNC=1"]),
    ("ffma_f64_smem_func.o", "ffma_inst.cu", ["-DPINN_INST_REAL=double", "-DPINN_INST_BUFS=1", "-DPINN_INST_INTEG=1",
                                             "-DPINN_INST_FIXED=1", "-DPINN_INST_FUNC=1"]),
    ("ffma_f64_gmem_func.o", "ffma_inst.cu", ["-DPINN_INST_REAL=double", "-DPINN_INST_BUFS=0", "-DPINN_INST_INTEG=1",
                                             "-DPINN_INST_FIXED=1", "-DPINN_INST_FUNC=1"]),
]
# PINN_MODE_TC_F64: the double instantiations again, with their layer products on the FP64 tensor cores (DMMA)
UNITS += [(obj.replace("ffma_f64_", "ffma_f64_dmma_"), src, defs + ["-DPINN_INST_DMMA=1"])
          for obj, src, defs in UNITS if obj.startswith("ffma_f64_")]


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; the engine has no non-CUDA build")


def _deps_mtime() -> float:
    m = 0.0
    for d in (CSRC, INCLUDE):
        for f in os.listdir(d):
            if f.endswith((".h", ".cuh")):
                m = max(m, os.path.getmtime(os.path.join(d, f)))
    return m


def _extra_units():
    """tensor-core translation units (tc_*.cu)."""
    return [(f[:-3] + ".o", f, []) for f in sorted(os.listdir(CSRC)) if f.startswith("tc_") and f.endswith(".cu")]


def build(verbose: bool = False, force: bool = False, debug: bool = False) -> str:
    """Default: the product library lib/libpinn_b200.so (no instrumentation).
    debug=True: lib/libpinn_b200_debug.so built in build_debug/ with -DPINN_DEBUG (phase timestamps for
    scripts/tc_timeline.py and scripts/tail_timeline.py; select it with PINN_B200_LIB)."""
    objdir, lib, flags = OBJDIR, LIB, list(NVCC_FLAGS)
    if debug:
        objdir = os.path.join(HERE, "build_debug")
        lib = os.path.join(LIBDIR, "libpinn_b200_debug.so")
        flags.append("-DPINN_DEBUG")
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(objdir, exist_ok=True)
    nvcc = _nvcc()
    hdr_m = _deps_mtime()
    units = UNITS + _extra_units()
    jobs = []
    for obj, src, defs in units:
        o = os.path.join(objdir, obj)
        s = os.path.join(CSRC, src)
        if force or not os.path.exists(o) or os.path.getmtime(o) < max(os.path.getmtime(s), hdr_m):
            jobs.append([nvcc, *flags, *defs, "-c", s, "-o", o] + (["-Xptxas", "-v"] if verbose else []))

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        return cmd, r

    if jobs:
        with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as ex:
            for cmd, r in ex.map(run, jobs):
                if verbose:
                    sys.stderr.write(r.stderr)
                if r.returncode != 0:
                    raise RuntimeError("nvcc failed: %s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
    objs = [os.path.join(objdir, u[0]) for u in units]
    if jobs or not os.path.exists(lib) or any(os.path.getmtime(o) > os.path.getmtime(lib) for o in objs):
        cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", lib, *objs, "-ldl"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed: %s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
    return lib


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="-f" in sys.argv, debug="--debug" in sys.argv))
