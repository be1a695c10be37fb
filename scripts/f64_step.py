"""Float64 on the FP64 tensor cores: device time of one loss + gradient evaluation (the fused kernel and its tail, CUDA
events) in mode "ffma" (FP64 FMA pipe) and "tc_f64" (the same kernel with its layer products on DMMA), alternated over
several rounds in one process, with a 256 MB L2 flush before every timed evaluation.  Cases: config 2 (128^2 grid, 4 x 64),
config 3 (65 536 + 3 x 4 096 points, 5 x 128) and config 4 (4 networks, 6 x 256).  The algorithmic rate is the engine's
flops_per_eval (6 C S N summed over terms and networks) over the median kernel time, printed beside the H100 SXM data
sheet's 67 TFLOP/s FP64 tensor and 34 TFLOP/s FP64 vector figures (not reached or measured here).  One JSON line per
(round, case, mode), led by a line with the card's name and power limit.
usage: f64_step.py [--rounds R] [--evals K] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch                                    # noqa: E402
import neuralpde_jl_b200 as npde                # noqa: E402
from neuralpde_jl_b200 import configs           # noqa: E402

DATASHEET_TFLOPS = {"fp64_tensor": 67.0, "fp64_vector": 34.0}
CASES = {"cfg2": (lambda: configs.config2(), 1.0),
         "cfg3": (lambda: configs.config3(), 1.0),
         "cfg4": (lambda: configs.config4(nodes=32, bc_nodes=16), 0.2)}   # slow in fp64: a fifth of the evaluations


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def setup(name, mode):
    cfg = CASES[name][0]()
    rep = npde.symbolic_discretize(cfg.pde_system, cfg.discretization(dtype=np.float64, mode=mode))
    if hasattr(rep.strategy, "points") and rep.point_sets[0] is None:
        rep.loss_functions.full_loss_function(rep.flat_init_params)   # Stochastic: draws and uploads the (fixed) sample
    return rep


def time_evals(rep, evals, flush):
    eng, th = rep.engine, rep.flat_init_params
    eng.set_timing(True)
    for _ in range(3):
        eng.loss_grad_host(th, None, True)
    ms = []
    for _ in range(evals):
        flush.zero_()
        torch.cuda.synchronize()
        eng.loss_grad_host(th, None, True)
        ms.append(eng.last_kernel_ms())
    eng.set_timing(False)
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--evals", type=int, default=50)
    ap.add_argument("--cases", default="cfg2,cfg3,cfg4")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("f64_step.py measures on a CUDA device; none is visible")
    torch.cuda.init()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    lines = [json.dumps({"card": card(), "note": "name, power.limit, clocks.max.sm",
                         "datasheet_tflops": DATASHEET_TFLOPS})]
    print(lines[0], flush=True)
    reps = {(c, m): setup(c, m) for c in a.cases.split(",") for m in ("ffma", "tc_f64")}
    for r in range(a.rounds):
        for (c, m), rep in reps.items():
            ms = time_evals(rep, max(3, int(a.evals * CASES[c][1])), flush)
            med = float(np.median(ms))
            fl = rep.engine.flops_per_eval()
            lines.append(json.dumps({"round": r, "case": c, "mode": m, "dtype": "float64", "n_theta": rep.engine.n_theta,
                                     "evals": len(ms), "kernel_ms_median": med, "kernel_ms_min": float(np.min(ms)),
                                     "flops_per_eval": fl, "algorithmic_tflops": fl / med * 1e-9}))
            print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
