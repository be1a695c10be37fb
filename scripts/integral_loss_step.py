"""Cost of an integral constraint on the device: device time of one loss + gradient evaluation (the fused kernel and its
tail, CUDA events, median) of the reference's Fokker-Planck problem (GridTraining(0.01), 3 x 18 sigmoid network) with
and without its normalisation constraint (IntegralLoss, 16 Gauss-Legendre nodes), FFMA fp32 and fp64.  One JSON line
per case, led by a line with the card's name and power limit.
usage: integral_loss_step.py [--evals K] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch                                    # noqa: E402
import neuralpde_jl_b200 as npde                # noqa: E402
import integral_loss_cases as LC                # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def run(constraint, dtype, evals):
    sys_, chains, strategy, add, _ = LC.fokker_planck()
    disc = LC.discretization((sys_, chains, strategy, add if constraint else None, False), dtype)
    rep = npde.symbolic_discretize(sys_, disc)
    eng = rep.engine
    th = rep.flat_init_params
    eng.set_timing(True)
    for _ in range(5):
        eng.loss_grad_host(th, None, True)
    ms = []
    for _ in range(evals):
        eng.loss_grad_host(th, None, True)
        ms.append(eng.last_kernel_ms())
    eng.set_timing(False)
    return {"case": "fokker_planck", "constraint": constraint, "dtype": np.dtype(dtype).name,
            "terms": rep.term_names, "n_theta": eng.n_theta, "flops_per_eval": eng.flops_per_eval(),
            "kernel_ms_median": float(np.median(ms)), "kernel_ms_min": float(np.min(ms))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--evals", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("integral_loss_step.py measures on a CUDA device; none is visible")
    torch.cuda.init()
    lines = [json.dumps({"card": card(), "note": "name, power.limit, clocks.max.sm"})]
    print(lines[0], flush=True)
    for dtype in (np.float32, np.float64):
        for constraint in (False, True):
            lines.append(json.dumps(run(constraint, dtype, a.evals)))
            print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
