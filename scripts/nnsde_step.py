"""NNSDE cost on the device, float64, FFMA kernel, for test/NNSDE1 test 2's shape (GBM, 4 -> 16 -> 16 -> 1 sigmoid,
n_z = 3, 51 times x sub_batch 10 = 510 points):
- the kernel time of one loss + gradient evaluation (the fused kernel and its tail, CUDA events, median over --evals),
  weak (one MEAN term) and strong (one WSUM term) GridTraining;
- the wall time per device Adam iteration (pinn_adam_iterate, chunks of 50) of StochasticTraining(51) with sub_batch 10,
  which redraws the 510 points with the KKL sampler before every step (one sampler launch + one fused launch);
- the KKL sampler kernel alone (CUDA events around --evals pinn_resample calls, per call).
One JSON line per (round, case), led by a line with the card's name and power limit.
usage: nnsde_step.py [--rounds R] [--evals K] [--iters M] [--out FILE]
(profiles/h100_nnsde_step.jsonl: --rounds 3 --evals 200 --iters 1000)"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch                                    # noqa: E402
import neuralpde_jl_b200 as npde                # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def problem():
    return npde.SDEProblem(lambda u, p, t: 1.2 * u, lambda u, p, t: 1.1 * u, 0.5, (0.0, 1.0))


def chain():
    return npde.Chain(npde.Dense(4, 16, "sigmoid"), npde.Dense(16, 16, "sigmoid"), npde.Dense(16, 1))


def rep_of(strategy, strong):
    return npde.NNSDERepresentation(problem(), npde.NNSDE(chain(), npde.Adam(1e-3), strategy=strategy, sub_batch=10,
                                                          strong_loss=strong, seed=100))


def kernel_ms(rep, evals):
    eng, th = rep.engine, rep.flat_init_params
    eng.set_timing(True)
    for _ in range(3):
        rep.loss_grad(th)
    ms = []
    for _ in range(evals):
        rep.loss_grad(th)
        ms.append(eng.last_kernel_ms())
    eng.set_timing(False)
    return float(np.median(ms))


def adam_us(rep, iters):
    eng = rep.engine
    eng.adam_begin(rep.flat_init_params, 1e-3)
    eng.adam_iterate(50, rep.term_weights)              # warm-up: graph capture
    l0 = eng.launch_count()
    t = time.perf_counter()
    for _ in range(iters // 50):
        eng.adam_iterate(50, rep.term_weights)          # ends in a device synchronise (loss read-back)
    dt = time.perf_counter() - t
    return 1e6 * dt / (iters // 50 * 50), (eng.launch_count() - l0) / (iters // 50 * 50)


def sampler_us(rep, evals):
    eng = rep.engine
    for _ in range(10):
        eng.resample()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(torch.cuda.default_stream())
    for _ in range(evals):
        eng.resample()
    b.record(torch.cuda.default_stream())
    b.synchronize()
    return 1e3 * a.elapsed_time(b) / evals


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--evals", type=int, default=200)
    ap.add_argument("--iters", type=int, default=1000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lines = [{"card": card()}]
    torch.cuda.init()
    grid = {s: rep_of(npde.GridTraining(1 / 50), s) for s in (False, True)}
    stoch = rep_of(npde.StochasticTraining(51, seed=3), False)
    for r in range(a.rounds):
        for strong in (False, True):
            lines.append({"round": r, "case": "grid_%s" % ("strong" if strong else "weak"), "points": 510,
                          "kernel_ms_per_eval": kernel_ms(grid[strong], a.evals)})
        us, launches = adam_us(stoch, a.iters)
        lines.append({"round": r, "case": "stochastic_weak_device_adam", "points": 510, "us_per_iter": us,
                      "launches_per_iter": launches})
        lines.append({"round": r, "case": "kkl_sampler", "points": 510, "us_per_draw": sampler_us(stoch, a.evals)})
        for ln in lines[-4:]:
            print(json.dumps(ln), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
