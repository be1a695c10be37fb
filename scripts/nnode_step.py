"""NNODE cost on the device: the kernel time of one loss + gradient evaluation (the fused kernel and its tail, CUDA
events, median over --evals), and the wall time per Adam iteration of the host loop (one evaluation and a host update
per iteration) against the device loop (pinn_adam_iterate, chunks of 50), float64; the wall time covers the optimizer
loop only, on a handle built and warmed up before.  Cases, the reference's test/NNODE
problems: Lorenz parameter estimation (1 -> 8 -> 8 -> 3 sigmoid, GridTraining(0.01) and 101 observations), the
Lotka-Volterra WeightedIntervalTraining problem with 400 tstops (1 -> 16 x 4 -> 2 sigmoid), the gelu WeightedInterval
problem (1 -> 64 x 4 -> 2) and ODE Example 3 (1 -> 10 -> 2 sigmoid, 16 Gauss-Legendre nodes).  One JSON line per
(round, case), led by a line with the card's name and power limit.
usage: nnode_step.py [--rounds R] [--evals K] [--iters M] [--out FILE]
(profiles/h100_nnode_step.jsonl: --rounds 3 --evals 100 --iters 1000)"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch                                    # noqa: E402
import neuralpde_jl_b200 as npde                # noqa: E402
from neuralpde_jl_b200.ode import _train         # noqa: E402
from test_nnode_host import chain, example3, lorenz, lotka_volterra   # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def cases():
    t = np.linspace(0.0, 1.0, 101)
    ds = [list(np.cos(t)), list(np.sin(t)), list(t), list(t), list(np.ones(101))]
    rng = np.random.default_rng(100)
    tstops = np.concatenate([rng.random(280), rng.random(80) + 1, rng.random(40) + 2])
    gelu = npde.Chain(npde.Dense(1, 64, "gelu"), *[npde.Dense(64, 64, "gelu") for _ in range(3)], npde.Dense(64, 2))
    return {
        "lorenz_param_estim": (lorenz(), npde.NNODE(chain(3, 8, "sigmoid", 2), npde.Adam(0.01),
                                                    strategy=npde.GridTraining(0.01), dataset=ds, param_estim=True), {}),
        "lv_wit_tstops": (lotka_volterra(), npde.NNODE(chain(2, 16, "sigmoid", 4), npde.Adam(0.01),
                                                       strategy=npde.WeightedIntervalTraining([0.3, 0.3, 0.4], 3)),
                          {"tstops": tstops}),
        "lv_wit_gelu": (lotka_volterra(), npde.NNODE(gelu, npde.Adam(0.01),
                                                     strategy=npde.WeightedIntervalTraining([0.7, 0.2, 0.1], 200)), {}),
        "ode_example_3": (example3(), npde.NNODE(chain(2, 10, "sigmoid"), npde.Adam(0.1)), {}),
    }


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
    return ms


def wall_per_iter(rep, iters, device_loop):
    """the optimizer loop alone (ode._train: no tracing, handle creation or solution building), after a warm-up run
    of the same loop on the same handle"""
    _train(rep, rep.alg.opt, 50, 0.0, False, device_loop, 50)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    _train(rep, rep.alg.opt, iters, 0.0, False, device_loop, 50)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / iters * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--evals", type=int, default=200)
    ap.add_argument("--iters", type=int, default=1000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("nnode_step.py measures on a CUDA device; none is visible")
    torch.cuda.init()
    lines = [json.dumps({"card": card(), "note": "name, power.limit, clocks.max.sm"})]
    print(lines[0], flush=True)
    cs = cases()
    for r in range(a.rounds):
        for name, (prob, alg, kw) in cs.items():
            rep = npde.NNODERepresentation(prob, alg, **kw)
            ms = kernel_ms(rep, a.evals)
            rec = {"round": r, "case": name, "dtype": "float64", "n_theta": rep.engine.n_theta, "terms": len(rep.specs),
                   "points": int(sum(0 if X is None else X.shape[1] for X in rep.point_sets)),
                   "kernel_ms_median": float(np.median(ms)), "kernel_ms_min": float(np.min(ms)),
                   "host_loop_ms_per_iter": wall_per_iter(rep, a.iters, False),
                   "device_loop_ms_per_iter": wall_per_iter(rep, a.iters, True)}
            lines.append(json.dumps(rec))
            print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
