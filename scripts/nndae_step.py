"""NNDAE cost on the device: the kernel time of one loss + gradient evaluation (the fused kernel and its tail, CUDA
events, median over --evals) with the launches it takes, and the wall time per Adam iteration of the host loop (one
evaluation and a host update per iteration) against the device loop (pinn_adam_iterate, chunks of 50), float64; the
wall time covers the optimizer loop only, on a handle built and warmed up before.  Cases, the reference's test/NNODE
DAE problems: Case I (1 -> 15 cos -> 15 sin -> 2, 101 grid points) and Case II (1 -> 15 sigmoid -> 2, 158 grid
points), each one functional term.  One JSON line per (round, case), led by a line with the card's name and power limit.
usage: nndae_step.py [--rounds R] [--evals K] [--iters M] [--out FILE]
(profiles/h100_nndae_step.jsonl: --rounds 3 --evals 200 --iters 1000)"""
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
from nndae_oracle import DT, case_i, case_ii     # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def cases():
    out = {}
    for name, case, lr in (("dae_case_i", case_i, 0.01), ("dae_case_ii", case_ii, 0.1)):
        prob, chain = case()
        out[name] = (prob, npde.NNDAE(chain, npde.Adam(lr)))
    return out


def kernel_ms(rep, evals):
    """(per-evaluation kernel times, launches per evaluation)"""
    eng, th = rep.engine, rep.flat_init_params
    eng.set_timing(True)
    for _ in range(3):
        rep.loss_grad(th)
    ms = []
    l0 = eng.launch_count()
    for _ in range(evals):
        rep.loss_grad(th)
        ms.append(eng.last_kernel_ms())
    launches = (eng.launch_count() - l0) / evals
    eng.set_timing(False)
    return ms, launches


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
        raise SystemExit("nndae_step.py measures on a CUDA device; none is visible")
    torch.cuda.init()
    lines = [json.dumps({"card": card(), "note": "name, power.limit, clocks.max.sm"})]
    print(lines[0], flush=True)
    cs = cases()
    for r in range(a.rounds):
        for name, (prob, alg) in cs.items():
            rep = npde.NNDAERepresentation(prob, alg, dt=DT)
            ms, launches = kernel_ms(rep, a.evals)
            rec = {"round": r, "case": name, "dtype": "float64", "n_theta": rep.engine.n_theta, "terms": len(rep.specs),
                   "points": int(rep.ts.size), "kernel_ms_median": float(np.median(ms)),
                   "kernel_ms_min": float(np.min(ms)), "launches_per_eval": launches,
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
