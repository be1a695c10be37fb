"""SDEPINN cost on the device, float64, FFMA kernel, on the shape of the reference's test/NNSDE2 OU problem (2 -> 20 ->
20 -> 1, tanh, tanh, logcosh; 161 x 21 = 3381 Fokker-Planck points, 1 initial point, 2 x 21 flux points and the norm
term's 21 owners x 64 Gauss-Legendre nodes):
- the kernel time of one loss + gradient evaluation (the fused kernel and its tail, CUDA events, median over --evals)
  and the launches it takes;
- the same for the norm term alone in an engine problem of its own (21 owners x 64 nodes in one owner tile), to show
  what share of the evaluation it takes;
- the wall time of one device BFGS iteration (pinn_qn_iterate, --iters iterations from θ0 in one call, which ends in a
  device synchronise) and its launches and loss evaluations per iteration.
One JSON line per (round, case), led by a line with the card's name and power limit.
usage: sdepinn_step.py [--rounds R] [--evals K] [--iters M] [--out FILE]
(profiles/h100_sdepinn_step.jsonl: --rounds 3 --evals 200 --iters 50)"""
import argparse
import dataclasses
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
from neuralpde_jl_b200 import engine as E       # noqa: E402
from neuralpde_jl_b200.sde_weak import SDEPINNProblem      # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def problem():
    prob = npde.SDEProblem(lambda u, p, t: -1 * u, lambda u, p, t: 1, 0.5, (0.0, 1.0))
    ch = npde.Chain(npde.Dense(2, 20, "tanh"), npde.Dense(20, 20, "tanh"), npde.Dense(20, 1, "logcosh"))
    alg = npde.SDEPINN(chain=ch, optimalg=npde.BFGS(), x_0=-4.0, x_end=4.0, distrib=npde.Normal(0.5, 0.05))
    opt_prob = SDEPINNProblem(prob, alg).discretize()
    w = opt_prob.representation.weights
    return opt_prob, np.concatenate([w["pde"], w["bc"], w["add"]])


def norm_engine(opt_prob):
    """the norm term of the problem, on its own"""
    rep = opt_prob.representation
    spec = rep.engine.spec
    i = len(spec.terms) - 1
    alone = E.ProblemSpec(nets=spec.nets, terms=[spec.terms[i]], n_theta=spec.n_theta, dtype=spec.dtype,
                          integrals=[dataclasses.replace(it, owner=0) for it in spec.integrals if it.owner == i])
    eng = E.Engine(alone)
    eng.set_points_host(0, rep.point_sets[i], rep.quad_weights[i])
    return eng


def kernel_ms(eng, th, weights, evals):
    eng.set_timing(True)
    for _ in range(3):
        eng.loss_grad_host(th, weights, True)
    ms = []
    l0 = eng.launch_count()
    for _ in range(evals):
        eng.loss_grad_host(th, weights, True)
        ms.append(eng.last_kernel_ms())
    launches = (eng.launch_count() - l0) / evals
    eng.set_timing(False)
    return float(np.median(ms)), launches


def bfgs_ms(opt_prob, weights, iters):
    eng = opt_prob.representation.engine
    eng.qn_begin(opt_prob.u0, E.QN_BFGS, linesearch=E.LS_HAGERZHANG, weights=weights)
    eng.qn_iterate(0)
    eng.qn_iterate(2)                                   # warm-up
    l0 = eng.launch_count()
    _, _, _, it0, ev0 = eng.qn_iterate(0)
    t = time.perf_counter()
    _, _, status, it, ev = eng.qn_iterate(iters)        # ends in a device synchronise (loss read-back)
    dt = time.perf_counter() - t
    n = max(it - it0, 1)
    return 1e3 * dt / n, (eng.launch_count() - l0) / n, (ev - ev0) / n, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--evals", type=int, default=200)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lines = [{"card": card()}]
    torch.cuda.init()
    opt_prob, weights = problem()
    norm = norm_engine(opt_prob)
    for r in range(a.rounds):
        ms, launches = kernel_ms(opt_prob.representation.engine, opt_prob.u0, weights, a.evals)
        lines.append({"round": r, "case": "ou_loss_grad", "points": 3381 + 1 + 42 + 21 * 64,
                      "kernel_ms_per_eval": ms, "launches_per_eval": launches})
        ms, launches = kernel_ms(norm, opt_prob.u0, None, a.evals)
        lines.append({"round": r, "case": "ou_norm_term_alone", "points": 21 * 64, "kernel_ms_per_eval": ms,
                      "launches_per_eval": launches})
        ms, launches, evals, n = bfgs_ms(opt_prob, weights, a.iters)
        lines.append({"round": r, "case": "ou_device_bfgs", "iterations": n, "ms_per_iter": ms,
                      "launches_per_iter": launches, "evals_per_iter": evals})
        for ln in lines[-3:]:
            print(json.dumps(ln), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
