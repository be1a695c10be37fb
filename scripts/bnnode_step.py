"""Per-transition cost of ahmc_bayesian_pinn_ode's device chain: wall time per transition and per leapfrog step
(graph replay, one read-back per call) and launches per transition.  Cases: the reference's ODEBPINN test i
(u' = cos 2πt on [0, 2], 1 -> 7 -> 1 tanh, GridTraining(1/20)), the same problem under StochasticTraining(100), which
draws fresh times on the device before every evaluation (PINN_HMC_REDRAW), and test iv (Lotka-Volterra, 1 -> 7 -> 7 -> 2
tanh, GridTraining(1/20), a 20-point dataset, estim_collocate, two Normal priors on θ.p), all FFMA fp64.
The chains run with a fixed step of 1e-5 and no adaptation, so that every transition does the full 30 steps.  One JSON
line per case, led by a line with the card's name and power limit.
usage: bnnode_step.py [--transitions K] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import sympy as sp

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch                                    # noqa: E402
import neuralpde_jl_b200 as npde                # noqa: E402
from neuralpde_jl_b200 import engine as E      # noqa: E402

N_LEAPFROG = 30


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def make(case):
    if case in ("i_grid", "i_stochastic"):
        prob = npde.ODEProblem(lambda u, p, t: sp.cos(2 * sp.pi * t), 0.0, (0.0, 2.0))
        chain = npde.Chain(npde.Dense(1, 7, "tanh"), npde.Dense(7, 1))
        strategy = npde.GridTraining if case == "i_grid" else npde.StochasticTraining(100)
        return npde.BNNODELogDensity(prob, chain, strategy=strategy)

    def lv(u, p, t):
        return [(p[0] - u[1]) * u[0], (u[0] - p[1]) * u[1]]
    prob = npde.ODEProblem(lv, [1.0, 1.0], (0.0, 4.0), [1.5, 3.0])
    chain = npde.Chain(npde.Dense(1, 7, "tanh"), npde.Dense(7, 7, "tanh"), npde.Dense(7, 2))
    t = np.linspace(0.0, 4.0, 20)
    data = [1.0 + 0.5 * np.sin(t), 1.0 + 0.5 * np.cos(t), t, np.full(20, 0.2)]
    return npde.BNNODELogDensity(prob, chain, dataset=data, l2std=[0.5, 0.5], phystd=[0.5, 0.5],
                                 phynewstd=lambda p: [0.5, 0.5], param=[npde.Normal(-7, 2), npde.Normal(-7, 2)],
                                 estim_collocate=True)


def run(case, transitions):
    ld = make(case)
    eng = ld.engine
    eng.hmc_begin(ld.theta0, n_leapfrog=N_LEAPFROG, adaptor=E.HMC_ADAPT_NONE, metric=E.HMC_METRIC_UNIT,
                  step_size=1e-5, prior_std=2.0, weights=ld.c, ll_const=ld.const, tail_priors=ld.tail or None,
                  tail_logabs=ld.tail_logabs, redraw=bool(ld.sampled))
    eng.hmc_iterate(5)                                   # warm-up: graph capture, module loads
    l0 = eng.launch_count()
    t0 = time.perf_counter()
    _, st = eng.hmc_iterate(transitions)
    wall = time.perf_counter() - t0
    ms = 1e3 * wall / transitions
    return {"case": case, "mode": "ffma", "dtype": eng.spec.dtype, "n_theta": eng.n_theta, "terms": len(ld.specs),
            "sampled_terms": len(ld.sampled), "transitions": transitions, "n_leapfrog": N_LEAPFROG,
            "ms_per_transition": ms, "ms_per_leapfrog_step": ms / N_LEAPFROG,
            "launches_per_transition": (eng.launch_count() - l0) / transitions,
            "acceptance_rate": float(np.mean(st[:, 1])), "numerical_errors": int(st[:, 6].sum())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--transitions", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bnnode_step.py measures on a CUDA device; none is visible")
    torch.cuda.init()
    lines = [json.dumps({"card": card(), "note": "name, power.limit, clocks.max.sm"})]
    print(lines[0], flush=True)
    for case in ("i_grid", "i_stochastic", "iv_lotka_volterra"):
        lines.append(json.dumps(run(case, a.transitions)))
        print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
