"""Per-transition cost of the device-resident HMC sampler (pinn_hmc_*): wall time per transition and per leapfrog step
(profiler off, graph replay, one read-back per call), launches per transition, then, in a second profiled window, the
share of device time spent in the fused kernels (torch.profiler, CUDA activities).  Cases: the reference's 2-D Poisson
BayesianPINN test (iv_2d_poisson: 2 -> 9 -> 9 -> 1 sigmoid, GridTraining(0.04), FFMA fp32), config 2 (tc_split) and the
reference's inverse Lorenz test (inv_ii_lorenz: three 1 -> 7 -> 7 -> 1 tanh networks, GridTraining(0.01), a 21-point
dataset per variable, σ_ estimated under a Normal(12, 2) prior, FFMA fp32).
The chains run with a fixed step of 1e-5 and no adaptation, so that no trajectory stops early at a non-finite value and
every transition does the full 30 steps.  One JSON line per case, led by a line with the card's name and power limit.
usage: hmc_step.py [--transitions K] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch                                    # noqa: E402
import neuralpde_jl_b200 as npde                # noqa: E402
from neuralpde_jl_b200 import configs, engine as E   # noqa: E402

N_LEAPFROG = 30


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def make(case):
    if case == "iv_2d_poisson":
        cfg = configs.config2(n=26)
        chain = npde.Chain(npde.Dense(2, 9, "sigmoid"), npde.Dense(9, 9, "sigmoid"), npde.Dense(9, 1))
        init = npde.initialparameters(np.random.default_rng(0), chain, np.float32)
        disc = npde.BayesianPINN([chain], npde.GridTraining(0.04), init_params=init, mode="ffma")
        std = [[0.003], [0.003] * 4, [0.05]]
    elif case == "inv_ii_lorenz":
        sys_, chains, data = configs.lorenz_bpinn()
        rng = np.random.default_rng(0)
        init = np.concatenate([npde.initialparameters(rng, c, np.float32) for c in chains] + [np.ones(1, np.float32)])
        disc = npde.BayesianPINN(chains, npde.GridTraining([0.01]), init_params=init, mode="ffma", param_estim=True,
                                 dataset=[data, None])
        rep = npde.symbolic_discretize(sys_, disc)
        return rep, [[0.1] * 3, [0.3] * 3, [1.0] * 3], [(E.HMC_PRIOR_NORMAL, 12.0, 2.0)]
    else:
        cfg = configs.config2()
        disc = npde.BayesianPINN(cfg.chains[0], cfg.strategy, init_params=cfg.init_params(np.float32), mode="tc_split")
        std = [[0.05], [0.05] * 4, [0.05]]
    rep = npde.symbolic_discretize(cfg.pde_system, disc)
    return rep, std, None


def run(case, transitions):
    rep, std, tail = make(case)
    eng = rep.engine
    c, const = rep.loglik_weights(std, data=True)
    th0 = rep.flat_init_params.astype(np.float64)
    if tail:
        th0[-len(tail):] = [a for _, a, _ in tail]
    eng.hmc_begin(th0, n_leapfrog=N_LEAPFROG, adaptor=E.HMC_ADAPT_NONE, metric=E.HMC_METRIC_UNIT,
                  step_size=1e-5, prior_std=10.0, weights=c, ll_const=const, tail_priors=tail)
    eng.hmc_iterate(5)                                   # warm-up: graph capture, module loads
    l0 = eng.launch_count()
    t0 = time.perf_counter()
    _, st = eng.hmc_iterate(transitions)
    wall = time.perf_counter() - t0
    ms = 1e3 * wall / transitions
    row = {"case": case, "mode": ["ffma", "tc_bf16", "tc_split"][eng.spec.mode],
           "dtype": eng.spec.dtype, "n_theta": eng.n_theta, "transitions": transitions, "n_leapfrog": N_LEAPFROG,
           "ms_per_transition": ms, "ms_per_leapfrog_step": ms / N_LEAPFROG,
           "launches_per_transition": (eng.launch_count() - l0) / transitions,
           "acceptance_rate": float(np.mean(st[:, 1])), "numerical_errors": int(st[:, 6].sum())}
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.hmc_iterate(transitions)
        torch.cuda.synchronize()
    fused = other = 0.0
    for evt in prof.key_averages():
        t = getattr(evt, "device_time_total", None)
        if t is None:
            t = evt.cuda_time_total
        if not t or "Memcpy" in evt.key or "Memset" in evt.key:
            continue
        if "hmc_" in evt.key:
            other += t
        else:
            fused += t
    row["device_ms_per_transition"] = (fused + other) / 1e3 / transitions
    row["fused_share_of_device_time"] = fused / max(fused + other, 1e-30)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--transitions", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("hmc_step.py measures on a CUDA device; none is visible")
    torch.cuda.init()
    lines = [json.dumps({"card": card(), "note": "name, power.limit, clocks.max.sm"})]
    print(lines[0], flush=True)
    for case in ("iv_2d_poisson", "cfg2", "inv_ii_lorenz"):
        lines.append(json.dumps(run(case, a.transitions)))
        print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
