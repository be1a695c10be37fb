"""Per-iteration cost of the device-resident quasi-Newton driver (pinn_qn_*): wall time per iteration and evaluations
per iteration (profiler off), then, in a second profiled window, the device time of the fused kernels, of the optimizer's
qn_* kernels and of the samplers per iteration (torch.profiler, CUDA activities).  The host gap per evaluation is the
wall time per evaluation minus the device time per evaluation: launch latency plus the one 16-byte
read-back and synchronisation per evaluation.  One JSON line per case, led by a line with the card's name and power limit.
usage: qn_step.py [--iters K] [--out FILE]"""
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

CASES = [("cfg2", "lbfgs", "ffma"), ("cfg2", "lbfgs", "tc_split"), ("cfg2", "bfgs", "ffma"), ("cfg2", "bfgs", "tc_split"),
         ("cfg3", "lbfgs", "ffma"), ("cfg3", "lbfgs", "tc_bf16")]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def make(which, mode):
    cfg = configs.config2() if which == "cfg2" else configs.config3()
    if which == "cfg3":
        cfg.strategy.device_sampler = True     # quasi-Newton needs device-resident point sets
    return npde.symbolic_discretize(cfg.pde_system, cfg.discretization(dtype=np.float32, mode=mode))


def classify(name):
    if "qn_" in name:
        return "qn"
    if "sample" in name:
        return "sampler"
    return "fused"


def run(which, method, mode, iters):
    rep = make(which, mode)
    eng = rep.engine
    eng.qn_begin(rep.flat_init_params, E.QN_LBFGS if method == "lbfgs" else E.QN_BFGS)
    eng.qn_iterate(3)                                    # warm-up: module loads, first shapes
    _, _, _, it0, ev0 = eng.qn_iterate(0)
    l0 = eng.launch_count()
    t0 = time.perf_counter()
    for _ in range(iters):
        f, gn, status, it, ev = eng.qn_iterate(1)
    wall = time.perf_counter() - t0
    n_it, n_ev = it - it0, ev - ev0
    row = {"cfg": which, "method": method, "mode": mode, "n_theta": eng.n_theta, "iters": n_it, "evals": n_ev,
           "evals_per_iter": n_ev / max(n_it, 1), "wall_ms_per_iter": 1e3 * wall / max(n_it, 1),
           "launches_per_iter": (eng.launch_count() - l0) / max(n_it, 1), "loss": f, "status": status}
    if status != E.QN_RUNNING or n_it == 0:
        return row
    from torch.profiler import ProfilerActivity, profile
    _, _, _, it1, ev1 = eng.qn_iterate(0)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            eng.qn_iterate(1)
        torch.cuda.synchronize()
    _, _, _, it2, ev2 = eng.qn_iterate(0)
    dev = {"fused": 0.0, "qn": 0.0, "sampler": 0.0}
    for evt in prof.key_averages():
        t = getattr(evt, "device_time_total", None)
        if t is None:
            t = evt.cuda_time_total
        if t and "Memcpy" not in evt.key and "Memset" not in evt.key:
            dev[classify(evt.key)] += t / 1e3             # us -> ms
    p_it, p_ev = max(it2 - it1, 1), max(ev2 - ev1, 1)
    for k in dev:
        row["device_ms_per_iter_" + k] = dev[k] / p_it
    row["fused_ms_per_eval"] = dev["fused"] / p_ev
    # per evaluation, because the profiled window may take a different number of evaluations per iteration
    row["wall_ms_per_eval"] = 1e3 * wall / max(n_ev, 1)
    row["host_gap_ms_per_eval"] = row["wall_ms_per_eval"] - sum(dev.values()) / p_ev
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("qn_step.py measures on a CUDA device; none is visible")
    torch.cuda.init()
    lines = [json.dumps({"card": card(), "note": "name, power.limit, clocks.max.sm"})]
    print(lines[0], flush=True)
    for which, method, mode in CASES:
        row = run(which, method, mode, a.iters)
        lines.append(json.dumps(row))
        print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
