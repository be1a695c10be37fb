"""Cost of integral terms on the device: device time of one loss + gradient evaluation (the fused kernel, CUDA events)
and wall time per BFGS iteration (the device-resident driver, pinn_qn_*), on the reference's IntegroDiff example 1
(1-D, ∫_0^t, 15-wide sigmoid network) and example 4 (2-D, ∫_0^1 ∫_0^x, 16 x 16 nodes per point), both at
GridTraining(0.01), FFMA fp32 and fp64.  One JSON line per case, led by a line with the card's name and power limit.
usage: ide_step.py [--evals K] [--iters K] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import torch                                    # noqa: E402
import neuralpde_jl_b200 as npde                # noqa: E402
from neuralpde_jl_b200 import engine as E      # noqa: E402
import integral_cases as IC                     # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def run(case, dtype, evals, iters):
    sys_, chains, _ = IC.REFERENCE[case]()
    disc = IC.discretization(chains, 0.01, dtype)
    rep = npde.symbolic_discretize(sys_, disc)
    eng = rep.engine
    th = rep.flat_init_params
    eng.set_timing(True)
    for _ in range(3):
        eng.loss_grad_host(th, None, True)
    ms = []
    for _ in range(evals):
        eng.loss_grad_host(th, None, True)
        ms.append(eng.last_kernel_ms())
    eng.set_timing(False)
    eng.qn_begin(th, E.QN_BFGS)
    t0 = time.perf_counter()
    f, _, status, it, ev = eng.qn_iterate(iters)
    wall = time.perf_counter() - t0
    return {"case": case, "dtype": np.dtype(dtype).name, "owner_points": int(np.prod([round((d.domain.hi - d.domain.lo) / 0.01) + 1
                                                                 for d in sys_.domain])),
            "n_theta": eng.n_theta, "flops_per_eval": eng.flops_per_eval(),
            "kernel_ms_median": float(np.median(ms)), "kernel_ms_min": float(np.min(ms)),
            "bfgs_iters": it, "bfgs_evals": ev, "ms_per_bfgs_iter": 1e3 * wall / max(it, 1),
            "ms_per_bfgs_eval": 1e3 * wall / max(ev - 1, 1), "bfgs_status": status, "loss_after": f}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--evals", type=int, default=50)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ide_step.py measures on a CUDA device; none is visible")
    torch.cuda.init()
    lines = [json.dumps({"card": card(), "note": "name, power.limit, clocks.max.sm"})]
    print(lines[0], flush=True)
    for case in ("ide1", "ide4"):
        for dtype in (np.float32, np.float64):
            lines.append(json.dumps(run(case, dtype, a.evals, a.iters)))
            print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
