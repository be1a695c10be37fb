"""Compare the device HMC chain of this checkout with another checkout of the project (for example its parent commit),
both with their libraries built: `scripts/hmc_step.py` of the two trees alternated R rounds in one call (time and
launches per transition of its fixed-point chains), then two seeded chains of each tree (the 2-D Poisson and the
inverse Lorenz BayesianPINN of hmc_step.py, find_good_stepsize and 10 Stan-adapted transitions of 30) compared bit for
bit: step size, samples and statistics.  Each tree runs in its own process with its own package and library.
One JSON line per measurement, led by hmc_step.py's card line; the last line holds the bit comparison.
usage: hmc_compare_builds.py --other ROOT [--rounds R] [--transitions K] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# runs in the tree given as argv[1]: two seeded chains, saved to argv[2]
CHAINS = r"""
import importlib.util, os, sys
import numpy as np
root, out = sys.argv[1], sys.argv[2]
sys.path.insert(0, root)
spec = importlib.util.spec_from_file_location("hmc_step", os.path.join(root, "scripts", "hmc_step.py"))
hs = importlib.util.module_from_spec(spec)
spec.loader.exec_module(hs)
res = {}
for case in ("iv_2d_poisson", "inv_ii_lorenz"):
    rep, std, tail = hs.make(case)
    c, const = rep.loglik_weights(std, data=True)
    th0 = rep.flat_init_params.astype(np.float64)
    if tail:
        th0[-len(tail):] = [a for _, a, _ in tail]
    eps = rep.engine.hmc_begin(th0, n_leapfrog=30, n_adapts=10, prior_std=2.0, seed=4, weights=c, ll_const=const,
                               tail_priors=tail)
    s, st = rep.engine.hmc_iterate(30)
    res[case + "_eps"], res[case + "_samples"], res[case + "_stats"] = np.array([eps]), s, st
np.savez(out, **res)
"""


def step_lines(root, transitions):
    r = subprocess.run([sys.executable, os.path.join("scripts", "hmc_step.py"), "--transitions", str(transitions)],
                       cwd=root, capture_output=True, text=True, check=True)
    out = []
    for line in r.stdout.splitlines():
        try:
            out.append(json.loads(line))
        except ValueError:
            pass
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other", required=True, help="root of the other checkout (library built)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--transitions", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    trees = {"other": os.path.abspath(a.other), "this": HERE}
    lines = []
    for r in range(1, a.rounds + 1):
        for build, root in trees.items():
            for d in step_lines(root, a.transitions):
                if "card" in d:
                    if not lines:
                        lines.append(d)
                    continue
                lines.append({"build": build, "round": r, "case": d["case"],
                              "ms_per_transition": round(d["ms_per_transition"], 4),
                              "launches_per_transition": d["launches_per_transition"]})
                print(json.dumps(lines[-1]), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        got = {}
        for build, root in trees.items():
            path = os.path.join(tmp, build + ".npz")
            subprocess.run([sys.executable, "-c", CHAINS, root, path], check=True)
            got[build] = np.load(path)
        equal = {k: bool(np.array_equal(got["other"][k], got["this"][k])) for k in got["this"].files}
    lines.append({"bits": "two seeded chains (iv_2d_poisson, inv_ii_lorenz: 30 transitions, 10 Stan-adapted), "
                          "step size / samples / statistics array_equal between the two trees", "equal": equal})
    print(json.dumps(lines[-1]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write("\n".join(json.dumps(x) for x in lines) + "\n")


if __name__ == "__main__":
    main()
