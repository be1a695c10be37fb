"""Alternate bench.py between builds of the library in one process tree, so that the builds see the same card and load.

    python scripts/bench_alternate.py --build parent=PATH/libpinn_b200.so --build new=PATH/libpinn_b200.so \
        [--rounds 3] [--steps 200] [--warmup 5] [--out FILE] [--args "ARGS" ...]

Every round runs every --args set on every build in turn (PINN_B200_LIB selects the library) and writes bench.py's JSON
line tagged with "build" and "args".  The first line names the card, its power limit and its maximum SM clock.
Default --args sets: cfg 2 in tc_split (with the other modes), cfg 2 in tc_bf16, cfg 3.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULT_ARGS = ["--no-cpu-baseline", "--mode tc_bf16 --no-alt-modes --no-cpu-baseline", "--config cfg3 --no-cpu-baseline"]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--build", action="append", required=True, metavar="NAME=LIB")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--args", action="append", default=None, help="one bench.py argument set (repeatable)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    builds = [b.split("=", 1) for b in a.build]
    for name, lib in builds:
        if not os.path.exists(lib):
            sys.exit("no such library: %s" % lib)
    out = open(a.out, "w") if a.out else sys.stdout
    out.write(json.dumps({"card": card(), "builds": dict(builds)}) + "\n")
    for _ in range(a.rounds):
        for name, lib in builds:
            for args in a.args or DEFAULT_ARGS:
                cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(a.steps), "--warmup", str(a.warmup)]
                r = subprocess.run(cmd + args.split(), capture_output=True, text=True, cwd=ROOT,
                                   env=dict(os.environ, PINN_B200_LIB=os.path.abspath(lib)))
                lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
                if r.returncode != 0 or not lines:
                    sys.exit("bench.py %s failed on build %s:\n%s" % (args, name, r.stderr[-2000:]))
                rec = json.loads(lines[-1])
                rec["build"], rec["args"] = name, args
                out.write(json.dumps(rec) + "\n")
                out.flush()


if __name__ == "__main__":
    main()
