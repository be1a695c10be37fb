"""Kernel time per evaluation (loss + gradient) of neural adapter problems on the GPU: the cost of evaluating the
teachers inside the fused kernel.

  one_teacher    the 2-D Poisson adapter (test/NeuralAdapter/neural_adapter__neural_adapter_2d_poisson.jl): student and
                 teacher Chain(Dense(2, 8, tanh), Dense(8, 8, tanh), Dense(8, 1)), GridTraining(0.01) on the unit square
  ten_teachers   the domain decomposition's list form: ten teachers over ten x-strips, one term each,
                 GridTraining([0.001, 0.01]), the 18-wide 4-hidden-layer student
  precomputed    one_teacher with the teacher's values as a precomputed point row instead (mean(abs2, u(X) - row)):
                 what the same loss costs without the in-kernel teacher

Prints one JSON line per case (median of CUDA-event kernel times over --evals evaluations), with the GPU's name and
power limit.  Usage: python scripts/adapter_step.py [--evals 200] [--dtype float32]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import neuralpde_jl_b200 as npde                                     # noqa: E402
from neuralpde_jl_b200 import engine as E                            # noqa: E402
from neuralpde_jl_b200.strategies import adapter_training_set        # noqa: E402


def _chain(dims):
    acts = ["tanh"] * (len(dims) - 2) + ["identity"]
    return npde.Chain(*[npde.Dense(a, b, f) for a, b, f in zip(dims[:-1], dims[1:], acts)])


def _teacher(dims, seed, name):
    c = _chain(dims)
    th = npde.initialparameters(np.random.default_rng(seed), c)
    return npde.register_symbolic(npde.Phi(c, 0, c.n_params, np.float64), th, name)


def _time(eng, theta, evals):
    for _ in range(20):
        eng.loss_grad_host(theta, None, True)
    eng.set_timing(True)
    ms = []
    for _ in range(evals):
        eng.loss_grad_host(theta, None, True)
        ms.append(eng.last_kernel_ms())
    eng.set_timing(False)
    return float(np.median(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--evals", type=int, default=200)
    ap.add_argument("--dtype", default="float32")
    a = ap.parse_args()
    dt = np.dtype(a.dtype)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    x, y = npde.parameters("x y")
    u = npde.variables("u")
    Dxx, Dyy = npde.Differential(x) ** 2, npde.Differential(y) ** 2
    eq = npde.Eq(Dxx(u(x, y)) + Dyy(u(x, y)), 0)

    def system(x0, x1):
        return npde.PDESystem([eq], [npde.Eq(u(0, y), 0)], [npde.In(x, x0, x1), npde.In(y, 0.0, 1.0)], [x, y], [u(x, y)])

    out = []
    small = [2, 8, 8, 1]
    student = _chain(small)
    th = npde.initialparameters(np.random.default_rng(1), student).astype(dt)
    pt = _teacher(small, 0, "phi")
    prob = npde.neural_adapter(npde.NeuralAdapterLoss(student, pt(x, y)), th, system(0.0, 1.0), npde.GridTraining(0.01))
    eng = prob.representation.engine
    n = adapter_training_set(system(0.0, 1.0).domain, 0.01, np.float64).shape[1]
    out.append(dict(case="one_teacher", points=n, kernel_ms=_time(eng, th, a.evals), flops=eng.flops_per_eval()))

    # the same loss with the teacher's values as a third point row
    pts = adapter_training_set(system(0.0, 1.0).domain, 0.01, np.float64)
    tv = npde.Phi(_chain(small), 0, student.n_params, np.float64)
    vals = tv(pts, pt.fixed_net.params).reshape(1, -1)
    spec = E.ProblemSpec(nets=[E.NetSpec(small, student.acts, 0)],
                         terms=[E.TermSpec(dim=3, taps=[E.TapSpec(net=0)], net_rows=[[0, 1]],
                                           prog=[("tap", 0, 0, 0.0), ("coord", 2, 0, 0.0), ("sub", 0, 1, 0.0)])],
                         n_theta=student.n_params, dtype=dt.name)
    e2 = E.Engine(spec)
    e2.set_points_host(0, np.concatenate([pts, vals]))
    out.append(dict(case="precomputed", points=n, kernel_ms=_time(e2, th, a.evals), flops=e2.flops_per_eval()))

    wide = [2, 18, 18, 18, 18, 1]
    student = _chain(wide)
    th = npde.initialparameters(np.random.default_rng(2), student).astype(dt)
    losses, systems = [], []
    for i in range(10):
        losses.append(npde.NeuralAdapterLoss(student, _teacher(small, 10 + i, "phi_%d" % i)(x, y)))
        systems.append(system(i / 10, (i + 1) / 10))
    prob = npde.neural_adapter(losses, th, systems, npde.GridTraining([0.001, 0.01]))
    eng = prob.representation.engine
    n = sum(adapter_training_set(s.domain, [0.001, 0.01], np.float64).shape[1] for s in systems)
    out.append(dict(case="ten_teachers", points=n, kernel_ms=_time(eng, th, a.evals), flops=eng.flops_per_eval()))
    for r in out:
        r.update(dtype=dt.name, evals=a.evals, gpu=gpu)
        print(json.dumps(r))


if __name__ == "__main__":
    main()
