"""The reference's test/NeuralAdapter/ group on the device, at its stated bounds (∞-norm against the analytic solution
on the 0.01 grid), and the optimizers of `solve` on a neural adapter problem.

- neural_adapter__neural_adapter_2d_poisson.jl: a 2-D Poisson PINN (5e-2), then a new network fitted to it with
  `neural_adapter` under Grid, Quadrature, Stochastic and QuasiRandom training (8e-2 each);
- neural_adapter__neural_adapter_2d_poisson_domain_decomposition.jl: ten sub-domain PINNs solved one after another, each
  bc at the sub-domain's left edge reading the previous sub-domain's trained network through `register_symbolic` (the
  composed solution: 5e-2), then the list form of `neural_adapter` merging the ten into one network, on the
  sub-domains' grid and then on the 0.01 grid (5e-2 after each stage).

Initial parameters come from this project's RNG (numpy, seed 100), not Julia's."""
import numpy as np
import pytest
import sympy as sp

import neuralpde_jl_b200 as npde
from neuralpde_jl_b200.strategies import _julia_range

pytestmark = pytest.mark.gpu

x, y = npde.parameters("x y")
u = npde.variables("u")
Dxx, Dyy = npde.Differential(x) ** 2, npde.Differential(y) ** 2
EQ = npde.Eq(Dxx(u(x, y)) + Dyy(u(x, y)), -sp.sin(sp.pi * x) * sp.sin(sp.pi * y))


def analytic(xv, yv):
    return np.sin(np.pi * xv) * np.sin(np.pi * yv) / (2 * np.pi ** 2)


def analytic_expr(xv, yv):
    return sp.sin(sp.pi * xv) * sp.sin(sp.pi * yv) / (2 * sp.pi ** 2)


def _chain(widths):
    acts = ["tanh"] * (len(widths) - 2) + [None]
    return npde.Chain(*[npde.Dense(a, b, f) for a, b, f in zip(widths[:-1], widths[1:], acts)])


GRID = np.stack(np.meshgrid(_julia_range(0.0, 0.01, 1.0), _julia_range(0.0, 0.01, 1.0), indexing="ij")).reshape(2, -1)


def _err(chain, theta, pts=GRID):
    pred = npde.Phi(chain, 0, chain.n_params, np.float64)(pts, theta).reshape(-1)
    return float(np.max(np.abs(pred - analytic(pts[0], pts[1]))))


def _train(prob, iters):
    return npde.solve(prob, npde.Adam(5e-3), maxiters=iters, device_loop=True)


@pytest.fixture(scope="module")
def poisson():
    """the 2-D Poisson PINN of the adapter test: QuadratureTraining, Adam(5e-3) for 2000 iterations"""
    rng = np.random.default_rng(100)
    chain1 = _chain([2, 8, 8, 1])
    bcs = [npde.Eq(u(0, y), 0.0), npde.Eq(u(1, y), -sp.sin(sp.pi) * sp.sin(sp.pi * y)),
           npde.Eq(u(x, 0), 0.0), npde.Eq(u(x, 1), -sp.sin(sp.pi * x) * sp.sin(sp.pi))]
    sys_ = npde.PDESystem([EQ], bcs, [npde.In(x, 0.0, 1.0), npde.In(y, 0.0, 1.0)], [x, y], [u(x, y)])
    disc = npde.PhysicsInformedNN(chain1, npde.QuadratureTraining(),
                                  init_params=npde.initialparameters(rng, chain1))
    prob = npde.discretize(sys_, disc)
    res = _train(prob, 2000)
    return sys_, chain1, res, prob.representation.phi, rng


def test_poisson_pinn(poisson):
    _, chain1, res, _, _ = poisson
    e = _err(chain1, res.u)
    print("2-D Poisson PINN: inf-norm error %.3e (bound 5e-2)" % e)
    assert e <= 5e-2


@pytest.mark.parametrize("strategy", [npde.GridTraining(0.05), npde.QuadratureTraining(),
                                      npde.StochasticTraining(1000, seed=1),
                                      npde.QuasiRandomTraining(1000, minibatch=200, resampling=True, seed=2)],
                         ids=["grid", "quadrature", "stochastic", "quasirandom"])
def test_adapter_strategies(poisson, strategy):
    sys_, _, res, phi, _ = poisson
    chain2 = _chain([2, 8, 8, 1])
    init2 = npde.initialparameters(np.random.default_rng(101), chain2)
    teacher = npde.register_symbolic(phi, res.u, "phi")
    prob = npde.neural_adapter(npde.NeuralAdapterLoss(chain2, teacher(x, y)), init2, sys_, strategy)
    res_ = _train(prob, 1500)
    e = _err(chain2, res_.u)
    print("adapter %s: inf-norm error %.3e (bound 8e-2)" % (type(strategy).__name__, e))
    assert e <= 8e-2


def test_solve_paths_on_an_adapter(poisson):
    """the host Adam loop and the device loop take the same steps; BFGS and L-BFGS run on the device and lower the loss"""
    sys_, _, res, phi, _ = poisson
    chain2 = _chain([2, 8, 8, 1])
    init2 = npde.initialparameters(np.random.default_rng(102), chain2)
    loss = npde.NeuralAdapterLoss(chain2, npde.register_symbolic(phi, res.u, "phi")(x, y))
    host = npde.solve(npde.neural_adapter(loss, init2, sys_, npde.GridTraining(0.05)), npde.Adam(5e-3), maxiters=20)
    dev = _train(npde.neural_adapter(loss, init2, sys_, npde.GridTraining(0.05)), 20)
    np.testing.assert_allclose(dev.u, host.u, rtol=1e-9, atol=1e-12)
    prob = npde.neural_adapter(loss, init2, sys_, npde.GridTraining(0.05))
    f0 = prob.f.f(init2)
    for opt in (npde.BFGS(), npde.LBFGS()):
        sol = npde.solve(npde.neural_adapter(loss, init2, sys_, npde.GridTraining(0.05)), opt, maxiters=30)
        assert sol.retcode in ("Success", "MaxIters") and sol.objective < 0.1 * f0, (opt, sol.retcode, sol.objective, f0)
        assert sol.u.shape == init2.shape


def test_domain_decomposition():
    rng = np.random.default_rng(100)
    n_dec = 10
    edges = [i / n_dec for i in range(n_dec + 1)]
    chains = [_chain([2, 8, 8, 1]) for _ in range(n_dec)]
    reses, phis, systems = [], [], []
    for i in range(n_dec):
        x0, xe = edges[i], edges[i + 1]
        doms = [npde.In(x, x0, xe), npde.In(y, 0.0, 1.0)]
        if i == 0:
            left = npde.Eq(u(0, y), 0.0)
        else:
            phi_bound = npde.register_symbolic(phis[i - 1], reses[i - 1].u, "phi_bound")
            left = npde.Eq(u(x0, y), phi_bound(x0, y))
        bcs = [left, npde.Eq(u(xe, y), analytic_expr(xe, y)), npde.Eq(u(x, 0), 0.0),
               npde.Eq(u(x, 1), -sp.sin(sp.pi * x) * sp.sin(sp.pi))]
        sys_ = npde.PDESystem([EQ], bcs, doms, [x, y], [u(x, y)])
        systems.append(sys_)
        disc = npde.PhysicsInformedNN(chains[i], npde.GridTraining([0.1 / n_dec, 0.1]),
                                      init_params=npde.initialparameters(rng, chains[i]))
        prob = npde.discretize(sys_, disc)
        reses.append(_train(prob, 2000))
        phis.append(prob.representation.phi)

    # the composed solution: each x of the 0.01 grid from the first sub-domain whose interval holds it
    xs, ys = _julia_range(0.0, 0.01, 1.0), _julia_range(0.0, 0.01, 1.0)
    err = 0.0
    for xv in xs:
        i = next(k for k in range(n_dec) if edges[k] <= xv <= edges[k + 1])
        pts = np.stack([np.full_like(ys, xv), ys])
        pred = phis[i](pts, reses[i].u).reshape(-1)
        err = max(err, float(np.max(np.abs(pred - analytic(xv, ys)))))
    print("domain decomposition, composed: inf-norm error %.3e (bound 5e-2)" % err)
    assert err <= 5e-2

    chain2 = _chain([2, 18, 18, 18, 18, 1])
    init2 = npde.initialparameters(rng, chain2)
    losses = [npde.NeuralAdapterLoss(chain2, npde.register_symbolic(phis[i], reses[i].u, "phi_%d" % i)(x, y))
              for i in range(n_dec)]
    res_ = _train(npde.neural_adapter(losses, init2, systems, npde.GridTraining([0.1 / n_dec, 0.1])), 2000)
    e1 = _err(chain2, res_.u)
    res_ = _train(npde.neural_adapter(losses, res_.u, systems, npde.GridTraining(0.01)), 2000)
    e2 = _err(chain2, res_.u)
    print("domain decomposition, merged: inf-norm error %.3e then %.3e (bound 5e-2)" % (e1, e2))
    assert e1 <= 5e-2 and e2 <= 5e-2
