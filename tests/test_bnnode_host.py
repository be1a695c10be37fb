"""ahmc_bayesian_pinn_ode / BNNODE on the host: the log density's term table (weights, constants, point sets) against a
literal restatement of the reference's LogTargetDensity (tests/bnnode_oracle.py), the σ(p) tracing, the θ.p priors,
the BNNODE indexing and the refusals.  No GPU."""
import math

import numpy as np
import pytest
import sympy as sp
import torch

import neuralpde_jl_b200 as npde
from neuralpde_jl_b200 import bpinn_ode as B
from neuralpde_jl_b200 import engine as E
from bnnode_oracle import BNNODEOracle
from test_nnode_host import chain, host_terms

KIND = {npde.Normal: "normal", npde.LogNormal: "lognormal", npde.Uniform: "uniform"}


def linear():                 # ODEBPINN i
    return npde.ODEProblem(lambda u, p, t: sp.cos(2 * sp.pi * t), 0.0, (0.0, 2.0))


def linear_inverse():         # ODEBPINN ii / iii: -u / p1 + exp(t / p2) cos t
    return npde.ODEProblem(lambda u, p, t: -u / p[0] + sp.exp(t / p[1]) * sp.cos(t), 0.0, (0.0, 4.0), [5.0, -5.0])


def scalar_p():               # iii_inverse_solve_improvement: one parameter
    return npde.ODEProblem(lambda u, p, t: -u / p + sp.exp(t / 5.0) * sp.cos(t), 0.0, (0.0, 4.0), 5.0)


def lotka_volterra():         # ODEBPINN iv
    def f(u, p, t):
        a, d = p
        x, y = u
        return [(a - y) * x, (x - d) * y]
    return npde.ODEProblem(f, [1.0, 1.0], (0.0, 4.0), [1.5, 3.0])


def _dataset(prob, n_pts=12, W=True):
    t = np.linspace(prob.tspan[0], prob.tspan[1], n_pts)
    n = 1 if np.ndim(prob.u0) == 0 else len(prob.u0)
    xs = [np.sin(t + k) * 0.3 + 1.0 for k in range(n)]
    return xs + [t] + ([np.linspace(0.5, 1.5, n_pts)] if W else [])


def _cases():
    st = npde.StochasticTraining(9, seed=3)
    wi = npde.WeightedIntervalTraining([0.2, 0.5, 0.3], 20, seed=1)
    q = npde.QuadratureTraining(nodes_per_dim=12)
    g = npde.GridTraining(0.25)
    return [
        ("grid scalar forward", linear, dict(strategy=g, phystd=[0.05])),
        ("stochastic scalar forward", linear, dict(strategy=st, phystd=[0.07])),
        ("weighted interval forward", linear, dict(strategy=wi, phystd=[0.05])),
        ("quadrature forward", linear, dict(strategy=q, phystd=[0.1])),
        ("grid forward with dataset", linear, dict(strategy=g, dataset=True, l2std=[0.02])),
        ("grid inverse", linear_inverse, dict(strategy=g, dataset=True, param=[npde.Normal(6.5, 0.5),
                                                                               npde.Normal(-3.0, 0.5)])),
        ("stochastic inverse collocate σ(p)", linear_inverse,
         dict(strategy=st, dataset=True, param=[npde.Normal(6.5, 0.5), npde.LogNormal(1.0, 0.5)], estim_collocate=True,
              phynewstd=lambda p: [0.1 / p[0] * p[1] ** 2])),
        ("scalar p collocate", scalar_p, dict(strategy=g, dataset=True, param=[npde.Normal(4.0, 2.0)],
                                              estim_collocate=True, phynewstd=lambda p: [0.1 / p])),
        ("vector grid inverse collocate", lotka_volterra,
         dict(strategy=g, dataset=True, param=[npde.Normal(-7, 2), npde.Uniform(1.0, 4.0)], estim_collocate=True,
              l2std=[0.5, 0.4], phystd=[0.5, 0.3], phynewstd=lambda p: [0.5, 0.2])),
        ("vector weighted interval forward collocate", lotka_volterra,
         dict(strategy=wi, dataset=True, estim_collocate=True, l2std=[0.5, 0.4], phystd=[0.5, 0.3],
              phynewstd=lambda p: [0.3, 0.6])),
        ("vector quadrature with dataset", lotka_volterra, dict(strategy=q, dataset=True, l2std=[0.5, 0.4],
                                                                phystd=[0.5, 0.3])),
    ]


def build(make, kw, width=5):
    prob = make()
    kw = dict(kw)
    if kw.pop("dataset", False):
        kw["dataset"] = _dataset(prob, W=True)
    n = 1 if np.ndim(prob.u0) == 0 else len(prob.u0)
    ch = chain(n, width=width, act_="tanh")
    ld = npde.BNNODELogDensity(prob, ch, seed=7, **kw)
    orc = BNNODEOracle(prob, ch, param=[(KIND[type(p)], *p.params()) for p in kw.get("param", [])],
                       dataset=ld.dataset, phystd=kw.get("phystd", [0.05]), l2std=kw.get("l2std", [0.05]),
                       phynewstd=kw.get("phynewstd"), estim_collocate=kw.get("estim_collocate", False))
    return prob, ld, orc


def fill_sampled(ld, rng):
    """fixed stand-ins for the device draws of the sampled terms; returns per component the physics times"""
    times = [[] for _ in range(ld.n)]
    for i, m, lo, hi in ld.sampled:
        ld.point_sets[i] = (lo + (hi - lo) * rng.random(m)).reshape(1, -1)
    for i, nm in enumerate(ld.term_names):
        if nm.startswith("phys_") and ld.kinds[i] == "phys":
            times[int(nm.split("_")[1]) - 1].append(ld.point_sets[i][0])
    return [np.concatenate(t) for t in times]


def host_loglik(ld, orc, theta):
    return float(np.dot(ld.c, host_terms(ld, orc.o, theta))) + ld.const + (
        0.0 if ld.tail_logabs is None else float(np.dot(ld.tail_logabs, np.log(np.abs(theta[ld.n_net:])))))


@pytest.mark.parametrize("i", range(len(_cases())), ids=[c[0] for c in _cases()])
def test_terms_match_literal_log_target_density(i):
    _, make, kw = _cases()[i]
    prob, ld, orc = build(make, kw)
    rng = np.random.default_rng(i)
    times = fill_sampled(ld, rng)
    quad = None
    if isinstance(ld.strategy, npde.QuadratureTraining):
        quad = (ld.point_sets[0][0], ld.quad_weights[0])
    for theta in (ld.theta0, ld.theta0 + 0.1 * rng.standard_normal(ld.theta0.size)):
        th = torch.tensor(theta)
        ref = float(orc.loglik(th, times, quad))
        got = host_loglik(ld, orc, theta)
        assert abs(got - ref) <= 1e-12 * max(1.0, abs(ref)), (got, ref)
        # the priors: the device's Normal on the network entries plus the forward-order tail table
        net = theta[:ld.n_net]
        mu, sd = orc.priorsNNw
        p_host = (-0.5 * net.size * math.log(2 * math.pi * sd * sd) - 0.5 * np.sum((net - mu) ** 2) / sd ** 2
                  + sum(B._logpdf(k, a, b, x) for (k, a, b), x in zip(ld.tail, theta[ld.n_net:])))
        assert abs(p_host - float(orc.priorweights(th))) <= 1e-12 * abs(p_host)


def test_point_sets_and_sampler_boxes():
    _, ld, _ = build(linear, dict(strategy=npde.GridTraining(0.25), dataset=True))
    assert np.allclose(ld.point_sets[0][0], np.concatenate([np.arange(9) * 0.25, np.linspace(0, 2, 12)]), atol=0)
    _, ld, _ = build(linear, dict(strategy=npde.WeightedIntervalTraining([0.2, 0.5, 0.3], 20)))
    assert [(m, lo, hi) for _, m, lo, hi in ld.sampled] == [(4, 0.0, 2 / 3), (10, 2 / 3, 4 / 3), (6, 4 / 3, 2.0)]
    assert list(ld.c) == [-0.5 * m / 0.05 ** 2 for m in (4, 10, 6)]
    _, ld, _ = build(lotka_volterra, dict(strategy=npde.StochasticTraining(30), dataset=True, l2std=[0.5, 0.5],
                                          phystd=[0.5, 0.5]))
    assert ld.term_names == ["phys_1", "phys_1_data", "phys_2", "phys_2_data", "l2_data_1", "l2_data_2"]
    assert [s[0] for s in ld.sampled] == [0, 2]


def test_sigma_tracing():
    prob = linear_inverse()
    ps = sp.symbols("p1 p2", real=True)
    assert B._sigma_monomials(lambda p: [0.1 / p[0]], list(ps), list(ps), 1)[0][0] == pytest.approx(0.1)
    a, e = B._sigma_monomials(lambda p: [0.1 / p[0]], list(ps), list(ps), 1)[0]
    assert list(e) == [-1.0, 0.0]
    a, e = B._sigma_monomials(lambda p: [3 * p[1] ** 2 * p[0]], list(ps), list(ps), 1)[0]
    assert (a, list(e)) == (3.0, [1.0, 2.0])
    assert B._sigma_monomials(lambda p: [0.05], list(ps), list(ps), 1)[0][0] == 0.05
    for bad in (lambda p: [0.1 + p[0]], lambda p: [sp.exp(p[0])], lambda p: [0 * p[0]], lambda p: [p[0] ** p[1]]):
        with pytest.raises(ValueError, match="monomial"):
            B._sigma_monomials(bad, list(ps), list(ps), 1)
    # through the front end: the log|p| coefficients are -n e_j
    _, ld, _ = build(linear_inverse, dict(strategy=npde.GridTraining(0.5), dataset=True, estim_collocate=True,
                                          param=[npde.Normal(5, 1), npde.Normal(-5, 1)],
                                          phynewstd=lambda p: [0.1 / p[0] * p[1] ** 2]))
    assert list(ld.tail_logabs) == [12.0, -24.0]
    with pytest.raises(ValueError, match="monomial"):
        build(linear_inverse, dict(strategy=npde.GridTraining(0.5), dataset=True, estim_collocate=True,
                                   param=[npde.Normal(5, 1), npde.Normal(-5, 1)], phynewstd=lambda p: [0.1 + p[0]]))
    assert prob.p == [5.0, -5.0]


def test_forward_prior_order_and_theta_p_start():
    param = [npde.Normal(6.5, 0.5), npde.LogNormal(1.0, 0.3), npde.Uniform(-2.0, 3.0)]
    prob = npde.ODEProblem(lambda u, p, t: -u / p[0] + p[1] * t + p[2], 0.0, (0.0, 1.0), [1.0, 2.0, 3.0])
    ld = npde.BNNODELogDensity(prob, chain(1), dataset=_dataset(prob), param=param)
    assert ld.tail == [(E.HMC_PRIOR_NORMAL, 6.5, 0.5), (E.HMC_PRIOR_LOGNORMAL, 1.0, 0.3),
                       (E.HMC_PRIOR_UNIFORM, -2.0, 3.0)]
    assert list(ld.theta0[-3:]) == [6.5, 1.0, -2.0]
    assert ld.spec.n_params == 3 and ld.spec.param_offset == ld.n_net


def test_bnnode_indexing_on_a_synthetic_sample_matrix(monkeypatch):
    ds, ne, ninv = 10, 3, 2
    samples = np.arange(ds * 4, dtype=np.float64).reshape(ds, 4)     # 2 network entries + 2 θ.p
    seen = {}

    def fake_outputs(chain_, dtype, device, ts, thetas):
        seen["thetas"] = thetas.copy()
        # N_k(t) = θ_0 + k / 3 + t: exercises the Float32 rounding of several outputs
        return np.stack([[th[0] + k / 3.0 + ts for k in range(2)] for th in thetas])

    monkeypatch.setattr(B, "_network_outputs", fake_outputs)
    prob = npde.ODEProblem(lambda u, p, t: [u[0], u[1]], [0.5, -1.0], (1.0, 2.0), [1.0, 1.0])
    t = np.array([1.0, 1.5, 2.0])
    curves, nnp, dep = B._bnnode_inference(prob, None, samples, ne, ninv, t, np.float64, 0)
    # curves: the first numensemble of the 1-based samples (ds - ne):ds -> 0-based 6, 7, 8
    assert np.array_equal(seen["thetas"], samples[6:9, :2])
    for k, u0 in enumerate((0.5, -1.0)):
        N = np.stack([(samples[i, 0] + k / 3.0 + t).astype(np.float32).astype(np.float64) for i in (6, 7, 8)])
        assert np.array_equal(curves[k], u0 + N * (t - 1.0))
    # parameter ensembles: samples[(end - ne):end] -> 0-based 6..9
    assert len(nnp) == 2 and all(np.array_equal(nnp[i], samples[6:, i]) for i in range(2))
    assert len(dep) == 2 and all(np.array_equal(dep[j], samples[6:, 2 + j]) for j in range(2))
    _, _, dep0 = B._bnnode_inference(prob, None, samples[:, :2], ne, 0, t, np.float64, 0)
    assert dep0 == [None]
    # one output: no Float32 rounding
    monkeypatch.setattr(B, "_network_outputs", lambda c, d, dv, ts, th: np.stack([[x[0] / 3.0 + ts] for x in th]))
    prob1 = npde.ODEProblem(lambda u, p, t: u, 0.25, (1.0, 2.0))
    curves, _, _ = B._bnnode_inference(prob1, None, samples[:, :2], ne, 0, t, np.float64, 0)
    assert np.array_equal(curves[0], 0.25 + np.stack([samples[i, 0] / 3.0 + t for i in (6, 7, 8)]) * (t - 1.0))
    assert npde.BNNODE(chain(1), draw_samples=2500).numensemble == 833


def test_exact_time_derivative_against_forward_difference_at_theta0():
    """autodiff = false: the reference's forward difference, replaced by exact taps; the log densities at θ0 agree"""
    for make, kw in ((linear, dict(strategy=npde.GridTraining(0.05))),
                     (lotka_volterra, dict(strategy=npde.GridTraining(0.05), dataset=True, estim_collocate=True,
                                           param=[npde.Normal(1.5, 0.5), npde.Normal(3.0, 0.5)],
                                           l2std=[0.5, 0.5], phystd=[0.5, 0.5], phynewstd=lambda p: [0.5, 0.5]))):
        prob, ld, orc = build(make, kw)
        th = torch.tensor(ld.theta0)
        times = [ld.point_sets[i][0] for i, nm in enumerate(ld.term_names) if nm.startswith("phys_")]
        exact = float(orc.logdensity(th, times))
        orc.derivative = "fd"
        fd = float(orc.logdensity(th, times))
        assert abs(exact - fd) <= 1e-6 * abs(exact), (exact, fd)


def test_refusals():
    ch = chain(1)
    prob = linear()
    with pytest.raises(ValueError, match="out-of-place"):
        npde.ODEProblem(lambda du, u, p, t: None, 0.0, (0.0, 1.0))
    with pytest.raises(ValueError, match="complex"):
        npde.ODEProblem(lambda u, p, t: u, 1j, (0.0, 1.0))
    with pytest.raises(ValueError, match="Dataset is Required for Inverse problems"):
        npde.BNNODELogDensity(linear_inverse(), ch, param=[npde.Normal(), npde.Normal()])
    with pytest.raises(ValueError, match="Dataset is Required for using the Data Quadrature"):
        npde.BNNODELogDensity(prob, ch, estim_collocate=True)
    with pytest.raises(ValueError, match=r"Invalid dataset for Inverse solve\. The dataset would be a timeseries \(x̂,t\)"):
        npde.BNNODELogDensity(prob, ch, dataset=[np.ones(3)])
    with pytest.raises(ValueError, match="Invalid dataset for Inverse solve with Data Quadrature loss"):
        npde.BNNODELogDensity(prob, ch, dataset=[np.ones(3), np.ones(3)], estim_collocate=True)
    with pytest.raises(ValueError, match="Invalid dataset for Inverse solve"):
        npde.BNNODELogDensity(prob, ch, dataset=[np.ones(3), [1, 2, 3]])
    with pytest.raises(ValueError, match="equal lengths"):
        npde.BNNODELogDensity(prob, ch, dataset=[np.ones(3), np.ones(4)])
    # [x̂, t] is padded with W = 1
    ld = npde.BNNODELogDensity(prob, ch, dataset=[np.ones(3), np.linspace(0, 1, 3)])
    assert np.array_equal(ld.dataset[-1], np.ones(3))
    lv = lotka_volterra()
    with pytest.raises(ValueError, match="phystd has 1 entries for 2"):
        npde.BNNODELogDensity(lv, chain(2))
    with pytest.raises(ValueError, match="l2std has 1 entries for 2"):
        npde.BNNODELogDensity(lv, chain(2), phystd=[0.1, 0.1], dataset=_dataset(lv))
    with pytest.raises(ValueError, match="nchains"):
        npde.ahmc_bayesian_pinn_ode(prob, ch, nchains=2)
    with pytest.raises(ValueError, match="NUTS and HMCDA"):
        npde.ahmc_bayesian_pinn_ode(prob, ch, Kernel="NUTS")
    with pytest.raises(ValueError, match="DenseEuclideanMetric"):
        npde.ahmc_bayesian_pinn_ode(prob, ch, Adaptorkwargs={"Metric": "DenseEuclideanMetric"})
    with pytest.raises(ValueError, match="JitteredLeapfrog"):
        npde.ahmc_bayesian_pinn_ode(prob, ch, Integratorkwargs={"Integrator": npde.Leapfrog, "jitter_rate": 1.0})
    with pytest.raises(ValueError, match="JitteredLeapfrog"):
        npde.ahmc_bayesian_pinn_ode(prob, ch, Integratorkwargs={"Integrator": "TemperedLeapfrog"})
    for mode in ("tc_bf16", "tc_split"):
        with pytest.raises(ValueError, match="FFMA kernel"):
            npde.BNNODELogDensity(prob, ch, mode=mode)
    with pytest.raises(ValueError, match="max 32"):
        npde.BNNODELogDensity(prob, ch, strategy=npde.WeightedIntervalTraining([1.0] * 33, 330))
    with pytest.raises(ValueError, match="ahmc_bayesian_pinn_ode: prior"):
        npde.BNNODELogDensity(linear_inverse(), ch, dataset=_dataset(linear_inverse()),
                              param=[npde.Normal(0.0, -1.0), npde.Normal()])
    with pytest.raises(ValueError, match="numensemble"):
        npde.solve(prob, npde.BNNODE(ch, draw_samples=3, numensemble=3))


def test_chain_seed_keys_the_point_draws():
    st = npde.StochasticTraining(8, seed=5)
    a = npde.BNNODELogDensity(linear(), chain(1), strategy=st, seed=0)
    b = npde.BNNODELogDensity(linear(), chain(1), strategy=st, seed=1)
    c = npde.BNNODELogDensity(linear(), chain(1), strategy=st, seed=2)
    assert a.sampler_seed == 5                      # seed 0: the strategy's own draws
    assert len({a.sampler_seed, b.sampler_seed, c.sampler_seed}) == 3
