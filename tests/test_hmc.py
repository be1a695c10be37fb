"""HMC sampler, host side: the float64 oracle (tests/hmc_oracle.py) against hand-derived Stan schedules, a hand-computed
dual-averaging sequence, Philox's published known answer and a Gaussian target, and the refusals of
npde.ahmc_bayesian_pinn_pde, which are raised before any engine exists."""
import numpy as np
import pytest
import sympy as sp

import neuralpde_jl_b200 as npde
import hmc_oracle as Q


def test_philox_known_answer():
    """Random123's kat_vectors entry for philox4x32-10 with zero counter and key"""
    w = Q.philox4x32_10([np.zeros(1)] * 4, 0, 0)
    assert [int(v[0]) for v in w] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]


def test_normals_are_standard_and_counter_keyed():
    z = Q.normals(7, 3, Q.TAG_MOMENTUM, 200001)
    assert abs(z.mean()) < 0.01 and abs(z.var() - 1.0) < 0.01
    assert np.array_equal(z[:10], Q.normals(7, 3, Q.TAG_MOMENTUM, 10))       # a prefix of the same stream
    assert not np.array_equal(z[:10], Q.normals(7, 4, Q.TAG_MOMENTUM, 10))
    assert not np.array_equal(z[:10], Q.normals(7, 3, Q.TAG_STEPSIZE_MOMENTUM, 10))
    u = [Q.uniform(7, t) for t in range(2000)]
    assert 0.0 <= min(u) and max(u) < 1.0 and abs(np.mean(u) - 0.5) < 0.02


def test_stan_windows_for_1000_adaptation_steps():
    init, windows, term = Q.stan_windows(1000)
    assert init == 75 and term == 50
    assert windows == [(76, 100), (101, 150), (151, 250), (251, 450), (451, 950)]


def test_stan_windows_for_short_adaptation():
    """the 200-draw reference tests adapt for 20 transitions: 15 % / the rest / 10 %"""
    init, windows, term = Q.stan_windows(20)
    assert (init, windows, term) == (3, [(4, 18)], 2)
    init, windows, term = Q.stan_windows(150)
    assert (init, windows, term) == (75, [(76, 100)], 50)
    assert Q.stan_windows(0)[1] == []


def test_dual_averaging_three_steps_by_hand():
    da = Q.DualAveraging(0.5, delta=0.8)
    mu = np.log(5.0)
    h = x_bar = 0.0
    for m, alpha in zip((1, 2, 3), (0.9, 0.3, 0.6)):
        da.update(alpha)
        h = (1 - 1 / (m + 10)) * h + (0.8 - alpha) / (m + 10)
        x = mu - h * np.sqrt(m) / 0.05
        x_bar = (1 - m ** -0.75) * x_bar + m ** -0.75 * x
        assert da.eps == pytest.approx(np.exp(x), rel=1e-14)
        assert da.x_bar == pytest.approx(x_bar, rel=1e-14)
    # step 1 by hand: h = -0.1 / 11, x = log 5 + 2 / 11, x_bar = x
    assert np.log(Q.DualAveraging(0.5).eps * 10) == pytest.approx(mu)
    d1 = Q.DualAveraging(0.5)
    d1.update(0.9)
    assert d1.eps == pytest.approx(5.0 * np.exp(2.0 / 11.0), rel=1e-14)
    d1.finalize()
    assert d1.eps == pytest.approx(5.0 * np.exp(2.0 / 11.0), rel=1e-14)
    d1.reset()
    assert (d1.m, d1.x_bar, d1.h_bar) == (0.0, 0.0, 0.0) and d1.mu == pytest.approx(np.log(50.0 * np.exp(2.0 / 11.0)))


def test_welford_regularised_variance():
    x = np.random.default_rng(0).normal(size=(40, 3)) * [1.0, 2.0, 0.5]
    mean, m2 = np.zeros(3), np.zeros(3)
    for k, row in enumerate(x, 1):
        d = row - mean
        mean = mean + d / k
        m2 = m2 + d * (row - mean)
    n = len(x)
    ref = (n / (n + 5.0)) * x.var(axis=0, ddof=1) + 1e-3 * 5.0 / (n + 5.0)
    assert np.allclose(Q.welford_variance(n, m2), ref, rtol=1e-12)


def test_oracle_samples_a_gaussian():
    """the oracle itself targets the right distribution: N(m, diag(s^2)) with a flat-ish prior, Stan adaptation"""
    m, s = np.array([1.0, -2.0]), np.array([0.5, 3.0])
    logp = lambda th: (-0.5 * float(np.sum(((th - m) / s) ** 2)), -(th - m) / s ** 2)   # noqa: E731
    ch = Q.sample(logp, np.zeros(2), 1500, n_leapfrog=10, n_adapts=300, prior_std=1e3, seed=11)
    post = ch.samples[300:]
    assert np.all(np.abs(post.mean(0) - m) < 0.25 * s)
    assert np.all(np.abs(post.std(0) / s - 1.0) < 0.25)
    assert 0.5 < ch.stats[300:, 1].mean() <= 1.0
    assert np.allclose(ch.minv / s ** 2, 1.0, rtol=0.6)          # the mass matrix learned the scales


def _ode_system():
    th = npde.parameters("θ")
    u = npde.variables("u")
    D = npde.Differential(th)
    q = (1 + 3 * th ** 2) / (1 + th + th ** 3)
    eq = npde.Eq(D(u(th)), th ** 3 + 2 * th + th ** 2 * q - u(th) * (th + q))
    return npde.PDESystem(eq, [npde.Eq(u(0.0), 1.0)], [npde.In(th, 0.0, 1.0)], [th], [u(th)])


def _disc(**kw):
    return npde.BayesianPINN([npde.Chain(npde.Dense(1, 12, "sigmoid"), npde.Dense(12, 1))], npde.GridTraining([0.01]),
                             **kw)


class _Marker:
    def __init__(self, name):
        self.name = name

    def __repr__(self):
        return self.name


@pytest.mark.parametrize("kw,msg", [
    ({"Kernel": _Marker("NUTS(0.8)")}, "NUTS and HMCDA"),
    ({"Kernel": _Marker("HMCDA(0.8, 1.0)")}, "NUTS and HMCDA"),
    ({"Adaptorkwargs": {"Metric": _Marker("DenseEuclideanMetric")}}, "DenseEuclideanMetric"),
    ({"Integratorkwargs": {"Integrator": _Marker("JitteredLeapfrog")}}, "JitteredLeapfrog"),
    ({"Integratorkwargs": {"Integrator": _Marker("TemperedLeapfrog")}}, "TemperedLeapfrog"),
    ({"nchains": 2}, "one chain"),
    ({"param": [_Marker("Normal(1, 2)")]}, "parameter estimation"),
    ({"Dict_differentials": {}}, "Dict_differentials"),
])
def test_refusals(kw, msg):
    with pytest.raises(ValueError, match=msg):
        npde.ahmc_bayesian_pinn_pde(_ode_system(), _disc(), **kw)


def test_refusals_of_the_discretization():
    with pytest.raises(ValueError, match="parameter estimation"):
        npde.ahmc_bayesian_pinn_pde(_ode_system(), _disc(param_estim=True))
    data = npde.DataLoss("u", np.array([[0.5]]), np.array([1.0]))
    with pytest.raises(ValueError, match="additional_loss"):
        npde.ahmc_bayesian_pinn_pde(_ode_system(), _disc(additional_loss=data))
    # a dataset and a non-Grid strategy reach symbolic_discretize's refusals unchanged
    with pytest.raises(ValueError, match="dataset points"):
        npde.ahmc_bayesian_pinn_pde(_ode_system(), _disc(dataset=[np.zeros((2, 2)), None]))
    with pytest.raises(ValueError, match="GridTraining only"):
        npde.ahmc_bayesian_pinn_pde(_ode_system(), npde.BayesianPINN(
            [npde.Chain(npde.Dense(1, 4, "tanh"), npde.Dense(4, 1))], npde.StochasticTraining(16)))


def test_log_likelihood_weights_helper():
    """c_k = -W n_k / (2 σ_k²) and the Gaussian normalisation, per group weight W = the group's weight sum"""
    from neuralpde_jl_b200.pinn import _loglik_weights
    w = {"pde": np.array([2.0]), "bc": np.array([1.0, 3.0])}
    n_k = np.array([100.0, 1.0, 5.0])
    c, const = _loglik_weights(w, n_k, 1, [[0.5], [0.1, 0.2], [0.05]])
    assert np.allclose(c, [-2.0 * 100 / 0.5, -4.0 * 1 / 0.02, -4.0 * 5 / 0.08])
    ref = 2.0 * (-50 * np.log(2 * np.pi) - 100 * np.log(0.5)) + 4.0 * (-0.5 * np.log(2 * np.pi) - np.log(0.1)) + \
        4.0 * (-2.5 * np.log(2 * np.pi) - 5 * np.log(0.2))
    assert const == pytest.approx(ref, rel=1e-14)
    with pytest.raises(ValueError, match="standard deviations"):
        _loglik_weights(w, n_k, 1, [[0.5], [0.1], [0.05]])
