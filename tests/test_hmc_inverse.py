"""BayesianPINN parameter estimation, host side: the per-entry priors of tests/hmc_prior_oracle.py against scipy.stats, the prior table and
starting θ.p that npde.ahmc_bayesian_pinn_pde builds, the log-likelihood weights over dataset and L2 data terms, and
the refusals, which are all raised before any engine exists."""
import numpy as np
import pytest
import sympy as sp
from scipy import stats

import neuralpde_jl_b200 as npde
from neuralpde_jl_b200 import engine as E
from neuralpde_jl_b200.pinn import _initial_theta, _loglik_weights, _loglik_weights_all, _tail_priors
import hmc_oracle as Q
import hmc_prior_oracle as P

XS = [-2.0, -1e-3, 0.0, 1e-3, 0.3, 1.0, 2.5, 7.0]


@pytest.mark.parametrize("kind,a,b,ref", [
    (P.PRIOR_NORMAL, 1.0, 0.5, stats.norm(loc=1.0, scale=0.5)),
    (P.PRIOR_LOGNORMAL, 0.3, 0.8, stats.lognorm(s=0.8, scale=np.exp(0.3))),
    (P.PRIOR_UNIFORM, -1e-3, 2.5, stats.uniform(loc=-1e-3, scale=2.5 + 1e-3)),
])
def test_oracle_priors_match_scipy(kind, a, b, ref):
    for x in XS:
        got, want = P.prior_logpdf(kind, a, b, x), float(ref.logpdf(x))
        if np.isinf(want):
            assert got == -np.inf, (x, got)
            assert np.isnan(P.prior_grad(kind, a, b, x)), x
            continue
        assert abs(got - want) <= 1e-12 * max(1.0, abs(want)), (x, got, want)
        # the gradient against a central difference of scipy's logpdf
        h = 1e-6 * max(1.0, abs(x))
        if kind == P.PRIOR_LOGNORMAL:
            h = min(h, 0.5 * x)
        fd = (float(ref.logpdf(x + h)) - float(ref.logpdf(x - h))) / (2 * h)
        if kind == P.PRIOR_UNIFORM:
            assert P.prior_grad(kind, a, b, x) == 0.0
        else:
            assert abs(P.prior_grad(kind, a, b, x) - fd) <= 1e-6 * max(1.0, abs(fd)), (x, P.prior_grad(kind, a, b, x), fd)
    # Distributions.jl's insupport: both bounds of Uniform belong to it, 0 does not belong to LogNormal
    if kind == P.PRIOR_UNIFORM:
        assert P.prior_logpdf(kind, a, b, a) == P.prior_logpdf(kind, a, b, b) == -np.log(b - a)
        assert P.prior_logpdf(kind, a, b, np.nextafter(b, np.inf)) == -np.inf


def test_oracle_target_with_tail_priors():
    """hmc_oracle's target around with_tail_priors: N(0.1, 2²) on the network entries only, the tail priors on the rest"""
    f = lambda th: (-0.5 * float(np.sum(th * th)), -th)      # noqa: E731
    th = np.array([0.3, -0.2, 1.5, 0.7])
    d = th - 0.1
    tail = [(P.PRIOR_LOGNORMAL, 0.0, 1.0), (P.PRIOR_NORMAL, 1.0, 0.5)]
    target = Q._Target(P.with_tail_priors(f, tail, 0.1, 2.0), 0.1, 2.0, 4)
    l1, g1 = target(th)
    ref = -0.5 * float(np.sum(th * th)) + stats.norm(0.1, 2.0).logpdf(th[:2]).sum() + \
        stats.lognorm(s=1.0).logpdf(th[2]) + stats.norm(1.0, 0.5).logpdf(th[3])
    assert l1 == pytest.approx(ref, rel=1e-13)
    assert np.allclose(g1, [-th[0] - d[0] / 4, -th[1] - d[1] / 4, -th[2] - (1 + np.log(th[2])) / th[2],
                            -th[3] - (th[3] - 1.0) / 0.25], rtol=1e-13)
    l2, g2 = target(np.array([0.3, -0.2, -1.5, 0.7]))
    assert l2 == -np.inf and np.isnan(g2[2])
    # no tail: the physics part unchanged
    assert P.with_tail_priors(f, [], 0.1, 2.0)(th)[0] == f(th)[0]


def test_tail_table_is_reversed_and_starts_at_the_first_parameter():
    param = [npde.Normal(1, .5), npde.LogNormal(0, 1)]
    assert _tail_priors(param) == [(E.HMC_PRIOR_LOGNORMAL, 0.0, 1.0), (E.HMC_PRIOR_NORMAL, 1.0, 0.5)]
    th = _initial_theta(np.array([0.1, 0.2, 0.3, 4.0, 4.0], dtype=np.float32), param)
    assert th.dtype == np.float64 and np.array_equal(th, np.array([0.1, 0.2, 0.3, 1.0, 0.0], dtype=np.float32))
    # LogNormal starts at μ of log x, Uniform at its lower bound; a problem without parameters keeps every entry
    assert list(_initial_theta(np.zeros(3), [npde.LogNormal(6.0, 0.5), npde.Uniform(-1.0, 2.0)])) == [0.0, 6.0, -1.0]
    assert np.array_equal(_initial_theta(np.arange(3.0), []), np.arange(3.0))
    assert npde.Uniform(2, 3).params() == (2, 3) and npde.LogNormal(6.0, 0.5).params() == (6.0, 0.5)


def test_log_likelihood_weights_over_dataset_and_data_terms():
    """grid terms as _loglik_weights; dataset term j in its group with that group's σ_j; L2 terms with l2std only"""
    w = {"pde": np.array([2.0, 1.0]), "bc": np.array([1.0, 3.0])}
    # grid: 2 pde, 2 bc; dataset: 2 pde terms, 1 bc term; 2 L2 terms
    n_k = np.array([100.0, 80.0, 1.0, 5.0, 21.0, 22.0, 4.0, 30.0, 31.0])
    allstd = [[0.5, 0.25], [0.1, 0.2], [0.05, 2.0]]
    c, const = _loglik_weights_all(w, n_k, (2, 2, 2, 1), allstd)
    c0, const0 = _loglik_weights(w, n_k[:4], 2, allstd)
    assert np.array_equal(c[:4], c0)
    assert np.allclose(c[4:], [-3.0 * 21 / (2 * 0.25), -3.0 * 22 / (2 * 0.0625), -4.0 * 4 / (2 * 0.01), 0.0, 0.0],
                       rtol=1e-15)
    ref = const0 + 3.0 * (-10.5 * np.log(2 * np.pi) - 21 * np.log(0.5)) + 3.0 * (-11 * np.log(2 * np.pi) - 22 * np.log(0.25)) \
        + 4.0 * (-2 * np.log(2 * np.pi) - 4 * np.log(0.1))
    assert const == pytest.approx(ref, rel=1e-14)
    cd, constd = _loglik_weights_all(w, n_k, (2, 2, 2, 1), allstd, data=True)
    assert np.array_equal(cd[:7], c[:7])
    assert np.allclose(cd[7:], [-30 / (2 * 0.0025), -31 / 8.0], rtol=1e-15)
    assert constd == pytest.approx(const - 15 * np.log(2 * np.pi) - 30 * np.log(0.05) - 15.5 * np.log(2 * np.pi)
                                   - 31 * np.log(2.0), rel=1e-14)
    # without dataset terms the helper is _loglik_weights
    c1, const1 = _loglik_weights_all(w, n_k[:4], (2, 2, 0, 0), allstd, data=True)
    assert np.array_equal(c1, c0) and const1 == const0
    with pytest.raises(ValueError, match="l2std"):
        _loglik_weights_all(w, n_k, (2, 2, 2, 1), [[0.5, 0.25], [0.1, 0.2], [0.05]], data=True)


def _periodic(param=True):
    """reference test/PDEBPINN/bpinn_pde__bpinn_pde_inv_i_1d_periodic_system.jl"""
    t, p = npde.parameters("t p")
    u = npde.variables("u")
    eq = npde.Eq(npde.Differential(t)(u(t)) - sp.cos(p * t), 0.0)
    return npde.PDESystem(eq, [npde.Eq(u(0.0), 0.0)], [npde.In(t, 0.0, 2.0)], [t], [u(t)], [p] if param else [],
                          defaults={p: 4.0} if param else {})


def _dataset(n=11):
    ts = np.linspace(0.0, 2.0, n)
    return [np.stack([np.sin(2 * np.pi * ts) / (2 * np.pi), ts], axis=1)]


def _disc(**kw):
    return npde.BayesianPINN([npde.Chain(npde.Dense(1, 6, "tanh"), npde.Dense(6, 1))], npde.GridTraining([0.02]), **kw)


class _Marker:
    def __init__(self, name):
        self.name = name

    def __repr__(self):
        return self.name


@pytest.mark.parametrize("disc_kw,kw,msg", [
    ({"param_estim": True, "dataset": [_dataset(), None]}, {}, "parameter estimation.*needs `param`"),
    ({"dataset": [_dataset(), None]}, {"param": [npde.Normal(1, 2)]}, "parameter estimation.*param_estim = true"),
    ({"param_estim": True}, {"param": [npde.LogNormal(6, 0.5)]}, "needs a dataset"),
    ({"param_estim": True, "dataset": [_dataset(), None]}, {"param": [npde.LogNormal(6, 0.5)], "l2std": [0.1, 0.1]},
     "L2 stds length"),
    ({"param_estim": True, "dataset": [_dataset(), None]}, {"param": [npde.Normal(1, 2), npde.Normal(1, 2)]},
     "2 priors in `param` for the 1 equation parameters"),
    ({"param_estim": True, "dataset": [_dataset(), None]}, {"param": [_Marker("Gamma(2, 1)")]},
     r"prior Gamma\(2, 1\) is not supported"),
    ({"param_estim": True, "dataset": [_dataset(), None]}, {"param": [npde.Normal(1, 0)]}, "σ > 0"),
    ({"param_estim": True, "dataset": [_dataset(), None]}, {"param": [npde.LogNormal(1, -1)]}, "σ > 0"),
    ({"param_estim": True, "dataset": [_dataset(), None]}, {"param": [npde.Uniform(2, 2)]}, "a < b"),
    ({"param_estim": True, "dataset": [_dataset(), None]}, {"param": [npde.Normal(np.inf, 1)]}, "finite"),
    ({"param_estim": True, "dataset": [_dataset(), None]}, {"param": [npde.Normal(1, 2)], "Dict_differentials": {}},
     "Dict_differentials"),
    ({"param_estim": True, "dataset": [_dataset()[0], None]}, {"param": [npde.Normal(1, 2)]}, "dataset points"),
    ({"param_estim": True, "dataset": [[np.zeros((4, 3))], None]}, {"param": [npde.Normal(1, 2)]},
     r"dataset points.*expected n × 2"),
    ({"param_estim": True, "dataset": [_dataset() * 2, None]}, {"param": [npde.Normal(1, 2)]}, "list of 1 arrays"),
    ({"param_estim": True, "dataset": [_dataset()]}, {"param": [npde.Normal(1, 2)]}, "dataset points"),
    ({"dataset": [_dataset(), None]}, {"Kernel": _Marker("NUTS(0.8)")}, "NUTS and HMCDA"),
])
def test_refusals(disc_kw, kw, msg):
    with pytest.raises(ValueError, match=msg):
        npde.ahmc_bayesian_pinn_pde(_periodic(), _disc(**disc_kw), **kw)


def test_dataset_coordinates_must_match_the_equation():
    """equation 1 has the variable t only, but dataset_pde[1] belongs to u(x, t) and has two coordinate columns"""
    x, t = npde.parameters("x t")
    u, v = npde.variables("u v")
    Dt = npde.Differential(t)
    eqs = [npde.Eq(Dt(v(t)), 0.0), npde.Eq(Dt(u(x, t)), v(t))]
    bcs = [npde.Eq(u(x, 0.0), 0.0), npde.Eq(v(0.0), 1.0)]
    sys_ = npde.PDESystem(eqs, bcs, [npde.In(x, 0.0, 1.0), npde.In(t, 0.0, 1.0)], [x, t], [u(x, t), v(t)])
    chains = [npde.Chain(npde.Dense(2, 4, "tanh"), npde.Dense(4, 1)), npde.Chain(npde.Dense(1, 4, "tanh"), npde.Dense(4, 1))]
    disc = npde.BayesianPINN(chains, npde.GridTraining(0.1), dataset=[[np.zeros((5, 3)), np.zeros((5, 2))], None])
    with pytest.raises(ValueError, match=r"dataset 1 has 2 coordinate columns but equation 1 has the variables \['t'\]"):
        npde.ahmc_bayesian_pinn_pde(sys_, disc, saveats=[0.5, 0.5])
