"""BayesianPINN parameter estimation on the device (pinn_hmc_begin_ex, npde.ahmc_bayesian_pinn_pde with param_estim):
the log density against a float64 restatement of the reference's PDELogTargetDensity, trajectory parity with the
oracle (tests/hmc_oracle.py with tests/hmc_prior_oracle.py) under per-entry priors, a closed-form Gaussian posterior over (w, b, p), the priors'
supports, bit-reproducibility, a tensor-core chain and the reference's inverse tests inv_i and inv_ii."""
import numpy as np
import pytest
import sympy as sp
import torch
from scipy import stats

import neuralpde_jl_b200 as npde
from neuralpde_jl_b200 import configs, engine as E
from neuralpde_jl_b200.pinn import _initial_theta, _tail_priors
from oracle import reference as R
from helpers import rel
import hmc_oracle as Q
import hmc_prior_oracle as P

pytestmark = pytest.mark.gpu

LOG2PI = np.log(2.0 * np.pi)


def _periodic_system():
    """reference test/PDEBPINN/bpinn_pde__bpinn_pde_inv_i_1d_periodic_system.jl: u' = cos(p t), u(0) = 0, p = 2π"""
    t, p = npde.parameters("t p")
    u = npde.variables("u")
    eq = npde.Eq(npde.Differential(t)(u(t)) - sp.cos(p * t), 0.0)
    return npde.PDESystem(eq, [npde.Eq(u(0.0), 0.0)], [npde.In(t, 0.0, 2.0)], [t], [u(t)], [p], defaults={p: 4.0})


def _periodic_data(seed=100):
    """201 points on [0, 2] with 20 % multiplicative noise, as the reference (seeded numpy in place of Julia's RNG)"""
    ts = np.linspace(0.0, 2.0, 201)
    u = np.sin(2 * np.pi * ts) / (2 * np.pi)
    u = u + 0.2 * u * np.random.default_rng(seed).standard_normal(ts.size)
    return [np.stack([u, ts], axis=1)]


def _two_param_system():
    """u' = a cos(2π t) + b, u(0) = 0 on [0, 1]; the data come from a = 1, b = 0"""
    t, a, b = npde.parameters("t a b")
    u = npde.variables("u")
    eq = npde.Eq(npde.Differential(t)(u(t)), a * sp.cos(2 * sp.pi * t) + b)
    return npde.PDESystem(eq, [npde.Eq(u(0.0), 0.0)], [npde.In(t, 0.0, 1.0)], [t], [u(t)], [a, b])


def _two_param_data():
    ts = np.linspace(0.0, 1.0, 41)
    u = np.sin(2 * np.pi * ts) / (2 * np.pi) + 0.01 * np.random.default_rng(3).standard_normal(ts.size)
    return [np.stack([u, ts], axis=1)]


PERIODIC = dict(system=_periodic_system, data=_periodic_data, chains=lambda: [npde.Chain(
    npde.Dense(1, 6, "tanh"), npde.Dense(6, 6, "tanh"), npde.Dense(6, 1))], dx=[0.02],
    param=[npde.LogNormal(6.0, 0.5)], allstd=[[0.02], [0.02], [0.02]], prior=(0.0, 1.0))
TWO = dict(system=_two_param_system, data=_two_param_data, chains=lambda: [npde.Chain(
    npde.Dense(1, 6, "tanh"), npde.Dense(6, 6, "tanh"), npde.Dense(6, 1))], dx=[0.05],
    param=[npde.Normal(1, .5), npde.LogNormal(0, 1)], allstd=[[0.05], [0.05], [0.05]], prior=(0.0, 2.0))


def _rep(case, **kw):
    disc = npde.BayesianPINN(case["chains"](), npde.GridTraining(case["dx"]), param_estim=True,
                             dataset=[case["data"](), None], **kw)
    return npde.symbolic_discretize(case["system"](), disc)


def _logpdf(prior, x):
    if isinstance(prior, npde.Normal):
        return stats.norm(prior.mu, prior.sigma).logpdf(x)
    if isinstance(prior, npde.LogNormal):
        return stats.lognorm(s=prior.sigma, scale=np.exp(prior.mu)).logpdf(x)
    return stats.uniform(prior.a, prior.b - prior.a).logpdf(x)


class _InverseOracle:
    """float64 restatement of the reference's log density (ext/bpinn/PDE_BPINN.jl:16-27): full_loss_function over the
    grid and dataset points (each group's sum times its weight sum, here the group's term count) + priorlogpdf +
    L2LossData, with exact derivative taps (oracle/reference.py)"""

    def __init__(self, case, rep):
        self.sys = case["system"]()
        self.chains = case["chains"]()
        self.prob = R.Problem(self.sys, [(c.dims, c.acts) for c in self.chains], param_estim=True, derivative="exact")
        self.grid = rep.point_sets[:len(self.sys.eqs) + len(self.sys.bcs)]
        self.data = case["data"]()
        self.param, self.allstd, self.prior = case["param"], case["allstd"], case["prior"]

    @staticmethod
    def _lp(r, s):
        n = r.numel()
        return -0.5 * n * LOG2PI - n * np.log(s) - (r * r).sum() / (2.0 * s * s)

    def loglik(self, theta, l2=True):
        eqs, bcs = list(self.sys.eqs), list(self.sys.bcs)
        stdpdes, stdbcs, l2std = self.allstd
        res = lambda eq, pts: self.prob.residual(eq, torch.as_tensor(pts, dtype=torch.float64), theta)   # noqa: E731
        pde = sum(self._lp(res(eq, s), stdpdes[i]) for i, (eq, s) in enumerate(zip(eqs, self.grid)))
        pde = pde + sum(self._lp(res(eq, m[:, 1:].T), stdpdes[j]) for j, (eq, m) in enumerate(zip(eqs, self.data)))
        bc = sum(self._lp(res(eq, s), stdbcs[j]) for j, (eq, s) in enumerate(zip(bcs, self.grid[len(eqs):])))
        ll = len(eqs) * pde + len(bcs) * bc
        if l2:
            for i, m in enumerate(self.data):
                u = self.prob._u(i, theta)(torch.as_tensor(m[:, 1:].T, dtype=torch.float64))[0]
                ll = ll + self._lp(u - torch.as_tensor(m[:, 0]), l2std[i])
        return ll

    def logp_grad(self, th):
        theta = torch.tensor(np.asarray(th, dtype=np.float64), requires_grad=True)
        ll = self.loglik(theta)
        (g,) = torch.autograd.grad(ll, theta)
        return float(ll.detach()), g.numpy().copy()

    def log_density(self, th):
        """loglik + priorlogpdf, the inverse priors applied as the reference does: invpriors[length(θ) - i + 1] to θ[i]"""
        n, ninv = th.size, len(self.param)
        lp = float(self.loglik(torch.tensor(th)).detach())
        lp += float(np.sum(stats.norm(self.prior[0], self.prior[1]).logpdf(th[:n - ninv])))
        for i in range(n - ninv + 1, n + 1):                   # 1-based, as ext/bpinn/PDE_BPINN.jl:194-196
            lp += float(_logpdf(self.param[n - i + 1 - 1], th[i - 1]))
        return lp


def _begin(rep, case, **kw):
    c, const = rep.loglik_weights(case["allstd"], data=True)
    th0 = _initial_theta(rep.flat_init_params, case["param"])
    kw = dict(dict(prior_mean=case["prior"][0], prior_std=case["prior"][1], weights=c, ll_const=const,
                   tail_priors=_tail_priors(case["param"])), **kw)
    return th0, rep.engine.hmc_begin(th0, **kw)


@pytest.mark.parametrize("case", [PERIODIC, TWO], ids=["inv_i", "two_params"])
def test_log_density_matches_the_float64_target(case):
    rep = _rep(case, init_params=None)
    assert rep.term_names == ["pde_1", "bc_1", "dataset_pde_1", "l2_data_u"]
    orc = _InverseOracle(case, rep)
    # at θ0: one transition with a huge step is rejected, so its row carries l(θ0)
    th0, _ = _begin(rep, case, n_leapfrog=5, adaptor=E.HMC_ADAPT_NONE, metric=E.HMC_METRIC_UNIT, step_size=5.0)
    _, st = rep.engine.hmc_iterate(1)
    assert st[0, 2] == 0.0
    ref = orc.log_density(th0)
    assert abs(st[0, 3] - ref) <= 1e-10 * abs(ref), (st[0, 3], ref)
    # full_loss_function holds the grid and dataset terms, not L2LossData
    fl = rep.loss_functions.full_loss_function(th0, case["allstd"])
    ref_fl = float(orc.loglik(torch.tensor(th0), l2=False))
    assert abs(fl - ref_fl) <= 1e-10 * abs(ref_fl), (fl, ref_fl)
    # along an adapting chain
    _begin(rep, case, n_adapts=10, seed=4)
    samples, st = rep.engine.hmc_iterate(15)
    assert st[:, 2].sum() > 0
    for k in (4, 9, 14):
        ref = orc.log_density(samples[k])
        assert abs(st[k, 3] - ref) <= 1e-10 * abs(ref), (k, st[k, 3], ref)


def test_trajectory_matches_the_float64_oracle():
    """two parameters (LogNormal and Normal after the reversal), FFMA fp64, find_good_stepsize and Stan adaptation over
    10 of 20 transitions, against the oracle with the same Philox draws"""
    rep = _rep(TWO, init_params=None)
    kw = dict(n_leapfrog=30, n_adapts=10, prior_mean=0.0, prior_std=2.0, seed=5)
    th0, eps0 = _begin(rep, TWO, **kw)
    samples, stats_ = rep.engine.hmc_iterate(20)
    orc = _InverseOracle(TWO, rep)
    tail = [(P.PRIOR_LOGNORMAL, 0.0, 1.0), (P.PRIOR_NORMAL, 1.0, 0.5)]
    ch = Q.sample(P.with_tail_priors(orc.logp_grad, tail, 0.0, 2.0), th0, 20, **kw)
    assert abs(eps0 - ch.eps0) <= 1e-9 * ch.eps0, (eps0, ch.eps0)
    assert np.allclose(stats_[:, 0], ch.stats[:, 0], rtol=1e-9, atol=0), (stats_[:, 0], ch.stats[:, 0])
    assert np.array_equal(stats_[:, 2], ch.stats[:, 2]), (stats_[:, 2], ch.stats[:, 2])
    assert 0 < stats_[:, 2].sum()
    for k in range(20):
        assert rel(samples[k], ch.samples[k]) <= 1e-7, (k, rel(samples[k], ch.samples[k]))


def _linear_system():
    """u(x) = w x + b with u' = p, u(0) = 0 and observations of u: every residual is linear in (w, b, p), so the
    posterior is Gaussian"""
    x, p = npde.parameters("x p")
    u = npde.variables("u")
    return npde.PDESystem(npde.Eq(npde.Differential(x)(u(x)), p), [npde.Eq(u(0.0), 0.0)], [npde.In(x, 0.0, 1.0)], [x],
                          [u(x)], [p])


def _linear_disc():
    xs = np.linspace(0.0, 1.0, 11)
    ys = 2.0 * xs + 0.1 * np.random.default_rng(7).standard_normal(xs.size)
    return npde.BayesianPINN([npde.Chain(npde.Dense(1, 1))], npde.GridTraining(0.1), param_estim=True,
                             dataset=[[np.stack([ys, xs], axis=1)], None])


def test_known_gaussian_posterior():
    allstd = [[0.5], [0.5], [0.5]]
    rep = npde.symbolic_discretize(_linear_system(), _linear_disc())
    c, _ = rep.loglik_weights(allstd, data=True)
    prior_g = lambda th: np.array([-th[0] / 4.0, -th[1] / 4.0, -(th[2] - 1.0) / 0.25])   # noqa: E731
    grad = lambda th: rep.engine.loss_grad_host(th, c, True)[2] + prior_g(th)            # noqa: E731
    g0 = grad(np.zeros(3))
    P = -np.stack([grad(e) - g0 for e in np.eye(3)], axis=1)
    P = 0.5 * (P + P.T)
    mean, cov = np.linalg.solve(P, g0), np.linalg.inv(P)
    sol = npde.ahmc_bayesian_pinn_pde(_linear_system(), _linear_disc(), draw_samples=4000, phystd=allstd[0],
                                      bcstd=allstd[1], l2std=allstd[2], priorsNNw=(0.0, 2.0), saveats=[0.5],
                                      param=[npde.Normal(1.0, 0.5)], seed=1)
    post = sol.original.samples[400:]
    assert np.mean(sol.original.statistics["numerical_error"]) == 0.0
    batches = post.reshape(40, -1, 3).mean(axis=1)
    se = batches.std(axis=0, ddof=1) / np.sqrt(40)
    assert np.all(np.abs(post.mean(0) - mean) <= 5 * se), (post.mean(0), mean, se)
    assert np.all(np.abs(post.var(0) / np.diag(cov) - 1.0) <= 0.2), (post.var(0), np.diag(cov))
    assert len(sol.estimated_de_params) == 1 and sol.estimated_de_params[0].shape == (1334,)
    assert np.array_equal(sol.estimated_de_params[0], sol.original.samples[-1334:, 2])


@pytest.mark.parametrize("prior,inside", [(npde.Uniform(0.0, 10.0), lambda p: (p >= 0.0) & (p <= 10.0)),
                                          (npde.LogNormal(0.05, 3.0), lambda p: p > 0.0)], ids=["uniform", "lognormal"])
def test_proposals_outside_the_support_are_rejected(prior, inside):
    """chains started on (Uniform: at a) or next to (LogNormal(0.05, 3), whose mode is near 0) the support's bound with
    a large fixed step: leaving the support ends the trajectory as a numerical error and a rejection"""
    case = dict(PERIODIC, param=[prior])
    rep = _rep(case, init_params=None)
    th0, _ = _begin(rep, case, n_leapfrog=10, adaptor=E.HMC_ADAPT_NONE, metric=E.HMC_METRIC_UNIT, step_size=0.05,
                    seed=9)
    samples, st = rep.engine.hmc_iterate(60)
    err = st[:, 6] == 1.0
    assert err.sum() > 0
    assert np.all(st[err, 2] == 0.0) and np.all(st[err, 1] == 0.0)
    assert np.all(inside(samples[:, -1])) and np.all(np.isfinite(st[:, 3]))
    assert np.all(np.isfinite(samples))


def _two_run(n=30, seed=2):
    rep = _rep(TWO, init_params=None)
    _, eps0 = _begin(rep, TWO, n_adapts=10, seed=seed)
    s, st = rep.engine.hmc_iterate(n)
    return eps0, s, st, rep


def test_runs_are_bit_identical_with_and_without_the_graph(monkeypatch):
    a = _two_run()
    b = _two_run()
    assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
    monkeypatch.setenv("PINN_B200_NO_GRAPH", "1")
    c = _two_run()
    assert a[0] == c[0] and np.array_equal(a[1], c[1]) and np.array_equal(a[2], c[2])
    monkeypatch.delenv("PINN_B200_NO_GRAPH")
    d = _two_run(n=12)
    s2, st2 = d[3].engine.hmc_iterate(18)
    assert np.array_equal(np.concatenate([d[1], s2]), a[1]) and np.array_equal(np.concatenate([d[2], st2]), a[2])
    # still momentum + 30 x (kick / drift, fused kernel) + closing kick + accept + select
    l0 = d[3].engine.launch_count()
    d[3].engine.hmc_iterate(2)
    assert d[3].engine.launch_count() - l0 == 2 * (4 + 2 * 30)


def test_begin_ex_without_tail_is_hmc_begin():
    rep = _rep(PERIODIC, init_params=None)
    c, const = rep.loglik_weights(PERIODIC["allstd"], data=True)
    th0 = _initial_theta(rep.flat_init_params, PERIODIC["param"])
    runs = []
    for tail in (None, []):
        eps0 = rep.engine.hmc_begin(th0, n_adapts=10, prior_std=3.0, seed=6, weights=c, ll_const=const, tail_priors=tail)
        runs.append((eps0,) + rep.engine.hmc_iterate(15))
    assert runs[0][0] == runs[1][0] and np.array_equal(runs[0][1], runs[1][1]) and np.array_equal(runs[0][2], runs[1][2])


def test_abi_refusals():
    rep = _rep(PERIODIC, init_params=None)
    eng = rep.engine
    th0 = _initial_theta(rep.flat_init_params, PERIODIC["param"])
    n = th0.size
    N, LN, U = E.HMC_PRIOR_NORMAL, E.HMC_PRIOR_LOGNORMAL, E.HMC_PRIOR_UNIFORM
    for tail, msg in (([(N, 0.0, 1.0)] * 17, "n_tail = 17"), ([(N, 0.0, 1.0)] * n, "n_tail = %d" % n),
                      ([(7, 0.0, 1.0)], "unknown kind 7"), ([(N, 0.0, 0.0)], "sigma 0"), ([(LN, 0.0, -1.0)], "sigma -1"),
                      ([(U, 2.0, 2.0)], "needs a < b"), ([(N, np.nan, 1.0)], "non-finite"),
                      ([(U, 7.0, 8.0)], "log density or its gradient is not finite at theta0")):
        with pytest.raises(E.EngineError, match=msg):
            eng.hmc_begin(th0, step_size=0.01, tail_priors=tail)
    th_neg = th0.copy()
    th_neg[-1] = -1.0
    with pytest.raises(E.EngineError, match="not finite at theta0"):
        eng.hmc_begin(th_neg, step_size=0.01, tail_priors=[(LN, 0.0, 1.0)])
    with pytest.raises(E.EngineError, match="call pinn_hmc_begin first"):
        eng.hmc_iterate(1)
    eng.hmc_begin(th0, step_size=0.01, tail_priors=[(U, 0.0, th0[-1])])          # the bound itself is in the support
    assert np.all(np.isfinite(eng.hmc_iterate(2)[1][:, 3]))


def test_tc_split_inverse_chain_runs():
    chains = [npde.Chain(npde.Dense(1, 16, "tanh"), npde.Dense(16, 16, "tanh"), npde.Dense(16, 1))]
    init = np.concatenate([npde.initialparameters(np.random.default_rng(1), chains[0], np.float32),
                           np.ones(1, np.float32)])
    disc = npde.BayesianPINN(chains, npde.GridTraining([0.02]), init_params=init, mode="tc_split", param_estim=True,
                             dataset=[_periodic_data(), None])
    sol = npde.ahmc_bayesian_pinn_pde(_periodic_system(), disc, draw_samples=60, bcstd=[0.05], phystd=[0.05],
                                      l2std=[0.05], priorsNNw=(0.0, 1.0), saveats=[1 / 50.0],
                                      param=[npde.LogNormal(6.0, 0.5)])
    st = sol.original.statistics
    assert all(np.all(np.isfinite(v)) for v in st.values())
    assert st["acceptance_rate"].mean() > 0
    assert np.all(np.isfinite(sol.estimated_de_params[0])) and np.all(sol.estimated_de_params[0] > 0)


# ---- the reference's inverse BayesianPINN tests (test/PDEBPINN/), bounds as stated there ------------------------------
def test_reference_inv_i_1d_periodic_system():
    disc = npde.BayesianPINN(PERIODIC["chains"](), npde.GridTraining([0.02]), param_estim=True,
                             dataset=[_periodic_data(), None])
    sol = npde.ahmc_bayesian_pinn_pde(_periodic_system(), disc, draw_samples=1500, bcstd=[0.02], phystd=[0.02],
                                      l2std=[0.02], priorsNNw=(0.0, 1.0), saveats=[1 / 50.0],
                                      param=[npde.LogNormal(6.0, 0.5)])
    ts = sol.timepoints[0][0]
    err = np.mean(np.abs(npde.pmean(sol.ensemblesol[0]) - np.sin(2 * np.pi * ts) / (2 * np.pi)))
    p = float(npde.pmean(sol.estimated_de_params[0]))
    assert err < 8e-2, (err, p)
    assert abs(p - 2 * np.pi) <= 0.1 * 2 * np.pi, (err, p)


def test_reference_inv_ii_lorenz_system():
    sys_, chains, data = configs.lorenz_bpinn()
    disc = npde.BayesianPINN(chains, npde.GridTraining([0.01]), param_estim=True, dataset=[data, None])
    sol = npde.ahmc_bayesian_pinn_pde(sys_, disc, draw_samples=50, bcstd=[0.3] * 3, phystd=[0.1] * 3,
                                      l2std=[1.0] * 3, priorsNNw=(0.0, 1.0), saveats=[0.01], param=[npde.Normal(12.0, 2)])
    p = float(npde.pmean(sol.estimated_de_params[0]))
    assert abs(p - 10.0) < 0.3 * 10.0, p
