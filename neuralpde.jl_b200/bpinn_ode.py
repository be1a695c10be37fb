"""Bayesian ODE posteriors: ``ahmc_bayesian_pinn_ode(prob, chain; ...)`` and ``solve(prob, BNNODE(chain; ...))``
(reference ext/bpinn/advancedHMC_MCMC.jl, ext/bpinn/BPINN_ode.jl).

The log density is the reference's ``LogTargetDensity``, term by term, as engine terms with fixed weights c_k and a
constant: l(θ) = Σ_k c_k L_k(θ) + const + the priors, where L_k is the k-th term loss of the fused kernel (the ODE
residuals of ode.py's lowering).  The chain is the device HMC sampler (csrc/hmc.cu).  StochasticTraining and
WeightedIntervalTraining draw fresh times on the device before every evaluation (PINN_HMC_REDRAW), and a data noise
σ_k(p) = a_k Π_j p_j^e_jk adds Σ_j c_j log|θ.p_j| on the device (``tail_logabs``).  DESIGN section 4.13 lists the terms.
"""
from __future__ import annotations

import math
from typing import List, Optional

import numpy as np
import sympy as sp

from . import engine as _eng
from .engine import Engine, TapSpec, TermSpec, REDUCE_MEAN, REDUCE_WSUM
from .ode import ODEProblem, _Evaluator, _Lowering, _TrialRepresentation, _check_mode, _init_array
from .pinn import BPINNsolution, BPINNstats, HMC, Leapfrog, _hmc_adaptation, _tail_priors, initialparameters
from .strategies import (GridTraining, QuadratureTraining, StochasticTraining, WeightedIntervalTraining, _julia_range,
                         gauss_legendre_box)

_LOG2PI = math.log(2.0 * math.pi)
_SEED_MIX = 0xD1B54A32D192ED03      # odd: seed -> sampler key is a bijection for a fixed strategy seed


def _default_phynewstd(p):
    return [0.05]


# ---- σ(p) -------------------------------------------------------------------------------------------------------
def _sigma_monomials(phynewstd, p_arg, p_syms: List[sp.Symbol], n: int):
    """phynewstd(p) traced with the θ.p symbols: per component k, (a_k, e_k) with σ_k(p) = a_k Π_j p_j^e_kj"""
    out = phynewstd(p_arg)
    vals = list(np.ravel(np.asarray(out, dtype=object)))
    if len(vals) < n:
        raise ValueError("ahmc_bayesian_pinn_ode: phynewstd returns %d standard deviations for %d components"
                         % (len(vals), n))
    form = "a constant or a monomial a * p_1^e_1 * ... * p_m^e_m in the ODE parameters with a != 0 (e.g. 0.1 / p)"
    res = []
    for v in vals[:n]:
        e = sp.sympify(v)
        coeff, rest = e.as_coeff_Mul()
        exps = np.zeros(len(p_syms))
        for base, ex in rest.as_powers_dict().items():
            if base == 1:
                continue
            if base not in p_syms or not ex.is_number or not ex.is_real:
                raise ValueError("ahmc_bayesian_pinn_ode: phynewstd(p) = %s is not supported; the device sampler needs %s"
                                 % (e, form))
            exps[p_syms.index(base)] += float(ex)
        if not coeff.is_number or not coeff.is_real or float(coeff) == 0.0 or not math.isfinite(float(coeff)):
            raise ValueError("ahmc_bayesian_pinn_ode: phynewstd(p) = %s is not supported; the device sampler needs %s"
                             % (e, form))
        res.append((float(coeff), exps))
    return res


# ---- the log density --------------------------------------------------------------------------------------------
class BNNODELogDensity(_TrialRepresentation):
    """The engine problem of ``LogTargetDensity``: terms (``term_names``, ``kinds``), weights ``c``, constant ``const``,
    θ0, the θ.p priors in forward order (``tail``), the log|θ.p| coefficients (``tail_logabs``) and the sampled terms'
    boxes (``sampled``: (term, n, lo, hi))."""

    def __init__(self, prob: ODEProblem, chain, *, strategy=GridTraining, dataset=(), init_params=None, physdt=1 / 20.0,
                 l2std=(0.05,), phystd=(0.05,), phynewstd=_default_phynewstd, param=(), estim_collocate=False,
                 mode="ffma", device=0, seed=0):
        if not isinstance(prob, ODEProblem):
            raise TypeError("ahmc_bayesian_pinn_ode: prob must be an ODEProblem")
        _check_mode(mode, "ahmc_bayesian_pinn_ode", "the tensor-core bf16 modes propagate 1-output networks")
        param = list(param or [])
        ninv = len(param)
        dataset = list(dataset or [])
        lw = _Lowering(prob, ninv > 0, ["t"])
        n = lw.n
        t0, t1 = prob.tspan
        if chain.dims[0] != 1 or chain.dims[-1] != n:
            raise ValueError("ahmc_bayesian_pinn_ode: the chain maps t to the %d components of u0: it needs 1 input and "
                             "%d outputs, has %d and %d" % (n, n, chain.dims[0], chain.dims[-1]))
        strategy = GridTraining(physdt) if strategy is GridTraining else strategy
        if not isinstance(strategy, (GridTraining, StochasticTraining, WeightedIntervalTraining, QuadratureTraining)):
            raise TypeError("ahmc_bayesian_pinn_ode: unsupported training strategy %r" % (strategy,))

        # dataset (advancedHMC_MCMC.jl:409-445)
        if not dataset and ninv > 0:
            raise ValueError("Dataset is Required for Inverse problems performing Parameter Estimation.")
        if not dataset and estim_collocate:
            raise ValueError("Dataset is Required for using the Data Quadrature loglikelihood term.")
        if dataset:
            typed = all(np.ndim(v) == 1 and np.size(v) > 0 and not np.iscomplexobj(v)
                        and np.issubdtype(np.asarray(v).dtype, np.floating) for v in dataset)
            if estim_collocate and (len(dataset) < 3 or not typed):
                raise ValueError("Invalid dataset for Inverse solve with Data Quadrature loss. The dataset would be a "
                                 "timeseries (x̂,t,W) with type: Vector{Vector{AbstractFloat}}")
            if not estim_collocate and (len(dataset) < 2 or not typed):
                raise ValueError("Invalid dataset for Inverse solve. The dataset would be a timeseries (x̂,t) with type: "
                                 "Vector{Vector{AbstractFloat}}")
            if not estim_collocate and len(dataset) == n + 1:     # [x̂..., t]: a uniform W = 1 column (:437-444)
                dataset = dataset + [np.ones(len(dataset[-1]))]
            if len(dataset) != n + 2 or len({np.size(v) for v in dataset}) != 1:
                raise ValueError("Invalid dataset: expected [x̂_1, ..., x̂_%d, t(, W)] of equal lengths, got %d vectors "
                                 "of lengths %s" % (n, len(dataset), [int(np.size(v)) for v in dataset]))
        phystd = np.ravel(np.asarray(phystd, dtype=np.float64))
        l2std = np.ravel(np.asarray(l2std, dtype=np.float64))
        if phystd.size < n:
            raise ValueError("ahmc_bayesian_pinn_ode: phystd has %d entries for %d components" % (phystd.size, n))
        if dataset and l2std.size < n:
            raise ValueError("ahmc_bayesian_pinn_ode: l2std has %d entries for %d components" % (l2std.size, n))

        # θ = [network, θ.p]; θ.p starts at params(param[k])[1] (:468-474), its priors in FORWARD order (priorweights
        # broadcasts invpriors against θ.p, :243-254)
        n_net = chain.n_params
        tail = _tail_priors(param, "ahmc_bayesian_pinn_ode")[::-1] if ninv else []
        if ninv:
            if prob.p is None or np.size(prob.p) != ninv:
                raise ValueError("ahmc_bayesian_pinn_ode: %d priors in `param` for the problem's %d parameters"
                                 % (ninv, 0 if prob.p is None else np.size(prob.p)))
        if init_params is None:
            net0 = initialparameters(np.random.default_rng(seed), chain, np.float64)
        else:
            net0 = _init_array(init_params, mode, "ahmc_bayesian_pinn_ode")
            if net0.shape not in ((n_net,), (n_net + ninv,)):
                raise ValueError("init_params has length %d, the chain needs %d" % (net0.size, n_net))
            net0 = net0[:n_net]
        self.theta0 = np.concatenate([net0.astype(np.float64), [float(p.params()[0]) for p in param]])

        super().__init__(prob, chain, strategy, lw, net0.dtype)
        self.kinds: List[str] = []
        consts = {"phys": 0.0, "data": 0.0, "collocation": 0.0}

        def add(spec, pts, w, weight, name, kind):
            self.add(spec, pts, w, weight, name)
            self.kinds.append(kind)

        # physloglikelihood (:136-238): Σ_k logpdf(MvNormal(r_k(t), phystd_k^2 I), 0)
        res = lw.residuals()
        t_d = np.asarray(dataset[-2], dtype=np.float64) if dataset else np.zeros(0)
        for k in range(n):
            s2 = phystd[k] ** 2
            if isinstance(strategy, QuadratureTraining):
                # ∫ innerdiff(t) dt with innerdiff's one-point logpdf, on a fixed Gauss-Legendre rule
                X, w, _ = gauss_legendre_box((np.array([t0]), np.array([t1])), int(strategy.nodes_per_dim), np.float64)
                add(lw.term(res[k], ["t"], REDUCE_WSUM), X, w, -0.5 / s2, "phys_%d" % (k + 1), "phys")
                consts["phys"] += -0.5 * (t1 - t0) * (_LOG2PI + math.log(s2))
                continue
            if isinstance(strategy, GridTraining):
                ts = np.concatenate([_julia_range(t0, float(strategy.dx), t1), t_d])
                add(lw.term(res[k], ["t"], REDUCE_WSUM), ts, np.ones(ts.size), -0.5 / s2, "phys_%d" % (k + 1), "phys")
                consts["phys"] += -0.5 * ts.size * (_LOG2PI + math.log(s2))
                continue
            if isinstance(strategy, StochasticTraining):
                boxes = [(int(strategy.points), t0, t1)]
            else:
                w = np.asarray(strategy.weights, dtype=np.float64)
                w = w / w.sum()
                h = (t1 - t0) / w.size
                boxes = [(int(strategy.points * wi), t0 + i * h, t0 + (i + 1) * h) for i, wi in enumerate(w)]
            for i, (m, lo, hi) in enumerate(boxes):
                if m < 1:
                    continue
                self.sampled.append((len(self.specs), m, lo, hi))
                add(lw.term(res[k], ["t"], REDUCE_MEAN), None, None, -0.5 * m / s2,
                    "phys_%d" % (k + 1) if len(boxes) == 1 else "phys_%d_interval_%d" % (k + 1, i + 1), "phys")
                consts["phys"] += -0.5 * m * (_LOG2PI + math.log(s2))
            if t_d.size:
                add(lw.term(res[k], ["t"], REDUCE_WSUM), t_d, np.ones(t_d.size), -0.5 / s2, "phys_%d_data" % (k + 1),
                    "phys")
                consts["phys"] += -0.5 * t_d.size * (_LOG2PI + math.log(s2))
        # L2LossData (:110-131): Σ_k logpdf(MvNormal(φ_k(t), l2std_k^2 I), x̂_k)
        if dataset:
            for k in range(n):
                s2 = l2std[k] ** 2
                xk = sp.Symbol("xhat", real=True)
                add(lw.term(lw.phi(k) - xk, ["t", "xhat"], REDUCE_WSUM),
                    np.stack([t_d, np.asarray(dataset[k], dtype=np.float64)]), np.ones(t_d.size), -0.5 / s2,
                    "l2_data_%d" % (k + 1), "data")
                consts["data"] += -0.5 * t_d.size * (_LOG2PI + math.log(s2))
        # L2loss2 (:57-105): Σ_k logpdf(MvNormal((dφ_k/dt - f_k(x̂, p, t)) W, σ_k(p)^2 I), 0), σ_k(p) a monomial:
        # the residual carries 1/σ_k(p), the normalisation -n log|a_k| goes into const and -n e_kj log|p_j| to the device
        logabs = np.zeros(ninv)
        if estim_collocate:
            p_syms = []
            if ninv:
                p_syms = [lw.p_arg] if np.ndim(prob.p) == 0 else list(lw.p_arg)
            sig = _sigma_monomials(phynewstd, lw.p_arg, p_syms, n)
            rows = ["t"] + ["uhat%d" % (j + 1) for j in range(n)]
            pts = np.stack([t_d] + [np.asarray(dataset[j], dtype=np.float64) for j in range(n)])
            W = np.asarray(dataset[-1], dtype=np.float64)
            for k, r in enumerate(lw.collocation_residuals()):
                a_k, e_k = sig[k]
                inv = sp.Float(1.0 / a_k) * sp.Mul(*[ps ** (-sp.nsimplify(e)) for ps, e in zip(p_syms, e_k) if e != 0])
                add(lw.term(r * inv, rows, REDUCE_WSUM), pts, W * W, -0.5, "collocation_%d" % (k + 1), "collocation")
                consts["collocation"] += -0.5 * t_d.size * _LOG2PI - t_d.size * math.log(abs(a_k))
                logabs -= t_d.size * e_k
        self._close("ahmc_bayesian_pinn_ode", ninv, mode, device, "log-likelihood terms")
        self.ninv = ninv
        self.consts, self.const = consts, float(sum(consts.values()))
        self.tail = tail
        self.tail_logabs = logabs if np.any(logabs != 0) else None
        self.dataset = dataset
        self.seed = seed
        # the device samplers' key: the strategy's seed, mixed with the chain's seed so that chains with different
        # seeds see independent point draws (seed = 0 leaves the strategy's draws as NNODE makes them)
        self.sampler_seed = (int(getattr(strategy, "seed", 0)) + _SEED_MIX * int(seed)) % 2 ** 64

    @property
    def c(self) -> np.ndarray:
        """the terms' fixed weights c_k"""
        return self.term_weights

    def _set_samplers(self, eng: Engine):
        for i, m, lo, hi in self.sampled:
            eng.set_sampler(i, m, [lo], [hi], self.sampler_seed)

    def pieces(self, theta, prior_mean: float, prior_std: float) -> dict:
        """The reference's four log-density parts at θ on the handle's current points: "phys", "prior", "data",
        "collocation" (one fused evaluation)"""
        th = np.asarray(theta, dtype=np.float64)
        _, terms, _ = self.engine.loss_grad_host(th.astype(self.dtype), self.c, False)
        v = self.c * np.asarray(terms, dtype=np.float64)
        kinds = np.asarray(self.kinds)
        out = {k: float(v[kinds == k].sum()) + self.consts[k] for k in ("phys", "data", "collocation")}
        if self.tail_logabs is not None:
            out["collocation"] += float(np.dot(self.tail_logabs, np.log(np.abs(th[self.n_net:]))))
        net = th[:self.n_net]
        out["prior"] = float(-0.5 * net.size * (_LOG2PI + 2.0 * math.log(prior_std))
                             - 0.5 * np.sum((net - prior_mean) ** 2) / prior_std ** 2)
        out["prior"] += sum(_logpdf(kind, a, b, x) for (kind, a, b), x in zip(self.tail, th[self.n_net:]))
        return out


def _logpdf(kind: int, a: float, b: float, x: float) -> float:
    """Distributions.jl's logpdf of the tail priors"""
    if kind == _eng.HMC_PRIOR_UNIFORM:
        return -math.log(b - a) if a <= x <= b else -math.inf
    if kind == _eng.HMC_PRIOR_LOGNORMAL:
        if not x > 0:
            return -math.inf
        z = (math.log(x) - a) / b
        return -(z * z + _LOG2PI) / 2 - math.log(b) - math.log(x)
    z = (x - a) / b
    return -(z * z + _LOG2PI) / 2 - math.log(b)


# ---- the sampler ------------------------------------------------------------------------------------------------
def ahmc_bayesian_pinn_ode(prob: ODEProblem, chain, *, strategy=GridTraining, dataset=(), init_params=None,
                           draw_samples: int = 1000, physdt: float = 1 / 20.0, l2std=(0.05,), phystd=(0.05,),
                           phynewstd=_default_phynewstd, priorsNNw=(0.0, 2.0), param=(), nchains: int = 1,
                           autodiff: bool = False, Kernel=HMC, Adaptorkwargs=None, Integratorkwargs=None,
                           MCMCkwargs=None, progress: bool = False, verbose: bool = False, estim_collocate: bool = False,
                           mode: str = "ffma", device: int = 0, seed: int = 0):
    """``ahmc_bayesian_pinn_ode(prob, chain; strategy, dataset, draw_samples, physdt, l2std, phystd, phynewstd,
    priorsNNw, param, ...)`` (reference ext/bpinn/advancedHMC_MCMC.jl:390-581): HMC over θ = [network, θ.p] for the
    log density ``LogTargetDensity`` of the trial solution u0 + (t - t0) N(t).  Returns ``(chain, samples, stats)``:
    the [draw_samples, n_θ] samples (twice) and a dict of AdvancedHMC's statistics, one [draw_samples] array each.

    As the reference: ``HMC`` with ``MCMCkwargs["n_leapfrog"]`` (30) steps from ``find_good_stepsize``, Stan adaptation
    (dual averaging to ``targetacceptancerate``, diagonal mass matrix) over the first ``min(draw_samples ÷ 10, 1000)``
    transitions, warm-up samples kept; θ.p starts at ``params(param[k])[1]``; a ``[x̂, t]`` dataset is padded with
    W = 1.  The chain runs on the device; ``seed`` keys its Philox streams, the initial network parameters and,
    mixed with the strategy's ``seed``, the device point draws of Stochastic / WeightedInterval training (the
    reference uses the global RNG), ``mode`` is "ffma" or "tc_f64".  d/dt is exact for both ``autodiff`` values (the
    reference's default is a forward difference).  ``phynewstd(p)`` must return constants or monomials in p.
    Refused with a message: NUTS / HMCDA, several chains, DenseEuclideanMetric, jittered / tempered leapfrog."""
    ik = dict(Integratorkwargs or {"Integrator": Leapfrog})
    mk = dict({"n_leapfrog": 30}, **(MCMCkwargs or {}))
    if not (Kernel is HMC or isinstance(Kernel, HMC)):
        raise ValueError("ahmc_bayesian_pinn_ode: Kernel %r is not implemented; the device sampler runs HMC with "
                         "MCMCkwargs n_leapfrog (NUTS and HMCDA are not supported)" % (Kernel,))
    adaptor, metric, target_accept = _hmc_adaptation(Adaptorkwargs, nchains, "ahmc_bayesian_pinn_ode")
    if ik.get("Integrator", Leapfrog) is not Leapfrog or set(ik) - {"Integrator"}:
        raise ValueError("ahmc_bayesian_pinn_ode: Integratorkwargs %r are not implemented; JitteredLeapfrog / "
                         "TemperedLeapfrog (jitter_rate, tempering_rate) are not supported (Leapfrog)" % (ik,))
    draw_samples = int(draw_samples)
    if draw_samples < 1:
        raise ValueError("ahmc_bayesian_pinn_ode: draw_samples = %d must be >= 1" % draw_samples)
    ld = BNNODELogDensity(prob, chain, strategy=strategy, dataset=dataset, init_params=init_params, physdt=physdt,
                          l2std=l2std, phystd=phystd, phynewstd=phynewstd, param=param,
                          estim_collocate=estim_collocate, mode=mode, device=device, seed=seed)
    mu_p, sd_p = float(priorsNNw[0]), float(priorsNNw[1])
    th0 = ld.theta0

    def report(when, th):
        pc = ld.pieces(th, mu_p, sd_p)
        print("%s Physics Log-likelihood: %g" % (when, pc["phys"]))
        print("%s Prior Log-likelihood: %g" % (when, pc["prior"]))
        print("%s SSE against dataset Log-likelihood: %g" % (when, pc["data"]))
        if estim_collocate:
            print("%s gradient loss against dataset Log-likelihood: %g" % (when, pc["collocation"]))

    if verbose:
        report("Current", th0)
    eng = ld.engine
    eng.hmc_begin(th0, n_leapfrog=int(mk["n_leapfrog"]), adaptor=adaptor, metric=metric,
                  n_adapts=min(draw_samples // 10, 1000), target_accept=target_accept, step_size=0.0, prior_mean=mu_p, prior_std=sd_p, seed=seed, weights=ld.c, ll_const=ld.const,
                  tail_priors=ld.tail or None, tail_logabs=ld.tail_logabs, redraw=bool(ld.sampled))
    samples, st = eng.hmc_iterate(draw_samples)
    stats = {name: st[:, j].copy() for j, name in enumerate(_eng.HMC_STATS)}
    if verbose:
        print("Sampling Complete.")
        report("Final", samples[-1])
    return samples, samples, stats


# ---- BNNODE and solve -------------------------------------------------------------------------------------------
class BNNODE:
    """``BNNODE(chain, kernel = HMC; strategy, draw_samples, priorsNNw, param, l2std, phystd, phynewstd, dataset,
    physdt, MCMCkwargs, nchains, init_params, Adaptorkwargs, Integratorkwargs, numensemble, estim_collocate, autodiff,
    progress, verbose)`` (reference ext/bpinn/BPINN_ode.jl:5-24), plus the engine options ``mode``, ``device`` and
    ``seed`` of ``ahmc_bayesian_pinn_ode``.  ``numensemble`` defaults to ``floor(draw_samples / 3)``."""

    def __init__(self, chain, kernel=HMC, *, strategy=None, draw_samples: int = 1000, priorsNNw=(0.0, 2.0), param=None,
                 l2std=(0.05,), phystd=(0.05,), phynewstd=_default_phynewstd, dataset=(), physdt: float = 1 / 20.0,
                 MCMCkwargs=None, nchains: int = 1, init_params=None, Adaptorkwargs=None, Integratorkwargs=None,
                 numensemble: Optional[int] = None, estim_collocate: bool = False, autodiff: bool = False,
                 progress: bool = False, verbose: bool = False, mode: str = "ffma", device: int = 0, seed: int = 0):
        self.chain, self.kernel, self.strategy, self.draw_samples = chain, kernel, strategy, int(draw_samples)
        self.priorsNNw, self.param, self.l2std, self.phystd, self.phynewstd = priorsNNw, param, l2std, phystd, phynewstd
        self.dataset, self.physdt, self.MCMCkwargs, self.nchains = dataset, physdt, MCMCkwargs, nchains
        self.init_params, self.Adaptorkwargs, self.Integratorkwargs = init_params, Adaptorkwargs, Integratorkwargs
        self.numensemble = int(math.floor(self.draw_samples / 3)) if numensemble is None else int(numensemble)
        self.estim_collocate, self.autodiff, self.progress, self.verbose = estim_collocate, autodiff, progress, verbose
        self.mode, self.device, self.seed = mode, device, seed


def _network_outputs(chain, dtype, device, ts: np.ndarray, thetas: np.ndarray) -> np.ndarray:
    """N(t) for each row of thetas (network parameters): [len(thetas), n_out, len(ts)], one value-only term per output"""
    n_out = chain.dims[-1]
    network = _Evaluator([TermSpec(dim=1, taps=[TapSpec(net=0, order=0, out=k)], prog=[("tap", 0, 0, 0.0)],
                                   net_rows=[[0]]) for k in range(n_out)], chain, 0, dtype, device)
    network.at(ts)
    out = np.empty((len(thetas), n_out, ts.size))
    for i, th in enumerate(thetas):
        out[i] = network(th)
    return out


def _bnnode_inference(prob: ODEProblem, chain, samples: np.ndarray, numensemble: int, ninv: int, t: np.ndarray, dtype,
                      device: int):
    """The reference's solve-side indexing, literally (BPINN_ode.jl:50-108): curves from the FIRST numensemble of the
    1-based samples (draw_samples - numensemble):draw_samples, parameter ensembles from samples[(end - numensemble):end]
    (numensemble + 1 each); several outputs pass through Float32.  Returns (curves, nn_params, de_params)."""
    ds = samples.shape[0]
    n_net = samples.shape[1] - ninv
    curve_theta = samples[ds - numensemble - 1:ds - 1, :n_net]
    N = _network_outputs(chain, dtype, device, t, curve_theta)
    n_out = N.shape[1]
    if n_out > 1:
        N = N.astype(np.float32).astype(np.float64)
    u0 = np.ravel(np.asarray(prob.u0, dtype=np.float64))
    curves = [u0[k] + N[:, k, :] * (t - prob.tspan[0]) for k in range(n_out)]
    kept = samples[ds - numensemble - 1:]
    nn_params = [kept[:, i].copy() for i in range(n_net)]
    de_params = [kept[:, n_net + j].copy() for j in range(ninv)] if ninv else [None]
    return curves, nn_params, de_params


def solve_bnnode(prob: ODEProblem, alg: BNNODE, *, saveat: float = 1 / 50.0) -> BPINNsolution:
    """``solve(prob::ODEProblem, alg::BNNODE; saveat)`` (reference ext/bpinn/BPINN_ode.jl:26-109): ahmc_bayesian_pinn_ode,
    then ``ensemblesol[k]`` = u0[k] + (t - t0) N_k(t) per kept sample ([numensemble, len(t)]) on t = t0:saveat:t1,
    ``estimated_nn_params`` (one array over the numensemble + 1 last samples per network parameter) and
    ``estimated_de_params`` (one such array per entry of θ.p; ``[None]`` without ``param``); ``timepoints`` is t."""
    if alg.draw_samples < 0:
        raise ValueError("Number of samples to be drawn has to be >=0.")
    if not 0 <= alg.numensemble < alg.draw_samples:
        raise ValueError("BNNODE: need 0 <= numensemble < draw_samples (numensemble = %d, draw_samples = %d)"
                         % (alg.numensemble, alg.draw_samples))
    param = [] if alg.param is None else list(alg.param)
    strategy = GridTraining if alg.strategy is None else alg.strategy
    chain_s, samples, stats = ahmc_bayesian_pinn_ode(
        prob, alg.chain, strategy=strategy, dataset=alg.dataset, draw_samples=alg.draw_samples,
        init_params=alg.init_params, physdt=alg.physdt, l2std=alg.l2std, phystd=alg.phystd, phynewstd=alg.phynewstd,
        priorsNNw=alg.priorsNNw, param=param, nchains=alg.nchains, autodiff=alg.autodiff, Kernel=alg.kernel,
        Adaptorkwargs=alg.Adaptorkwargs, Integratorkwargs=alg.Integratorkwargs, MCMCkwargs=alg.MCMCkwargs,
        progress=alg.progress, verbose=alg.verbose, estim_collocate=alg.estim_collocate, mode=alg.mode,
        device=alg.device, seed=alg.seed)
    t = _julia_range(prob.tspan[0], float(saveat), prob.tspan[1])
    dtype = np.float64 if alg.init_params is None else np.asarray(alg.init_params).dtype
    curves, nn_params, de_params = _bnnode_inference(prob, alg.chain, samples, alg.numensemble, len(param), t, dtype,
                                                     alg.device)
    return BPINNsolution(BPINNstats(chain_s, samples, stats), curves, nn_params, de_params, t)
