"""Float64 restatement of the per-entry priors of csrc/hmc.cu (pinn_hmc_begin_ex): Distributions.jl's Normal(μ, σ),
LogNormal(μ, σ) and Uniform(a, b) on theta's last entries, and a wrapper that lets hmc_oracle.sample run on the
log density the engine samples with such a table.

hmc_oracle.sample adds N(prior_mean, prior_std²) to every entry of theta.  ``with_tail_priors`` hands it a physics
log-likelihood that already holds the tail priors and gives back that Normal prior's share on the tail entries, so the
sampler's target is N over the network entries + the tail priors + the physics part, as on the device."""
from __future__ import annotations

import numpy as np

PRIOR_NORMAL, PRIOR_LOGNORMAL, PRIOR_UNIFORM = 0, 1, 2


def _insupport(kind: int, a: float, b: float, x: float) -> bool:
    """Distributions.jl's insupport: LogNormal x > 0, Uniform a <= x <= b"""
    if kind == PRIOR_LOGNORMAL:
        return x > 0.0
    if kind == PRIOR_UNIFORM:
        return a <= x <= b
    return True


def prior_logpdf(kind: int, a: float, b: float, x: float) -> float:
    """logpdf of one entry; -inf outside the support"""
    if not _insupport(kind, a, b, x):
        return -np.inf
    if kind == PRIOR_UNIFORM:
        return -np.log(b - a)
    lx = np.log(x) if kind == PRIOR_LOGNORMAL else x
    v = -(((lx - a) / b) ** 2 + np.log(2.0 * np.pi)) / 2.0 - np.log(b)
    return v - lx if kind == PRIOR_LOGNORMAL else v


def prior_grad(kind: int, a: float, b: float, x: float) -> float:
    """d/dx prior_logpdf; NaN outside the support"""
    if not _insupport(kind, a, b, x):
        return np.nan
    if kind == PRIOR_NORMAL:
        return -(x - a) / (b * b)
    if kind == PRIOR_LOGNORMAL:
        return -(1.0 + (np.log(x) - a) / (b * b)) / x
    return 0.0


def with_tail_priors(logp_grad, tail, prior_mean: float, prior_std: float):
    """``logp_grad`` for hmc_oracle.sample(..., prior_mean, prior_std) when ``tail`` = [(PRIOR_*, a, b), ...] holds the
    priors of theta's last len(tail) entries: adds them, and removes the N(prior_mean, prior_std²) logpdf and gradient
    that the sampler's target adds on those entries."""
    tail = list(tail)
    iv = 1.0 / (prior_std * prior_std)
    norm_const = 0.5 * np.log(2.0 * np.pi) + np.log(prior_std)

    def f(th):
        l, g = logp_grad(th)
        g = np.asarray(g, dtype=np.float64).copy()
        tt = th[th.size - len(tail):]
        d = tt - prior_mean
        l = l + sum(prior_logpdf(k, a, b, x) for (k, a, b), x in zip(tail, tt))
        l = l + 0.5 * float(np.sum(d * d)) * iv + len(tail) * norm_const
        g[th.size - len(tail):] += [prior_grad(k, a, b, x) for (k, a, b), x in zip(tail, tt)]
        g[th.size - len(tail):] += d * iv
        return l, g

    return f
