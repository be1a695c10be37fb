"""Float64 numpy restatement of the HMC sampler of csrc/hmc.cu, written from AdvancedHMC's documented behaviour
(HMC with a fixed number of leapfrog steps, end-point Metropolis acceptance, find_good_stepsize, Nesterov dual averaging,
Stan's windowed diagonal mass-matrix adaptation) and from the engine's Philox streams, so that a GPU run can be replayed
draw for draw.  ``logp_grad(theta) -> (l, grad)`` is the physics log-likelihood; the Normal prior is added here."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, List, Optional

import numpy as np

M32 = 0xFFFFFFFF
TAG_MOMENTUM, TAG_STEPSIZE_MOMENTUM, TAG_ACCEPT = 0, 1, 2
STATS = ("step_size", "acceptance_rate", "is_accept", "log_density", "hamiltonian_energy",
         "hamiltonian_energy_error", "numerical_error", "is_adapt")


# ---- Philox4x32-10 (Salmon et al., SC'11), vectorised over counters -------------------------------------------------
def philox4x32_10(c, k0: int, k1: int):
    """c: four uint64 arrays holding 32-bit words; returns the four output words."""
    c0, c1, c2, c3 = (np.asarray(x, dtype=np.uint64) & M32 for x in c)
    k0, k1 = np.uint64(k0 & M32), np.uint64(k1 & M32)
    for _ in range(10):
        p0 = c0 * np.uint64(0xD2511F53)
        p1 = c2 * np.uint64(0xCD9E8D57)
        hi0, lo0 = p0 >> np.uint64(32), p0 & np.uint64(M32)
        hi1, lo1 = p1 >> np.uint64(32), p1 & np.uint64(M32)
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0 = (k0 + np.uint64(0x9E3779B9)) & np.uint64(M32)
        k1 = (k1 + np.uint64(0xBB67AE85)) & np.uint64(M32)
    return c0, c1, c2, c3


def _u53(hi, lo):
    bits = (np.asarray(hi, dtype=np.uint64) << np.uint64(32)) | np.asarray(lo, dtype=np.uint64)
    return (bits >> np.uint64(11)).astype(np.float64) * (1.0 / 9007199254740992.0)


def sampler_uniform_f64(n: int, dim: int, seed: int, term: int = 0, draw: int = 0) -> np.ndarray:
    """The fp64 draws of the engine's StochasticTraining sampler (pinn_set_sampler with lb = 0, ub = 1): (dim, n)."""
    key = (seed + 0x9E3779B97F4A7C15 * (term + 1)) & (2 ** 64 - 1)
    p = np.arange(n, dtype=np.uint64)
    out = np.empty((dim, n))
    for r0 in range(0, dim, 2):
        c = (p & np.uint64(M32), p >> np.uint64(32), np.full(n, (r0 ^ (draw << 8)) & M32, dtype=np.uint64),
             np.full(n, (draw >> 24) & M32, dtype=np.uint64))
        w = philox4x32_10(c, key, key >> 32)
        for j in range(2):
            if r0 + j < dim:
                out[r0 + j] = _u53(w[2 * j], w[2 * j + 1])
    return out


def normals(seed: int, t: int, tag: int, n: int) -> np.ndarray:
    """Standard normals 0..n-1 of transition t in stream tag: Box-Muller on one Philox draw per pair (2j, 2j+1)."""
    j = np.arange((n + 1) // 2, dtype=np.uint64)
    c = (j, np.full(j.size, t & M32, dtype=np.uint64), np.full(j.size, (t >> 32) & M32, dtype=np.uint64),
         np.full(j.size, tag, dtype=np.uint64))
    w = philox4x32_10(c, seed, seed >> 32)
    u1 = _u53(w[0], w[1]) + 1.0 / 9007199254740992.0
    u2 = _u53(w[2], w[3])
    rad = np.sqrt(-2.0 * np.log(u1))
    z = np.empty(2 * j.size)
    z[0::2] = rad * np.cos(2.0 * np.pi * u2)
    z[1::2] = rad * np.sin(2.0 * np.pi * u2)
    return z[:n]


def uniform(seed: int, t: int, tag: int = TAG_ACCEPT) -> float:
    w = philox4x32_10((np.zeros(1), np.array([t & M32]), np.array([(t >> 32) & M32]), np.array([tag])), seed, seed >> 32)
    return float(_u53(w[0], w[1])[0])


# ---- adaptation -----------------------------------------------------------------------------------------------------
def stan_windows(n_adapts: int):
    """(init buffer, [(first, last) of each window], term buffer), 1-based transitions (Stan's windowed_adaptation)."""
    init, term, win = 75, 50, 25
    if init + win + term > n_adapts:
        init, term = int(np.floor(0.15 * n_adapts)), int(np.floor(0.1 * n_adapts))
        win = n_adapts - init - term
    start, end = init + 1, n_adapts - term
    windows = []
    if end >= start:
        first, last = start, start + win - 1
        while True:
            windows.append((first, last))
            if last >= end:
                break
            win *= 2
            nxt = last + win
            if nxt + 2 * win > end:
                nxt = end
            first, last = last + 1, nxt
    return init, windows, term


@dataclass
class DualAveraging:
    """Nesterov dual averaging of log(step size) (Hoffman & Gelman 2014; AdvancedHMC's defaults)."""
    eps: float
    delta: float = 0.8
    gamma: float = 0.05
    t0: float = 10.0
    kappa: float = 0.75
    m: float = 0.0
    x_bar: float = 0.0
    h_bar: float = 0.0
    mu: float = field(init=False)

    def __post_init__(self):
        self.mu = np.log(10.0 * self.eps)

    def update(self, alpha: float):
        m = self.m + 1.0
        eta_h = 1.0 / (m + self.t0)
        h_bar = (1.0 - eta_h) * self.h_bar + eta_h * (self.delta - alpha)
        x = self.mu - h_bar * np.sqrt(m) / self.gamma
        eta_x = m ** (-self.kappa)
        x_bar = (1.0 - eta_x) * self.x_bar + eta_x * x
        eps = np.exp(x)
        if np.isfinite(eps):
            self.m, self.h_bar, self.x_bar, self.eps = m, h_bar, x_bar, eps

    def reset(self):
        self.mu = np.log(10.0 * self.eps)
        self.m = self.x_bar = self.h_bar = 0.0

    def finalize(self):
        self.eps = float(np.exp(self.x_bar))


def welford_variance(n: int, m2: np.ndarray) -> np.ndarray:
    return (n / ((n + 5.0) * (n - 1.0))) * m2 + 1e-3 * (5.0 / (n + 5.0))


# ---- sampler --------------------------------------------------------------------------------------------------------
class _Target:
    def __init__(self, logp_grad, prior_mean, prior_std, n):
        self.f, self.mu, self.iv = logp_grad, prior_mean, 1.0 / (prior_std * prior_std)
        self.const = -0.5 * n * np.log(2.0 * np.pi) - n * np.log(prior_std)

    def __call__(self, th):
        l, g = self.f(th)
        d = th - self.mu
        return l + self.const - 0.5 * float(np.sum(d * d)) * self.iv, np.asarray(g, dtype=np.float64) - d * self.iv


def _leapfrog(target, th, r, g, eps, minv, n_steps):
    """(theta, r, l, g, finite) after n_steps leapfrog steps; stops at the first non-finite value"""
    h = 0.5 * eps
    l = np.nan
    for _ in range(n_steps):
        r = r + h * g
        th = th + eps * (minv * r)
        l, g = target(th)
        if not (np.isfinite(l) and np.all(np.isfinite(g))):
            return th, r, l, g, False
        r = r + h * g
    ok = np.isfinite(l) and all(np.all(np.isfinite(v)) for v in (th, r, g))
    return th, r, l, g, ok


def _energy(l, r, minv, ok):
    return -l + 0.5 * float(np.sum(minv * r * r)) if ok else np.inf


def find_good_stepsize(target, th0, l0, g0, seed: int, trace: Optional[list] = None) -> float:
    """AdvancedHMC's find_good_stepsize with one momentum draw (unit metric)."""
    r0 = normals(seed, 0, TAG_STEPSIZE_MOMENTUM, th0.size)
    minv = np.ones_like(th0)
    h0 = _energy(l0, r0, minv, True)

    def dh(eps):
        th, r, l, g, ok = _leapfrog(target, th0, r0, g0, eps, minv, 1)
        v = h0 - _energy(l, r, minv, ok)
        if trace is not None:
            trace.append((eps, v))
        return v

    a_min, a_cross, a_max, d = 0.25, 0.5, 0.75, 2.0
    eps = eps1 = 0.1
    direction = 1 if dh(eps) > np.log(a_cross) else -1
    for _ in range(100):
        eps1 = d * eps if direction == 1 else eps / d
        v = dh(eps)                      # AdvancedHMC evaluates the current eps and moves to eps1 afterwards
        if direction == 1 and not (v > np.log(a_cross)):
            break
        if direction == -1 and not (v < np.log(a_cross)):
            break
        eps = eps1
    if eps > eps1:
        eps, eps1 = eps1, eps
    for _ in range(100):
        mid = 0.5 * (eps + eps1)
        v = dh(mid)
        if np.exp(v) > a_max:
            eps = mid
        elif np.exp(v) < a_min:
            eps1 = mid
        else:
            eps = mid
            break
    return eps


@dataclass
class Chain:
    eps0: float
    samples: np.ndarray
    stats: np.ndarray
    minv: np.ndarray


def sample(logp_grad: Callable, theta0, n: int, *, n_leapfrog: int = 30, adapt: bool = True, diag: bool = True,
           n_adapts: int = 0, delta: float = 0.8, step_size: float = 0.0, prior_mean: float = 0.0,
           prior_std: float = 1.0, seed: int = 0) -> Chain:
    th = np.asarray(theta0, dtype=np.float64).copy()
    target = _Target(logp_grad, prior_mean, prior_std, th.size)
    l, g = target(th)
    eps0 = step_size if step_size > 0 else find_good_stepsize(target, th, l, g, seed)
    da = DualAveraging(eps0, delta)
    _, windows, _ = stan_windows(n_adapts)
    ends = {w[1] for w in windows}
    minv = np.ones_like(th)
    wn, wmean, wm2 = 0, np.zeros_like(th), np.zeros_like(th)
    samples, stats = np.empty((n, th.size)), np.empty((n, len(STATS)))
    for t in range(n):
        i = t + 1
        r = normals(seed, t, TAG_MOMENTUM, th.size) / np.sqrt(minv)
        h0 = _energy(l, r, minv, True)
        th1, r1, l1, g1, ok = _leapfrog(target, th, r, g, da.eps, minv, n_leapfrog)
        h1 = _energy(l1, r1, minv, ok)
        alpha = min(1.0, float(np.exp(h0 - h1))) if ok else 0.0
        accept = uniform(seed, t) < alpha
        adapting = adapt and i <= n_adapts
        stats[t] = (da.eps, alpha, accept, l1 if accept else l, h1 if accept else h0, h1 - h0 if accept else 0.0,
                    not ok, adapting)
        if accept:
            th, l, g = th1, l1, g1
        samples[t] = th
        if adapting:
            da.update(alpha)
            in_window = any(a <= i <= b for a, b in windows)
            if in_window and diag:
                wn += 1
                dlt = th - wmean
                wmean = wmean + dlt / wn
                wm2 = wm2 + dlt * (th - wmean)
            if i in ends:
                if diag and wn >= 2:
                    minv = welford_variance(wn, wm2)
                wn, wmean, wm2 = 0, np.zeros_like(th), np.zeros_like(th)
                da.reset()
            if i == n_adapts:
                da.finalize()
    return Chain(eps0, samples, stats, minv)
