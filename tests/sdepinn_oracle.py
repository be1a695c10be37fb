"""Float64 restatement of SDEPINN's loss (reference src/NN_SDE_weaksolve.jl:121-272) with torch autograd, independent
of the engine's lowering and kernel.  The drift f, the noise g and the x-derivatives of f and g² are written out per
case.  The network is a torch MLP in Lux's parameter layout; its derivatives are exact (autograd) or the reference's
central-difference stencils (ε = eps^(1/(2 + order)), src/pinn_types.jl:445-482).  The flux at x_b is the reference's
f p̂ - ½ g² ∂x p̂ (``flux="quirk"``) or the exact f p̂ - ½ ∂x(g² p̂) (``flux="exact"``).  The norm integral is a
Gauss-Legendre rule of q nodes over [x_0, x_end]."""
import math
from dataclasses import dataclass
from typing import Callable

import numpy as np
import torch


def act(name, z):
    if name == "identity":
        return z
    if name == "tanh":
        return torch.tanh(z)
    if name == "logcosh":       # NNlib: x + softplus(-2x) - log 2
        # softplus as log1p(exp(y)) for every y used here (|y| <= 2000): smooth at 0, where autograd through |y| or
        # relu(y) would take the subgradient 0, and exact up to y = 2000, where torch's default threshold of 20 is not
        return z + torch.nn.functional.softplus(-2 * z, threshold=2000.0) - math.log(2.0)
    raise ValueError(name)


def mlp(theta, dims, acts, x):
    """x (d, m) -> (out, m); θ per layer: W (out × in, column-major) then b"""
    o, h = 0, x
    for a, (i, j) in zip(acts, zip(dims[:-1], dims[1:])):
        W = theta[o:o + i * j].reshape(i, j).T
        o += i * j
        b = theta[o:o + j]
        o += j
        h = act(a, W @ h + b[:, None])
    return h


@dataclass
class Case:
    """f(x), f'(x), g²(x), (g²)'(x), (g²)''(x) as torch functions; u0, the initial pdf value and the domain"""
    f: Callable
    df: Callable
    g2: Callable
    dg2: Callable
    d2g2: Callable
    u0: float
    pdf0: float
    tspan: tuple
    x_0: float
    x_end: float


def ou_case():
    """test/NNSDE2 OU: f = -u, g = 1, u0 = 0.5, Normal(0.5, 0.05), x in [-4, 4]"""
    z = lambda x: torch.zeros_like(x)      # noqa: E731
    pdf0 = 1.0 / (0.05 * math.sqrt(2 * math.pi))
    return Case(lambda x: -x, lambda x: -torch.ones_like(x), lambda x: torch.ones_like(x), z, z, 0.5, pdf0,
                (0.0, 1.0), -4.0, 4.0)


def gbm_case():
    """test/NNSDE2 GBM: f = 0.2 u, g = 0.3 u, u0 = 1, LogNormal(0, 0.05), x in [0, 3]"""
    pdf0 = 1.0 / (0.05 * math.sqrt(2 * math.pi))
    return Case(lambda x: 0.2 * x, lambda x: 0.2 * torch.ones_like(x), lambda x: 0.09 * x * x, lambda x: 0.18 * x,
                lambda x: 0.18 * torch.ones_like(x), 1.0, pdf0, (0.0, 1.0), 0.0, 3.0)


def julia_range(lo, step, hi):
    n = int(np.floor((hi - lo) / step + 1e-10)) + 1
    return lo + step * np.arange(n, dtype=np.float64)


class SDEPINNOracle:
    def __init__(self, case: Case, dims, acts, Nt=20, dx=0.05, lam=1.0, q=64, deriv="exact", flux="quirk"):
        self.c, self.dims, self.acts = case, list(dims), list(acts)
        self.lam, self.q, self.deriv, self.flux = lam, q, deriv, flux
        t0, t1 = case.tspan
        dt = (t1 - t0) / Nt
        self.xs, self.ts = julia_range(case.x_0, dx, case.x_end), julia_range(t0, dt, t1)
        gx, gt = np.meshgrid(self.xs, self.ts, indexing="ij")
        self.grid = np.stack([gx.ravel(order="F"), gt.ravel(order="F")])      # x fastest
        self.flux_at = [xb for xb in (case.x_0, case.x_end)
                        if not (abs(case.f(torch.tensor(xb))) == 0 and abs(case.g2(torch.tensor(xb))) == 0)]
        nodes, w = np.polynomial.legendre.leggauss(q)
        h = 0.5 * (case.x_end - case.x_0)
        self.nodes, self.w = case.x_0 + h * (nodes + 1.0), h * w

    # -- p̂ and its derivatives ----------------------------------------------------------------------------------
    def p(self, th, x, t):
        return mlp(th, self.dims, self.acts, torch.stack([x, t]))[0]

    def _derivs(self, th, x, t):
        """p, p_t, p_x, p_xx at the points (x, t)"""
        if self.deriv == "exact":
            x, t = x.clone().requires_grad_(True), t.clone().requires_grad_(True)
            p = self.p(th, x, t)
            px, pt = torch.autograd.grad(p.sum(), (x, t), create_graph=True)
            pxx = torch.autograd.grad(px.sum(), x, create_graph=True)[0]
            return p, pt, px, pxx
        e1, e2 = np.finfo(np.float64).eps ** (1 / 3), np.finfo(np.float64).eps ** (1 / 4)
        p = self.p(th, x, t)
        pt = (self.p(th, x, t + e1) - self.p(th, x, t - e1)) / (2 * e1)
        px = (self.p(th, x + e1, t) - self.p(th, x - e1, t)) / (2 * e1)
        pxx = (self.p(th, x + e2, t) + self.p(th, x - e2, t) - 2 * p) / e2 ** 2
        return p, pt, px, pxx

    # -- residuals ----------------------------------------------------------------------------------------------
    def pde_residual(self, th, X):
        c = self.c
        x, t = torch.tensor(X[0]), torch.tensor(X[1])
        p, pt, px, pxx = self._derivs(th, x, t)
        # Dt p + Dx(f p) - ½ Dxx(g² p), product rule written out
        return pt + c.df(x) * p + c.f(x) * px - 0.5 * (c.d2g2(x) * p + 2 * c.dg2(x) * px + c.g2(x) * pxx)

    def flux_residual(self, th, xb):
        c = self.c
        t = torch.tensor(self.ts)
        x = torch.full_like(t, xb)
        p, _, px, _ = self._derivs(th, x, t)
        J = c.f(x) * p - 0.5 * c.g2(x) * px
        return J - 0.5 * c.dg2(x) * p if self.flux == "exact" else J

    def ic_residual(self, th):
        c = self.c
        return self.p(th, torch.tensor([c.u0]), torch.tensor([c.tspan[0]])) - c.pdf0

    def integrals(self, th):
        """∫ p̂(x, t_i) dx for every grid time (Gauss-Legendre)"""
        xs, w = torch.tensor(self.nodes), torch.tensor(self.w)
        out = []
        for ti in self.ts:
            out.append((w * self.p(th, xs, torch.full_like(xs, ti))).sum())
        return torch.stack(out)

    def term_losses(self, th):
        """[pde, ic, flux at each kept boundary..., norm]: means of squares, and Σ_t (I_t - 1)² unweighted"""
        terms = [self.pde_residual(th, self.grid).pow(2).mean(), self.ic_residual(th).pow(2).mean()]
        terms += [self.flux_residual(th, xb).pow(2).mean() for xb in self.flux_at]
        terms.append((self.integrals(th) - 1.0).pow(2).sum())
        return terms

    def loss_and_grad(self, theta):
        th = torch.tensor(np.asarray(theta, dtype=np.float64), requires_grad=True)
        terms = self.term_losses(th)
        total = sum(terms[:-1]) + self.lam * terms[-1]
        g, = torch.autograd.grad(total, th)
        return float(total), np.array([float(v) for v in terms]), g.numpy()
