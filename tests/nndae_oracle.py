"""Float64 restatement of NNDAE's loss (reference src/dae_solve.jl:48-82) with torch autograd, independent of the
engine's lowering and kernel: f(du, u, p, t) is evaluated through ``sympy.lambdify`` of f traced with plain symbols, the
network is a torch MLP in Lux's parameter layout, and d/dt is either the reference's forward difference with
ε = sqrt(eps(Float64)) or exact (autograd).  Also the two reference problems (test/NNODE/nndae__dae_case_*.jl) and the
closed-form solutions of their mass-matrix ODEs."""
import math

import numpy as np
import sympy as sp
import torch

import neuralpde_jl_b200 as npde
from nnode_oracle import act as _act

_TORCH = {"sin": torch.sin, "cos": torch.cos, "exp": torch.exp, "log": torch.log, "tanh": torch.tanh,
          "sqrt": torch.sqrt, "Abs": torch.abs, "pi": math.pi, "E": math.e}


def act(name, z):
    return torch.cos(z) if name == "cos" else _act(name, z)


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


class NNDAEOracle:
    def __init__(self, prob, chain):
        self.prob, self.dims, self.acts = prob, list(chain.dims), list(chain.acts)
        self.n = 1 if np.ndim(prob.u0) == 0 else len(np.ravel(prob.u0))
        self.u0 = torch.tensor(np.ravel(np.asarray(prob.u0, dtype=np.float64)))
        self.t0 = prob.tspan[0]
        self.dv = list(prob.differential_vars)
        dus = [sp.Symbol("du%d" % j) for j in range(self.n)]
        us = [sp.Symbol("u%d" % j) for j in range(self.n)]
        t = sp.Symbol("t")
        out = prob.f.f(dus, us, prob.p, t)
        self.f = [sp.lambdify(dus + us + [t], sp.sympify(e), modules=[_TORCH, "math"]) for e in np.ravel(np.asarray(out, dtype=object))]

    def phi(self, theta, t):
        """(n, m): u0 + (t - t0) N(t)"""
        return self.u0[:, None] + (t[None, :] - self.t0) * mlp(theta, self.dims, self.acts, t[None, :])

    def dfdx(self, theta, t, derivative="fd"):
        """(n, m): dφ/dt of the differential components, 0 for the algebraic ones (:48-62)"""
        if derivative == "fd":
            e = math.sqrt(np.finfo(np.float64).eps)
            d = (self.phi(theta, t + e) - self.phi(theta, t)) / e
        else:
            tt = t.detach().clone().requires_grad_(True)
            ph = self.phi(theta, tt)
            d = torch.stack([torch.autograd.grad(ph[k].sum(), tt, create_graph=True)[0] for k in range(self.n)])
        return torch.stack([d[k] if self.dv[k] else torch.zeros_like(t) for k in range(self.n)])

    def per_point(self, theta, t, derivative="fd"):
        """(m,): Σ_k f_k(dφ(t_i), φ(t_i), p, t_i)²"""
        du, u = self.dfdx(theta, t, derivative), self.phi(theta, t)
        args = [du[k] for k in range(self.n)] + [u[k] for k in range(self.n)] + [t]
        return sum((torch.as_tensor(fk(*args), dtype=torch.float64) * torch.ones_like(t)) ** 2 for fk in self.f)

    def inner_loss(self, theta, t, derivative="fd"):
        """Σ_i Σ_k f_k² / n (:64-73)"""
        return self.per_point(theta, t, derivative).sum() / t.numel()

    def loss(self, theta, t, derivative="fd"):
        """sum(abs2, inner_loss) (:75-82): the square of the mean"""
        return self.inner_loss(theta, t, derivative) ** 2

    def loss_and_grad(self, theta, t, derivative="exact"):
        th = torch.tensor(np.asarray(theta, dtype=np.float64)).requires_grad_(True)
        L = self.loss(th, torch.tensor(np.asarray(t, dtype=np.float64)), derivative)
        (G,) = torch.autograd.grad(L, th)
        return float(L.detach()), G.numpy()


# ---- the reference problems ---------------------------------------------------------------------------------------
def case_i():
    """nndae__dae_case_i.jl: u₁' = cos 2πt, 0 = u₂ + cos 2πt on (0, 1)"""
    f = lambda du, u, p, t: [sp.cos(2 * sp.pi * t) - du[0], u[1] + sp.cos(2 * sp.pi * t) - du[1]]   # noqa: E731
    prob = npde.DAEProblem(f, [0.0, 0.0], [1.0, -1.0], (0.0, 1.0), differential_vars=[True, False])
    chain = npde.Chain(npde.Dense(1, 15, "cos"), npde.Dense(15, 15, "sin"), npde.Dense(15, 2))
    return prob, chain


def case_ii():
    """nndae__dae_case_ii.jl: 0 = u₁ - t, u₂' = u₂ - t on (0, π/2) (Float32 tspan)"""
    f = lambda du, u, p, t: [u[0] - t - du[0], u[1] - t - du[1]]   # noqa: E731
    prob = npde.DAEProblem(f, [0.0, 0.0], [0.0, 0.0], (0.0, float(np.float32(np.pi / 2))), differential_vars=[False, True])
    chain = npde.Chain(npde.Dense(1, 15, "sigmoid"), npde.Dense(15, 2))
    return prob, chain


def ground_i(t):
    t = np.asarray(t, dtype=np.float64)
    return np.stack([1 + np.sin(2 * np.pi * t) / (2 * np.pi), -np.cos(2 * np.pi * t)])


def ground_ii(t):
    t = np.asarray(t, dtype=np.float64)
    return np.stack([t, 1 + t - np.exp(t)])


DT = float(np.float32(1 / 100.0))      # dt = 1 / 100.0f0
