"""Float64 restatement of NNODE's loss (reference src/ode_solve.jl) with torch autograd, independent of the engine's
lowering and kernel: f is evaluated through ``sympy.lambdify`` of f traced with plain symbols, the network is a torch
MLP in Lux's parameter layout, d/dt is either exact (autograd) or the reference's forward difference with
ε = sqrt(eps(Float64)) (:206-213)."""
import math

import numpy as np
import sympy as sp
import torch

_TORCH = {"sin": torch.sin, "cos": torch.cos, "exp": torch.exp, "log": torch.log, "tanh": torch.tanh,
          "sqrt": torch.sqrt, "Abs": torch.abs, "pi": math.pi, "E": math.e}


def act(name, z):
    if name == "identity":
        return z
    if name == "tanh":
        return torch.tanh(z)
    if name == "sigmoid":
        return torch.sigmoid(z)
    if name == "sin":
        return torch.sin(z)
    if name == "softplus":
        return torch.nn.functional.softplus(z)
    if name == "swish":
        return z * torch.sigmoid(z)
    if name == "gelu":      # NNlib's gelu (tanh form)
        return 0.5 * z * (1 + torch.tanh(math.sqrt(2 / math.pi) * (z + 0.044715 * z ** 3)))
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


class NNODEOracle:
    def __init__(self, prob, chain, param_estim=False):
        self.prob, self.dims, self.acts = prob, list(chain.dims), list(chain.acts)
        self.n_net = chain.n_params
        self.n = 1 if np.ndim(prob.u0) == 0 else len(np.ravel(prob.u0))
        self.u0 = torch.tensor(np.ravel(np.asarray(prob.u0, dtype=np.float64)))
        self.t0 = prob.tspan[0]
        self.param_estim = param_estim
        us = [sp.Symbol("u%d" % j) for j in range(self.n)]
        np_ = 0 if prob.p is None else np.size(prob.p)
        ps = [sp.Symbol("q%d" % j) for j in range(np_)]
        t = sp.Symbol("t")
        u_arg = us[0] if np.ndim(prob.u0) == 0 else us
        p_arg = (ps[0] if np.ndim(prob.p) == 0 else ps) if param_estim else prob.p
        out = prob.f.f(u_arg, p_arg, t)
        outs = [out] if np.ndim(prob.u0) == 0 else list(out)
        self.f = [sp.lambdify(us + ps + [t], sp.sympify(e), modules=[_TORCH, "math"]) for e in outs]
        self.np = np_

    def p_of(self, theta):
        if self.param_estim:
            return [theta[self.n_net + j] for j in range(self.np)]
        return [torch.tensor(float(v), dtype=torch.float64) for v in np.ravel(np.asarray(self.prob.p if self.np else [],
                                                                                           dtype=np.float64))]

    def phi(self, theta, t):
        """(n, m)"""
        return self.u0[:, None] + (t[None, :] - self.t0) * mlp(theta, self.dims, self.acts, t[None, :])

    def dphi(self, theta, t, derivative="exact"):
        if derivative == "fd":
            e = math.sqrt(np.finfo(np.float64).eps)
            return (self.phi(theta, t + e) - self.phi(theta, t)) / e
        tt = t.detach().clone().requires_grad_(True)
        ph = self.phi(theta, tt)
        return torch.stack([torch.autograd.grad(ph[k].sum(), tt, create_graph=True)[0] for k in range(self.n)])

    def fval(self, u, theta, t):
        """f(u, p, t) with u (n, m) -> (n, m)"""
        args = [u[j] for j in range(self.n)] + self.p_of(theta) + [t]
        return torch.stack([torch.as_tensor(fk(*args), dtype=torch.float64) * torch.ones_like(t) for fk in self.f])

    def residual(self, theta, t, derivative="exact"):
        """(n, m): dφ/dt - f(φ, p, t)"""
        return self.dphi(theta, t, derivative) - self.fval(self.phi(theta, t), theta, t)

    # ---- the reference's loss pieces -------------------------------------------------------------------------
    def inner_loss(self, theta, t, batch, derivative="exact"):
        """batch: sum(abs2, r) / length(t) (:227-239); else Σ_t sum(abs2, r(t)) (:222-225, :275)"""
        r = self.residual(theta, t, derivative)
        return (r ** 2).sum() / t.numel() if batch else (r ** 2).sum()

    def quadrature_loss(self, theta, nodes, weights, derivative="exact"):
        """∫ abs2(Σ_k r_k^2) dt by the given rule (:246-267)"""
        s = (self.residual(theta, nodes, derivative) ** 2).sum(0)
        return (weights * s ** 2).sum()

    def l2_data(self, theta, dataset):
        """generate_L2lossData (:338-346)"""
        t = torch.tensor(np.asarray(dataset[-2], dtype=np.float64))
        ph = self.phi(theta, t)
        return sum(((ph[k] - torch.tensor(np.asarray(dataset[k], dtype=np.float64))) ** 2).sum() for k in range(self.n))

    def l2_collocate(self, theta, dataset, derivative="exact"):
        """generate_L2loss2 (:352-380)"""
        t = torch.tensor(np.asarray(dataset[-2], dtype=np.float64))
        W = torch.tensor(np.asarray(dataset[-1], dtype=np.float64))
        uh = torch.stack([torch.tensor(np.asarray(dataset[j], dtype=np.float64)) for j in range(self.n)])
        d = self.dphi(theta, t, derivative) - self.fval(uh, theta, t)
        return sum(((d[k] ** 2) * W).sum() for k in range(self.n))

    def data_loss(self, theta, k, t, y):
        """the structured additional loss: mean(abs2, φ_k(t) - y)"""
        t = torch.tensor(np.asarray(t, dtype=np.float64))
        return ((self.phi(theta, t)[k] - torch.tensor(np.asarray(y, dtype=np.float64))) ** 2).mean()

    def total_loss(self, theta, main, extras=(), tstops=None, n_orig=None, batch=True, derivative="exact"):
        """total_loss (:471-501): main + extras, then the tstops combination (n_orig None: Quadrature, L + L_t)"""
        L = main + sum(extras)
        if tstops is None:
            return L
        Lt = self.inner_loss(theta, torch.tensor(np.asarray(tstops, dtype=np.float64)), batch, derivative)
        if n_orig is None:
            return L + Lt
        nt = len(tstops)
        return (L * n_orig + Lt * nt) / (n_orig + nt)
