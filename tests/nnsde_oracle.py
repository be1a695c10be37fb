"""Float64 restatement of NNSDE's loss (reference src/NN_SDE_solve.jl) with torch autograd, independent of the engine's
lowering and kernel: inner_sde_loss (:243-342) over the reference's input layout (a Vector of (1 + n_z) x n_samples
matrices, one per time), the Quadrature integrand (:498-507) and generate_EM_L2loss (:452-484).  f and g are evaluated
through ``sympy.lambdify``; d/dt is exact (autograd) or the reference's forward difference with ε = sqrt(eps(Float64))
(:213-224).  Also the numpy replay of the device KKL sampler (include/pinn_b200.h)."""
import math

import numpy as np
import sympy as sp
import torch

from nnode_oracle import _TORCH, mlp


class NNSDEOracle:
    def __init__(self, prob, chain, param_estim=False):
        self.prob, self.dims, self.acts = prob, list(chain.dims), list(chain.acts)
        self.n_net = chain.n_params
        self.n_z = self.dims[0] - 1
        self.n = 1 if np.ndim(prob.u0) == 0 else len(np.ravel(prob.u0))
        self.u0 = torch.tensor(np.ravel(np.asarray(prob.u0, dtype=np.float64)))
        self.t0 = prob.tspan[0] / prob.tspan[1]
        self.param_estim = param_estim
        us = [sp.Symbol("u%d" % j) for j in range(self.n)]
        self.np = 0 if prob.p is None else np.size(prob.p)
        ps = [sp.Symbol("q%d" % j) for j in range(self.np)]
        t = sp.Symbol("t")
        u_arg = us[0] if np.ndim(prob.u0) == 0 else us
        p_arg = (ps[0] if np.ndim(prob.p) == 0 else ps) if param_estim else prob.p

        def lam(fn):
            out = fn(u_arg, p_arg, t)
            outs = [out] if np.ndim(prob.u0) == 0 else list(out)
            return [sp.lambdify(us + ps + [t], sp.sympify(e), modules=[_TORCH, "math"]) for e in outs]
        self.f, self.g = lam(prob.f.f), lam(prob.g)

    def p_of(self, theta):
        if self.param_estim:
            return [theta[self.n_net + j] for j in range(self.np)]
        return [torch.tensor(float(v), dtype=torch.float64)
                for v in np.ravel(np.asarray(self.prob.p if self.np else [], dtype=np.float64))]

    def _eval(self, fns, u, theta, t):
        args = [u[j] for j in range(self.n)] + self.p_of(theta) + [t]
        return torch.stack([torch.as_tensor(fk(*args), dtype=torch.float64) * torch.ones_like(t) for fk in fns])

    def phi(self, theta, X):
        """SDEPhi on a (1 + n_z, m) matrix: (n, m)"""
        return self.u0[:, None] + (X[0][None, :] - self.t0) * mlp(theta, self.dims, self.acts, X)

    def dudt(self, theta, X, derivative="exact"):
        if derivative == "fd":
            e = math.sqrt(np.finfo(np.float64).eps)
            return (self.phi(theta, torch.cat([X[:1] + e, X[1:]])) - self.phi(theta, X)) / e
        t = X[0].detach().clone().requires_grad_(True)
        ph = self.phi(theta, torch.cat([t[None, :], X[1:]]))
        return torch.stack([torch.autograd.grad(ph[k].sum(), t, create_graph=True)[0] for k in range(self.n)])

    def fs(self, theta, X):
        """f(u) + g(u) √2 Σ_j z_j cos((j - ½) π t) at u = φ(X), (n, m)"""
        u, t = self.phi(theta, X), X[0]
        w = math.sqrt(2) * sum(X[1 + j] * torch.cos((j + 1 - 0.5) * math.pi * t) for j in range(self.n_z))
        return self._eval(self.f, u, theta, t) + self._eval(self.g, u, theta, t) * w

    def residual(self, theta, X, derivative="exact"):
        return self.fs(theta, X) - self.dudt(theta, X, derivative)

    def inner(self, theta, X, train_type, derivative="exact"):
        """inner_sde_loss on one matrix: sum over outputs of train_type over samples (:283)"""
        r2 = self.residual(theta, X, derivative) ** 2
        return (r2.mean(1) if train_type == "mean" else r2.sum(1)).sum()

    def inner_batch(self, theta, inputs, train_type, derivative="exact"):
        """inner_sde_loss on a Vector of matrices (:338-341)"""
        return sum(self.inner(theta, X, train_type, derivative) for X in inputs) / len(inputs)

    def grid_loss(self, theta, inputs, batch, train_type, derivative="exact"):
        """generate_loss(::GridTraining / ::WeightedIntervalTraining / ::StochasticTraining) (:547-567)"""
        if batch:
            return self.inner_batch(theta, inputs, train_type, derivative)
        return sum(self.inner(theta, X, train_type, derivative) for X in inputs)

    def quadrature_loss(self, theta, nodes, weights, train_type, derivative="exact"):
        """Σ_q w_q abs2(inner_sde_loss(node q's (1 + n_z) x 1 matrix)) (:510-521)"""
        return sum(weights[q] * self.inner(theta, nodes[:, q:q + 1], train_type, derivative) ** 2
                   for q in range(nodes.shape[1]))

    def em_loss(self, theta, dataset):
        """generate_EM_L2loss (:452-484): Σ (ΔX - f Δt)^2 + Σ ((ΔX - f Δt)^2 - g^2 Δt)^2"""
        t = torch.tensor(np.asarray(dataset[1], dtype=np.float64))
        proc = torch.stack([torch.tensor(np.asarray(x, dtype=np.float64)) for x in dataset[0]], dim=1)   # (n+1, m)
        dt = (t[1:] - t[:-1])[:, None]
        dX = proc[1:] - proc[:-1]
        X, tt = proc[:-1], t[:-1][:, None].expand_as(proc[:-1])
        f = self._eval(self.f, X.reshape(1, -1), theta, tt.reshape(-1))[0].reshape(X.shape)
        g = self._eval(self.g, X.reshape(1, -1), theta, tt.reshape(-1))[0].reshape(X.shape)
        fx, gx = f * dt, g ** 2 * dt
        return ((dX - fx) ** 2).sum() + (((dX - fx) ** 2 - gx) ** 2).sum()


# ---- numpy replay of the device KKL sampler ------------------------------------------------------------------------
M32 = 0xFFFFFFFF


def philox4x32_10(c, k0, k1):
    c = [int(v) & M32 for v in c]
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        hi0, lo0, hi1, lo1 = p0 >> 32, p0 & M32, p1 >> 32, p1 & M32
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        k0, k1 = (k0 + 0x9E3779B9) & M32, (k1 + 0xBB67AE85) & M32
    return c


def u53(a, b):
    return float(((a << 32) | b) >> 11) * (1.0 / 9007199254740992.0)


def kkl_points(n_times, sub, n_z, t_lb, t_ub, seed, draw, strong):
    """the (1 + n_z, n_times * sub) points of draw `draw` (float64)"""
    key = (seed ^ 0xD6E8FEB86659FD93) & 0xFFFFFFFFFFFFFFFF
    k0, k1 = key & M32, key >> 32
    d0, d1 = draw & M32, (draw >> 32) & M32
    out = np.empty((1 + n_z, n_times * sub))
    zc = {}
    for i in range(n_times):
        c = philox4x32_10([i, M32, d0, d1], k0, k1)
        t = t_lb + (t_ub - t_lb) * u53(c[0], c[1])
        for s in range(sub):
            p = i * sub + s
            q = s if strong else p
            out[0, p] = t
            if q not in zc:
                z = np.empty(n_z)
                for j in range((n_z + 1) // 2):
                    w = philox4x32_10([q, j, d0, d1 ^ 0x4B4B4C00], k0, k1)
                    u1, u2 = 1.0 - u53(w[0], w[1]), u53(w[2], w[3])
                    r = math.sqrt(-2.0 * math.log(u1))
                    z[2 * j] = r * math.cos(6.283185307179586 * u2)
                    if 2 * j + 1 < n_z:
                        z[2 * j + 1] = r * math.sin(6.283185307179586 * u2)
                zc[q] = z
            out[1:, p] = zc[q]
    return out
