"""Float64 restatement of fixed (registered) networks for the tests: oracle.reference's Problem, extended so that an
application of a registered network function -- and a Differential of one -- evaluates the trained network with its
parameters held constant (derivatives by nested autograd), and the neural adapter's loss
mean(abs2, chain(cord, θ) - target(cord)) over a point matrix."""
import numpy as np
import sympy as sp
import torch

from neuralpde_jl_b200.symbolic import fixed_net_of
from oracle import reference as R


def fixed_forward(fn, X: torch.Tensor, dirs=()) -> torch.Tensor:
    """value (dirs = ()) or partial derivative along input positions ``dirs`` of fixed network fn at X (d, N); its
    parameters are a constant tensor, so no gradient reaches them"""
    p = torch.tensor(np.asarray(fn.params, dtype=np.float64))
    if not dirs:
        return R.phi(X, p, fn.dims, fn.acts)
    xg = X.detach().clone().requires_grad_(True)
    v = R.phi(xg, p, fn.dims, fn.acts)
    for d in dirs:
        (g,) = torch.autograd.grad(v.sum(), xg, create_graph=True)
        v = g[d:d + 1, :]
    return v


def _fixed_app(e):
    """(application, derivative variables) when e is a registered function or a derivative of one, else None"""
    dv, inner = [], e
    while isinstance(inner, sp.Derivative):
        for v, n in inner.variable_count:
            dv += [str(v)] * int(n)
        inner = inner.expr
    return (inner, dv) if fixed_net_of(inner) is not None else None


class FixedProblem(R.Problem):
    """oracle.reference.Problem with registered network functions"""

    def _eval(self, e, env, cords, theta):
        hit = _fixed_app(e)
        if hit is None:
            return super()._eval(e, env, cords, theta)
        app, dv = hit
        n = max(v.shape[1] for v in env.values())
        cols = [env[str(a)].expand(1, n) if isinstance(a, sp.Symbol) else torch.full((1, n), float(a), dtype=torch.float64)
                for a in app.args]
        dirs = [next(i for i, a in enumerate(app.args) if isinstance(a, sp.Symbol) and str(a) == v) for v in dv]
        return fixed_forward(fixed_net_of(app), torch.cat(cols, dim=0), dirs)


def adapter_loss_and_grad(chain, theta_np, terms):
    """Σ_k mean(abs2, chain(cord_k, θ) - target_k(cord_k)) (Σ_k scale_k Σ w r² for weighted terms) and its θ-gradient.
    terms: list of (row names, target expression, (d, N) points, weights or None, scale)."""
    theta = torch.tensor(np.asarray(theta_np, dtype=np.float64), requires_grad=True)
    prob = FixedProblem.__new__(FixedProblem)
    prob.param_names, prob.defaults = [], {}
    losses = []
    for names, target, pts, w, scale in terms:
        X = torch.as_tensor(np.asarray(pts, dtype=np.float64))
        env = {n: X[i:i + 1, :] for i, n in enumerate(names) if isinstance(n, str)}
        r = R.phi(X, theta, chain.dims, chain.acts) - prob._eval(sp.sympify(target), env, {}, theta)
        losses.append(torch.mean(r * r) if w is None else scale * torch.sum(torch.as_tensor(w) * r[0] ** 2))
    total = sum(losses)
    (g,) = torch.autograd.grad(total, theta)
    return float(total.detach()), np.array([float(l.detach()) for l in losses]), g.numpy().copy()
