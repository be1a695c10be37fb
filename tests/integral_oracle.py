"""Float64 restatement of the reference's integral terms (get_numeric_integral, src/discretize.jl:334-397, with the
infinite-bound substitution of src/transform_inf_integral.jl), on top of the loss oracle in oracle/reference.py.

``IntegralProblem(..., quad="gauss")`` evaluates every integral with the engine's fixed Gauss-Legendre rule (the same
node table, the same substitution), so loss and gradient (torch autograd) are what the engine computes up to rounding.
``quad="adaptive"`` integrates each point's integrand with scipy's adaptive ``quad`` / ``dblquad`` at the reference's
tolerances (reltol = abstol = 1e-3): it stands in for ``CubatureJLh`` when the fixed rule is pinned to the reference.

The reference writes the node into ``cord_ = cord; cord_[integrating_var_id] .= x`` (:355-358).  ``cord`` there is
``cord[:, i]``, a fresh copy of one point made by the slice in the loop over points (:389-393), so the aliasing only
ever touches that copy: the owner's residual, and the other points, keep their own coordinates.  Every integrand call
overwrites all integrating rows before it reads them, so the copy's previous contents never leak into a value either.
Bounds that are functions of the coordinates are evaluated at the owner point (``lb_[i, :] = l(cord, ...)``), before
any node is written; the restatement follows that, also for the second bound of ``[0,1] x [0,x]``.
"""
from __future__ import annotations

import itertools
from typing import Callable, Dict, Optional

import numpy as np
import sympy as sp
import torch
from scipy import integrate

from oracle import reference as R
from neuralpde_jl_b200.symbolic import IntegralOp

EPS = 1.0 / 20          # transform_inf_integral.jl: ϵ = 1 / 20
REL_TOL = ABS_TOL = 1e-3


def substitution(lo, hi):
    """(t bounds, x(t), dx/dt) of one integrating variable with bounds lo, hi (sympy), as transform_inf_integral.jl
    builds them: v_inf, v_semiinf and get_inf_transformation_jacobian."""
    lo, hi = sp.sympify(lo), sp.sympify(hi)
    if lo == -sp.oo and hi == sp.oo:
        return (-1 + EPS, 1 - EPS), (lambda t: t / (1 - t ** 2)), (lambda t: (1 + t ** 2) / (1 - t ** 2) ** 2)
    if hi == sp.oo:
        if lo.is_number:
            a = float(lo)
            return (0.0, 1 - EPS), (lambda t: a + t / (1 - t)), (lambda t: 1 / (1 - t) ** 2)
        return (lo / (1 + lo), 1 - EPS), (lambda t: t / (1 - t)), (lambda t: 1 / (1 - t) ** 2)
    if lo == -sp.oo:
        b = float(hi)
        return (-1 + EPS, 0.0), (lambda t: b + t / (1 + t)), (lambda t: 1 / (1 + t) ** 2)
    return (lo, hi), (lambda t: t), None


class IntegralProblem(R.Problem):
    """``R.Problem`` whose generated residual also evaluates ``Integral`` terms.  ``closures``: depvar name -> a
    function of the (d, N) coordinates that replaces that variable's network (forward__integral.jl's chains are
    closures, not MLPs)."""

    def __init__(self, *args, quad: str = "gauss", q: int = 16, closures: Optional[Dict[str, Callable]] = None, **kw):
        kw.setdefault("derivative", "exact")
        super().__init__(*args, **kw)
        self.quad, self.q = quad, q
        self.closures = closures or {}

    def _u(self, k, theta):
        nm = self.names[k]
        if nm in self.closures:
            return self.closures[nm]
        return super()._u(k, theta)

    def _eval(self, e, env, cords, theta):
        if isinstance(e, IntegralOp):
            return self._integral(e, env, theta)
        return super()._eval(e, env, cords, theta)

    def _at(self, integrand, env, theta):
        """the integrand at the coordinates env (each (1, N))"""
        cords = {nm: torch.cat([env[v] for v in self.inputs[nm]], dim=0)
                 for nm in self.names if all(v in env for v in self.inputs[nm])}
        return self._eval(integrand, env, cords, theta)

    def _integral(self, e, env, theta):
        integrand, vs, lbs, ubs = e.args
        integrand = self._expand(integrand)
        names = [str(v) for v in vs]
        n = next(iter(env.values())).shape[1]
        subs = [substitution(lo, hi) for lo, hi in zip(lbs, ubs)]
        # bounds in t, per owner point (evaluated at the owner's coordinates)
        bnds = []
        for (lo_t, hi_t), _, _ in subs:
            bnds.append([self._eval(sp.sympify(b), env, {}, theta).expand(1, n) for b in (lo_t, hi_t)])
        if self.quad == "gauss":
            xi, wq = np.polynomial.legendre.leggauss(self.q)
            total = 0
            for js in itertools.product(range(self.q), repeat=len(names)):
                env2, w = dict(env), 1
                for k, (j, v) in enumerate(zip(js, names)):
                    lo, hi = bnds[k]
                    h = 0.5 * (hi - lo)
                    t = lo + h * (1 + float(xi[j]))
                    _, xmap, jac = subs[k]
                    env2[v] = xmap(t)
                    w = w * h * float(wq[j]) * (jac(t) if jac is not None else 1)
                total = total + w * self._at(integrand, env2, theta).expand(1, n)
            return total
        # adaptive: one scipy integration per owner point (value only)
        out = np.empty(n)
        for p in range(n):
            env_p = {k_: v_[:, p:p + 1].detach() for k_, v_ in env.items()}

            def g(*ts):
                env2, w = dict(env_p), 1.0
                for k, (t, v) in enumerate(zip(ts, names)):
                    _, xmap, jac = subs[k]
                    tt = torch.tensor([[float(t)]])
                    env2[v] = xmap(tt)
                    w *= float(jac(tt)) if jac is not None else 1.0
                with torch.no_grad():
                    return w * float(self._at(integrand, env2, theta).reshape(-1)[0])

            lims = [(float(bnds[k][0][0, p]), float(bnds[k][1][0, p])) for k in range(len(names))]
            if len(names) == 1:
                out[p] = integrate.quad(g, *lims[0], epsabs=ABS_TOL, epsrel=REL_TOL)[0]
            else:                     # dblquad integrates func(y, x): x = first variable (outer), y = second (inner)
                out[p] = integrate.dblquad(lambda y, x: g(x, y), lims[0][0], lims[0][1], lims[1][0], lims[1][1],
                                           epsabs=ABS_TOL, epsrel=REL_TOL)[0]
        return torch.tensor(out).reshape(1, n)
