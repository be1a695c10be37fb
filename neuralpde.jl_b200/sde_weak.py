"""SDEPINN: ``solve(SDEProblem(f, g, u0, tspan, p), SDEPINN(chain = ..., x_0, x_end, ...))`` on the fused kernel
(reference src/NN_SDE_weaksolve.jl:121-272).

The network p̂(X, T) is the density of the scalar process.  It is trained as an ordinary PhysicsInformedNN problem
under GridTraining([dx, dt]) on the Fokker-Planck equation of the SDE, Dt(p̂) ~ -Dx(f p̂) + ½ Dxx(g² p̂), with f and g
traced once with sympy on the X, T symbols, plus three boundary conditions: the initial density at the single point
(u0, t0), and a zero probability flux J(x, T) = f p̂ - ½ (g² Dx(p̂) + p̂ Dx(g²)) at x_0 and x_end.  The reference forms
J by calling a Julia function on the number x_b, so g(x_b, p, T)² is a number before Dx reaches it and that part
expands to 0; the flux terms keep the same quirk (DESIGN section 4.15).  The norm loss
λ_norm Σ_t (∫_{x_0}^{x_end} p̂(x, t) dx - 1)² over the Nt + 1 grid times is one weighted-sum term whose program reads
one integral (64 Gauss-Legendre nodes over row X).
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import sympy as sp

from .ode import _check_mode
from .pinn import (BFGS, LBFGS, Adam, NonAdaptiveLoss, Normal, PhysicsInformedNN, _ResidualSumLoss, discretize,
                   solve)
from .strategies import GridTraining, _julia_range
from .symbolic import ClosedInterval, Differential, Eq, In, Integral, PDESystem

X_SYM, T_SYM = sp.Symbol("X", real=True), sp.Symbol("T", real=True)
P_HAT = sp.Function("p")


class SDEPINN:
    """``SDEPINN(; chain, x_0, x_end, optimalg, norm_loss_alg, initial_parameters, Nt = 20, dx = 0.05, σ_var_bc,
    λ_ic, λ_norm = 1, distrib = Normal(0.5, 0.01), strategy, autodiff, batch, param_estim, dataset, additional_loss)``
    (src/NN_SDE_weaksolve.jl:44-119).  ``chain`` maps (x, t) to the density.  ``optimalg``: ``BFGS()`` / ``LBFGS()``
    (device quasi-Newton) or ``Adam(...)`` (host loop).  ``distrib`` is a ``Normal`` or ``LogNormal``; the
    initial condition is its pdf at u0.  As in the reference, ``norm_loss_alg``, ``σ_var_bc``, ``λ_ic``,
    ``strategy``, ``autodiff``, ``batch``, ``param_estim``, ``dataset`` and ``additional_loss`` are accepted and not
    used; the norm integral is a fixed 64-node Gauss-Legendre rule.  Engine options: ``mode`` ("ffma" | "tc_f64"),
    ``device``."""

    def __init__(self, *, chain, x_0, x_end, optimalg=None, norm_loss_alg=None, initial_parameters=None, Nt=20,
                 dx=0.05, σ_var_bc=0.05, λ_ic=1.0, λ_norm=1.0, distrib=Normal(0.5, 0.01), strategy=None,
                 autodiff=True, batch=False, param_estim=False, dataset=None, additional_loss=None, mode="ffma",
                 device=0, **kwargs):
        _check_mode(mode, "SDEPINN", "the tensor-core modes refuse integral terms and logcosh layers")
        if optimalg is None:
            raise ValueError("SDEPINN: optimalg is required (BFGS(), LBFGS() or Adam(...))")
        if not isinstance(optimalg, (Adam, BFGS, LBFGS)):
            raise TypeError("SDEPINN: optimalg must be Adam(...), BFGS() or LBFGS(), got %r" % (optimalg,))
        if not hasattr(distrib, "pdf"):
            raise TypeError("SDEPINN: distrib must be a Normal or a LogNormal, got %r" % (distrib,))
        if not x_0 < x_end:
            raise ValueError("SDEPINN: need x_0 < x_end, got [%s, %s]" % (x_0, x_end))
        if int(Nt) < 1 or not dx > 0:
            raise ValueError("SDEPINN: need Nt >= 1 and dx > 0, got Nt = %s, dx = %s" % (Nt, dx))
        self.chain, self.optimalg, self.norm_loss_alg = chain, optimalg, norm_loss_alg
        self.initial_parameters = initial_parameters
        self.x_0, self.x_end, self.Nt, self.dx = float(x_0), float(x_end), int(Nt), float(dx)
        self.σ_var_bc, self.λ_ic, self.λ_norm, self.distrib = σ_var_bc, λ_ic, float(λ_norm), distrib
        self.strategy, self.autodiff, self.batch = strategy, autodiff, batch
        self.param_estim, self.dataset, self.additional_loss = param_estim, dataset, additional_loss
        self.mode, self.device, self.kwargs = mode, device, kwargs


# ---- the PDE system -----------------------------------------------------------------------------------------------
def _traced(fn, x, p, t) -> sp.Expr:
    return sp.sympify(fn(x, p, t))


def flux(prob, x_b: float) -> sp.Expr:
    """J(x_b, T) = f p̂ - ½ (g² Dx(p̂) + p̂ Dx(g²)) with f and g evaluated at the number x_b (:160-164); Dx(g²) of that
    number is 0.  p̂ keeps the X slot, which the point set fixes at x_b."""
    fb, gb = _traced(prob.f.f, sp.Float(x_b), prob.p, T_SYM), _traced(prob.g, sp.Float(x_b), prob.p, T_SYM)
    Dx = Differential(X_SYM)
    p = P_HAT(X_SYM, T_SYM)
    return fb * p - sp.Rational(1, 2) * (gb ** 2 * Dx(p) + p * Dx(gb ** 2))


def fokker_planck(prob) -> tuple:
    """(lhs, rhs) of Dt(p̂) ~ -Dx(f p̂) + ½ Dxx(g² p̂) (:173-174)"""
    Dx, Dxx, Dt = Differential(X_SYM), Differential(X_SYM) ** 2, Differential(T_SYM)
    p = P_HAT(X_SYM, T_SYM)
    f, g = _traced(prob.f.f, X_SYM, prob.p, T_SYM), _traced(prob.g, X_SYM, prob.p, T_SYM)
    return Dt(p), -Dx(f * p) + sp.Rational(1, 2) * Dxx(g ** 2 * p)


class SDEPINNProblem:
    """The PhysicsInformedNN problem of one ``solve(prob, alg)``: ``pde_system``, ``discretization`` (its
    ``additional_loss`` is the norm term), the flux boundaries it keeps (``flux_at``: a flux that vanishes identically
    is a zero loss and has no term) and the grid times ``ts``.  ``discretize()`` builds the engine problem."""

    def __init__(self, prob, alg: SDEPINN):
        if not isinstance(alg, SDEPINN):
            raise TypeError("solve(::SDEProblem, alg): alg must be an SDEPINN")
        if not prob.scalar:
            raise ValueError("SDEPINN: u0 must be a number: the Fokker-Planck PDE has one space variable X (the "
                             "reference's vector-u0 branch is a TODO, src/NN_SDE_weaksolve.jl:214)")
        t0, t1 = prob.tspan
        dt = (t1 - t0) / alg.Nt
        u0 = float(prob.u0)
        self.ts = _julia_range(t0, dt, t1)
        lhs, rhs = fokker_planck(prob)
        ic = Eq(P_HAT(sp.Float(u0), sp.Float(t0)) - alg.distrib.pdf(u0), 0)
        bcs, self.flux_at = [ic], []
        for x_b in (alg.x_0, alg.x_end):
            J = flux(prob, x_b)
            if J != 0:
                bcs.append(Eq(J, 0))
                self.flux_at.append(x_b)
        domains = [In(X_SYM, alg.x_0, alg.x_end), In(T_SYM, t0, t1)]
        self.pde_system = PDESystem([Eq(lhs, rhs)], bcs, domains, [X_SYM, T_SYM], [P_HAT(X_SYM, T_SYM)])
        Ix = Integral(X_SYM, ClosedInterval(alg.x_0, alg.x_end))
        norm = _ResidualSumLoss(Eq(Ix(P_HAT(X_SYM, T_SYM)), 1), np.vstack([np.full(self.ts.size, alg.x_0), self.ts]))
        init = alg.initial_parameters
        self.discretization = PhysicsInformedNN(
            alg.chain, GridTraining([alg.dx, dt]), init_params=None if init is None else np.asarray(init),
            additional_loss=norm, adaptive_loss=NonAdaptiveLoss(additional_loss_weights=alg.λ_norm),
            mode=alg.mode, device=alg.device)

    def flux_points(self, x_b: float) -> np.ndarray:
        """(x_b, t_i) for the grid times: GridTraining's points of J(x_b, T) ~ 0"""
        return np.vstack([np.full(self.ts.size, x_b), self.ts])

    def discretize(self):
        """the OptimizationProblem; its representation's terms are pde_1, bc_1 (the initial density), the flux terms
        and the norm term ("additional")"""
        opt_prob = discretize(self.pde_system, self.discretization)
        for j, x_b in enumerate(self.flux_at):        # the flux terms' points lie on the line X = x_b
            opt_prob.representation.set_points(2 + j, self.flux_points(x_b))
        return opt_prob


def solve_sdepinn(prob, alg: SDEPINN, *, maxiters: int = 200, verbose: bool = False, dt=None, abtol=None,
                  reltol=None, saveat=None, tstops=None):
    """``solve(prob::SDEProblem, alg::SDEPINN; maxiters = 200, verbose)`` (:121-272): ``(res, phi)``, ``res.u`` the
    trained θ and ``phi([x, t], θ)`` the density at (x, t), evaluated on the device.  ``dt``, ``abtol``, ``reltol``,
    ``saveat`` and ``tstops`` are accepted and not used, as in the reference."""
    opt_prob = SDEPINNProblem(prob, alg).discretize()
    rep = opt_prob.representation
    callback: Optional[object] = None
    if verbose:
        lf = rep.loss_functions

        def callback(state, loss):
            th = state["u"]
            print("loss = ", loss)
            if th is not None:
                print("pde = ", [f(th) for f in lf.pde_loss_functions])
                print("bc  = ", [f(th) for f in lf.bc_loss_functions])
            return False
    res = solve(opt_prob, alg.optimalg, maxiters=int(maxiters), callback=callback)
    return res, rep.phi
