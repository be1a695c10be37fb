"""NNDAE: ``solve(DAEProblem(f, du0, u0, tspan, p; differential_vars), NNDAE(chain, opt))`` on the fused kernel
(reference src/dae_solve.jl).

The trial solution is NNODE's φ(t) = u0 + (t - t0) · N(t).  ``f(du, u, p, t)`` is traced once with sympy: u_k is φ_k,
du_k is dφ_k/dt (the exact d/dt tap of output k) for a differential component and 0 for an algebraic one.  The
reference's objective is the square of a mean, (1/n Σ_i Σ_k f_k(dφ(t_i), φ(t_i), p, t_i)²)² over the grid
tspan[1]:dt:tspan[2] (:64-82), so the per-point value v(t) = Σ_k f_k² is one functional term of the FFMA kernel with
g = (.)² and scale 1/n.  Every loss and gradient evaluation is one launch.  DESIGN section 4.16 maps the reference onto
the engine.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Sequence

import numpy as np
import sympy as sp

from .engine import Engine, REDUCE_SQUARE_OF_SUM
from .ode import (ComponentVector, ODEFunction, ODESolution, _Lowering, _TrialProblem, _TrialRepresentation, _check_mode,
                  _save_times, _theta0, _train)
from .strategies import _julia_range


# ---- problem and algorithm ------------------------------------------------------------------------------------
@dataclass
class DAEFunction(ODEFunction):
    """``DAEFunction(f; analytic)``: out-of-place residual ``f(du, u, p, t)``; ``analytic(du0, u0, p, t)`` the exact
    solution."""


@dataclass
class DAEProblem(_TrialProblem):
    """``DAEProblem(f, du0, u0, tspan, p; differential_vars)``: ``f(du, u, p, t)`` out-of-place, returning one residual
    per component of ``u0`` (a number or a vector); ``differential_vars[k]`` is true when f reads du_k as a derivative.
    ``du0`` is never read, as in the reference."""
    f: object
    du0: object
    u0: object
    tspan: Sequence[float]
    p: object = None
    differential_vars: object = field(default=None, kw_only=True)
    _solver = "NNDAE"
    _out_of_place = "The NNODE solver only supports out-of-place DAE definitions, i.e. du=f(u,p,t)."
    _inplace_args = 5          # f(out, du, u, p, t)

    def __post_init__(self):
        if not isinstance(self.f, ODEFunction):
            self.f = DAEFunction(self.f)
        super().__post_init__()
        n = 1 if self.scalar else len(np.ravel(self.u0))
        if self.differential_vars is None:
            raise ValueError("NNDAE: DAEProblem needs differential_vars, one Bool per component of u0 (true where f "
                             "reads du_k as a derivative)")
        dv = np.ravel(np.asarray(self.differential_vars, dtype=object))
        if dv.size != n:
            raise ValueError("NNDAE: differential_vars has %d entries, u0 has %d components" % (dv.size, n))
        self.differential_vars = [bool(v) for v in dv]

    def _analytic(self, t: float):
        return self.f.analytic(self.du0, self.u0, self.p, t)


class NNDAE:
    """``NNDAE(chain, opt, init_params; strategy, autodiff)`` (src/dae_solve.jl:32-46).  ``chain`` has one input and
    one output per component of u0.  ``opt``: ``Adam(...)`` (host loop, or the device loop with
    ``solve(...; device_loop=True)``), ``BFGS()`` or ``LBFGS()``.  Training runs on ``GridTraining(dt)`` only: as in
    the reference, ``strategy`` must be None and ``autodiff`` false.  Engine options: ``mode`` ("ffma" | "tc_f64"),
    ``device``, and ``seed`` for the initial parameters (the reference uses the global RNG)."""
    def __init__(self, chain, opt, init_params=None, *, strategy=None, autodiff=False, mode="ffma", device=0, seed=0):
        self.chain, self.opt, self.init_params = chain, opt, init_params
        self.strategy, self.autodiff = strategy, bool(autodiff)
        self.mode, self.device, self.seed = mode, device, seed
        _check_mode(mode, "NNDAE", "the tensor-core modes propagate 1-output networks and refuse functional terms")


class _DAELowering(_Lowering):
    def value(self, differential_vars) -> sp.Expr:
        """v = Σ_k f_k(du, φ, p, t)², du_k = dφ_k/dt for a differential component and 0 for an algebraic one"""
        du = [self.dphi(k) if differential_vars[k] else sp.Integer(0) for k in range(self.n)]
        fs = self._trace("f", [self.phi(k) for k in range(self.n)], du=du)
        return sp.Add(*[e ** 2 for e in fs])


# ---- the engine problem -----------------------------------------------------------------------------------------
class NNDAERepresentation(_TrialRepresentation):
    """The engine problem of one ``solve(prob, alg; dt)``: the one functional term (``term_names == ["loss"]``) over the
    grid tspan[1]:dt:tspan[2] and θ0 (network parameters only).  ``loss_grad(θ)`` is one evaluation; its total is the
    reference's objective."""

    def __init__(self, prob: DAEProblem, alg: NNDAE, dt=None):
        if not isinstance(alg, NNDAE):
            raise TypeError("solve(::DAEProblem, alg): alg must be an NNDAE")
        chain = alg.chain
        lw = _DAELowering(prob, False, ["t"])
        n = lw.n
        if chain.dims[0] != 1 or chain.dims[-1] != n:
            raise ValueError("NNDAE: the chain maps t to the %d components of u0: it needs 1 input and %d outputs, has "
                             "%d and %d" % (n, n, chain.dims[0], chain.dims[-1]))
        # src/dae_solve.jl:108-111, :79: alg.strategy leaves `strategy` nothing, which generate_loss does not take
        if alg.strategy is not None:
            raise ValueError("NNDAE: only GridTraining(dt) is supported: leave alg.strategy as None and pass dt to solve")
        if dt is None:
            raise ValueError("`dt` is not defined")
        if alg.autodiff:
            raise ValueError("autodiff not supported for GridTraining.")
        flat = _theta0(alg, chain, np.zeros(0), "NNDAE")
        super().__init__(prob, chain, None, lw, flat.dtype)
        t0, t1 = prob.tspan
        self.ts = _julia_range(t0, float(dt), t1)
        # (mean_i Σ_k f_k²)²: g = (.)² of 1/n Σ_i v(t_i), no point weights, term weight 1
        self.add(lw.term(lw.value(prob.differential_vars), ["t"], REDUCE_SQUARE_OF_SUM, 1.0 / self.ts.size), self.ts,
                 None, 1.0, "loss")
        self._close("NNDAE", 0, alg.mode, alg.device)
        self.alg = alg
        self.loss_const = 0.0
        self.flat_init_params = ComponentVector(flat, self.n_net)

    def _set_samplers(self, eng: Engine):
        pass


# ---- solution and solve -----------------------------------------------------------------------------------------
class DAESolution(ODESolution):
    """``t``, ``u`` (one value per time: a number for scalar u0, else an (n,) array), ``sol(t; idxs)`` through the
    trained network, ``k`` the optimization solution (``k.u``: θ as a ComponentVector with an empty ``.p``), ``resid``
    its objective, ``retcode``, ``errors`` with an analytic solution (src/dae_solve.jl:133-162)."""


def solve_nndae(prob: DAEProblem, alg: NNDAE, *, maxiters: int, dt=None, abstol: float = 1e-6, saveat=None,
                save_everystep: bool = True, verbose: bool = False, device_loop: bool = False,
                chunk: int = 50) -> DAESolution:
    """``solve(prob::DAEProblem, alg::NNDAE; maxiters, dt, abstol, saveat, save_everystep, verbose)``
    (src/dae_solve.jl:84-163).  Training stops as soon as a loss is below ``abstol`` (:118-128), as NNODE's loops do."""
    rep = NNDAERepresentation(prob, alg, dt=dt)
    res = _train(rep, alg.opt, int(maxiters), float(abstol), verbose, device_loop, chunk, who="NNDAE")
    return DAESolution(rep, res, _save_times(*prob.tspan, saveat, dt, save_everystep))
