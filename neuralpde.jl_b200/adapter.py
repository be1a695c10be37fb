"""Neural adapters: fit a new network to already trained ones (reference src/neural_adapter.jl).

``neural_adapter(loss, init_params, pde_system, strategy)`` builds the problem ``mean(abs2, loss(cord, θ))`` over the
strategy's points, where the reference's ``loss(cord, θ) = chain2(cord, θ) .- phi(cord, res.u)`` is a Julia closure.  A
closure cannot run inside a CUDA kernel, so the loss takes a structured form here, as ``DataLoss`` does for
``additional_loss``: ``NeuralAdapterLoss(chain2, target)`` means ``chain2(cord, θ) - target(cord)``, with ``target`` an
expression of the system's independent variables and registered network functions (``register_symbolic``).  The
teachers run inside the fused kernel as fixed networks, so device-sampled point sets need no precomputed values.
"""
from __future__ import annotations

import dataclasses
from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np
import sympy as sp

from . import engine as _eng
from .engine import Engine, NetSpec, ProblemSpec, TermSpec, REDUCE_MEAN, REDUCE_WSUM
from .lowering import LoweringError, _Emitter
from .pinn import (Chain, NonAdaptiveLoss, OptimizationFunction, OptimizationProblem, _fixed_specs, _upload_fixed)
from .strategies import (GridTraining, QuadratureTraining, QuasiRandomTraining, StochasticTraining, adapter_training_set,
                         gauss_legendre_box, get_bounds_)
from .symbolic import FixedNet, PDESystem, VarInfo, expand_derivatives, get_vars


@dataclass
class NeuralAdapterLoss:
    """``loss(cord, θ) = chain(cord, θ) .- target(cord)``: the student ``chain`` (its inputs are the rows of ``cord``
    in order) minus ``target``, an expression of the system's independent variables and registered network
    functions, e.g. ``phi_teacher(x, y)``."""
    chain: Chain
    target: object


@dataclass
class AdapterRepresentation:
    """What ``solve`` reads from a neural adapter problem: one term per system, fixed loss weights."""
    engine: Engine
    strategy: object
    eqs: list                                   # the losses, one per term
    rows: List[list]                            # per term: the point rows (variable names, or numbers)
    fixed: List[FixedNet]
    point_sets: List[Optional[np.ndarray]]
    bcs: list = field(default_factory=list)
    adaloss: NonAdaptiveLoss = field(default_factory=NonAdaptiveLoss)
    additional_loss: object = None
    iteration: list = field(default_factory=lambda: [0])
    weights: dict = None

    def resample(self):
        pass


def _adapter_term(loss: NeuralAdapterLoss, rows: list, defaults: dict, fixed: List[FixedNet]) -> TermSpec:
    """The residual chain(cord) - target(cord) over point rows ``rows``: the student is network 0 (its inputs are the
    rows in order), the target's registered functions are fixed networks 1, 2, ..."""
    names = [r if isinstance(r, str) else "__row%d" % i for i, r in enumerate(rows)]
    c = loss.chain
    if c.dims[0] != len(names):
        raise ValueError("NeuralAdapterLoss: the chain has %d inputs, the training points have %d rows %s"
                         % (c.dims[0], len(names), rows))
    if c.dims[-1] != 1:
        raise ValueError("NeuralAdapterLoss: the chain must have a 1-dimensional output")
    vi = VarInfo(["__student"], names, {n: i for i, n in enumerate(names)}, {"__student": 0}, {"__student": names})
    em = _Emitter(vi, names, {}, defaults, fixed=fixed)
    try:
        a = em.emit(sp.Function("__student")(*[sp.Symbol(n, real=True) for n in names]))
        b = em.emit(expand_derivatives(sp.sympify(loss.target)))
    except LoweringError as ex:
        raise ValueError(str(ex)) from ex
    em.prog.append(("sub", a, b, 0.0))
    return TermSpec(dim=len(names), taps=em.taps, prog=em.prog, net_rows=[list(range(len(names)))] + em.fixed_net_rows(),
                    reduction=REDUCE_MEAN)


def neural_adapter(loss, init_params, pde_system, strategy, device: int = 0, seed: Optional[int] = None
                   ) -> OptimizationProblem:
    """``neural_adapter(loss, init_params, pde_system, strategy)`` and the list form
    ``neural_adapter(losses, init_params, pde_systems, strategy)`` (one term per system, summed), as in
    src/neural_adapter.jl.  Training sets: Grid uses the adapter's own product grid over the domains (:1-6);
    Stochastic and QuasiRandom draw ``points`` per evaluation on the device inside the bounds of the first equation's
    arguments (:8-23); Quadrature uses the engine's fixed Gauss-Legendre box on those bounds.  Returns an
    ``OptimizationProblem`` over the student's θ only."""
    single = not isinstance(loss, (list, tuple))
    losses = [loss] if single else list(loss)
    systems = [pde_system] if single else list(pde_system)
    if len(losses) != len(systems):
        raise ValueError("neural_adapter: %d losses for %d systems" % (len(losses), len(systems)))
    for l in losses:
        if not isinstance(l, NeuralAdapterLoss):
            raise TypeError("neural_adapter: `loss` must be a NeuralAdapterLoss(chain, target) -- chain(cord, θ) minus a "
                            "target expression of registered network functions; a Python callable cannot run inside "
                            "the CUDA kernel (got %r)" % type(l).__name__)
    chain = losses[0].chain
    if any(l.chain.dims != chain.dims or l.chain.acts != chain.acts for l in losses):
        raise ValueError("neural_adapter: every loss must train the same chain")
    if not isinstance(systems[0], PDESystem):
        raise TypeError("neural_adapter: expected a PDESystem")
    theta0 = np.asarray(init_params)
    if theta0.dtype not in (np.float32, np.float64):
        theta0 = theta0.astype(np.float64)
    if theta0.shape != (chain.n_params,):
        raise ValueError("init_params has length %d, the chain needs %d" % (theta0.size, chain.n_params))
    dtype = theta0.dtype
    sampled = isinstance(strategy, (StochasticTraining, QuasiRandomTraining))
    if isinstance(strategy, QuasiRandomTraining) and not strategy.resampling:
        raise ValueError("neural_adapter: QuasiRandomTraining(resampling=false) minibatches are not supported; the "
                         "device draws a fresh Latin hypercube sample per evaluation (resampling=true)")
    if not isinstance(strategy, (GridTraining, QuadratureTraining, StochasticTraining, QuasiRandomTraining)):
        raise TypeError("unsupported training strategy %r" % (strategy,))

    fixed: List[FixedNet] = []
    specs, rows_all, sets, quad_w, boxes = [], [], [], [], []
    for l, sys_ in zip(losses, systems):
        vi = get_vars(sys_.ivs, sys_.dvs)
        defaults = {str(k): float(v) for k, v in sys_.defaults.items()}
        if isinstance(strategy, GridTraining):
            rows = [str(d.variables) for d in sys_.domain]
            pts, w, box = adapter_training_set(sys_.domain, strategy.dx, dtype.type), None, None
        else:
            rows, lb, ub = get_bounds_(sys_.domain, sys_.eqs, dtype.type, vi)
            box = (lb, ub)
            pts, w = None, None
        tm = _adapter_term(l, rows, defaults, fixed)
        if isinstance(strategy, QuadratureTraining):
            pts, w, area = gauss_legendre_box(box, strategy.nodes_per_dim, dtype.type)
            tm.reduction, tm.scale = REDUCE_WSUM, 1.0 / area
        specs.append(tm)
        rows_all.append(rows)
        sets.append(pts)
        quad_w.append(w)
        boxes.append(box)
    if not fixed:
        raise ValueError("neural_adapter: the targets apply no registered network function: there is nothing to adapt to")

    spec = ProblemSpec(nets=[NetSpec(chain.dims, chain.acts, 0)], terms=specs, n_theta=chain.n_params,
                       dtype=dtype.name, mode=_eng.MODE_FFMA, device=device, fixed=_fixed_specs(fixed))
    eng = Engine(spec)
    _upload_fixed(eng, fixed)
    for i, (pts, w) in enumerate(zip(sets, quad_w)):
        if pts is not None:
            eng.set_points_host(i, pts, w)
    if sampled:
        kind = "lhs" if isinstance(strategy, QuasiRandomTraining) else "uniform"
        s0 = strategy.seed if seed is None else seed
        for i, (lb, ub) in enumerate(boxes):
            eng.set_sampler(i, strategy.points, np.asarray(lb, np.float64), np.asarray(ub, np.float64), s0, kind=kind)
        strategy = dataclasses.replace(strategy, device_sampler=True)   # the points live on the device
    n = len(specs)
    rep = AdapterRepresentation(engine=eng, strategy=strategy, eqs=losses, rows=rows_all, fixed=fixed, point_sets=sets,
                                weights={"pde": np.ones(n), "bc": np.zeros(0), "add": np.ones(1)})
    state = {"calls": 0}

    def _evaluate(theta, want_grad: bool):
        if sampled and state["calls"] > 0:
            eng.resample()                   # a fresh sample per evaluation, as the reference draws per loss call
        state["calls"] += 1
        rep.iteration[0] += 1
        return eng.loss_grad_host(np.asarray(theta, dtype=dtype), None, want_grad)

    def f(theta, p=None) -> float:
        return _evaluate(theta, False)[0]

    def grad(theta, p=None):
        total, _, g = _evaluate(theta, True)
        return total, g

    return OptimizationProblem(OptimizationFunction(f, grad), theta0.copy(), None, rep)
