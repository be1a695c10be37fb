"""NNODE: ``solve(ODEProblem(f, u0, tspan, p), NNODE(chain, opt; ...))`` on the fused kernel (reference
src/ode_solve.jl).

The trial solution is φ(t) = u0 + (t - t0) · N(t) for one network N with one output per component
(src/ode_solve.jl:186-197).  ``f(u, p, t)`` is traced once with sympy symbols; the residual of component k,
dφ_k/dt - f_k(φ, p, t) = N_k + (t - t0) ∂N_k/∂t - f_k(u0 + (t - t0) N, p, t), is lowered by the equation emitter of
lowering.py to value and d/dt taps of output k.  Every loss and gradient evaluation is one launch of the FFMA kernel.
DESIGN section 4.12 maps the reference's loss terms onto the engine's terms.

This module also holds the front end that NNODE, NNSDE (sde.py) and BNNODE (bpinn_ode.py) share: the problem checks
(``_TrialProblem``), the lowering of φ and its residuals (``_Lowering``), the term table and engine handle
(``_TrialRepresentation``), the value-only evaluator (``_Evaluator``), the strategy, mode and init_params checks, the
analytic errors and the optimizer loops (``_train``).
"""
from __future__ import annotations

import inspect
from dataclasses import dataclass
from typing import Callable, List, Optional, Sequence

import numpy as np
import sympy as sp

from . import engine as _eng
from .engine import Engine, NetSpec, ProblemSpec, TapSpec, TermSpec, REDUCE_MEAN, REDUCE_WSUM
from .lowering import LoweringError, _Emitter
from .pinn import BFGS, LBFGS, MODES, Adam, DataLoss, _linesearch_kind, _qn_run, initialparameters
from .strategies import (GridTraining, QuadratureTraining, QuasiRandomTraining, StochasticTraining,
                         WeightedIntervalTraining, _julia_range, gauss_legendre_box)
from .symbolic import VarInfo, expand_derivatives


# ---- problem and algorithm ------------------------------------------------------------------------------------
@dataclass
class ODEFunction:
    """``ODEFunction(f; analytic)``: out-of-place ``f(u, p, t)``; ``analytic(u0, p, t)`` the exact solution."""
    f: Callable
    analytic: Optional[Callable] = None


class _TrialProblem:
    """What ODEProblem, SDEProblem and DAEProblem share: the checks of their fields, ``scalar``, and the name and
    out-of-place message of the solver that traces their functions of (u, p, t) (DAEProblem: (du, u, p, t))"""
    _solver = "NNODE"
    _out_of_place = "The NNODE solver only supports out-of-place ODE definitions, i.e. du=f(u,p,t)."
    _components_note = ""      # appended to the component-count refusal
    _traced = ("f",)           # the functions of (u, p, t) the solver traces
    _inplace_args = 4          # the argument count of an in-place function: f(du, u, p, t)

    def __post_init__(self):
        if not isinstance(self.f, ODEFunction):
            self.f = ODEFunction(self.f)
        if _has_complex(self.u0) or _has_complex(self.p):
            raise ValueError("%s: complex u0 or p are not supported (the engine trains real networks)" % self._solver)
        for name in self._traced:
            try:
                n_args = len(inspect.signature(self._function(name)).parameters)
            except (TypeError, ValueError):
                n_args = self._inplace_args - 1
            if n_args == self._inplace_args:
                raise ValueError(self._out_of_place)
        self.tspan = (float(self.tspan[0]), float(self.tspan[1]))

    def _function(self, name: str) -> Callable:
        return self.f.f if name == "f" else getattr(self, name)

    @property
    def scalar(self) -> bool:
        return np.ndim(self.u0) == 0

    def _analytic(self, t: float):
        return self.f.analytic(self.u0, self.p, t)


@dataclass
class ODEProblem(_TrialProblem):
    """``ODEProblem(f, u0, tspan, p)``: ``u0`` a number or a vector, ``f(u, p, t)`` out-of-place."""
    f: object
    u0: object
    tspan: Sequence[float]
    p: object = None


def _has_complex(p) -> bool:
    return p is not None and any(isinstance(v, complex) or np.iscomplexobj(v) for v in np.ravel(np.asarray(p, dtype=object)))


def _check_mode(mode: str, who: str, why: str):
    """The ODE family runs on the FFMA kernel (``ffma``, or ``tc_f64`` for Float64); `why` says why the others cannot"""
    if mode not in MODES:
        raise ValueError("unknown mode %r (one of %s)" % (mode, sorted(MODES)))
    if mode not in ("ffma", "tc_f64"):
        raise ValueError("%s runs on the FFMA kernel: mode=\"ffma\" (or \"tc_f64\" for Float64); %s" % (who, why))


class NNODE:
    """``NNODE(chain, opt, init_params; strategy, autodiff, batch, param_estim, additional_loss, dataset,
    estim_collocate)`` (src/ode_solve.jl:143-153).  ``chain`` has one input and one output per component of u0.
    ``opt``: ``Adam(...)`` (host loop, or the device loop with ``solve(...; device_loop=True)``), ``BFGS()`` or
    ``LBFGS()``.  ``additional_loss``: a ``DataLoss`` whose ``depvar`` is a component index (0-based), the structured
    form of the reference's closure.  ``dataset = [x̂_1, ..., x̂_n, t, W]``.  Engine options: ``mode`` ("ffma" |
    "tc_f64"), ``device``, and ``seed`` for the initial parameters (the reference uses the global RNG)."""
    def __init__(self, chain, opt, init_params=None, *, strategy=None, autodiff=False, batch=True, param_estim=False,
                 additional_loss=None, dataset=(), estim_collocate=False, mode="ffma", device=0, seed=0):
        self.chain, self.opt, self.init_params = chain, opt, init_params
        self.strategy, self.autodiff, self.batch = strategy, bool(autodiff), bool(batch)
        self.param_estim, self.additional_loss = bool(param_estim), additional_loss
        self.dataset, self.estim_collocate = list(dataset), bool(estim_collocate)
        self.mode, self.device, self.seed = mode, device, seed
        _check_mode(mode, "NNODE", "the tensor-core modes propagate 1-output networks, NNODE's network has one output "
                                   "per component")
        if additional_loss is not None and not isinstance(additional_loss, DataLoss):
            raise ValueError("NNODE: additional_loss must be a DataLoss(depvar=k, points=t, values=u_k) with a component "
                             "index k in place of the depvar name (the structured form of the reference's "
                             "additional_loss(phi, θ) closure); arbitrary closures cannot run inside the CUDA kernel")


class ComponentVector(np.ndarray):
    """θ as the reference's ``ComponentArray(; depvar, p)``: the flat vector, with ``.depvar`` (network parameters)
    and ``.p`` (the ODE parameters under ``param_estim``; empty otherwise)."""

    def __new__(cls, flat, n_net: int):
        obj = np.asarray(flat).view(cls)
        obj.n_net = n_net
        return obj

    def __array_finalize__(self, obj):
        self.n_net = getattr(obj, "n_net", None)

    @property
    def depvar(self) -> np.ndarray:
        return np.asarray(self)[:self.n_net]

    @property
    def p(self) -> np.ndarray:
        return np.asarray(self)[self.n_net:]


@dataclass
class OptimizationSolution:
    """``sol.k``: the optimizer's result; ``u`` is θ (a ComponentVector)."""
    u: ComponentVector
    objective: float
    iterations: int
    retcode: str


# ---- the trial solution and its residuals -----------------------------------------------------------------------
T_SYM = sp.Symbol("t", real=True)


def _p_symbols(p):
    """θ.p symbols shaped like the problem's p (a number or a vector)"""
    if np.ndim(p) == 0:
        return sp.Symbol("p1", real=True), ["p1"]
    names = ["p%d" % (i + 1) for i in range(len(np.ravel(p)))]
    return [sp.Symbol(nm, real=True) for nm in names], names


class _Lowering:
    """The trial solution φ_k = u0_k + (t - t0) N_k of one network N whose inputs are the point rows `rows` (["t"] for
    NNODE and BNNODE, ["t", "z1", ...] for NNSDE): the symbols of N's outputs, the θ.p symbols under `param_estim`,
    the residuals of the problem's f and the TermSpec of an expression in them"""

    def __init__(self, prob: _TrialProblem, param_estim: bool, rows: List[str]):
        self.prob, self.rows = prob, list(rows)
        self.n = 1 if prob.scalar else len(np.ravel(prob.u0))
        self.u0 = np.ravel(np.asarray(prob.u0, dtype=np.float64))
        self.t0 = prob.tspan[0]
        self.N = [sp.Function("N%d" % (k + 1))(*[sp.Symbol(r, real=True) for r in self.rows]) for k in range(self.n)]
        names = ["N%d" % (k + 1) for k in range(self.n)]
        self.vi = VarInfo(depvars=names, indvars=list(self.rows), dict_indvars={r: i for i, r in enumerate(self.rows)},
                          dict_depvars={nm: k for k, nm in enumerate(names)},
                          dict_depvar_input={nm: list(self.rows) for nm in names})
        if param_estim:
            if prob.p is None:
                raise ValueError("%s: param_estim starts θ.p at the problem's p, and the problem has none" % prob._solver)
            self.p_arg, pnames = _p_symbols(prob.p)
            self.param_index = {nm: i for i, nm in enumerate(pnames)}
        else:
            self.p_arg, self.param_index = prob.p, {}

    def _trace(self, name: str, comps: List[sp.Expr], du: Optional[List[sp.Expr]] = None) -> List[sp.Expr]:
        """the problem's function `name` (f or g) of (u, p, t) at u = comps, with symbols: one expression per
        component.  With `du`, f is a DAE residual f(du, u, p, t), and du and u are lists even for a scalar u0."""
        who = self.prob._solver
        try:
            fn = self.prob._function(name)
            if du is not None:
                out = fn(list(du), list(comps), self.p_arg, T_SYM)
            else:
                out = fn(comps[0] if self.prob.scalar else list(comps), self.p_arg, T_SYM)
        except Exception as ex:      # noqa: BLE001 -- any failure to trace is the user's function, reported with its message
            args = "u, p" if du is None else "du, u, p"
            raise ValueError("%s: %s(%s, t) could not be traced with symbolic %s and t (write it with sympy functions "
                             "such as sympy.cos): %s: %s" % (who, name, args, args, type(ex).__name__, ex)) from ex
        if out is None:
            raise ValueError(self.prob._out_of_place)
        outs = list(np.ravel(np.asarray(out, dtype=object)))      # a number, or a sequence of one for a scalar u0
        if len(outs) != self.n:
            raise ValueError("%s: %s returns %d components, u0 has %d%s"
                             % (who, name, len(outs), self.n, self.prob._components_note))
        exprs = [sp.sympify(e) for e in outs]
        for e in exprs:
            if e.has(sp.I) or any(a.is_real is False for a in e.atoms(sp.Number)):
                raise ValueError("%s: %s is complex-valued; the engine trains real networks" % (who, name))
        return exprs

    def phi(self, k: int) -> sp.Expr:
        return self.u0[k] + (T_SYM - self.t0) * self.N[k]

    def dphi(self, k: int) -> sp.Expr:
        return self.N[k] + (T_SYM - self.t0) * sp.Derivative(self.N[k], T_SYM)

    def residuals(self) -> List[sp.Expr]:
        """r_k = dφ_k/dt - f_k(φ, p, t)"""
        fs = self._trace("f", [self.phi(k) for k in range(self.n)])
        return [self.dphi(k) - fs[k] for k in range(self.n)]

    def collocation_residuals(self) -> List[sp.Expr]:
        """dφ_k/dt - f_k(û, θ.p, t), û read from point rows 1..n (the observations)"""
        fs = self._trace("f", [sp.Symbol("uhat%d" % (j + 1), real=True) for j in range(self.n)])
        return [self.dphi(k) - fs[k] for k in range(self.n)]

    def term(self, expr: sp.Expr, rows: List[str], reduction: int, scale: float = 1.0) -> TermSpec:
        """TermSpec of the residual expr over point rows `rows`; taps of N_k become taps of output k of network 0, whose
        inputs are the lowering's rows.  A residual without taps is a parameter-only term, which the engine accepts
        only if it reads θ.p (NNSDE's Euler-Maruyama loss).  NNODE's and BNNODE's residuals always have taps: f sees φ
        or û but never ∂N/∂t, so it cannot cancel the (t - t0) ∂N_k/∂t of dφ_k/dt, nor the N_k of φ_k - x̂."""
        em = _Emitter(self.vi, rows, self.param_index, {})
        try:
            v = em.emit(expand_derivatives(expr))
        except LoweringError as ex:
            raise ValueError("%s: %s" % (self.prob._solver, ex)) from ex
        em.prog.append(("sub", v, em.const(0.0), 0.0))       # the last instruction is the residual
        taps = [TapSpec(net=0, order=tp.order, dirs=tp.dirs, out=tp.net) for tp in em.taps]
        return TermSpec(dim=len(rows), taps=taps, prog=em.prog,
                        net_rows=[[rows.index(r) for r in self.rows]] if taps else None, reduction=reduction,
                        scale=scale)


class _Evaluator:
    """A value-only engine of one network: the value-only terms `terms` (one per quantity, all over the same point
    rows) evaluated at the columns of the point matrix given to ``at``, for one θ per call"""

    def __init__(self, terms: List[TermSpec], chain, n_params: int, dtype, device: int):
        self.n_rows, self.dtype = terms[0].dim, np.dtype(dtype)
        self.engine = Engine(ProblemSpec(nets=[NetSpec(chain.dims, chain.acts, 0)], terms=terms, n_params=n_params,
                                         param_offset=chain.n_params, n_theta=chain.n_params + n_params,
                                         dtype=self.dtype.name, mode=_eng.MODE_FFMA, device=device))
        self.m = 0

    def at(self, X):
        """evaluate at the columns of X, (rows, m) or, with one row, any shape of m values"""
        X = np.asarray(X, dtype=np.float64).reshape(self.n_rows, -1).astype(self.dtype)
        for k in range(len(self.engine.spec.terms)):
            self.engine.set_points_host(k, X)
        self.m = X.shape[1]

    def __call__(self, theta) -> np.ndarray:
        """(len(terms), m) values at θ"""
        th = np.asarray(theta, dtype=self.dtype)
        out = np.empty((len(self.engine.spec.terms), self.m))
        for k in range(out.shape[0]):
            out[k] = self.engine.term_residual_host(k, th, self.m)
        return out


# ---- the engine problem -----------------------------------------------------------------------------------------
def _strategy(alg, dt):
    """NNODE's and NNSDE's training strategy (src/ode_solve.jl:439-451): alg.strategy, by default GridTraining(dt)
    with a dt and QuadratureTraining without, and its refusals"""
    strategy = alg.strategy
    if strategy is None:
        strategy = GridTraining(dt) if dt is not None else QuadratureTraining()
    if isinstance(strategy, QuasiRandomTraining):
        raise ValueError("QuasiRandomTraining is not supported by NNODE since it's for high dimensional spaces only. "
                         "Use StochasticTraining instead.")
    if alg.autodiff:
        for cls in (GridTraining, StochasticTraining, WeightedIntervalTraining):
            if isinstance(strategy, cls):
                raise ValueError("autodiff not supported for %s." % cls.__name__)
    if not isinstance(strategy, (GridTraining, StochasticTraining, WeightedIntervalTraining, QuadratureTraining)):
        raise TypeError("unsupported training strategy %r" % (strategy,))
    return strategy


def _init_array(init_params, mode: str, who: str) -> np.ndarray:
    """init_params as a float32 or float64 array (other real dtypes become float64), as PhysicsInformedNN takes them;
    complex parameters, and float32 ones under tc_f64, are refused"""
    init = np.asarray(init_params)
    if np.iscomplexobj(init):
        raise ValueError("%s: complex parameters are not supported (the engine trains real networks)" % who)
    if init.dtype not in (np.float32, np.float64):
        init = init.astype(np.float64)
    if mode == "tc_f64" and init.dtype != np.float64:
        raise ValueError("mode=\"tc_f64\" runs the layer products on the FP64 tensor cores and needs float64 "
                         "parameters (init_params is %s); use mode=\"ffma\" for float32" % init.dtype.name)
    return init


def _theta0(alg, chain, p0: np.ndarray, who: str) -> np.ndarray:
    """NNODE's and NNSDE's θ0 = [depvar, p] (ComponentArray(; depvar, p), src/ode_solve.jl:431-435): θ.p starts at
    p0 unless init_params gives it"""
    n_net = chain.n_params
    if alg.init_params is None:
        return np.concatenate([initialparameters(np.random.default_rng(alg.seed), chain, np.float64), p0])
    init = _init_array(alg.init_params, alg.mode, who)
    if init.shape == (n_net,):
        init = np.concatenate([init, p0.astype(init.dtype)])
    if init.shape != (n_net + p0.size,):
        raise ValueError("init_params has length %d, the chain%s needs %d"
                         % (init.size, " + p" if p0.size else "", n_net + p0.size))
    return init


class _TrialRepresentation:
    """What the engine problems of NNODE, NNSDE and BNNODE share: the term table (``specs``, ``point_sets``,
    ``quad_weights``, ``term_weights``, ``term_names``) that ``add`` fills and ``_close`` turns into the ProblemSpec;
    the engine handle, created at first use with every fixed point set uploaded and the sampled terms' device
    samplers registered by the subclass's ``_set_samplers``; ``loss_grad`` and ``trial``."""

    def __init__(self, prob: _TrialProblem, chain, strategy, lowering: _Lowering, dtype):
        self.prob, self.chain, self.strategy, self.lowering, self.dtype = prob, chain, strategy, lowering, dtype
        self.n, self.n_net = lowering.n, chain.n_params
        self.specs: List[TermSpec] = []
        self.point_sets: List[Optional[np.ndarray]] = []
        self.quad_weights: List[Optional[np.ndarray]] = []
        self.term_weights: List[float] = []      # an array once closed
        self.term_names: List[str] = []
        self.sampled: list = []
        self._engine, self._calls, self._phi = None, 0, None

    def add(self, spec: TermSpec, pts, w, weight: float, name: str):
        self.specs.append(spec)
        self.point_sets.append(None if pts is None else np.asarray(pts, dtype=np.float64).reshape(spec.dim, -1))
        self.quad_weights.append(None if w is None else np.asarray(w, dtype=np.float64))
        self.term_weights.append(float(weight))
        self.term_names.append(name)

    def _close(self, who: str, n_params: int, mode: str, device: int, what: str = "loss terms"):
        if len(self.specs) > _eng.MAX_TERMS:
            raise ValueError("%s: %d %s (max %d)" % (who, len(self.specs), what, _eng.MAX_TERMS))
        self.term_weights = np.asarray(self.term_weights)
        self.spec = ProblemSpec(nets=[NetSpec(self.chain.dims, self.chain.acts, 0)], terms=self.specs,
                                n_params=n_params, param_offset=self.n_net, n_theta=self.n_net + n_params,
                                dtype=self.dtype.name, mode=MODES[mode], device=device)

    @property
    def engine(self) -> Engine:
        """The engine handle, created at first use with every fixed point set uploaded and the sampled terms' device
        samplers registered"""
        if self._engine is None:
            eng = Engine(self.spec)
            for i, (X, w) in enumerate(zip(self.point_sets, self.quad_weights)):
                if X is not None:
                    eng.set_points_host(i, X.astype(self.dtype), None if w is None else w.astype(self.dtype))
            self._set_samplers(eng)
            self._engine = eng
        return self._engine

    def loss_grad(self, theta, want_grad: bool = True):
        """(total of the engine's terms, term losses, gradient or None) at θ: one fused launch (a fresh sample of the
        sampled terms each call after the first, as the reference draws one per loss call)"""
        if self.sampled and self._calls > 0:
            self.engine.resample()
        self._calls += 1
        return self.engine.loss_grad_host(np.asarray(theta, dtype=self.dtype), self.term_weights, want_grad)

    def trial(self, theta, X) -> np.ndarray:
        """φ at the columns of the (rows, m) inputs X (NNODE: any shape of m times), (n, m), evaluated on the device"""
        if self._phi is None:
            lw = self.lowering
            self._phi = _Evaluator([lw.term(lw.phi(k), lw.rows, REDUCE_MEAN) for k in range(self.n)], self.chain,
                                   self.spec.n_params, self.dtype, self.spec.device)
        self._phi.at(X)
        return self._phi(theta)


class NNODERepresentation(_TrialRepresentation):
    """The engine problem of one ``solve(prob, alg)``: terms (``term_names``), their weights, point sets and θ0.
    ``loss_grad(θ)`` is one evaluation (a fresh stochastic sample each call, as the reference draws one per loss call)."""

    def __init__(self, prob: ODEProblem, alg: NNODE, dt=None, tstops=None):
        if not isinstance(alg, NNODE):
            raise TypeError("solve(::ODEProblem, alg): alg must be an NNODE")
        chain = alg.chain
        lw = _Lowering(prob, alg.param_estim, ["t"])
        n = lw.n
        t0, t1 = prob.tspan
        if chain.dims[0] != 1 or chain.dims[-1] != n:
            raise ValueError("NNODE: the chain maps t to the %d components of u0: it needs 1 input and %d outputs, has "
                             "%d and %d" % (n, n, chain.dims[0], chain.dims[-1]))
        strategy = _strategy(alg, dt)

        # dataset (src/ode_solve.jl:455-464)
        ds = alg.dataset
        if ds and (len(ds) < 3 or not all(np.ndim(v) == 1 and np.size(v) > 0 and not np.iscomplexobj(v)
                                          and np.issubdtype(np.asarray(v).dtype, np.floating) for v in ds)):
            raise ValueError("Invalid dataset. The dataset would be a timeseries (x̂,t,W) with type: "
                             "Vector{Vector{AbstractFloat}")
        if not ds and alg.param_estim and alg.additional_loss is None:
            raise ValueError("Dataset or an additional loss is required for Inverse problems performing Parameter "
                             "Estimation.")
        if not ds and alg.estim_collocate:
            raise ValueError("Dataset is required for Inverse problems performing Parameter Estimation using the Data "
                             "Quadrature loss function.")
        if ds and len(ds) - 2 != n:
            raise ValueError("Invalid dataset: %d observation vectors for %d components (dataset = [x̂_1, ..., x̂_n, t, W])"
                             % (len(ds) - 2, n))

        p0 = np.ravel(np.asarray(prob.p, dtype=np.float64)) if alg.param_estim else np.zeros(0)
        flat = _theta0(alg, chain, p0, "NNODE")
        super().__init__(prob, chain, strategy, lw, flat.dtype)
        add = self.add
        res = lw.residuals()
        if isinstance(strategy, QuadratureTraining):
            # ∫ abs2(inner_loss(t)) dt with inner_loss(t) = Σ_k r_k(t)^2 (:250): one term with residual Σ_k r_k^2
            X, w, _ = gauss_legendre_box((np.array([t0]), np.array([t1])), int(strategy.nodes_per_dim), np.float64)
            s = sp.Add(*[r ** 2 for r in res])
            add(lw.term(s, ["t"], REDUCE_WSUM, 1.0), X, w, 1.0, "quadrature")
            n_orig = None
        else:
            if isinstance(strategy, GridTraining):
                ts = _julia_range(t0, float(strategy.dx), t1)
                n_orig = ts.size
            elif isinstance(strategy, WeightedIntervalTraining):
                ts, n_orig = strategy.sample(t0, t1), int(strategy.points)
            else:
                ts, n_orig = None, int(strategy.points)
            for k in range(n):
                if ts is None:     # fresh uniform points in [t0, t1] at every evaluation (:283-294), drawn on the device
                    self.sampled.append(len(self.specs))
                    add(lw.term(res[k], ["t"], REDUCE_MEAN), None, None, 1.0 if alg.batch else n_orig, "residual_%d" % (k + 1))
                else:
                    add(lw.term(res[k], ["t"], REDUCE_WSUM, 1.0 / ts.size if alg.batch else 1.0), ts, np.ones(ts.size),
                        1.0, "residual_%d" % (k + 1))
        if alg.param_estim and ds:
            t_d = np.asarray(ds[-2], dtype=np.float64)
            for k in range(n):      # generate_L2lossData (:338-346): Σ_t (φ_k(t) - x̂_k(t))^2
                xk = sp.Symbol("xhat", real=True)
                add(lw.term(lw.phi(k) - xk, ["t", "xhat"], REDUCE_WSUM, 1.0),
                    np.stack([t_d, np.asarray(ds[k], dtype=np.float64)]), np.ones(t_d.size), 1.0, "l2_data_%d" % (k + 1))
            if alg.estim_collocate:     # generate_L2loss2 (:352-380): Σ_t W_t (dφ_k/dt - f_k(û, θ.p, t))^2
                rows = ["t"] + ["uhat%d" % (j + 1) for j in range(n)]
                pts = np.stack([t_d] + [np.asarray(ds[j], dtype=np.float64) for j in range(n)])
                W = np.asarray(ds[-1], dtype=np.float64)
                for k, r in enumerate(lw.collocation_residuals()):
                    add(lw.term(r, rows, REDUCE_WSUM, 1.0), pts, W, 1.0, "collocation_%d" % (k + 1))
        dl = alg.additional_loss
        if dl is not None:
            k = dl.depvar
            if not isinstance(k, (int, np.integer)) or not 0 <= k < n:
                raise ValueError("NNODE: DataLoss.depvar must be a component index in [0, %d), got %r" % (n, k))
            y = np.ravel(np.asarray(dl.values, dtype=np.float64))
            td = np.ravel(np.asarray(dl.points, dtype=np.float64))
            if td.shape != y.shape:
                raise ValueError("DataLoss: points must be (1, n) or (n,) times and values (n,)")
            yk = sp.Symbol("y", real=True)
            add(lw.term(lw.phi(k) - yk, ["t", "y"], REDUCE_MEAN), np.stack([td, y]), None, 1.0, "additional")
        if tstops is not None:
            tt = np.ravel(np.asarray(tstops, dtype=np.float64))
            if n_orig is not None:     # (L N + L_t N_t) / (N + N_t) (:482-499); Quadrature: L + L_t
                self.term_weights = [w_ * n_orig / (n_orig + tt.size) for w_ in self.term_weights]
            wt = 1.0 if n_orig is None else tt.size / (n_orig + tt.size)
            for k in range(n):
                add(lw.term(res[k], ["t"], REDUCE_WSUM, 1.0 / tt.size if alg.batch else 1.0), tt, np.ones(tt.size),
                    wt, "tstops_%d" % (k + 1))
        self._close("NNODE", p0.size, alg.mode, alg.device)
        self.alg = alg
        self.loss_const = 0.0      # added to every reported loss (NNSDE's constant Euler-Maruyama terms)
        self.flat_init_params = ComponentVector(flat, self.n_net)

    def _set_samplers(self, eng: Engine):
        t0, t1 = self.prob.tspan
        for i in self.sampled:
            eng.set_sampler(i, int(self.strategy.points), [t0], [t1], int(self.strategy.seed))


def _analytic_errors(prob: _TrialProblem, ts: np.ndarray, U: np.ndarray) -> dict:
    """SciMLBase's timeseries errors of the (n, len(ts)) values U against prob.f.analytic (``analytic(u0, p, t)``;
    DAEProblem: ``analytic(du0, u0, p, t)``): the final, maximum and root-mean-square errors; empty without an analytic
    solution"""
    an = prob.f.analytic
    if an is None:
        return {}
    A = np.stack([np.ravel(np.asarray(prob._analytic(float(ti)), dtype=np.float64)) for ti in ts], axis=1)
    E = U - A
    return {"final": float(np.mean(np.abs(E[:, -1]))), "l∞": float(np.max(np.abs(E))),
            "l2": float(np.sqrt(np.mean(E ** 2)))}


# ---- solution ---------------------------------------------------------------------------------------------------
class ODESolution:
    """``t``, ``u`` (one value per time: a number for scalar u0, else an (n,) array), ``sol(t; idxs)`` through the
    trained network (NNODEInterpolation, :382-398), ``k`` the optimization solution, ``errors`` with an analytic
    solution (SciMLBase's timeseries errors: "final", "l∞", "l2")."""

    def __init__(self, rep: NNODERepresentation, res: OptimizationSolution, ts: np.ndarray):
        self.prob, self.alg, self.k, self.original = rep.prob, rep.alg, res, res
        self.retcode, self.resid = "Success", res.objective
        self._rep = rep
        self.t = np.asarray(ts, dtype=np.float64)
        U = rep.trial(res.u, self.t)
        self.u = [float(U[0, i]) for i in range(self.t.size)] if rep.prob.scalar else [U[:, i].copy() for i in range(self.t.size)]
        self.errors = _analytic_errors(rep.prob, self.t, U)

    def __call__(self, t, idxs=None):
        """φ(t): for a number t a number (scalar u0 or an integer idxs) or a vector; for an array of times one column
        per time"""
        U = self._rep.trial(self.k.u, t)
        if idxs is not None:
            U = U[idxs]
        elif self.prob.scalar:
            U = U[0]
        if np.ndim(t) == 0:
            U = U[..., 0]
        return float(U) if np.ndim(U) == 0 else U


def _save_times(t0, t1, saveat, dt, save_everystep) -> np.ndarray:
    """:521-532"""
    if saveat is not None and np.ndim(saveat) == 0:
        return _julia_range(t0, float(saveat), t1)
    if saveat is not None:
        return np.asarray(saveat, dtype=np.float64)
    if dt is not None:
        return _julia_range(t0, float(dt), t1)
    if save_everystep:
        return np.linspace(t0, t1, 100)
    return np.array([t0, t1])


# ---- solve ------------------------------------------------------------------------------------------------------
def solve_nnode(prob: ODEProblem, alg: NNODE, *, maxiters: int, dt=None, abstol: float = 1e-6, saveat=None,
                save_everystep: bool = True, tstops=None, verbose: bool = False, device_loop: bool = False,
                chunk: int = 50) -> ODESolution:
    """``solve(prob::ODEProblem, alg::NNODE; maxiters, dt, abstol, saveat, save_everystep, tstops, verbose)``
    (src/ode_solve.jl:403-552).  Training stops as soon as a loss is below ``abstol`` (:507-516): the host Adam loop
    checks every iteration before its update; ``device_loop=True`` checks every ``chunk`` iterations; BFGS / LBFGS check
    after every accepted iteration."""
    rep = NNODERepresentation(prob, alg, dt=dt, tstops=tstops)
    res = _train(rep, alg.opt, int(maxiters), float(abstol), verbose, device_loop, chunk)
    return ODESolution(rep, res, _save_times(*prob.tspan, saveat, dt, save_everystep))


def _train(rep: NNODERepresentation, opt, maxiters: int, abstol: float, verbose: bool, device_loop: bool,
           chunk: int, who: str = "NNODE") -> OptimizationSolution:
    """the optimizer loops of NNODE and NNSDE; every reported loss is the engine's total plus rep.loss_const"""
    c = rep.loss_const

    def log(it, l):
        if verbose:
            print("[%s]\tIter: [%*d/%d]\tLoss: %g" % (who, len(str(maxiters)), it, maxiters, l))

    def stop(state, l):
        log(state["iter"], l + c)
        return l + c < abstol

    eng, w = rep.engine, rep.term_weights
    if isinstance(opt, (BFGS, LBFGS)):
        th, f, iters, _, retcode = _qn_run(eng, rep.flat_init_params, opt, _linesearch_kind(opt.linesearch), maxiters,
                                           stop, w)
        return OptimizationSolution(ComponentVector(th, rep.n_net), f + c, iters, retcode)
    if not isinstance(opt, Adam):
        raise TypeError("%s: opt must be Adam(...), BFGS() or LBFGS(), got %r" % (who, opt))
    if device_loop:
        eng.adam_begin(rep.flat_init_params, opt.lr, opt.beta1, opt.beta2, opt.eps)
        done, obj = 0, float("nan")
        while done < maxiters:
            n = min(chunk, maxiters - done)
            obj, _ = eng.adam_iterate(n, w)
            done += n
            if stop({"iter": done}, obj):
                break
        return OptimizationSolution(ComponentVector(eng.adam_theta(), rep.n_net), obj + c, done, "Success")
    u = np.asarray(rep.flat_init_params, dtype=np.float64).copy()
    m, v = np.zeros_like(u), np.zeros_like(u)
    obj, it = float("nan"), 0
    for it in range(1, maxiters + 1):
        obj, _, g = rep.loss_grad(u)
        if stop({"iter": it}, obj):
            break
        g = g.astype(np.float64)
        m = opt.beta1 * m + (1 - opt.beta1) * g
        v = opt.beta2 * v + (1 - opt.beta2) * g * g
        u -= opt.lr * (m / (1 - opt.beta1 ** it)) / (np.sqrt(v / (1 - opt.beta2 ** it)) + opt.eps)
    return OptimizationSolution(ComponentVector(u.astype(rep.dtype), rep.n_net), obj + c, it, "Success")
