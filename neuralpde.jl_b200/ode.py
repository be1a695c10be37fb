"""NNODE: ``solve(ODEProblem(f, u0, tspan, p), NNODE(chain, opt; ...))`` on the fused kernel (reference
src/ode_solve.jl).

The trial solution is φ(t) = u0 + (t - t0) · N(t) for one network N with one output per component
(src/ode_solve.jl:186-197).  ``f(u, p, t)`` is traced once with sympy symbols; the residual of component k,
dφ_k/dt - f_k(φ, p, t) = N_k + (t - t0) ∂N_k/∂t - f_k(u0 + (t - t0) N, p, t), is lowered by the equation emitter of
lowering.py to value and d/dt taps of output k.  Every loss and gradient evaluation is one launch of the FFMA kernel.
DESIGN section 4.12 maps the reference's loss terms onto the engine's terms.
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

# the modes that run the FFMA kernel; the tensor-core modes propagate 1-output networks only
_NNODE_MODES = ("ffma", "tc_f64")


# ---- problem and algorithm ------------------------------------------------------------------------------------
@dataclass
class ODEFunction:
    """``ODEFunction(f; analytic)``: out-of-place ``f(u, p, t)``; ``analytic(u0, p, t)`` the exact solution."""
    f: Callable
    analytic: Optional[Callable] = None


@dataclass
class ODEProblem:
    """``ODEProblem(f, u0, tspan, p)``: ``u0`` a number or a vector, ``f(u, p, t)`` out-of-place."""
    f: object
    u0: object
    tspan: Sequence[float]
    p: object = None

    def __post_init__(self):
        if not isinstance(self.f, ODEFunction):
            self.f = ODEFunction(self.f)
        if _has_complex(self.u0) or _has_complex(self.p):
            raise ValueError("NNODE: complex u0 or p are not supported (the engine trains real networks)")
        f = self.f.f
        try:
            n_args = len(inspect.signature(f).parameters)
        except (TypeError, ValueError):
            n_args = 3
        if n_args == 4:
            raise ValueError("The NNODE solver only supports out-of-place ODE definitions, i.e. du=f(u,p,t).")
        self.tspan = (float(self.tspan[0]), float(self.tspan[1]))

    @property
    def scalar(self) -> bool:
        return np.ndim(self.u0) == 0


def _has_complex(p) -> bool:
    return p is not None and any(isinstance(v, complex) or np.iscomplexobj(v) for v in np.ravel(np.asarray(p, dtype=object)))


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
        if mode not in MODES:
            raise ValueError("unknown mode %r (one of %s)" % (mode, sorted(MODES)))
        if mode not in _NNODE_MODES:
            raise ValueError("NNODE runs on the FFMA kernel: mode=\"ffma\" (or \"tc_f64\" for Float64); the tensor-core "
                             "modes propagate 1-output networks, NNODE's network has one output per component")
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


# ---- tracing f --------------------------------------------------------------------------------------------------
T_SYM = sp.Symbol("t", real=True)


def _trace(prob: ODEProblem, u_syms, p_arg) -> List[sp.Expr]:
    """f(u, p, t) with symbols, as a list of one expression per component"""
    try:
        out = prob.f.f(u_syms, p_arg, T_SYM)
    except Exception as ex:      # noqa: BLE001 -- any failure to trace is the user's f, reported with its message
        raise ValueError("NNODE: f(u, p, t) could not be traced with symbolic u, p and t (write it with sympy "
                         "functions such as sympy.cos): %s: %s" % (type(ex).__name__, ex)) from ex
    if out is None:
        raise ValueError("The NNODE solver only supports out-of-place ODE definitions, i.e. du=f(u,p,t).")
    n = 1 if prob.scalar else len(np.ravel(prob.u0))
    outs = list(np.ravel(np.asarray(out, dtype=object)))      # a number, or a sequence of one for a scalar u0
    if len(outs) != n:
        raise ValueError("NNODE: f returns %d components, u0 has %d" % (len(outs), n))
    exprs = [sp.sympify(e) for e in outs]
    for e in exprs:
        if e.has(sp.I) or any(a.is_real is False for a in e.atoms(sp.Number)):
            raise ValueError("NNODE: f is complex-valued; the engine trains real networks")
    return exprs


def _p_symbols(p):
    """θ.p symbols shaped like the problem's p (a number or a vector)"""
    if p is None:
        raise ValueError("NNODE: param_estim starts θ.p at the problem's p, and the problem has none")
    if np.ndim(p) == 0:
        return sp.Symbol("p1", real=True), ["p1"]
    names = ["p%d" % (i + 1) for i in range(len(np.ravel(p)))]
    return [sp.Symbol(nm, real=True) for nm in names], names


class _Lowering:
    """The symbols of the network outputs N_k(t) and the rows / parameters the emitter reads."""

    def __init__(self, prob: ODEProblem, alg: NNODE):
        self.prob = prob
        self.n = 1 if prob.scalar else len(np.ravel(prob.u0))
        self.u0 = np.ravel(np.asarray(prob.u0, dtype=np.float64))
        self.t0 = prob.tspan[0]
        self.N = [sp.Function("N%d" % (k + 1))(T_SYM) for k in range(self.n)]
        names = ["N%d" % (k + 1) for k in range(self.n)]
        self.vi = VarInfo(depvars=names, indvars=["t"], dict_indvars={"t": 0},
                          dict_depvars={nm: k for k, nm in enumerate(names)}, dict_depvar_input={nm: ["t"] for nm in names})
        if alg.param_estim:
            self.p_arg, pnames = _p_symbols(prob.p)
            self.param_index = {nm: i for i, nm in enumerate(pnames)}
        else:
            self.p_arg, self.param_index = prob.p, {}

    def phi(self, k: int) -> sp.Expr:
        return self.u0[k] + (T_SYM - self.t0) * self.N[k]

    def dphi(self, k: int) -> sp.Expr:
        return self.N[k] + (T_SYM - self.t0) * sp.Derivative(self.N[k], T_SYM)

    def u_arg(self, comps: List[sp.Expr]):
        return comps[0] if self.prob.scalar else list(comps)

    def residuals(self) -> List[sp.Expr]:
        """r_k = dφ_k/dt - f_k(φ, p, t)"""
        fs = _trace(self.prob, self.u_arg([self.phi(k) for k in range(self.n)]), self.p_arg)
        return [self.dphi(k) - fs[k] for k in range(self.n)]

    def collocation_residuals(self) -> List[sp.Expr]:
        """dφ_k/dt - f_k(û, θ.p, t), û read from point rows 1..n (the observations)"""
        uh = [sp.Symbol("uhat%d" % (j + 1), real=True) for j in range(self.n)]
        fs = _trace(self.prob, self.u_arg(uh), self.p_arg)
        return [self.dphi(k) - fs[k] for k in range(self.n)]

    def term(self, expr: sp.Expr, rows: List[str], reduction: int, scale: float = 1.0) -> TermSpec:
        """TermSpec of the residual expr over point rows `rows`; taps of N_k become taps of output k of network 0"""
        em = _Emitter(self.vi, rows, self.param_index, {})
        try:
            v = em.emit(expand_derivatives(expr))
        except LoweringError as ex:
            raise ValueError("NNODE: %s" % ex) from ex
        em.prog.append(("sub", v, em.const(0.0), 0.0))       # the last instruction is the residual
        taps = [TapSpec(net=0, order=tp.order, dirs=tp.dirs, out=tp.net) for tp in em.taps]
        if not taps:
            raise ValueError("NNODE: the residual %s reads no network output" % expr)
        return TermSpec(dim=len(rows), taps=taps, prog=em.prog, net_rows=[[rows.index("t")]], reduction=reduction,
                        scale=scale)


# ---- the engine problem -----------------------------------------------------------------------------------------
class NNODERepresentation:
    """The engine problem of one ``solve(prob, alg)``: terms (``term_names``), their weights, point sets and θ0.
    ``loss_grad(θ)`` is one evaluation (a fresh stochastic sample each call, as the reference draws one per loss call)."""

    def __init__(self, prob: ODEProblem, alg: NNODE, dt=None, tstops=None):
        if not isinstance(alg, NNODE):
            raise TypeError("solve(::ODEProblem, alg): alg must be an NNODE")
        chain = alg.chain
        lw = _Lowering(prob, alg)
        n = lw.n
        t0, t1 = prob.tspan
        if chain.dims[0] != 1 or chain.dims[-1] != n:
            raise ValueError("NNODE: the chain maps t to the %d components of u0: it needs 1 input and %d outputs, has "
                             "%d and %d" % (n, n, chain.dims[0], chain.dims[-1]))

        # strategy (src/ode_solve.jl:439-451) and its refusals
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

        # θ = [depvar, p] (ComponentArray(; depvar, p), :431-435); dtype as PhysicsInformedNN
        n_net = chain.n_params
        p0 = np.ravel(np.asarray(prob.p, dtype=np.float64)) if alg.param_estim else np.zeros(0)
        if alg.init_params is None:
            flat = np.concatenate([initialparameters(np.random.default_rng(alg.seed), chain, np.float64), p0])
        else:
            init = np.asarray(alg.init_params)
            if np.iscomplexobj(init):
                raise ValueError("NNODE: complex parameters are not supported (the engine trains real networks)")
            if init.dtype not in (np.float32, np.float64):
                init = init.astype(np.float64)
            if init.shape == (n_net,):
                init = np.concatenate([init, p0.astype(init.dtype)])
            if init.shape != (n_net + p0.size,):
                raise ValueError("init_params has length %d, the chain%s needs %d"
                                 % (init.size, " + p" if p0.size else "", n_net + p0.size))
            flat = init
        dtype = flat.dtype
        if alg.mode == "tc_f64" and dtype != np.float64:
            raise ValueError("mode=\"tc_f64\" runs the layer products on the FP64 tensor cores and needs float64 "
                             "parameters (init_params is %s); use mode=\"ffma\" for float32" % dtype.name)

        # terms, point sets, weights, names
        specs: List[TermSpec] = []
        sets: List[Optional[np.ndarray]] = []
        qw: List[Optional[np.ndarray]] = []
        weights: List[float] = []
        names: List[str] = []
        res = lw.residuals()

        def add(spec, pts, w, weight, name):
            specs.append(spec)
            sets.append(None if pts is None else np.asarray(pts, dtype=np.float64).reshape(spec.dim, -1))
            qw.append(w)
            weights.append(float(weight))
            names.append(name)

        sampled: List[int] = []      # StochasticTraining's terms
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
                    sampled.append(len(specs))
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
                weights = [w_ * n_orig / (n_orig + tt.size) for w_ in weights]
            wt = 1.0 if n_orig is None else tt.size / (n_orig + tt.size)
            for k in range(n):
                add(lw.term(res[k], ["t"], REDUCE_WSUM, 1.0 / tt.size if alg.batch else 1.0), tt, np.ones(tt.size),
                    wt, "tstops_%d" % (k + 1))
        if len(specs) > _eng.MAX_TERMS:
            raise ValueError("NNODE: %d loss terms (max %d)" % (len(specs), _eng.MAX_TERMS))

        self.spec = ProblemSpec(nets=[NetSpec(chain.dims, chain.acts, 0)], terms=specs, n_params=p0.size,
                                param_offset=n_net, n_theta=n_net + p0.size, dtype=dtype.name, mode=MODES[alg.mode],
                                device=alg.device)
        self.prob, self.alg, self.strategy, self.lowering = prob, alg, strategy, lw
        self.n, self.n_net, self.dtype = n, n_net, dtype
        self.specs, self.point_sets, self.quad_weights = specs, sets, qw
        self.term_weights = np.asarray(weights)
        self.term_names = names
        self.sampled = sampled
        self.loss_const = 0.0      # added to every reported loss (NNSDE's constant Euler-Maruyama terms)
        self.flat_init_params = ComponentVector(flat, n_net)
        self._engine = None
        self._calls = 0

    @property
    def engine(self) -> Engine:
        """The engine handle, created at first use with every fixed point set uploaded and the stochastic terms'
        device samplers registered"""
        if self._engine is None:
            eng = Engine(self.spec)
            for i, (X, w) in enumerate(zip(self.point_sets, self.quad_weights)):
                if X is not None:
                    eng.set_points_host(i, X.astype(self.dtype), None if w is None else w.astype(self.dtype))
            t0, t1 = self.prob.tspan
            for i in self.sampled:
                eng.set_sampler(i, int(self.strategy.points), [t0], [t1], int(self.strategy.seed))
            self._engine = eng
        return self._engine

    def loss_grad(self, theta, want_grad: bool = True):
        """(total, term losses, gradient or None) at θ: one fused launch"""
        if self.sampled and self._calls > 0:
            self.engine.resample()
        self._calls += 1
        return self.engine.loss_grad_host(np.asarray(theta, dtype=self.dtype), self.term_weights, want_grad)

    def trial(self, theta, ts) -> np.ndarray:
        """φ(t) at the times ts, (n, len(ts)), evaluated on the device through value-only terms"""
        ts = np.ravel(np.asarray(ts, dtype=np.float64))
        if not hasattr(self, "_phi_engine"):
            lw = self.lowering
            terms = [lw.term(lw.phi(k), ["t"], REDUCE_MEAN) for k in range(self.n)]
            self._phi_engine = Engine(ProblemSpec(nets=[NetSpec(self.alg.chain.dims, self.alg.chain.acts, 0)], terms=terms,
                                                  n_params=self.spec.n_params, param_offset=self.n_net,
                                                  n_theta=self.spec.n_theta, dtype=self.dtype.name,
                                                  mode=_eng.MODE_FFMA, device=self.alg.device))
        e = self._phi_engine
        th = np.asarray(theta, dtype=self.dtype)
        out = np.empty((self.n, ts.size))
        for k in range(self.n):
            e.set_points_host(k, ts.reshape(1, -1).astype(self.dtype))
            out[k] = e.term_residual_host(k, th, ts.size)
        return out


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
        self.errors = {}
        an = rep.prob.f.analytic
        if an is not None:
            A = np.stack([np.ravel(np.asarray(an(rep.prob.u0, rep.prob.p, float(ti)), dtype=np.float64))
                          for ti in self.t], axis=1)
            E = U - A
            self.errors = {"final": float(np.mean(np.abs(E[:, -1]))), "l∞": float(np.max(np.abs(E))),
                           "l2": float(np.sqrt(np.mean(E ** 2)))}

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
