"""Host-side mirror of the reference's PINN interface for the hot path:
``PhysicsInformedNN(chain, strategy; ...)``, ``symbolic_discretize`` -> ``PINNRepresentation``,
``discretize`` -> ``OptimizationProblem`` (reference src/pinn_types.jl:147-211, :257-440;
src/discretize.jl:413-780).  Same names, argument meaning and error behaviour; every
loss / gradient / residual evaluation goes through the C ABI (engine.py) to the CUDA
kernels -- there is no CPU code path here.
"""
from __future__ import annotations

import dataclasses
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Sequence, Union

import numpy as np

from . import engine as _eng
from .engine import (Engine, EngineError, FixedNetSpec, IntegralSpec, NetSpec, ProblemSpec, TapSpec, TermSpec,
                     REDUCE_ABS_OF_SUM, REDUCE_MEAN, REDUCE_SQUARE_OF_SUM, REDUCE_WSUM)
from .lowering import LoweredTerm, LoweringError, lower_equation, term_spec
from .strategies import (AbstractTrainingStrategy, GridTraining, QuadratureTraining, QuasiRandomTraining,
                         StochasticTraining, _julia_range, _product_columns, gauss_legendre_box, generate_quasi_random_points,
                         generate_random_points, generate_training_sets, get_bounds, shard_range)
from .symbolic import Equation, FixedNet, PDESystem, VarInfo, eq_indvars, fixed_function, get_vars

# PhysicsInformedNN(mode=...) -> PINN_MODE_*; "ffma" and "tc_f64" run the FFMA kernel (integral terms, fixed networks and
# functional terms evaluate there only)
MODES = {"ffma": _eng.MODE_FFMA, "tc_bf16": _eng.MODE_TC_BF16, "tc_split": _eng.MODE_TC_SPLIT, "tc_f64": _eng.MODE_TC_F64}
FFMA_KERNEL_MODES = (_eng.MODE_FFMA, _eng.MODE_TC_F64)

_ACT_NAMES = {"identity": "identity", "tanh": "tanh", "sigmoid": "sigmoid", "σ": "sigmoid", "sin": "sin",
              "softplus": "softplus", "swish": "swish", "gelu": "gelu", "logcosh": "logcosh", "cos": "cos",
              None: "identity"}


# ---- Lux stand-ins -----------------------------------------------------------------------------
@dataclass
class Dense:
    """``Dense(in => out, activation)``: ``activation.(W*x .+ b)``."""
    in_dims: int
    out_dims: int
    activation: Optional[str] = None

    def __post_init__(self):
        if self.activation not in _ACT_NAMES:
            raise ValueError("unsupported activation %r (supported: %s)" % (self.activation, sorted(
                k for k in _ACT_NAMES if k)))
        self.activation = _ACT_NAMES[self.activation]


@dataclass
class Chain:
    """``Chain(Dense(...), Dense(...), ...)`` of Dense layers."""
    layers: List[Dense]

    def __init__(self, *layers):
        if len(layers) == 1 and isinstance(layers[0], (list, tuple)):
            layers = tuple(layers[0])
        for a, b in zip(layers[:-1], layers[1:]):
            if a.out_dims != b.in_dims:
                raise ValueError("Chain: layer widths do not chain (%d -> %d)" % (a.out_dims, b.in_dims))
        self.layers = list(layers)

    @property
    def dims(self) -> List[int]:
        return [self.layers[0].in_dims] + [l.out_dims for l in self.layers]

    @property
    def acts(self) -> List[str]:
        return [l.activation for l in self.layers]

    @property
    def n_params(self) -> int:
        return sum(l.in_dims * l.out_dims + l.out_dims for l in self.layers)


def initialparameters(rng: np.random.Generator, chain: Chain, dtype=np.float64) -> np.ndarray:
    """Lux default init (glorot_uniform weights, zero bias), flattened in ComponentArray order:
    per layer weight (out x in, column-major) then bias."""
    parts = []
    for l in chain.layers:
        lim = np.sqrt(6.0 / (l.in_dims + l.out_dims))
        W = rng.uniform(-lim, lim, size=(l.out_dims, l.in_dims))
        parts += [W.ravel(order="F"), np.zeros(l.out_dims)]
    return np.concatenate(parts).astype(dtype)


# ---- logging (reference src/pinn_types.jl:7-68) ------------------------------------------------------
@dataclass
class LogOptions:
    log_frequency: int = 50


def logscalar(logger, scalar, name: str, step: int):
    """No-op fallback; loggers opt in by defining ``log_value(name, scalar, step=)``."""
    if logger is not None and hasattr(logger, "log_value"):
        logger.log_value(name, float(scalar), step=step)


def logvector(logger, vector, name: str, step: int):
    if logger is not None and hasattr(logger, "log_value"):
        for j, v in enumerate(vector):
            logger.log_value("%s/%d" % (name, j + 1), float(v), step=step)


# ---- adaptive losses (reference src/adaptive_losses.jl:22-42) -----------------------------------------
@dataclass
class NonAdaptiveLoss:
    pde_loss_weights: Union[float, Sequence[float]] = 1.0
    bc_loss_weights: Union[float, Sequence[float]] = 1.0
    additional_loss_weights: Union[float, Sequence[float]] = 1.0

    def reweights_at(self, iteration: int) -> bool:
        return False

    def update(self, iteration, pde_losses, bc_losses, weights, term_grad_stats=None):   # Returns(nothing)
        return None


@dataclass
class Adam:
    """``Optimisers.Adam(η, (β1, β2), ϵ)`` hyper-parameters (also the rule of ``solve``)."""
    lr: float = 1e-3
    beta1: float = 0.9
    beta2: float = 0.999
    eps: float = 1e-8


@dataclass
class HagerZhang:
    """``LineSearches.HagerZhang()`` with its defaults (Hager & Zhang 2006): Wolfe / approximate-Wolfe parameters δ, σ,
    ε; bisection weight θ; interval shrink γ; bracket expansion ρ; step shrink ψ₃ after a non-finite value; iteration
    cap.  The device driver implements these values only."""
    delta: float = 0.1
    sigma: float = 0.9
    epsilon: float = 1e-6
    theta: float = 0.5
    gamma: float = 0.66
    rho: float = 5.0
    psi3: float = 0.1
    linesearchmax: int = 50


@dataclass
class BackTracking:
    """``LineSearches.BackTracking()`` with its defaults: Armijo constant c₁, step clamp [ρ_lo, ρ_hi], cubic
    interpolation (order 3), iteration cap.  The device driver implements these values only."""
    c_1: float = 1e-4
    rho_hi: float = 0.5
    rho_lo: float = 0.1
    iterations: int = 1000
    order: int = 3


@dataclass
class LBFGS:
    """``Optim.LBFGS(m = 10, linesearch = HagerZhang())``: α₀ = 1 every iteration (InitialStatic), initial inverse
    Hessian γI with γ = sᵀy / yᵀy of the newest pair (scaleinvH0); the first step is along -g."""
    m: int = 10
    linesearch: object = field(default_factory=HagerZhang)


@dataclass
class BFGS:
    """``Optim.BFGS(linesearch = HagerZhang(), initial_stepnorm = nothing)``: dense inverse Hessian,
    H₀ = I or I · initial_stepnorm / ‖g₀‖∞."""
    linesearch: object = field(default_factory=HagerZhang)
    initial_stepnorm: Optional[float] = None


@dataclass
class Descent:
    """``Optimisers.Descent(η)``."""
    lr: float = 0.1


class _RuleState:
    """``Optimisers.setup(rule, x)`` + ``Optimisers.update!(state, x, dx)`` for the two rules the adaptive losses use:
    x .-= step(dx).  Adam: mt, vt moments with bias correction by running powers of β (Optimisers.jl's `apply!`)."""

    def __init__(self, rule, n: int):
        self.rule = rule
        self.m, self.v = np.zeros(n), np.zeros(n)
        self.b1t, self.b2t = 1.0, 1.0

    def update(self, x: np.ndarray, dx: np.ndarray):
        r = self.rule
        dx = np.asarray(dx, dtype=np.float64)
        if isinstance(r, Descent):
            x -= r.lr * dx
            return
        self.b1t *= r.beta1
        self.b2t *= r.beta2
        self.m = r.beta1 * self.m + (1.0 - r.beta1) * dx
        self.v = r.beta2 * self.v + (1.0 - r.beta2) * dx * dx
        x -= self.m / (1.0 - self.b1t) / (np.sqrt(self.v / (1.0 - self.b2t)) + r.eps) * r.lr


def _softmax(x: np.ndarray) -> np.ndarray:
    e = np.exp(x - np.max(x))          # reference src/adaptive_losses.jl:242-245
    return e / e.sum()


@dataclass
class MiniMaxAdaptiveLoss:
    """Weights are MAXIMISED by an internal optimiser fed with ``-losses`` every ``reweight_every`` iterations
    (reference src/adaptive_losses.jl:183-239; defaults ``Adam(1e-4)`` for the pde weights and ``Adam(0.5)`` for the
    bc weights, any ``Adam(...)`` / ``Descent(...)`` rule accepted)."""
    reweight_every: int
    pde_max_optimiser: object = field(default_factory=lambda: Adam(1e-4))
    bc_max_optimiser: object = field(default_factory=lambda: Adam(0.5))
    pde_loss_weights: Union[float, Sequence[float]] = 1.0
    bc_loss_weights: Union[float, Sequence[float]] = 1.0
    additional_loss_weights: Union[float, Sequence[float]] = 1.0

    def reweights_at(self, iteration: int) -> bool:
        return iteration % self.reweight_every == 0

    def update(self, iteration, pde_losses, bc_losses, weights, term_grad_stats=None):
        if not hasattr(self, "_pde_state"):      # Optimisers.setup at generate_adaptive_loss_function time (:205-210)
            self._pde_state = _RuleState(self.pde_max_optimiser, len(weights["pde"]))
            self._bc_state = _RuleState(self.bc_max_optimiser, len(weights["bc"]))
        if iteration % self.reweight_every == 0:
            self._pde_state.update(weights["pde"], -np.asarray(pde_losses, dtype=np.float64))
            self._bc_state.update(weights["bc"], -np.asarray(bc_losses, dtype=np.float64))


@dataclass
class SoftAdaptAdaptiveLoss:
    """``λ = softmax(α · (L(t) − L(t_prev)) / (L(t_prev) + ε)) · N`` over all pde and bc terms every ``reweight_every``
    iterations (reference src/adaptive_losses.jl:247-364; Heydari et al., arXiv:1912.12355).  The previous losses are
    seeded by the very first call (:335-339) and replaced at every reweighting."""
    reweight_every: int
    alpha: float = 0.1
    pde_loss_weights: Union[float, Sequence[float]] = 1.0
    bc_loss_weights: Union[float, Sequence[float]] = 1.0
    additional_loss_weights: Union[float, Sequence[float]] = 1.0

    def reweights_at(self, iteration: int) -> bool:
        return iteration % self.reweight_every == 0

    def update(self, iteration, pde_losses, bc_losses, weights, term_grad_stats=None):
        cur = np.concatenate([np.asarray(pde_losses, dtype=np.float64), np.asarray(bc_losses, dtype=np.float64)])
        if not hasattr(self, "_prev"):
            self._prev = cur.copy()
        if iteration % self.reweight_every == 0:
            rates = (cur - self._prev) / (self._prev + 1e-8)
            w = _softmax(self.alpha * rates) * cur.size
            n_pde = len(pde_losses)
            weights["pde"][:] = w[:n_pde]
            weights["bc"][:] = w[n_pde:]
            self._prev = cur.copy()


@dataclass
class ReLoBRaLoAdaptiveLoss:
    """Relative loss balancing with random lookback: ``λ = softmax(α · L(t) / (L(t0) + ε)) · N`` where t0 is the
    previous reweighting with probability β and the first call otherwise (reference src/adaptive_losses.jl:366-491;
    Bischof & Kraus, arXiv:2110.09813).  ``seed`` fixes the Bernoulli draws (the reference uses the global RNG)."""
    reweight_every: int
    alpha: float = 1.0
    beta: float = 0.9
    pde_loss_weights: Union[float, Sequence[float]] = 1.0
    bc_loss_weights: Union[float, Sequence[float]] = 1.0
    additional_loss_weights: Union[float, Sequence[float]] = 1.0
    seed: Optional[int] = None

    def reweights_at(self, iteration: int) -> bool:
        return iteration % self.reweight_every == 0

    def update(self, iteration, pde_losses, bc_losses, weights, term_grad_stats=None):
        cur = np.concatenate([np.asarray(pde_losses, dtype=np.float64), np.asarray(bc_losses, dtype=np.float64)])
        if not hasattr(self, "_init"):
            self._init, self._prev = cur.copy(), cur.copy()
            self._rng = np.random.default_rng(self.seed)
        if iteration % self.reweight_every == 0:
            use_prev = self._rng.random() < self.beta
            ref = self._prev if use_prev else self._init
            w = _softmax(self.alpha * cur / (ref + 1e-8)) * cur.size
            n_pde = len(pde_losses)
            weights["pde"][:] = w[:n_pde]
            weights["bc"][:] = w[n_pde:]
            self._prev = cur.copy()
            self.last_use_prev = bool(use_prev)


@dataclass
class GradientScaleAdaptiveLoss:
    """Boundary weights follow ``max|grad L_pde| / mean|grad L_bc_j|`` through an exponential moving average
    (reference src/adaptive_losses.jl:76-134, after Wang, Teng & Perdikaris).  The reference differentiates every term
    closure with Zygote on each reweighting; here ``term_grad_stats(i)`` is one fused engine evaluation of term i with
    the two reductions done on the device (``pinn_term_grad_stats``)."""
    reweight_every: int
    weight_change_inertia: float = 0.9
    pde_loss_weights: Union[float, Sequence[float]] = 1.0
    bc_loss_weights: Union[float, Sequence[float]] = 1.0
    additional_loss_weights: Union[float, Sequence[float]] = 1.0

    def reweights_at(self, iteration: int) -> bool:
        return iteration % self.reweight_every == 0

    def update(self, iteration, pde_losses, bc_losses, weights, term_grad_stats=None):
        if iteration % self.reweight_every != 0:
            return
        if term_grad_stats is None:
            raise ValueError("GradientScaleAdaptiveLoss needs per-term gradient statistics from the engine")
        n_pde, n_bc = len(pde_losses), len(bc_losses)
        # the paper assumes one PDE loss: the reference takes the maximum of the per-equation maxima (:107-110)
        pde_grads_max = max(term_grad_stats(i)[0] for i in range(n_pde))
        bc_grads_mean = np.array([term_grad_stats(n_pde + j)[1] for j in range(n_bc)], dtype=np.float64)
        # `adaloss_T isa Float64` in the reference (:117) tests a type against a type and is always false,
        # so the divisor guard is 1e-7 for every element type; kept as is
        eps = 1e-7
        proposed = pde_grads_max / (bc_grads_mean + eps)
        a = float(self.weight_change_inertia)
        weights["bc"][:] = a * weights["bc"] + (1.0 - a) * proposed
        self.last = {"pde_grad_max": pde_grads_max, "bc_grads_mean": bc_grads_mean}


@dataclass
class DataLoss:
    """Native ``additional_loss``: ``mean(abs2, u_k(X) .- y)`` over observations.

    The reference accepts an arbitrary Julia closure ``additional_loss(phi, θ, p)``
    differentiated by Zygote (src/discretize.jl:590-598); a closure cannot run inside a CUDA
    kernel, so the engine takes the structured form of the common case (SURVEY section 8(f)
    item 3; fixture test/NNPDE2/additional_loss__lorenz_system.jl:60-69)."""
    depvar: str
    points: np.ndarray        # (d, n) inputs of the dependent variable
    values: np.ndarray        # (n,) observations


@dataclass
class IntegralLoss:
    """Native non-data ``additional_loss``: an integral constraint ``g(Σ_p w_p v_p - target)``, ``g = |·|``
    (``norm="abs"``) or ``(·)²`` (``norm="abs2"``), ``v_p`` the integrand at node p.

    The reference states such constraints as closures (test/NNPDE2/additional_loss__fokker_planck.jl:42-46,
    docs/src/tutorials/constraints.md:58-71); a closure cannot run inside a CUDA kernel, so the engine takes this
    structured form, as ``DataLoss`` does for data.  ``integrand`` is an expression in the independent variables, the
    dependent variables and their derivatives, parameters and registered functions, lowered like an equation side.
    The nodes are the engine's fixed Gauss-Legendre box on ``domains`` (``nodes_per_dim`` per variable), or explicit
    ``points`` ((d, n), one row per argument of the dependent variables the integrand applies) with ``weights``
    (1 when omitted).  The reference's adaptive cubature is replaced by the fixed rule.  The term runs on the FFMA
    path; with several ranks its whole node set stays on rank 0."""
    integrand: object
    domains: Optional[Sequence] = None
    _: dataclasses.KW_ONLY
    points: Optional[np.ndarray] = None
    weights: Optional[np.ndarray] = None
    target: float = 0.0
    norm: str = "abs"
    nodes_per_dim: int = 16

    def __post_init__(self):
        if self.norm not in ("abs", "abs2"):
            raise ValueError("IntegralLoss: norm must be \"abs\" or \"abs2\", got %r" % (self.norm,))
        if (self.domains is None) == (self.points is None):
            raise ValueError("IntegralLoss: give either domains (Gauss-Legendre nodes) or explicit points")
        if self.weights is not None and self.points is None:
            raise ValueError("IntegralLoss: weights go with explicit points")
        if int(self.nodes_per_dim) < 1:
            raise ValueError("IntegralLoss: nodes_per_dim must be >= 1")

    def nodes(self, rows: List[str]):
        """(points (len(rows), n), weights (n,)) in float64; row i is the variable rows[i]"""
        if self.points is not None:
            X = np.asarray(self.points, dtype=np.float64)
            X = X.reshape(1, -1) if X.ndim == 1 else X
            if X.ndim != 2 or X.shape[0] != len(rows):
                raise ValueError("IntegralLoss: points must be (%d, n) for the variables %s, got shape %s"
                                 % (len(rows), rows, np.shape(self.points)))
            w = np.ones(X.shape[1]) if self.weights is None else np.asarray(self.weights, dtype=np.float64)
            if np.ndim(w) == 0:
                w = np.full(X.shape[1], float(w))
            if w.shape != (X.shape[1],):
                raise ValueError("IntegralLoss: weights must have shape (%d,), got %s" % (X.shape[1], w.shape))
            return X, w
        box = {str(d.variables): (float(d.domain.lo), float(d.domain.hi)) for d in self.domains}
        missing = [r for r in rows if r not in box]
        if missing:
            raise ValueError("IntegralLoss: no domain for the variables %s" % missing)
        lb = np.array([box[r][0] for r in rows])
        ub = np.array([box[r][1] for r in rows])
        X, w, _ = gauss_legendre_box((lb, ub), int(self.nodes_per_dim), np.float64)
        return X, w


@dataclass
class _ResidualSumLoss:
    """``additional_loss`` Σ_p (lhs - rhs)² of ``eq`` at the columns of ``points`` (one row per variable of the
    equation): a weighted-sum term with unit weights and scale 1, whose integrals take ``q`` Gauss-Legendre nodes.
    SDEPINN's norm loss Σ_t (∫ p̂(x, t) dx - 1)² is one (sde_weak.py)."""
    eq: Equation
    points: np.ndarray
    q: int = _eng.MAX_QUAD


def _integral_loss_term(add: IntegralLoss, vi: VarInfo, param_index, param_values, fixed):
    """(TermSpec, points, weights) of the functional term: the program yields v_p - target / Σw, so that
    Σ_p w_p (v_p - target / Σw) = Σ_p w_p v_p - target"""
    import sympy as sp
    if callable(add.integrand) and not isinstance(add.integrand, sp.Basic):
        raise ValueError("IntegralLoss: the integrand must be an expression, not a callable")
    integrand = sp.sympify(add.integrand)
    rows = eq_indvars(Equation(integrand, sp.Integer(0)), vi)
    if not rows:
        raise ValueError("IntegralLoss: the integrand %s applies no dependent variable: nothing to train on" % integrand)
    X, w = add.nodes(rows)
    sw = float(np.sum(w))
    if add.target != 0 and sw == 0:
        raise ValueError("IntegralLoss: the weights sum to 0, so a nonzero target cannot be folded into the integrand")
    shift = float(add.target) / sw if add.target != 0 else 0.0
    lt = lower_equation(Equation(integrand, sp.Float(shift)), vi, param_index, param_values, hoist=False, fixed=fixed)
    if lt.integrals:
        raise ValueError("IntegralLoss: the integrand may not contain an Integral")
    red = REDUCE_ABS_OF_SUM if add.norm == "abs" else REDUCE_SQUARE_OF_SUM
    return term_spec(lt, red, 1.0), X, w


# ---- PhysicsInformedNN -------------------------------------------------------------------------------
class AbstractPINN:
    pass


@dataclass
class PhysicsInformedNN(AbstractPINN):
    """``PhysicsInformedNN(chain, strategy; init_params, phi, derivative, param_estim,
    additional_loss, adaptive_loss, logger, log_options, iteration)``
    (reference src/pinn_types.jl:165-211).  ``chain``: one Chain, or a list with one
    1-output Chain per dependent variable.  Engine options arrive as extra keywords:
    ``mode`` ("ffma" | "tc_bf16" | "tc_split" | "tc_f64"), ``device``.  The bf16 tensor-core modes need float32 and
    1-output networks with a linear last layer; "tc_split" takes hidden widths 16 / 32 / 48 / 64, "tc_bf16" also 64 / 128
    and any multiple of 64 up to 256 (include/pinn_b200.h lists the shapes; anything else is refused with a message).
    "tc_f64" needs float64 and takes everything "ffma" takes: the same kernel with its layer products on the FP64 tensor
    cores."""
    chain: Union[Chain, List[Chain]]
    strategy: AbstractTrainingStrategy
    init_params: Optional[np.ndarray] = None
    phi: Optional[object] = None
    derivative: Optional[object] = None
    param_estim: bool = False
    additional_loss: Optional[object] = None
    adaptive_loss: Optional[object] = None
    logger: Optional[object] = None
    log_options: LogOptions = field(default_factory=LogOptions)
    iteration: Optional[list] = None
    mode: str = "ffma"
    device: int = 0
    seed: int = 0

    def __post_init__(self):
        if self.derivative is not None:
            raise ValueError("a custom `derivative` cannot be injected: derivatives are exact forward-mode "
                             "taps evaluated inside the CUDA kernel")
        if self.phi is not None:
            raise ValueError("a custom trial solution `phi` is not supported by the engine (MLP chains only)")
        self.multioutput = isinstance(self.chain, (list, tuple))
        if self.iteration is None:
            self.iteration = [0]
            self.self_increment = True
        else:
            self.self_increment = False


class BayesianPINN(AbstractPINN):
    """``BayesianPINN(args...; dataset = nothing, kwargs...)`` (reference src/pinn_types.jl:214-245): wraps a
    PhysicsInformedNN; ``symbolic_discretize`` then builds ``full_loss_function(θ, allstd)`` = the weighted
    log-likelihood (src/discretize.jl:653-757) that the HMC samplers of ext/bpinn consume; ``ahmc_bayesian_pinn_pde``
    samples its posterior on the device.  The likelihood and its θ-gradient come from the same fused kernel.
    ``dataset = [dataset_pde, dataset_bc]``: each None or a list with one ``n × (1 + d_k)`` array per dependent
    variable, observed values in column 1 and the variable's d_k inputs after it.  Equation (bc) j is also evaluated at
    the coordinates of dataset_pde[j] (dataset_bc[j]); with ``param_estim`` the observations enter as L2LossData."""

    def __init__(self, *args, dataset=None, **kwargs):
        self.pinn = PhysicsInformedNN(*args, **kwargs)
        self.dataset = (None, None) if dataset is None else tuple(dataset)

    def __getattr__(self, name):                  # Base.getproperty forwarding (:236-240)
        return getattr(self.pinn, name)


@dataclass
class PINNLossFunctions:
    bc_loss_functions: List[Callable]
    pde_loss_functions: List[Callable]
    full_loss_function: Callable
    additional_loss_function: Optional[object]
    datafree_pde_loss_functions: List[Callable]
    datafree_bc_loss_functions: List[Callable]
    full_loss_gradient: Optional[Callable] = None     # explicit gradient (replaces AutoZygote)


@dataclass
class PINNRepresentation:
    eqs: list
    bcs: list
    domains: list
    eq_params: list
    defaults: dict
    default_p: Optional[list]
    param_estim: bool
    additional_loss: object
    adaloss: object
    depvars: list
    indvars: list
    dict_indvars: dict
    dict_depvars: dict
    dict_depvar_input: dict
    logger: object
    multioutput: bool
    iteration: list
    init_params: np.ndarray
    flat_init_params: np.ndarray
    phi: object
    derivative: object
    strategy: object
    pde_indvars: list
    bc_indvars: list
    symbolic_pde_loss_functions: List[LoweredTerm]
    symbolic_bc_loss_functions: List[LoweredTerm]
    loss_functions: Optional[PINNLossFunctions] = None
    engine: Optional[Engine] = None
    term_names: List[str] = field(default_factory=list)


class Phi:
    """Trial solution ``phi(x, θ)`` (reference src/pinn_types.jl:79-90), evaluated on the GPU
    through a value-only term of an auxiliary engine handle."""

    def __init__(self, chain: Chain, theta_offset: int, n_theta: int, dtype, device: int = 0):
        self.chain, self.theta_offset, self.n_theta = chain, theta_offset, n_theta
        self.dtype, self.device = np.dtype(dtype), device
        self._engine = None

    def _get(self) -> Engine:
        if self._engine is None:
            net = NetSpec(self.chain.dims, self.chain.acts, self.theta_offset)
            term = TermSpec(dim=self.chain.dims[0], taps=[TapSpec(net=0, order=0)], prog=[("tap", 0, 0, 0.0)],
                            net_rows=[list(range(self.chain.dims[0]))])
            self._engine = Engine(ProblemSpec(nets=[net], terms=[term], n_theta=self.n_theta,
                                              dtype=self.dtype.name, device=self.device))
        return self._engine

    def __call__(self, x, theta) -> np.ndarray:
        x = np.asarray(x, dtype=self.dtype)
        scalar = x.ndim == 0
        x = x.reshape(self.chain.dims[0], -1) if x.ndim <= 1 else x
        if x.shape[0] != self.chain.dims[0]:
            raise ValueError("phi: expected %d input rows, got %d" % (self.chain.dims[0], x.shape[0]))
        eng = self._get()
        eng.set_points_host(0, x)
        r = eng.term_residual_host(0, np.asarray(theta, dtype=self.dtype), x.shape[1])
        return r[0] if scalar else r.reshape(1, -1)


def register_symbolic(phi: Phi, theta, name: str = "phi_registered"):
    """``phi_bound(x, y) = first(phi(vcat(x, y), θ))`` followed by ``@register_symbolic phi_bound(x, y)``: a function
    usable in equations -- applications and ``Differential``s of them -- that evaluates the trained network ``phi`` at
    parameters ``theta`` (the full θ ``phi`` was trained with).  The network runs inside the fused kernel as a fixed
    network: its parameters are not trained and receive no gradient."""
    if not isinstance(phi, Phi):
        raise TypeError("register_symbolic: expected a trained network's Phi (discretization.phi), got %r" % type(phi))
    if phi.chain.dims[-1] != 1:
        raise ValueError("register_symbolic: the network must have a 1-dimensional output")
    th = np.asarray(theta, dtype=np.float64).reshape(-1)
    if th.size < phi.theta_offset + phi.chain.n_params:
        raise ValueError("register_symbolic: theta has %d entries, the network needs [%d, %d)"
                         % (th.size, phi.theta_offset, phi.theta_offset + phi.chain.n_params))
    params = th[phi.theta_offset:phi.theta_offset + phi.chain.n_params].copy()
    return fixed_function(name, FixedNet(list(phi.chain.dims), list(phi.chain.acts), params))


def _fixed_specs(fixed: List[FixedNet]) -> List[FixedNetSpec]:
    return [FixedNetSpec(f.dims, f.acts) for f in fixed]


def _upload_fixed(eng: Engine, fixed: List[FixedNet]):
    for j, f in enumerate(fixed):
        eng.set_fixed_params_host(j, f.params)


# ---- discretization --------------------------------------------------------------------------------------
def _per_term(w, n: int, what: str) -> np.ndarray:
    if np.isscalar(w):
        return np.full(n, float(w))
    w = np.asarray(w, dtype=np.float64)
    if w.shape != (n,):
        raise ValueError("%s: expected %d weights, got %s" % (what, n, w.shape))
    return w.copy()


def symbolic_discretize(pde_system: PDESystem, discretization: PhysicsInformedNN, rank: int = 0,
                        world: int = 1) -> PINNRepresentation:
    """Build the engine problem for a PDESystem (reference src/discretize.jl:413-767).
    ``rank`` / ``world`` shard every term's point set contiguously (SURVEY section 8(e))."""
    bayes = isinstance(discretization, BayesianPINN)
    if bayes:
        dataset = discretization.dataset
        if not isinstance(discretization.pinn.strategy, GridTraining):
            raise ValueError("BayesianPINN: the reference defines the log-likelihood form for GridTraining only "
                             "(merge_strategy_with_loglikelihood_function, src/training_strategies.jl:50-113)")
        if discretization.pinn.adaptive_loss is not None and not isinstance(discretization.pinn.adaptive_loss, NonAdaptiveLoss):
            raise ValueError("BayesianPINN: adaptive loss weights are not supported with the log-likelihood form")
        discretization = discretization.pinn
    else:
        dataset = (None, None)
    if not isinstance(discretization, PhysicsInformedNN):
        raise TypeError("symbolic_discretize: expected a PhysicsInformedNN or BayesianPINN")
    d = discretization
    eqs, bcs, domains = list(pde_system.eqs), list(pde_system.bcs), list(pde_system.domain)
    if len(bcs) == 0:
        # reference: builds, then solve throws MethodError
        # (test/direct_function__empty_boundary_condition_fails_in_solve_phase.jl:15-25)
        raise ValueError("PDESystem has no boundary conditions: the loss has no bc terms to sum")
    vi: VarInfo = get_vars(pde_system.ivs, pde_system.dvs)
    chains = list(d.chain) if d.multioutput else [d.chain]
    if len(chains) != len(vi.depvars):
        raise ValueError("need one chain per dependent variable (%d chains, %d depvars)"
                         % (len(chains), len(vi.depvars)))
    for c, name in zip(chains, vi.depvars):
        if c.dims[0] != len(vi.dict_depvar_input[name]):
            raise ValueError("chain for %s has %d inputs, the variable has %d arguments"
                             % (name, c.dims[0], len(vi.dict_depvar_input[name])))
        if c.dims[-1] != 1:
            raise ValueError("chain for %s must have a 1-dimensional output" % name)
    ds_pde, ds_bc = _bayes_dataset(dataset, vi)

    # ---- parameters: θ = [depvar blocks..., p] (src/discretize.jl:432-472) -----------------------------
    eq_params = [str(p) for p in pde_system.ps]
    defaults = {str(k): float(v) for k, v in pde_system.defaults.items()}
    n_net = sum(c.n_params for c in chains)
    n_p = len(eq_params) if d.param_estim else 0
    if d.init_params is None:
        rng = np.random.default_rng(d.seed)
        flat = np.concatenate([initialparameters(rng, c, np.float64) for c in chains])   # Float64 default
        if d.param_estim:
            flat = np.concatenate([flat, np.array([defaults.get(p, 1.0) for p in eq_params])])
    else:
        flat = np.asarray(d.init_params)
        if flat.dtype not in (np.float32, np.float64):
            flat = flat.astype(np.float64)
        if flat.shape != (n_net + n_p,):
            raise ValueError("init_params has length %d, the chains%s need %d"
                             % (flat.size, " + p" if n_p else "", n_net + n_p))
    dtype = flat.dtype
    if d.mode == "tc_f64" and dtype != np.float64:
        raise ValueError("mode=\"tc_f64\" runs the layer products on the FP64 tensor cores and needs float64 parameters "
                         "(init_params is %s); use mode=\"ffma\", \"tc_bf16\" or \"tc_split\" for float32" % dtype.name)
    offs, o = [], 0
    for c in chains:
        offs.append(o)
        o += c.n_params
    param_index = {p: i for i, p in enumerate(eq_params)} if d.param_estim else {}
    param_values = {} if d.param_estim else defaults
    default_p = None if d.param_estim or not eq_params else [defaults[p] for p in eq_params]
    if eq_params and not d.param_estim:
        missing = [p for p in eq_params if p not in defaults]
        if missing:
            raise ValueError("parameters %s have no default value and param_estim=false" % missing)

    # ---- lower equations (src/discretize.jl:505-539) -------------------------------------------------------
    try:
        # points drawn on the device carry only coordinates: no host-evaluated (hoisted) rows then
        hoist = not getattr(d.strategy, "device_sampler", False)
        fixed: List[FixedNet] = []          # registered network functions the equations apply
        pde_terms = [lower_equation(e, vi, param_index, param_values, hoist=hoist, fixed=fixed) for e in eqs]
        bc_terms = [lower_equation(e, vi, param_index, param_values, hoist=hoist, fixed=fixed) for e in bcs]
        add = d.additional_loss
        if isinstance(add, _ResidualSumLoss):
            add_lt = lower_equation(add.eq, vi, param_index, param_values, fixed=fixed)
            add_lt.integrals = [dataclasses.replace(it, q=int(add.q)) for it in add_lt.integrals]
        elif add is not None and not isinstance(add, (DataLoss, IntegralLoss)):
            raise ValueError("additional_loss must be a DataLoss (data term) or an IntegralLoss (integral constraint); "
                             "arbitrary closures cannot run inside the CUDA kernel")
        if isinstance(add, IntegralLoss):
            if bayes:
                raise ValueError("BayesianPINN: an IntegralLoss has no log-likelihood form (the reference adds "
                                 "additional_loss values as one observation); use PhysicsInformedNN")
            if d.mode not in ("ffma", "tc_f64"):
                raise ValueError("IntegralLoss: functional terms run on the FFMA path: use mode=\"ffma\"")
            func_spec, func_pts, func_w = _integral_loss_term(add, vi, param_index, param_values, fixed)
    except LoweringError as ex:
        raise ValueError(str(ex)) from ex

    # ---- adaptive weights (src/discretize.jl:548-564) -------------------------------------------------------
    adaloss = d.adaptive_loss if d.adaptive_loss is not None else NonAdaptiveLoss()
    weights = {"pde": _per_term(adaloss.pde_loss_weights, len(eqs), "pde_loss_weights"),
               "bc": _per_term(adaloss.bc_loss_weights, len(bcs), "bc_loss_weights"),
               "add": _per_term(adaloss.additional_loss_weights, 1, "additional_loss_weights")}

    # ---- point sets per strategy (src/training_strategies.jl) ------------------------------------------------
    strategy = d.strategy
    specs: List[TermSpec] = []
    reductions = []
    for lt in pde_terms + bc_terms:
        if isinstance(strategy, QuadratureTraining):
            specs.append(term_spec(lt, REDUCE_WSUM, 1.0))      # scale filled below
        else:
            specs.append(term_spec(lt, REDUCE_MEAN))
    # BayesianPINN dataset terms (src/training_strategies.jl:84-108): equation / bc j's residual at the coordinates of
    # dataset j, paired by zip (so the shorter list decides how many), then with param_estim one L2LossData term per
    # dependent variable (ext/bpinn/PDE_BPINN.jl:147-180) over the dataset_pde and dataset_bc rows of that variable
    ds_terms: List[tuple] = []           # (lowered term, (d, n) coordinates)
    n_ds = []
    for ds, lts, what in ((ds_pde, pde_terms, "equation"), (ds_bc, bc_terms, "boundary condition")):
        for j, (lt, m) in enumerate(zip(lts, ds or [])):
            X = m[:, 1:].T
            if X.shape[0] != len(lt.indvars):
                raise ValueError("BayesianPINN: dataset %d has %d coordinate columns but %s %d has the variables %s"
                                 % (j + 1, X.shape[0], what, j + 1, lt.indvars))
            specs.append(term_spec(lt, REDUCE_MEAN))
            ds_terms.append((lt, X))
        n_ds.append(min(len(lts), len(ds or [])))
    l2_sets: List[np.ndarray] = []
    if bayes and d.param_estim and (ds_pde is not None or ds_bc is not None):
        for k, c in enumerate(chains):
            m = np.concatenate([ds[k] for ds in (ds_pde, ds_bc) if ds is not None], axis=0)
            din = c.dims[0]
            rows = [None] * len(chains)
            rows[k] = list(range(din))
            specs.append(TermSpec(dim=din + 1, taps=[TapSpec(net=k, order=0)],
                                  prog=[("tap", 0, 0, 0.0), ("coord", din, 0, 0.0), ("sub", 0, 1, 0.0)],
                                  net_rows=rows, reduction=REDUCE_MEAN))
            l2_sets.append(np.concatenate([m[:, 1:].T, m[:, :1].T], axis=0))
    if isinstance(add, IntegralLoss):
        specs.append(func_spec)
    if isinstance(add, _ResidualSumLoss):
        specs.append(term_spec(add_lt, REDUCE_WSUM, 1.0))
    if isinstance(add, DataLoss):
        if add.depvar not in vi.dict_depvars:
            raise ValueError("DataLoss: unknown dependent variable %s" % add.depvar)
        k = vi.dict_depvars[add.depvar]
        din = chains[k].dims[0]
        rows = [None] * len(chains)
        rows[k] = list(range(din))
        specs.append(TermSpec(dim=din + 1, taps=[TapSpec(net=k, order=0)],
                              prog=[("tap", 0, 0, 0.0), ("coord", din, 0, 0.0), ("sub", 0, 1, 0.0)],
                              net_rows=rows, reduction=REDUCE_MEAN))

    # integral terms (get_numeric_integral, src/discretize.jl:334-397): one set per term that reads them -- a dataset
    # term re-reads its equation's integrals at the dataset's coordinates -- numbered in term order
    integrals: List[IntegralSpec] = []
    owners = list(enumerate(pde_terms + bc_terms + [lt for lt, _ in ds_terms]))
    if isinstance(add, _ResidualSumLoss):
        owners.append((len(specs) - 1, add_lt))
    for i, lt in owners:
        if lt.integrals:
            base = len(integrals)
            integrals += [dataclasses.replace(it, owner=i) for it in lt.integrals]
            specs[i].prog = [("integral", base + ins[1], 0, 0.0) if ins[0] == "integral" else ins
                             for ins in specs[i].prog]
    if len(integrals) > _eng.MAX_INTEGRALS:
        raise ValueError("the system has %d integral terms (max %d)" % (len(integrals), _eng.MAX_INTEGRALS))

    nets = [NetSpec(c.dims, c.acts, off) for c, off in zip(chains, offs)]
    mode = MODES[d.mode]
    if fixed and mode not in FFMA_KERNEL_MODES:
        raise ValueError("registered network functions run on the FFMA path: use mode=\"ffma\"")
    spec = ProblemSpec(nets=nets, terms=specs, n_params=n_p, param_offset=n_net, n_theta=n_net + n_p,
                       dtype=dtype.name, mode=mode, device=d.device, integrals=integrals, fixed=_fixed_specs(fixed))

    n_pde, n_bc = len(eqs), len(bcs)
    point_sets: List[Optional[np.ndarray]] = [None] * len(specs)
    quad_w: List[Optional[np.ndarray]] = [None] * len(specs)
    bounds_all = None
    if isinstance(strategy, GridTraining):
        pde_sets, bc_sets = generate_training_sets(domains, strategy.dx, eqs, bcs, dtype.type, vi)
        for i, s in enumerate(pde_sets + bc_sets):
            point_sets[i] = s
    elif isinstance(strategy, (StochasticTraining, QuasiRandomTraining)):
        pb, bb = get_bounds(domains, eqs, bcs, dtype.type, vi, strategy)
        bounds_all = pb + bb
    elif isinstance(strategy, QuadratureTraining):
        pb, bb = get_bounds(domains, eqs, bcs, dtype.type, vi, strategy)
        for i, b in enumerate(pb + bb):
            npd = strategy.nodes_per_dim if i < n_pde else strategy.bc_nodes_per_dim
            pts, w, area = gauss_legendre_box(b, npd, dtype.type)
            point_sets[i], quad_w[i] = pts, w
            specs[i].scale = 1.0 / area
    else:
        raise TypeError("unsupported training strategy %r" % (strategy,))
    o = n_pde + n_bc
    for i, (_, X) in enumerate(ds_terms):
        point_sets[o + i] = X.astype(dtype)
    o += len(ds_terms)
    for i, m in enumerate(l2_sets):
        point_sets[o + i] = m.astype(dtype)
    n_main = o + len(l2_sets)             # every term but the additional loss
    if isinstance(add, DataLoss):
        X = np.asarray(add.points, dtype=dtype)
        y = np.asarray(add.values, dtype=dtype).reshape(1, -1)
        if X.ndim != 2 or X.shape[1] != y.shape[1]:
            raise ValueError("DataLoss: points must be (d, n) and values (n,)")
        point_sets[-1] = np.concatenate([X, y], axis=0)
    if isinstance(add, _ResidualSumLoss):
        point_sets[-1] = np.asarray(add.points, dtype=dtype)
        quad_w[-1] = np.ones(point_sets[-1].shape[1], dtype=dtype)
    func_term = len(specs) - 1 if isinstance(add, IntegralLoss) else -1

    eng = Engine(spec)
    _upload_fixed(eng, fixed)
    n_terms = len(specs)
    sampler_rng = np.random.default_rng(getattr(strategy, "seed", 0) + 7919 * rank)
    state = {"calls": 0}

    lowered = pde_terms + bc_terms + [lt for lt, _ in ds_terms]

    def augment(i: int, pts: np.ndarray) -> np.ndarray:
        """append the hoisted coordinate-only rows of term i (float64 evaluation, then theta's eltype)"""
        return lowered[i].augment(pts) if i < len(lowered) else pts

    def upload(i: int, pts: np.ndarray, w: Optional[np.ndarray] = None, shard: bool = True):
        n = pts.shape[1]
        lo, hi = shard_range(n, rank, world) if shard else (0, n)
        eng.set_points_host(i, augment(i, np.asarray(pts, dtype=dtype)[:, lo:hi]), None if w is None else w[lo:hi])
        if world > 1 and shard:
            eng.set_global_count(i, n)

    for i in range(n_terms):
        if point_sets[i] is not None:
            upload(i, point_sets[i], quad_w[i])
    if func_term >= 0:
        # g(Σ_r S_r) is not Σ_r g(S_r): the whole node set stays on rank 0, the other ranks hold none and add exactly 0
        point_sets[func_term], quad_w[func_term] = func_pts.astype(dtype), func_w.astype(dtype)
        n_f = func_pts.shape[1] if rank == 0 else 0
        eng.set_points_host(func_term, point_sets[func_term][:, :n_f], quad_w[func_term][:n_f])

    device_sampler = isinstance(strategy, (StochasticTraining, QuasiRandomTraining)) and strategy.device_sampler
    if device_sampler:
        # SURVEY 8(f).1: the reference draws on the host and uploads every call (training_strategies.jl:277-281);
        # here each term's box is registered once and every draw is one small kernel per term
        for i, b in enumerate(bounds_all):
            npts = strategy.points if i < n_pde else strategy.bcs_points
            lo, hi = shard_range(npts, rank, world)
            lb, ub = (np.asarray(v_, dtype=np.float64) for v_ in b)
            eng.set_sampler(i, hi - lo, lb, ub, strategy.seed + 7919 * rank,
                            kind="lhs" if isinstance(strategy, QuasiRandomTraining) else "uniform")
            if world > 1:
                eng.set_global_count(i, npts)

    def resample():
        """Stochastic: fresh uniform points each call (training_strategies.jl:277-281);
        QuasiRandom(resampling=true): a fresh scrambled sequence each call (:375-380)."""
        if bounds_all is None:
            return
        if device_sampler:
            if state["calls"] > 0:
                eng.resample()
            for i in range(len(bounds_all)):
                point_sets[i] = None            # fetched on demand (rep.current_points)
            return
        if isinstance(strategy, QuasiRandomTraining) and not strategy.resampling and state["calls"] > 0:
            return
        for i, b in enumerate(bounds_all):
            npts = strategy.points if i < n_pde else strategy.bcs_points
            if isinstance(strategy, StochasticTraining):
                lo, hi = shard_range(npts, rank, world)
                pts = generate_random_points(hi - lo, b, dtype.type, sampler_rng)
                eng.set_points_host(i, augment(i, pts))
                if world > 1:
                    eng.set_global_count(i, npts)
            else:
                pts = generate_quasi_random_points(npts, b, dtype.type, strategy.seed + state["calls"] * 1009 + i)
                upload(i, pts)
            point_sets[i] = pts

    def term_weights() -> np.ndarray:
        w = np.concatenate([weights["pde"], weights["bc"], np.zeros(n_main - n_pde - n_bc)])
        if add is not None:
            w = np.concatenate([w, weights["add"]])
        return w

    iteration = d.iteration
    logger, log_frequency = d.logger, d.log_options.log_frequency

    def _evaluate(theta, want_grad: bool):
        """src/discretize.jl:567-598: term losses, iteration += 1, reweight, THEN the weighted sum -- the returned loss
        and gradient use the weights the reweighting just produced.  On a reweighting iteration that takes a loss-only
        evaluation first (a third of a step); every other iteration is a single fused call."""
        resample()
        state["calls"] += 1
        th = np.asarray(theta, dtype=dtype)
        stats = lambda i: eng.term_grad_stats_host(i, th)           # noqa: E731
        it = iteration[0] + 1 if d.self_increment else iteration[0]   # :574-576
        if adaloss.reweights_at(it):
            _, terms0, _ = eng.loss_grad_host(th, term_weights(), False)
            iteration[0] = it
            adaloss.update(it, terms0[:n_pde], terms0[n_pde:n_pde + n_bc], weights, term_grad_stats=stats)   # :578-580
            total, terms, grad = eng.loss_grad_host(th, term_weights(), want_grad)
        else:
            total, terms, grad = eng.loss_grad_host(th, term_weights(), want_grad)
            iteration[0] = it
            adaloss.update(it, terms[:n_pde], terms[n_pde:n_pde + n_bc], weights, term_grad_stats=stats)
        pde_losses, bc_losses = terms[:n_pde], terms[n_pde:n_pde + n_bc]
        if logger is not None and iteration[0] % log_frequency == 0:  # :600-645
            it = iteration[0]
            logvector(logger, pde_losses, "unweighted_loss/pde_losses", it)
            logvector(logger, bc_losses, "unweighted_loss/bc_losses", it)
            logvector(logger, weights["pde"] * pde_losses, "weighted_loss/weighted_pde_losses", it)
            logvector(logger, weights["bc"] * bc_losses, "weighted_loss/weighted_bc_losses", it)
            logscalar(logger, total, "weighted_loss/full_weighted_loss", it)
            logvector(logger, weights["pde"], "adaptive_loss/pde_loss_weights", it)
            logvector(logger, weights["bc"], "adaptive_loss/bc_loss_weights", it)
        return total, terms, grad

    def full_loss_function(theta, p=None) -> float:
        return _evaluate(theta, False)[0]

    def full_loss_gradient(theta, p=None):
        total, _, grad = _evaluate(theta, True)
        return total, grad

    def make_term_loss(i):
        def loss(theta):
            resample()
            _, terms, _ = eng.loss_grad_host(np.asarray(theta, dtype=dtype), term_weights(), False)
            return float(terms[i])
        return loss

    def make_datafree(i):
        def residual(points, theta):
            pts = np.asarray(points, dtype=dtype)
            if pts.ndim == 1:
                pts = pts.reshape(specs[i].dim, -1)
            old = point_sets[i]
            eng.set_points_host(i, augment(i, pts), None if quad_w[i] is None else np.ones(pts.shape[1], dtype=dtype))
            r = eng.term_residual_host(i, np.asarray(theta, dtype=dtype), pts.shape[1])
            if old is not None:
                upload(i, old, quad_w[i])
            return r.reshape(1, -1)
        return residual

    phis = [Phi(c, off, n_net + n_p, dtype, d.device) for c, off in zip(chains, offs)]
    phi = phis if d.multioutput else phis[0]
    lf = PINNLossFunctions(
        bc_loss_functions=[make_term_loss(n_pde + j) for j in range(n_bc)],
        pde_loss_functions=[make_term_loss(i) for i in range(n_pde)],
        full_loss_function=full_loss_function,
        additional_loss_function=add,
        datafree_pde_loss_functions=[make_datafree(i) for i in range(n_pde)],
        datafree_bc_loss_functions=[make_datafree(n_pde + j) for j in range(n_bc)],
        full_loss_gradient=full_loss_gradient,
    )
    rep = PINNRepresentation(
        eqs=eqs, bcs=bcs, domains=domains, eq_params=eq_params, defaults=defaults, default_p=default_p,
        param_estim=d.param_estim, additional_loss=add, adaloss=adaloss, depvars=vi.depvars, indvars=vi.indvars,
        dict_indvars=vi.dict_indvars, dict_depvars=vi.dict_depvars, dict_depvar_input=vi.dict_depvar_input,
        logger=logger, multioutput=d.multioutput, iteration=iteration, init_params=flat, flat_init_params=flat,
        phi=phi, derivative=None, strategy=strategy,
        pde_indvars=[lt.indvars for lt in pde_terms], bc_indvars=[lt.indvars for lt in bc_terms],
        symbolic_pde_loss_functions=pde_terms, symbolic_bc_loss_functions=bc_terms, loss_functions=lf, engine=eng,
        term_names=["pde_%d" % (i + 1) for i in range(n_pde)] + ["bc_%d" % (j + 1) for j in range(n_bc)]
        + ["dataset_pde_%d" % (j + 1) for j in range(n_ds[0])] + ["dataset_bc_%d" % (j + 1) for j in range(n_ds[1])]
        + ["l2_data_%s" % name for name in (vi.depvars if l2_sets else [])]
        + (["additional"] if add is not None else []))
    rep.point_sets = point_sets
    rep.resample = resample
    rep.quad_weights = quad_w
    rep.weights = weights

    def set_points(i: int, pts, w=None, n_global: Optional[int] = None):
        """Replace term i's point set ((d, N) coordinates; hoisted rows are appended here)."""
        point_sets[i] = np.asarray(pts, dtype=dtype)
        if world > 1 and n_global is None:
            raise ValueError("set_points on a sharded problem replaces this rank's shard: pass n_global (the term's "
                             "point count over all ranks) so the mean is scaled correctly")
        upload(i, point_sets[i], w, shard=False)
        if n_global is not None:
            eng.set_global_count(i, n_global)
    rep.set_points = set_points
    if bayes:
        # BayesianPINN (src/discretize.jl:653-757): the objective is the weighted LOG-LIKELIHOOD of zero residuals under
        # independent Gaussians, logpdf(MvNormal(r, sigma^2 I), 0) = -n/2 log(2 pi) - n log(sigma) - sum(r^2) / (2 sigma^2) per
        # term (get_points_loss_functions, src/training_strategies.jl:115-128) -- the sum of squares is n * mean(abs2, r),
        # which the fused kernel returns per term, and its theta-gradient is the engine's weighted gradient with weights
        # -W n / (2 sigma^2).  As in the reference the per-group log-likelihoods are SUMMED before the weight vector
        # multiplies them (:682-738): every weight of a group scales the whole group sum.  Dataset terms join their
        # group's sum; L2LossData (data=True) is the sampler's and is not part of full_loss_function.
        n_k = np.array([point_sets[i].shape[1] for i in range(n_main)], dtype=np.float64)
        counts = (n_pde, n_bc, n_ds[0], n_ds[1])
        rep.loglik_weights = lambda allstd, data=False: _loglik_weights_all(weights, n_k, counts, allstd, data)

        def _loglik(theta, allstd, want_grad):
            stdpdes, stdbcs, stdextra = allstd
            c, const = rep.loglik_weights(allstd)
            th = np.asarray(theta, dtype=dtype)
            has_add = isinstance(add, DataLoss)
            if has_add:
                _, t0, _ = eng.loss_grad_host(th, np.concatenate([c, [0.0]]), False)
                A = float(t0[-1])                  # the additional loss VALUE is one observation of Normal(0, stdextra) (:745)
                c_all = np.concatenate([c, [-weights["add"][0] * A / float(stdextra) ** 2]])
            else:
                c_all = c
            total, terms, grad = eng.loss_grad_host(th, c_all, want_grad)
            ll = const + float(np.dot(c, np.asarray(terms[:n_main], dtype=np.float64)))
            if has_add:
                s_e = float(stdextra)
                ll += weights["add"][0] * (-np.log(s_e * np.sqrt(2.0 * np.pi)) - A * A / (2.0 * s_e ** 2))
            if d.self_increment:
                iteration[0] += 1
            return ll, grad

        lf.full_loss_function = lambda theta, allstd: _loglik(theta, allstd, False)[0]
        lf.full_loss_gradient = lambda theta, allstd: _loglik(theta, allstd, True)
    return rep


def _loglik_weights(weights, n_k: np.ndarray, n_pde: int, allstd):
    """Per-term weights c_k = -W n_k / (2 σ_k²) and the constant Σ W (-n_k/2 log 2π - n_k log σ_k) of the BayesianPINN
    log-likelihood Σ_k c_k L_k + const, L_k = mean(abs2, r_k) (src/training_strategies.jl:115-128; every weight of a
    group scales the whole group sum, src/discretize.jl:682-738)."""
    stdpdes, stdbcs = allstd[0], allstd[1]
    n_bc = n_k.size - n_pde
    sig = np.concatenate([np.asarray(stdpdes, dtype=np.float64), np.asarray(stdbcs, dtype=np.float64)])
    if sig.shape != (n_pde + n_bc,):
        raise ValueError("allstd: need %d pde and %d bc standard deviations" % (n_pde, n_bc))
    Wg = np.concatenate([np.full(n_pde, weights["pde"].sum()), np.full(n_bc, weights["bc"].sum())])
    c = -Wg * n_k / (2.0 * sig ** 2)
    const = float(np.sum(Wg * (-0.5 * n_k * np.log(2.0 * np.pi) - n_k * np.log(sig))))
    return c, const


def _loglik_weights_all(weights, n_k: np.ndarray, counts, allstd, data: bool = False):
    """Weights c and constant of the BayesianPINN log-likelihood over all its terms.  n_k holds the point counts of the
    grid pde and bc terms, the dataset pde and bc terms (counts: the four numbers) and then the L2 data terms.

    - grid terms: ``_loglik_weights``;
    - dataset term j: c = -W n / (2 σ²) with its group's weight sum W and σ = stdpdes[j] (stdbcs[j]), plus
      W (-n/2 log 2π - n log σ) in the constant (src/training_strategies.jl:115-128, src/discretize.jl:699-717);
    - L2 data term i (``data``; zero otherwise): c = -n / (2 l2std[i]²) and -n/2 log 2π - n log l2std[i], no adaptive
      weight (L2LossData, ext/bpinn/PDE_BPINN.jl:147-180)."""
    n_pde, n_bc, n_dp, n_db = counts
    c, const = _loglik_weights(weights, n_k[:n_pde + n_bc], n_pde, allstd)
    o = n_pde + n_bc
    nd, nl = n_k[o:o + n_dp + n_db], n_k[o + n_dp + n_db:]
    sig = np.concatenate([np.asarray(allstd[0], dtype=np.float64)[:n_dp],
                          np.asarray(allstd[1], dtype=np.float64)[:n_db]])
    Wg = np.concatenate([np.full(n_dp, weights["pde"].sum()), np.full(n_db, weights["bc"].sum())])
    c_d = -Wg * nd / (2.0 * sig ** 2)
    const += float(np.sum(Wg * (-0.5 * nd * np.log(2.0 * np.pi) - nd * np.log(sig))))
    c_l = np.zeros(nl.size)
    if data and nl.size:
        l2 = np.asarray(allstd[2], dtype=np.float64).reshape(-1)
        if l2.shape != nl.shape:
            raise ValueError("allstd: need %d l2std values, one per dependent variable" % nl.size)
        c_l = -nl / (2.0 * l2 ** 2)
        const += float(np.sum(-0.5 * nl * np.log(2.0 * np.pi) - nl * np.log(l2)))
    return np.concatenate([c, c_d, c_l]), const


def _bayes_dataset(dataset, vi: VarInfo):
    """BayesianPINN's ``dataset = [dataset_pde, dataset_bc]``, each None or a list with one n × (1 + d_k) array per
    dependent variable (d_k: its inputs).  Returns the two lists as float64 arrays (or None)."""
    if len(dataset) != 2:
        raise ValueError("BayesianPINN: dataset points: expected dataset = [dataset_pde, dataset_bc], got %d entries"
                         % len(dataset))
    out = []
    for what, ds in zip(("dataset_pde", "dataset_bc"), dataset):
        if ds is None:
            out.append(None)
            continue
        if not isinstance(ds, (list, tuple)) or len(ds) != len(vi.depvars):
            raise ValueError("BayesianPINN: dataset points: %s must be None or a list of %d arrays, one per dependent "
                             "variable %s, each n × (1 + inputs) with the observed values in column 1"
                             % (what, len(vi.depvars), vi.depvars))
        mats = []
        for name, m in zip(vi.depvars, ds):
            a = np.asarray(m, dtype=np.float64)
            cols = 1 + len(vi.dict_depvar_input[name])
            if a.ndim != 2 or a.shape[0] < 1 or a.shape[1] != cols:
                raise ValueError("BayesianPINN: dataset points: %s for %s has shape %s, expected n × %d"
                                 % (what, name, a.shape, cols))
            mats.append(a)
        out.append(mats)
    return out


@dataclass
class OptimizationFunction:
    """``OptimizationFunction(f; grad)``: ``f(θ, p)`` and an explicit gradient
    ``grad(θ, p) -> (f, ∇f)`` that replaces AutoZygote (src/discretize.jl:778)."""
    f: Callable
    grad: Callable


@dataclass
class OptimizationProblem:
    f: OptimizationFunction
    u0: np.ndarray
    p: object = None
    representation: Optional[PINNRepresentation] = None


def discretize(pde_system: PDESystem, discretization: PhysicsInformedNN, rank: int = 0,
               world: int = 1) -> OptimizationProblem:
    """``discretize(pde_system, discretization)`` (src/discretize.jl:776-780)."""
    rep = symbolic_discretize(pde_system, discretization, rank, world)
    lf = rep.loss_functions
    return OptimizationProblem(OptimizationFunction(lf.full_loss_function, lf.full_loss_gradient),
                               rep.flat_init_params.copy(), None, rep)


@dataclass
class Solution:
    u: np.ndarray
    objective: float
    iterations: int
    retcode: str = "Default"     # quasi-Newton runs: "Success", "MaxIters", "Failure" or "Terminated" (by the callback)


def _host_resampled(rep) -> bool:
    return (isinstance(rep.strategy, StochasticTraining) and not rep.strategy.device_sampler) or \
           (isinstance(rep.strategy, QuasiRandomTraining) and rep.strategy.resampling and
            not rep.strategy.device_sampler) if rep is not None else True


_DEVICE_LOOP_SETS = ("point sets that live on the device: Grid, Quadrature, non-resampled QuasiRandom, or "
                     "StochasticTraining(..., device_sampler=True)")


def _linesearch_kind(ls) -> int:
    if isinstance(ls, HagerZhang) and ls == HagerZhang():
        return _eng.LS_HAGERZHANG
    if isinstance(ls, BackTracking) and ls == BackTracking():
        return _eng.LS_BACKTRACKING
    raise ValueError("linesearch must be HagerZhang() or BackTracking() with their default parameters, got %r" % (ls,))


def _qn_run(eng: Engine, u0: np.ndarray, opt, ls_kind: int, maxiters: int, callback: Optional[Callable], term_w):
    """The device quasi-Newton run from u0: one ``maxiters`` call without a callback, one iteration per call with one.
    Returns (θ, objective, iterations, evaluations, retcode)."""
    if isinstance(opt, LBFGS):
        eng.qn_begin(u0, _eng.QN_LBFGS, m=opt.m, linesearch=ls_kind, weights=term_w)
    else:
        eng.qn_begin(u0, _eng.QN_BFGS, linesearch=ls_kind, initial_stepnorm=opt.initial_stepnorm, weights=term_w)
    f, _, status, iters, evals = eng.qn_iterate(0)
    retcode = None
    if callback is None:
        f, _, status, iters, evals = eng.qn_iterate(maxiters)
    else:
        while status == _eng.QN_RUNNING and iters < maxiters:
            f, _, status, iters, evals = eng.qn_iterate(1)
            if callback({"iter": iters, "u": eng.qn_theta()}, f):
                retcode = "Terminated"
                break
    if retcode is None:
        retcode = {_eng.QN_CONVERGED: "Success", _eng.QN_LS_FAILED: "Failure"}.get(status, "MaxIters")
    return eng.qn_theta(), f, iters, evals, retcode


def _solve_quasi_newton(prob: OptimizationProblem, opt, maxiters: int, callback: Optional[Callable]) -> Solution:
    """BFGS / L-BFGS with theta, the gradient and the curvature history on the device (pinn_qn_*); the line search runs
    on the host with one 16-byte read-back per evaluation."""
    rep = prob.representation
    if _host_resampled(rep):
        raise ValueError("BFGS / LBFGS need " + _DEVICE_LOOP_SETS)
    if not isinstance(rep.adaloss, NonAdaptiveLoss):
        raise ValueError("BFGS / LBFGS need fixed loss weights (NonAdaptiveLoss): an adaptive loss would change the "
                         "objective between the line search's trial points")
    ls_kind = _linesearch_kind(opt.linesearch)
    if isinstance(rep.strategy, QuasiRandomTraining) and not rep.strategy.device_sampler:
        rep.resample()                               # non-resampled QuasiRandom places its points at the first loss call
    w = rep.weights
    term_w = np.concatenate([w["pde"], w["bc"]] + ([w["add"]] if rep.additional_loss is not None else []))
    theta, f, iters, evals, retcode = _qn_run(rep.engine, prob.u0, opt, ls_kind, maxiters, callback, term_w)
    rep.iteration[0] += evals                        # one loss call per evaluation, as the reference counts them
    return Solution(theta.astype(prob.u0.dtype), f, iters, retcode)


class _DefaultMaxiters(int):
    """``solve``'s default ``maxiters`` (100 for an OptimizationProblem); an ODEProblem needs it given"""


_MAXITERS_DEFAULT = _DefaultMaxiters(100)


def solve(prob: OptimizationProblem, opt: Union[Adam, LBFGS, BFGS], maxiters: int = _MAXITERS_DEFAULT, callback: Optional[Callable] = None,
          device_loop: bool = False, chunk: int = 50, **ode_kwargs) -> Solution:
    """Minimal stand-in for ``Optimization.solve(prob, opt; maxiters, callback)``.

    ``LBFGS()`` / ``BFGS()``: the device-resident quasi-Newton driver (pinn_qn_*), whatever ``device_loop`` says; one
    ``maxiters`` call without a callback, one iteration per call with one (the callback sees θ and the loss after every
    accepted step, and returning True halts the run).  Point sets as for ``device_loop=True``; the loss weights must be
    fixed (NonAdaptiveLoss).

    Default: a host Adam loop that calls the engine's loss+gradient once per iteration.
    ``device_loop=True`` (fixed point sets, or StochasticTraining with the device-side sampler, which then draws fresh
    points before every step): theta, m, v stay on the device and the Adam update is fused into the gradient reduction
    (pinn_adam_iterate); the callback sees the loss every `chunk` steps.

    ``solve(prob::ODEProblem, alg::NNODE; maxiters, dt, abstol, saveat, ...)`` trains an NNODE (ode.py) and takes the
    keywords of ``ode.solve``.  ``solve(prob::ODEProblem, alg::BNNODE; saveat)`` samples the Bayesian ODE posterior
    (bpinn_ode.py) and returns a BPINNsolution.  ``solve(prob::SDEProblem, alg::NNSDE; maxiters, dt, abstol, saveat,
    ...)`` trains an NNSDE (sde.py) and returns an SDEsol.  ``solve(prob::SDEProblem, alg::SDEPINN; maxiters = 200,
    verbose)`` trains the density of the SDE's Fokker-Planck equation (sde_weak.py) and returns ``(res, phi)``.
    ``solve(prob::DAEProblem, alg::NNDAE; maxiters, dt, abstol, saveat, ...)`` trains an NNDAE (dae.py) and returns a
    DAESolution."""
    from .bpinn_ode import BNNODE, solve_bnnode
    from .dae import DAEProblem, solve_nndae
    from .ode import ODEProblem, solve_nnode
    from .sde import SDEProblem, solve_nnsde
    from .sde_weak import SDEPINN, solve_sdepinn
    if isinstance(prob, SDEProblem) and isinstance(opt, SDEPINN):
        if callback is not None or chunk != 50 or device_loop:
            raise TypeError("solve(::SDEProblem, ::SDEPINN) takes no callback, chunk or device_loop")
        return solve_sdepinn(prob, opt, maxiters=200 if maxiters is _MAXITERS_DEFAULT else maxiters, **ode_kwargs)
    if isinstance(prob, DAEProblem):
        if callback is not None or chunk != 50:
            raise TypeError("solve(::DAEProblem, ::NNDAE) takes no callback or chunk: it stops at abstol")
        if maxiters is _MAXITERS_DEFAULT:
            raise TypeError("solve(::DAEProblem, ::NNDAE) needs maxiters")
        return solve_nndae(prob, opt, maxiters=maxiters, device_loop=device_loop, **ode_kwargs)
    if isinstance(prob, SDEProblem):
        if callback is not None or chunk != 50:
            raise TypeError("solve(::SDEProblem, ::NNSDE) takes no callback or chunk: it stops at abstol")
        if maxiters is _MAXITERS_DEFAULT:
            raise TypeError("solve(::SDEProblem, ::NNSDE) needs maxiters")
        return solve_nnsde(prob, opt, maxiters=maxiters, device_loop=device_loop, **ode_kwargs)
    if isinstance(prob, ODEProblem) and isinstance(opt, BNNODE):
        if callback is not None or chunk != 50 or device_loop or maxiters is not _MAXITERS_DEFAULT:
            raise TypeError("solve(::ODEProblem, ::BNNODE) takes no maxiters, callback, chunk or device_loop")
        return solve_bnnode(prob, opt, **ode_kwargs)
    if isinstance(prob, ODEProblem):
        if callback is not None or chunk != 50:
            raise TypeError("solve(::ODEProblem, ::NNODE) takes no callback or chunk: it stops at abstol")
        if maxiters is _MAXITERS_DEFAULT:
            raise TypeError("solve(::ODEProblem, ::NNODE) needs maxiters")
        return solve_nnode(prob, opt, maxiters=maxiters, device_loop=device_loop, **ode_kwargs)
    if ode_kwargs:
        raise TypeError("solve() got unexpected keyword arguments %s" % sorted(ode_kwargs))
    if isinstance(opt, (LBFGS, BFGS)):
        return _solve_quasi_newton(prob, opt, maxiters, callback)
    rep = prob.representation
    if device_loop:
        if _host_resampled(rep):
            raise ValueError("device_loop needs " + _DEVICE_LOOP_SETS)
        eng = rep.engine
        eng.adam_begin(prob.u0, opt.lr, opt.beta1, opt.beta2, opt.eps)
        done, obj = 0, float("nan")
        adaloss, weights, iteration = rep.adaloss, rep.weights, rep.iteration
        n_pde, n_bc = len(rep.eqs), len(rep.bcs)

        def term_w():
            return np.concatenate([weights["pde"], weights["bc"]] + ([weights["add"]] if rep.additional_loss is not None else []))

        adaptive = not isinstance(adaloss, NonAdaptiveLoss)

        def reweight(it):
            """what full_loss_function does at iteration `it` before forming the weighted sum (src/discretize.jl:574-588):
            theta is read back once, the term losses are evaluated and handed to the adaptive loss"""
            th = eng.adam_theta()
            _, terms0, _ = eng.loss_grad_host(th, term_w(), False)
            adaloss.update(it, terms0[:n_pde], terms0[n_pde:n_pde + n_bc], weights,
                           term_grad_stats=lambda i: eng.term_grad_stats_host(i, th))

        if adaptive and (iteration[0] + 1) % adaloss.reweight_every != 0:
            reweight(iteration[0] + 1)          # the reference's closures see every iteration: SoftAdapt / ReLoBRaLo seed here
        while done < maxiters:
            n = min(chunk, maxiters - done)
            if adaptive:
                # iterations before the next reweighting run on the device with the current weights; the reweighting
                # iteration itself updates the weights first and takes its step with the new ones
                nxt = (iteration[0] // adaloss.reweight_every + 1) * adaloss.reweight_every
                if nxt - iteration[0] == 1:
                    reweight(nxt)
                    n = 1
                else:
                    n = min(n, nxt - iteration[0] - 1)
            obj, _ = eng.adam_iterate(n, term_w())
            done += n
            iteration[0] += n
            if callback is not None and callback({"iter": done, "u": None}, obj):
                break
        return Solution(eng.adam_theta(), obj, done)
    u = prob.u0.astype(np.float64).copy()
    m, v = np.zeros_like(u), np.zeros_like(u)
    obj = float("nan")
    it = 0
    for it in range(1, maxiters + 1):
        obj, g = prob.f.grad(u.astype(prob.u0.dtype), prob.p)
        g = g.astype(np.float64)
        m = opt.beta1 * m + (1 - opt.beta1) * g
        v = opt.beta2 * v + (1 - opt.beta2) * g * g
        u -= opt.lr * (m / (1 - opt.beta1 ** it)) / (np.sqrt(v / (1 - opt.beta2 ** it)) + opt.eps)
        if callback is not None and callback({"iter": it, "u": u}, obj):
            break
    return Solution(u.astype(prob.u0.dtype), obj, it)


# ---- Bayesian PINN sampling (reference ext/bpinn/PDE_BPINN.jl) --------------------------------------------------------
@dataclass
class HMC:
    """``AdvancedHMC.HMC(ϵ, n_leapfrog)``: fixed-length trajectories.  As in the reference, ``ϵ`` is not used: the
    initial step size comes from ``find_good_stepsize``."""
    step_size: float = 0.1
    n_leapfrog: int = 30


class StanHMCAdaptor:
    """``Adaptor = StanHMCAdaptor``: dual averaging of the step size and Stan's windowed mass-matrix estimate."""


class NoAdaptation:
    """``Adaptor = NoAdaptation``: step size and metric stay as found."""


class DiagEuclideanMetric:
    """``Metric = DiagEuclideanMetric``: diagonal M⁻¹, adapted by the Stan adaptor."""


class UnitEuclideanMetric:
    """``Metric = UnitEuclideanMetric``: M = I."""


class Leapfrog:
    """``Integrator = Leapfrog``."""


@dataclass(frozen=True)
class Normal:
    """``Distributions.Normal(μ, σ)``, a prior of an equation parameter (``param``)."""
    mu: float = 0.0
    sigma: float = 1.0

    def params(self):
        return (self.mu, self.sigma)

    def pdf(self, x: float) -> float:
        """``Distributions.pdf``"""
        return float(np.exp(-0.5 * ((x - self.mu) / self.sigma) ** 2) / (self.sigma * np.sqrt(2.0 * np.pi)))


@dataclass(frozen=True)
class LogNormal:
    """``Distributions.LogNormal(μ, σ)``: log x ~ Normal(μ, σ); ``params`` are (μ, σ) of log x, not the mean."""
    mu: float = 0.0
    sigma: float = 1.0

    def params(self):
        return (self.mu, self.sigma)

    def pdf(self, x: float) -> float:
        """``Distributions.pdf``: 0 for x <= 0"""
        if x <= 0:
            return 0.0
        return float(np.exp(-0.5 * ((np.log(x) - self.mu) / self.sigma) ** 2) / (x * self.sigma * np.sqrt(2.0 * np.pi)))


@dataclass(frozen=True)
class Uniform:
    """``Distributions.Uniform(a, b)`` on [a, b]."""
    a: float = 0.0
    b: float = 1.0

    def params(self):
        return (self.a, self.b)


_PRIOR_KINDS = {Normal: _eng.HMC_PRIOR_NORMAL, LogNormal: _eng.HMC_PRIOR_LOGNORMAL, Uniform: _eng.HMC_PRIOR_UNIFORM}


def _tail_priors(param, who: str = "ahmc_bayesian_pinn_pde") -> List[tuple]:
    """The device's table for θ.p: (kind, a, b) per parameter, in the reference's order -- priorlogpdf applies
    ``param[length(θ) - i + 1]`` to θ[i] (ext/bpinn/PDE_BPINN.jl:194-196), so θ.p[k] gets param[end - k].  ``who``
    names the calling sampler in the refusals."""
    out = []
    for prior in param:
        kind = _PRIOR_KINDS.get(type(prior))
        if kind is None:
            raise ValueError("%s: prior %r is not supported (Normal, LogNormal or Uniform)" % (who, prior))
        a, b = (float(v) for v in prior.params())
        if not (np.isfinite(a) and np.isfinite(b)) or (kind == _eng.HMC_PRIOR_UNIFORM and not a < b) or \
                (kind != _eng.HMC_PRIOR_UNIFORM and not b > 0.0):
            raise ValueError("%s: prior %r: needs finite parameters with σ > 0 (Uniform: a < b)" % (who, prior))
        out.append((kind, a, b))
    return out[::-1]


def _initial_theta(flat_init_params, param) -> np.ndarray:
    """float64 θ0: the network part of flat_init_params, then θ.p[k] = params(param[k])[1] in FORWARD order
    (ext/bpinn/PDE_BPINN.jl:476, :499): Normal's μ, LogNormal's μ of log x, Uniform's a."""
    th = np.array(flat_init_params, dtype=np.float64)
    th[th.size - len(param):] = [float(p.params()[0]) for p in param]
    return th


@dataclass
class BPINNstats:
    """``BPINNstats(mcmc_chain, samples, statistics)``: ``chain`` / ``samples`` are the [draw_samples, n_θ] draws,
    ``statistics`` maps each AdvancedHMC statistic (step_size, acceptance_rate, is_accept, log_density,
    hamiltonian_energy, hamiltonian_energy_error, numerical_error, is_adapt) to its [draw_samples] values."""
    chain: np.ndarray
    samples: np.ndarray
    statistics: Dict[str, np.ndarray]


@dataclass
class BPINNsolution:
    """``BPINNsolution(original, ensemblesol, estimated_nn_params, estimated_de_params, timepoints)``:
    ``ensemblesol[k]`` is φ_k on ``timepoints[k]`` ((d_k, n_points), first input fastest) for each of the last
    ``numensemble + 1`` samples, an array [numensemble + 1, n_points]; ``estimated_nn_params[k]`` holds network k's
    parameters in those samples."""
    original: BPINNstats
    ensemblesol: List[np.ndarray]
    estimated_nn_params: List[np.ndarray]
    estimated_de_params: list
    timepoints: List[np.ndarray]


def pmean(x) -> np.ndarray:
    """MonteCarloMeasurements' ``pmean``: the mean over samples (axis 0) of an ensemble array."""
    return np.mean(np.asarray(x, dtype=np.float64), axis=0)


_DEFAULT_ADAPTOR = {"Adaptor": StanHMCAdaptor, "Metric": DiagEuclideanMetric, "targetacceptancerate": 0.8}


def _hmc_adaptation(Adaptorkwargs, nchains: int, who: str):
    """The Adaptor / Metric / nchains options of the HMC samplers, checked: (adaptor, metric, target acceptance) for
    Engine.hmc_begin"""
    ak = dict(_DEFAULT_ADAPTOR, **(Adaptorkwargs or {}))
    if ak["Adaptor"] not in (StanHMCAdaptor, NoAdaptation):
        raise ValueError("%s: Adaptor %r is not implemented (StanHMCAdaptor or NoAdaptation)" % (who, ak["Adaptor"]))
    if ak["Metric"] not in (DiagEuclideanMetric, UnitEuclideanMetric):
        raise ValueError("%s: Metric %r is not implemented; DenseEuclideanMetric is not supported "
                         "(DiagEuclideanMetric or UnitEuclideanMetric)" % (who, ak["Metric"]))
    if nchains != 1:
        raise ValueError("%s: nchains = %r; one chain per call is supported" % (who, nchains))
    return (_eng.HMC_ADAPT_STAN if ak["Adaptor"] is StanHMCAdaptor else _eng.HMC_ADAPT_NONE,
            _eng.HMC_METRIC_DIAG if ak["Metric"] is DiagEuclideanMetric else _eng.HMC_METRIC_UNIT,
            float(ak["targetacceptancerate"]))


def ahmc_bayesian_pinn_pde(pde_system: PDESystem, discretization: BayesianPINN, *, draw_samples: int = 1000,
                           bcstd=(0.01,), l2std=(0.05,), phystd=(0.05,), phynewstd=(0.05,), priorsNNw=(0.0, 2.0),
                           param=(), nchains: int = 1, Kernel=None, Adaptorkwargs=None, Integratorkwargs=None,
                           saveats=(1 / 10,), numensemble: Optional[int] = None, Dict_differentials=None,
                           progress: bool = False, verbose: bool = False, seed: int = 0) -> BPINNsolution:
    """``ahmc_bayesian_pinn_pde(pde_system, discretization; draw_samples, bcstd, phystd, priorsNNw, saveats, ...)``
    (reference ext/bpinn/PDE_BPINN.jl:371-635): Hamiltonian Monte Carlo over the network parameters of a BayesianPINN,
    target ``full_loss_function(θ, [phystd, bcstd, l2std]) + log N(θ; μ_p, σ_p² I)`` with ``priorsNNw = (μ_p, σ_p)``.

    Defaults as the reference: ``HMC(0.1, 30)`` started at ``find_good_stepsize``, Stan adaptation (dual averaging to
    acceptance 0.8, diagonal mass matrix) over the first ``min(draw_samples ÷ 10, 1000)`` transitions, warm-up samples
    kept.  The chain runs on the device (``pinn_hmc_*``); ``seed`` keys its Philox streams (the reference uses the global
    RNG).  ``phynewstd`` is accepted and unused (it belongs to ``Dict_differentials``).

    Parameter estimation (``BayesianPINN(...; param_estim = true, dataset)`` with ``param = [prior, ...]``, one
    Normal / LogNormal / Uniform per equation parameter): the target gains L2LossData, the observations' Gaussian
    log-likelihood with standard deviations ``l2std`` (one per dependent variable), and θ.p gets the priors of
    ``param`` in REVERSED order, as the reference's priorlogpdf applies them; θ.p starts at ``params(param[k])[1]``
    (LogNormal: μ of log x).  ``estimated_de_params[k]`` holds θ.p[k] over the ensemble's samples.
    Not supported (refused with a message): NUTS / HMCDA kernels, ``DenseEuclideanMetric``, jittered / tempered
    leapfrog, several chains, ``Dict_differentials`` and an ``additional_loss``."""
    Kernel = HMC() if Kernel is None else Kernel
    ik = dict({"Integrator": Leapfrog}, **(Integratorkwargs or {}))
    if not isinstance(Kernel, HMC):
        raise ValueError("ahmc_bayesian_pinn_pde: Kernel %r is not implemented; the device sampler runs HMC(ϵ, n_leapfrog) "
                         "(NUTS and HMCDA are not supported)" % (Kernel,))
    adaptor, metric, target_accept = _hmc_adaptation(Adaptorkwargs, nchains, "ahmc_bayesian_pinn_pde")
    if ik["Integrator"] is not Leapfrog:
        raise ValueError("ahmc_bayesian_pinn_pde: Integrator %r is not implemented; JitteredLeapfrog / TemperedLeapfrog "
                         "are not supported (Leapfrog)" % (ik["Integrator"],))
    if not isinstance(discretization, BayesianPINN):
        raise TypeError("ahmc_bayesian_pinn_pde: expected a BayesianPINN discretization")
    param_estim = discretization.pinn.param_estim
    if len(param) > 0 and not param_estim:
        raise ValueError("ahmc_bayesian_pinn_pde: parameter estimation: `param` priors need "
                         "BayesianPINN(...; param_estim = true)")
    if param_estim and len(param) == 0:       # the reference throws UndefVarError(:param) (PDE_BPINN.jl:454-455)
        raise ValueError("ahmc_bayesian_pinn_pde: parameter estimation (param_estim = true) needs `param`, one prior "
                         "per equation parameter")
    if Dict_differentials is not None:
        raise ValueError("ahmc_bayesian_pinn_pde: Dict_differentials (the data-collocation loss) is not supported")
    if discretization.pinn.additional_loss is not None:
        raise ValueError("ahmc_bayesian_pinn_pde: an additional_loss enters the log-likelihood with a weight that depends "
                         "on its value, two evaluations per gradient; the device sampler does not support it")
    tail = []
    if param_estim:
        if all(ds is None for ds in discretization.dataset):      # UndefVarError(:dataset) (:456-457)
            raise ValueError("ahmc_bayesian_pinn_pde: parameter estimation (param_estim = true) needs a dataset")
        n_dv = len(get_vars(pde_system.ivs, pde_system.dvs).depvars)
        if len(l2std) != n_dv:                                     # :458-459
            raise ValueError("ahmc_bayesian_pinn_pde: L2 stds length must match number of dependant variables "
                             "(%d l2std values, %d dependent variables)" % (len(l2std), n_dv))
        if len(param) != len(pde_system.ps):
            raise ValueError("ahmc_bayesian_pinn_pde: parameter estimation: %d priors in `param` for the %d equation "
                             "parameters %s" % (len(param), len(pde_system.ps), [str(p) for p in pde_system.ps]))
        tail = _tail_priors(param)
    rep = symbolic_discretize(pde_system, discretization)
    if len(rep.domains) != len(saveats):
        raise ValueError("Number of independent variables must match saveat inference discretization steps")
    draw_samples = int(draw_samples)
    numensemble = int(np.floor(draw_samples / 3)) if numensemble is None else int(numensemble)
    if draw_samples < 1 or not 0 <= numensemble < draw_samples:
        raise ValueError("ahmc_bayesian_pinn_pde: need draw_samples >= 1 and 0 <= numensemble < draw_samples")
    allstd = [phystd, bcstd, l2std]
    c, const = rep.loglik_weights(allstd, data=True)
    mu_p, sd_p = float(priorsNNw[0]), float(priorsNNw[1])
    n_adapts = min(draw_samples // 10, 1000)
    eng = rep.engine
    ninv = len(tail)
    theta0 = _initial_theta(rep.flat_init_params, param)
    n_net = theta0.size - ninv
    eps0 = eng.hmc_begin(theta0, n_leapfrog=Kernel.n_leapfrog, adaptor=adaptor, metric=metric, n_adapts=n_adapts,
                         target_accept=target_accept, step_size=0.0,
                         prior_mean=mu_p, prior_std=sd_p, seed=seed, weights=c, ll_const=const,
                         tail_priors=tail if ninv else None)
    if verbose:
        print("Initial step size %g; current physics log-likelihood %g"
              % (eps0, rep.loss_functions.full_loss_function(theta0, allstd)))
        if ninv:
            c_phys, const_phys = rep.loglik_weights(allstd)
            _, terms, _ = eng.loss_grad_host(theta0.astype(rep.flat_init_params.dtype), c, False)
            sse = float(np.dot(c - c_phys, np.asarray(terms, dtype=np.float64))) + (const - const_phys)
            print("Current SSE against dataset Log-likelihood : %g" % sse)
    samples, st = eng.hmc_iterate(draw_samples)
    statistics = {name: st[:, j].copy() for j, name in enumerate(_eng.HMC_STATS)}
    if verbose:
        print("Sampling complete: acceptance rate %.3f" % float(np.mean(statistics["acceptance_rate"])))

    # inference (PDE_BPINN.jl:222-312): the last numensemble + 1 samples on the saveat grid of each network's inputs
    kept = samples[draw_samples - numensemble - 1:]
    ranges = {str(dm.variables): _julia_range(dm.domain.lo, float(h), dm.domain.hi) for dm, h in zip(rep.domains, saveats)}
    phis = rep.phi if rep.multioutput else [rep.phi]
    timepoints, ensemble, nn_params = [], [], []
    for name, ph in zip(rep.depvars, phis):
        tp = _product_columns([ranges[v] for v in rep.dict_depvar_input[name]])
        timepoints.append(tp)
        ensemble.append(np.stack([np.asarray(ph(tp, th), dtype=np.float64).reshape(-1) for th in kept]))
        nn_params.append(kept[:, ph.theta_offset:ph.theta_offset + ph.chain.n_params].copy())
    de_params = [kept[:, n_net + k].copy() for k in range(ninv)] if ninv else [None]
    return BPINNsolution(BPINNstats(samples, samples, statistics), ensemble, nn_params, de_params, timepoints)
