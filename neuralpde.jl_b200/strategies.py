"""Training strategies: the collocation point sets and the per-term reduction.

Mirrors reference src/training_strategies.jl (GridTraining :13, StochasticTraining :235,
QuasiRandomTraining :311, QuadratureTraining :412) and the set construction in
src/discretize.jl:185-324.  Only the *data* side lives here; the reduction
``mean(abs2, residual)`` runs inside the CUDA kernel.
"""
from __future__ import annotations

import itertools
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np

from .symbolic import Equation, VarDomain, VarInfo, get_argument


class AbstractTrainingStrategy:
    pass


@dataclass
class GridTraining(AbstractTrainingStrategy):
    """``GridTraining(dx)``: dx scalar or one per domain (training_strategies.jl:13-19)."""
    dx: object


@dataclass
class StochasticTraining(AbstractTrainingStrategy):
    """``StochasticTraining(points; bcs_points = points)`` (training_strategies.jl:235-240)."""
    points: int
    bcs_points: Optional[int] = None
    seed: int = 0          # the reference uses the global RNG; a seed makes runs reproducible
    device_sampler: bool = False   # draw on the GPU (Philox, pinn_set_sampler / pinn_resample) instead of host rand + upload

    def __post_init__(self):
        if self.bcs_points is None:
            self.bcs_points = self.points


@dataclass
class QuasiRandomTraining(AbstractTrainingStrategy):
    """``QuasiRandomTraining(points; bcs_points, resampling, minibatch)``
    (training_strategies.jl:311-334).  Sampling: a scrambled Sobol sequence
    (``sampling_alg = LatinHypercubeSample()`` by default in the reference; any
    QuasiMonteCarlo sampler is allowed there)."""
    points: int
    bcs_points: Optional[int] = None
    resampling: bool = True
    minibatch: int = 0
    seed: int = 0
    device_sampler: bool = False   # resampling on the GPU: a Latin hypercube sample per call (pinn_set_sampler_ex, kind LHS)

    def __post_init__(self):
        if self.bcs_points is None:
            self.bcs_points = self.points
        if self.device_sampler and not self.resampling:
            raise ValueError("QuasiRandomTraining(device_sampler=True) resamples on every call: it needs resampling=True")


@dataclass
class WeightedIntervalTraining(AbstractTrainingStrategy):
    """``WeightedIntervalTraining(weights, points)`` (training_strategies.jl, NNODE only): the time span is cut into
    ``len(weights)`` equal sub-intervals and sub-interval i gets ``trunc(points * w_i)`` uniform points, w normalised
    to sum 1.  The points are drawn once (src/ode_solve.jl:297-316).  ``seed`` fixes the draw (the reference uses the
    global RNG)."""
    weights: Sequence[float]
    points: int
    seed: int = 0

    def sample(self, t0: float, t1: float) -> np.ndarray:
        w = np.asarray(self.weights, dtype=np.float64)
        w = w / w.sum()
        h = (t1 - t0) / w.size
        rng = np.random.default_rng(self.seed)
        return np.concatenate([rng.random(int(self.points * wi)) * h + t0 + i * h for i, wi in enumerate(w)])


@dataclass
class QuadratureTraining(AbstractTrainingStrategy):
    """Fixed-node tensor Gauss-Legendre quadrature of ``r^2`` over the domain:
    ``loss = sum_i w_i r(x_i)^2 / area``.

    The reference integrates ``r^2`` adaptively with CubatureJLh on the CPU
    (training_strategies.jl:451-481); the adaptive host loop is out of scope (SURVEY section 2
    row 12, section 8 A5), the *fixed-node* form is what shards over GPUs (BASELINE config 4)."""
    nodes_per_dim: int = 16
    bc_nodes_per_dim: Optional[int] = None

    def __post_init__(self):
        if self.bc_nodes_per_dim is None:
            self.bc_nodes_per_dim = self.nodes_per_dim


# ---- Grid (reference src/discretize.jl:185-241) ------------------------------------------------------
def _julia_range(lo: float, dx: float, hi: float) -> np.ndarray:
    """``lo:dx:hi`` (Julia StepRangeLen semantics: the last element never exceeds hi)."""
    n = int(np.floor((hi - lo) / dx + 1e-10)) + 1
    return lo + dx * np.arange(n, dtype=np.float64)


def _product_columns(spans: Sequence[np.ndarray]) -> np.ndarray:
    """``reduce(hcat, vec(map(collect, Iterators.product(span...))))``: (d, N), first variable fastest."""
    if len(spans) == 0:
        return np.zeros((0, 1))
    grids = np.meshgrid(*spans, indexing="ij")
    return np.stack([g.ravel(order="F") for g in grids], axis=0)


def generate_training_sets(domains: Sequence[VarDomain], dx, eqs: Sequence[Equation], bcs: Sequence[Equation],
                           eltype, vi: VarInfo) -> Tuple[List[np.ndarray], List[np.ndarray]]:
    """Grid training sets for the equations and the boundary conditions.

    Follows reference src/discretize.jl:201-240 literally, including that the list of
    boundary values removed from the PDE spans (``dif``) is built from ``get_variables`` --
    symbols only -- and therefore stays empty: the PDE set is the *full* grid."""
    dxs = list(dx) if isinstance(dx, (list, tuple, np.ndarray)) else [dx] * len(domains)
    spans = {str(d.variables): _julia_range(d.domain.lo, float(h), d.domain.hi) for d, h in zip(domains, dxs)}
    # dif[i] would hold numbers found among the *symbolic* bc arguments: always empty (see docstring)
    spans_pde = {k: v.copy() for k, v in spans.items()}

    def sets(eq_list, span_dict):
        out = []
        for args in get_argument(eq_list, vi):
            cols = [span_dict[a] if isinstance(a, str) else np.array([float(a)]) for a in args]
            out.append(_product_columns(cols).astype(eltype))
        return out

    return sets(eqs, spans_pde), sets(bcs, spans)


# ---- bounds for the sampling strategies (reference src/discretize.jl:299-324) ------------------------------
def get_bounds(domains: Sequence[VarDomain], eqs: Sequence[Equation], bcs: Sequence[Equation], eltype, vi: VarInfo,
               strategy) -> Tuple[List[Tuple[np.ndarray, np.ndarray]], List[Tuple[np.ndarray, np.ndarray]]]:
    """Per-term (lower, upper) bounds.  Stochastic / QuasiRandom: the interior shrinks by
    ``1/points`` on each side and numeric bc arguments give degenerate intervals
    (src/discretize.jl:299-324).  Quadrature: the plain domain bounds (the reference's
    ``+cbrt(eps)`` shift at :264-297 protects its adaptive integrator from the singular
    boundary and is not needed for fixed interior Gauss nodes)."""
    if isinstance(strategy, QuadratureTraining):
        span = {str(d.variables): (d.domain.lo, d.domain.hi) for d in domains}
    else:
        dx = 1.0 / strategy.points
        span = {str(d.variables): (d.domain.lo + dx, d.domain.hi - dx) for d in domains}

    def bounds(eq_list):
        out = []
        for args in get_argument(eq_list, vi):
            lo = np.array([span[a][0] if isinstance(a, str) else float(a) for a in args], dtype=eltype)
            hi = np.array([span[a][1] if isinstance(a, str) else float(a) for a in args], dtype=eltype)
            out.append((lo, hi))
        return out

    return bounds(eqs), bounds(bcs)


def generate_random_points(points: int, bound, eltype, rng: np.random.Generator) -> np.ndarray:
    """``rand(eltype, d, points) .* (ub .- lb) .+ lb`` (training_strategies.jl:242-245)."""
    lb, ub = bound
    u = rng.random((len(lb), points)).astype(eltype)
    return (u * (ub - lb)[:, None] + lb[:, None]).astype(eltype)


def generate_quasi_random_points(points: int, bound, eltype, seed: int) -> np.ndarray:
    """Low-discrepancy points in the box (training_strategies.jl:336-389 uses QuasiMonteCarlo.sample)."""
    from scipy.stats import qmc
    lb, ub = bound
    d = len(lb)
    u = qmc.Sobol(d=d, scramble=True, seed=seed).random(points)
    return (u.T * (ub - lb)[:, None] + lb[:, None]).astype(eltype)


def gauss_legendre_box(bound, nodes_per_dim: int, eltype) -> Tuple[np.ndarray, np.ndarray, float]:
    """Tensor Gauss-Legendre nodes / weights on a box; degenerate dimensions get one node.
    Returns (points (d, N), weights (N), area) with ``sum(weights) == area`` over the
    non-degenerate dimensions."""
    lb, ub = bound
    xs, ws, area = [], [], 1.0
    g, w = np.polynomial.legendre.leggauss(nodes_per_dim)
    for a, b in zip(lb.astype(np.float64), ub.astype(np.float64)):
        if b > a:
            xs.append(0.5 * (b - a) * g + 0.5 * (b + a))
            ws.append(0.5 * (b - a) * w)
            area *= (b - a)
        else:
            xs.append(np.array([a]))
            ws.append(np.array([1.0]))
    pts = _product_columns(xs)
    # weights with the same (first variable fastest) ordering as the points
    wl = np.meshgrid(*ws, indexing="ij")
    wt = np.ones_like(wl[0])
    for m in wl:
        wt = wt * m
    return pts.astype(eltype), wt.ravel(order="F").astype(eltype), float(area)


# ---- neural adapter sets (reference src/neural_adapter.jl:1-23) --------------------------------------------------
def adapter_training_set(domains: Sequence[VarDomain], dx, eltype) -> np.ndarray:
    """The neural adapter's Grid set: every domain's ``infimum:dx:supremum`` span, product in domain order (first
    variable fastest), one (d, N) matrix for the whole system (src/neural_adapter.jl:1-6)."""
    dxs = list(dx) if isinstance(dx, (list, tuple, np.ndarray)) else [dx] * len(domains)
    return _product_columns([_julia_range(d.domain.lo, float(h), d.domain.hi) for d, h in zip(domains, dxs)]).astype(eltype)


def get_bounds_(domains: Sequence[VarDomain], eqs: Sequence[Equation], eltype, vi: VarInfo):
    """``get_bounds_`` of the neural adapter (src/neural_adapter.jl:8-23): the first equation's arguments, each a
    variable's [infimum, supremum] -- the plain domain, not shrunk as get_bounds does -- or a number's degenerate
    interval.  Returns (args, lb, ub)."""
    span = {str(d.variables): (d.domain.lo, d.domain.hi) for d in domains}
    args = get_argument(list(eqs), vi)[0]
    lb = np.array([span[a][0] if isinstance(a, str) else float(a) for a in args], dtype=eltype)
    ub = np.array([span[a][1] if isinstance(a, str) else float(a) for a in args], dtype=eltype)
    return args, lb, ub


def shard_range(n: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous shard [lo, hi) of n points for `rank` of `world` (SURVEY section 8(e))."""
    base, rem = divmod(n, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)
