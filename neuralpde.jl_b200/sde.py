"""NNSDE: ``solve(SDEProblem(f, g, u0, tspan, p), NNSDE(chain, opt; ...))`` on the fused kernel (reference
src/NN_SDE_solve.jl).

The network N(t, z_1..z_n) takes the time and n = chain.dims[0] - 1 N(0, 1) coefficients of the truncated
Karhunen-Loeve (KKL) expansion of the Wiener process, W'(t) ≈ √2 Σ_j z_j cos((j - ½) π t).  The trial solution is
φ = u0 + (t - t0) N(t, z) and the residual of component k is r_k = dφ_k/dt - f_k(φ, p, t) - g_k(φ, p, t) W'(t)
(:256-283).  f and g are traced once with sympy symbols and lowered by ode.py's shared lowering to value and d/dt
taps of output k.  Time is rescaled to tspan ./ tspan[end] (:774-779), and f and g see the scaled t.  DESIGN
section 4.14 maps the reference's loss terms onto the engine's terms.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np
import sympy as sp

from . import engine as _eng
from .engine import Engine, REDUCE_MEAN, REDUCE_WSUM, TermSpec
from .ode import (T_SYM, ComponentVector, OptimizationSolution, _Lowering, _TrialProblem, _TrialRepresentation,
                  _analytic_errors, _check_mode, _save_times, _strategy, _theta0, _train)
from .strategies import GridTraining, QuadratureTraining, StochasticTraining, _julia_range, gauss_legendre_box

_OUT_OF_PLACE = "The NNSDE solver only supports out-of-place SDE definitions, i.e. du=f(u,p,t) + g(u,p,t)*dW(t)"


# ---- problem and algorithm ------------------------------------------------------------------------------------
@dataclass
class SDEProblem(_TrialProblem):
    """``SDEProblem(f, g, u0, tspan, p)``: out-of-place drift ``f(u, p, t)`` and diagonal noise ``g(u, p, t)``, ``u0`` a
    number or a vector.  ``f`` may be an ``ODEFunction(f, analytic)`` whose ``analytic(u0, p, t)`` is the expected
    solution E[u(t)]; the solution then carries errors of the ensemble mean."""
    f: object
    g: object
    u0: object
    tspan: Sequence[float]
    p: object = None
    _solver = "NNSDE"
    _out_of_place = _OUT_OF_PLACE
    _components_note = " (g is diagonal noise: one per component)"
    _traced = ("f", "g")

    def __post_init__(self):
        super().__post_init__()
        if self.tspan[1] == 0.0:
            raise ValueError("NNSDE rescales time to tspan ./ tspan[end]; tspan[end] = 0 cannot be rescaled")


class NNSDE:
    """``NNSDE(chain, opt, init_params; strategy, autodiff, batch, sub_batch, strong_loss, moment_loss, param_estim,
    dataset, numensemble, additional_loss)`` (src/NN_SDE_solve.jl:149-160).  ``chain`` has 1 + n_z inputs (t and the
    KKL coefficients) and one output per component of u0.  ``opt``: ``Adam(...)`` (host loop, or the device loop with
    ``solve(...; device_loop=True)``), ``BFGS()`` or ``LBFGS()``.  ``dataset = [[x_1, ..., x_m], t]``: m observed paths
    of a scalar process at the times t, for ``param_estim``.  Engine options: ``mode`` ("ffma" | "tc_f64"),
    ``device``, and ``seed`` for the initial parameters and the host draws of z (the reference uses the global RNG)."""
    def __init__(self, chain, opt, init_params=None, *, strategy=None, autodiff=False, batch=True, sub_batch=1,
                 strong_loss=False, moment_loss=False, param_estim=False, dataset=(), data_sub_batch=1, numensemble=10,
                 additional_loss=None, mode="ffma", device=0, seed=0):
        self.chain, self.opt, self.init_params = chain, opt, init_params
        self.strategy, self.autodiff, self.batch = strategy, bool(autodiff), bool(batch)
        self.sub_batch, self.strong_loss, self.moment_loss = int(sub_batch), bool(strong_loss), bool(moment_loss)
        self.param_estim, self.dataset, self.data_sub_batch = bool(param_estim), list(dataset), int(data_sub_batch)
        self.numensemble, self.additional_loss = int(numensemble), additional_loss
        self.mode, self.device, self.seed = mode, device, seed
        _check_mode(mode, "NNSDE", "the tensor-core modes propagate 1-output networks and no parameter-only terms")
        if self.sub_batch < 1:
            raise ValueError("NNSDE: sub_batch must be >= 1, got %d" % self.sub_batch)
        if additional_loss is not None:
            raise ValueError("NNSDE: additional_loss(phi, θ) closures cannot run inside the CUDA kernel")
        if self.moment_loss:
            raise ValueError("NNSDE: moment_loss is not supported: generate_DataMoments_loss squares per-time sample "
                             "means, one functional per time, and the engine evaluates at most one functional term")


# ---- the residuals ----------------------------------------------------------------------------------------------
def kkl_noise(z: Sequence[sp.Expr], t) -> sp.Expr:
    """√2 Σ_j z_j cos((j - ½) π t), the truncated KKL series of dW/dt (:262)"""
    return sp.sqrt(2) * sp.Add(*[zj * sp.cos((j + sp.Rational(1, 2)) * sp.pi * t) for j, zj in enumerate(z)])


class _SDELowering(_Lowering):
    """The trial solution of N(t, z_1..z_n_z) on time rescaled to tspan ./ tspan[end], its KKL residuals and the
    Euler-Maruyama data terms"""

    def __init__(self, prob: SDEProblem, param_estim: bool, n_z: int):
        super().__init__(prob, param_estim, ["t"] + ["z%d" % (j + 1) for j in range(n_z)])
        self.t0 = prob.tspan[0] / prob.tspan[1]

    def residuals(self) -> List[sp.Expr]:
        """r_k = dφ_k/dt - f_k(φ, p, t) - g_k(φ, p, t) √2 Σ_j z_j cos((j - ½) π t)"""
        ph = [self.phi(k) for k in range(self.n)]
        fs, gs = self._trace("f", ph), self._trace("g", ph)
        w = kkl_noise([sp.Symbol(r, real=True) for r in self.rows[1:]], T_SYM)
        return [self.dphi(k) - fs[k] - gs[k] * w for k in range(self.n)]

    def em_residuals(self) -> List[sp.Expr]:
        """generate_EM_L2loss (:452-484) on rows X, t, Δt, ΔX: ΔX - f Δt and (ΔX - f Δt)^2 - g^2 Δt"""
        X, dt, dX = (sp.Symbol(s, real=True) for s in ("X", "dt", "dX"))
        f, g = self._trace("f", [X])[0], self._trace("g", [X])[0]
        e = dX - f * dt
        return [e, e ** 2 - g ** 2 * dt]


def reads_param(spec: TermSpec) -> bool:
    return any(ins[0] == "param" for ins in spec.prog)


def add_rand_coeff(ts, n_z: int, sub_batch: int, rng) -> List[np.ndarray]:
    """one (1 + n_z, sub_batch) matrix per time, an independent N(0, 1) draw per column (:353-362)"""
    return [np.vstack([np.full(sub_batch, t), rng.standard_normal((sub_batch, n_z)).T]) for t in np.ravel(ts)]


def add_rand_coeff_2(ts, n_z: int, sub_batch: int, rng) -> List[np.ndarray]:
    """one (1 + n_z, sub_batch) matrix per time; column s has path s's z at every time (:372-382)"""
    z = rng.standard_normal((sub_batch, n_z)).T
    return [np.vstack([np.full(sub_batch, t), z]) for t in np.ravel(ts)]


def em_points(dataset):
    """rows X, t, Δt, ΔX of the n · n_samples increments, path by path (dataset times are not rescaled)"""
    t = np.asarray(dataset[1], dtype=np.float64)
    cols = []
    for x in dataset[0]:
        x = np.asarray(x, dtype=np.float64)
        cols.append(np.stack([x[:-1], t[:-1], np.diff(t), np.diff(x)]))
    return np.concatenate(cols, axis=1)


def _valid_dataset(ds) -> bool:
    if len(ds) < 2 or not isinstance(ds[0], (list, tuple)) or len(ds[0]) == 0:
        return False
    t = ds[1]
    if np.ndim(t) != 1 or np.size(t) < 2 or np.iscomplexobj(t):
        return False
    return all(np.ndim(x) == 1 and np.size(x) == np.size(t) and not np.iscomplexobj(x) for x in ds[0])


# ---- the engine problem -----------------------------------------------------------------------------------------
class NNSDERepresentation(_TrialRepresentation):
    """The engine problem of one ``solve(prob, alg)``: terms (``term_names``), their weights, point sets, θ0 and
    ``loss_const`` (the Euler-Maruyama terms that do not depend on θ).  ``loss_grad(θ)`` is one evaluation of the
    engine's terms (a fresh StochasticTraining draw each call); the reference's objective is its total plus
    ``loss_const``."""

    def __init__(self, prob: SDEProblem, alg: NNSDE, dt=None, tstops=None):
        if not isinstance(alg, NNSDE):
            raise TypeError("solve(::SDEProblem, alg): alg must be an NNSDE")
        if tstops is not None:
            raise ValueError("NNSDE: tstops are not supported (the reference's evaluate_tstops_loss reads an undefined "
                             "`ts`, src/NN_SDE_solve.jl:651, so every tstops solve throws there)")
        chain = alg.chain
        n_z = chain.dims[0] - 1
        t0, t1 = prob.tspan[0] / prob.tspan[1], 1.0          # tspan_scale = tspan ./ tspan[end]
        if dt is not None:
            dt = dt / abs(t1 - t0)
        lw = _SDELowering(prob, alg.param_estim, n_z)
        n = lw.n
        if chain.dims[-1] != n or n_z < 0:
            raise ValueError("NNSDE: the chain maps (t, z_1..z_n_z) to the %d components of u0: it needs %d outputs, "
                             "has %d" % (n, n, chain.dims[-1]))
        if 1 + n_z > _eng.MAX_IN:
            raise ValueError("NNSDE: the chain has %d inputs (t and %d KKL coefficients); the engine's networks take at "
                             "most %d (PINN_MAX_DIM)" % (1 + n_z, n_z, _eng.MAX_IN))

        strategy = _strategy(alg, dt)
        S = alg.sub_batch
        if isinstance(strategy, QuadratureTraining) and S > 1:
            raise ValueError("NNSDE: QuadratureTraining with sub_batch > 1 is not supported: its integrand squares a "
                             "sample mean, (mean_s Σ_k r_k^2)^2, which is not a sum of per-point squares")

        ds = alg.dataset
        if not ds and alg.param_estim:
            raise ValueError("Dataset or an additional loss is required for Inverse problems performing Parameter "
                             "Estimation.")
        if ds and not _valid_dataset(ds):
            raise ValueError("Invalid dataset. The dataset would be a timeseries (x̂,t) where x̂ is of type: "
                             "Vector{<:Vector{<:AbstractFloat}} and t is type: Vector{AbstractFloat}.")
        if ds and alg.param_estim and not prob.scalar:
            raise ValueError("NNSDE: the Euler-Maruyama data loss (generate_EM_L2loss) observes a scalar process; u0 has "
                             "%d components" % n)

        p0 = np.ravel(np.asarray(prob.p, dtype=np.float64)) if alg.param_estim else np.zeros(0)
        flat = _theta0(alg, chain, p0, "NNSDE")
        super().__init__(prob, chain, strategy, lw, flat.dtype)
        add = self.add
        rng = np.random.default_rng([int(alg.seed), 1])      # the host draws of z (training sets)
        res = lw.residuals()
        rows = lw.rows
        strong = alg.strong_loss
        training_sets: list = []
        if isinstance(strategy, QuadratureTraining):
            # ∫ abs2(inner_sde_loss) dt with one z per node and sub_batch 1: residual Σ_k r_k^2 (:498-531)
            T, w, _ = gauss_legendre_box((np.array([t0]), np.array([t1])), int(strategy.nodes_per_dim), np.float64)
            X = np.vstack([T, rng.standard_normal((T.size, n_z)).T])
            add(lw.term(sp.Add(*[r ** 2 for r in res]), rows, REDUCE_WSUM, 1.0), X, w, 1.0, "quadrature")
        elif isinstance(strategy, StochasticTraining):
            # a fresh draw of N_t times x S samples per evaluation (:570-603), on the device KKL sampler
            nt = int(strategy.points)
            wt = {(False, True): 1.0, (False, False): nt, (True, True): S, (True, False): nt * S}[(strong, alg.batch)]
            for k in range(n):
                self.sampled.append(len(self.specs))
                add(lw.term(res[k], rows, REDUCE_MEAN), None, None, wt, "residual_%d" % (k + 1))
        else:
            ts = (_julia_range(t0, float(strategy.dx), t1) if isinstance(strategy, GridTraining)
                  else strategy.sample(t0, t1))
            training_sets = (add_rand_coeff_2 if strong else add_rand_coeff)(ts, n_z, S, rng)
            X = np.concatenate(training_sets, axis=1) if training_sets else np.zeros((1 + n_z, 0))
            nt = ts.size
            for k in range(n):
                if not strong and alg.batch:        # (1/N_t) Σ_i mean_s = mean over the N_t·S points
                    add(lw.term(res[k], rows, REDUCE_MEAN), X, None, 1.0, "residual_%d" % (k + 1))
                else:                               # Σ_i mean_s / (1/N_t) Σ_i Σ_s / Σ_i Σ_s
                    scale = {(False, False): 1.0 / S, (True, True): 1.0 / nt, (True, False): 1.0}[(strong, alg.batch)]
                    add(lw.term(res[k], rows, REDUCE_WSUM, scale), X, np.ones(X.shape[1]), 1.0, "residual_%d" % (k + 1))

        loss_const = 0.0
        if alg.param_estim and ds:
            P = em_points(ds)
            for j, e in enumerate(lw.em_residuals()):
                spec = lw.term(e, ["X", "t", "dt", "dX"], REDUCE_WSUM, 1.0)
                if reads_param(spec):
                    add(spec, P, np.ones(P.shape[1]), 1.0, "em_%d" % (j + 1))
                else:       # f (or g) does not read θ.p: a constant of the objective
                    fn = sp.lambdify([sp.Symbol(s, real=True) for s in ("X", "t", "dt", "dX")], e, "numpy")
                    loss_const += float(np.sum(np.asarray(fn(*P), dtype=np.float64) ** 2 * np.ones(P.shape[1])))
        self._close("NNSDE", p0.size, alg.mode, alg.device)
        self.alg, self.n_z = alg, n_z
        self.tspan_scale, self.dt = (t0, t1), dt
        self.training_sets = training_sets
        self.loss_const = loss_const
        self.flat_init_params = ComponentVector(flat, self.n_net)

    def _set_samplers(self, eng: Engine):
        """the StochasticTraining terms on the device KKL sampler, all with one seed, so that every component sees the
        same draw"""
        t0, t1 = self.tspan_scale
        for i in self.sampled:
            eng.set_sampler_kkl(i, int(self.strategy.points), self.alg.sub_batch, t0, t1, int(self.strategy.seed),
                                strong=self.alg.strong_loss)


# ---- solution ---------------------------------------------------------------------------------------------------
class SDEPhi:
    """``phi(inp, θ)``: φ = u0 + (t - t0) N(inp) at a (1 + n_z,) input (a number for scalar u0, else (n,)) or at the
    columns of a (1 + n_z, m) matrix ((n, m))"""

    def __init__(self, rep: NNSDERepresentation):
        self._rep = rep

    def __call__(self, inp, theta):
        inp = np.asarray(inp, dtype=np.float64)
        U = self._rep.trial(theta, inp)
        if inp.ndim == 1:
            return float(U[0, 0]) if self._rep.prob.scalar else U[:, 0]
        return U


@dataclass
class NNSDEInterpolation:
    phi: SDEPhi
    θ: ComponentVector


@dataclass
class RODESolution:
    """``t``, ``u`` (the ensemble, as ``SDEsol.estimated_sol``), ``interp`` (``phi``, ``θ``), ``errors``"""
    t: np.ndarray
    u: list
    interp: NNSDEInterpolation
    errors: dict
    retcode: str = "Success"


@dataclass
class SDEsol:
    """(:745-756) ``estimated_sol[k]``: output k at every timepoint for each of the numensemble validation inputs,
    ``[numensemble, len(timepoints)]`` (``pmean`` gives the weak solution); ``ensemble_fits[i]`` the (n, numensemble)
    outputs at ``ensemble_inputs[i]``, the (1 + n_z, numensemble) inputs of timepoint i; ``training_sets`` the
    per-time input matrices of the fixed-point strategies (empty for Stochastic and Quadrature training)."""
    original: OptimizationSolution
    rode_solution: RODESolution
    estimated_sol: List[np.ndarray]
    timepoints: np.ndarray
    estimated_params: Optional[np.ndarray]
    ensemble_fits: List[np.ndarray]
    ensemble_inputs: List[np.ndarray]
    numensemble: int
    training_sets: list
    dataset_training_sets: Optional[list]


# ---- solve ------------------------------------------------------------------------------------------------------
def solve_nnsde(prob: SDEProblem, alg: NNSDE, *, maxiters: int, dt=None, abstol: float = 1e-6, saveat=None,
                save_everystep: bool = True, tstops=None, verbose: bool = False, device_loop: bool = False,
                chunk: int = 50) -> SDEsol:
    """``solve(prob::SDEProblem, alg::NNSDE; maxiters, dt, abstol, saveat, save_everystep, verbose)``
    (src/NN_SDE_solve.jl:758-943).  Training stops as soon as a loss is below ``abstol``, as NNODE's loops do."""
    rep = NNSDERepresentation(prob, alg, dt=dt, tstops=tstops)
    res = _train(rep, alg.opt, int(maxiters), float(abstol), verbose, device_loop, chunk, who="NNSDE")
    t0, t1 = rep.tspan_scale
    ts = _save_times(t0, t1, saveat, rep.dt, save_everystep)
    inputs = add_rand_coeff(ts, rep.n_z, alg.numensemble, np.random.default_rng([int(alg.seed), 2]))
    U = rep.trial(res.u, np.concatenate(inputs, axis=1)).reshape(rep.n, ts.size, alg.numensemble)
    fits = [U[:, i, :].copy() for i in range(ts.size)]
    est = [U[k].T.copy() for k in range(rep.n)]
    errors = _analytic_errors(prob, ts, np.stack([e.mean(axis=0) for e in est]))
    rode = RODESolution(ts, est, NNSDEInterpolation(SDEPhi(rep), res.u), errors)
    return SDEsol(res, rode, est, ts, np.asarray(res.u.p).copy() if alg.param_estim else None, fits, inputs,
                  alg.numensemble, rep.training_sets, None)
