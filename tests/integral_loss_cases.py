"""Problems with an integral constraint (pinn.IntegralLoss) for the CPU and GPU tests.  Each case returns
(pde_system, chains, strategy, IntegralLoss, param_estim)."""
import numpy as np
import sympy as sp

import neuralpde_jl_b200 as npde
from neuralpde_jl_b200.pinn import Chain, Dense

import integral_cases as IC

ALPHA, BETA, SIGMA = 0.3, 0.5, 0.5
X0, X1, DX = -2.2, 2.2, 0.01
C_TEST = 142.88418699042          # test/NNPDE2/additional_loss__fokker_planck.jl:75
C_TUTORIAL = 32.47                # 0.01 Σ p Δx = 1 (docs/src/tutorials/constraints.md:58-71) gives ∫p ≈ 100


def fokker_planck_system():
    """the stationary Fokker-Planck equation of additional_loss__fokker_planck.jl:11-28"""
    x = npde.parameters("x")
    p = npde.variables("p")
    Dx, Dxx = npde.Differential(x), npde.Differential(x) ** 2
    eq = npde.Eq(Dx((ALPHA * x - BETA * x ** 3) * p(x)), (SIGMA ** 2 / 2) * Dxx(p(x)))
    bcs = [npde.Eq(p(X0), 0.0), npde.Eq(p(X1), 0.0)]
    return npde.PDESystem([eq], bcs, [npde.In(x, X0, X1)], [x], [p(x)]), x, p


def fp_chain(width=18):
    return Chain(Dense(1, width, "sigmoid"), Dense(width, width, "sigmoid"), Dense(width, width, "sigmoid"),
                 Dense(width, 1))


def fokker_planck(norm="abs", target=0.0):
    """the reference test's constraint |∫(dx p(x) - 1) dx| on [-2.2, 2.2], GridTraining(0.01)"""
    sys_, x, p = fokker_planck_system()
    add = npde.IntegralLoss(DX * p(x) - 1, list(sys_.domain), norm=norm, target=target)
    return sys_, [fp_chain()], npde.GridTraining(DX), add, False


def fokker_planck_tutorial():
    """the tutorial's constraint |0.01 Σ_i p(x_i) Δx - 1| over 200 uniform points, QuadratureTraining()"""
    sys_, x, p = fokker_planck_system()
    xs = np.linspace(X0, X1, 200)
    dxs = xs[1] - xs[0]
    add = npde.IntegralLoss(p(x), points=xs.reshape(1, -1), weights=np.full(xs.size, 0.01 * dxs), target=1.0,
                            norm="abs")
    return sys_, [fp_chain()], npde.QuadratureTraining(), add, False


def neumann2d():
    """pure-Neumann Poisson problem on the unit square, Δu = -2π² cos(πx) cos(πy), zero normal derivative: the solution
    is fixed up to a constant, pinned by a zero mean ((∫u)² on a Gauss-Legendre box)"""
    x, y = npde.parameters("x y")
    u = npde.variables("u")
    Dx, Dy = npde.Differential(x), npde.Differential(y)
    Dxx, Dyy = Dx ** 2, Dy ** 2
    eq = npde.Eq(Dxx(u(x, y)) + Dyy(u(x, y)), -2 * sp.pi ** 2 * sp.cos(sp.pi * x) * sp.cos(sp.pi * y))
    bcs = [npde.Eq(Dx(u(0.0, y)), 0.0), npde.Eq(Dx(u(1.0, y)), 0.0), npde.Eq(Dy(u(x, 0.0)), 0.0),
           npde.Eq(Dy(u(x, 1.0)), 0.0)]
    doms = [npde.In(x, 0.0, 1.0), npde.In(y, 0.0, 1.0)]
    sys_ = npde.PDESystem([eq], bcs, doms, [x, y], [u(x, y)])
    add = npde.IntegralLoss(u(x, y), doms, norm="abs2", nodes_per_dim=8)
    return sys_, [Chain(Dense(2, 16, "tanh"), Dense(16, 16, "tanh"), Dense(16, 1))], npde.GridTraining(0.1), add, False


def taps_and_param():
    """an integrand with a first and a second derivative tap and a trainable parameter: u'' + a u' = 0 on [0, 1] with
    u(0) = 0 and the constraint |∫ (a x u' + u'' + sin(u)) dx - 0.3|"""
    x = npde.parameters("x")
    a = npde.parameters("a")
    u = npde.variables("u")
    Dx, Dxx = npde.Differential(x), npde.Differential(x) ** 2
    eq = npde.Eq(Dxx(u(x)) + a * Dx(u(x)), 0)
    sys_ = npde.PDESystem([eq], [npde.Eq(u(0.0), 0.0)], [npde.In(x, 0.0, 1.0)], [x], [u(x)], [a], defaults={a: 0.7})
    add = npde.IntegralLoss(a * x * Dx(u(x)) + Dxx(u(x)) + sp.sin(u(x)), list(sys_.domain), target=0.3,
                            nodes_per_dim=12)
    return sys_, [Chain(Dense(1, 12, "tanh"), Dense(12, 12, "sin"), Dense(12, 1))], npde.GridTraining(0.05), add, True


CASES = {"fokker_planck": fokker_planck, "tutorial": fokker_planck_tutorial, "neumann2d": neumann2d,
         "taps_and_param": taps_and_param}


def discretization(case, dtype=np.float64, seed=110, adaptive_loss=None, **kw):
    sys_, chains, strategy, add, pe = case
    flat = IC.init_params(chains, np.float64, seed)
    if pe:
        flat = np.concatenate([flat, [0.7]])
    return npde.PhysicsInformedNN(chains if len(chains) > 1 else chains[0], strategy, init_params=flat.astype(dtype),
                                  additional_loss=add, param_estim=pe, adaptive_loss=adaptive_loss, **kw)


def analytic(x, C):
    return C * np.exp((1 / (2 * SIGMA ** 2)) * (2 * ALPHA * x ** 2 - BETA * x ** 4))
