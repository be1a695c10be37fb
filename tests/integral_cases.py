"""The reference's integro-differential test problems (test/IntegroDiff/, seven files) as PDESystems, plus the shapes
the GPU tests add.  Each case: (pde_system, chains, GridTraining dx)."""
import numpy as np
import sympy as sp

import neuralpde_jl_b200 as npde
from neuralpde_jl_b200.pinn import Chain, Dense, initialparameters


def ide1(act="sigmoid"):
    """ide__integrodiff_example_1_1d.jl: Di(i) + 2 i + 5 ∫_0^t i ~ 1, i(0) ~ 0 on [0, 2]."""
    t = npde.parameters("t")
    i = npde.variables("i")
    Di = npde.Differential(t)
    Ii = npde.Integral(t, npde.ClosedInterval(0, t))
    eq = npde.Eq(Di(i(t)) + 2 * i(t) + 5 * Ii(i(t)), 1)
    sys_ = npde.PDESystem([eq], [npde.Eq(i(0.0), 0.0)], [npde.In(t, 0.0, 2.0)], [t], [i(t)])
    return sys_, [Chain(Dense(1, 15, act), Dense(15, 1))], 0.1


def ide2(act="sigmoid"):
    """ide__integrodiff_example_2_1d.jl: ∫_0^x u cos ~ x^3 / 3, u(0) ~ 0 on [0, 1]."""
    x = npde.parameters("x")
    u = npde.variables("u")
    Ix = npde.Integral(x, npde.ClosedInterval(0, x))
    eq = npde.Eq(Ix(u(x) * sp.cos(x)), x ** 3 / 3)
    sys_ = npde.PDESystem([eq], [npde.Eq(u(0.0), 0.0)], [npde.In(x, 0.0, 1.0)], [x], [u(x)])
    return sys_, [Chain(Dense(1, 15, act), Dense(15, 1))], 0.1


def ide3(act="sigmoid"):
    """ide__integrodiff_example_3_2_inputs_1_output.jl: ∫∫_[0,1]^2 u ~ 1/3 with derivative bcs."""
    x, y = npde.parameters("x y")
    u = npde.variables("u")
    Dx, Dy = npde.Differential(x), npde.Differential(y)
    Ix = npde.Integral((x, y), npde.UnitSquare())
    eq = npde.Eq(Ix(u(x, y)), sp.Rational(1, 3))
    bcs = [npde.Eq(u(0.0, 0.0), 1), npde.Eq(Dx(u(x, y)), -2 * x), npde.Eq(Dy(u(x, y)), -2 * y)]
    sys_ = npde.PDESystem([eq], bcs, [npde.In(x, 0.0, 1.0), npde.In(y, 0.0, 1.0)], [x, y], [u(x, y)])
    return sys_, [Chain(Dense(2, 15, act), Dense(15, 1))], 0.1


def ide4(act="sigmoid", dx=0.1):
    """ide__integrodiff_example_4_2_inputs_1_output.jl: ∫_0^1 ∫_0^x u dy dx ~ 5/12 (the y bound is the owner's x)."""
    x, y = npde.parameters("x y")
    u = npde.variables("u")
    Dy = npde.Differential(y)
    Ix = npde.Integral((x, y), npde.ProductDomain(npde.UnitInterval(), npde.ClosedInterval(0, x)))
    eq = npde.Eq(Ix(u(x, y)), sp.Rational(5, 12))
    bcs = [npde.Eq(u(0.0, 0.0), 0), npde.Eq(Dy(u(x, y)), 2 * y), npde.Eq(u(x, 0), x)]
    sys_ = npde.PDESystem([eq], bcs, [npde.In(x, 0.0, 1.0), npde.In(y, 0.0, 1.0)], [x, y], [u(x, y)])
    return sys_, [Chain(Dense(2, 15, act), Dense(15, 1))], dx


def ide5(act="sigmoid"):
    """ide__integrodiff_example_5_1_input_2_outputs.jl: ∫_1^x u w ~ log|x|, Dx(w) ~ -2/x^3, u ~ x (two networks in one
    integrand)."""
    x = npde.parameters("x")
    u, w = npde.variables("u w")
    Dx = npde.Differential(x)
    Ix = npde.Integral(x, npde.ClosedInterval(1, x))
    eqs = [npde.Eq(Ix(u(x) * w(x)), sp.log(sp.Abs(x))), npde.Eq(Dx(w(x)), -2 / x ** 3), npde.Eq(u(x), x)]
    bcs = [npde.Eq(u(1.0), 1.0), npde.Eq(w(1.0), 1.0)]
    sys_ = npde.PDESystem(eqs, bcs, [npde.In(x, 1.0, 2.0)], [x], [u(x), w(x)])
    return sys_, [Chain(Dense(1, 15, act), Dense(15, 1)) for _ in range(2)], 0.1


def ide6(act="sigmoid"):
    """ide__integrodiff_example_6_infinity.jl: ∫_1^x u ~ ∫_1^∞ u - 1/x ([a, ∞) bound)."""
    x = npde.parameters("x")
    u = npde.variables("u")
    I = npde.Integral(x, npde.ClosedInterval(1, x))
    Iinf = npde.Integral(x, npde.ClosedInterval(1, npde.Inf))
    eq = npde.Eq(I(u(x)), Iinf(u(x)) - 1 / x)
    sys_ = npde.PDESystem([eq], [npde.Eq(u(1), 1)], [npde.In(x, 1.0, 2.0)], [x], [u(x)])
    return sys_, [Chain(Dense(1, 10, act), Dense(10, 1))], 0.1


def ide7(act="tanh"):
    """ide__integrodiff_example_7_infinity.jl: ∫_x^∞ u ~ 1/x ([x, ∞) bound)."""
    x = npde.parameters("x")
    u = npde.variables("u")
    I = npde.Integral(x, npde.ClosedInterval(x, npde.Inf))
    eq = npde.Eq(I(u(x)), 1 / x)
    sys_ = npde.PDESystem([eq], [npde.Eq(u(1), 1)], [npde.In(x, 1.0, 2.0)], [x], [u(x)])
    return sys_, [Chain(Dense(1, 12, act), Dense(12, 1))], 0.1


REFERENCE = {"ide1": ide1, "ide2": ide2, "ide3": ide3, "ide4": ide4, "ide5": ide5, "ide6": ide6, "ide7": ide7}


def discretization(chains, dx, dtype=np.float64, seed=110, **kw):
    return npde.PhysicsInformedNN(chains if len(chains) > 1 else chains[0], npde.GridTraining(dx),
                                  init_params=init_params(chains, dtype, seed), **kw)


def init_params(chains, dtype=np.float64, seed=110):
    rng = np.random.default_rng(seed)
    flat = np.concatenate([initialparameters(rng, c, np.float64) for c in chains])
    # a non-zero bias so every activation is evaluated away from its symmetric point
    flat = flat + 0.05 * rng.standard_normal(flat.shape)
    return flat.astype(dtype)


def chain_specs(chains):
    return [(c.dims, c.acts) for c in chains]
