"""Problems for the tensor-core precision-model tests (tests/tc_model.py): one small PDESystem per channel structure that
PINN_TC_DISPATCH instantiates, with all-tanh and generic-activation networks, plus shapes, networks and terms the
tensor-core kernels take other branches for.  Each builder returns a Config (neuralpde_jl_b200.configs)."""
from contextlib import contextmanager

import numpy as np
import sympy as sp

from neuralpde_jl_b200 import pinn
from neuralpde_jl_b200.configs import Config
from neuralpde_jl_b200.pinn import Chain, DataLoss, Dense
from neuralpde_jl_b200.strategies import GridTraining, QuadratureTraining
from neuralpde_jl_b200.symbolic import Differential, Eq, In, PDESystem, parameters, variables

from tc_model import SpecRecorder

GENERIC = ["sigmoid", "sin", "softplus", "swish", "identity"]


def net(d_in, widths, acts):
    layers, prev = [], d_in
    for w, a in zip(widths, acts):
        layers.append(Dense(prev, w, a))
        prev = w
    return Chain(*layers, Dense(prev, 1))


def _box(names, lo=0.0, hi=1.0):
    syms = parameters(" ".join(names))
    syms = syms if isinstance(syms, (list, tuple)) else [syms]
    return list(syms), [In(s, lo, hi) for s in syms]


# ---- one PDESystem per channel structure (n1, n2, pure) of the PDE term ------------------------------------------
def _value():                         # (0, 0)
    (x, y), dom = _box("x y")
    u = variables("u")
    return PDESystem(Eq(u(x, y), sp.sin(sp.pi * x) * y), [Eq(u(0, y), 0.0)], dom, [x, y], [u(x, y)]), 0.05


def _ux():                            # (1, 0)
    (x, y), dom = _box("x y")
    u = variables("u")
    return PDESystem(Eq(Differential(x)(u(x, y)), sp.cos(x) * y), [Eq(u(0, y), y)], dom, [x, y], [u(x, y)]), 0.05


def _transport2():                    # (2, 0)
    (x, y), dom = _box("x y")
    u = variables("u")
    U = u(x, y)
    return PDESystem(Eq(Differential(x)(U) + Differential(y)(U), 0.0), [Eq(u(x, 0), sp.sin(sp.pi * x))], dom, [x, y],
                     [U]), 0.05


def _transport3():                    # (3, 0)
    (t, x, y), dom = _box("t x y")
    u = variables("u")
    U = u(t, x, y)
    eq = Eq(Differential(t)(U) + Differential(x)(U) + 0.5 * Differential(y)(U), 0.0)
    return PDESystem(eq, [Eq(u(0, x, y), sp.sin(sp.pi * x) * sp.sin(sp.pi * y))], dom, [t, x, y], [U]), 0.125


def _transport4():                    # (4, 0): four inputs, the d_in > 3 first-layer branch
    (t, x, y, z), dom = _box("t x y z")
    u = variables("u")
    U = u(t, x, y, z)
    D = Differential
    eq = Eq(D(t)(U) + D(x)(U) - D(y)(U) + 0.5 * D(z)(U), 0.0)
    return PDESystem(eq, [Eq(u(0, x, y, z), x * y - z)], dom, [t, x, y, z], [U]), 0.25


def _uxx():                           # (1, 1), Neumann bc (1, 0)
    (x,), dom = _box("x")
    u = variables("u")
    Dx = Differential(x)
    eq = Eq((Dx ** 2)(u(x)), -sp.pi ** 2 * sp.sin(sp.pi * x))
    return PDESystem(eq, [Eq(u(0.0), 0.0), Eq(Dx(u(1.0)), -sp.pi)], dom, [x], [u(x)]), 1.0 / 99


def _burgers():                       # (2, 1) pure
    t, x = parameters("t x")
    u = variables("u")
    U = u(t, x)
    Dt, Dx = Differential(t), Differential(x)
    eq = Eq(Dt(U) + U * Dx(U) - (0.01 / sp.pi) * (Dx ** 2)(U), 0)
    bcs = [Eq(u(0, x), -sp.sin(sp.pi * x)), Eq(u(t, -1), 0.0), Eq(u(t, 1), 0.0)]
    return PDESystem(eq, bcs, [In(t, 0.0, 1.0), In(x, -1.0, 1.0)], [t, x], [U]), 0.05


def _mixed21():                       # (2, 1) mixed: u_xy + u_x
    (x, y), dom = _box("x y")
    u = variables("u")
    U = u(x, y)
    Dx, Dy = Differential(x), Differential(y)
    return PDESystem(Eq(Dx(Dy(U)) + Dx(U), x * y), [Eq(u(x, 0), x)], dom, [x, y], [U]), 0.05


def _mixed31():                       # (3, 1) mixed: u_xy + u_z
    (x, y, z), dom = _box("x y z")
    u = variables("u")
    U = u(x, y, z)
    D = Differential
    return PDESystem(Eq(D(x)(D(y)(U)) + D(z)(U), 1.0), [Eq(u(x, y, 0), x * y)], dom, [x, y, z], [U]), 0.125


def _pure31():                        # (3, 1) pure: u_t + u_x + u_y - u_xx
    (t, x, y), dom = _box("t x y")
    u = variables("u")
    U = u(t, x, y)
    D = Differential
    eq = Eq(D(t)(U) + D(x)(U) + D(y)(U) - 0.1 * (D(x) ** 2)(U), 0.0)
    return PDESystem(eq, [Eq(u(0, x, y), sp.sin(sp.pi * x) * y)], dom, [t, x, y], [U]), 0.125


def _mixed22():                       # (2, 2) mixed: u_xx + u_xy
    (x, y), dom = _box("x y")
    u = variables("u")
    U = u(x, y)
    Dx, Dy = Differential(x), Differential(y)
    return PDESystem(Eq((Dx ** 2)(U) + Dx(Dy(U)), 1.0), [Eq(u(0, y), y ** 2)], dom, [x, y], [U]), 0.05


def _poisson():                       # (2, 2) pure; on the wide kernel two (1, 1) passes
    (x, y), dom = _box("x y")
    u = variables("u")
    U = u(x, y)
    Dxx, Dyy = Differential(x) ** 2, Differential(y) ** 2
    eq = Eq(Dxx(U) + Dyy(U), -sp.sin(sp.pi * x) * sp.sin(sp.pi * y))
    bcs = [Eq(u(0, y), 0.0), Eq(u(1, y), 0.0), Eq(u(x, 0), 0.0), Eq(u(x, 1), 0.0)]
    return PDESystem(eq, bcs, dom, [x, y], [U]), 0.05


# name -> (system builder, runs on the wide kernel)
STRUCTURES = {
    "value": (_value, True), "ux": (_ux, True), "transport2": (_transport2, True), "transport3": (_transport3, True),
    "transport4": (_transport4, False), "uxx": (_uxx, True), "burgers": (_burgers, True), "mixed21": (_mixed21, True),
    "mixed31": (_mixed31, False), "pure31": (_pure31, False), "mixed22": (_mixed22, False), "poisson": (_poisson, True),
}
NARROW_WIDTHS = [[16, 16], [32, 32], [48, 48], [64, 64], [48, 16, 64], [16, 32]]


def _acts(i, depth, generic):
    if not generic:
        return ["tanh"] * depth
    return [GENERIC[(i + k) % len(GENERIC)] for k in range(depth)]


def structure_case(name, kernel, generic):
    """Config of structure `name` on the narrow ("tc") or wide ("tw") kernel, all-tanh or generic hidden layers."""
    build, _ = STRUCTURES[name]
    i = sorted(STRUCTURES).index(name)
    sys_, dx = build()
    d_in = len(sys_.ivs)
    widths = NARROW_WIDTHS[i % len(NARROW_WIDTHS)] if kernel == "tc" else [[128, 128], [128, 64, 128]][i % 2]
    chain = net(d_in, widths, _acts(i, len(widths), generic))
    return Config("%s_%s_%s" % (name, kernel, "generic" if generic else "tanh"), sys_, [chain], GridTraining(dx))


def matrix():
    """(id, kernel, Config factory) of every structure x activation kind on each kernel where it fits."""
    out = []
    for name, (_, wide_ok) in sorted(STRUCTURES.items()):
        for kernel in ("tc", "tw") if wide_ok else ("tc",):
            for generic in (False, True):
                out.append(("%s-%s-%s" % (name, kernel, "generic" if generic else "tanh"), kernel,
                            (lambda n=name, k=kernel, g=generic: structure_case(n, k, g))))
    return out


# ---- shapes, networks and terms -----------------------------------------------------------------------------------
def poisson_depth(tl, width=16):
    """2-D Poisson (5 channels) with tl tensor layers (0..6)."""
    sys_, dx = _poisson()
    return Config("poisson_tl%d" % tl, sys_, [net(2, [width] * (tl + 1), ["tanh"] * (tl + 1))], GridTraining(0.1))


def wide_deep():
    """Burgers on a 2 -> 128 x 7 -> 1 network: six tensor layers on the wide kernel."""
    sys_, dx = _burgers()
    return Config("burgers_wide_tl6", sys_, [net(2, [128] * 7, ["tanh"] * 7)], GridTraining(0.1))


def coupled_narrow():
    """Two networks of different width and depth, terms that tap both."""
    x, y = parameters("x y")
    u, v = variables("u v")
    U, V = u(x, y), v(x, y)
    Dx, Dy = Differential(x), Differential(y)
    eqs = [Eq((Dx ** 2)(U) + Dy(V), sp.sin(x)), Eq(Dx(V) + U * V, x * y)]
    bcs = [Eq(u(0, y), 0.0), Eq(v(x, 0), x)]
    sys_ = PDESystem(eqs, bcs, [In(x, 0.0, 1.0), In(y, 0.0, 1.0)], [x, y], [U, V])
    chains = [net(2, [32, 32], ["tanh", "tanh"]), net(2, [48, 16, 64], ["sigmoid", "swish", "tanh"])]
    return Config("coupled_narrow", sys_, chains, GridTraining(0.05), multioutput=True)


def coupled_wide():
    """Two 128-wide networks, one term taps both."""
    t, x = parameters("t x")
    u, v = variables("u v")
    U, V = u(t, x), v(t, x)
    Dt, Dx = Differential(t), Differential(x)
    eqs = [Eq(Dt(U) + V * Dx(U), 0.0), Eq((Dx ** 2)(V), U)]
    bcs = [Eq(u(0, x), sp.sin(sp.pi * x)), Eq(v(t, 0), 0.0)]
    sys_ = PDESystem(eqs, bcs, [In(t, 0.0, 1.0), In(x, 0.0, 1.0)], [t, x], [U, V])
    chains = [net(2, [128, 128], ["tanh", "tanh"]), net(2, [64, 128, 64], ["tanh", "softplus", "sin"])]
    return Config("coupled_wide", sys_, chains, GridTraining(0.05), multioutput=True)


def quadrature(width=32):
    """2-D Poisson with Gauss-Legendre quadrature weights (WSUM terms)."""
    sys_, _ = _poisson()
    chain = net(2, [width, width] if width <= 64 else [128, 128], ["tanh", "sigmoid"])
    return Config("poisson_quadrature", sys_, [chain], QuadratureTraining(nodes_per_dim=20, bc_nodes_per_dim=12))


def heat_param_estim():
    """u_t = a u_xx with the diffusivity a in theta.p and a DataLoss term on the analytic solution (narrow: 4 channels)."""
    t, x = parameters("t x")
    a = parameters("a")
    u = variables("u")
    U = u(t, x)
    Dt, Dxx = Differential(t), Differential(x) ** 2
    eq = Eq(Dt(U), a * Dxx(U))
    bcs = [Eq(u(0, x), sp.sin(sp.pi * x)), Eq(u(t, 0), 0.0), Eq(u(t, 1), 0.0)]
    sys_ = PDESystem(eq, bcs, [In(t, 0.0, 1.0), In(x, 0.0, 1.0)], [t, x], [U], ps=[a], defaults={a: 0.5})
    rng = np.random.default_rng(4)
    X = rng.random((2, 300))
    yobs = np.exp(-np.pi ** 2 * 0.1 * X[0]) * np.sin(np.pi * X[1])
    return Config("heat_param_estim", sys_, [net(2, [32, 32], ["tanh", "tanh"])], GridTraining(0.05),
                  param_estim=True, additional_loss=DataLoss("u", X, yobs))


def many_rows(kernel="tc"):
    """3-D transport with coordinate-only coefficients: hoisted rows make the PDE term's point matrix 7 rows deep."""
    (x, y, z), dom = _box("x y z")
    u = variables("u")
    U = u(x, y, z)
    D = Differential
    eq = Eq(sp.sin(x * y) * D(x)(U) + sp.cos(y + z) * D(y)(U) + sp.exp(x * z) * D(z)(U), sp.sin(x * y * z))
    sys_ = PDESystem(eq, [Eq(u(x, y, 0), x + y)], dom, [x, y, z], [U])
    widths = [32, 32] if kernel == "tc" else [128, 128]
    return Config("many_rows_%s" % kernel, sys_, [net(3, widths, ["tanh", "softplus"])], GridTraining(0.125))


def coords_above_one():
    """u_yy + u = g with x in (1 + 2^-9, 1 + 2^-8): every x rounds down to bf16 1.0, so the coordinates' lo (x - 1 > 0)
    enters the x column of the first layer's weight gradient with one sign at every point (the narrow kernel adds it
    for terms with second-derivative channels)."""
    x, y = parameters("x y")
    u = variables("u")
    U = u(x, y)
    eq = Eq((Differential(y) ** 2)(U) + U, sp.sin(sp.pi * y))
    lo, hi = 1 + 2.0 ** -9, 1 + 2.0 ** -8
    d = (hi - lo) / 12
    sys_ = PDESystem(eq, [Eq(u(x, 0), 0.0)], [In(x, lo + d / 2, hi - d / 2), In(y, 0.0, 1.0)], [x, y], [U])
    return Config("coords_above_one", sys_, [net(2, [32, 32], ["tanh", "tanh"])], GridTraining([d, 0.05]))


def point_count(kernel="tc"):
    """1-D u_xx; the tests set the PDE term's point count."""
    sys_, _ = _uxx()
    widths = [32, 32] if kernel == "tc" else [128, 128]
    return Config("uxx_points_%s" % kernel, sys_, [net(1, widths, ["tanh", "tanh"])], GridTraining(1.0 / 99))


# ---- capture without a GPU -----------------------------------------------------------------------------------------
@contextmanager
def engine_class(cls):
    """symbolic_discretize constructs `cls` instead of the engine."""
    old = pinn.Engine
    pinn.Engine = cls
    try:
        yield
    finally:
        pinn.Engine = old


def capture(cfg, mode="tc_bf16", dtype=np.float32):
    """(rep, SpecRecorder) of a Config: the spec and uploaded points symbolic_discretize hands to the engine."""
    with engine_class(SpecRecorder):
        rep = pinn.symbolic_discretize(cfg.pde_system, cfg.discretization(dtype=dtype, mode=mode))
    return rep, rep.engine


def make_theta(cfg, seed=3):
    """Glorot weights with every entry perturbed (non-zero biases), rounded to fp32."""
    th = cfg.init_params(np.float64, seed=seed)
    th = th + 0.05 * np.random.default_rng(seed).standard_normal(th.size)
    return th.astype(np.float32)
