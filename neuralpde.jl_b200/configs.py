"""The five BASELINE.json configurations as PDESystem + discretization builders.

Problem statements follow the reference where it has one (2-D Poisson: README.md:58-77;
Burgers: docs/src/tutorials/low_level.md:27-37 with the 3-bc form of
test/DGM/dgm__burger_s_equation.jl:39-46); configs 4 and 5 have no counterpart in the
reference tree (SURVEY section 4) and are fixed here.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional

import numpy as np
import sympy as sp

from .pinn import Chain, DataLoss, Dense, PhysicsInformedNN, initialparameters
from .strategies import GridTraining, QuadratureTraining, QuasiRandomTraining, StochasticTraining
from .symbolic import Differential, Eq, In, PDESystem, parameters, variables


@dataclass
class Config:
    name: str
    pde_system: PDESystem
    chains: List[Chain]
    strategy: object
    multioutput: bool = False
    param_estim: bool = False
    additional_loss: Optional[DataLoss] = None
    n_pde_points: int = 0
    note: str = ""

    def init_params(self, dtype=np.float32, seed: int = 1) -> np.ndarray:
        """Glorot-uniform weights, zero bias, generated in float64 then cast (SURVEY section 8(d))."""
        rng = np.random.default_rng(seed)
        parts = [initialparameters(rng, c, np.float64) for c in self.chains]
        if self.param_estim:
            parts.append(np.array([self.pde_system.defaults.get(p, 1.0) for p in self.pde_system.ps], dtype=np.float64))
        return np.concatenate(parts).astype(dtype)

    def discretization(self, dtype=np.float32, mode: str = "ffma", device: int = 0, seed: int = 1, **kw):
        chain = self.chains if self.multioutput else self.chains[0]
        return PhysicsInformedNN(chain, self.strategy, init_params=self.init_params(dtype, seed),
                                 param_estim=self.param_estim, additional_loss=self.additional_loss, mode=mode,
                                 device=device, **kw)

    def chain_specs(self):
        return [(c.dims, c.acts) for c in self.chains]


def mlp(n_in: int, width: int, hidden: int, act: str = "tanh") -> Chain:
    layers = [Dense(n_in, width, act)] + [Dense(width, width, act) for _ in range(hidden - 1)] + [Dense(width, 1)]
    return Chain(*layers)


def config1(n: int = 256) -> Config:
    """1-D Poisson u'' = f, Dirichlet BC, Chain(Dense(1,16,tanh), Dense(16,1)), GridTraining, 256 points."""
    x = parameters("x")
    u = variables("u")
    Dxx = Differential(x) ** 2
    eq = Eq(Dxx(u(x)), -sp.pi ** 2 * sp.sin(sp.pi * x))
    bcs = [Eq(u(0.0), 0.0), Eq(u(1.0), 0.0)]
    sys_ = PDESystem(eq, bcs, [In(x, 0.0, 1.0)], [x], [u(x)])
    return Config("cfg1_poisson1d", sys_, [Chain(Dense(1, 16, "tanh"), Dense(16, 1))], GridTraining(1.0 / (n - 1)),
                  n_pde_points=n)


def config2(n: int = 128, width: int = 64, hidden: int = 4) -> Config:
    """2-D Poisson on [0,1]^2 (README.md:58-69), 4x64 tanh MLP, GridTraining with n^2 points."""
    x, y = parameters("x y")
    u = variables("u")
    Dxx, Dyy = Differential(x) ** 2, Differential(y) ** 2
    eq = Eq(Dxx(u(x, y)) + Dyy(u(x, y)), -sp.sin(sp.pi * x) * sp.sin(sp.pi * y))
    bcs = [Eq(u(0, y), 0.0), Eq(u(1, y), 0.0), Eq(u(x, 0), 0.0), Eq(u(x, 1), 0.0)]
    sys_ = PDESystem(eq, bcs, [In(x, 0.0, 1.0), In(y, 0.0, 1.0)], [x, y], [u(x, y)])
    return Config("cfg2_poisson2d", sys_, [mlp(2, width, hidden)], GridTraining(1.0 / (n - 1)), n_pde_points=n * n)


def config3(points: int = 65536, bcs_points: int = 4096, width: int = 128, hidden: int = 5) -> Config:
    """Burgers u_t + u u_x - (0.01/pi) u_xx = 0 on (t,x) in [0,1]x[-1,1], 5x128 MLP, StochasticTraining."""
    t, x = parameters("t x")
    u = variables("u")
    Dt, Dx, Dxx = Differential(t), Differential(x), Differential(x) ** 2
    eq = Eq(Dt(u(t, x)) + u(t, x) * Dx(u(t, x)) - (0.01 / sp.pi) * Dxx(u(t, x)), 0)
    bcs = [Eq(u(0, x), -sp.sin(sp.pi * x)), Eq(u(t, -1), 0.0), Eq(u(t, 1), 0.0)]
    sys_ = PDESystem(eq, bcs, [In(t, 0.0, 1.0), In(x, -1.0, 1.0)], [t, x], [u(t, x)])
    return Config("cfg3_burgers", sys_, [mlp(2, width, hidden)],
                  StochasticTraining(points, bcs_points=bcs_points, seed=2), n_pde_points=points,
                  note="bcs_points=%d (the reference default would be bcs_points=points)" % bcs_points)


def config4(nodes: int = 128, bc_nodes: int = 32, width: int = 256, hidden: int = 6, nu: float = 0.01) -> Config:
    """Steady 3-D Navier-Stokes lid-driven cavity, one 3->256x6->1 network per (u, v, w, p), fixed-node
    quadrature with nodes^3 points."""
    x, y, z = parameters("x y z")
    u, v, w, p = variables("u v w p")
    D = {s: Differential(s) for s in (x, y, z)}
    D2 = {s: Differential(s) ** 2 for s in (x, y, z)}
    U = {"u": u(x, y, z), "v": v(x, y, z), "w": w(x, y, z)}
    P = p(x, y, z)

    def momentum(q, s):
        adv = U["u"] * D[x](q) + U["v"] * D[y](q) + U["w"] * D[z](q)
        return Eq(adv + D[s](P) - nu * (D2[x](q) + D2[y](q) + D2[z](q)), 0)

    eqs = [momentum(U["u"], x), momentum(U["v"], y), momentum(U["w"], z),
           Eq(D[x](U["u"]) + D[y](U["v"]) + D[z](U["w"]), 0)]
    bcs = []
    for f in (u, v, w):
        for axis in range(3):
            for val in (0.0, 1.0):
                args = [x, y, z]
                args[axis] = val
                lid = 1.0 if (f is u and axis == 2 and val == 1.0) else 0.0
                bcs.append(Eq(f(*args), lid))
    bcs.append(Eq(p(0.0, 0.0, 0.0), 0.0))          # pressure gauge
    sys_ = PDESystem(eqs, bcs, [In(x, 0.0, 1.0), In(y, 0.0, 1.0), In(z, 0.0, 1.0)], [x, y, z],
                     [u(x, y, z), v(x, y, z), w(x, y, z), p(x, y, z)])
    return Config("cfg4_ns_cavity", sys_, [mlp(3, width, hidden) for _ in range(4)],
                  QuadratureTraining(nodes, bc_nodes_per_dim=bc_nodes), multioutput=True,
                  n_pde_points=4 * nodes ** 3)


def config5(points: int = 1 << 20, bcs_points: int = 16384, n_obs: int = 4096, width: int = 128, hidden: int = 4) -> Config:
    """Parametric heat equation u_t = a*kappa*(u_xx + u_yy), inputs (t, x, y, kappa), unknown scalar a in
    theta.p (true value 1), data loss on the analytic solution exp(-2 pi^2 kappa t) sin(pi x) sin(pi y)."""
    t, x, y, k = parameters("t x y kappa")
    a = parameters("a")
    u = variables("u")
    Dt, Dxx, Dyy = Differential(t), Differential(x) ** 2, Differential(y) ** 2
    U = u(t, x, y, k)
    eq = Eq(Dt(U), a * k * (Dxx(U) + Dyy(U)))
    bcs = [Eq(u(0, x, y, k), sp.sin(sp.pi * x) * sp.sin(sp.pi * y)),
           Eq(u(t, 0, y, k), 0.0), Eq(u(t, 1, y, k), 0.0), Eq(u(t, x, 0, k), 0.0), Eq(u(t, x, 1, k), 0.0)]
    doms = [In(t, 0.0, 1.0), In(x, 0.0, 1.0), In(y, 0.0, 1.0), In(k, 0.1, 1.0)]
    sys_ = PDESystem(eq, bcs, doms, [t, x, y, k], [U], ps=[a], defaults={a: 0.5})
    rng = np.random.default_rng(5)
    X = rng.random((4, n_obs))
    X[3] = 0.1 + 0.9 * X[3]
    yobs = np.exp(-2 * np.pi ** 2 * X[3] * X[0]) * np.sin(np.pi * X[1]) * np.sin(np.pi * X[2])
    return Config("cfg5_heat_inverse", sys_, [mlp(4, width, hidden)],
                  QuasiRandomTraining(points, bcs_points=bcs_points, resampling=False, seed=5), multioutput=True,
                  param_estim=True, additional_loss=DataLoss("u", X, yobs), n_pde_points=points)


def lorenz_bpinn(seed: int = 100, width: int = 7):
    """The reference's inverse BayesianPINN Lorenz test (test/PDEBPINN/bpinn_pde__bpinn_pde_inv_ii_lorenz_system.jl):
    unknown σ_ in x' = σ_ (y - x), three 1 -> width -> width -> 1 tanh networks, observations of (x, y, z) at
    t = 0, 0.05, ..., 1 with 5 % multiplicative noise (seeded numpy in place of Julia's RNG; the ODE solved with
    scipy's RK45 at rtol 1e-10).  Returns (pde_system, chains, dataset_pde)."""
    from scipy.integrate import solve_ivp
    t, s_ = parameters("t σ_")
    x, y, z = variables("x y z")
    Dt = Differential(t)
    eqs = [Eq(Dt(x(t)), s_ * (y(t) - x(t))), Eq(Dt(y(t)), x(t) * (28.0 - z(t)) - y(t)),
           Eq(Dt(z(t)), x(t) * y(t) - 8.0 / 3.0 * z(t))]
    bcs = [Eq(x(0.0), 1.0), Eq(y(0.0), 0.0), Eq(z(0.0), 0.0)]
    sys_ = PDESystem(eqs, bcs, [In(t, 0.0, 1.0)], [t], [x(t), y(t), z(t)], ps=[s_], defaults={s_: 1.0})
    chains = [Chain(Dense(1, width, "tanh"), Dense(width, width, "tanh"), Dense(width, 1)) for _ in range(3)]
    f = lambda _, u: [10.0 * (u[1] - u[0]), u[0] * (28.0 - u[2]) - u[1], u[0] * u[1] - 8.0 / 3.0 * u[2]]   # noqa: E731
    ts = np.linspace(0.0, 1.0, 21)
    us = solve_ivp(f, (0.0, 1.0), [1.0, 0.0, 0.0], t_eval=ts, rtol=1e-10, atol=1e-12).y
    us = us + 0.05 * np.random.default_rng(seed).standard_normal(us.shape) * us
    return sys_, chains, [np.stack([us[i], ts], axis=1) for i in range(3)]


ALL = {"cfg1": config1, "cfg2": config2, "cfg3": config3, "cfg4": config4, "cfg5": config5}
