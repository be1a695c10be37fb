"""NNODE host side (no GPU): tracing and lowering of f, point sets and weights of every strategy, loss assembly against
the float64 oracle, gelu's derivatives, and the refusals (reference src/ode_solve.jl)."""
import math

import numpy as np
import pytest
import sympy as sp
import torch

import neuralpde_jl_b200 as npde
from neuralpde_jl_b200.engine import REDUCE_MEAN, REDUCE_WSUM
from nnode_oracle import NNODEOracle, act, mlp

torch.set_default_dtype(torch.float64)


# ---- problems (the reference's test/NNODE files) -------------------------------------------------------------------
def scalar_cos():                       # nnode__scalar.jl, nnode__training_strategy_others.jl
    return npde.ODEProblem(npde.ODEFunction(lambda u, p, t: sp.cos(2 * sp.pi * t),
                                            analytic=lambda u0, p, t: math.sin(2 * math.pi * t) / (2 * math.pi)),
                           0.0, (0.0, 1.0))


def example2():                         # nnode__ode_example_2.jl
    return npde.ODEProblem(npde.ODEFunction(lambda u, p, t: -u / 5 + sp.exp(-t / 5) * sp.cos(t),
                                            analytic=lambda u0, p, t: math.exp(-t / 5) * (u0 + math.sin(t))),
                           0.0, (0.0, 1.0))


def example3():                         # nnode__ode_example_3.jl
    return npde.ODEProblem(npde.ODEFunction(lambda u, p, t: [sp.cos(2 * sp.pi * t), sp.sin(2 * sp.pi * t)],
                                            analytic=lambda u0, p, t: [math.sin(2 * math.pi * t) / (2 * math.pi),
                                                                       -math.cos(2 * math.pi * t) / (2 * math.pi)]),
                           [0.0, -1.0 / (2 * math.pi)], (0.0, 1.0))


def ode_i():                            # nnode__ode_i.jl
    def f(u, p, t):
        return [t ** 3 + 2 * t + t ** 2 * ((1 + 3 * t ** 2) / (1 + t + t ** 3))
                - u[0] * (t + (1 + 3 * t ** 2) / (1 + t + t ** 3))]
    return npde.ODEProblem(npde.ODEFunction(f, analytic=lambda u0, p, t: [math.exp(-t ** 2 / 2) / (1 + t + t ** 3) + t ** 2]),
                           [1.0], (0.0, 1.0))


def lotka_volterra():                   # nnode__training_strategy_with_tstops.jl / _weightedintervaltraining.jl
    return npde.ODEProblem(lambda u, p, t: [p[0] * u[0] - p[1] * u[0] * u[1], -p[2] * u[1] + p[3] * u[0] * u[1]],
                           [1.0, 1.0], (0.0, 3.0), [1.5, 1.0, 3.0, 1.0])


def lorenz(p=(1.0, 1.0, 1.0), tspan=(0.0, 1.0)):   # nnode__ode_parameter_estimation*.jl
    return npde.ODEProblem(lambda u, p, t: [p[0] * (u[1] - u[0]), u[0] * (p[1] - u[2]) - u[1], u[0] * u[1] - p[2] * u[2]],
                           [1.0, 0.0, 0.0], tspan, list(p))


def chain(n_out, width=5, act_="sigmoid", hidden=1):
    layers = [npde.Dense(1, width, act_)] + [npde.Dense(width, width, act_) for _ in range(hidden - 1)]
    return npde.Chain(*layers, npde.Dense(width, n_out))


def _run_prog(spec, rows, taps, params):
    val = []
    for op, a, b, imm in spec.prog:
        f = {"const": lambda: np.full(rows.shape[1], imm), "coord": lambda: rows[a], "tap": lambda: taps[a],
             "param": lambda: np.full(rows.shape[1], params[a]),
             "add": lambda: val[a] + val[b], "sub": lambda: val[a] - val[b], "mul": lambda: val[a] * val[b],
             "div": lambda: val[a] / val[b], "neg": lambda: -val[a], "powi": lambda: val[a] ** int(imm),
             "pow": lambda: val[a] ** val[b], "sin": lambda: np.sin(val[a]), "cos": lambda: np.cos(val[a]),
             "exp": lambda: np.exp(val[a]), "log": lambda: np.log(val[a]), "tanh": lambda: np.tanh(val[a]),
             "sqrt": lambda: np.sqrt(val[a]), "abs": lambda: np.abs(val[a])}[op]
        val.append(f())
    return val[-1]


def oracle_taps(spec, oracle, th, t):
    """the network outputs N_k and dN_k/dt the term's taps name, from the oracle's MLP"""
    tt = torch.tensor(t).requires_grad_(True)
    N = mlp(th, oracle.dims, oracle.acts, tt[None, :])
    dN = torch.stack([torch.autograd.grad(N[k].sum(), tt, retain_graph=True)[0] for k in range(oracle.n)])
    return [(dN if tp.order else N)[tp.out].detach().numpy() for tp in spec.taps]


def host_terms(rep, oracle, theta):
    """every term's loss, the engine's reduction restated on the host, from the program run on oracle taps"""
    th = torch.tensor(np.asarray(theta, dtype=np.float64))
    out = []
    for i, spec in enumerate(rep.specs):
        X = rep.point_sets[i]
        taps = oracle_taps(spec, oracle, th, X[0])
        r = _run_prog(spec, X, taps, np.asarray(theta)[rep.n_net:])
        if spec.reduction == REDUCE_MEAN:
            out.append(np.mean(r ** 2))
        else:
            out.append(spec.scale * np.sum(rep.quad_weights[i] * r ** 2))
    return np.array(out)


# ---- tracing and lowering ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("make, estim", [(scalar_cos, False), (example2, False), (example3, False), (ode_i, False),
                                         (lotka_volterra, False), (lotka_volterra, True), (lorenz, True)])
def test_lowered_program_matches_oracle_residual(make, estim):
    prob = make()
    n = 1 if np.ndim(prob.u0) == 0 else len(prob.u0)
    ch = chain(n, 6, "tanh")
    ds = [list(np.linspace(0, 1, 4)) for _ in range(n)] + [list(np.linspace(0, 1, 4)), [1.0] * 4] if estim else []
    alg = npde.NNODE(ch, npde.Adam(0.1), strategy=npde.GridTraining(0.1), param_estim=estim, dataset=ds)
    rep = npde.NNODERepresentation(prob, alg)
    theta = np.asarray(rep.flat_init_params, dtype=np.float64).copy()
    if estim:
        theta[rep.n_net:] += np.linspace(0.1, 0.3, theta.size - rep.n_net)
    orc = NNODEOracle(prob, ch, param_estim=estim)
    t = np.linspace(prob.tspan[0] + 0.05, prob.tspan[1] - 0.05, 9)
    R = orc.residual(torch.tensor(theta), torch.tensor(t)).detach().numpy()
    for k in range(n):
        spec = rep.specs[k]
        assert [tp.net for tp in spec.taps] == [0] * len(spec.taps) and {tp.out for tp in spec.taps} <= set(range(n))
        r = _run_prog(spec, t[None, :], oracle_taps(spec, orc, torch.tensor(theta), t), theta[rep.n_net:])
        np.testing.assert_allclose(r, R[k], rtol=1e-13, atol=1e-13)


def test_scalar_and_vector_tracing_shapes():
    assert npde.NNODERepresentation(scalar_cos(), npde.NNODE(chain(1), npde.Adam(0.1)), dt=0.1).n == 1
    rep = npde.NNODERepresentation(example3(), npde.NNODE(chain(2), npde.Adam(0.1)), dt=0.1)
    assert rep.n == 2 and rep.term_names == ["residual_1", "residual_2"]
    # param_estim: θ = [network, p], p starting at the problem's p
    rep = npde.NNODERepresentation(lorenz(), npde.NNODE(chain(3), npde.Adam(0.1), param_estim=True,
                                                         dataset=[[1.0], [0.0], [0.0], [0.0], [1.0]]), dt=0.1)
    assert list(rep.flat_init_params.p) == [1.0, 1.0, 1.0] and rep.flat_init_params.depvar.size == rep.n_net


# ---- point sets and weights --------------------------------------------------------------------------------------
def test_point_sets_of_every_strategy():
    prob = lotka_volterra()
    ch = chain(2)
    rep = npde.NNODERepresentation(prob, npde.NNODE(ch, npde.Adam(0.1), strategy=npde.GridTraining(0.3)))
    np.testing.assert_allclose(rep.point_sets[0][0], 0.3 * np.arange(11))        # Julia range 0:0.3:3
    assert all(s.reduction == REDUCE_WSUM and s.scale == 1 / 11 for s in rep.specs)
    rep = npde.NNODERepresentation(prob, npde.NNODE(ch, npde.Adam(0.1), strategy=npde.GridTraining(0.3), batch=False))
    assert all(s.scale == 1.0 for s in rep.specs)
    # dt without a strategy: GridTraining(dt); neither: Gauss-Legendre on [t0, t1]
    rep = npde.NNODERepresentation(prob, npde.NNODE(ch, npde.Adam(0.1)), dt=0.5)
    np.testing.assert_allclose(rep.point_sets[0][0], 0.5 * np.arange(7))
    rep = npde.NNODERepresentation(prob, npde.NNODE(ch, npde.Adam(0.1)))
    g, w = np.polynomial.legendre.leggauss(16)
    np.testing.assert_allclose(rep.point_sets[0][0], 1.5 * g + 1.5)
    np.testing.assert_allclose(rep.quad_weights[0], 1.5 * w)
    assert rep.term_names == ["quadrature"] and rep.specs[0].scale == 1.0
    # WeightedIntervalTraining: trunc(points * w_i) uniform points in sub-interval i
    wit = npde.WeightedIntervalTraining([0.7, 0.2, 0.1], 200)
    ts = wit.sample(0.0, 3.0)
    assert ts.size == 140 + 40 + 20
    assert np.all((ts[:140] >= 0) & (ts[:140] < 1)) and np.all((ts[140:180] >= 1) & (ts[140:180] < 2))
    assert np.all((ts[180:] >= 2) & (ts[180:] < 3))
    assert npde.WeightedIntervalTraining([0.3, 0.3, 0.4], 3).sample(0.0, 3.0).size == 0 + 0 + 1
    # StochasticTraining: device-sampled mean terms, weight N without batch
    rep = npde.NNODERepresentation(prob, npde.NNODE(ch, npde.Adam(0.1), strategy=npde.StochasticTraining(100), batch=False))
    assert rep.point_sets == [None, None] and all(s.reduction == REDUCE_MEAN for s in rep.specs)
    np.testing.assert_array_equal(rep.term_weights, [100.0, 100.0])
    # tstops: (L N + L_t N_t) / (N + N_t) through the weights, L + L_t for Quadrature
    rep = npde.NNODERepresentation(prob, npde.NNODE(ch, npde.Adam(0.1), strategy=npde.GridTraining(0.3)), tstops=[0.5, 1.5])
    np.testing.assert_allclose(rep.term_weights, [11 / 13, 11 / 13, 2 / 13, 2 / 13])
    assert rep.term_names[2:] == ["tstops_1", "tstops_2"] and rep.specs[2].scale == 0.5
    rep = npde.NNODERepresentation(prob, npde.NNODE(ch, npde.Adam(0.1)), tstops=[0.5, 1.5])
    np.testing.assert_array_equal(rep.term_weights, [1.0, 1.0, 1.0])
    rep = npde.NNODERepresentation(prob, npde.NNODE(ch, npde.Adam(0.1), strategy=wit), tstops=[0.5, 1.5])
    np.testing.assert_allclose(rep.term_weights, [200 / 202, 200 / 202, 2 / 202, 2 / 202])


# ---- loss assembly against the oracle -----------------------------------------------------------------------------
def _cases():
    lv, lz = lotka_volterra(), lorenz()
    t_d = np.linspace(0.0, 1.0, 6)
    ds = [list(np.cos(t_d)), list(np.sin(t_d)), list(t_d ** 2), list(t_d), list(np.full(6, 0.2))]
    out = []
    for batch in (True, False):
        out += [("grid", lv, dict(strategy=npde.GridTraining(0.25), batch=batch), {}),
                ("grid_tstops", lv, dict(strategy=npde.GridTraining(0.25), batch=batch), dict(tstops=[0.3, 1.7, 2.9])),
                ("wit", lv, dict(strategy=npde.WeightedIntervalTraining([0.5, 0.5], 20), batch=batch), {}),
                ("quad", lv, dict(batch=batch), {}),
                ("quad_tstops", lv, dict(batch=batch), dict(tstops=[0.3, 1.7])),
                ("data", lz, dict(strategy=npde.GridTraining(0.1), batch=batch, param_estim=True, dataset=ds), {}),
                ("collocate", lz, dict(strategy=npde.GridTraining(0.1), batch=batch, param_estim=True, dataset=ds,
                                       estim_collocate=True), {}),
                ("additional", scalar_cos(), dict(strategy=npde.GridTraining(0.1), batch=batch,
                                                  additional_loss=npde.DataLoss(0, t_d, np.sin(2 * np.pi * t_d) / 6)),
                 dict(tstops=[0.35]))]
    return out


def oracle_total(rep, orc, theta, alg, kw, derivative="exact"):
    """the reference's total_loss at θ (a tensor to differentiate, or an array)"""
    th = theta if isinstance(theta, torch.Tensor) else torch.tensor(np.asarray(theta, dtype=np.float64))
    s = rep.strategy
    if isinstance(s, npde.QuadratureTraining):
        main = orc.quadrature_loss(th, torch.tensor(rep.point_sets[0][0]), torch.tensor(rep.quad_weights[0]), derivative)
        n_orig = None
    else:
        t = torch.tensor(rep.point_sets[0][0])
        main = orc.inner_loss(th, t, alg.batch, derivative)
        n_orig = t.numel() if isinstance(s, npde.GridTraining) else s.points
    extras = []
    if alg.param_estim and alg.dataset:
        extras.append(orc.l2_data(th, alg.dataset))
        if alg.estim_collocate:
            extras.append(orc.l2_collocate(th, alg.dataset, derivative))
    if alg.additional_loss is not None:
        dl = alg.additional_loss
        extras.append(orc.data_loss(th, dl.depvar, dl.points, dl.values))
    return orc.total_loss(th, main, extras, kw.get("tstops"), n_orig, alg.batch, derivative)


def oracle_terms(rep, orc, theta, alg, kw):
    """each engine term's loss restated from the oracle's per-component pieces (exact d/dt), by term name"""
    th = theta if isinstance(theta, torch.Tensor) else torch.tensor(np.asarray(theta, dtype=np.float64))
    T = lambda v: torch.tensor(np.asarray(v, dtype=np.float64))          # noqa: E731
    red = (lambda q: q.mean()) if alg.batch else (lambda q: q.sum())     # noqa: E731
    ds = alg.dataset
    out = []
    for i, name in enumerate(rep.term_names):
        kind, _, k = name.rpartition("_")
        k = int(k) - 1 if k.isdigit() else 0
        if name == "quadrature":
            t, w = T(rep.point_sets[i][0]), T(rep.quad_weights[i])
            out.append((w * (orc.residual(th, t) ** 2).sum(0) ** 2).sum())
        elif kind in ("residual", "tstops"):
            t = T(rep.point_sets[i][0] if kind == "residual" else kw["tstops"])
            out.append(red(orc.residual(th, t)[k] ** 2))
        elif kind == "l2_data":
            out.append(((orc.phi(th, T(ds[-2]))[k] - T(ds[k])) ** 2).sum())
        elif kind == "collocation":
            t = T(ds[-2])
            uh = torch.stack([T(ds[j]) for j in range(orc.n)])
            out.append((T(ds[-1]) * (orc.dphi(th, t)[k] - orc.fval(uh, th, t)[k]) ** 2).sum())
        else:
            dl = alg.additional_loss
            out.append(orc.data_loss(th, dl.depvar, dl.points, dl.values))
    return out


@pytest.mark.parametrize("i", range(16))
def test_loss_assembly_matches_oracle(i):
    name, prob, akw, kw = _cases()[i]
    n = 1 if np.ndim(prob.u0) == 0 else len(prob.u0)
    ch = chain(n, 6, "tanh", hidden=2)
    alg = npde.NNODE(ch, npde.Adam(0.1), **akw)
    rep = npde.NNODERepresentation(prob, alg, **kw)
    orc = NNODEOracle(prob, ch, param_estim=alg.param_estim)
    theta = rep.flat_init_params
    total = float(np.dot(rep.term_weights, host_terms(rep, orc, theta)))
    ref = float(oracle_total(rep, orc, theta, alg, kw).detach())
    assert abs(total - ref) <= 1e-12 * abs(ref), (name, total, ref)
    terms = [float(v.detach()) for v in oracle_terms(rep, orc, theta, alg, kw)]
    np.testing.assert_allclose(host_terms(rep, orc, theta), terms, rtol=1e-12)


def test_fixed_quadrature_within_reltol_of_adaptive():
    """16 Gauss-Legendre nodes against scipy's adaptive quad at θ0, within the reference's default reltol 1e-3"""
    from scipy.integrate import quad
    for prob, n in ((scalar_cos(), 1), (example2(), 1), (example3(), 2), (ode_i(), 1)):
        ch = chain(n, 5, "sigmoid")
        rep = npde.NNODERepresentation(prob, npde.NNODE(ch, npde.Adam(0.1)))
        orc = NNODEOracle(prob, ch)
        th = torch.tensor(np.asarray(rep.flat_init_params))
        fixed = float(orc.quadrature_loss(th, torch.tensor(rep.point_sets[0][0]), torch.tensor(rep.quad_weights[0])).detach())
        g = lambda t: float((orc.residual(th, torch.tensor([t])) ** 2).sum().detach() ** 2)   # noqa: E731
        adaptive = quad(g, *prob.tspan, epsabs=1e-14, epsrel=1e-12)[0]
        assert abs(fixed - adaptive) <= 1e-3 * abs(adaptive), (fixed, adaptive)


def test_fd_and_exact_time_derivative_distance():
    """the reference's default forward difference (ε = sqrt(eps)) against the exact d/dt the engine takes: the relative
    loss difference at θ0 on the test problems, pinned at its measured size"""
    dist = []
    for prob, n in ((scalar_cos(), 1), (example2(), 1), (example3(), 2), (ode_i(), 1), (lotka_volterra(), 2)):
        ch = chain(n, 5, "sigmoid")
        alg = npde.NNODE(ch, npde.Adam(0.1), strategy=npde.GridTraining(0.05))
        rep = npde.NNODERepresentation(prob, alg)
        orc = NNODEOracle(prob, ch)
        ex = float(oracle_total(rep, orc, rep.flat_init_params, alg, {}, "exact").detach())
        fd = float(oracle_total(rep, orc, rep.flat_init_params, alg, {}, "fd").detach())
        dist.append(abs(fd - ex) / ex)
    # measured (float64, torch's CPU kernels): scalar 2.345e-9, example 2 3.659e-9, example 3 9.41e-12, ODE I 7.18e-11,
    # Lotka-Volterra 2.225e-10 -- the forward difference's truncation error, far below every bound the tests apply
    np.testing.assert_allclose(dist, [2.345e-9, 3.659e-9, 9.41e-12, 7.18e-11, 2.225e-10], rtol=0.1)


# ---- gelu ------------------------------------------------------------------------------------------------------------
def gelu_derivs(z):
    """the closed form the kernel evaluates (ffma_kernel.cuh gelu_eval4), restated"""
    c, k = math.sqrt(2 / math.pi), 0.044715
    t = np.tanh(c * (z + k * z ** 3))
    t1 = 1 - t * t
    t2, t3, t4 = -2 * t * t1, t1 * (6 * t * t - 2), 8 * t * t1 * (2 - 3 * t * t)
    u1, u2, u3 = c * (1 + 3 * k * z * z), 6 * c * k * z, 6 * c * k
    T1, T2 = t1 * u1, t2 * u1 ** 2 + t1 * u2
    T3 = t3 * u1 ** 3 + 3 * t2 * u1 * u2 + t1 * u3
    T4 = t4 * u1 ** 4 + 6 * t3 * u1 ** 2 * u2 + t2 * (3 * u2 ** 2 + 4 * u1 * u3)
    return 0.5 * z * (1 + t), 0.5 * (1 + t + z * T1), 0.5 * (2 * T1 + z * T2), 0.5 * (3 * T2 + z * T3), 0.5 * (4 * T3 + z * T4)


def test_gelu_derivatives_against_autograd():
    z = torch.linspace(-6, 6, 241).requires_grad_(True)
    ds = [act("gelu", z)]
    for _ in range(4):
        ds.append(torch.autograd.grad(ds[-1].sum(), z, create_graph=True)[0])
    for mine, ref in zip(gelu_derivs(z.detach().numpy()), ds):
        np.testing.assert_allclose(mine, ref.detach().numpy(), rtol=1e-12, atol=1e-11)
    assert npde.Dense(2, 3, "gelu").activation == "gelu" and npde.engine.ACT["gelu"] == 6


# ---- refusals --------------------------------------------------------------------------------------------------------
def test_refusals():
    ch, opt = chain(1), npde.Adam(0.1)
    prob = scalar_cos()
    R = npde.NNODERepresentation
    for s in (npde.GridTraining(0.1), npde.StochasticTraining(10), npde.WeightedIntervalTraining([1.0], 10)):
        with pytest.raises(ValueError, match="autodiff not supported for %s" % type(s).__name__):
            R(prob, npde.NNODE(ch, opt, strategy=s, autodiff=True))
    with pytest.raises(ValueError, match="QuasiRandomTraining is not supported by NNODE"):
        R(prob, npde.NNODE(ch, opt, strategy=npde.QuasiRandomTraining(10)))
    with pytest.raises(ValueError, match="complex"):
        npde.ODEProblem(lambda u, p, t: u, 1.0 + 2.0j, (0.0, 1.0))
    with pytest.raises(ValueError, match="complex"):
        npde.ODEProblem(lambda u, p, t: u, 1.0, (0.0, 1.0), [1j])
    with pytest.raises(ValueError, match="complex"):
        R(prob, npde.NNODE(ch, opt, np.zeros(ch.n_params, dtype=complex)))
    with pytest.raises(ValueError, match="out-of-place"):
        npde.ODEProblem(lambda du, u, p, t: None, 1.0, (0.0, 1.0))
    with pytest.raises(ValueError, match="DataLoss.*component index"):
        npde.NNODE(ch, opt, additional_loss=lambda phi, th: 0.0)
    for bad in ([[1.0], [0.0]], [[1.0], [0.0], "x"], [[1, 2], [0, 1], [1, 1]]):
        with pytest.raises(ValueError, match="Invalid dataset"):
            R(prob, npde.NNODE(ch, opt, dataset=bad), dt=0.1)
    with pytest.raises(ValueError, match="Dataset or an additional loss is required"):
        R(lorenz(), npde.NNODE(chain(3), opt, param_estim=True), dt=0.1)
    with pytest.raises(ValueError, match="Dataset is required"):
        R(prob, npde.NNODE(ch, opt, estim_collocate=True), dt=0.1)
    for mode in ("tc_bf16", "tc_split"):
        with pytest.raises(ValueError, match="FFMA kernel"):
            npde.NNODE(ch, opt, mode=mode)
    with pytest.raises(ValueError, match="could not be traced"):
        R(npde.ODEProblem(lambda u, p, t: math.cos(t), 0.0, (0.0, 1.0)), npde.NNODE(ch, opt), dt=0.1)
    with pytest.raises(ValueError, match="unsupported expression node"):
        R(npde.ODEProblem(lambda u, p, t: sp.erf(t), 0.0, (0.0, 1.0)), npde.NNODE(ch, opt), dt=0.1)
    with pytest.raises(ValueError, match="1 input and 2 outputs"):
        R(example3(), npde.NNODE(ch, opt), dt=0.1)
    with pytest.raises(ValueError, match="tc_f64"):
        R(prob, npde.NNODE(ch, opt, np.zeros(ch.n_params, dtype=np.float32), mode="tc_f64"), dt=0.1)
    # solve on an OptimizationProblem keeps its keywords
    with pytest.raises(TypeError, match="unexpected keyword"):
        npde.solve(npde.OptimizationProblem(None, np.zeros(1)), opt, saveat=0.1)
    # maxiters is required for an ODE problem (no silent default)
    with pytest.raises(TypeError, match="needs maxiters"):
        npde.solve(prob, npde.NNODE(ch, opt), dt=0.1)


def test_scalar_u0_accepts_a_one_element_result():
    prob = npde.ODEProblem(lambda u, p, t: [sp.cos(2 * sp.pi * t)], 0.0, (0.0, 1.0))
    rep = npde.NNODERepresentation(prob, npde.NNODE(chain(1), npde.Adam(0.1)), dt=0.1)
    ref = npde.NNODERepresentation(scalar_cos(), npde.NNODE(chain(1), npde.Adam(0.1)), dt=0.1)
    assert rep.specs[0].prog == ref.specs[0].prog
    with pytest.raises(ValueError, match="f returns 2 components, u0 has 1"):
        npde.NNODERepresentation(npde.ODEProblem(lambda u, p, t: [t, t], 0.0, (0.0, 1.0)),
                                 npde.NNODE(chain(1), npde.Adam(0.1)), dt=0.1)


def test_save_times():
    from neuralpde_jl_b200.ode import _save_times
    np.testing.assert_allclose(_save_times(0.0, 1.0, 0.25, None, True), [0, 0.25, 0.5, 0.75, 1.0])
    np.testing.assert_allclose(_save_times(0.0, 1.0, [0.1, 0.7], None, True), [0.1, 0.7])
    np.testing.assert_allclose(_save_times(0.0, 1.0, None, 0.5, True), [0, 0.5, 1.0])
    assert _save_times(0.0, 1.0, None, None, True).size == 100
    np.testing.assert_allclose(_save_times(0.0, 1.0, None, None, False), [0.0, 1.0])
