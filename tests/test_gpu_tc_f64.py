"""PINN_MODE_TC_F64 (mode="tc_f64"): the FFMA kernel with its layer products on the FP64 tensor cores (DMMA).

It is held to the float64 goldens at DESIGN section 3's fp64 tolerances (loss 1e-10, gradient 1e-9), and to the FFMA fp64
path on the same inputs at 1e-12 norm-relative (only the summation order of the layer products differs), over a sweep of
widths, input counts, channel counts, point counts and both activation-buffer / weight placements, and on the integral,
fixed-network and functional-term instantiations against their float64 oracles."""
import os

import numpy as np
import pytest

import neuralpde_jl_b200 as npde
from neuralpde_jl_b200 import engine as E
from oracle import reference as R

from cases import CASES, FULL_CASES, point_sets
from helpers import engine_eval_sets, load_golden, rel

pytestmark = pytest.mark.gpu

GOLDEN = ["cfg1", "cfg2_small", "cfg2_full", "cfg3_small", "cfg5_small", "mixed", "neumann_sin", "third_order_ode",
          "third_order_2d", "poisson1d_wide", "burgers_wide", "cfg4_tiny"]


def _close(a, b, tol=1e-12):
    """(total, terms, grad) of two evaluations agree to tol, norm-relative"""
    assert abs(a[0] - b[0]) <= tol * abs(b[0]), (a[0], b[0])
    assert rel(a[1], b[1]) <= tol, rel(a[1], b[1])
    if b[2] is not None:
        assert rel(a[2], b[2]) <= tol, rel(a[2], b[2])


@pytest.mark.parametrize("name", GOLDEN)
def test_golden_and_ffma(name):
    if name == "cfg2_full":       # the full-shape golden keeps checksums of its inputs; they are regenerated from seeds
        g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", name + ".npz"))
        sets, qw, _ = point_sets(FULL_CASES[name]())
        g = dict(g, theta=FULL_CASES[name]().init_params(np.float64, seed=1))
    else:
        g, sets, qw = load_golden(name)
    cfg = (FULL_CASES if name == "cfg2_full" else CASES)[name]
    _, total, terms, grad = engine_eval_sets(cfg(), np.float64, sets, qw, mode="tc_f64", theta=g["theta"])
    assert abs(total - float(g["total"])) <= 1e-10 * abs(float(g["total"]))
    np.testing.assert_allclose(terms, g["terms"], rtol=1e-9, atol=1e-300)
    # the full-shape golden stores its gradient in float32 (tests/golden/make_golden_full.py): rounding is 3e-8 there
    assert rel(grad, g["grad"]) < (1e-7 if name == "cfg2_full" else 1e-9)
    _, *ref = engine_eval_sets(cfg(), np.float64, sets, qw, mode="ffma", theta=g["theta"])
    _close((total, terms, grad), ref)


# ---- shape sweep through the engine spec: one term whose program sums C channels' worth of taps -----------------------
def _spec(mode, width, n_in, C, hidden=2, outs=1):
    dims = [n_in] + [width] * hidden + [outs]
    net = E.NetSpec(dims, ["tanh"] * hidden + ["identity"], 0)
    n1 = min(C - 1, n_in)
    n2 = min(C - 1 - n1, n1)
    n3 = C - 1 - n1 - n2                       # pure third derivatives (along dir1's directions that have a second)
    assert n3 <= n2
    taps = [E.TapSpec(net=0, out=outs - 1)]
    taps += [E.TapSpec(net=0, order=1, dirs=[i]) for i in range(n1)]
    taps += [E.TapSpec(net=0, order=2, dirs=[i, i]) for i in range(n2)]
    taps += [E.TapSpec(net=0, order=3, dirs=[i, i, i]) for i in range(n3)]
    prog = [("tap", t, 0, 0.0) for t in range(len(taps))]
    acc = 0
    for t in range(1, len(taps)):
        prog.append(("add", acc, t, 0.0))
        acc = len(prog) - 1
    prog.append(("coord", 0, 0, 0.0))
    prog.append(("mul", acc, len(prog) - 1, 0.0))
    term = E.TermSpec(dim=n_in, taps=taps, prog=prog)
    return E.ProblemSpec(nets=[net], terms=[term], n_theta=net.n_params, dtype="float64", mode=mode)


def _eval(mode, width, n_in, C, n, hidden=2, outs=1, seed=0):
    spec = _spec(mode, width, n_in, C, hidden, outs)
    rng = np.random.default_rng(seed)
    th = rng.uniform(-1, 1, spec.n_theta) / np.sqrt(width)
    eng = E.Engine(spec)
    eng.set_points_host(0, rng.uniform(-1, 1, (n_in, n)))
    return eng, th, eng.loss_grad_host(th, None, True)


SWEEP = ([(w, 2, 3, 1000, 2, 1) for w in (12, 15, 18, 64, 128, 256)]       # widths
         + [(18, 8, c, 33, 2, 1) for c in range(1, 11)]                    # C = 1..10 on 8 inputs
         + [(15, 1, c, 31, 3, 1) for c in range(1, 5)]                     # 1 input, up to a third derivative
         + [(64, 2, 3, n, 2, 1) for n in (1, 31, 32, 33, 1000)]            # partial and whole tiles
         + [(18, 2, 3, 100, 2, 3)]                                         # a tap of output 3 of 3
         + [(64, 2, 2, 200, 6, 1)]                                         # smem buffers, streamed weights
         + [(128, 2, 3, 200, 3, 1), (256, 8, 10, 64, 2, 1)])               # global buffers, streamed weights


@pytest.mark.parametrize("width,n_in,C,n,hidden,outs", SWEEP)
def test_shape_sweep_matches_ffma(width, n_in, C, n, hidden, outs):
    _, _, got = _eval(E.MODE_TC_F64, width, n_in, C, n, hidden, outs)
    _, _, ref = _eval(E.MODE_FFMA, width, n_in, C, n, hidden, outs)
    _close(got, ref)


def test_loss_only_residual_probe_and_grad_stats():
    eng, th, (total, terms, grad) = _eval(E.MODE_TC_F64, 64, 2, 3, 333)
    ref, _, _ = _eval(E.MODE_FFMA, 64, 2, 3, 333)
    t2, terms2, g2 = eng.loss_grad_host(th, None, False)
    assert g2 is None and t2 == total and np.array_equal(terms2, terms)
    np.testing.assert_allclose(eng.term_residual_host(0, th, 333), ref.term_residual_host(0, th, 333), rtol=1e-11,
                               atol=1e-13)
    np.testing.assert_allclose(eng.term_grad_stats_host(0, th), ref.term_grad_stats_host(0, th), rtol=1e-11)


def test_two_runs_bit_identical_and_one_launch():
    eng, th, a = _eval(E.MODE_TC_F64, 128, 2, 3, 1000)
    n0 = eng.launch_count()
    b = eng.loss_grad_host(th, None, True)
    assert eng.launch_count() - n0 == 1
    assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


def test_device_adam_takes_the_host_loops_steps():
    eng, th0, _ = _eval(E.MODE_TC_F64, 64, 2, 3, 500)
    th = th0.copy()
    lr, b1, b2, eps = 1e-3, 0.9, 0.999, 1e-8
    m, v = np.zeros_like(th), np.zeros_like(th)
    for t in range(1, 6):
        _, _, g = eng.loss_grad_host(th, None, True)
        m = b1 * m + (1 - b1) * g
        v = b2 * v + (1 - b2) * g * g
        c2 = np.sqrt(1 - b2 ** t)
        th = th - lr * c2 / (1 - b1 ** t) * m / (np.sqrt(v) + eps * c2)
    eng.adam_begin(th0, lr, b1, b2, eps)
    n0 = eng.launch_count()
    eng.adam_iterate(5)
    assert eng.launch_count() - n0 == 5
    assert rel(eng.adam_theta(), th) < 1e-9


@pytest.mark.parametrize("opt", ["LBFGS", "BFGS"])
def test_quasi_newton_iterates_like_ffma(opt):
    from neuralpde_jl_b200 import configs
    cfg = configs.config2(n=16, width=16, hidden=3)
    res = {}
    for mode in ("ffma", "tc_f64"):
        prob = npde.discretize(cfg.pde_system, cfg.discretization(dtype=np.float64, mode=mode))
        res[mode] = npde.solve(prob, getattr(npde, opt)(), maxiters=10)
    assert rel(res["tc_f64"].u, res["ffma"].u) < 1e-9
    assert abs(res["tc_f64"].objective - res["ffma"].objective) <= 1e-9 * abs(res["ffma"].objective)


# ---- the integral, fixed-network and functional-term instantiations against their float64 oracles ----------------------
def test_integro_differential_equation():
    import integral_cases as IC
    from integral_oracle import IntegralProblem
    sys_, chains, dx = IC.ide1()
    rep = npde.symbolic_discretize(sys_, IC.discretization(chains, dx, np.float64, mode="tc_f64"))
    total, _, grad = rep.engine.loss_grad_host(rep.flat_init_params, None, True)
    ps, bs = R.generate_training_sets(sys_.domain, dx, sys_.eqs, sys_.bcs, sys_.ivs, sys_.dvs)
    L, _, G = IntegralProblem(sys_, IC.chain_specs(chains)).loss_and_grad(rep.flat_init_params, ps, bs)
    assert abs(total - L) <= 1e-10 * abs(L) and rel(grad, G) < 1e-9


def test_fixed_network():
    from adapter_oracle import FixedProblem
    x, y = npde.parameters("x y")
    u = npde.variables("u")
    Dx, Dy = npde.Differential(x), npde.Differential(y)
    student = npde.Chain(npde.Dense(2, 12, "tanh"), npde.Dense(12, 12, "tanh"), npde.Dense(12, 1))
    teacher = npde.Chain(npde.Dense(2, 6, "sigmoid"), npde.Dense(6, 5, "sin"), npde.Dense(5, 1))
    rng = np.random.default_rng(3)
    tt = npde.initialparameters(rng, teacher, np.float64)
    pb = npde.register_symbolic(npde.Phi(teacher, 0, teacher.n_params, np.float64), tt, "phi_tc_f64")
    eq = npde.Eq((Dx**2)(u(x, y)) + (Dy**2)(u(x, y)), Dx(pb(x, y)) + (Dy**2)(pb(x, y)))
    bcs = [npde.Eq(u(0.2, y), pb(0.2, y)), npde.Eq(u(x, 0), 0.0)]
    sys_ = npde.PDESystem([eq], bcs, [npde.In(x, 0.2, 1.0), npde.In(y, 0.0, 1.0)], [x, y], [u(x, y)])
    th = npde.initialparameters(np.random.default_rng(5), student, np.float64)
    got = {}
    for mode in ("ffma", "tc_f64"):
        rep = npde.symbolic_discretize(sys_, npde.PhysicsInformedNN(student, npde.GridTraining(0.1), init_params=th,
                                                                    mode=mode))
        got[mode] = rep.engine.loss_grad_host(th, None, True)
    ps, bs = R.generate_training_sets(sys_.domain, 0.1, sys_.eqs, sys_.bcs, sys_.ivs, sys_.dvs)
    L, _, G = FixedProblem(sys_, [(student.dims, student.acts)], derivative="exact").loss_and_grad(th, ps, bs)
    assert abs(got["tc_f64"][0] - L) <= 1e-10 * abs(L) and rel(got["tc_f64"][2], G) < 1e-9
    _close(got["tc_f64"], got["ffma"])


def test_fokker_planck_integral_loss():
    import integral_loss_cases as LC
    from integral_loss_oracle import IntegralLossProblem
    case = LC.fokker_planck()
    sys_, chains, strategy, add, pe = case
    rep = npde.symbolic_discretize(sys_, LC.discretization(case, np.float64, mode="tc_f64"))
    th = rep.flat_init_params
    total, terms, grad = rep.engine.loss_grad_host(th, None, True)
    n_pde = len(sys_.eqs)
    sets = [np.asarray(rep.point_sets[i], dtype=np.float64) for i in range(n_pde + len(sys_.bcs))]
    prob = IntegralLossProblem(sys_, LC.IC.chain_specs(chains), param_estim=pe, integrand=add.integrand,
                               X=np.asarray(rep.point_sets[-1], dtype=np.float64),
                               w=np.asarray(rep.quad_weights[-1], dtype=np.float64), target=add.target, norm=add.norm,
                               w_add=rep.weights["add"][0])
    L, T, G = prob.loss_and_grad(np.asarray(th, dtype=np.float64), sets[:n_pde], sets[n_pde:])
    assert abs(total - L) <= 1e-10 * abs(L) and rel(grad, G) < 1e-9
    ref = npde.symbolic_discretize(sys_, LC.discretization(case, np.float64, mode="ffma"))
    _close((total, terms, grad), ref.engine.loss_grad_host(th, None, True))


def test_refusals():
    with pytest.raises(E.EngineError, match="PINN_MODE_TC_F64 .* needs dtype PINN_F64"):
        spec = _spec(E.MODE_TC_F64, 16, 2, 3)
        spec.dtype = "float32"
        E.Engine(spec)
    with pytest.raises(E.EngineError, match="unknown mode 4"):
        spec = _spec(E.MODE_TC_F64, 16, 2, 3)
        spec.mode = 4
        E.Engine(spec)
