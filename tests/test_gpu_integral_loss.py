"""Integral constraints on the device (pinn.IntegralLoss, PINN_REDUCE_*_OF_SUM): the FFMA kernel's functional term and the
tail's g'(S) scaling against the float64 restatement (tests/integral_loss_oracle.py) at DESIGN section 3's tolerances
(fp64: loss 1e-10, gradient 1e-9; fp32: loss 1e-5, gradient 5e-4), the loss-only and residual-probe paths,
reproducibility, the launch count, the device loops, two ranks, the ABI's refusals, and the reference's Fokker-Planck
test and tutorial."""
import dataclasses

import numpy as np
import pytest
import torch

import neuralpde_jl_b200 as npde
from neuralpde_jl_b200 import engine as E

import integral_loss_cases as LC
from integral_loss_oracle import IntegralLossProblem
from helpers import rel

pytestmark = pytest.mark.gpu

TOL = {np.float64: (1e-10, 1e-9), np.float32: (1e-5, 5e-4)}


def _setup(name, dtype, case=None, **kw):
    case = case or LC.CASES[name]()
    rep = npde.symbolic_discretize(case[0], LC.discretization(case, dtype, **kw))
    return case, rep


def _oracle(case, rep):
    """the restatement on the engine's own point sets, nodes and weights"""
    sys_, chains, strategy, add, pe = case
    n_pde, n_bc = len(sys_.eqs), len(sys_.bcs)
    sets = [np.asarray(rep.point_sets[i], dtype=np.float64) for i in range(n_pde + n_bc)]
    kw = {}
    if isinstance(strategy, npde.QuadratureTraining):
        kw = dict(qweights=[np.asarray(rep.quad_weights[i], dtype=np.float64) for i in range(n_pde + n_bc)],
                  qscales=[rep.engine.spec.terms[i].scale for i in range(n_pde + n_bc)])
    prob = IntegralLossProblem(sys_, LC.IC.chain_specs(chains), param_estim=pe, integrand=add.integrand,
                               X=np.asarray(rep.point_sets[-1], dtype=np.float64),
                               w=np.asarray(rep.quad_weights[-1], dtype=np.float64), target=add.target, norm=add.norm,
                               w_add=rep.weights["add"][0])
    return prob, sets[:n_pde], sets[n_pde:], kw


def _check(rep, prob, ps, bs, kw, dtype, th=None):
    th = rep.flat_init_params if th is None else th
    total, terms, grad = rep.engine.loss_grad_host(th, None, True)
    L, T, G = prob.loss_and_grad(np.asarray(th, dtype=np.float64), ps, bs, **kw)
    lt, gt = TOL[dtype]
    assert abs(total - L) <= lt * abs(L), (total, L)
    np.testing.assert_allclose(terms, T, rtol=lt, atol=lt * 1e-4 * abs(L))
    assert rel(grad, G) < gt, rel(grad, G)
    return total, terms, grad


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name", ["fokker_planck", "neumann2d", "taps_and_param", "tutorial"])
def test_matches_oracle(name, dtype):
    case, rep = _setup(name, dtype)
    assert rep.term_names[-1] == "additional"
    prob, ps, bs, kw = _oracle(case, rep)
    _check(rep, prob, ps, bs, kw, dtype)


@pytest.mark.parametrize("side", [-1.0, 1.0])
def test_both_sides_of_the_kink(side):
    """|S| with S = Σ w v - target above and below 0: the constraint's gradient changes sign with S"""
    case0, rep0 = _setup("fokker_planck", np.float64)
    prob0, _, _, _ = _oracle(case0, rep0)
    s0 = float(torch.sum(prob0.w * prob0.values(torch.as_tensor(rep0.flat_init_params))))
    case = LC.fokker_planck(target=s0 + side * 0.05)
    case, rep = _setup(None, np.float64, case=case)
    prob, ps, bs, kw = _oracle(case, rep)
    th = torch.as_tensor(rep.flat_init_params)
    assert np.sign(float(torch.sum(prob.w * prob.values(th))) - case[3].target) == -side
    _, terms, _ = _check(rep, prob, ps, bs, kw, np.float64)
    assert terms[-1] == pytest.approx(0.05, rel=1e-8)


def test_loss_only_and_residual_probe():
    case, rep = _setup("taps_and_param", np.float64)
    th = rep.flat_init_params
    total, terms, _ = rep.engine.loss_grad_host(th, None, True)
    total2, terms2, g2 = rep.engine.loss_grad_host(th, None, False)
    assert g2 is None and abs(total2 - total) <= 1e-13 * abs(total)
    np.testing.assert_allclose(terms2, terms, rtol=1e-13)
    prob, _, _, _ = _oracle(case, rep)
    n = rep.point_sets[-1].shape[1]
    v = rep.engine.term_residual_host(rep.engine.n_terms - 1, th, n)
    vo = prob.values(torch.as_tensor(th)).numpy() - case[3].target / prob.w.sum().item()
    np.testing.assert_allclose(v, vo, rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_two_runs_bit_identical(dtype):
    for name in ("fokker_planck", "neumann2d"):
        _, rep = _setup(name, dtype)
        th = rep.flat_init_params
        a = rep.engine.loss_grad_host(th, None, True)
        b = rep.engine.loss_grad_host(th, None, True)
        assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


def test_one_launch_per_evaluation():
    _, rep = _setup("neumann2d", np.float64)
    eng = rep.engine
    n0 = eng.launch_count()
    eng.loss_grad_host(rep.flat_init_params, None, True)
    assert eng.launch_count() - n0 == 1
    eng.adam_begin(rep.flat_init_params, 1e-3)
    n0 = eng.launch_count()
    eng.adam_iterate(4)
    assert eng.launch_count() - n0 == 4


def test_device_adam_takes_the_host_loops_steps():
    _, rep = _setup("fokker_planck", np.float64)
    eng = rep.engine
    th = rep.flat_init_params.copy()
    lr, b1, b2, eps = 1e-3, 0.9, 0.999, 1e-8
    m, v = np.zeros_like(th), np.zeros_like(th)
    for t in range(1, 6):
        _, _, g = eng.loss_grad_host(th, None, True)
        m = b1 * m + (1 - b1) * g
        v = b2 * v + (1 - b2) * g * g
        c2 = np.sqrt(1 - b2 ** t)
        th = th - lr * c2 / (1 - b1 ** t) * m / (np.sqrt(v) + eps * c2)
    eng.adam_begin(rep.flat_init_params, lr, b1, b2, eps)
    eng.adam_iterate(5)
    assert rel(eng.adam_theta(), th) < 1e-9


@pytest.mark.parametrize("opt", ["LBFGS", "BFGS"])
def test_quasi_newton_lowers_the_loss(opt):
    case = LC.fokker_planck()
    prob = npde.discretize(case[0], LC.discretization(case, np.float64))
    l0 = prob.f.f(prob.u0, None)
    res = npde.solve(prob, getattr(npde, opt)(), maxiters=30)
    assert np.isfinite(res.objective) and res.objective < l0


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_ranks_reproduce_one_rank(tmp_path):
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = str(tmp_path / "r0.npz")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29571", os.path.join(root, "tests", "integral_loss_mgpu_worker.py"), out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    res = np.load(out)
    _, rep = _setup("neumann2d", np.float64)
    tot, terms, g = rep.engine.loss_grad_host(rep.flat_init_params, None, True)
    assert abs(float(res["tot"]) - tot) <= 1e-11 * abs(tot)
    np.testing.assert_allclose(res["terms"], terms, rtol=1e-11)
    assert rel(res["g"], g) < 1e-11


# ---- refusals of the ABI ---------------------------------------------------------------------------------------------------
def _term(reduction=E.REDUCE_MEAN, prog=None):
    return E.TermSpec(dim=1, taps=[E.TapSpec(net=0)], prog=prog or [("tap", 0, 0, 0.0)], net_rows=[[0]],
                      reduction=reduction, scale=1.0)


def _spec(mode=E.MODE_FFMA, terms=None, **kw):
    net = E.NetSpec([1, 8, 1], ["tanh", "identity"])
    terms = terms or [_term(), _term(E.REDUCE_ABS_OF_SUM)]
    return E.ProblemSpec(nets=[net], terms=terms, n_theta=net.n_params, dtype="float32", mode=mode, **kw)


@pytest.mark.parametrize("spec,msg", [
    (lambda: _spec(mode=E.MODE_TC_BF16), "functional terms run on the FFMA path"),
    (lambda: _spec(mode=E.MODE_TC_SPLIT), "functional terms run on the FFMA path"),
    (lambda: _spec(terms=[_term(E.REDUCE_SQUARE_OF_SUM), _term(E.REDUCE_ABS_OF_SUM)]), "second functional term"),
    (lambda: _spec(terms=[_term(), _term(E.REDUCE_ABS_OF_SUM, [("tap", 0, 0, 0.0), ("integral", 0, 0, 0.0),
                                                               ("add", 0, 1, 0.0)])],
                   integrals=[E.IntegralSpec(owner=1, n_dims=1, q=4, ub=[1.0, 0.0], taps=[E.TapSpec(net=0)],
                                             prog=[("tap", 0, 0, 0.0)], net_rows=[[0]])]),
     "functional term and owns integral terms"),
    (lambda: _spec(terms=[_term(reduction=7)]), "unknown reduction 7"),
])
def test_create_refusals(spec, msg):
    with pytest.raises(E.EngineError, match=msg):
        E.Engine(spec())


def _engine_with_points():
    eng = E.Engine(_spec())
    x = np.linspace(0, 1, 40).reshape(1, -1)
    eng.set_points_host(0, x)
    eng.set_points_host(1, x)
    return eng


def test_call_refusals():
    eng = _engine_with_points()
    th = np.random.default_rng(0).standard_normal(eng.n_theta).astype(np.float32)
    with pytest.raises(E.EngineError, match="functional term; its nodes are fixed"):
        eng.set_sampler(1, 64, [0.0], [1.0])
    with pytest.raises(E.EngineError, match="functional term"):
        eng.term_grad_stats_host(1, th)
    with pytest.raises(E.EngineError, match="global count is the local count 40"):
        eng.set_global_count(1, 80)
    eng.set_global_count(1, 40)
    with pytest.raises(E.EngineError, match="pinn_hmc_begin: term 1 is a functional term"):
        eng.hmc_begin(th.astype(np.float64))
    # the other term keeps its behaviour
    eng.term_grad_stats_host(0, th)
    eng.set_global_count(0, 80)


def test_nullable_weights_mean_one():
    eng = _engine_with_points()
    th = np.random.default_rng(1).standard_normal(eng.n_theta).astype(np.float32)
    a = eng.loss_grad_host(th, None, True)
    eng.set_points_host(1, np.linspace(0, 1, 40).reshape(1, -1), np.ones(40, dtype=np.float32))
    b = eng.loss_grad_host(th, None, True)
    assert a[0] == b[0] and np.array_equal(a[2], b[2])
    v = eng.term_residual_host(1, th, 40).astype(np.float64)
    assert a[1][1] == pytest.approx(abs(v.sum()), rel=1e-5)


# ---- the reference's test and tutorial --------------------------------------------------------------------------------------
def _fp_error(rep, theta, C):
    xs = np.arange(LC.X0, LC.X1 + 1e-9, LC.DX)
    u = np.asarray(rep.phi(xs.reshape(1, -1), theta), dtype=np.float64).ravel()
    ur = LC.analytic(xs, C)
    return float(np.linalg.norm(u - ur) / np.linalg.norm(ur))


@pytest.mark.parametrize("with_init", [True, False])
def test_reference_fokker_planck(with_init):
    """additional_loss__fokker_planck.jl:71-81 / :104-109: L-BFGS for 400 iterations, then BFGS for 2000, fp64;
    ‖u_predict - u_real‖ ≤ 1e-3 ‖u_real‖ with C = 142.88418699042"""
    case = LC.fokker_planck()
    sys_, chains, strategy, add, _ = case
    if with_init:
        disc = LC.discretization(case, np.float64)
    else:
        disc = npde.PhysicsInformedNN(chains[0], strategy, additional_loss=add)
    prob = npde.discretize(sys_, disc)
    res = npde.solve(prob, npde.LBFGS(), maxiters=400)
    res = npde.solve(dataclasses.replace(prob, u0=res.u), npde.BFGS(), maxiters=2000)
    err = _fp_error(prob.representation, res.u, LC.C_TEST)
    print("fokker_planck(init_params=%s): loss %.6g after %d BFGS iterations, rel. error %.3e"
          % (with_init, res.objective, res.iterations, err))
    assert err <= 1e-3


def test_reference_tutorial():
    """docs/src/tutorials/constraints.md: QuadratureTraining(), BFGS(linesearch = BackTracking()), 600 iterations; the
    constraint 0.01 Σ p Δx = 1 holds to 1e-3 (the error against C = 32.47 is printed)"""
    case = LC.fokker_planck_tutorial()
    prob = npde.discretize(case[0], LC.discretization(case, np.float64))
    res = npde.solve(prob, npde.BFGS(linesearch=npde.BackTracking()), maxiters=600)
    rep = prob.representation
    _, terms, _ = rep.engine.loss_grad_host(res.u, None, False)
    err = _fp_error(rep, res.u, LC.C_TUTORIAL)
    print("tutorial: loss %.6g, constraint %.3e, rel. error against C = %.2f: %.3e"
          % (res.objective, terms[-1], LC.C_TUTORIAL, err))
    assert terms[-1] <= 1e-3
