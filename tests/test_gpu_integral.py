"""Integral terms on the device: the FFMA kernel's node tiles against the float64 restatement (tests/integral_oracle.py)
with the same Gauss-Legendre rule, at DESIGN section 3's tolerances (fp64: loss 1e-10, gradient 1e-9; fp32: loss
1e-5, gradient 5e-4), the loss-only and residual-probe paths, reproducibility, a device-sampled owner term, the
ABI's refusals, and the reference's seven IntegroDiff tests under the device BFGS."""
import numpy as np
import pytest
import torch

import neuralpde_jl_b200 as npde
from neuralpde_jl_b200 import engine as E
from neuralpde_jl_b200.pinn import initialparameters
from oracle import reference as R

import integral_cases as IC
from integral_oracle import IntegralProblem
from helpers import rel

pytestmark = pytest.mark.gpu

# every shape the kernel dispatches: 1-D with a variable bound (ide1, ide2), the unit square (ide3), [0,1] x [0,x]
# (ide4), two networks in one integrand (ide5), [a, Inf) next to a finite integral (ide6), [x, Inf) (ide7); across the
# three activations
SHAPES = [("ide1", "sigmoid"), ("ide1", "sin"), ("ide2", "tanh"), ("ide3", "sigmoid"), ("ide4", "tanh"),
          ("ide4", "sin"), ("ide5", "sigmoid"), ("ide6", "sigmoid"), ("ide6", "tanh"), ("ide7", "tanh"),
          ("ide7", "sin")]


def _engine(name, act, dtype, **kw):
    sys_, chains, dx = IC.REFERENCE[name](act)
    rep = npde.symbolic_discretize(sys_, IC.discretization(chains, dx, dtype, **kw))
    return sys_, chains, dx, rep


def _oracle(sys_, chains, dx, theta64, sets=None):
    prob = IntegralProblem(sys_, IC.chain_specs(chains))
    if sets is None:
        ps, bs = R.generate_training_sets(sys_.domain, dx, sys_.eqs, sys_.bcs, sys_.ivs, sys_.dvs)
    else:
        ps, bs = sets[:len(sys_.eqs)], sets[len(sys_.eqs):]
    return prob, prob.loss_and_grad(theta64, ps, bs)


@pytest.mark.parametrize("name,act", SHAPES)
def test_fp64_matches_oracle(name, act):
    sys_, chains, dx, rep = _engine(name, act, np.float64)
    th = rep.flat_init_params
    total, terms, grad = rep.engine.loss_grad_host(th, None, True)
    _, (L, T, G) = _oracle(sys_, chains, dx, th)
    assert abs(total - L) <= 1e-10 * abs(L), (total, L)
    np.testing.assert_allclose(terms, T, rtol=1e-10, atol=1e-14)
    assert rel(grad, G) < 1e-9


@pytest.mark.parametrize("name,act", SHAPES)
def test_fp32_matches_oracle(name, act):
    sys_, chains, dx, rep = _engine(name, act, np.float32)
    th = rep.flat_init_params
    total, terms, grad = rep.engine.loss_grad_host(th, None, True)
    _, (L, T, G) = _oracle(sys_, chains, dx, th.astype(np.float64))
    assert abs(total - L) <= 1e-5 * abs(L), (total, L)
    np.testing.assert_allclose(terms, T, rtol=1e-5, atol=1e-9)
    assert rel(grad, G) < 5e-4


@pytest.mark.parametrize("name", ["ide1", "ide4", "ide6", "ide7"])
def test_loss_only_and_residual_probe(name):
    sys_, chains, dx, rep = _engine(name, IC.REFERENCE[name].__defaults__[0], np.float64)
    th = rep.flat_init_params
    total, terms, grad = rep.engine.loss_grad_host(th, None, True)
    total2, terms2, g2 = rep.engine.loss_grad_host(th, None, False)
    assert g2 is None and abs(total2 - total) <= 1e-13 * abs(total)
    np.testing.assert_allclose(terms2, terms, rtol=1e-13)
    prob = IntegralProblem(sys_, IC.chain_specs(chains))
    ps, _ = R.generate_training_sets(sys_.domain, dx, sys_.eqs, sys_.bcs, sys_.ivs, sys_.dvs)
    r = rep.loss_functions.datafree_pde_loss_functions[0](ps[0], th)
    ro = prob.residual(sys_.eqs[0], torch.as_tensor(ps[0]), torch.as_tensor(th)).numpy().ravel()
    np.testing.assert_allclose(np.ravel(r), ro, rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_two_runs_bit_identical(dtype):
    for name in ("ide4", "ide6"):
        _, _, _, rep = _engine(name, "sigmoid", dtype)
        th = rep.flat_init_params
        a = rep.engine.loss_grad_host(th, None, True)
        b = rep.engine.loss_grad_host(th, None, True)
        assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


def test_device_sampled_owner_term_matches_oracle_on_drawn_points():
    """StochasticTraining with the device sampler: the owner's points are drawn on the GPU; the oracle evaluates the
    same loss at the points the engine drew (ide1: the integral's bound is the owner's own coordinate row)."""
    sys_, chains, _ = IC.ide1()
    disc = npde.PhysicsInformedNN(chains[0], npde.StochasticTraining(200, bcs_points=1, seed=5, device_sampler=True),
                                  init_params=IC.init_params(chains))
    rep = npde.symbolic_discretize(sys_, disc)
    eng = rep.engine
    th = rep.flat_init_params
    total, terms, grad = eng.loss_grad_host(th, None, True)
    sets = [eng.get_points_host(0, 200), eng.get_points_host(1, 1)]
    _, (L, T, G) = _oracle(sys_, chains, 0.1, th, sets=sets)
    assert abs(total - L) <= 1e-10 * abs(L)
    assert rel(grad, G) < 1e-9


def test_flops_count_the_node_evaluations():
    _, chains, _, rep = _engine("ide1", "sigmoid", np.float64)
    S = sum(a * b for a, b in zip(chains[0].dims[:-1], chains[0].dims[1:]))
    n_pde = 21
    # owner: value + first derivative channel (C = 2), integrand C = 1 at 16 nodes, forward and reverse; bc: C = 1
    assert rep.engine.flops_per_eval() == pytest.approx(n_pde * 6 * S * (2 + 2 * 16) + 1 * 6 * S)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_ranks_reproduce_one_rank(tmp_path):
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = str(tmp_path / "r0.npz")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29563", os.path.join(root, "tests", "ide_mgpu_worker.py"), out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    res = np.load(out)
    _, _, _, rep = _engine("ide4", "sigmoid", np.float64)
    tot, terms, g = rep.engine.loss_grad_host(rep.flat_init_params, None, True)
    assert abs(float(res["tot"]) - tot) <= 1e-11 * abs(tot)
    np.testing.assert_allclose(res["terms"], terms, rtol=1e-10)
    assert rel(res["g"], g) < 1e-10


# ---- refusals of pinn_create_ex ------------------------------------------------------------------------------------------
def _spec(mode=E.MODE_FFMA, **integral):
    net = E.NetSpec([1, 8, 1], ["tanh", "identity"])
    term = E.TermSpec(dim=1, taps=[E.TapSpec(net=0)], prog=[("tap", 0, 0, 0.0), ("integral", 0, 0, 0.0),
                                                            ("sub", 0, 1, 0.0)], net_rows=[[0]])
    it = E.IntegralSpec(owner=0, n_dims=1, q=8, ub=[1.0, 0.0], taps=[E.TapSpec(net=0)], prog=[("tap", 0, 0, 0.0)],
                        net_rows=[[0]])
    for k, v in integral.items():
        setattr(it, k, v)
    return E.ProblemSpec(nets=[net], terms=[term], n_theta=net.n_params, dtype="float32", mode=mode, integrals=[it])


@pytest.mark.parametrize("kw,msg", [
    (dict(mode=E.MODE_TC_BF16), "integral terms run on the FFMA path"),
    (dict(n_dims=3), "3 integrating dimensions"),
    (dict(q=0), "q=0 Gauss-Legendre nodes"),
    (dict(q=65), "q=65 Gauss-Legendre nodes"),
    (dict(ub_row=[3, -1]), "bound row out of range"),
    (dict(prog=[("tap", 2, 0, 0.0)]), "integral 0 instr 0 TAP 2 out of range"),
    (dict(net_rows=[[5]]), "integral 0 network 0 input 0 maps to point row 5"),
])
def test_create_ex_refusals(kw, msg):
    mode = kw.pop("mode", E.MODE_FFMA)
    with pytest.raises(E.EngineError, match=msg):
        E.Engine(_spec(mode=mode, **kw))


def test_integral_opcode_refused_by_pinn_create():
    spec = _spec()
    spec.integrals = []
    with pytest.raises(E.EngineError, match="integral terms are created with pinn_create_ex"):
        E.Engine(spec)


def test_create_ex_valid_spec_builds():
    E.Engine(_spec())


# ---- the reference's IntegroDiff tests, solved with BFGS on the device ---------------------------------------------------
def _predict(rep, k, pts, theta):
    return np.asarray(rep.phi[k](pts, theta) if isinstance(rep.phi, list) else rep.phi(pts, theta)).ravel()


def _solve(name):
    sys_, chains, dx = IC.REFERENCE[name]()
    rng = np.random.default_rng(110)                 # Lux's default init (glorot_uniform, zero bias), as the tests use
    init = np.concatenate([initialparameters(rng, c) for c in chains])
    disc = npde.PhysicsInformedNN(chains if len(chains) > 1 else chains[0], npde.GridTraining(dx), init_params=init)
    prob = npde.discretize(sys_, disc)
    maxiters = {"ide5": 200, "ide6": 200, "ide7": 300}.get(name, 100)
    res = npde.solve(prob, npde.BFGS(), maxiters=maxiters)
    return prob.representation, res


def _grid1(lo, hi):
    return np.arange(lo, hi + 1e-9, 0.01)


def test_reference_ide1():
    rep, res = _solve("ide1")
    ts = _grid1(0.0, 2.0)
    u = _predict(rep, 0, ts.reshape(1, -1), res.u)
    assert np.mean((0.5 * np.exp(-ts) * np.sin(2 * ts) - u) ** 2) < 0.02


def test_reference_ide2():
    rep, res = _solve("ide2")
    xs = _grid1(0.0, 1.0)
    u = _predict(rep, 0, xs.reshape(1, -1), res.u)
    assert np.mean((xs ** 2 / np.cos(xs) - u) ** 2) < 0.02


def _grid2():
    xs = np.arange(0.0, 1.0 + 1e-9, 0.01)
    X, Y = np.meshgrid(xs, xs)                       # (y, x) order, as the reference's comprehension
    return X.ravel(), Y.ravel()


def test_reference_ide3():
    rep, res = _solve("ide3")
    X, Y = _grid2()
    u = _predict(rep, 0, np.stack([X, Y]), res.u)
    assert np.mean((1 - X ** 2 - Y ** 2 - u) ** 2) < 0.001


def test_reference_ide4():
    rep, res = _solve("ide4")
    X, Y = _grid2()
    u = _predict(rep, 0, np.stack([X, Y]), res.u)
    assert np.mean((X + Y ** 2 - u) ** 2) < 0.02


def test_reference_ide5():
    rep, res = _solve("ide5")
    xs = _grid1(1.0, 2.0)
    u = _predict(rep, 0, xs.reshape(1, -1), res.u)
    w = _predict(rep, 1, xs.reshape(1, -1), res.u)
    assert np.mean((xs - u) ** 2) < 0.001
    assert np.mean((1 / xs ** 2 - w) ** 2) < 0.001


def _isapprox(a, b, rtol):
    return np.linalg.norm(a - b) <= rtol * max(np.linalg.norm(a), np.linalg.norm(b))


def test_reference_ide6():
    rep, res = _solve("ide6")
    xs = _grid1(1.0, 2.0)
    assert _isapprox(1 / xs ** 2, _predict(rep, 0, xs.reshape(1, -1), res.u), 0.1)


def test_reference_ide7():
    rep, res = _solve("ide7")
    xs = _grid1(1.0, 2.0)
    assert _isapprox(1 / xs ** 2, _predict(rep, 0, xs.reshape(1, -1), res.u), 0.02)
