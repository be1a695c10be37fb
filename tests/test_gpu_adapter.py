"""Fixed networks on the device: neural adapters and registered network functions in the FFMA kernel against the
float64 restatement (tests/adapter_oracle.py) at DESIGN section 3's tolerances (fp64: loss 1e-10, gradient 1e-9; fp32:
loss 1e-5, gradient 5e-4); device-sampled sets, the loss-only and residual paths, reproducibility, launches, re-pointed
parameters, the ABI's refusals and a two-rank sum."""
import os
import subprocess
import sys

import numpy as np
import pytest
import sympy as sp
import torch

import neuralpde_jl_b200 as npde
from neuralpde_jl_b200 import engine as E
from neuralpde_jl_b200.strategies import adapter_training_set
from oracle import reference as R

from adapter_oracle import FixedProblem, adapter_loss_and_grad
from helpers import rel
from integral_oracle import IntegralProblem

pytestmark = pytest.mark.gpu
TOL = {np.float64: (1e-10, 1e-9), np.float32: (1e-5, 5e-4)}

x, y = npde.parameters("x y")
u = npde.variables("u")
Dx, Dy = npde.Differential(x), npde.Differential(y)


def _chain(dims, acts):
    return npde.Chain(*[npde.Dense(a, b, act) for a, b, act in zip(dims[:-1], dims[1:], acts)])


def _teacher(dims=(2, 8, 8, 1), acts=("tanh", "tanh", "identity"), seed=0, name="phi"):
    chain = _chain(dims, acts)
    rng = np.random.default_rng(seed)
    theta = npde.initialparameters(rng, chain) + 0.05 * rng.standard_normal(chain.n_params)
    return chain, theta, npde.register_symbolic(npde.Phi(chain, 0, chain.n_params, np.float64), theta, name)


STUDENT = _chain((2, 8, 8, 1), ("tanh", "tanh", "identity"))


def _theta0(chain, dtype, seed=7):
    rng = np.random.default_rng(seed)
    return (npde.initialparameters(rng, chain) + 0.05 * rng.standard_normal(chain.n_params)).astype(dtype)


def _box(x0=0.0, x1=1.0):
    return [npde.In(x, x0, x1), npde.In(y, 0.0, 1.0)]


def _system(doms):
    return npde.PDESystem([npde.Eq((Dx**2)(u(x, y)) + (Dy**2)(u(x, y)), -sp.sin(sp.pi * x) * sp.sin(sp.pi * y))],
                          [npde.Eq(u(0, y), 0)], doms, [x, y], [u(x, y)])


def _check(dtype, got, want):
    (total, terms, grad), (L, T, G) = got, want
    lt, gt = TOL[dtype]
    assert abs(total - L) <= lt * abs(L), (total, L)
    np.testing.assert_allclose(terms, T, rtol=lt * 10, atol=1e-14)
    assert rel(grad, G) < gt, rel(grad, G)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_one_teacher_matches_oracle(dtype):
    _, _, pt = _teacher()
    sys_ = _system(_box())
    th = _theta0(STUDENT, dtype)
    prob = npde.neural_adapter(npde.NeuralAdapterLoss(STUDENT, pt(x, y)), th, sys_, npde.GridTraining(0.05))
    eng = prob.representation.engine
    got = eng.loss_grad_host(th, None, True)
    assert got[2].shape == (STUDENT.n_params,)                  # the gradient covers the student's θ only
    pts = adapter_training_set(sys_.domain, 0.05, np.float64)
    want = adapter_loss_and_grad(STUDENT, th.astype(np.float64), [(["x", "y"], pt(x, y), pts, None, 1.0)])
    _check(dtype, got, want)
    # loss-only path, residual probe, one launch per evaluation, bit-reproducible
    n0 = eng.launch_count()
    t2, terms2, g2 = eng.loss_grad_host(th, None, True)
    assert eng.launch_count() - n0 == 1
    assert t2 == got[0] and np.array_equal(g2, got[2]) and np.array_equal(terms2, got[1])
    t3, _, _ = eng.loss_grad_host(th, None, False)
    assert abs(t3 - got[0]) <= TOL[dtype][0] * abs(got[0])
    r = eng.term_residual_host(0, th, pts.shape[1])
    rw = R.phi(torch.tensor(pts), torch.tensor(th.astype(np.float64)), STUDENT.dims, STUDENT.acts).numpy()[0] - \
        R.phi(torch.tensor(pts), torch.tensor(pt.fixed_net.params), pt.fixed_net.dims, pt.fixed_net.acts).numpy()[0]
    np.testing.assert_allclose(r, rw, rtol=0, atol=1e-12 if dtype == np.float64 else 1e-5)
    assert eng.flops_per_eval() == pytest.approx(pts.shape[1] * (6 + 2) * (2 * 8 + 8 * 8 + 8))


def test_ten_teachers_list_form():
    systems, losses, terms = [], [], []
    for i in range(10):
        _, _, pt = _teacher(seed=10 + i, name="phi_%d" % i)
        sys_ = _system(_box(i / 10, (i + 1) / 10))
        systems.append(sys_)
        losses.append(npde.NeuralAdapterLoss(STUDENT, pt(x, y)))
        terms.append((["x", "y"], pt(x, y), adapter_training_set(sys_.domain, [0.01, 0.1], np.float64), None, 1.0))
    th = _theta0(STUDENT, np.float64)
    prob = npde.neural_adapter(losses, th, systems, npde.GridTraining([0.01, 0.1]))
    assert len(prob.representation.fixed) == 10
    got = prob.representation.engine.loss_grad_host(th, None, True)
    _check(np.float64, got, adapter_loss_and_grad(STUDENT, th, terms))
    total, g = prob.f.grad(th)
    assert total == got[0] and np.array_equal(g, got[2])


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_bc_and_pde_on_a_fixed_network(dtype):
    # a teacher of another width, depth and activation than the student; a bc on its value at a constant x_0 and a pde
    # term on its first and second derivatives
    _, _, pb = _teacher(dims=(2, 6, 5, 1), acts=("sigmoid", "sin", "identity"), seed=3, name="phi_bound")
    eq = npde.Eq((Dx**2)(u(x, y)) + (Dy**2)(u(x, y)), Dx(pb(x, y)) + (Dy**2)(pb(x, y)) + Dx(Dy(pb(x, y))))
    bcs = [npde.Eq(u(0.2, y), pb(0.2, y)), npde.Eq(u(x, 0), 0.0), npde.Eq(u(x, 1), pb(x, 1.0) * x)]
    sys_ = npde.PDESystem([eq], bcs, _box(0.2, 1.0), [x, y], [u(x, y)])
    th = _theta0(STUDENT, dtype)
    rep = npde.symbolic_discretize(sys_, npde.PhysicsInformedNN(STUDENT, npde.GridTraining(0.1), init_params=th))
    got = rep.engine.loss_grad_host(th, None, True)
    ps, bs = R.generate_training_sets(sys_.domain, 0.1, sys_.eqs, sys_.bcs, sys_.ivs, sys_.dvs)
    prob = FixedProblem(sys_, [(STUDENT.dims, STUDENT.acts)], derivative="exact")
    _check(dtype, got, prob.loss_and_grad(th.astype(np.float64), ps, bs))


class _FixedIntegralProblem(FixedProblem, IntegralProblem):
    pass


def test_fixed_tap_inside_an_integrand():
    t = npde.parameters("t")
    i = npde.variables("i")
    teacher = _chain((1, 6, 1), ("tanh", "identity"))
    rng = np.random.default_rng(5)
    tt = npde.initialparameters(rng, teacher) + 0.05 * rng.standard_normal(teacher.n_params)
    pt = npde.register_symbolic(npde.Phi(teacher, 0, teacher.n_params, np.float64), tt, "w")
    Ii = npde.Integral(t, npde.ClosedInterval(0, t))
    eq = npde.Eq(npde.Differential(t)(i(t)) + 5 * Ii(i(t) * pt(t) + npde.Differential(t)(pt(t))), pt(t))
    sys_ = npde.PDESystem([eq], [npde.Eq(i(0.0), 0.0)], [npde.In(t, 0.0, 2.0)], [t], [i(t)])
    chain = _chain((1, 12, 1), ("sigmoid", "identity"))
    th = _theta0(chain, np.float64)
    rep = npde.symbolic_discretize(sys_, npde.PhysicsInformedNN(chain, npde.GridTraining(0.1), init_params=th))
    got = rep.engine.loss_grad_host(th, None, True)
    ps, bs = R.generate_training_sets(sys_.domain, 0.1, sys_.eqs, sys_.bcs, sys_.ivs, sys_.dvs)
    prob = _FixedIntegralProblem(sys_, [(chain.dims, chain.acts)])
    _check(np.float64, got, prob.loss_and_grad(th, ps, bs))


@pytest.mark.parametrize("strategy", [npde.StochasticTraining(300, seed=11),
                                      npde.QuasiRandomTraining(300, resampling=True, seed=12)])
def test_device_sampled_sets(strategy):
    _, _, pt = _teacher(seed=2)
    sys_ = _system(_box())
    th = _theta0(STUDENT, np.float64)
    prob = npde.neural_adapter(npde.NeuralAdapterLoss(STUDENT, pt(x, y)), th, sys_, strategy)
    eng = prob.representation.engine
    for _ in range(2):                                          # the second evaluation draws a fresh sample first
        n0 = eng.launch_count()
        total, g = prob.f.grad(th)
        pts = eng.get_points_host(0, 300)
        assert pts.min() >= 0.0 and pts.max() <= 1.0
        want = adapter_loss_and_grad(STUDENT, th, [(["x", "y"], pt(x, y), pts, None, 1.0)])
        assert abs(total - want[0]) <= 1e-10 * want[0] and rel(g, want[2]) < 1e-9
    assert eng.launch_count() - n0 == 2                         # one sampler launch + one fused launch


def test_quadrature_box():
    _, _, pt = _teacher(seed=6)
    sys_ = _system(_box())
    th = _theta0(STUDENT, np.float64)
    prob = npde.neural_adapter(npde.NeuralAdapterLoss(STUDENT, pt(x, y)), th, sys_, npde.QuadratureTraining(12))
    got = prob.representation.engine.loss_grad_host(th, None, True)
    pts, w, area = npde.strategies.gauss_legendre_box((np.zeros(2), np.ones(2)), 12, np.float64)
    _check(np.float64, got, adapter_loss_and_grad(STUDENT, th, [(["x", "y"], pt(x, y), pts, w, 1.0 / area)]))


def _engine_spec(n_fixed=1, mode=E.MODE_FFMA, tap_net=1, dims=(2, 8, 1)):
    net = E.NetSpec([2, 8, 1], ["tanh", "identity"], 0)
    fixed = [E.FixedNetSpec(list(dims), ["tanh", "identity"]) for _ in range(n_fixed)]
    term = E.TermSpec(dim=2, taps=[E.TapSpec(net=0), E.TapSpec(net=tap_net)],
                      prog=[("tap", 0, 0, 0.0), ("tap", 1, 0, 0.0), ("sub", 0, 1, 0.0)])
    return E.ProblemSpec(nets=[net], terms=[term], n_theta=net.n_params, dtype="float32" if mode else "float64",
                         mode=mode, fixed=fixed)


def test_repointed_parameters():
    spec = _engine_spec()
    eng = E.Engine(spec)
    pts = np.random.default_rng(0).uniform(0, 1, size=(2, 100))
    eng.set_points_host(0, pts)
    student = teacher = _chain((2, 8, 1), ("tanh", "identity"))
    th = _theta0(student, np.float64)
    a, b = _theta0(teacher, np.float64, 1), _theta0(teacher, np.float64, 2)

    def want(p):
        f = npde.symbolic.FixedNet([2, 8, 1], ["tanh", "identity"], p)
        return adapter_loss_and_grad(student, th, [(["x", "y"], npde.symbolic.fixed_function("f", f)(x, y), pts, None,
                                                    1.0)])
    eng.set_fixed_params_host(0, a)
    ta = eng.loss_grad_host(th, None, True)
    _check(np.float64, ta, want(a))
    eng.set_fixed_params_host(0, b)                              # copy into the same engine buffer
    _check(np.float64, eng.loss_grad_host(th, None, True), want(b))
    dev = torch.tensor(a, device="cuda")
    eng.set_fixed_params(0, dev)                                 # alias a device buffer
    assert eng.loss_grad_host(th, None, True)[0] == ta[0]
    dev2 = torch.tensor(b, device="cuda")
    eng.set_fixed_params(0, dev2)
    _check(np.float64, eng.loss_grad_host(th, None, True), want(b))
    # the device Adam loop sees re-pointed parameters too
    eng.adam_begin(th, 1e-3)
    l1, _ = eng.adam_iterate(3)
    eng.set_fixed_params(0, dev)
    eng.adam_begin(th, 1e-3)
    l2, _ = eng.adam_iterate(3)
    assert l1 != l2


def test_repointing_between_replays_of_a_captured_adam_graph():
    # the captured graph reads the fixed network's parameters through the device copy of the problem: re-pointing
    # between two pinn_adam_iterate calls of the same length (one graph, replayed) takes effect without a re-capture
    student = teacher = _chain((2, 8, 1), ("tanh", "identity"))
    pts = np.random.default_rng(0).uniform(0, 1, size=(2, 100))
    th = _theta0(student, np.float64)
    a, b = _theta0(teacher, np.float64, 1), _theta0(teacher, np.float64, 2)
    eng = E.Engine(_engine_spec())
    eng.set_points_host(0, pts)
    dev_a, dev_b = torch.tensor(a, device="cuda"), torch.tensor(b, device="cuda")
    eng.set_fixed_params(0, dev_a)
    eng.adam_begin(th, 1e-2)
    eng.adam_iterate(1)
    eng.adam_iterate(1)                      # replays the graph captured by the first call
    th2 = eng.adam_theta()
    eng.set_fixed_params(0, dev_b)
    loss_b, _ = eng.adam_iterate(1)          # the loss at th2, before this step, with the teacher's parameters b
    ref = E.Engine(_engine_spec())
    ref.set_points_host(0, pts)
    ref.set_fixed_params_host(0, b)
    assert loss_b == pytest.approx(ref.loss_grad_host(th2, None, False)[0], rel=1e-12)
    ref.set_fixed_params_host(0, a)
    assert abs(loss_b - ref.loss_grad_host(th2, None, False)[0]) > 1e-6 * loss_b


def test_abi_refusals():
    with pytest.raises(E.EngineError, match="fixed networks run on the FFMA path"):
        E.Engine(_engine_spec(mode=E.MODE_TC_BF16))
    with pytest.raises(E.EngineError, match="n_fixed=17 out of range"):
        E.Engine(_engine_spec(n_fixed=17))
    with pytest.raises(E.EngineError, match="names network 3"):
        E.Engine(_engine_spec(n_fixed=2, tap_net=3))
    many = _engine_spec(n_fixed=9)                                # the student and 9 fixed networks in one term
    many.terms[0] = E.TermSpec(dim=2, taps=[E.TapSpec(net=k) for k in range(10)],
                               prog=[("tap", k, 0, 0.0) for k in range(10)] + [("add", 0, 1, 0.0)])
    with pytest.raises(E.EngineError, match="taps more than 8 networks"):
        E.Engine(many)
    eng = E.Engine(_engine_spec())
    eng.set_points_host(0, np.zeros((2, 4)))
    with pytest.raises(E.EngineError, match="fixed network 0 has no parameters"):
        eng.loss_grad_host(np.zeros(eng.n_theta), None, True)
    with pytest.raises(E.EngineError, match="fixed network 1 out of range"):
        E._check(eng.lib.pinn_set_fixed_params(eng._h, 1, E.C.c_void_p(16)))
    with pytest.raises(ValueError, match="parameters"):
        eng.set_fixed_params_host(0, np.zeros(3))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks(tmp_path):
    out = str(tmp_path / "r.npz")
    here = os.path.dirname(os.path.abspath(__file__))
    subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nproc_per_node=2",
                    os.path.join(here, "adapter_mgpu_worker.py"), out], check=True, timeout=600)
    r = np.load(out)
    _, _, pt = _teacher(seed=1)
    th = _theta0(STUDENT, np.float64)
    pts = adapter_training_set(_box(), 0.05, np.float64)
    want = adapter_loss_and_grad(STUDENT, th, [(["x", "y"], pt(x, y), pts, None, 1.0)])
    assert abs(float(r["tot"]) - want[0]) <= 1e-10 * want[0] and rel(r["g"], want[2]) < 1e-9
