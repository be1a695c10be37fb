"""Registered network functions and neural adapters on the host: their lowering to fixed-network taps, the adapter's
training sets against a restatement of src/neural_adapter.jl, the float64 oracle of a fixed network, and the refusals.
No GPU needed."""
import numpy as np
import pytest
import sympy as sp
import torch

import neuralpde_jl_b200 as npde
from neuralpde_jl_b200.adapter import _adapter_term
from neuralpde_jl_b200.engine import TapSpec
from neuralpde_jl_b200.lowering import LoweringError, lower_equation
from neuralpde_jl_b200.strategies import adapter_training_set, get_bounds_

from adapter_oracle import FixedProblem, fixed_forward

x, y = npde.parameters("x y")
u = npde.variables("u")
Dx, Dy = npde.Differential(x), npde.Differential(y)


def _teacher(dims=(2, 8, 1), acts=("tanh", "identity"), seed=0, name="phi_bound"):
    chain = npde.Chain(*[npde.Dense(a, b, act) for a, b, act in zip(dims[:-1], dims[1:], acts)])
    theta = npde.initialparameters(np.random.default_rng(seed), chain)
    return chain, theta, npde.register_symbolic(npde.Phi(chain, 0, chain.n_params, np.float64), theta, name)


VI = npde.get_vars([x, y], [u(x, y)])


def test_constant_argument_binds_to_the_bc_row():
    _, _, pb = _teacher()
    fixed = []
    lt = lower_equation(npde.Eq(u(0.3, y), pb(0.3, y)), VI, fixed=fixed)
    assert lt.indvars == ["x", "y"]
    assert lt.taps == [TapSpec(net=0, order=0, dirs=()), TapSpec(net=1, order=0, dirs=())]
    assert lt.prog == [("tap", 0, 0, 0.0), ("tap", 1, 0, 0.0), ("sub", 0, 1, 0.0)]
    assert lt.net_rows == [[0, 1], [0, 1]]             # x_0 sits in row 0 of the bc's points (get_argument)
    assert len(fixed) == 1 and fixed[0] is pb.fixed_net


def test_derivatives_of_a_registered_function():
    _, _, pb = _teacher()
    fixed = []
    lt = lower_equation(npde.Eq((Dx**2)(u(x, y)), Dx(pb(x, y)) + (Dy**2)(pb(x, y)) + Dx(Dy(pb(x, y)))), VI,
                        fixed=fixed)
    fixed_taps = sorted((t.order, tuple(t.dirs)) for t in lt.taps if t.net == 1)
    assert fixed_taps == [(1, (0,)), (2, (0, 1)), (2, (1, 1))]
    assert [t for t in lt.taps if t.net == 0] == [TapSpec(net=0, order=2, dirs=(0, 0))]


def test_swapped_arguments_map_to_their_rows():
    _, _, pb = _teacher()
    lt = lower_equation(npde.Eq(u(x, y), Dx(pb(y, x))), VI, fixed=[])
    assert lt.net_rows[1] == [1, 0]
    assert lt.taps[1] == TapSpec(net=1, order=1, dirs=(1,))        # d/dx is the teacher's second input


def test_two_teachers_get_their_own_networks():
    _, _, p1 = _teacher(name="phi")
    _, _, p2 = _teacher(seed=1, name="phi")                          # same name, distinct functions
    fixed = []
    lower_equation(npde.Eq(u(x, y), p1(x, y)), VI, fixed=fixed)
    lt = lower_equation(npde.Eq(u(x, y), p2(x, y) - p1(x, y)), VI, fixed=fixed)
    assert len(fixed) == 2 and {t.net for t in lt.taps} == {0, 1, 2}


def test_registered_applications_are_never_hoisted():
    _, _, pb = _teacher()
    lt = lower_equation(npde.Eq(u(x, y), pb(x, y) * sp.sin(x) * sp.cos(y) + sp.exp(x * y)), VI, hoist=True, fixed=[])
    assert lt.extra_exprs and not any(e.has(sp.core.function.AppliedUndef) for e in lt.extra_exprs)
    assert any(t.net == 1 for t in lt.taps)


def test_unregistered_function_still_raises():
    g = sp.Function("phi_bound")
    with pytest.raises(LoweringError, match="unknown function phi_bound"):
        lower_equation(npde.Eq(u(x, y), g(x, y)), VI, fixed=[])


def test_constant_without_a_row_is_refused():
    _, _, pb = _teacher()
    with pytest.raises(LoweringError, match="arguments of a registered function"):
        lower_equation(npde.Eq(u(x, y), pb(0.5, y)), VI, fixed=[])


def test_adapter_term_ir():
    chain, _, pb = _teacher()
    student = npde.Chain(npde.Dense(2, 4, "tanh"), npde.Dense(4, 1))
    fixed = []
    tm = _adapter_term(npde.NeuralAdapterLoss(student, pb(x, y)), ["x", "y"], {}, fixed)
    assert tm.taps == [TapSpec(net=0, order=0, dirs=()), TapSpec(net=1, order=0, dirs=())]
    assert tm.prog == [("tap", 0, 0, 0.0), ("tap", 1, 0, 0.0), ("sub", 0, 1, 0.0)]
    assert tm.net_rows == [[0, 1], [0, 1]] and tm.dim == 2
    # rows in another order: the student reads them in order, the teacher by name
    tm = _adapter_term(npde.NeuralAdapterLoss(student, pb(x, y)), ["y", "x"], {}, [])
    assert tm.net_rows == [[0, 1], [1, 0]]


def _julia_range(lo, h, hi):
    n = int(np.floor((hi - lo) / h + 1e-10)) + 1
    return lo + h * np.arange(n)


def test_adapter_grid_set_matches_reference():
    # src/neural_adapter.jl:1-6: reduce(hcat, vec(map(collect, Iterators.product(spans...)))), first variable fastest
    doms = [npde.In(x, 0.0, 1.0), npde.In(y, 0.0, 0.5)]
    got = adapter_training_set(doms, [0.25, 0.1], np.float64)
    xs, ys = _julia_range(0.0, 0.25, 1.0), _julia_range(0.0, 0.1, 0.5)
    want = np.array([[a, b] for b in ys for a in xs]).T
    np.testing.assert_array_equal(got, want)


def test_adapter_bounds_match_reference():
    # src/neural_adapter.jl:8-23: the first equation's arguments, each its domain's [infimum, supremum] (no shrink)
    doms = [npde.In(x, 0.0, 1.0), npde.In(y, -1.0, 2.0)]
    sys_ = npde.PDESystem([npde.Eq(u(x, y), 0), npde.Eq(u(0.5, y), 1)], [npde.Eq(u(0, y), 0)], doms, [x, y], [u(x, y)])
    args, lb, ub = get_bounds_(sys_.domain, sys_.eqs, np.float64, npde.get_vars(sys_.ivs, sys_.dvs))
    assert args == ["x", "y"]
    np.testing.assert_array_equal(lb, [0.0, -1.0])
    np.testing.assert_array_equal(ub, [1.0, 2.0])
    sys2 = npde.PDESystem([npde.Eq(u(0.5, y), 1)], [npde.Eq(u(0, y), 0)], doms, [x, y], [u(x, y)])
    args, lb, ub = get_bounds_(sys2.domain, sys2.eqs, np.float64, npde.get_vars(sys2.ivs, sys2.dvs))
    assert args == [0.5, "y"]
    np.testing.assert_array_equal(lb, [0.5, -1.0])
    np.testing.assert_array_equal(ub, [0.5, 2.0])


def test_oracle_fixed_forward_against_numpy():
    chain, theta, pb = _teacher(dims=(2, 5, 3, 1), acts=("sigmoid", "tanh", "identity"), seed=4)
    X = np.random.default_rng(1).uniform(-1, 1, size=(2, 7))
    h, o = X, 0
    for l in chain.layers:                     # Lux layout: W (out x in, column-major), then b
        W = theta[o:o + l.in_dims * l.out_dims].reshape(l.out_dims, l.in_dims, order="F")
        o += l.in_dims * l.out_dims
        b = theta[o:o + l.out_dims]
        o += l.out_dims
        z = W @ h + b[:, None]
        h = {"sigmoid": lambda v: 1 / (1 + np.exp(-v)), "tanh": np.tanh, "identity": lambda v: v}[l.activation](z)
    got = fixed_forward(pb.fixed_net, torch.tensor(X))
    np.testing.assert_allclose(got.numpy(), h, rtol=1e-13, atol=1e-14)
    # through the Problem oracle: the student's θ gets a gradient, the teacher's parameters none
    sys_ = npde.PDESystem([npde.Eq(u(x, y), pb(x, y))], [npde.Eq(u(0, y), 0)], [npde.In(x, 0, 1), npde.In(y, 0, 1)],
                          [x, y], [u(x, y)])
    student = ((2, 3, 1), ("tanh", "identity"))
    prob = FixedProblem(sys_, [student], derivative="exact")
    th = torch.tensor(np.random.default_rng(2).normal(size=13), requires_grad=True)
    r = prob.residual(sys_.eqs[0], torch.tensor(X), th)
    (g,) = torch.autograd.grad((r ** 2).sum(), th)
    assert torch.all(torch.isfinite(g)) and g.abs().sum() > 0
    from oracle import reference as R
    want = R.phi(torch.tensor(X), th.detach(), *student) - torch.tensor(h)
    np.testing.assert_allclose(r.detach().numpy(), want.numpy(), rtol=1e-12, atol=1e-13)


def test_callable_loss_is_refused():
    _, _, pb = _teacher()
    sys_ = npde.PDESystem([npde.Eq(u(x, y), 0)], [npde.Eq(u(0, y), 0)], [npde.In(x, 0, 1), npde.In(y, 0, 1)],
                          [x, y], [u(x, y)])
    with pytest.raises(TypeError, match="NeuralAdapterLoss"):
        npde.neural_adapter(lambda cord, th: cord, np.zeros(3), sys_, npde.GridTraining(0.1))
    with pytest.raises(TypeError, match="NeuralAdapterLoss"):
        npde.neural_adapter([lambda cord, th: cord], np.zeros(3), [sys_], npde.GridTraining(0.1))


def test_register_symbolic_refusals():
    chain = npde.Chain(npde.Dense(2, 4, "tanh"), npde.Dense(4, 2))
    with pytest.raises(ValueError, match="1-dimensional output"):
        npde.register_symbolic(npde.Phi(chain, 0, chain.n_params, np.float64), np.zeros(chain.n_params))
    chain = npde.Chain(npde.Dense(2, 4, "tanh"), npde.Dense(4, 1))
    with pytest.raises(ValueError, match="theta has"):
        npde.register_symbolic(npde.Phi(chain, 0, chain.n_params, np.float64), np.zeros(3))
    with pytest.raises(TypeError):
        npde.register_symbolic(lambda c, t: c, np.zeros(3))
