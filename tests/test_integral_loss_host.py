"""Integral constraints (pinn.IntegralLoss) without a GPU: lowering of the integrand and the target fold, both node
rules, the float64 restatement (tests/integral_loss_oracle.py) against scipy's adaptive quadrature, the normalisation
constants of the reference's two Fokker-Planck forms, and every refusal on the Python side."""
import numpy as np
import pytest
import sympy as sp
import torch
from scipy import integrate

import neuralpde_jl_b200 as npde
from neuralpde_jl_b200 import engine as E
from neuralpde_jl_b200.pinn import Phi, _integral_loss_term, register_symbolic
from neuralpde_jl_b200.symbolic import get_vars
from oracle import reference as R

import integral_loss_cases as LC
from integral_loss_oracle import IntegralLossProblem


def _lower(add, sys_, param_index=None, param_values=None, fixed=None):
    vi = get_vars(sys_.ivs, sys_.dvs)
    return _integral_loss_term(add, vi, param_index or {}, param_values or {}, [] if fixed is None else fixed)


def test_lowering_taps_param_and_target_fold():
    sys_, chains, _, add, _ = LC.taps_and_param()
    spec, X, w = _lower(add, sys_, param_index={"a": 0})
    assert spec.reduction == E.REDUCE_ABS_OF_SUM and spec.scale == 1.0 and spec.dim == 1
    assert sorted(t.order for t in spec.taps) == [0, 1, 2]
    assert any(ins[0] == "param" for ins in spec.prog)
    # the last instruction is v - target / Σw
    op, a, b, _ = spec.prog[-1]
    assert op == "sub" and spec.prog[b][0] == "const"
    assert spec.prog[b][3] == pytest.approx(0.3 / w.sum(), rel=1e-15)
    # with the default parameter substituted instead (param_estim = false): no PARAM instruction
    spec2, _, _ = _lower(add, sys_, param_values={"a": 0.7})
    assert not any(ins[0] == "param" for ins in spec2.prog)


def test_lowering_abs2_without_target_has_zero_shift():
    sys_, _, _, add, _ = LC.neumann2d()
    spec, X, w = _lower(add, sys_)
    assert spec.reduction == E.REDUCE_SQUARE_OF_SUM and X.shape == (2, 64)
    op, a, b, _ = spec.prog[-1]
    assert op == "sub" and spec.prog[b] == ("const", 0, 0, 0.0)


def test_lowering_registered_function():
    sys_, x, p = LC.fokker_planck_system()
    teacher = LC.fp_chain(6)
    th = np.random.default_rng(0).standard_normal(teacher.n_params)
    f = register_symbolic(Phi(teacher, 0, teacher.n_params, np.float64), th, "teacher")
    fixed = []
    spec, _, _ = _lower(npde.IntegralLoss(p(x) * f(x), list(sys_.domain)), sys_, fixed=fixed)
    assert len(fixed) == 1 and sorted(t.net for t in spec.taps) == [0, 1]
    assert spec.net_rows[1] == [0]


def test_gauss_legendre_nodes():
    sys_, _, _, add, _ = LC.neumann2d()
    X, w = add.nodes(["x", "y"])
    xi, wq = np.polynomial.legendre.leggauss(8)
    assert X.shape == (2, 64) and w.sum() == pytest.approx(1.0, rel=1e-14)
    np.testing.assert_allclose(np.unique(X[0]), 0.5 * xi + 0.5, rtol=1e-14)
    # the rule integrates x^3 y^2 exactly
    assert np.sum(w * X[0] ** 3 * X[1] ** 2) == pytest.approx(1 / 12, rel=1e-13)


def test_explicit_nodes_and_default_weights():
    _, _, _, add, _ = LC.fokker_planck_tutorial()
    X, w = add.nodes(["x"])
    assert X.shape == (1, 200) and w.shape == (200,)
    assert w[0] == pytest.approx(0.01 * 4.4 / 199, rel=1e-14)
    X2, w2 = npde.IntegralLoss(add.integrand, points=np.linspace(0, 1, 5)).nodes(["x"])
    assert X2.shape == (1, 5) and np.all(w2 == 1.0)
    _, w3 = npde.IntegralLoss(add.integrand, points=np.linspace(0, 1, 5), weights=0.25).nodes(["x"])
    assert np.all(w3 == 0.25)


def test_oracle_against_adaptive_quadrature():
    """the restatement's Gauss-Legendre sum of a network integrand against scipy.integrate.quad of the same function"""
    sys_, chains, _, _, _ = LC.fokker_planck()
    x, p = sys_.ivs[0], sys_.dvs[0].func
    integrand = p(x) * x ** 2 + sp.sin(x)
    th = torch.as_tensor(LC.IC.init_params(chains))
    add = npde.IntegralLoss(integrand, list(sys_.domain), nodes_per_dim=40)
    X, w = add.nodes(["x"])
    prob = IntegralLossProblem(sys_, LC.IC.chain_specs(chains), integrand=integrand, X=X, w=w, target=0.25, norm="abs2")
    c = chains[0]

    def f(t):
        v = R.phi(torch.tensor([[t]]), th, c.dims, c.acts)
        return float(v) * t ** 2 + np.sin(t)

    ref = integrate.quad(f, LC.X0, LC.X1, epsabs=1e-12, epsrel=1e-12)[0]
    assert float(torch.sum(prob.w * prob.values(th))) == pytest.approx(ref, rel=1e-10)
    assert float(prob.functional(th)) == pytest.approx((ref - 0.25) ** 2, rel=1e-9)


def test_normalisation_constants():
    """C of the test's constraint |0.01 ∫p - 4.4| = 0 and of the tutorial's 0.01 Σ p Δx = 1"""
    I = integrate.quad(lambda t: np.exp((2 * LC.ALPHA * t ** 2 - LC.BETA * t ** 4) / (2 * LC.SIGMA ** 2)),
                       LC.X0, LC.X1, epsabs=1e-13, epsrel=1e-13)[0]
    assert I == pytest.approx(3.07978, abs=1e-5)
    assert 440.0 / I == pytest.approx(LC.C_TEST, abs=1e-1)
    assert abs(440.0 / I - LC.C_TEST) < 2e-2
    assert 100.0 / I == pytest.approx(LC.C_TUTORIAL, abs=5e-3)


# ---- refusals ----------------------------------------------------------------------------------------------------------
def _disc(case, **kw):
    return LC.discretization(case, **kw)


def test_refuses_callable_additional_loss():
    sys_, chains, strategy, _, _ = LC.fokker_planck()
    d = npde.PhysicsInformedNN(chains[0], strategy, additional_loss=lambda phi, th, p: 0.0)
    with pytest.raises(ValueError, match="DataLoss .* IntegralLoss"):
        npde.symbolic_discretize(sys_, d)


def test_refuses_callable_integrand():
    sys_, _, _, _, _ = LC.fokker_planck()
    with pytest.raises(ValueError, match="not a callable"):
        _lower(npde.IntegralLoss(lambda x: x, list(sys_.domain)), sys_)


@pytest.mark.parametrize("mode", ["tc_bf16", "tc_split"])
def test_refuses_tensor_core_modes(mode):
    case = LC.fokker_planck()
    with pytest.raises(ValueError, match="FFMA path"):
        npde.symbolic_discretize(case[0], _disc(case, dtype=np.float32, mode=mode))


def test_refuses_bayesian_pinn():
    sys_, chains, _, add, _ = LC.fokker_planck()
    d = npde.BayesianPINN(chains[0], npde.GridTraining(0.1), additional_loss=add)
    with pytest.raises(ValueError, match="BayesianPINN: an IntegralLoss"):
        npde.symbolic_discretize(sys_, d)
    with pytest.raises(ValueError, match="additional_loss"):
        npde.ahmc_bayesian_pinn_pde(sys_, d, draw_samples=10, bcstd=[0.1, 0.1], phystd=[0.1])


@pytest.mark.parametrize("kw,msg", [
    (dict(norm="l1"), "norm must be"),
    (dict(), "either domains .* or explicit points"),
    (dict(domains=[1], points=np.zeros((1, 3))), "either domains"),
    (dict(points=None, weights=np.ones(3), domains=[1]), "weights go with explicit points"),
    (dict(domains=[1], nodes_per_dim=0), "nodes_per_dim"),
])
def test_refuses_bad_arguments(kw, msg):
    args = dict(domains=None)
    args.update(kw)
    domains = args.pop("domains")
    with pytest.raises(ValueError, match=msg):
        npde.IntegralLoss(sp.Symbol("x"), domains, **args)


def test_refuses_bad_nodes():
    sys_, x, p = LC.fokker_planck_system()
    with pytest.raises(ValueError, match=r"points must be \(1, n\)"):
        _lower(npde.IntegralLoss(p(x), points=np.zeros((2, 4))), sys_)
    with pytest.raises(ValueError, match="weights must have shape"):
        _lower(npde.IntegralLoss(p(x), points=np.zeros((1, 4)), weights=np.ones(3)), sys_)
    with pytest.raises(ValueError, match="weights sum to 0"):
        _lower(npde.IntegralLoss(p(x), points=np.zeros((1, 2)), weights=np.array([1.0, -1.0]), target=1.0), sys_)
    y = npde.parameters("y")
    with pytest.raises(ValueError, match="no domain for the variables"):
        _lower(npde.IntegralLoss(p(x), [npde.In(y, 0.0, 1.0)]), sys_)
    with pytest.raises(ValueError, match="applies no dependent variable"):
        _lower(npde.IntegralLoss(x ** 2, list(sys_.domain)), sys_)


def test_refuses_integral_in_integrand():
    sys_, x, p = LC.fokker_planck_system()
    Ix = npde.Integral(x, npde.ClosedInterval(0, x))
    with pytest.raises(ValueError, match="may not contain an Integral"):
        _lower(npde.IntegralLoss(p(x) + Ix(p(x)), list(sys_.domain)), sys_)
