"""Integral terms on the host: lowering, the Gauss-Legendre rule against the reference's adaptive integral, the
reference's own known answers (test/Forward/forward__integral.jl) and the refusals of the Python layer."""
import numpy as np
import pytest
import sympy as sp
import torch

import neuralpde_jl_b200 as npde
from neuralpde_jl_b200 import engine as E
from neuralpde_jl_b200.lowering import DEFAULT_QUAD_NODES, LoweringError, lower_equation
from neuralpde_jl_b200.symbolic import get_vars
from oracle import reference as R

import integral_cases as IC
from integral_oracle import IntegralProblem


def _lower(case, k=0, hoist=True):
    sys_, chains, _ = case()
    vi = get_vars(sys_.ivs, sys_.dvs)
    return lower_equation(sys_.eqs[k], vi, hoist=hoist)


# ---- lowering ----------------------------------------------------------------------------------------------------------
def test_lowering_ide1_variable_upper_bound():
    lt = _lower(IC.ide1)
    assert lt.indvars == ["t"] and not lt.extra_exprs
    assert ("integral", 0, 0, 0.0) in lt.prog and lt.prog[-1][0] == "sub"
    (it,) = lt.integrals
    assert (it.n_dims, it.q, it.rows[0]) == (1, DEFAULT_QUAD_NODES, 0)
    assert (it.lb[0], it.lb_row[0], it.ub_row[0], it.inf_kind[0]) == (0.0, -1, 0, E.INF_NONE)
    assert it.prog == [("tap", 0, 0, 0.0)] and it.taps[0].order == 0 and it.net_rows == [[0]]


def test_lowering_ide2_coordinate_in_integrand():
    (it,) = _lower(IC.ide2).integrals
    ops = [p[0] for p in it.prog]
    assert sorted(ops) == ["coord", "cos", "mul", "tap"] and ops[-1] == "mul"   # u(x) * cos(x) at the node coordinate
    assert ("coord", 0, 0, 0.0) in it.prog and it.ub_row[0] == 0


def test_lowering_ide3_unit_square():
    lt = _lower(IC.ide3)
    (it,) = lt.integrals
    assert it.n_dims == 2 and it.rows == [0, 1]
    assert (it.lb, it.ub, it.lb_row, it.ub_row) == ([0.0, 0.0], [1.0, 1.0], [-1, -1], [-1, -1])
    assert not lt.taps                                    # the owner reads only the integral
    assert lt.prog == [("integral", 0, 0, 0.0), ("const", 0, 0, 1 / 3), ("sub", 0, 1, 0.0)]


def test_lowering_ide4_bound_is_owner_row():
    (it,) = _lower(IC.ide4).integrals
    assert it.n_dims == 2 and it.rows == [0, 1]
    assert (it.lb_row, it.ub_row, it.ub) == ([-1, -1], [-1, 0], [1.0, 0.0])


def test_lowering_ide5_two_networks():
    (it,) = _lower(IC.ide5).integrals
    assert sorted(t.net for t in it.taps) == [0, 1]
    assert [p[0] for p in it.prog] == ["tap", "tap", "mul"]
    assert it.net_rows == [[0], [0]] and (it.lb[0], it.ub_row[0]) == (1.0, 0)


def test_lowering_ide6_two_integrals_and_semi_infinite():
    lt = _lower(IC.ide6)
    fin, inf = lt.integrals
    assert sum(1 for p in lt.prog if p[0] == "integral") == 2
    assert fin.inf_kind[0] == E.INF_NONE and (fin.lb[0], fin.ub_row[0]) == (1.0, 0)
    # [1, Inf): x = 1 + t / (1 - t), t in [0, 1 - 1/20], Jacobian 1 / (1 - t)^2 read from the t row, which follows the
    # owner's rows (x, and 1/x hoisted)
    assert inf.inf_kind[0] == E.INF_UPPER and inf.shift[0] == 1.0
    assert (inf.lb[0], inf.ub[0], inf.lb_row[0], inf.ub_row[0]) == (0.0, 0.95, -1, -1)
    assert lt.dim == 2 and ("coord", 2, 0, 0.0) in inf.prog and inf.prog[-1][0] == "div"


def test_lowering_ide7_coordinate_lower_bound_to_infinity():
    lt = _lower(IC.ide7)
    (it,) = lt.integrals
    # [x, Inf): x = t / (1 - t) from t = x / (1 + x), a hoisted owner row; the t row follows it
    assert lt.extra_exprs == [sp.Symbol("x", real=True) / (1 + sp.Symbol("x", real=True))]
    assert it.inf_kind[0] == E.INF_UPPER and it.shift[0] == 0.0 and it.lb_row[0] == 1
    assert ("coord", 2, 0, 0.0) in it.prog


# ---- Gauss-Legendre table -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("q", [1, 2, 5, 16, 33, 64])
def test_node_table_matches_leggauss(q):
    x, w = E.quadrature_nodes(q)
    xr, wr = np.polynomial.legendre.leggauss(q)
    np.testing.assert_allclose(x, xr, rtol=0, atol=2e-15)
    # leggauss's own weights drift to ~1.3e-12 relative near the ends at q = 64 (against a 40-digit evaluation, where the
    # engine's table stays below 1e-13)
    np.testing.assert_allclose(w, wr, rtol=2e-12, atol=1e-15)
    assert abs(w.sum() - 2) < 1e-14


# ---- the fixed rule against the reference's adaptive integral ---------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(IC.REFERENCE))
def test_gauss_matches_adaptive_within_reference_tolerance(name):
    sys_, chains, dx = IC.REFERENCE[name]()
    theta = torch.as_tensor(IC.init_params(chains))
    sets, _ = R.generate_training_sets(sys_.domain, dx, sys_.eqs, sys_.bcs, sys_.ivs, sys_.dvs)
    step = 3 if len(sys_.ivs) == 2 else 1                # every third point of the 2-D grids keeps dblquad quick
    for k, (eq, s) in enumerate(zip(sys_.eqs, sets)):
        pts = torch.as_tensor(s[:, ::step])
        g = IntegralProblem(sys_, IC.chain_specs(chains), quad="gauss").residual(eq, pts, theta)
        a = IntegralProblem(sys_, IC.chain_specs(chains), quad="adaptive").residual(eq, pts, theta)
        err = (g - a).abs().max().item()
        assert err <= 1e-3 * max(1.0, a.abs().max().item()), (name, k, err)


# ---- test/Forward/forward__integral.jl ---------------------------------------------------------------------------------------
def _forward_integral_system(lo, hi):
    x = npde.parameters("x")
    u = npde.variables("u")
    I = npde.Integral(x, npde.ClosedInterval(lo, hi))
    return npde.PDESystem([npde.Eq(I(u(x)), 0)], [npde.Eq(u(1.0), 0)], [npde.In(x, 1.0, 2.0)], [x], [u(x)])


def test_forward_integral_zero_to_infinity_rtol_1e5():
    sys_ = _forward_integral_system(0, npde.Inf)
    prob = IntegralProblem(sys_, [([1, 1], ["identity"])],
                           closures={"u": lambda c: torch.exp(c) / (torch.exp(2 * c) + 3)})
    v = prob.residual(sys_.eqs[0], torch.ones(1, 1, dtype=torch.float64), torch.zeros(2)).item()
    assert v == pytest.approx(np.pi / (3 * np.sqrt(3)), rel=1e-5)


def test_forward_integral_whole_line_atol_1e13():
    sys_ = _forward_integral_system(-npde.Inf, npde.Inf)
    prob = IntegralProblem(sys_, [([1, 1], ["identity"])], closures={"u": lambda c: c * torch.exp(-c ** 2)})
    v = prob.residual(sys_.eqs[0], torch.ones(1, 1, dtype=torch.float64), torch.zeros(2)).item()
    assert abs(v) <= 1e-13


def test_default_node_count_is_needed():
    """12 nodes still meet rtol = 1e-5 on [0, Inf), 10 do not: the default (16) is not arbitrary slack."""
    sys_ = _forward_integral_system(0, npde.Inf)
    exact = np.pi / (3 * np.sqrt(3))
    errs = {}
    for q in (10, 12):
        prob = IntegralProblem(sys_, [([1, 1], ["identity"])], q=q,
                               closures={"u": lambda c: torch.exp(c) / (torch.exp(2 * c) + 3)})
        errs[q] = abs(prob.residual(sys_.eqs[0], torch.ones(1, 1, dtype=torch.float64), torch.zeros(2)).item() - exact)
    assert errs[12] <= 1e-5 * exact < errs[10]


# ---- refusals of the Python layer --------------------------------------------------------------------------------------------
def test_refuses_three_integrating_dimensions():
    x, y, z = npde.parameters("x y z")
    u = npde.variables("u")
    I = npde.Integral((x, y, z), npde.ProductDomain(npde.UnitInterval(), npde.UnitInterval(), npde.UnitInterval()))
    vi = get_vars([x, y, z], [u(x, y, z)])
    with pytest.raises(LoweringError, match="at most 2 integrating dimensions"):
        lower_equation(npde.Eq(I(u(x, y, z)), 0), vi)


def test_refuses_nested_integral():
    x = npde.parameters("x")
    u = npde.variables("u")
    I = npde.Integral(x, npde.ClosedInterval(0, x))
    with pytest.raises(LoweringError, match="nested"):
        lower_equation(npde.Eq(I(I(u(x))), 0), get_vars([x], [u(x)]))


def test_refuses_bound_depending_on_a_dependent_variable():
    x = npde.parameters("x")
    u = npde.variables("u")
    I = npde.Integral(x, npde.ClosedInterval(0, u(x)))
    with pytest.raises(LoweringError, match="dependent variables"):
        lower_equation(npde.Eq(I(u(x)), 0), get_vars([x], [u(x)]))


def test_refuses_expression_bound_without_host_rows():
    """device-sampled point sets carry coordinates only: a bound x / (1 + x) has no row to live in"""
    with pytest.raises(LoweringError, match="device-sampled"):
        _lower(IC.ide7, hoist=False)


def test_refuses_infinite_bounds_in_two_dimensions():
    x, y = npde.parameters("x y")
    u = npde.variables("u")
    I = npde.Integral((x, y), npde.ProductDomain(npde.ClosedInterval(0, npde.Inf), npde.UnitInterval()))
    with pytest.raises(LoweringError, match="1-dimensional integrals only"):
        lower_equation(npde.Eq(I(u(x, y)), 0), get_vars([x, y], [u(x, y)]))


def test_refuses_integrand_without_network():
    x = npde.parameters("x")
    u = npde.variables("u")
    I = npde.Integral(x, npde.ClosedInterval(0, x))
    with pytest.raises(LoweringError, match="no dependent variable"):
        lower_equation(npde.Eq(u(x) + I(x ** 2), 0), get_vars([x], [u(x)]))
