"""Symbolic front end: a thin sympy stand-in for the ModelingToolkit objects a NeuralPDE
user writes (``@parameters``, ``@variables u(..)``, ``Differential``, ``~``, ``x ∈
Interval``, ``PDESystem``), plus the variable bookkeeping helpers of the reference
(``get_vars``, ``get_argument``, ``get_variables``; reference
src/symbolic_utilities.jl:401-526).

In the real deployment this layer stays in Julia (SURVEY section 1, L4-L5); it exists here
so that the parity tests read like the reference's own tests.
"""
from __future__ import annotations

import itertools
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Union

import sympy as sp
from sympy.core.function import AppliedUndef

Number = (int, float, sp.Number)


def parameters(names: str):
    """``@parameters x y`` -> sympy symbols (independent variables or equation parameters)."""
    syms = sp.symbols(names, real=True)
    return syms


def variables(names: str):
    """``@variables u(..) v(..)`` -> undefined functions; call them as ``u(x, y)``."""
    fs = [sp.Function(n) for n in names.replace(",", " ").split()]
    return fs[0] if len(fs) == 1 else tuple(fs)


class Differential:
    """``Dxx = Differential(x)^2``: ``Differential(x)**2`` or nested application.

    Applying it builds an *unevaluated* ``sympy.Derivative`` so that ``Dx(u(0, y))`` keeps
    meaning "partial derivative with respect to the input slot named x, evaluated at
    (0, y)" exactly as in the reference (src/symbolic_utilities.jl:160-201)."""

    def __init__(self, var: sp.Symbol, order: int = 1):
        self.x = var
        self.order = int(order)

    def __pow__(self, n: int) -> "Differential":
        return Differential(self.x, self.order * int(n))

    def __call__(self, expr):
        expr = sp.sympify(expr)
        if expr.is_number:          # Dx(c) = 0: SDEPINN's flux applies Dx to g(x_0, p, t)^2, a number
            return sp.Integer(0)
        return sp.Derivative(expr, (self.x, self.order), evaluate=False)


@dataclass(frozen=True)
class Equation:
    """``lhs ~ rhs``"""
    lhs: sp.Expr
    rhs: sp.Expr

    def __repr__(self):
        return "%s ~ %s" % (self.lhs, self.rhs)


def Eq(lhs, rhs) -> Equation:
    return Equation(sp.sympify(lhs), sp.sympify(rhs))


@dataclass(frozen=True)
class Interval:
    lo: float
    hi: float


@dataclass(frozen=True)
class VarDomain:
    """``x ∈ Interval(lo, hi)``"""
    variables: sp.Symbol
    domain: Interval


def In(var: sp.Symbol, lo: float, hi: float) -> VarDomain:
    return VarDomain(var, Interval(float(lo), float(hi)))


@dataclass
class PDESystem:
    """``PDESystem(eqs, bcs, domains, ivs, dvs, ps; defaults)``"""
    eqs: List[Equation]
    bcs: List[Equation]
    domain: List[VarDomain]
    ivs: List[sp.Symbol]
    dvs: List[sp.Expr]                    # e.g. [u(x, y)]
    ps: List[sp.Symbol] = field(default_factory=list)
    defaults: Dict[sp.Symbol, float] = field(default_factory=dict)

    def __post_init__(self):
        if isinstance(self.eqs, Equation):
            self.eqs = [self.eqs]
        if isinstance(self.bcs, Equation):
            self.bcs = [self.bcs]
        self.eqs = list(self.eqs)
        self.bcs = list(self.bcs)


# ---- variable bookkeeping (reference src/symbolic_utilities.jl:401-426) -------------------------
@dataclass
class VarInfo:
    depvars: List[str]
    indvars: List[str]
    dict_indvars: Dict[str, int]          # name -> 0-based index
    dict_depvars: Dict[str, int]
    dict_depvar_input: Dict[str, List[str]]


def get_vars(indvars_: Sequence[sp.Symbol], depvars_: Sequence[sp.Expr]) -> VarInfo:
    indvars = [str(v) for v in indvars_]
    depvars, dep_in = [], {}
    for d in depvars_:
        if isinstance(d, AppliedUndef):
            name = d.func.__name__
            depvars.append(name)
            dep_in[name] = [str(a) for a in d.args]
        else:                                   # bare name: defaults to all inputs
            name = str(d)
            depvars.append(name)
            dep_in[name] = list(indvars)
    return VarInfo(depvars, indvars, {n: i for i, n in enumerate(indvars)},
                   {n: i for i, n in enumerate(depvars)}, dep_in)


def _depvar_apps(expr: sp.Expr, vi: VarInfo) -> List[AppliedUndef]:
    """Applications of dependent variables in first-seen (pre-order) order, de-duplicated."""
    seen, out = set(), []
    for node in sp.preorder_traversal(expr):
        if isinstance(node, AppliedUndef) and node.func.__name__ in vi.dict_depvars and node not in seen:
            seen.add(node)
            out.append(node)
    return out


def _eq_expr(eq: Equation) -> sp.Expr:
    # a container holding both sides; traversal order lhs then rhs like the reference's toexpr(eq)
    return sp.Tuple(eq.lhs, eq.rhs)


def get_argument(eqs: Sequence[Equation], vi: VarInfo) -> List[list]:
    """Arguments used in each equation: for every dependent variable (in depvar order) the
    arguments of its first occurrence; symbols are de-duplicated, numbers are kept
    (reference src/symbolic_utilities.jl:498-526)."""
    out = []
    for eq in eqs:
        apps = _depvar_apps(_eq_expr(eq), vi)
        first = {}
        for a in apps:
            first.setdefault(a.func.__name__, a)
        args, syms = [], set()
        for name in vi.depvars:
            if name not in first:
                continue
            for a in first[name].args:
                if isinstance(a, sp.Symbol):
                    if str(a) in syms:
                        continue
                    syms.add(str(a))
                    args.append(str(a))
                else:
                    args.append(float(a))
        out.append(args)
    return out


def get_variables(eqs: Sequence[Equation], vi: VarInfo) -> List[List[str]]:
    """Only the symbolic arguments (reference src/symbolic_utilities.jl:456-468)."""
    return [[a for a in args if isinstance(a, str)] for args in get_argument(eqs, vi)]


def eq_depvars(eq: Equation, vi: VarInfo) -> List[str]:
    """Dependent variables appearing in an equation, in depvar order (``pair``,
    reference src/symbolic_utilities.jl:391-399)."""
    names = {a.func.__name__ for a in _depvar_apps(_eq_expr(eq), vi)}
    return [n for n in vi.depvars if n in names]


def eq_indvars(eq: Equation, vi: VarInfo) -> List[str]:
    """``this_eq_indvars``: ordered union of the declared inputs of the equation's dependent
    variables (reference src/discretize.jl:43-44).  Row i of the term's point matrix is
    bound to the i-th name (src/discretize.jl:126)."""
    out: List[str] = []
    for n in eq_depvars(eq, vi):
        for v in vi.dict_depvar_input[n]:
            if v not in out:
                out.append(v)
    return out


def expand_derivatives(expr: sp.Expr) -> sp.Expr:
    """``expand_derivatives`` with the reference's fallback: keep the raw form when the
    expansion vanishes (reference src/symbolic_utilities.jl:360-364)."""
    expr = sp.sympify(expr)
    try:
        ex = expr.doit()
    except Exception:
        return expr
    return expr if ex == 0 else ex


# ---- integral terms (Symbolics.Integral with DomainSets domains; reference src/symbolic_utilities.jl:203-320) ------
Inf = sp.oo


@dataclass(frozen=True)
class ClosedInterval:
    """``ClosedInterval(lo, hi)``: each bound a number, ±``Inf`` or an expression of the coordinates."""
    lo: object
    hi: object


def UnitInterval() -> ClosedInterval:
    return ClosedInterval(0, 1)


@dataclass(frozen=True)
class ProductDomain:
    """``ProductDomain(d1, d2)``: one interval per integrating variable, in order."""
    domains: tuple

    def __init__(self, *domains):
        object.__setattr__(self, "domains", tuple(domains))


def UnitSquare() -> ProductDomain:
    return ProductDomain(UnitInterval(), UnitInterval())


class IntegralOp(sp.Function):
    """Unevaluated ``Integral(vars in domain)(integrand)``: args (integrand, Tuple(vars), Tuple(lbs), Tuple(ubs))."""
    nargs = 4

    @classmethod
    def eval(cls, *args):
        return None


class Integral:
    """``Integral(x in ClosedInterval(0, x))`` -> ``Integral(x, ClosedInterval(0, x))``;
    ``Integral((x, y) in UnitSquare())`` -> ``Integral((x, y), UnitSquare())``.  Applying it to an expression gives
    the unevaluated integral, evaluated per collocation point of the equation (lowering.py)."""

    def __init__(self, variables, domain):
        vs = tuple(variables) if isinstance(variables, (tuple, list)) else (variables,)
        doms = domain.domains if isinstance(domain, ProductDomain) else (domain,)
        if len(vs) != len(doms):
            raise ValueError("Integral: %d variables over a %d-dimensional domain" % (len(vs), len(doms)))
        if not all(isinstance(d_, ClosedInterval) for d_ in doms):
            raise TypeError("Integral: domains are ClosedInterval / UnitInterval / UnitSquare / ProductDomain")
        self.variables = vs
        self.lbs = tuple(sp.sympify(d_.lo) for d_ in doms)
        self.ubs = tuple(sp.sympify(d_.hi) for d_ in doms)

    def __call__(self, expr):
        return IntegralOp(sp.sympify(expr), sp.Tuple(*self.variables), sp.Tuple(*self.lbs), sp.Tuple(*self.ubs))


# ---- registered network functions (``@register_symbolic phi_bound(x, y)``) ------------------------------------------
@dataclass(eq=False)
class FixedNet:
    """A trained 1-output Dense MLP whose parameters stay fixed: dims, activations and its flat Lux parameters."""
    dims: List[int]
    acts: List[str]
    params: "object"          # numpy array (float64 copy)


_fixed_ids = itertools.count()


def fixed_function(name: str, net: FixedNet):
    """A sympy function whose applications (and derivatives of them) the lowering evaluates with the fixed network
    ``net``.  Every call gives a distinct function, even under one name, so two teachers never compare equal."""
    f = sp.Function(name, real=True, fixed_id=next(_fixed_ids))
    f.fixed_net = net
    return f


def fixed_net_of(e) -> Optional[FixedNet]:
    """The fixed network of an application of a registered function, or None."""
    return getattr(e.func, "fixed_net", None) if isinstance(e, AppliedUndef) else None
