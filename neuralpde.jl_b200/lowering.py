"""Lowering of one equation / boundary condition to the engine's residual IR.

Input: the equation after ``expand_derivatives`` (so every derivative chain ends directly on
a dependent-variable call -- the invariant the reference's tap extractor relies on,
src/symbolic_utilities.jl:160-174).  Output: the tap list (pure partial derivatives of one
network each) and an SSA program computing ``lhs - rhs`` per point from taps, coordinate
rows and parameters -- the same quantity the reference's generated function returns
(src/symbolic_utilities.jl:360-370, src/discretize.jl:126-151).

In deployment this is what the Julia shim does with ``pinnrep.symbolic_*_loss_functions``
(INTEGRATION.md); it lives here in Python because Julia is absent from the build image.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import sympy as sp
from sympy.core.function import AppliedUndef

from .engine import (DEFAULT_QUAD_NODES, INF_BOTH, INF_LOWER, INF_NONE, INF_UPPER, IntegralSpec, TapSpec, TermSpec,
                     REDUCE_MEAN)
from .symbolic import (Equation, FixedNet, IntegralOp, VarInfo, _depvar_apps, _eq_expr, eq_indvars, expand_derivatives,
                       fixed_net_of)


class LoweringError(ValueError):
    pass


@dataclass
class LoweredTerm:
    taps: List[TapSpec]
    prog: List[tuple]
    indvars: List[str]               # row i of the term's point matrix is this variable
    net_rows: List[Optional[List[int]]]
    # coordinate-only subexpressions hoisted out of the per-step program: evaluated once per point set
    # (float64, on the host) and appended as extra rows dim, dim+1, ... of the point matrix
    extra_exprs: List[sp.Expr] = None
    # integral terms the program reads with ("integral", k): owner -1 and k local to this term until
    # symbolic_discretize places them
    integrals: List[IntegralSpec] = None

    @property
    def dim(self) -> int:
        return len(self.indvars) + len(self.extra_exprs or [])

    def augment(self, pts):
        """(d, N) coordinates -> (d + n_extra, N) with the hoisted rows appended."""
        import numpy as np
        pts = np.asarray(pts)
        if not self.extra_exprs:
            return pts
        if pts.shape[0] != len(self.indvars):
            raise ValueError("expected %d coordinate rows, got %d" % (len(self.indvars), pts.shape[0]))
        rows64 = [pts[i].astype(np.float64) for i in range(pts.shape[0])]
        fns = getattr(self, "_extra_fns", None)
        if fns is None:          # compiled once per term: resampling strategies call augment on every loss evaluation
            syms = [sp.Symbol(v, real=True) for v in self.indvars]
            fns = [sp.lambdify(syms, e, "numpy") for e in self.extra_exprs]
            self._extra_fns = fns
        extra = []
        for f in fns:
            extra.append(np.broadcast_to(np.asarray(f(*rows64), dtype=np.float64), rows64[0].shape))
        return np.concatenate([pts, np.stack(extra).astype(pts.dtype)], axis=0)


MAX_DIM = 8   # PINN_MAX_DIM
MAX_FIXED_NETS = 16   # PINN_MAX_FIXED_NETS
# the reference truncates the substituted intervals of infinite bounds by 1/20 (src/transform_inf_integral.jl)
INF_EPS = 1.0 / 20


def _hoist_coordinate_terms(expr, coord_names, blocked_names, extras, base_dim):
    """Replace maximal coordinate-only subexpressions (no network tap, no trainable parameter) by fresh
    symbols __c<i>; trivial ones (a bare symbol / number, or fewer than 2 operations) stay inline."""
    def has_net(e):
        return e.has(AppliedUndef) or e.has(sp.Derivative) or e.has(IntegralOp) or \
            any(str(q) in blocked_names for q in e.free_symbols)

    def rec(e):
        if isinstance(e, (AppliedUndef, sp.Derivative, sp.Subs, IntegralOp)):
            return e
        if not has_net(e):
            names = {str(q) for q in e.free_symbols}
            if names and names <= coord_names and not isinstance(e, sp.Symbol) and e.count_ops() >= 2 \
                    and base_dim + len(extras) < MAX_DIM:
                for i, old in enumerate(extras):
                    if old == e:
                        return sp.Symbol("__c%d" % i, real=True)
                extras.append(e)
                return sp.Symbol("__c%d" % (len(extras) - 1), real=True)
            return e
        if isinstance(e, (sp.Add, sp.Mul)):
            pure = [a for a in e.args if not has_net(a)]
            rest = [rec(a) for a in e.args if has_net(a)]
            if pure:
                rest.append(rec(e.func(*pure)))
            return e.func(*rest, evaluate=False) if len(rest) > 1 else rest[0]
        if e.args:
            return e.func(*[rec(a) for a in e.args])
        return e

    return rec(sp.sympify(expr))


class _Emitter:
    def __init__(self, vi: VarInfo, rows: List[str], param_index: Dict[str, int], param_values: Dict[str, float],
                 extras: Optional[List[sp.Expr]] = None, hoist: bool = False, node_vars: Optional[Dict[str, int]] = None,
                 fixed: Optional[List[FixedNet]] = None, const_rows: Optional[Dict[float, int]] = None):
        self.vi = vi
        self.rows = rows
        self.param_index = param_index
        self.param_values = param_values
        self.prog: List[tuple] = []
        self.taps: List[TapSpec] = []
        self._tap_ids: Dict[tuple, int] = {}
        self._cse: Dict[object, int] = {}
        self.extras = extras if extras is not None else []   # hoisted rows (an integral's expression bounds land here)
        self.hoist = hoist
        self.node_vars = node_vars or {}    # integrand: quadrature variable t_k -> ("coord", -1 - k) until placed
        self.integrals: List[IntegralSpec] = []
        # registered network functions: the problem's fixed networks (shared by its equations; tap network
        # len(depvars) + j is fixed[j]), the point rows each one reads here, and the rows that hold constant arguments
        self.fixed = fixed if fixed is not None else []
        self.fixed_rows: Dict[int, List[int]] = {}
        self.const_rows = const_rows or {}

    def _push(self, op, a=0, b=0, imm=0.0) -> int:
        key = (op, a, b, float(imm))
        if key in self._cse:
            return self._cse[key]
        self.prog.append((op, int(a), int(b), float(imm)))
        self._cse[key] = len(self.prog) - 1
        return len(self.prog) - 1

    def const(self, v: float) -> int:
        return self._push("const", imm=float(v))

    def tap(self, depvar: str, dirs: Tuple[int, ...]) -> int:
        return self._tap_net(self.vi.dict_depvars[depvar], depvar, dirs)

    def fixed_tap(self, app: AppliedUndef, dirvars: List[str]) -> int:
        """A value or partial derivative of a registered network function at its arguments: coordinates of the
        equation, or constants bound to the rows that hold them (``phi_bound(x_0, y)``)."""
        name, fn = app.func.__name__, fixed_net_of(app)
        if len(app.args) != fn.dims[0]:
            raise LoweringError("%s called with %d arguments; its network has %d inputs" % (name, len(app.args), fn.dims[0]))
        rows = []
        for a in app.args:
            if isinstance(a, sp.Symbol) and str(a) in self.rows:
                rows.append(self.rows.index(str(a)))
            elif a.is_number and float(a) in self.const_rows:
                rows.append(self.const_rows[float(a)])
            else:
                raise LoweringError("%s(%s): arguments of a registered function are the equation's coordinates %s or "
                                    "constants that a dependent variable of the equation takes at the same position"
                                    % (name, ", ".join(map(str, app.args)), self.rows))
        j = next((i for i, f in enumerate(self.fixed) if f is fn), None)
        if j is None:
            if len(self.fixed) >= MAX_FIXED_NETS:
                raise LoweringError("more than %d registered network functions in one problem" % MAX_FIXED_NETS)
            self.fixed.append(fn)
            j = len(self.fixed) - 1
        net = len(self.vi.depvars) + j
        if self.fixed_rows.setdefault(net, rows) != rows:
            raise LoweringError("%s is applied to different arguments in one equation" % name)
        dirs = []
        for v in dirvars:
            pos = [i for i, a in enumerate(app.args) if isinstance(a, sp.Symbol) and str(a) == v]
            if len(pos) != 1:
                raise LoweringError("derivative of %s with respect to %s, which is not exactly one of its arguments %s"
                                    % (app, v, list(app.args)))
            dirs.append(pos[0])
        return self._tap_net(net, name, tuple(dirs))

    def _tap_net(self, net: int, depvar: str, dirs: Tuple[int, ...]) -> int:
        dirs = tuple(sorted(dirs))
        key = (net, dirs)
        if key not in self._tap_ids:
            if len(dirs) > 3 or (len(dirs) == 3 and len(set(dirs)) != 1):
                raise LoweringError(
                    "derivative of order %d of %s along %s: this engine propagates exact taps up to order 2 in any "
                    "directions and pure third derivatives (the reference's order-4 stencil and the recursive mixed "
                    "forms, src/pinn_types.jl:454-474, are not covered)" % (len(dirs), depvar, list(dirs)))
            self._tap_ids[key] = len(self.taps)
            self.taps.append(TapSpec(net=net, order=len(dirs), dirs=dirs))
        return self._push("tap", a=self._tap_ids[key])

    # -- expression walk -----------------------------------------------------------------------
    def emit(self, e: sp.Expr) -> int:
        e = sp.sympify(e)
        if isinstance(e, (sp.Number, sp.NumberSymbol)) or e.is_number and not e.free_symbols and not e.has(AppliedUndef):
            return self.const(float(e))
        if isinstance(e, sp.Symbol):
            name = str(e)
            if name in self.rows:
                return self._push("coord", a=self.rows.index(name))
            if name.startswith("__c"):
                return self._push("coord", a=len(self.rows) + int(name[3:]))
            if name in self.node_vars:
                return self._push("coord", a=-1 - self.node_vars[name])
            if name in self.param_index:
                return self._push("param", a=self.param_index[name])
            if name in self.param_values:
                return self.const(self.param_values[name])
            if name in self.vi.dict_indvars:
                raise LoweringError(
                    "independent variable %s is not an input of any dependent variable in this equation" % name)
            raise LoweringError("unknown symbol %s (not an independent variable or a parameter with a default)" % name)
        if isinstance(e, IntegralOp):
            if self.node_vars:
                raise LoweringError("integral nested in an integrand: not supported")
            return self._push("integral", a=self.integral(e))
        if isinstance(e, AppliedUndef) and fixed_net_of(e) is not None:
            return self.fixed_tap(e, [])
        if isinstance(e, AppliedUndef):
            name = e.func.__name__
            if name not in self.vi.dict_depvars:
                raise LoweringError("unknown function %s" % name)
            if len(e.args) != len(self.vi.dict_depvar_input[name]):
                raise LoweringError("%s called with %d arguments, declared with %d"
                                    % (name, len(e.args), len(self.vi.dict_depvar_input[name])))
            return self.tap(name, ())
        if isinstance(e, sp.Subs):
            # Subs(Derivative(u(x,y), x), x, 0): the evaluation point lives in the data
            return self.emit(e.args[0])
        if isinstance(e, sp.Derivative):
            dvars: List[str] = []
            inner = e
            while isinstance(inner, sp.Derivative):
                for v, n in inner.variable_count:
                    dvars += [str(v)] * int(n)
                inner = inner.expr
            if isinstance(inner, sp.Subs):
                inner = inner.args[0]
                while isinstance(inner, sp.Derivative):
                    for v, n in inner.variable_count:
                        dvars += [str(v)] * int(n)
                    inner = inner.expr
            if fixed_net_of(inner) is not None:
                return self.fixed_tap(inner, dvars)
            if not (isinstance(inner, AppliedUndef) and inner.func.__name__ in self.vi.dict_depvars):
                raise LoweringError("derivative of a non-network expression survived expand_derivatives: %s" % e)
            name = inner.func.__name__
            slots = self.vi.dict_depvar_input[name]
            dirs = []
            for v in dvars:
                if v not in slots:
                    raise LoweringError("derivative of %s with respect to %s, which is not one of its inputs %s"
                                        % (name, v, slots))
                dirs.append(slots.index(v))
            return self.tap(name, tuple(dirs))
        if isinstance(e, sp.Add):
            terms = list(e.args)
            acc = None
            for t in terms:
                coeff, rest = t.as_coeff_Mul()
                if coeff == -1 and rest != 1 and acc is not None:
                    acc = self._push("sub", a=acc, b=self.emit(rest))
                else:
                    v = self.emit(t)
                    acc = v if acc is None else self._push("add", a=acc, b=v)
            return acc
        if isinstance(e, sp.Mul):
            coeff, rest = e.as_coeff_Mul()
            if coeff == -1 and rest != 1:
                return self._push("neg", a=self.emit(rest))
            num, den = [], []
            for f in e.args:
                if isinstance(f, sp.Pow) and f.exp.is_number and f.exp.is_negative:
                    den.append(sp.Pow(f.base, -f.exp))
                else:
                    num.append(f)
            acc = None
            for f in num:
                v = self.emit(f)
                acc = v if acc is None else self._push("mul", a=acc, b=v)
            if acc is None:
                acc = self.const(1.0)
            for f in den:
                acc = self._push("div", a=acc, b=self.emit(f))
            return acc
        if isinstance(e, sp.Pow):
            base, ex = e.args
            if base == sp.E:
                return self._push("exp", a=self.emit(ex))
            if ex.is_Integer:
                n = int(ex)
                if n == 2:
                    b = self.emit(base)
                    return self._push("mul", a=b, b=b)
                return self._push("powi", a=self.emit(base), imm=float(n))
            if ex == sp.Rational(1, 2):
                return self._push("sqrt", a=self.emit(base))
            if ex == sp.Rational(-1, 2):
                return self._push("div", a=self.const(1.0), b=self._push("sqrt", a=self.emit(base)))
            return self._push("pow", a=self.emit(base), b=self.emit(ex))
        unary = {sp.sin: "sin", sp.cos: "cos", sp.exp: "exp", sp.log: "log", sp.tanh: "tanh", sp.Abs: "abs"}
        for f, op in unary.items():
            if isinstance(e, f):
                return self._push(op, a=self.emit(e.args[0]))
        if isinstance(e, sp.tan):
            a = self.emit(e.args[0])
            return self._push("div", a=self._push("sin", a=a), b=self._push("cos", a=a))
        if isinstance(e, sp.cosh) or isinstance(e, sp.sinh):
            a = self.emit(e.args[0])
            ep = self._push("exp", a=a)
            en = self._push("exp", a=self._push("neg", a=a))
            s = self._push("add" if isinstance(e, sp.cosh) else "sub", a=ep, b=en)
            return self._push("mul", a=s, b=self.const(0.5))
        raise LoweringError("unsupported expression node %s in %s" % (type(e).__name__, e))

    # -- integral terms --------------------------------------------------------------------------
    def _bound_row(self, b: sp.Expr):
        """(constant, row): a number, a coordinate row, or a coordinate expression hoisted into a row of its own."""
        b = sp.sympify(b)
        if b.is_number:
            return float(b), -1
        names = {str(q) for q in b.free_symbols}
        if b.has(AppliedUndef) or b.has(sp.Derivative) or not names <= set(self.rows):
            raise LoweringError("integral bound %s: bounds are numbers or functions of the equation's coordinates %s "
                                "(bounds that depend on dependent variables are not supported)" % (b, self.rows))
        if isinstance(b, sp.Symbol):
            return 0.0, self.rows.index(str(b))
        if not self.hoist:
            raise LoweringError("integral bound %s is an expression of the coordinates; it becomes a host-evaluated row, "
                                "which device-sampled point sets do not carry" % b)
        for i, old in enumerate(self.extras):
            if old == b:
                return 0.0, len(self.rows) + i
        if len(self.rows) + len(self.extras) >= MAX_DIM:
            raise LoweringError("integral bound %s: no point row left (max %d)" % (b, MAX_DIM))
        self.extras.append(b)
        return 0.0, len(self.rows) + len(self.extras) - 1

    def integral(self, e: IntegralOp) -> int:
        """Lower one integral: the quadrature geometry, and the integrand (times the Jacobian of the reference's
        infinite-bound substitution, src/transform_inf_integral.jl) as its own IR over the node point."""
        integrand, vars_, lbs, ubs = e.args
        names = [str(v) for v in vars_]
        if len(names) > 2:
            raise LoweringError("integral over %d variables: at most 2 integrating dimensions are supported" % len(names))
        if len(set(names)) != len(names):
            raise LoweringError("integral over %s names a variable twice" % names)
        spec = IntegralSpec(owner=-1, n_dims=len(names), q=DEFAULT_QUAD_NODES)
        tsyms = [sp.Symbol("__t%d" % k, real=True) for k in range(len(names))]
        jac = sp.Integer(1)
        for k, (v, lo, hi) in enumerate(zip(names, lbs, ubs)):
            if v not in self.rows:
                raise LoweringError("integrating variable %s is not a coordinate of the equation %s" % (v, self.rows))
            lo_inf, hi_inf = lo == -sp.oo, hi == sp.oo
            if lo == sp.oo or hi == -sp.oo:
                raise LoweringError("integral over %s: empty interval [%s, %s]" % (v, lo, hi))
            if (lo_inf or hi_inf) and len(names) > 1:
                raise LoweringError("infinite bounds are supported for 1-dimensional integrals only")
            t = tsyms[k]
            kind, shift = INF_NONE, 0.0
            if lo_inf and hi_inf:                       # x = t / (1 - t^2), t in [-1 + eps, 1 - eps]
                kind, lo_t, hi_t = INF_BOTH, -1.0 + INF_EPS, 1.0 - INF_EPS
                jac = jac * (1 + t ** 2) / (1 - t ** 2) ** 2
            elif hi_inf:                                # x = a + t / (1 - t), or t / (1 - t) from a / (1 + a)
                kind, hi_t = INF_UPPER, 1.0 - INF_EPS
                if sp.sympify(lo).is_number:
                    shift, lo_t = float(lo), 0.0
                else:
                    lo_t = lo / (1 + lo)
                jac = jac / (1 - t) ** 2
            elif lo_inf:                                # x = b + t / (1 + t), t in [-1 + eps, 0]
                if not sp.sympify(hi).is_number:
                    raise LoweringError("integral over (-Inf, %s]: an upper bound that depends on the coordinates "
                                        "with an infinite lower bound is not supported" % hi)
                kind, shift, lo_t, hi_t = INF_LOWER, float(hi), -1.0 + INF_EPS, 0.0
                jac = jac / (1 + t) ** 2
            else:
                lo_t, hi_t = lo, hi
            spec.rows[k] = self.rows.index(v)
            spec.lb[k], spec.lb_row[k] = self._bound_row(lo_t)
            spec.ub[k], spec.ub_row[k] = self._bound_row(hi_t)
            spec.inf_kind[k], spec.shift[k] = kind, shift
        body = expand_derivatives(integrand)
        if not (body.has(AppliedUndef) or body.has(sp.Derivative)):
            raise LoweringError("integrand %s contains no dependent variable: nothing to train on" % integrand)
        em = _Emitter(self.vi, self.rows, self.param_index, self.param_values,
                      node_vars={str(t): k for k, t in enumerate(tsyms)}, fixed=self.fixed, const_rows=self.const_rows)
        v = em.emit(body * jac if jac != 1 else body)
        if v != len(em.prog) - 1:              # the last instruction is the integrand's value
            em.prog.append(("mul", v, em.const(1.0), 0.0))
        spec.taps, spec.prog = em.taps, em.prog
        spec.net_rows = _net_rows(self.vi, self.rows) + em.fixed_net_rows()
        for i, old in enumerate(self.integrals):
            if old == spec:
                return i
        self.integrals.append(spec)
        return len(self.integrals) - 1


    def fixed_net_rows(self) -> List[Optional[List[int]]]:
        """net_rows entries of the fixed networks (after the dependent variables'): None where this body taps none"""
        n = len(self.vi.depvars)
        return [self.fixed_rows.get(n + j) for j in range(len(self.fixed))]


def _const_rows(eq: Equation, vi: VarInfo, rows: List[str]) -> Dict[float, int]:
    """constant arguments of the equation's dependent variables and the point row each sits in: row i of a bc such as
    u(x_0, y) ~ ... holds x_0 (get_argument), so a registered function applied to x_0 reads that row"""
    out: Dict[float, int] = {}
    for app in _depvar_apps(_eq_expr(eq), vi):
        for a, v in zip(app.args, vi.dict_depvar_input[app.func.__name__]):
            if a.is_number and v in rows:
                out.setdefault(float(a), rows.index(v))
    return out


def _net_rows(vi: VarInfo, rows: List[str]) -> List[Optional[List[int]]]:
    out: List[Optional[List[int]]] = []
    for name in vi.depvars:
        ins = vi.dict_depvar_input[name]
        out.append([rows.index(v) for v in ins] if all(v in rows for v in ins) else None)
    return out


def lower_equation(eq: Equation, vi: VarInfo, param_index: Optional[Dict[str, int]] = None,
                   param_values: Optional[Dict[str, float]] = None, hoist: bool = False,
                   fixed: Optional[List[FixedNet]] = None) -> LoweredTerm:
    """Equation -> taps + residual program (``lhs - rhs``), and the IR of every integral it reads.  ``fixed``: the
    problem's fixed networks so far (registered network functions append theirs; shared by a problem's equations)."""
    rows = eq_indvars(eq, vi)
    extras: List[sp.Expr] = []
    em = _Emitter(vi, rows, param_index or {}, param_values or {}, extras=extras, hoist=hoist, fixed=fixed,
                  const_rows=_const_rows(eq, vi, rows))
    lhs = expand_derivatives(eq.lhs)
    rhs = expand_derivatives(eq.rhs)
    if hoist:
        # trainable parameters block hoisting; parameters with fixed defaults are substituted first
        subs = {sp.Symbol(k, real=True): v for k, v in (param_values or {}).items()}
        lhs = _hoist_coordinate_terms(lhs.subs(subs), set(rows), set(param_index or {}), extras, len(rows))
        rhs = _hoist_coordinate_terms(rhs.subs(subs), set(rows), set(param_index or {}), extras, len(rows))
    a = em.emit(lhs)
    b = em.emit(rhs)
    em.prog.append(("sub", a, b, 0.0))      # not CSE'd: must be the last instruction
    if not em.taps and not em.integrals:
        raise LoweringError("equation %s contains no dependent variable: nothing to train on" % (eq,))
    dim = len(rows) + len(extras)
    for spec in em.integrals:                # the quadrature variables follow the owner's rows (hoisted ones included)
        spec.prog = [("coord", dim - 1 - ins[1], 0, 0.0) if ins[0] == "coord" and ins[1] < 0 else ins
                     for ins in spec.prog]
    return LoweredTerm(em.taps, em.prog, rows, _net_rows(vi, rows) + em.fixed_net_rows(), extras, em.integrals)


def term_spec(lt: LoweredTerm, reduction: int = REDUCE_MEAN, scale: float = 1.0) -> TermSpec:
    return TermSpec(dim=lt.dim, taps=lt.taps, prog=lt.prog, net_rows=lt.net_rows,
                    reduction=reduction, scale=scale)
