"""SDEPINN host side (no GPU): logcosh's closed form against autograd, the Fokker-Planck, initial-condition and flux
terms as lowered for the engine against the float64 oracle (exact and finite-difference derivatives), the flux quirk,
the point sets and counts, the Gauss-Legendre norm against adaptive quadrature, and the refusals (reference
src/NN_SDE_weaksolve.jl)."""
import math

import numpy as np
import pytest
import sympy as sp
import torch
from scipy import integrate, stats

import neuralpde_jl_b200 as npde
from neuralpde_jl_b200 import engine as E
from neuralpde_jl_b200.lowering import lower_equation
from neuralpde_jl_b200.pinn import _ResidualSumLoss
from neuralpde_jl_b200 import sde_weak as SW
from neuralpde_jl_b200.sde_weak import SDEPINNProblem
from neuralpde_jl_b200.strategies import generate_training_sets
from neuralpde_jl_b200.symbolic import get_vars
from sdepinn_oracle import SDEPINNOracle, act, gbm_case, mlp, ou_case

torch.set_default_dtype(torch.float64)


# ---- problems (test/NNSDE2) ------------------------------------------------------------------------------------------
def ou():
    return npde.SDEProblem(lambda u, p, t: -1 * u, lambda u, p, t: 1, 0.5, (0.0, 1.0))


def gbm():
    return npde.SDEProblem(lambda u, p, t: 0.2 * u, lambda u, p, t: 0.3 * u, 1.0, (0.0, 1.0))


def chain(width=20):
    return npde.Chain(npde.Dense(2, width, "tanh"), npde.Dense(width, width, "tanh"), npde.Dense(width, 1, "logcosh"))


def make(name, **kw):
    ch = chain()
    if name == "ou":
        prob, case = ou(), ou_case()
        alg = npde.SDEPINN(chain=ch, optimalg=npde.BFGS(), x_0=-4.0, x_end=4.0, distrib=npde.Normal(0.5, 0.05), **kw)
    else:
        prob, case = gbm(), gbm_case()
        alg = npde.SDEPINN(chain=ch, optimalg=npde.BFGS(), x_0=0.0, x_end=3.0,
                           distrib=npde.LogNormal(math.log(1.0), 0.05), **kw)
    return prob, alg, case


def theta(ch, seed):
    return npde.initialparameters(np.random.default_rng(seed), ch, np.float64)


# ---- logcosh -----------------------------------------------------------------------------------------------------------
def logcosh_derivs(z):
    """the closed form the kernel evaluates (ffma_kernel.cuh logcosh_eval4), restated"""
    az = np.abs(z)
    t = np.tanh(z)
    s = 1 - t * t
    return [az + np.log1p(np.exp(-2 * az)) - math.log(2.0), t, s, -2 * t * s, s * (6 * t * t - 2)]


def test_logcosh_derivatives_against_autograd():
    z = torch.cat([torch.linspace(-40.0, 40.0, 801), torch.tensor([-1e-8, 0.0, 1e-8, 17.3, -23.9])]).requires_grad_(True)
    ds = [act("logcosh", z)]
    for _ in range(4):
        ds.append(torch.autograd.grad(ds[-1].sum(), z, create_graph=True)[0])
    for k, (mine, ref) in enumerate(zip(logcosh_derivs(z.detach().numpy()), ds)):
        np.testing.assert_allclose(mine, ref.detach().numpy(), rtol=1e-13, atol=1e-13, err_msg="derivative %d" % k)
    assert npde.Dense(2, 3, "logcosh").activation == "logcosh" and E.ACT["logcosh"] == 7


# ---- lowering against the oracle ---------------------------------------------------------------------------------------
def _run_prog(prog, rows, taps):
    val = []
    for op, a, b, imm in prog:
        f = {"const": lambda: np.full(rows.shape[1], imm), "coord": lambda: rows[a], "tap": lambda: taps[a],
             "add": lambda: val[a] + val[b], "sub": lambda: val[a] - val[b], "mul": lambda: val[a] * val[b],
             "div": lambda: val[a] / val[b], "neg": lambda: -val[a], "powi": lambda: val[a] ** int(imm),
             "pow": lambda: val[a] ** val[b]}[op]
        val.append(f())
    return val[-1]


def _taps(spec_taps, th, dims, acts, X):
    """the value and derivative taps of p̂ at the (2, m) points, by autograd"""
    x, t = torch.tensor(X[0]).requires_grad_(True), torch.tensor(X[1]).requires_grad_(True)
    out = []
    for tp in spec_taps:
        v = mlp(th, dims, acts, torch.stack([x, t]))[0]
        for d in tp.dirs:
            v = torch.autograd.grad(v.sum(), (x, t)[d], create_graph=True)[0]
        out.append(v.detach().numpy())
    return out


def lowered_terms(prob, alg, th):
    """each bc / pde term's loss: the lowered program run on autograd taps over the term's points"""
    s = SDEPINNProblem(prob, alg)
    vi = get_vars(s.pde_system.ivs, s.pde_system.dvs)
    pde_sets, bc_sets = generate_training_sets(s.pde_system.domain, s.discretization.strategy.dx, s.pde_system.eqs,
                                               s.pde_system.bcs, np.float64, vi)
    sets = pde_sets + bc_sets[:1] + [s.flux_points(xb) for xb in s.flux_at]
    out = []
    ch = alg.chain
    for eq, X in zip(s.pde_system.eqs + s.pde_system.bcs, sets):
        lt = lower_equation(eq, vi, hoist=False)
        assert lt.indvars == ["X", "T"]
        taps = _taps(lt.taps, th, ch.dims, ch.acts, X)
        out.append(np.mean(_run_prog(lt.prog, X, taps) ** 2))
    return np.array(out), s


@pytest.mark.parametrize("name", ["ou", "gbm"])
@pytest.mark.parametrize("seed", [0, 3])
def test_lowered_terms_match_oracle(name, seed):
    prob, alg, case = make(name)
    th = theta(alg.chain, seed)
    mine, s = lowered_terms(prob, alg, torch.tensor(th))
    orc = SDEPINNOracle(case, alg.chain.dims, alg.chain.acts)
    ref = np.array([float(v) for v in orc.term_losses(torch.tensor(th))])
    assert s.flux_at == orc.flux_at
    np.testing.assert_allclose(mine, ref[:-1], rtol=1e-11)


@pytest.mark.parametrize("name", ["ou", "gbm"])
def test_exact_taps_against_reference_stencils(name):
    """the deviation of exact taps from the reference's central differences, pinned at θ0: every term within 1e-7
    relative (the stencils' truncation and rounding; measured 3e-9 / 5e-9 on the PDE term)"""
    prob, alg, case = make(name)
    th = torch.tensor(theta(alg.chain, 1))
    with torch.no_grad():
        fd = SDEPINNOracle(case, alg.chain.dims, alg.chain.acts, deriv="fd").term_losses(th)
    ex = SDEPINNOracle(case, alg.chain.dims, alg.chain.acts).term_losses(th)
    rel = [abs(float(a) - float(b)) / abs(float(a)) for a, b in zip(ex, fd)]
    print("%s exact vs FD, relative per term: %s" % (name, " ".join("%.2e" % r for r in rel)))
    assert max(rel) < 1e-7


def test_flux_quirk_at_gbm_x_end():
    """the reference's flux drops p̂ ∂x(g²): the engine follows it.  At GBM's x_end = 3, ∂x(σ² x²) = 0.54 and the exact
    flux differs; at OU's boundaries (g constant) both agree"""
    th = torch.tensor(theta(chain(), 2))
    prob, alg, case = make("gbm")
    mine, s = lowered_terms(prob, alg, th)
    assert s.flux_at == [3.0]                # f = g = 0 at x_0 = 0: that flux vanishes identically
    quirk = SDEPINNOracle(case, alg.chain.dims, alg.chain.acts)
    exact = SDEPINNOracle(case, alg.chain.dims, alg.chain.acts, flux="exact")
    q, e = float(quirk.term_losses(th)[2]), float(exact.term_losses(th)[2])
    assert mine[2] == pytest.approx(q, rel=1e-11)
    assert abs(q - e) > 1e-3 * max(q, e)
    assert float(case.dg2(torch.tensor(3.0))) == pytest.approx(0.54)
    prob, alg, case = make("ou")
    a = SDEPINNOracle(case, alg.chain.dims, alg.chain.acts).term_losses(th)
    b = SDEPINNOracle(case, alg.chain.dims, alg.chain.acts, flux="exact").term_losses(th)
    assert float(a[2]) == float(b[2]) and float(a[3]) == float(b[3])


def test_flux_equation_form():
    prob, alg, _ = make("gbm")
    J = SW.flux(prob, 3.0)
    p = SW.P_HAT(SW.X_SYM, SW.T_SYM)
    dp = npde.Differential(SW.X_SYM)(p)
    assert set(sp.Add.make_args(sp.expand(J))) == {J.coeff(p) * p, J.coeff(dp) * dp}      # no p̂ ∂x(g²) part
    assert float(J.coeff(p)) == pytest.approx(0.6, rel=1e-15) and float(J.coeff(dp)) == pytest.approx(-0.405, rel=1e-15)
    assert npde.Differential(SW.X_SYM)(sp.Float(0.81)) == 0


# ---- point sets, counts and the norm term --------------------------------------------------------------------------------
def test_point_sets_and_counts():
    prob, alg, _ = make("ou")
    s = SDEPINNProblem(prob, alg)
    vi = get_vars(s.pde_system.ivs, s.pde_system.dvs)
    pde_sets, bc_sets = generate_training_sets(s.pde_system.domain, s.discretization.strategy.dx, s.pde_system.eqs,
                                               s.pde_system.bcs, np.float64, vi)
    assert pde_sets[0].shape == (2, 3381)
    np.testing.assert_array_equal(bc_sets[0], [[0.5], [0.0]])
    assert s.flux_at == [-4.0, 4.0]
    for xb in s.flux_at:
        P = s.flux_points(xb)
        assert P.shape == (2, 21) and np.all(P[0] == xb)
        np.testing.assert_allclose(P[1], np.arange(21) / 20, atol=1e-15)
    norm = s.discretization.additional_loss
    assert isinstance(norm, _ResidualSumLoss) and norm.points.shape == (2, 21) and norm.q == E.MAX_QUAD == 64
    lt = lower_equation(norm.eq, vi)
    assert [ins[0] for ins in lt.prog] == ["integral", "const", "sub"] and lt.prog[1][3] == 1.0
    assert len(lt.integrals) == 1 and lt.integrals[0].rows[0] == 0
    assert (lt.integrals[0].lb[0], lt.integrals[0].ub[0]) == (-4.0, 4.0)
    assert [ins[0] for ins in lt.integrals[0].prog] == ["tap"] and lt.integrals[0].taps[0].order == 0
    assert s.discretization.adaptive_loss.additional_loss_weights == 1.0
    g = make("gbm")
    assert SDEPINNProblem(g[0], g[1]).discretization.strategy.dx == [0.05, 0.05]


@pytest.mark.parametrize("name", ["ou", "gbm"])
def test_gauss_legendre_norm_against_adaptive_quadrature(name):
    """GL-64 against scipy's adaptive quad at θ0; G7K15 (a single HCubature rule over [x_0, x_end], one reading of the
    reference's maxiters = 10) is reported, not asserted"""
    prob, alg, case = make(name)
    th = torch.tensor(theta(alg.chain, 0))
    orc = SDEPINNOracle(case, alg.chain.dims, alg.chain.acts)
    gl = orc.integrals(th).numpy()
    for i, t in enumerate(orc.ts):
        f = lambda x: float(orc.p(th, torch.tensor([x]), torch.tensor([t]))[0])   # noqa: E731
        ref = integrate.quad(f, case.x_0, case.x_end, epsabs=1e-13, epsrel=1e-13, limit=200)[0]
        assert gl[i] == pytest.approx(ref, rel=1e-12, abs=1e-12)
        xk, wk = _kronrod15(case.x_0, case.x_end)
        g7k15 = float(sum(w * f(x) for x, w in zip(xk, wk)))
        if i in (0, len(orc.ts) - 1):
            print("%s t=%.2f GL64 %.15g G7K15 %.15g diff %.2e" % (name, t, gl[i], g7k15, g7k15 - gl[i]))


def _kronrod15(a, b):
    """the 15-point Kronrod nodes and weights on [a, b]"""
    xk = [0.991455371120812639206854697526329, 0.949107912342758524526189684047851, 0.864864423359769072789712788640926,
          0.741531185599394439863864773280788, 0.586087235467691130294144845693013, 0.405845151377397166906606412076961,
          0.207784955007898467600689403773245, 0.0]
    wk = [0.022935322010529224963732008058970, 0.063092092629978553290700663189204, 0.104790010322250183839876322541518,
          0.140653259715525918745189590510238, 0.169004726639267902826583426598550, 0.190350578064785409913256402421014,
          0.204432940075298892414161999234649, 0.209482141084727828012999174891714]
    h, c = 0.5 * (b - a), 0.5 * (a + b)
    xs = [c - h * x for x in xk[:-1]] + [c] + [c + h * x for x in reversed(xk[:-1])]
    ws = wk[:-1] + [wk[-1]] + list(reversed(wk[:-1]))
    return xs, [h * w for w in ws]


# ---- refusals -----------------------------------------------------------------------------------------------------------
def test_refusals():
    ch = chain(4)
    with pytest.raises(ValueError, match="optimalg is required"):
        npde.SDEPINN(chain=ch, x_0=-1.0, x_end=1.0)
    for mode in ("tc_bf16", "tc_split"):
        with pytest.raises(ValueError, match="SDEPINN runs on the FFMA kernel"):
            npde.SDEPINN(chain=ch, optimalg=npde.BFGS(), x_0=-1.0, x_end=1.0, mode=mode)
    vec = npde.SDEProblem(lambda u, p, t: [-u[0], -u[1]], lambda u, p, t: [1, 1], [0.5, 0.5], (0.0, 1.0))
    alg = npde.SDEPINN(chain=ch, optimalg=npde.BFGS(), x_0=-1.0, x_end=1.0)
    with pytest.raises(ValueError, match="u0 must be a number"):
        SDEPINNProblem(vec, alg)
    with pytest.raises(ValueError, match="u0 must be a number"):
        npde.solve(vec, alg)
    with pytest.raises(ValueError, match="only supports out-of-place"):
        npde.SDEProblem(lambda du, u, p, t: None, lambda u, p, t: 1, 0.5, (0.0, 1.0))
    with pytest.raises(ValueError, match="complex"):
        npde.SDEProblem(lambda u, p, t: -u, lambda u, p, t: 1, 0.5 + 1j, (0.0, 1.0))
    with pytest.raises(TypeError, match="takes no callback"):
        npde.solve(ou(), alg, callback=lambda *a: False)


def test_pdf():
    assert npde.Normal(0.5, 0.05).pdf(0.5) == pytest.approx(1 / (0.05 * math.sqrt(2 * math.pi)), rel=1e-15)
    assert npde.Normal(0.0, 2.0).pdf(1.0) == pytest.approx(0.17603266338214976, rel=1e-14)
    assert npde.LogNormal(0.0, 0.05).pdf(1.0) == pytest.approx(7.978845608028654, rel=1e-14)
    assert npde.LogNormal(0.3, 0.5).pdf(2.0) == pytest.approx(stats.lognorm(0.5, scale=math.exp(0.3)).pdf(2.0), rel=1e-14)
    assert npde.Normal(-0.2, 0.7).pdf(0.4) == pytest.approx(stats.norm(-0.2, 0.7).pdf(0.4), rel=1e-14)
    assert npde.LogNormal(0.0, 1.0).pdf(0.0) == 0.0
