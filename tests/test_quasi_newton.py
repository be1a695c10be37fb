"""CPU checks of the quasi-Newton oracle (tests/qn_oracle.py) and of the optimizer hyper-parameter types: the line searches
meet their own termination conditions, non-finite values are handled as documented, both methods solve Rosenbrock, and
the compact L-BFGS form the engine implements equals the two-loop recursion."""
import ctypes

import numpy as np
import pytest
from scipy.optimize import rosen, rosen_der

import neuralpde_jl_b200 as npde
import qn_oracle as Q

DELTA, SIGMA, EPS = 0.1, 0.9, 1e-6


def _slice(f, df, x0, d):
    x0, d = np.asarray(x0, dtype=np.float64), np.asarray(d, dtype=np.float64)
    return (lambda a: float(f(x0 + a * d))), (lambda a: float(df(x0 + a * d) @ d))


def _cases():
    quad = (lambda x: 3.0 * (x[0] - 0.7) ** 2 + 1.0, lambda x: np.array([6.0 * (x[0] - 0.7)]), [0.0], [1.0])
    quartic = (lambda x: (x[0] - 1.0) ** 4, lambda x: np.array([4.0 * (x[0] - 1.0) ** 3]), [-1.0], [1.0])  # flat at x = 1
    x0 = np.array([-1.2, 1.0])
    rng = np.random.default_rng(3)
    out = [quad, quartic, (rosen, rosen_der, x0, -rosen_der(x0)), (rosen, rosen_der, x0, -rosen_der(x0) / 50)]
    for _ in range(4):
        x = rng.uniform(-2, 2, size=5)
        d = -rosen_der(x) * rng.uniform(0.001, 0.3) + 0.01 * rng.standard_normal(5)
        if rosen_der(x) @ d < 0:
            out.append((rosen, rosen_der, x, d))
    return out


@pytest.mark.parametrize("case", range(8))
def test_hager_zhang_step_satisfies_wolfe_or_approximate_wolfe(case):
    cases = _cases()
    if case >= len(cases):
        pytest.skip("fewer random descent slices")
    phi, dphi = _slice(*cases[case])
    p0, d0 = phi(0.0), dphi(0.0)
    alpha, pa = Q.hager_zhang(lambda a: (phi(a), dphi(a)), p0, d0)
    assert alpha > 0 and pa == phi(alpha)
    da = dphi(alpha)
    wolfe = DELTA * d0 >= (pa - p0) / alpha and da >= SIGMA * d0
    approx = (2 * DELTA - 1) * d0 >= da >= SIGMA * d0 and pa <= p0 + EPS * abs(p0)
    assert wolfe or approx, (alpha, pa, da)


@pytest.mark.parametrize("case", range(8))
def test_backtracking_step_satisfies_armijo(case):
    cases = _cases()
    if case >= len(cases):
        pytest.skip("fewer random descent slices")
    phi, dphi = _slice(*cases[case])
    p0, d0 = phi(0.0), dphi(0.0)
    alpha, pa = Q.backtracking(phi, p0, d0)
    assert 0 < alpha <= 1 and pa == phi(alpha)
    assert pa <= p0 + 1e-4 * alpha * d0


def test_non_finite_values_shrink_the_step():
    calls = []

    def phi(a):
        calls.append(a)
        return np.inf if a > 0.3 else (a - 0.2) ** 2

    dphi = lambda a: np.nan if a > 0.3 else 2 * (a - 0.2)     # noqa: E731
    p0, d0 = phi(0.0), dphi(0.0)
    calls.clear()
    alpha, _ = Q.hager_zhang(lambda a: (phi(a), dphi(a)), p0, d0)
    assert calls[0] == 1.0 and calls[1] == pytest.approx(0.1)     # psi3 = 0.1 after the non-finite trial
    assert 0 < alpha <= 0.3
    calls.clear()
    alpha, pa = Q.backtracking(phi, p0, d0)
    assert calls[:3] == [1.0, 0.5, 0.25]                        # a non-finite value fails Armijo: step halves (rho_hi)
    assert np.isfinite(pa) and pa <= p0 + 1e-4 * alpha * d0
    with pytest.raises(Q.LineSearchFailed):
        Q.hager_zhang(lambda a: (np.nan, np.nan), 1.0, -1.0)
    with pytest.raises(Q.LineSearchFailed):
        Q.hager_zhang(lambda a: (1.0, 1.0), 1.0, 1.0)           # not a descent direction


@pytest.mark.parametrize("method,ls", [("lbfgs", "hagerzhang"), ("lbfgs", "backtracking"), ("bfgs", "hagerzhang"),
                                       ("bfgs", "backtracking")])
@pytest.mark.parametrize("n", [2, 10])
def test_oracle_solves_rosenbrock(method, ls, n):
    # (-1.2, 1) in 2-D; the origin in 10-D (from (-1.2, 1, ...) the N-D function has a second stationary point near x1 = -1)
    x0 = np.array([-1.2, 1.0]) if n == 2 else np.zeros(n)
    res = Q.minimize(lambda x: (rosen(x), rosen_der(x)), x0, method=method, linesearch=ls, maxiters=5000)
    assert res.retcode == "Success", (res.retcode, res.iterations)
    assert np.max(np.abs(res.g)) <= 1e-8
    np.testing.assert_allclose(res.x, np.ones(n), atol=1e-6)
    losses = [h[1] for h in res.history]
    assert all(b <= a for a, b in zip(losses, losses[1:]))     # every accepted step decreases the loss


@pytest.mark.parametrize("k", [1, 3, 10])
def test_compact_form_equals_two_loop_recursion(k):
    rng = np.random.default_rng(k)
    n = 40
    S = rng.standard_normal((k, n))
    A = rng.standard_normal((n, n))
    A = A @ A.T + n * np.eye(n)                               # SPD: every pair has s'y > 0
    Y = S @ A + 0.01 * rng.standard_normal((k, n))
    g = rng.standard_normal(n)
    gamma = (S[-1] @ Y[-1]) / (Y[-1] @ Y[-1])
    r2 = Q.two_loop(g, list(zip(S, Y)), gamma)
    rc = Q.compact_form(g, S, Y, gamma)
    assert np.linalg.norm(rc - r2) <= 1e-12 * np.linalg.norm(r2)


def test_optimizer_types_carry_the_documented_defaults():
    hz = npde.HagerZhang()
    assert (hz.delta, hz.sigma, hz.epsilon, hz.theta, hz.gamma, hz.rho, hz.psi3, hz.linesearchmax) == \
        (0.1, 0.9, 1e-6, 0.5, 0.66, 5.0, 0.1, 50)
    bt = npde.BackTracking()
    assert (bt.c_1, bt.rho_hi, bt.rho_lo, bt.iterations, bt.order) == (1e-4, 0.5, 0.1, 1000, 3)
    assert npde.LBFGS().m == 10 and npde.LBFGS().linesearch == npde.HagerZhang()
    b = npde.BFGS()
    assert b.linesearch == npde.HagerZhang() and b.initial_stepnorm is None
    assert npde.BFGS(linesearch=npde.BackTracking()).linesearch == npde.BackTracking()
    assert npde.BFGS(initial_stepnorm=0.01).initial_stepnorm == 0.01
    assert npde.Solution(np.zeros(1), 0.0, 0).retcode == "Default"


def test_quasi_newton_abi_is_declared():
    eng = npde.engine
    for sym in ("pinn_qn_begin", "pinn_qn_iterate", "pinn_qn_theta"):
        assert sym in eng.EXPORTS
    assert eng._QnOptions.initial_stepnorm.offset == 16 and ctypes.sizeof(eng._QnOptions) == 24
