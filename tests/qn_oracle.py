"""Float64 numpy restatement of the quasi-Newton methods behind ``npde.LBFGS`` / ``npde.BFGS``, for the tests.

Written from the published algorithms, independently of the engine's CUDA / C++ driver:
  - L-BFGS by the two-loop recursion (Nocedal & Wright, Algorithm 7.4) with H0 = gamma I, gamma = s'y / y'y of the
    newest pair; the engine uses the compact form of Byrd, Nocedal & Schnabel (1994) instead, so the two check each other.
  - BFGS with a dense inverse Hessian, H <- H + ((s'y + y'Hy) / (s'y)^2) s s' - (H y s' + s y'H) / s'y.
  - Hager & Zhang (2006) line search: bracket, update, secant^2, bisection; Wolfe or approximate-Wolfe termination.
  - Armijo backtracking with quadratic, then cubic interpolation (Nocedal & Wright, section 3.5).
Driven by any ``fg(theta) -> (loss, grad)``.  The driver rules are the ones the engine documents (include/pinn_b200.h):
alpha0 = 1, curvature guard s'y <= 0, reset to -g on a non-descent direction, one more evaluation when the accepted step
is not the last trial, stop at ||g||_inf <= 1e-8, an unchanged theta, a line-search failure or maxiters.
"""
import numpy as np


class LineSearchFailed(Exception):
    pass


ITER_FINITE_MAX = 53            # ceil(-log2(eps(Float64)))


def _spacing(x):
    return float(np.spacing(abs(x)))


def _up(x):
    return float(np.nextafter(x, np.inf))


def hager_zhang(phidphi, phi0, dphi0, c=1.0, delta=0.1, sigma=0.9, epsilon=1e-6, gamma=0.66, rho=5.0, psi3=0.1,
                linesearchmax=50):
    """Returns (alpha, phi(alpha)); raises LineSearchFailed.  phidphi(alpha) -> (phi, phi')."""
    if not (np.isfinite(phi0) and np.isfinite(dphi0)) or not dphi0 < 0:
        raise LineSearchFailed("not a descent direction")
    phi_lim = phi0 + epsilon * abs(phi0)
    al, va, sl = [0.0], [phi0], [dphi0]

    def finite(f, df):
        return np.isfinite(f) and np.isfinite(df)

    def ev(x):
        f, df = phidphi(x)
        if not finite(f, df):
            raise LineSearchFailed("non-finite value inside the bracket")
        al.append(x); va.append(f); sl.append(df)
        return len(al) - 1

    def wolfe(i):
        x, f, df = al[i], va[i], sl[i]
        exact = delta * dphi0 >= (f - phi0) / x and df >= sigma * dphi0
        approx = (2 * delta - 1) * dphi0 >= df >= sigma * dphi0 and f <= phi_lim
        return exact or approx

    def bisect(ia, ib):
        a, b = al[ia], al[ib]
        while b - a > _spacing(b):
            i = ev((a + b) / 2)
            if sl[i] >= 0:
                return ia, i
            if va[i] <= phi_lim:
                a, ia = al[i], i
            else:
                b, ib = al[i], i
        return ia, ib

    def update(ia, ib, ic):
        x = al[ic]
        if x < al[ia] or x > al[ib]:
            return ia, ib
        if sl[ic] >= 0:
            return ia, ic
        if va[ic] <= phi_lim:
            return ic, ib
        return bisect(ia, ic)

    def secant(a, b, da, db):
        return (a * db - b * da) / (db - da)

    def secant2(ia, ib):
        if not (sl[ia] < 0 and sl[ib] >= 0):
            raise LineSearchFailed("bad bracket")
        x = secant(al[ia], al[ib], sl[ia], sl[ib])
        if not np.isfinite(x):
            raise LineSearchFailed("non-finite secant step")
        ic = ev(x)
        if wolfe(ic):
            return True, ic, ic
        iA, iB = update(ia, ib, ic)
        a, b = al[iA], al[iB]
        x = None
        if iB == ic:
            x = secant(al[ib], al[iB], sl[ib], sl[iB])
        elif iA == ic:
            x = secant(al[ia], al[iA], sl[ia], sl[iA])
        if x is not None and a <= x <= b:
            ic = ev(x)
            if wolfe(ic):
                return True, ic, ic
            iA, iB = update(iA, iB, ic)
        return False, iA, iB

    f, df = phidphi(c)
    k = 1
    while not finite(f, df) and k < ITER_FINITE_MAX:     # a non-finite trial shrinks the step by psi3
        k += 1
        c *= psi3
        f, df = phidphi(c)
    if not finite(f, df):
        raise LineSearchFailed("no finite trial")
    al.append(c); va.append(f); sl.append(df)
    bracketed, ia, ib, it = False, 0, 1, 1
    alphamax = np.inf
    while not bracketed and it < linesearchmax:
        if df >= 0:
            ib = len(al) - 1
            for i in range(ib - 1, -1, -1):
                if va[i] <= phi_lim:
                    ia = i
                    break
            bracketed = True
        elif va[-1] > phi_lim:
            ia, ib = bisect(0, len(al) - 1)
            bracketed = True
        else:
            cold, phi_cold = c, f
            if _up(cold) >= alphamax:
                return cold, phi_cold
            c = min(c * rho, alphamax)
            f, df = phidphi(c)
            k = 1
            while not finite(f, df) and c > _up(cold) and k < ITER_FINITE_MAX:
                alphamax = c
                k += 1
                c = (cold + c) / 2
                f, df = phidphi(c)
            if not finite(f, df):
                return cold, phi_cold
            al.append(c); va.append(f); sl.append(df)
        it += 1
    while it < linesearchmax:
        a, b = al[ia], al[ib]
        if not b > a:
            raise LineSearchFailed("empty bracket")
        if b - a <= _spacing(b):
            return a, va[ia]
        ok, iA, iB = secant2(ia, ib)
        if ok:
            return al[iA], va[iA]
        A, B = al[iA], al[iB]
        if not B > A:
            raise LineSearchFailed("empty bracket")
        if B - A < gamma * (b - a):
            if _up(va[ia]) >= va[ib] and _up(va[iA]) >= va[iB]:
                return A, va[iA]
            ia, ib = iA, iB
        else:
            ic = ev((A + B) / 2)
            ia, ib = update(iA, iB, ic)
        it += 1
    raise LineSearchFailed("linesearchmax reached")


def backtracking(phi, phi0, dphi0, alpha=1.0, c_1=1e-4, rho_hi=0.5, rho_lo=0.1, iterations=1000, order=3):
    """Returns (alpha, phi(alpha)) satisfying Armijo; raises LineSearchFailed.  phi(alpha) -> value.
    A non-finite value fails the Armijo test and halves the step."""
    if not (np.isfinite(phi0) and np.isfinite(dphi0)) or not dphi0 < 0:
        raise LineSearchFailed("not a descent direction")
    a_prev, f_prev = alpha, phi0
    a, f = alpha, phi(alpha)
    it = 0
    while not f <= phi0 + c_1 * a * dphi0:
        it += 1
        if it > iterations:
            raise LineSearchFailed("iterations reached")
        if not np.isfinite(f):
            t = rho_hi * a
        elif order == 2 or it == 1 or not np.isfinite(f_prev):
            t = -(dphi0 * a * a) / (2 * (f - phi0 - dphi0 * a))       # minimiser of the quadratic model
        else:                                                          # minimiser of the cubic through both trials
            e2, e1 = f - phi0 - dphi0 * a, f_prev - phi0 - dphi0 * a_prev
            div = 1.0 / (a_prev ** 2 * a ** 2 * (a - a_prev))
            ca = (a_prev ** 2 * e2 - a ** 2 * e1) * div
            cb = (-a_prev ** 3 * e2 + a ** 3 * e1) * div
            if abs(ca) <= np.finfo(np.float64).eps:
                t = -dphi0 / (2 * cb)
            else:
                t = (-cb + np.sqrt(max(cb * cb - 3 * ca * dphi0, 0.0))) / (3 * ca)
        t = np.fmax(np.fmin(t, a * rho_hi), a * rho_lo)                # fmin / fmax ignore NaN
        a_prev, f_prev = a, f
        a = float(t)
        f = phi(a)
    return a, f


def two_loop(g, pairs, gamma):
    """H g for the L-BFGS matrix of `pairs` [(s, y), oldest first] with H0 = gamma I."""
    q = np.array(g, dtype=np.float64)
    alphas = []
    for s, y in reversed(pairs):
        a = (s @ q) / (y @ s)
        alphas.append(a)
        q -= a * y
    r = gamma * q
    for (s, y), a in zip(pairs, reversed(alphas)):
        b = (y @ r) / (y @ s)
        r += s * (a - b)
    return r


def compact_form(g, S, Y, gamma):
    """H g by the compact representation (Byrd, Nocedal & Schnabel 1994); S, Y are k x n, oldest row first."""
    SY = S @ Y.T
    R = np.triu(SY)
    D = np.diag(np.diag(SY))
    a, b = S @ g, Y @ g
    q0 = np.linalg.solve(R, a)
    p = np.linalg.solve(R.T, (D + gamma * (Y @ Y.T)) @ q0 - gamma * b)
    return gamma * g + S.T @ p - gamma * (Y.T @ q0)


class Result:
    def __init__(self):
        self.history = []       # per accepted step: (theta, loss, evaluations so far)
        self.retcode = "MaxIters"


def minimize(fg, x0, method="lbfgs", m=10, linesearch="hagerzhang", initial_stepnorm=None, maxiters=100, g_abstol=1e-8):
    """fg(theta) -> (loss, grad).  Returns a Result with x, f, g, iterations, evals, retcode and history."""
    res = Result()
    x = np.array(x0, dtype=np.float64)
    cache = {}

    def evaluate(alpha, d):
        xt = x + alpha * d
        f, g = fg(xt)
        res.evals += 1
        cache["last"] = (alpha, float(f), np.array(g, dtype=np.float64))
        return float(f), np.array(g, dtype=np.float64)

    res.evals = 0
    f, g = evaluate(0.0, np.zeros_like(x))
    n = x.size
    pairs = []
    H = None
    if method == "bfgs":
        gn = np.max(np.abs(g))
        H = np.eye(n) * (initial_stepnorm / gn if initial_stepnorm and gn > 0 else 1.0)
    res.iterations = 0
    stop = np.max(np.abs(g)) <= g_abstol
    if stop:
        res.retcode = "Success"
    while not stop and res.iterations < maxiters:
        if method == "lbfgs":
            gamma = (pairs[-1][0] @ pairs[-1][1]) / (pairs[-1][1] @ pairs[-1][1]) if pairs else 1.0
            d = -two_loop(g, pairs, gamma)
        else:
            d = -(H @ g)
        if not g @ d < 0:                              # not a descent direction: forget the curvature, step along -g
            pairs, d = [], -g
            if H is not None:
                H = np.eye(n)
        dphi0 = float(g @ d)
        try:
            if linesearch == "hagerzhang":
                def phidphi(a):
                    fa, ga = evaluate(a, d)
                    return fa, float(ga @ d)
                alpha, _ = hager_zhang(phidphi, f, dphi0)
            else:
                alpha, _ = backtracking(lambda a: evaluate(a, d)[0], f, dphi0)
        except LineSearchFailed:
            res.retcode = "Failure"
            break
        res.iterations += 1
        if alpha == 0.0:
            res.retcode = "Success"
            break
        if cache["last"][0] != alpha:
            evaluate(alpha, d)
        _, f_new, g_new = cache["last"]
        s = alpha * d
        x_new = x + s
        y = g_new - g
        changed = not np.array_equal(x_new, x)
        x, f, g = x_new, f_new, g_new
        sy = float(s @ y)
        if sy > 0:                                     # curvature guard
            if method == "lbfgs":
                pairs.append((s, y))
                if len(pairs) > m:
                    pairs.pop(0)
            else:
                Hy = H @ y
                H = H + ((sy + y @ Hy) / sy ** 2) * np.outer(s, s) - (np.outer(Hy, s) + np.outer(s, Hy)) / sy
        res.history.append((x.copy(), f, res.evals))
        if not changed or np.max(np.abs(g)) <= g_abstol:
            res.retcode = "Success"
            break
    res.x, res.f, res.g = x, f, g
    return res
