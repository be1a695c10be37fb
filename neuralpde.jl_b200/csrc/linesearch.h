// linesearch.h -- the two line searches of the quasi-Newton driver (qn.cu), with the LineSearches.jl defaults.
// Pure host C++ (no CUDA): phi(alpha) = f(theta + alpha d) and phi'(alpha) = g(theta + alpha d)' d come from a callback
// `void eval(double alpha, double& phi, double& dphi)` that may throw to abort the search.
//   HagerZhang:   W. W. Hager and H. Zhang, "A new conjugate gradient method with guaranteed descent and an efficient
//                 line search", SIAM J. Optim. 16 (2006): bracket (B1-B3), update (U0-U3), secant^2 (S1-S4), bisection.
//   BackTracking: Armijo backtracking, quadratic then cubic interpolation (Nocedal & Wright, section 3.5).
#pragma once
#include <cmath>
#include <tuple>
#include <utility>
#include <vector>

namespace pinn {

enum { LS_OK = 0, LS_FAILED = 1 };
struct LsResult { int status; double alpha; double phi; };

struct HagerZhangParams {
  double delta = 0.1, sigma = 0.9, epsilon = 1e-6, gamma = 0.66, rho = 5.0, psi3 = 0.1;
  int linesearchmax = 50;
};
struct BackTrackingParams {
  double c1 = 1e-4, rho_hi = 0.5, rho_lo = 0.1;
  int iterations = 1000, order = 3;
};

namespace ls_detail {
constexpr int kIterFiniteMax = 53;   // ceil(-log2(eps(Float64)))
inline bool finite2(double f, double df) { return std::isfinite(f) && std::isfinite(df); }
inline double spacing(double x) { x = std::fabs(x); return std::nextafter(x, INFINITY) - x; }
inline double nanmin(double a, double b) { return std::isnan(a) ? b : std::isnan(b) ? a : std::fmin(a, b); }
inline double nanmax(double a, double b) { return std::isnan(a) ? b : std::isnan(b) ? a : std::fmax(a, b); }
struct Fail {};

template <class Eval>
struct HagerZhang {
  Eval& eval;
  const HagerZhangParams& P;
  double phi_lim;
  std::vector<double> al, va, sl;   // every finite trial: step, phi, phi'

  int push(double c, double f, double df) { al.push_back(c); va.push_back(f); sl.push_back(df); return (int)al.size() - 1; }
  int eval_push(double c) {
    double f, df;
    eval(c, f, df);
    if (!finite2(f, df)) throw Fail();
    return push(c, f, df);
  }
  // Wolfe, or approximate Wolfe when phi(c) <= phi(0) + epsilon |phi(0)|
  bool wolfe(int i) const {
    const double c = al[i], f = va[i], df = sl[i], phi0 = va[0], dphi0 = sl[0];
    const bool w1 = P.delta * dphi0 >= (f - phi0) / c && df >= P.sigma * dphi0;
    const bool w2 = (2 * P.delta - 1) * dphi0 >= df && df >= P.sigma * dphi0 && f <= phi_lim;
    return w1 || w2;
  }
  static double secant(double a, double b, double da, double db) { return (a * db - b * da) / (db - da); }
  // U3: [a, b] with phi'(a) < 0, phi(a) <= phi_lim and phi'(b) < 0, phi(b) > phi_lim; bisect until phi' >= 0 at b
  std::pair<int, int> bisect(int ia, int ib) {
    double a = al[ia], b = al[ib];
    while (b - a > spacing(b)) {
      const int id = eval_push((a + b) / 2);
      if (sl[id] >= 0) return {ia, id};
      if (va[id] <= phi_lim) { a = al[id]; ia = id; }
      else { b = al[id]; ib = id; }
    }
    return {ia, ib};
  }
  // U0-U3: shrink [a, b] with the trial c
  std::pair<int, int> update(int ia, int ib, int ic) {
    const double c = al[ic];
    if (c < al[ia] || c > al[ib]) return {ia, ib};
    if (sl[ic] >= 0) return {ia, ic};
    if (va[ic] <= phi_lim) return {ic, ib};
    return bisect(ia, ic);
  }
  // S1-S4; true when a trial satisfied the termination conditions (its index in iA == iB)
  bool secant2(int ia, int ib, int& iA, int& iB) {
    if (!(sl[ia] < 0 && sl[ib] >= 0)) throw Fail();
    double c = secant(al[ia], al[ib], sl[ia], sl[ib]);
    if (!std::isfinite(c)) throw Fail();
    int ic = eval_push(c);
    if (wolfe(ic)) { iA = iB = ic; return true; }
    std::tie(iA, iB) = update(ia, ib, ic);
    const double a = al[iA], b = al[iB];
    bool again = false;
    if (iB == ic) { c = secant(al[ib], al[iB], sl[ib], sl[iB]); again = true; }
    else if (iA == ic) { c = secant(al[ia], al[iA], sl[ia], sl[iA]); again = true; }
    if (again && a <= c && c <= b) {
      ic = eval_push(c);
      if (wolfe(ic)) { iA = iB = ic; return true; }
      std::tie(iA, iB) = update(iA, iB, ic);
    }
    return false;
  }

  LsResult run(double phi0, double dphi0, double c) {
    push(0.0, phi0, dphi0);
    double f, df;
    eval(c, f, df);
    // a non-finite trial shrinks the step by psi3
    for (int k = 1; !finite2(f, df) && k < kIterFiniteMax; ++k) { c *= P.psi3; eval(c, f, df); }
    if (!finite2(f, df)) return {LS_FAILED, 0.0, phi0};
    push(c, f, df);
    // bracketing (B1-B3)
    bool bracketed = false;
    int ia = 0, ib = 1, iter = 1;
    double alphamax = INFINITY;
    while (!bracketed && iter < P.linesearchmax) {
      if (df >= 0) {                                  // upward slope: b found, a = the last trial below phi_lim
        ib = (int)al.size() - 1;
        for (int i = ib - 1; i >= 0; --i) if (va[i] <= phi_lim) { ia = i; break; }
        bracketed = true;
      } else if (va.back() > phi_lim) {               // downward slope above phi_lim: a minimum lies before c
        std::tie(ia, ib) = bisect(0, (int)al.size() - 1);
        bracketed = true;
      } else {                                        // still descending: expand by rho
        const double cold = c, phi_cold = f;
        if (std::nextafter(cold, INFINITY) >= alphamax) return {LS_OK, cold, phi_cold};
        c = std::fmin(c * P.rho, alphamax);
        eval(c, f, df);
        for (int k = 1; !finite2(f, df) && c > std::nextafter(cold, INFINITY) && k < kIterFiniteMax; ++k) {
          alphamax = c;
          c = (cold + c) / 2;
          eval(c, f, df);
        }
        if (!finite2(f, df)) return {LS_OK, cold, phi_cold};
        push(c, f, df);
      }
      ++iter;
    }
    while (iter < P.linesearchmax) {
      const double a = al[ia], b = al[ib];
      if (!(b > a)) throw Fail();
      if (b - a <= spacing(b)) return {LS_OK, a, va[ia]};
      int iA, iB;
      if (secant2(ia, ib, iA, iB)) return {LS_OK, al[iA], va[iA]};
      const double A = al[iA], B = al[iB];
      if (!(B > A)) throw Fail();
      if (B - A < P.gamma * (b - a)) {
        // the interval shrank; stop when phi is flat at both ends
        if (std::nextafter(va[ia], INFINITY) >= va[ib] && std::nextafter(va[iA], INFINITY) >= va[iB])
          return {LS_OK, A, va[iA]};
        ia = iA; ib = iB;
      } else {                                        // secant^2 converges slowly: bisect
        const int ic = eval_push((A + B) / 2);
        std::tie(ia, ib) = update(iA, iB, ic);
      }
      ++iter;
    }
    throw Fail();
  }
};
}  // namespace ls_detail

// Returns the accepted step and phi there; LS_FAILED when the search cannot find one (phi'(0) >= 0, no finite trial,
// a non-finite value inside the bracket, or linesearchmax iterations).  Starts from the trial step c.
template <class Eval>
LsResult hager_zhang(Eval& eval, double phi0, double dphi0, double c, const HagerZhangParams& P = HagerZhangParams()) {
  if (!ls_detail::finite2(phi0, dphi0) || !(dphi0 < 0)) return {LS_FAILED, 0.0, phi0};
  ls_detail::HagerZhang<Eval> s{eval, P, phi0 + P.epsilon * std::fabs(phi0), {}, {}, {}};
  try {
    return s.run(phi0, dphi0, c);
  } catch (const ls_detail::Fail&) {
    return {LS_FAILED, 0.0, phi0};
  }
}

// Armijo backtracking from the trial step alpha.  A non-finite phi fails the Armijo test and halves the step (rho_hi);
// otherwise the first reduction minimises the quadratic through phi(0), phi'(0), phi(alpha), later ones the cubic that
// also passes through the previous trial; each new step is clamped to [rho_lo alpha, rho_hi alpha].
template <class Eval>
LsResult backtracking(Eval& eval, double phi0, double dphi0, double alpha, const BackTrackingParams& P = BackTrackingParams()) {
  using namespace ls_detail;
  if (!finite2(phi0, dphi0) || !(dphi0 < 0)) return {LS_FAILED, 0.0, phi0};
  double a1 = alpha, a2 = alpha;       // previous and current trial
  double f1 = phi0, f2, df;            // phi at a1 and a2
  eval(a2, f2, df);
  for (int it = 1; !(f2 <= phi0 + P.c1 * a2 * dphi0); ++it) {
    if (it > P.iterations) return {LS_FAILED, 0.0, phi0};
    double t;
    if (!std::isfinite(f2)) {
      t = P.rho_hi * a2;
    } else if (P.order == 2 || it == 1 || !std::isfinite(f1)) {
      t = -(dphi0 * a2 * a2) / (2 * (f2 - phi0 - dphi0 * a2));
    } else {
      const double e2 = f2 - phi0 - dphi0 * a2, e1 = f1 - phi0 - dphi0 * a1;
      const double div = 1.0 / (a1 * a1 * a2 * a2 * (a2 - a1));
      const double a = (a1 * a1 * e2 - a2 * a2 * e1) * div;
      const double b = (-a1 * a1 * a1 * e2 + a2 * a2 * a2 * e1) * div;
      if (std::fabs(a) <= 2.220446049250313e-16) t = -dphi0 / (2 * b);
      else t = (-b + std::sqrt(std::fmax(b * b - 3 * a * dphi0, 0.0))) / (3 * a);
    }
    t = nanmax(nanmin(t, a2 * P.rho_hi), a2 * P.rho_lo);
    a1 = a2; f1 = f2; a2 = t;
    eval(a2, f2, df);
  }
  return {LS_OK, a2, f2};
}

}  // namespace pinn
