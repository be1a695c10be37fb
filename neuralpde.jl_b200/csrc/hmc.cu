// hmc.cu -- device-resident Hamiltonian Monte Carlo: the pinn_hmc_* entry points of include/pinn_b200.h.
//
// theta, the momentum r, the gradient g of the log density, their start-of-transition copies, M^-1 and the Welford
// window statistics are float64 on the device for both engine dtypes; every evaluation is the fused kernel (eval_step) at
// theta rounded to the engine dtype, weighted by the fixed log-likelihood weights.  The prior's value and gradient are
// added here: N(mean, std^2) on the first n - n_tail entries and, for parameter estimation, one Normal / LogNormal /
// Uniform prior per entry of the last n_tail (theta.p), plus c_j log|theta.p_j| where a chain has tail_logabs (the
// normalisation of a noise that depends on theta.p).  A tail entry outside its prior's support, or at 0 under a c_j != 0,
// has a non-finite gradient, so the trajectory stops there like at any other non-finite value.  One transition is a fixed
// launch sequence that the host never inspects:
//
//   momentum | L x (kick / drift, [samplers,] fused evaluation) | closing kick + energy partials | accept (1 block) | select
//
// With PINN_HMC_REDRAW the device samplers draw fresh points before every evaluation: draw index = the number of
// evaluations since pinn_hmc_begin (S->draws, advanced by every kick / drift launch, stopped trajectory or not).
//
// so it is captured once into a CUDA graph and replayed.  Decisions (accept, step size, window ends) are made on the
// device by the single-block accept kernel; after a non-finite value the remaining kick / drift kernels are no-ops.
// Reductions are per-chunk partials combined in a fixed order on a grid that depends on n_theta only, and random numbers
// are Philox draws keyed by (seed, transition, index, stream), so runs and graph replays are bit-identical.
// find_good_stepsize runs on the host at pinn_hmc_begin (one read-back per trial).
#include <cuda_runtime.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "engine.h"
#include "philox.cuh"
#include "reduce.cuh"

namespace pinn {
namespace {

constexpr int kHmcThreads = 256;
constexpr long long kChunk = 2048;           // elements per block of a reduction
constexpr size_t kBufBytes = 64ull << 20;    // sample rows buffered on the device between copies to the host
constexpr int kMaxRows = 4096;
// Philox streams (counter word 3)
constexpr uint32_t kTagMomentum = 0, kTagStepsizeMomentum = 1, kTagAccept = 2;
// dual averaging (AdvancedHMC's NesterovDualAveraging defaults)
constexpr double kDaGamma = 0.05, kDaT0 = 10.0, kDaKappa = 0.75;
enum { kInit = 0, kTrial = 1, kTransition = 2 };

// device scalars of the chain
struct HmcScal {
  double eps;                    // step size of the next transition
  double trial_eps;              // step size of a find_good_stepsize trial (0 for the evaluation at theta0)
  double logp;                   // l(theta)
  double dh;                     // find_good_stepsize: H0 - H1 of the last trial
  double mu, m, x_bar, h_bar;    // dual-averaging state
  long long t;                   // transitions done
  long long row_base;            // the sample-buffer row of transition t is t - row_base
  long long row;                 // row of the current transition
  long long win_n;               // Welford count of the current window
  long long win_n_cur;           // ... after the current transition's push (read by the select kernel)
  long long win_size, next_split;   // Stan windows: size of the current window, its last transition (-1: none left)
  unsigned long long draws;      // evaluations since begin: the draw index of the next sampler launch
  int flag;                      // non-finite value in the current trajectory
  int accept, push, win_end;     // the current transition's decision, Welford push and window end
};

struct HmcArgs {
  long long n;
  int chunks;
  double *theta, *r, *g, *theta0, *g0, *minv, *wmean, *wm2;
  double* part;                  // [3][chunks]: K at the start, K at the end, sum (theta - mu)^2 at the end
  void* theta_r;                 // engine dtype: what the fused kernel evaluates
  const void* g_r;               // engine dtype: gradient of the weighted physics log-likelihood
  const void* total;             // engine dtype: its value (without ll_const)
  HmcScal* S;
  double *samples, *stats;       // [rows][n], [rows][PINN_HMC_N_STATS]
  double prior_mean, inv_var;    // prior N(mean, 1 / inv_var) of theta[0, n - n_tail)
  int n_tail;                    // tail[j] is the prior of theta[n - n_tail + j]
  pinn_hmc_prior tail[PINN_MAX_PARAMS];
  double tail_c[PINN_MAX_PARAMS];   // c_j of the c_j log|theta.p_j| terms (0: none)
  double lp_const;               // ll_const + the prior's normalisation
  double delta;                  // target acceptance
  int adapt, diag, n_adapts;
  long long window_start, window_end;
  unsigned long long seed;
};

__device__ __forceinline__ double u53(uint32_t hi, uint32_t lo) {
  return (double)((((unsigned long long)hi << 32) | lo) >> 11) * (1.0 / 9007199254740992.0);
}

// standard normal i of transition t in stream tag: Box-Muller on one Philox draw per pair (2j, 2j + 1)
__device__ __forceinline__ double normal_draw(unsigned long long seed, long long t, uint32_t tag, long long i) {
  const unsigned long long j = (unsigned long long)i >> 1;
  uint32_t c[4] = {(uint32_t)j, (uint32_t)(unsigned long long)t, (uint32_t)((unsigned long long)t >> 32), tag};
  philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
  const double u1 = u53(c[0], c[1]) + 1.0 / 9007199254740992.0;   // (0, 1]
  const double u2 = u53(c[2], c[3]);
  const double rad = sqrt(-2.0 * log(u1));
  double s, co;
  sincospi(2.0 * u2, &s, &co);
  return (i & 1) ? rad * s : rad * co;
}

// Distributions.jl's insupport: LogNormal x > 0, Uniform a <= x <= b
__device__ __forceinline__ bool tail_insupport(const pinn_hmc_prior& p, double x) {
  if (p.kind == PINN_HMC_PRIOR_LOGNORMAL) return x > 0.0;
  if (p.kind == PINN_HMC_PRIOR_UNIFORM) return x >= p.a && x <= p.b;
  return true;
}

// d/dx logpdf: Normal -(x - mu) / s^2, LogNormal -(1 + (log x - mu) / s^2) / x, Uniform 0; NaN outside the support
__device__ __forceinline__ double tail_grad(const pinn_hmc_prior& p, double x) {
  if (!tail_insupport(p, x)) return NAN;
  if (p.kind == PINN_HMC_PRIOR_NORMAL) return -(x - p.a) / (p.b * p.b);
  if (p.kind == PINN_HMC_PRIOR_LOGNORMAL) return -(1.0 + (log(x) - p.a) / (p.b * p.b)) / x;
  return 0.0;
}

// logpdf as Distributions.jl writes it; -Inf outside the support
__device__ __forceinline__ double tail_logpdf(const pinn_hmc_prior& p, double x) {
  if (!tail_insupport(p, x)) return -INFINITY;
  if (p.kind == PINN_HMC_PRIOR_UNIFORM) return -log(p.b - p.a);
  const double lx = p.kind == PINN_HMC_PRIOR_LOGNORMAL ? log(x) : x;
  const double z = (lx - p.a) / p.b;
  const double v = -(z * z + log(2.0 * M_PI)) / 2.0 - log(p.b);
  return p.kind == PINN_HMC_PRIOR_LOGNORMAL ? v - lx : v;
}

__device__ __forceinline__ double prior_grad(const HmcArgs& a, double th) { return -(th - a.prior_mean) * a.inv_var; }

// gradient of l at entry i: the physics part g_phys plus the prior's (network entries: the n_tail = 0 arithmetic)
__device__ __forceinline__ double grad_at(const HmcArgs& a, long long i, double th, double g_phys) {
  const long long j = i - (a.n - a.n_tail);
  if (j < 0) return g_phys + prior_grad(a, th);
  if (a.tail_c[j] != 0.0) return g_phys + (tail_grad(a.tail[j], th) + a.tail_c[j] / th);
  return g_phys + tail_grad(a.tail[j], th);
}

// start of a transition (restore = false: theta0 = theta, g0 = g) or of a find_good_stepsize trial (restore = true:
// theta = theta0, g = g0); r = z ./ sqrt(M^-1) and the chunk's partial of r' M^-1 r
__global__ void __launch_bounds__(kHmcThreads) hmc_momentum_kernel(HmcArgs a, bool restore, uint32_t tag) {
  const long long lo = (long long)blockIdx.x * kChunk, hi = min(a.n, lo + kChunk);
  const long long t = a.S->t;
  double acc = 0.0;
  for (long long i = lo + threadIdx.x; i < hi; i += kHmcThreads) {
    if (restore) { a.theta[i] = a.theta0[i]; a.g[i] = a.g0[i]; }
    else { a.theta0[i] = a.theta[i]; a.g0[i] = a.g[i]; }
    const double mi = a.minv[i];
    const double ri = normal_draw(a.seed, t, tag, i) / sqrt(mi);
    a.r[i] = ri;
    acc += mi * ri * ri;
  }
  acc = block_reduce<kHmcThreads, false>(acc);
  if (threadIdx.x == 0) {
    a.part[blockIdx.x] = acc;
    if (blockIdx.x == 0) a.S->flag = 0;
  }
}

// leapfrog step: (first ? nothing : g = gradient of the last evaluation, closing half kick), opening half kick, drift;
// theta_r = (real)theta for the next evaluation.  A no-op once the trajectory met a non-finite value.
template <typename real>
__global__ void __launch_bounds__(kHmcThreads) hmc_kick_drift_kernel(HmcArgs a, bool first, const double* eps) {
  const long long i = (long long)blockIdx.x * kHmcThreads + threadIdx.x;
  if (i == 0) a.S->draws += 1;   // the evaluation after this launch, whether or not the trajectory has stopped
  if (i >= a.n || a.S->flag) return;
  const double e = *eps, h = 0.5 * e;
  double th = a.theta[i], ri = a.r[i], gi;
  if (first) {
    gi = a.g[i];
  } else {
    gi = grad_at(a, i, th, (double)((const real*)a.g_r)[i]);
    a.g[i] = gi;
    if (!isfinite(gi) || (i == 0 && !isfinite((double)*(const real*)a.total))) { a.S->flag = 1; return; }
    ri += h * gi;
  }
  ri += h * gi;
  th += e * (a.minv[i] * ri);
  a.r[i] = ri;
  a.theta[i] = th;
  ((real*)a.theta_r)[i] = (real)th;
}

// after the last evaluation: g, the closing half kick, and the chunk's partials of r' M^-1 r and |theta - mu|^2 (the
// latter over the Normal prior's entries only)
template <typename real>
__global__ void __launch_bounds__(kHmcThreads) hmc_close_kernel(HmcArgs a, const double* eps) {
  const long long lo = (long long)blockIdx.x * kChunk, hi = min(a.n, lo + kChunk);
  const long long n_net = a.n - a.n_tail;
  const double h = 0.5 * *eps;
  const bool live = !a.S->flag;
  bool bad = blockIdx.x == 0 && threadIdx.x == 0 && !isfinite((double)*(const real*)a.total);
  double k = 0.0, p = 0.0;
  for (long long i = lo + threadIdx.x; i < hi; i += kHmcThreads) {
    const double th = a.theta[i];
    const double gi = grad_at(a, i, th, (double)((const real*)a.g_r)[i]);
    a.g[i] = gi;
    double ri = a.r[i];
    if (live) { ri += h * gi; a.r[i] = ri; }
    bad |= !isfinite(gi) || !isfinite(ri) || !isfinite(th);
    const double mi = a.minv[i];
    k += mi * ri * ri;
    if (i < n_net) {
      const double d = th - a.prior_mean;
      p += d * d;
    }
  }
  if (bad) a.S->flag = 1;
  k = block_reduce<kHmcThreads, false>(k);
  __syncthreads();
  p = block_reduce<kHmcThreads, false>(p);
  if (threadIdx.x == 0) {
    a.part[a.chunks + blockIdx.x] = k;
    a.part[2 * a.chunks + blockIdx.x] = p;
  }
}

__device__ double sum_chunks(const double* part, int chunks) {
  double v = 0.0;
  for (int c = threadIdx.x; c < chunks; c += kHmcThreads) v += part[c];
  v = block_reduce<kHmcThreads, false>(v);
  __syncthreads();
  return v;
}

// one block: the energies, then (kTransition) the Metropolis decision, the statistics row, dual averaging and the Stan
// window bookkeeping; kInit stores l(theta), kTrial the energy difference of a find_good_stepsize trial
template <typename real>
__global__ void __launch_bounds__(kHmcThreads) hmc_accept_kernel(HmcArgs a, int mode) {
  const double k0 = 0.5 * sum_chunks(a.part, a.chunks);
  const double k1 = 0.5 * sum_chunks(a.part + a.chunks, a.chunks);
  const double pp = sum_chunks(a.part + 2 * a.chunks, a.chunks);
  if (threadIdx.x) return;
  HmcScal& S = *a.S;
  double logp1 = (double)*(const real*)a.total + a.lp_const - 0.5 * pp * a.inv_var;
  for (int j = 0; j < a.n_tail; ++j) {
    const double x = a.theta[a.n - a.n_tail + j];
    logp1 += tail_logpdf(a.tail[j], x);
    if (a.tail_c[j] != 0.0) logp1 += a.tail_c[j] * log(fabs(x));
  }
  if (mode == kInit) { S.logp = logp1; return; }
  const double h0 = -S.logp + k0;
  double h1 = -logp1 + k1;
  const bool numerr = S.flag || !isfinite(h1);
  if (numerr) h1 = INFINITY;     // AdvancedHMC maps a non-finite phase point to H = +Inf
  if (mode == kTrial) { S.dh = h0 - h1; return; }
  const long long t = S.t;
  const double alpha = numerr ? 0.0 : fmin(1.0, exp(h0 - h1));
  uint32_t c[4] = {0u, (uint32_t)(unsigned long long)t, (uint32_t)((unsigned long long)t >> 32), kTagAccept};
  philox4x32_10(c, (uint32_t)a.seed, (uint32_t)(a.seed >> 32));
  const bool accept = u53(c[0], c[1]) < alpha;
  const long long i = t + 1;     // 1-based transition index, as the adaptor counts
  const bool adapting = a.adapt && i <= a.n_adapts;
  const long long row = t - S.row_base;
  double* st = a.stats + row * PINN_HMC_N_STATS;
  st[PINN_HMC_STAT_STEP_SIZE] = S.eps;
  st[PINN_HMC_STAT_ACCEPTANCE_RATE] = alpha;
  st[PINN_HMC_STAT_IS_ACCEPT] = accept ? 1.0 : 0.0;
  st[PINN_HMC_STAT_LOG_DENSITY] = accept ? logp1 : S.logp;
  st[PINN_HMC_STAT_HAMILTONIAN_ENERGY] = accept ? h1 : h0;
  st[PINN_HMC_STAT_HAMILTONIAN_ENERGY_ERROR] = accept ? h1 - h0 : 0.0;
  st[PINN_HMC_STAT_NUMERICAL_ERROR] = numerr ? 1.0 : 0.0;
  st[PINN_HMC_STAT_IS_ADAPT] = adapting ? 1.0 : 0.0;
  if (accept) S.logp = logp1;
  S.accept = accept;
  S.push = 0;
  S.win_end = 0;
  if (adapting) {
    // Nesterov dual averaging (Hoffman & Gelman 2014, as AdvancedHMC): a non-finite step size keeps the previous state
    const double m = S.m + 1.0;
    const double eta_h = 1.0 / (m + kDaT0);
    const double h_bar = (1.0 - eta_h) * S.h_bar + eta_h * (a.delta - alpha);
    const double x = S.mu - h_bar * sqrt(m) / kDaGamma;
    const double eta_x = pow(m, -kDaKappa);
    const double x_bar = (1.0 - eta_x) * S.x_bar + eta_x * x;
    const double eps = exp(x);
    if (isfinite(eps)) { S.m = m; S.h_bar = h_bar; S.x_bar = x_bar; S.eps = eps; }
    // Stan windows: theta joins the window's Welford estimate; at a window end M^-1 is set (select kernel) and both
    // the estimate and the dual averaging restart
    if (i >= a.window_start && i <= a.window_end) {
      S.win_n += 1;
      S.push = 1;
    }
    S.win_n_cur = S.win_n;
    if (i == S.next_split) {
      S.win_end = 1;
      S.win_n = 0;
      S.mu = log(10.0 * S.eps);
      S.m = 0.0; S.x_bar = 0.0; S.h_bar = 0.0;
      if (S.next_split >= a.window_end) {
        S.next_split = -1;
      } else {
        S.win_size *= 2;
        long long nxt = S.next_split + S.win_size;
        if (nxt + 2 * S.win_size > a.window_end) nxt = a.window_end;   // the last window runs to the term buffer
        S.next_split = nxt;
      }
    }
    if (i == a.n_adapts) S.eps = exp(S.x_bar);
  }
  S.row = row;
  S.t = t + 1;
}

// end of a transition: the rejected proposal restores theta0 / g0; the sample row; the Welford push and, at a window
// end, M^-1 = the regularised window variance (Stan: n / ((n + 5)(n - 1)) M2 + 1e-3 * 5 / (n + 5))
__global__ void __launch_bounds__(kHmcThreads) hmc_select_kernel(HmcArgs a) {
  const long long i = (long long)blockIdx.x * kHmcThreads + threadIdx.x;
  if (i >= a.n) return;
  const HmcScal& S = *a.S;
  double th = a.theta[i];
  if (!S.accept) { th = a.theta0[i]; a.theta[i] = th; a.g[i] = a.g0[i]; }
  a.samples[S.row * a.n + i] = th;
  if (!a.diag) return;
  if (S.push) {
    const double nn = (double)S.win_n_cur;
    const double d = th - a.wmean[i];
    const double mu = a.wmean[i] + d / nn;
    a.wmean[i] = mu;
    a.wm2[i] += d * (th - mu);
  }
  if (S.win_end) {
    const double nn = (double)S.win_n_cur;
    if (nn >= 2.0) a.minv[i] = (nn / ((nn + 5.0) * (nn - 1.0))) * a.wm2[i] + 1e-3 * (5.0 / (nn + 5.0));
    a.wmean[i] = 0.0;
    a.wm2[i] = 0.0;
  }
}

__global__ void hmc_fill_kernel(double* p, long long n, double v) {
  const long long i = (long long)blockIdx.x * kHmcThreads + threadIdx.x;
  if (i < n) p[i] = v;
}

template <typename real>
__global__ void hmc_narrow_kernel(const double* in, long long n, real* out) {
  const long long i = (long long)blockIdx.x * kHmcThreads + threadIdx.x;
  if (i < n) out[i] = (real)in[i];
}

}  // namespace

struct HmcState {
  pinn_hmc_options opt = {};
  double w[PINN_MAX_TERMS] = {};
  HmcArgs a = {};
  int rows = 1;                  // capacity of the sample / statistics buffers
  long long t = 0;               // transitions done (host copy)
  cudaGraphExec_t graph = nullptr;
  unsigned long long graph_key = 0;
  bool redraw = false;           // PINN_HMC_REDRAW: the device samplers draw before every evaluation
};

void hmc_release(pinn_engine* e) {
  HmcState* s = e->hmc;
  if (!s) return;
  if (s->graph) cudaGraphExecDestroy(s->graph);
  HmcArgs& a = s->a;
  double* dp[] = {a.theta, a.r, a.g, a.theta0, a.g0, a.minv, a.wmean, a.wm2, a.part, a.samples, a.stats};
  for (double* p : dp) if (p) cudaFree(p);
  void* vp[] = {a.theta_r, (void*)a.g_r, a.S};
  for (void* p : vp) if (p) cudaFree(p);
  delete s;
  e->hmc = nullptr;
}

namespace {

unsigned blocks_of(long long n) { return (unsigned)((n + kHmcThreads - 1) / kHmcThreads); }

template <typename T>
int alloc(T** p, size_t count, pinn_engine* e) { return dev_alloc((void**)p, count * sizeof(T), e); }

// Stan's windowed adaptation schedule (AdvancedHMC StanHMCAdaptor, Stan's windowed_adaptation): buffers 75 / 25 / 50,
// or 15 % / the rest / 10 % of n_adapts when n_adapts < 150
void stan_windows(long long n_adapts, long long* start, long long* end, long long* size) {
  long long init = 75, term = 50, win = 25;
  if (init + win + term > n_adapts) {
    init = (long long)floor(0.15 * (double)n_adapts);
    term = (long long)floor(0.1 * (double)n_adapts);
    win = n_adapts - init - term;
  }
  *start = init + 1;
  *end = n_adapts - term;
  *size = win;
}

int launch_check(pinn_engine* e, int count) {
  CUDA_TRY(cudaGetLastError());
  e->launches += count;
  return 0;
}

// evaluate the weighted physics log-likelihood and its gradient at theta_r (redraw: on fresh points of draw S->draws)
int evaluate(pinn_engine* e, HmcState* s, cudaStream_t st) {
  const HmcArgs& a = s->a;
  if (s->redraw)
    for (int t = 0; t < e->n_terms; ++t)
      if (e->term[t].sampler_on && draw_term(e, t, 0, &a.S->draws, st)) return 1;
  char* out = (char*)a.total - (size_t)e->n_terms * e->es;
  return eval_step(e, a.theta_r, s->w, (void*)a.g_r, out, (void*)a.total, false, st);
}

int momentum(pinn_engine* e, HmcState* s, bool restore, uint32_t tag, cudaStream_t st) {
  hmc_momentum_kernel<<<s->a.chunks, kHmcThreads, 0, st>>>(s->a, restore, tag);
  return launch_check(e, 1);
}

// leapfrog trajectory of n_steps from the current (theta, r, g), then the closing kick and the energy partials
int trajectory(pinn_engine* e, HmcState* s, int n_steps, const double* eps, cudaStream_t st) {
  const bool f64 = e->dtype == PINN_F64;
  const long long n = e->n_theta;
  for (int j = 0; j < n_steps; ++j) {
    if (f64) hmc_kick_drift_kernel<double><<<blocks_of(n), kHmcThreads, 0, st>>>(s->a, j == 0, eps);
    else hmc_kick_drift_kernel<float><<<blocks_of(n), kHmcThreads, 0, st>>>(s->a, j == 0, eps);
    if (launch_check(e, 1) || evaluate(e, s, st)) return 1;
  }
  if (f64) hmc_close_kernel<double><<<s->a.chunks, kHmcThreads, 0, st>>>(s->a, eps);
  else hmc_close_kernel<float><<<s->a.chunks, kHmcThreads, 0, st>>>(s->a, eps);
  return launch_check(e, 1);
}

int accept_launch(pinn_engine* e, HmcState* s, int mode, cudaStream_t st) {
  if (e->dtype == PINN_F64) hmc_accept_kernel<double><<<1, kHmcThreads, 0, st>>>(s->a, mode);
  else hmc_accept_kernel<float><<<1, kHmcThreads, 0, st>>>(s->a, mode);
  return launch_check(e, 1);
}

// one transition: the fixed launch sequence of the file comment
int enqueue_transition(pinn_engine* e, HmcState* s, cudaStream_t st) {
  if (momentum(e, s, false, kTagMomentum, st)) return 1;
  if (trajectory(e, s, s->opt.n_leapfrog, &s->a.S->eps, st)) return 1;
  if (accept_launch(e, s, kTransition, st)) return 1;
  hmc_select_kernel<<<blocks_of(e->n_theta), kHmcThreads, 0, st>>>(s->a);
  return launch_check(e, 1);
}

int read_scal(pinn_engine* e, HmcState* s, HmcScal* h) {
  CUDA_TRY(cudaMemcpyAsync(h, s->a.S, sizeof(HmcScal), cudaMemcpyDeviceToHost, e->own_stream));
  CUDA_TRY(cudaStreamSynchronize(e->own_stream));
  return 0;
}

// H0 - H1 of one leapfrog step of size eps from (theta0, the find_good_stepsize momentum)
int stepsize_trial(pinn_engine* e, HmcState* s, bool first, double eps, double* dh) {
  cudaStream_t st = e->own_stream;
  HmcScal* S = s->a.S;
  CUDA_TRY(cudaMemcpyAsync(&S->trial_eps, &eps, sizeof(double), cudaMemcpyHostToDevice, st));
  if (momentum(e, s, !first, kTagStepsizeMomentum, st) || trajectory(e, s, 1, &S->trial_eps, st) ||
      accept_launch(e, s, kTrial, st))
    return 1;
  HmcScal h;
  if (read_scal(e, s, &h)) return 1;
  *dh = h.dh;
  return 0;
}

// AdvancedHMC's find_good_stepsize: one momentum draw, direction from the first trial, doubling / halving until the
// acceptance ratio crosses 1/2, then bisection until exp(dH) lies in [0.25, 0.75] (100 trials at most each).  As there,
// each crossing trial evaluates the current eps and moves to the candidate eps' afterwards.
int find_good_stepsize(pinn_engine* e, HmcState* s, double* out) {
  const double a_min = 0.25, a_cross = 0.5, a_max = 0.75, d = 2.0;
  double eps = 0.1, eps1 = 0.1, dh;
  if (stepsize_trial(e, s, true, eps, &dh)) return 1;
  const int direction = dh > log(a_cross) ? 1 : -1;
  for (int it = 0; it < 100; ++it) {
    eps1 = direction == 1 ? d * eps : eps / d;
    if (stepsize_trial(e, s, false, eps, &dh)) return 1;
    if (direction == 1 && !(dh > log(a_cross))) break;
    if (direction == -1 && !(dh < log(a_cross))) break;
    eps = eps1;
  }
  if (eps > eps1) std::swap(eps, eps1);
  for (int it = 0; it < 100; ++it) {
    const double mid = 0.5 * (eps + eps1);
    if (stepsize_trial(e, s, false, mid, &dh)) return 1;
    if (exp(dh) > a_max) eps = mid;
    else if (exp(dh) < a_min) eps1 = mid;
    else { eps = mid; break; }
  }
  // the chain starts from theta0 and its gradient
  if (momentum(e, s, true, kTagStepsizeMomentum, e->own_stream)) return 1;
  *out = eps;
  return 0;
}

unsigned long long fnv1a(const void* p, size_t n, unsigned long long h) {
  const unsigned char* b = (const unsigned char*)p;
  for (size_t i = 0; i < n; ++i) { h ^= b[i]; h *= 1099511628211ull; }
  return h;
}

long long launches_per_transition(const pinn_engine* e, const HmcState* s) {
  long long per_step = 2 + (e->plan.wide ? 1 : 0);
  if (s->redraw)
    for (int t = 0; t < e->n_terms; ++t) per_step += e->term[t].sampler_on ? 1 : 0;
  return 4 + (long long)s->opt.n_leapfrog * per_step;
}

}  // namespace
}  // namespace pinn

using namespace pinn;

static int hmc_start(pinn_handle e, const double* host_theta0, const pinn_hmc_options* opts, const double* host_weights,
                     double ll_const, const pinn_hmc_prior* tail, int32_t n_tail, const double* tail_logabs,
                     uint32_t flags, double* step_size_out) {
  if (!host_theta0 || !opts) return fail("pinn_hmc_begin: null theta / options");
  if (n_tail < 0 || n_tail > PINN_MAX_PARAMS || (long long)n_tail >= e->n_theta)
    return fail("pinn_hmc_begin: n_tail = %d must lie in [0, min(%d, n_theta = %lld - 1)]", n_tail, PINN_MAX_PARAMS,
                (long long)e->n_theta);
  if (n_tail > 0 && !tail) return fail("pinn_hmc_begin: null tail priors with n_tail = %d", n_tail);
  for (int j = 0; j < n_tail; ++j) {
    const pinn_hmc_prior& p = tail[j];
    if (p.kind != PINN_HMC_PRIOR_NORMAL && p.kind != PINN_HMC_PRIOR_LOGNORMAL && p.kind != PINN_HMC_PRIOR_UNIFORM)
      return fail("pinn_hmc_begin: tail prior %d has unknown kind %d", j, p.kind);
    if (!isfinite(p.a) || !isfinite(p.b))
      return fail("pinn_hmc_begin: tail prior %d has a non-finite parameter (%g, %g)", j, p.a, p.b);
    if (p.kind == PINN_HMC_PRIOR_UNIFORM && !(p.a < p.b))
      return fail("pinn_hmc_begin: tail prior %d is Uniform(%g, %g): needs a < b", j, p.a, p.b);
    if (p.kind != PINN_HMC_PRIOR_UNIFORM && !(p.b > 0.0))
      return fail("pinn_hmc_begin: tail prior %d has sigma %g: must be positive", j, p.b);
  }
  if (tail_logabs && n_tail == 0) return fail("pinn_hmc_begin: tail_logabs needs n_tail >= 1");
  for (int j = 0; tail_logabs && j < n_tail; ++j)
    if (!isfinite(tail_logabs[j])) return fail("pinn_hmc_begin: tail_logabs[%d] = %g is not finite", j, tail_logabs[j]);
  if (flags & ~(uint32_t)PINN_HMC_REDRAW) return fail("pinn_hmc_begin: unknown flags 0x%x", flags);
  if (e->nranks > 1) return fail("pinn_hmc_begin: the sampler runs one chain on one GPU (communicator with %d ranks)", e->nranks);
  const bool redraw = (flags & PINN_HMC_REDRAW) != 0;
  if (any_sampler(e) && !redraw)
    return fail("pinn_hmc_begin: HMC needs a fixed log density; a device sampler redraws the points (use fixed point sets)");
  if (opts->n_leapfrog < 1) return fail("pinn_hmc_begin: n_leapfrog = %d must be >= 1", opts->n_leapfrog);
  if (opts->adaptor != PINN_HMC_ADAPT_NONE && opts->adaptor != PINN_HMC_ADAPT_STAN)
    return fail("pinn_hmc_begin: unknown adaptor %d", opts->adaptor);
  if (opts->metric != PINN_HMC_METRIC_UNIT && opts->metric != PINN_HMC_METRIC_DIAG)
    return fail("pinn_hmc_begin: unknown metric %d", opts->metric);
  if (opts->n_adapts < 0) return fail("pinn_hmc_begin: n_adapts = %d must be >= 0", opts->n_adapts);
  if (!(opts->target_accept > 0.0 && opts->target_accept < 1.0))
    return fail("pinn_hmc_begin: target acceptance %g outside (0, 1)", opts->target_accept);
  if (!(opts->prior_std > 0.0) || !isfinite(opts->prior_std) || !isfinite(opts->prior_mean))
    return fail("pinn_hmc_begin: prior std %g must be positive and finite (mean %g)", opts->prior_std, opts->prior_mean);
  if (!isfinite(opts->step_size) || !isfinite(ll_const)) return fail("pinn_hmc_begin: non-finite step size / ll_const");
  if (e->total_tiles <= 0) return fail("pinn_hmc_begin: no collocation points");
  CUDA_TRY(cudaSetDevice(e->device));
  hmc_release(e);
  HmcState* s = new HmcState();
  e->hmc = s;
  s->opt = *opts;
  s->redraw = redraw;
  for (int k = 0; k < e->n_terms; ++k) s->w[k] = host_weights ? host_weights[k] : 1.0;
  const long long n = e->n_theta;
  HmcArgs& a = s->a;
  a.n = n;
  a.chunks = (int)std::max<long long>(1, (n + kChunk - 1) / kChunk);
  s->rows = (int)std::max<long long>(1, std::min<long long>(kMaxRows, (long long)(kBufBytes / (8 * (size_t)n))));
  void* out = nullptr;
  int rc = alloc(&a.theta, n, e) || alloc(&a.r, n, e) || alloc(&a.g, n, e) || alloc(&a.theta0, n, e) ||
           alloc(&a.g0, n, e) || alloc(&a.minv, n, e) || alloc(&a.wmean, n, e) || alloc(&a.wm2, n, e) ||
           alloc(&a.part, 3 * (size_t)a.chunks, e) || alloc(&a.samples, (size_t)s->rows * n, e) ||
           alloc(&a.stats, (size_t)s->rows * PINN_HMC_N_STATS, e) || dev_alloc(&a.theta_r, n * e->es, e) ||
           dev_alloc(&out, (size_t)n * e->es + (PINN_MAX_TERMS + 1) * e->es, e) || alloc(&a.S, 1, e);
  if (rc) { a.g_r = out; return 1; }
  a.g_r = out;                                            // [gradient | term losses | total]
  a.total = (char*)out + (size_t)n * e->es + (size_t)e->n_terms * e->es;
  a.prior_mean = opts->prior_mean;
  a.inv_var = 1.0 / (opts->prior_std * opts->prior_std);
  a.n_tail = n_tail;
  for (int j = 0; j < n_tail; ++j) {
    a.tail[j] = tail[j];
    a.tail_c[j] = tail_logabs ? tail_logabs[j] : 0.0;
  }
  const long long n_net = n - n_tail;
  a.lp_const = ll_const - 0.5 * (double)n_net * log(2.0 * M_PI) - (double)n_net * log(opts->prior_std);
  a.delta = opts->target_accept;
  a.adapt = opts->adaptor == PINN_HMC_ADAPT_STAN;
  a.diag = opts->metric == PINN_HMC_METRIC_DIAG;
  a.n_adapts = opts->n_adapts;
  long long wsize = 0;
  stan_windows(opts->n_adapts, &a.window_start, &a.window_end, &wsize);
  a.seed = opts->seed;

  cudaStream_t st = e->own_stream;
  HmcScal h = {};
  CUDA_TRY(cudaMemcpyAsync(a.S, &h, sizeof h, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(a.theta, host_theta0, n * sizeof(double), cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemsetAsync(a.r, 0, n * sizeof(double), st));
  CUDA_TRY(cudaMemsetAsync(a.wmean, 0, n * sizeof(double), st));
  CUDA_TRY(cudaMemsetAsync(a.wm2, 0, n * sizeof(double), st));
  hmc_fill_kernel<<<blocks_of(n), kHmcThreads, 0, st>>>(a.minv, n, 1.0);
  if (e->dtype == PINN_F64) hmc_narrow_kernel<double><<<blocks_of(n), kHmcThreads, 0, st>>>(a.theta, n, (double*)a.theta_r);
  else hmc_narrow_kernel<float><<<blocks_of(n), kHmcThreads, 0, st>>>(a.theta, n, (float*)a.theta_r);
  if (launch_check(e, 2) || evaluate(e, s, st)) return 1;
  // l(theta0) and g(theta0): the closing kernel with step 0 (r = 0), then the accept kernel's initial mode
  if (e->dtype == PINN_F64) hmc_close_kernel<double><<<a.chunks, kHmcThreads, 0, st>>>(a, &a.S->trial_eps);
  else hmc_close_kernel<float><<<a.chunks, kHmcThreads, 0, st>>>(a, &a.S->trial_eps);
  if (launch_check(e, 1) || accept_launch(e, s, kInit, st) || read_scal(e, s, &h)) return 1;
  if (!isfinite(h.logp) || h.flag)
    return fail("pinn_hmc_begin: the log density or its gradient is not finite at theta0 (log density %g)", h.logp);
  double eps = opts->step_size;
  if (!(eps > 0.0) && find_good_stepsize(e, s, &eps)) return 1;
  if (read_scal(e, s, &h)) return 1;
  h.eps = eps;
  h.mu = log(10.0 * eps);
  h.m = h.x_bar = h.h_bar = 0.0;
  h.t = 0;
  h.win_n = 0;
  h.win_size = wsize;
  h.next_split = a.adapt && a.window_end >= a.window_start ? a.window_start + wsize - 1 : -1;
  h.flag = 0;
  CUDA_TRY(cudaMemcpyAsync(a.S, &h, sizeof h, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  if (step_size_out) *step_size_out = eps;
  return 0;
}

extern "C" {

int pinn_hmc_begin_ex2(pinn_handle e, const double* host_theta0, const pinn_hmc_options* opts, const double* host_weights,
                       double ll_const, const pinn_hmc_prior* tail, int32_t n_tail, const double* tail_logabs,
                       uint32_t flags, double* step_size_out) {
  if (!e) return fail("pinn_hmc_begin: null handle");
  if (e->plan.prob.func_term >= 0)
    return fail("pinn_hmc_begin: term %d is a functional term (an integral constraint); the log density of the sampler is "
                "built from mean-square terms only", e->plan.prob.func_term);
  if (hmc_start(e, host_theta0, opts, host_weights, ll_const, tail, n_tail, tail_logabs, flags, step_size_out)) {
    hmc_release(e);              // a failed start leaves no chain: pinn_hmc_iterate refuses until the next begin
    return 1;
  }
  return 0;
}

int pinn_hmc_begin_ex(pinn_handle e, const double* host_theta0, const pinn_hmc_options* opts, const double* host_weights,
                      double ll_const, const pinn_hmc_prior* tail, int32_t n_tail, double* step_size_out) {
  return pinn_hmc_begin_ex2(e, host_theta0, opts, host_weights, ll_const, tail, n_tail, nullptr, 0, step_size_out);
}

int pinn_hmc_begin(pinn_handle e, const double* host_theta0, const pinn_hmc_options* opts, const double* host_weights,
                   double ll_const, double* step_size_out) {
  return pinn_hmc_begin_ex(e, host_theta0, opts, host_weights, ll_const, nullptr, 0, step_size_out);
}

int pinn_hmc_iterate(pinn_handle e, int32_t n, double* host_samples, double* host_stats) {
  if (!e) return fail("pinn_hmc_iterate: null handle");
  if (e->plan.prob.func_term >= 0) return fail("pinn_hmc_iterate: the handle has a functional term");
  if (!e->hmc) return fail("pinn_hmc_iterate: call pinn_hmc_begin first");
  if (n < 0) return fail("pinn_hmc_iterate: n = %d must be >= 0", n);
  CUDA_TRY(cudaSetDevice(e->device));
  HmcState* s = e->hmc;
  cudaStream_t st = e->own_stream;
  const char* ng = getenv("PINN_B200_NO_GRAPH");
  const bool use_graph = !e->timing && !(ng && ng[0] == '1');
  if (use_graph) {
    // the graph holds one transition; its arguments change only with the point sets
    unsigned long long key = 1469598103934665603ull;
    key = fnv1a(e->dyn, sizeof e->dyn, key);
    for (const TermState& ts : e->term) key = fnv1a(&ts.n_global, sizeof ts.n_global, key);
    if (s->redraw)
      for (const TermState& ts : e->term) {
        const unsigned long long reg[6] = {ts.sampler_on, (unsigned long long)ts.sampler_kind, ts.sampler_seed,
                                           (unsigned long long)ts.sampler_n, (unsigned long long)ts.kkl_times,
                                           (unsigned long long)ts.kkl_sub << 32 | (unsigned)ts.kkl_flags};
        key = fnv1a(reg, sizeof reg, key);
        key = fnv1a(ts.sampler_lb, sizeof ts.sampler_lb, key);
        key = fnv1a(ts.sampler_ub, sizeof ts.sampler_ub, key);
      }
    if (!s->graph || s->graph_key != key) {
      if (s->graph) { cudaGraphExecDestroy(s->graph); s->graph = nullptr; }
      cudaGraph_t g = nullptr;
      CUDA_TRY(cudaStreamBeginCapture(st, cudaStreamCaptureModeRelaxed));
      const long long l0 = e->launches;
      const int rc = enqueue_transition(e, s, st);
      cudaError_t ce = cudaStreamEndCapture(st, &g);
      e->launches = l0;
      if (rc) { if (g) cudaGraphDestroy(g); return 1; }
      if (ce != cudaSuccess) return fail("pinn_hmc_iterate: graph capture failed: %s", cudaGetErrorString(ce));
      ce = cudaGraphInstantiate(&s->graph, g, 0);
      cudaGraphDestroy(g);
      if (ce != cudaSuccess) { s->graph = nullptr; return fail("pinn_hmc_iterate: graph instantiation failed: %s", cudaGetErrorString(ce)); }
      s->graph_key = key;
    }
  }
  const long long nt = e->n_theta;
  for (int done = 0; done < n;) {
    const int k = std::min(n - done, s->rows);
    CUDA_TRY(cudaMemcpyAsync(&s->a.S->row_base, &s->t, sizeof(long long), cudaMemcpyHostToDevice, st));
    for (int j = 0; j < k; ++j) {
      if (use_graph) {
        CUDA_TRY(cudaGraphLaunch(s->graph, st));
        e->launches += launches_per_transition(e, s);
      } else if (enqueue_transition(e, s, st)) {
        return 1;
      }
    }
    if (host_samples)
      CUDA_TRY(cudaMemcpyAsync(host_samples + (size_t)done * nt, s->a.samples, (size_t)k * nt * sizeof(double),
                               cudaMemcpyDeviceToHost, st));
    if (host_stats)
      CUDA_TRY(cudaMemcpyAsync(host_stats + (size_t)done * PINN_HMC_N_STATS, s->a.stats,
                               (size_t)k * PINN_HMC_N_STATS * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    s->t += k;
    done += k;
  }
  return 0;
}

int pinn_hmc_theta(pinn_handle e, double* host_theta_out) {
  if (!e || !host_theta_out) return fail("pinn_hmc_theta: null handle / output");
  if (!e->hmc) return fail("pinn_hmc_theta: call pinn_hmc_begin first");
  CUDA_TRY(cudaSetDevice(e->device));
  CUDA_TRY(cudaMemcpyAsync(host_theta_out, e->hmc->a.theta, e->n_theta * sizeof(double), cudaMemcpyDeviceToHost,
                           e->own_stream));
  CUDA_TRY(cudaStreamSynchronize(e->own_stream));
  return 0;
}

}  // extern "C"
