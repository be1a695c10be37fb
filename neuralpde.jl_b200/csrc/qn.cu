// qn.cu -- device-resident BFGS / L-BFGS: the pinn_qn_* entry points of include/pinn_b200.h.
//
// theta, g, the direction d, the L-BFGS pairs and BFGS's dense inverse Hessian live on the device in float64; every
// loss / gradient evaluation is the fused kernel (eval_step) at theta + alpha d rounded to the engine dtype.  The line
// search (linesearch.h) and the k x k algebra of the compact L-BFGS form run on the host.  Every reduction here is
// per-block partials in a fixed order followed by one fixed-order pass, on a grid that depends on n_theta only, so runs
// and ranks are bit-identical.
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "engine.h"
#include "linesearch.h"
#include "reduce.cuh"

namespace pinn {
namespace {

constexpr int kQnThreads = 256;
constexpr long long kChunk = 2048;           // elements per block of a reduction
constexpr int kMaxM = 32;                    // longest L-BFGS history
constexpr int kMaxItems = 4 * (kMaxM + 1) + 1;
constexpr int kPhi = kMaxItems;              // scal[kPhi], scal[kPhi + 1]: phi and phi' of the last evaluation
constexpr int kFlag = kMaxItems + 2;         // scal[kFlag] (as int): the accepted step changed theta
constexpr int kScal = kMaxItems + 4;
constexpr long long kMaxBfgsTheta = 16384;   // dense H of 16384^2 doubles = 2 GiB
constexpr double kGAbsTol = 1e-8;            // Optim's g_abstol

// reduction items: sum_i a[i] b[i], or max_i |a[i]| when b == nullptr (NaN propagates)
struct QnItems {
  int n;
  const double* a[kMaxItems];
  const double* b[kMaxItems];
};

// L-BFGS direction d = -(gamma g + sum_j p_j S_j + sum_j q_j Y_j)
struct QnCombine {
  int k;
  double gamma;
  const double* s[kMaxM];
  const double* y[kMaxM];
  double p[kMaxM], q[kMaxM];
};

// grid (chunks, items): part[chunk][item]
__global__ void __launch_bounds__(kQnThreads) qn_multidot_kernel(QnItems it, long long n, double* part) {
  const int j = blockIdx.y;
  const long long lo = (long long)blockIdx.x * kChunk, hi = min(n, lo + kChunk);
  const double* a = it.a[j];
  const double* b = it.b[j];
  double acc = 0.0;
  if (b) {
    for (long long i = lo + threadIdx.x; i < hi; i += kQnThreads) acc = fma(a[i], b[i], acc);
    acc = block_reduce<kQnThreads, false>(acc);
  } else {
    for (long long i = lo + threadIdx.x; i < hi; i += kQnThreads) acc = nan_max(acc, fabs(a[i]));
    acc = block_reduce<kQnThreads, true>(acc);
  }
  if (threadIdx.x == 0) part[(size_t)blockIdx.x * it.n + j] = acc;
}

// out[j] = the chunks' partials of item j combined in chunk order
__global__ void qn_finish_kernel(QnItems it, const double* part, int chunks, double* out) {
  const int j = threadIdx.x;
  if (j >= it.n) return;
  double r = part[j];
  for (int c = 1; c < chunks; ++c) {
    const double v = part[(size_t)c * it.n + j];
    r = it.b[j] ? r + v : nan_max(r, v);
  }
  out[j] = r;
}

// trial point: theta_real = (real)(theta + alpha d), rounded exactly as the accepted update rounds it
template <typename real>
__global__ void qn_trial_kernel(const double* theta, const double* d, double alpha, long long n, real* out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (real)__dadd_rn(theta[i], __dmul_rn(alpha, d[i]));
}

template <typename real>
__global__ void qn_widen_kernel(const real* in, long long n, double* out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (double)in[i];
}

template <typename real>
__global__ void qn_narrow_kernel(const double* in, long long n, real* out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (real)in[i];
}

// phi' = g_trial' d: per-chunk partials
template <typename real>
__global__ void __launch_bounds__(kQnThreads) qn_dot_kernel(const real* g, const double* d, long long n, double* part) {
  const long long lo = (long long)blockIdx.x * kChunk, hi = min(n, lo + kChunk);
  double acc = 0.0;
  for (long long i = lo + threadIdx.x; i < hi; i += kQnThreads) acc = fma((double)g[i], d[i], acc);
  acc = block_reduce<kQnThreads, false>(acc);
  if (threadIdx.x == 0) part[blockIdx.x] = acc;
}

// out2 = {phi, phi'}: the 16 bytes one evaluation sends to the host
template <typename real>
__global__ void qn_phi_kernel(const double* part, int chunks, const real* total, double* out2) {
  double r = part[0];
  for (int c = 1; c < chunks; ++c) r += part[c];
  out2[0] = (double)*total;
  out2[1] = r;
}

// accept the step: s = alpha d, theta += s, y = g_new - g, g = g_new
template <typename real>
__global__ void qn_accept_kernel(double* theta, const double* d, double alpha, double* g, const real* g_new, double* s_out,
                                 double* y_out, long long n, int* changed) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double s = __dmul_rn(alpha, d[i]);
  const double t = theta[i], tn = __dadd_rn(t, s);
  if (tn != t) *changed = 1;
  theta[i] = tn;
  const double gn = (double)g_new[i];
  y_out[i] = __dsub_rn(gn, g[i]);
  g[i] = gn;
  s_out[i] = s;
}

// L-BFGS combination pass: d and per-chunk partials of g'd
__global__ void __launch_bounds__(kQnThreads) qn_combine_kernel(QnCombine c, const double* g, long long n, double* d,
                                                                double* part) {
  const long long lo = (long long)blockIdx.x * kChunk, hi = min(n, lo + kChunk);
  double acc = 0.0;
  for (long long i = lo + threadIdx.x; i < hi; i += kQnThreads) {
    const double gi = g[i];
    double v = c.gamma * gi;
    for (int j = 0; j < c.k; ++j) v = fma(c.p[j], c.s[j][i], v);
    for (int j = 0; j < c.k; ++j) v = fma(c.q[j], c.y[j][i], v);
    d[i] = -v;
    acc = fma(gi, -v, acc);
  }
  acc = block_reduce<kQnThreads, false>(acc);
  if (threadIdx.x == 0) part[blockIdx.x] = acc;
}

// out = scale * H x, one warp per row
__global__ void __launch_bounds__(kQnThreads) qn_gemv_kernel(const double* H, const double* x, double scale, long long n,
                                                             double* out) {
  const long long r = (long long)blockIdx.x * (kQnThreads / 32) + (threadIdx.x >> 5);
  if (r >= n) return;
  const int lane = threadIdx.x & 31;
  const double* row = H + r * n;
  double acc = 0.0;
  for (long long c = lane; c < n; c += 32) acc = fma(row[c], x[c], acc);
  for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) out[r] = scale * acc;
}

// BFGS update H += c1 s s' - (u s' + s u') / s'y with u = H y, c1 = (s'y + y'u) / (s'y)^2; written without contractions
// so that H stays exactly symmetric.  grid (ceil(n / 256), n)
__global__ void __launch_bounds__(kQnThreads) qn_rank2_kernel(double* H, const double* s, const double* u, double c1,
                                                              double inv_sy, long long n) {
  const long long r = blockIdx.y, c = (long long)blockIdx.x * kQnThreads + threadIdx.x;
  if (c >= n) return;
  const double ss = __dmul_rn(s[r], s[c]);
  const double us = __dadd_rn(__dmul_rn(u[r], s[c]), __dmul_rn(s[r], u[c]));
  const size_t k = (size_t)r * n + c;
  H[k] = __dadd_rn(H[k], __dsub_rn(__dmul_rn(c1, ss), __dmul_rn(us, inv_sy)));
}

__global__ void __launch_bounds__(kQnThreads) qn_identity_kernel(double* H, double scale, long long n) {
  const long long r = blockIdx.y, c = (long long)blockIdx.x * kQnThreads + threadIdx.x;
  if (c < n) H[(size_t)r * n + c] = r == c ? scale : 0.0;
}

struct EvalError {};

}  // namespace

struct QnState {
  pinn_qn_options opt = {};
  bool has_w = false;
  double w[PINN_MAX_TERMS] = {};
  int status = PINN_QN_RUNNING;
  long long iters = 0, evals = 0;
  double f = NAN, gnorm = NAN, gtd = NAN;
  double last_alpha = NAN;       // the trial buffers hold the evaluation at this step
  int chunks = 1;
  // device (float64 unless noted)
  double *theta = nullptr, *g = nullptr, *d = nullptr;
  double *S = nullptr, *Y = nullptr;   // L-BFGS: [m + 1][n] ring with one staging slot; BFGS: the last s, y
  double *H = nullptr, *u = nullptr;   // BFGS: inverse Hessian, H y
  double *part = nullptr, *scal = nullptr;
  void *theta_r = nullptr, *g_r = nullptr, *out = nullptr;   // engine dtype: trial theta, its gradient, term losses + total
  double* h_scal = nullptr;      // pinned copy of scal
  // L-BFGS bookkeeping by slot: hist = stored pairs oldest -> newest, stage = the slot the next pair is written to
  std::vector<int> hist, free_slots;
  int stage = 0;
  std::vector<double> SY, YY;    // [(m + 1)^2]: SY[i][j] = s_i'y_j (i stored no later than j), YY[i][j] = y_i'y_j
  std::vector<double> a_slot, b_slot;   // S'g, Y'g of the current g
};

void qn_release(pinn_engine* e) {
  QnState* q = e->qn;
  if (!q) return;
  double* dp[] = {q->theta, q->g, q->d, q->S, q->Y, q->H, q->u, q->part, q->scal};
  for (double* p : dp) if (p) { cudaFree(p); }
  void* vp[] = {q->theta_r, q->g_r, q->out};
  for (void* p : vp) if (p) cudaFree(p);
  if (q->h_scal) cudaFreeHost(q->h_scal);
  delete q;
  e->qn = nullptr;
}

namespace {

bool lbfgs(const QnState* q) { return q->opt.kind == PINN_QN_LBFGS; }
unsigned blocks_of(long long n) { return (unsigned)((n + kQnThreads - 1) / kQnThreads); }

int launch_reduce(pinn_engine* e, QnState* q, const QnItems& it) {
  cudaStream_t st = e->own_stream;
  qn_multidot_kernel<<<dim3(q->chunks, it.n), kQnThreads, 0, st>>>(it, e->n_theta, q->part);
  CUDA_TRY(cudaGetLastError());
  qn_finish_kernel<<<1, 256, 0, st>>>(it, q->part, q->chunks, q->scal);
  CUDA_TRY(cudaGetLastError());
  e->launches += 2;
  return 0;
}

int fetch(pinn_engine* e, QnState* q, int first, int count) {
  CUDA_TRY(cudaMemcpyAsync(q->h_scal + first, q->scal + first, count * sizeof(double), cudaMemcpyDeviceToHost, e->own_stream));
  CUDA_TRY(cudaStreamSynchronize(e->own_stream));
  return 0;
}

// one loss / gradient evaluation at theta + alpha d: {phi, phi'} to the host, one synchronisation
int eval_at(pinn_engine* e, QnState* q, double alpha, double& f, double& df) {
  cudaStream_t st = e->own_stream;
  const long long n = e->n_theta;
  if (any_sampler(e) && pinn_resample(e, st)) return 1;     // a fresh sample per evaluation, as the reference's loss draws
  const bool f64 = e->dtype == PINN_F64;
  if (f64) qn_trial_kernel<double><<<blocks_of(n), kQnThreads, 0, st>>>(q->theta, q->d, alpha, n, (double*)q->theta_r);
  else qn_trial_kernel<float><<<blocks_of(n), kQnThreads, 0, st>>>(q->theta, q->d, alpha, n, (float*)q->theta_r);
  CUDA_TRY(cudaGetLastError());
  e->launches += 1;
  char* out = (char*)q->out;
  void* total = out + (size_t)e->n_terms * e->es;
  if (eval_step(e, q->theta_r, q->has_w ? q->w : nullptr, q->g_r, out, total, false, st)) return 1;
  if (f64) {
    qn_dot_kernel<double><<<q->chunks, kQnThreads, 0, st>>>((const double*)q->g_r, q->d, n, q->part);
    qn_phi_kernel<double><<<1, 1, 0, st>>>(q->part, q->chunks, (const double*)total, q->scal + kPhi);
  } else {
    qn_dot_kernel<float><<<q->chunks, kQnThreads, 0, st>>>((const float*)q->g_r, q->d, n, q->part);
    qn_phi_kernel<float><<<1, 1, 0, st>>>(q->part, q->chunks, (const float*)total, q->scal + kPhi);
  }
  CUDA_TRY(cudaGetLastError());
  e->launches += 2;
  q->last_alpha = NAN;
  if (fetch(e, q, kPhi, 2)) return 1;
  f = q->h_scal[kPhi];
  df = q->h_scal[kPhi + 1];
  q->evals += 1;
  q->last_alpha = alpha;
  return 0;
}

// theta += alpha d and g = the gradient of the last evaluation, which must be the one at alpha; s, y go to the staging slot
int accept(pinn_engine* e, QnState* q, double alpha) {
  cudaStream_t st = e->own_stream;
  const long long n = e->n_theta;
  double* s = lbfgs(q) ? q->S + (size_t)q->stage * n : q->S;
  double* y = lbfgs(q) ? q->Y + (size_t)q->stage * n : q->Y;
  int* changed = (int*)(q->scal + kFlag);
  CUDA_TRY(cudaMemsetAsync(changed, 0, sizeof(int), st));
  if (e->dtype == PINN_F64)
    qn_accept_kernel<double><<<blocks_of(n), kQnThreads, 0, st>>>(q->theta, q->d, alpha, q->g, (const double*)q->g_r, s, y, n, changed);
  else
    qn_accept_kernel<float><<<blocks_of(n), kQnThreads, 0, st>>>(q->theta, q->d, alpha, q->g, (const float*)q->g_r, s, y, n, changed);
  CUDA_TRY(cudaGetLastError());
  e->launches += 1;
  return 0;
}

int set_identity(pinn_engine* e, QnState* q, double scale) {
  const long long n = e->n_theta;
  qn_identity_kernel<<<dim3(blocks_of(n), (unsigned)n), kQnThreads, 0, e->own_stream>>>(q->H, scale, n);
  CUDA_TRY(cudaGetLastError());
  e->launches += 1;
  return 0;
}

// after an accepted step: one multi-dot pass gives S'g, Y'g, S'y_new, Y'y_new and ||g||_inf; a pair with s'y > 0 joins
// the history (the oldest pair leaves when m are stored).  Returns whether the step changed theta in *changed.
int lbfgs_absorb(pinn_engine* e, QnState* q, bool* changed) {
  const long long n = e->n_theta;
  const int M1 = q->opt.m + 1, stg = q->stage;
  const double* yn = q->Y + (size_t)stg * n;
  std::vector<int> rows = q->hist;
  rows.push_back(stg);
  QnItems it;
  it.n = 0;
  for (int h : rows) {
    const double* sh = q->S + (size_t)h * n;
    const double* yh = q->Y + (size_t)h * n;
    it.a[it.n] = sh; it.b[it.n++] = q->g;
    it.a[it.n] = yh; it.b[it.n++] = q->g;
    it.a[it.n] = sh; it.b[it.n++] = yn;
    it.a[it.n] = yh; it.b[it.n++] = yn;
  }
  it.a[it.n] = q->g; it.b[it.n++] = nullptr;
  if (launch_reduce(e, q, it) || fetch(e, q, 0, kScal)) return 1;
  const double* r = q->h_scal;
  for (size_t i = 0; i < rows.size(); ++i) { q->a_slot[rows[i]] = r[4 * i]; q->b_slot[rows[i]] = r[4 * i + 1]; }
  q->gnorm = r[4 * rows.size()];
  int flag;
  memcpy(&flag, r + kFlag, sizeof flag);
  *changed = flag != 0;
  const double sy = r[4 * (rows.size() - 1) + 2];
  if (sy > 0) {                  // curvature guard: a pair with s'y <= 0 is dropped
    for (size_t i = 0; i < rows.size(); ++i) {
      const int h = rows[i];
      q->SY[(size_t)h * M1 + stg] = r[4 * i + 2];
      q->YY[(size_t)h * M1 + stg] = q->YY[(size_t)stg * M1 + h] = r[4 * i + 3];
    }
    q->hist.push_back(stg);
    if ((int)q->hist.size() > q->opt.m) { q->stage = q->hist.front(); q->hist.erase(q->hist.begin()); }
    else { q->stage = q->free_slots.back(); q->free_slots.pop_back(); }
  }
  return 0;
}

// compact form (Byrd, Nocedal & Schnabel 1994): H g = gamma g + S R^-T ((D + gamma Y'Y) R^-1 a - gamma b) - gamma Y R^-1 a,
// a = S'g, b = Y'g, R = upper triangle of S'Y, D = diag(s_i'y_i); the k x k solves run here in double, then one pass
// writes d = -H g and g'd
int lbfgs_direction(pinn_engine* e, QnState* q) {
  const long long n = e->n_theta;
  const int M1 = q->opt.m + 1, k = (int)q->hist.size();
  QnCombine c = {};
  c.k = k;
  c.gamma = 1.0;
  if (k > 0) {
    const std::vector<int>& h = q->hist;
    auto R = [&](int i, int j) { return q->SY[(size_t)h[i] * M1 + h[j]]; };
    auto YY = [&](int i, int j) { return q->YY[(size_t)h[i] * M1 + h[j]]; };
    const double gamma = R(k - 1, k - 1) / YY(k - 1, k - 1);
    double q0[kMaxM], t[kMaxM], p[kMaxM];
    for (int i = k - 1; i >= 0; --i) {               // q0 = R^-1 a
      double v = q->a_slot[h[i]];
      for (int j = i + 1; j < k; ++j) v -= R(i, j) * q0[j];
      q0[i] = v / R(i, i);
    }
    for (int i = 0; i < k; ++i) {                    // t = (D + gamma Y'Y) q0 - gamma b
      double v = 0.0;
      for (int j = 0; j < k; ++j) v += YY(i, j) * q0[j];
      t[i] = R(i, i) * q0[i] + gamma * v - gamma * q->b_slot[h[i]];
    }
    for (int i = 0; i < k; ++i) {                    // p = R^-T t
      double v = t[i];
      for (int j = 0; j < i; ++j) v -= R(j, i) * p[j];
      p[i] = v / R(i, i);
    }
    c.gamma = gamma;
    for (int i = 0; i < k; ++i) {
      c.s[i] = q->S + (size_t)h[i] * n;
      c.y[i] = q->Y + (size_t)h[i] * n;
      c.p[i] = p[i];
      c.q[i] = -gamma * q0[i];
    }
  }
  cudaStream_t st = e->own_stream;
  qn_combine_kernel<<<q->chunks, kQnThreads, 0, st>>>(c, q->g, n, q->d, q->part);
  CUDA_TRY(cudaGetLastError());
  QnItems it;
  it.n = 1; it.a[0] = q->g; it.b[0] = q->d;
  qn_finish_kernel<<<1, 256, 0, st>>>(it, q->part, q->chunks, q->scal);
  CUDA_TRY(cudaGetLastError());
  e->launches += 2;
  if (fetch(e, q, 0, 1)) return 1;
  q->gtd = q->h_scal[0];
  return 0;
}

// after an accepted step: u = H y, then s'y, y'u and ||g||_inf; H gets the BFGS update when s'y > 0
int bfgs_absorb(pinn_engine* e, QnState* q, bool* changed) {
  const long long n = e->n_theta;
  cudaStream_t st = e->own_stream;
  qn_gemv_kernel<<<(unsigned)((n + 7) / 8), kQnThreads, 0, st>>>(q->H, q->Y, 1.0, n, q->u);
  CUDA_TRY(cudaGetLastError());
  e->launches += 1;
  QnItems it;
  it.n = 3;
  it.a[0] = q->S; it.b[0] = q->Y;
  it.a[1] = q->Y; it.b[1] = q->u;
  it.a[2] = q->g; it.b[2] = nullptr;
  if (launch_reduce(e, q, it) || fetch(e, q, 0, kScal)) return 1;
  const double sy = q->h_scal[0], yu = q->h_scal[1];
  q->gnorm = q->h_scal[2];
  int flag;
  memcpy(&flag, q->h_scal + kFlag, sizeof flag);
  *changed = flag != 0;
  if (sy > 0) {
    qn_rank2_kernel<<<dim3(blocks_of(n), (unsigned)n), kQnThreads, 0, st>>>(q->H, q->S, q->u, (sy + yu) / (sy * sy), 1.0 / sy, n);
    CUDA_TRY(cudaGetLastError());
    e->launches += 1;
  }
  return 0;
}

int bfgs_direction(pinn_engine* e, QnState* q) {
  const long long n = e->n_theta;
  qn_gemv_kernel<<<(unsigned)((n + 7) / 8), kQnThreads, 0, e->own_stream>>>(q->H, q->g, -1.0, n, q->d);
  CUDA_TRY(cudaGetLastError());
  e->launches += 1;
  QnItems it;
  it.n = 1; it.a[0] = q->g; it.b[0] = q->d;
  if (launch_reduce(e, q, it) || fetch(e, q, 0, 1)) return 1;
  q->gtd = q->h_scal[0];
  return 0;
}

int direction(pinn_engine* e, QnState* q) { return lbfgs(q) ? lbfgs_direction(e, q) : bfgs_direction(e, q); }

// a direction that is not a descent direction: forget the curvature information and step along -g
int reset_direction(pinn_engine* e, QnState* q) {
  if (lbfgs(q)) {
    for (int h : q->hist) q->free_slots.push_back(h);
    q->hist.clear();
  } else if (set_identity(e, q, 1.0)) {
    return 1;
  }
  return direction(e, q);
}

// one iteration: direction, line search, accepted step, history update, stopping tests
int qn_step(pinn_engine* e, QnState* q) {
  if (direction(e, q)) return 1;
  if (!(q->gtd < 0) && reset_direction(e, q)) return 1;
  auto ev = [&](double a, double& f, double& df) { if (eval_at(e, q, a, f, df)) throw EvalError(); };
  LsResult r;
  try {
    r = q->opt.linesearch == PINN_LS_HAGERZHANG ? hager_zhang(ev, q->f, q->gtd, 1.0) : backtracking(ev, q->f, q->gtd, 1.0);
  } catch (const EvalError&) {
    return 1;
  }
  if (r.status != LS_OK) { q->status = PINN_QN_LS_FAILED; return 0; }
  q->iters += 1;
  if (r.alpha == 0.0) { q->status = PINN_QN_CONVERGED; return 0; }   // theta unchanged
  double f = r.phi, df;
  // the trial buffers hold the last evaluation; the accepted step's gradient needs one more when it was an earlier trial
  if (!(q->last_alpha == r.alpha) && eval_at(e, q, r.alpha, f, df)) return 1;
  bool changed = false;
  if (accept(e, q, r.alpha)) return 1;
  if (lbfgs(q) ? lbfgs_absorb(e, q, &changed) : bfgs_absorb(e, q, &changed)) return 1;
  q->f = f;
  if (!changed || q->gnorm <= kGAbsTol) q->status = PINN_QN_CONVERGED;
  return 0;
}

template <typename T>
int alloc(T** p, size_t count, pinn_engine* e) { return dev_alloc((void**)p, count * sizeof(T), e); }

}  // namespace
}  // namespace pinn

using namespace pinn;

extern "C" {

int pinn_qn_begin(pinn_handle e, const void* host_theta0, const pinn_qn_options* opts, const double* host_weights) {
  if (!e) return fail("pinn_qn_begin: null handle");
  if (!host_theta0 || !opts) return fail("pinn_qn_begin: null theta / options");
  if (opts->kind != PINN_QN_LBFGS && opts->kind != PINN_QN_BFGS) return fail("pinn_qn_begin: unknown optimizer kind %d", opts->kind);
  if (opts->linesearch != PINN_LS_HAGERZHANG && opts->linesearch != PINN_LS_BACKTRACKING)
    return fail("pinn_qn_begin: unknown line search %d", opts->linesearch);
  if (opts->kind == PINN_QN_LBFGS && (opts->m < 1 || opts->m > kMaxM))
    return fail("pinn_qn_begin: L-BFGS history m = %d outside [1, %d]", opts->m, kMaxM);
  const long long n = e->n_theta;
  if (opts->kind == PINN_QN_BFGS && n > kMaxBfgsTheta)
    return fail("pinn_qn_begin: BFGS keeps a dense float64 n_theta x n_theta inverse Hessian; n_theta = %lld exceeds %lld "
                "(2 GiB) -- use L-BFGS (PINN_QN_LBFGS) for this network", n, kMaxBfgsTheta);
  if (e->total_tiles <= 0 && e->nranks <= 1) return fail("pinn_qn_begin: no collocation points");
  CUDA_TRY(cudaSetDevice(e->device));
  qn_release(e);
  QnState* q = new QnState();
  e->qn = q;
  q->opt = *opts;
  if (q->opt.kind == PINN_QN_BFGS) q->opt.m = 1;
  if (host_weights) { q->has_w = true; memcpy(q->w, host_weights, sizeof(double) * e->n_terms); }
  q->chunks = (int)std::max<long long>(1, (n + kChunk - 1) / kChunk);
  const size_t slots = lbfgs(q) ? (size_t)q->opt.m + 1 : 1;
  int rc = alloc(&q->theta, n, e) || alloc(&q->g, n, e) || alloc(&q->d, n, e) || alloc(&q->S, slots * n, e) ||
           alloc(&q->Y, slots * n, e) || alloc(&q->part, (size_t)q->chunks * kMaxItems, e) || alloc(&q->scal, kScal, e) ||
           dev_alloc(&q->theta_r, n * e->es, e) || dev_alloc(&q->g_r, n * e->es, e) ||
           dev_alloc(&q->out, (PINN_MAX_TERMS + 1) * e->es, e);
  if (!rc && !lbfgs(q)) rc = alloc(&q->u, n, e) || alloc(&q->H, (size_t)n * n, e);
  if (rc) { qn_release(e); return 1; }
  cudaError_t ce = cudaMallocHost((void**)&q->h_scal, kScal * sizeof(double));
  if (ce != cudaSuccess) { q->h_scal = nullptr; qn_release(e); return fail("pinn_qn_begin: pinned buffer: %s", cudaGetErrorString(ce)); }
  const int M1 = q->opt.m + 1;
  q->SY.assign((size_t)M1 * M1, 0.0);
  q->YY.assign((size_t)M1 * M1, 0.0);
  q->a_slot.assign(M1, 0.0);
  q->b_slot.assign(M1, 0.0);
  for (int s = M1 - 1; s >= 1; --s) q->free_slots.push_back(s);   // slots taken in order 1, 2, ...
  q->stage = 0;

  cudaStream_t st = e->own_stream;
  CUDA_TRY(cudaMemcpyAsync(q->theta_r, host_theta0, n * e->es, cudaMemcpyHostToDevice, st));
  if (e->dtype == PINN_F64) qn_widen_kernel<double><<<blocks_of(n), kQnThreads, 0, st>>>((const double*)q->theta_r, n, q->theta);
  else qn_widen_kernel<float><<<blocks_of(n), kQnThreads, 0, st>>>((const float*)q->theta_r, n, q->theta);
  CUDA_TRY(cudaGetLastError());
  e->launches += 1;
  CUDA_TRY(cudaMemsetAsync(q->d, 0, n * sizeof(double), st));
  CUDA_TRY(cudaMemsetAsync(q->g, 0, n * sizeof(double), st));
  double f, df;
  if (eval_at(e, q, 0.0, f, df) || accept(e, q, 0.0)) return 1;   // g = the gradient at theta0
  QnItems it;
  it.n = 1; it.a[0] = q->g; it.b[0] = nullptr;
  if (launch_reduce(e, q, it) || fetch(e, q, 0, 1)) return 1;
  q->f = f;
  q->gnorm = q->h_scal[0];
  if (!lbfgs(q)) {
    const double sn = q->opt.initial_stepnorm;
    if (set_identity(e, q, sn > 0 && q->gnorm > 0 ? sn / q->gnorm : 1.0)) return 1;
  }
  if (q->gnorm <= kGAbsTol) q->status = PINN_QN_CONVERGED;
  return 0;
}

int pinn_qn_iterate(pinn_handle e, int32_t n_iters, double* host_f, double* host_gnorm_inf, int32_t* host_status,
                    int64_t* host_iters, int64_t* host_evals) {
  if (!e) return fail("pinn_qn_iterate: null handle");
  if (!e->qn) return fail("pinn_qn_iterate: call pinn_qn_begin first");
  if (n_iters < 0) return fail("pinn_qn_iterate: n_iters must be >= 0");
  CUDA_TRY(cudaSetDevice(e->device));
  QnState* q = e->qn;
  for (int i = 0; i < n_iters && q->status == PINN_QN_RUNNING; ++i)
    if (qn_step(e, q)) return 1;
  if (host_f) *host_f = q->f;
  if (host_gnorm_inf) *host_gnorm_inf = q->gnorm;
  if (host_status) *host_status = q->status;
  if (host_iters) *host_iters = q->iters;
  if (host_evals) *host_evals = q->evals;
  return 0;
}

int pinn_qn_theta(pinn_handle e, void* host_theta_out) {
  if (!e || !host_theta_out) return fail("pinn_qn_theta: null handle / output");
  if (!e->qn) return fail("pinn_qn_theta: call pinn_qn_begin first");
  CUDA_TRY(cudaSetDevice(e->device));
  QnState* q = e->qn;
  const long long n = e->n_theta;
  cudaStream_t st = e->own_stream;
  if (e->dtype == PINN_F64) qn_narrow_kernel<double><<<blocks_of(n), kQnThreads, 0, st>>>(q->theta, n, (double*)q->theta_r);
  else qn_narrow_kernel<float><<<blocks_of(n), kQnThreads, 0, st>>>(q->theta, n, (float*)q->theta_r);
  CUDA_TRY(cudaGetLastError());
  e->launches += 1;
  q->last_alpha = NAN;           // the trial buffer now holds theta itself
  CUDA_TRY(cudaMemcpyAsync(host_theta_out, q->theta_r, n * e->es, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  return 0;
}

}  // extern "C"
