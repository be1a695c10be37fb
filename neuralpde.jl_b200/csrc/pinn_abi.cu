// pinn_abi.cu -- host side of the C ABI declared in include/pinn_b200.h: workspace ownership, kernel
// launch sequencing, host-buffer staging and the optional NCCL gradient allreduce.  Descriptor
// validation and lowering live in the planner (plan.cu), the handle struct in engine.h, the quasi-Newton driver in qn.cu, the HMC sampler in
// hmc.cu.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "engine.h"

namespace pinn {
cudaError_t ffma_launch(int dtype, bool bufs_smem, bool integ, bool fixed, bool func, bool dmma, const FfmaArgs& a,
                        int grid, size_t smem, cudaStream_t st);
cudaError_t grad_stats_launch(int dtype, const void* grad, long long n, double* out2, cudaStream_t st);
cudaError_t sample_uniform_launch(int dtype, void* pts, long long n, int dim, const double* lb, const double* ub,
                                  unsigned long long seed, unsigned long long draw, const unsigned long long* draw_dev,
                                  cudaStream_t st);
cudaError_t sample_lhs_launch(int dtype, void* pts, long long n, int dim, const double* lb, const double* ub,
                              unsigned long long seed, unsigned long long draw, const unsigned long long* draw_dev,
                              cudaStream_t st);
cudaError_t sample_kkl_launch(int dtype, void* pts, long long n_times, int sub, int n_z, double t_lb, double t_ub,
                              bool strong, unsigned long long seed, unsigned long long draw,
                              const unsigned long long* draw_dev, cudaStream_t st);
cudaError_t finish_launch(int dtype, const void* packed, long long n_grad, int n_terms, const ScaleW& scale_w, void* out_grad,
                          void* out_terms, void* out_total, cudaStream_t st);
}  // namespace pinn

using namespace pinn;

// ---- minimal NCCL binding (resolved at run time so single-GPU use has no dependency) ----
typedef struct { char internal[128]; } ncclUniqueId;
typedef int ncclResult_t;
enum { ncclInt8 = 0, ncclInt32 = 2, ncclFloat32 = 7, ncclFloat64 = 8, ncclSumOp = 0, ncclMinOp = 3 };
struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
};
static NcclApi g_nccl;

static bool load_nccl() {
  if (g_nccl.lib) return true;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  for (const char* n : names) {
    g_nccl.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (g_nccl.lib) break;
  }
  if (!g_nccl.lib) return false;
  g_nccl.GetUniqueId = (decltype(g_nccl.GetUniqueId))dlsym(g_nccl.lib, "ncclGetUniqueId");
  g_nccl.CommInitRank = (decltype(g_nccl.CommInitRank))dlsym(g_nccl.lib, "ncclCommInitRank");
  g_nccl.CommDestroy = (decltype(g_nccl.CommDestroy))dlsym(g_nccl.lib, "ncclCommDestroy");
  g_nccl.AllReduce = (decltype(g_nccl.AllReduce))dlsym(g_nccl.lib, "ncclAllReduce");
  g_nccl.AllGather = (decltype(g_nccl.AllGather))dlsym(g_nccl.lib, "ncclAllGather");
  g_nccl.GetErrorString = (decltype(g_nccl.GetErrorString))dlsym(g_nccl.lib, "ncclGetErrorString");
  return g_nccl.GetUniqueId && g_nccl.CommInitRank && g_nccl.CommDestroy && g_nccl.AllReduce;
}

int pinn::dev_alloc(void** p, size_t bytes, pinn_engine* e) {
  if (bytes == 0) bytes = 16;
  cudaError_t err = cudaMalloc(p, bytes);
  if (err != cudaSuccess) return fail("cudaMalloc(%zu bytes) failed: %s", bytes, cudaGetErrorString(err));
  e->ws_bytes += (long long)bytes;
  return 0;
}

static void retile(pinn_engine* e) {
  int t0 = 0;
  for (int t = 0; t < e->n_terms; ++t) {
    e->dyn[t].tile0 = t0;
    e->dyn[t].n_tiles = (int)((e->dyn[t].n + e->plan.tile_pts - 1) / e->plan.tile_pts);
    t0 += e->dyn[t].n_tiles;
  }
  e->total_tiles = t0;
}

// the handle's device buffers in every launch-argument template
static void bind_buffers(pinn_engine* e) {
  Plan& p = e->plan;
  FfmaArgs& f = p.ffma;
  f.prob = e->dprob; f.partial = e->partial; f.partial_stride = e->partial_stride; f.term_sums = e->term_sums;
  f.stash = e->stash; f.gbufs = e->gbufs;
  for (TcCommonArgs* c : {static_cast<TcCommonArgs*>(&p.tc), static_cast<TcCommonArgs*>(&p.tw)}) {
    c->prob = e->dprob; c->partial = (float*)e->partial; c->partial_stride = e->partial_stride; c->term_sums = e->term_sums;
    c->acc = e->tc_acc;
  }
  p.tc.stash = p.tw.hstash = (uint8_t*)e->stash;
  p.tw.zstash = (float*)e->tw_zstash; p.tw.wpack = (const uint8_t*)e->tw_wpack; p.tw.tile_counter = e->tw_counter;
  p.pack.prob = e->dprob; p.pack.wpack = (uint8_t*)e->tw_wpack; p.pack.tile_counter = e->tw_counter;
}

// per-call fields of a fused launch; everything else in the kernel arguments is fixed per handle (Plan)
struct LaunchCall {
  const void* theta;
  int tile_begin, tile_end, mode;  // mode 0 loss+grad, 1 loss only, 2 residual out
  void* resid_out;                 // mode 2: r[n] of the selected term
  double seed[PINN_MAX_TERMS];     // w_k * scale_k
  TailArgs tail;
};

// a kernel's arguments: the handle's template with the per-call fields of c and the current point sets
template <typename Args>
static Args with_call(Args a, const pinn_engine* e, const LaunchCall& c) {
  a.theta = (decltype(a.theta))c.theta; a.resid_out = (decltype(a.resid_out))c.resid_out;
  a.tile_begin = c.tile_begin; a.tile_end = c.tile_end; a.mode = c.mode;
  memcpy(a.seed, c.seed, sizeof a.seed); memcpy(a.dyn, e->dyn, sizeof a.dyn);
  a.tail = c.tail;
  return a;
}

extern "C" {

const char* pinn_last_error(void) { return last_error(); }
int pinn_abi_version(void) { return PINN_ABI_VERSION; }

int pinn_destroy(pinn_handle e) {
  if (!e) return 0;
  cudaSetDevice(e->device);
  if (e->adam_graph) cudaGraphExecDestroy(e->adam_graph);
  qn_release(e);
  hmc_release(e);
  if (e->p2p) {
    // peers may still be reading this rank's symmetric buffers inside their last step: callers synchronise the ranks
    // (any collective / barrier) before destroying handles; here only this device is drained
    cudaDeviceSynchronize();
    for (int r = 0; r < e->nranks; ++r)
      if (r != e->rank && e->peer_base[r]) cudaIpcCloseMemHandle(e->peer_base[r]);
  }
  if (e->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(e->comm);
  void* ptrs[] = {e->dprob, e->partial, e->term_sums, e->stash, e->gbufs, e->packed, e->d_state, e->sym,
                  e->d_theta, e->d_grad, e->d_out, e->adam_m, e->adam_v, e->tw_wpack, e->tw_zstash, e->tw_counter, e->tc_acc};
  for (void* p : ptrs) if (p) cudaFree(p);
  for (const TermState& ts : e->term) {
    if (ts.own_pts) cudaFree(ts.own_pts);
    if (ts.own_qw) cudaFree(ts.own_qw);
  }
  for (void* p : e->fixed_own) if (p) cudaFree(p);
  if (e->h_pin_in) cudaFreeHost(e->h_pin_in);
  if (e->h_pin_out) cudaFreeHost(e->h_pin_out);
  if (e->own_stream) cudaStreamDestroy(e->own_stream);
  if (e->ev0) cudaEventDestroy(e->ev0);
  if (e->ev1) cudaEventDestroy(e->ev1);
  delete e;
  return 0;
}

int pinn_create(const pinn_problem_desc* d, pinn_handle* out) { return pinn_create_ex(d, nullptr, 0, out); }

int pinn_quadrature_nodes(int32_t q, double* x, double* w) {
  if (q < 1 || q > PINN_MAX_QUAD) return fail("pinn_quadrature_nodes: q=%d out of range [1,%d]", q, PINN_MAX_QUAD);
  if (!x || !w) return fail("pinn_quadrature_nodes: null output");
  gauss_legendre(q, x, w);
  return 0;
}

int pinn_create_ex(const pinn_problem_desc* d, const pinn_integral_desc* integrals, int32_t n_integrals, pinn_handle* out) {
  return pinn_create_ex2(d, integrals, n_integrals, nullptr, 0, out);
}

int pinn_create_ex2(const pinn_problem_desc* d, const pinn_integral_desc* integrals, int32_t n_integrals,
                    const pinn_fixed_net_desc* fixed, int32_t n_fixed, pinn_handle* out) {
  if (!out) return fail("pinn_create: null output handle");
  *out = nullptr;
  if (!d) return fail("pinn_create: null descriptor");
  int ndev = 0;
  cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess || ndev == 0)
    return fail("pinn_create: no CUDA device available (%s); this engine has no CPU fallback",
                cudaGetErrorString(ce));
  if (d->device < 0 || d->device >= ndev) return fail("pinn_create: device %d not in [0,%d)", d->device, ndev);
  CUDA_TRY(cudaSetDevice(d->device));
  pinn_engine* e = new pinn_engine();
  e->dtype = d->dtype; e->mode = d->mode; e->device = d->device;
  e->es = d->dtype == PINN_F64 ? 8 : 4;
  e->n_terms = d->n_terms; e->n_theta = d->n_theta;
  int max_smem = 0;
  cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, e->device);
  if (max_smem <= 0) max_smem = 227 * 1024;
  if (plan_problem(d, integrals, n_integrals, fixed, n_fixed, max_smem, e->plan)) { pinn_destroy(e); return 1; }
  const Plan& p = e->plan;
  cudaDeviceGetAttribute(&e->num_sms, cudaDevAttrMultiProcessorCount, e->device);
  if (e->num_sms <= 0) e->num_sms = 132;

#define TRY_OR_DESTROY(x) do { if (x) { pinn_destroy(e); return 1; } } while (0)
  TRY_OR_DESTROY(dev_alloc((void**)&e->dprob, sizeof(DevProblem), e));
  cudaError_t err = cudaMemcpy(e->dprob, &p.prob, sizeof(DevProblem), cudaMemcpyHostToDevice);
  if (err != cudaSuccess) { fail("pinn_create: upload failed: %s", cudaGetErrorString(err)); pinn_destroy(e); return 1; }
  const size_t g = (size_t)e->num_sms;
  e->partial_stride = (e->n_theta + 3) & ~3LL;
  // a functional term's own partials G follow the ordinary ones (tail.cuh)
  const size_t n_partials = p.prob.func_term >= 0 ? 2 * g : g;
  TRY_OR_DESTROY(dev_alloc(&e->partial, n_partials * (size_t)e->partial_stride * e->es, e));
  TRY_OR_DESTROY(dev_alloc((void**)&e->term_sums, g * PINN_MAX_TERMS * sizeof(double), e));
  if (ffma_kernel_mode(e->mode)) {
    TRY_OR_DESTROY(dev_alloc(&e->stash, g * (size_t)p.ffma.stash_per_cta * e->es, e));
    if (!p.bufs_smem) TRY_OR_DESTROY(dev_alloc(&e->gbufs, g * 2 * (size_t)p.ffma.buf_elems * e->es, e));
  } else {
    TRY_OR_DESTROY(dev_alloc(&e->stash, g * (size_t)(p.wide ? p.tw.hstash_per_cta : p.tc.stash_per_cta), e));
    TRY_OR_DESTROY(dev_alloc((void**)&e->tc_acc, g * (size_t)kAccCols * kAccRows * sizeof(float), e));
    if (p.wide) {
      TRY_OR_DESTROY(dev_alloc(&e->tw_zstash, g * (size_t)p.tw.zstash_per_cta * sizeof(float), e));
      TRY_OR_DESTROY(dev_alloc(&e->tw_wpack, (size_t)std::max(p.pack.n_images, 1) * (p.x256 ? kTxImgBytes : kTwImgBytes), e));
      TRY_OR_DESTROY(dev_alloc((void**)&e->tw_counter, 64, e));
    }
  }
  TRY_OR_DESTROY(dev_alloc(&e->packed, ((size_t)e->n_theta + PINN_MAX_TERMS) * e->es, e));
  TRY_OR_DESTROY(dev_alloc((void**)&e->d_state, sizeof(TailState), e));
  {
    TailState st0;
    memset(&st0, 0, sizeof st0);
    st0.func_term = (short)p.prob.func_term; st0.func_square = (short)p.prob.func_square;
    err = cudaMemcpy(e->d_state, &st0, sizeof st0, cudaMemcpyHostToDevice);
  }
  if (err != cudaSuccess) { fail("pinn_create: state init failed: %s", cudaGetErrorString(err)); pinn_destroy(e); return 1; }
  {
    const char* to = getenv("PINN_B200_TAIL_TIMEOUT_S");
    if (to && atof(to) > 0) e->tail_timeout_ns = (unsigned long long)(atof(to) * 1e9);
  }
  TRY_OR_DESTROY(dev_alloc(&e->d_theta, (size_t)e->n_theta * e->es, e));
  TRY_OR_DESTROY(dev_alloc(&e->d_grad, (size_t)e->n_theta * e->es, e));
  TRY_OR_DESTROY(dev_alloc(&e->d_out, (PINN_MAX_TERMS + 1) * e->es, e));
  err = cudaMallocHost(&e->h_pin_in, (size_t)e->n_theta * e->es);
  if (err == cudaSuccess) err = cudaHostAlloc(&e->h_pin_out, ((size_t)e->n_theta + PINN_MAX_TERMS + 1) * e->es, cudaHostAllocMapped);
  if (err == cudaSuccess) {
    void* dptr = nullptr;
    e->zero_copy_out = cudaHostGetDevicePointer(&dptr, e->h_pin_out, 0) == cudaSuccess && dptr == e->h_pin_out;
    cudaGetLastError();
  }
  // a BLOCKING stream: the *_host entry points run here and must order after uploads / sampler draws that callers
  // enqueue on the legacy default stream (pinn_set_points_host, pinn_set_sampler, pinn_resample with stream = 0)
  if (err == cudaSuccess) err = cudaStreamCreate(&e->own_stream);
  if (err == cudaSuccess) err = cudaEventCreate(&e->ev0);
  if (err == cudaSuccess) err = cudaEventCreate(&e->ev1);
  if (err != cudaSuccess) { fail("pinn_create: host staging setup failed: %s", cudaGetErrorString(err)); pinn_destroy(e); return 1; }
#undef TRY_OR_DESTROY
  bind_buffers(e);
  retile(e);
  *out = e;
  return 0;
}

static int check_fixed(pinn_handle e, int32_t j, const char* fn) {
  if (!e) return fail("%s: null handle", fn);
  if (j < 0 || j >= e->plan.prob.n_fixed)
    return fail("%s: fixed network %d out of range [0,%d)", fn, j, e->plan.prob.n_fixed);
  return 0;
}

// point fixed network j at p in the device copy of the problem; evaluations still in flight finish with the old pointer
// first (the kernels read it from there, so captured Adam graphs need no re-capture)
static int bind_fixed(pinn_engine* e, int j, const void* p) {
  CUDA_TRY(cudaSetDevice(e->device));
  if (e->fixed_ptr[j] == p) return 0;
  CUDA_TRY(cudaDeviceSynchronize());
  CUDA_TRY(cudaMemcpy(&e->dprob->fixed_params[j], &p, sizeof p, cudaMemcpyHostToDevice));
  e->fixed_ptr[j] = p;
  return 0;
}

int pinn_set_fixed_params(pinn_handle e, int32_t j, const void* dev_params) {
  if (check_fixed(e, j, "pinn_set_fixed_params")) return 1;
  if (!dev_params) return fail("pinn_set_fixed_params: null parameters");
  return bind_fixed(e, j, dev_params);
}

int pinn_set_fixed_params_host(pinn_handle e, int32_t j, const void* host_params, void* stream) {
  if (check_fixed(e, j, "pinn_set_fixed_params_host")) return 1;
  if (!host_params) return fail("pinn_set_fixed_params_host: null parameters");
  CUDA_TRY(cudaSetDevice(e->device));
  const size_t bytes = (size_t)e->plan.fixed_len[j] * e->es;
  if (!e->fixed_own[j]) {
    if (dev_alloc(&e->fixed_own[j], bytes, e)) return 1;
  } else {
    CUDA_TRY(cudaDeviceSynchronize());   // evaluations in flight on any stream may still read the bound buffer
  }
  // complete before returning: later evaluations, on whatever stream, read the new parameters
  CUDA_TRY(cudaMemcpyAsync(e->fixed_own[j], host_params, bytes, cudaMemcpyHostToDevice, (cudaStream_t)stream));
  CUDA_TRY(cudaStreamSynchronize((cudaStream_t)stream));
  return bind_fixed(e, j, e->fixed_own[j]);
}

static int check_term(pinn_handle e, int32_t term, const char* fn) {
  if (!e) return fail("%s: null handle", fn);
  if (term < 0 || term >= e->n_terms) return fail("%s: term %d out of range [0,%d)", fn, term, e->n_terms);
  return 0;
}

int pinn_set_points(pinn_handle e, int32_t term, const void* dev_pts, int64_t n, const void* dev_w) {
  if (check_term(e, term, "pinn_set_points")) return 1;
  if (n < 0) return fail("pinn_set_points: negative point count");
  if (n > 0 && !dev_pts) return fail("pinn_set_points: null points");
  if (e->plan.term[term].reduction == PINN_REDUCE_WSUM && n > 0 && !dev_w)
    return fail("pinn_set_points: term %d is a weighted-sum (quadrature) term and needs weights", term);
  if (n > (int64_t)kTilePts * 60000000LL) return fail("pinn_set_points: too many points");
  e->dyn[term].pts = dev_pts; e->dyn[term].qw = dev_w; e->dyn[term].n = n;
  retile(e);
  return 0;
}

static int grow(void** p, size_t* cap, size_t need, pinn_engine* e) {
  if (need <= *cap) return 0;
  if (*p) { cudaFree(*p); e->ws_bytes -= (long long)*cap; *p = nullptr; *cap = 0; }
  size_t want = need + need / 8;
  if (dev_alloc(p, want, e)) return 1;
  *cap = want;
  return 0;
}

int pinn_set_points_host(pinn_handle e, int32_t term, const void* host_pts, int64_t n, const void* host_w,
                         void* stream) {
  if (check_term(e, term, "pinn_set_points_host")) return 1;
  if (n < 0) return fail("pinn_set_points_host: negative point count");
  if (n > 0 && !host_pts) return fail("pinn_set_points_host: null points");
  if (e->plan.term[term].reduction == PINN_REDUCE_WSUM && n > 0 && !host_w)
    return fail("pinn_set_points_host: term %d is a weighted-sum (quadrature) term and needs weights", term);
  CUDA_TRY(cudaSetDevice(e->device));
  const int dim = e->plan.prob.terms[term].dim;
  cudaStream_t st = (cudaStream_t)stream;
  size_t bytes = (size_t)n * dim * e->es;
  TermState& ts = e->term[term];
  if (grow(&ts.own_pts, &ts.own_pts_cap, bytes, e)) return 1;
  if (bytes) CUDA_TRY(cudaMemcpyAsync(ts.own_pts, host_pts, bytes, cudaMemcpyHostToDevice, st));
  const void* w = nullptr;
  if (host_w) {
    size_t wb = (size_t)n * e->es;
    if (grow(&ts.own_qw, &ts.own_qw_cap, wb, e)) return 1;
    if (wb) CUDA_TRY(cudaMemcpyAsync(ts.own_qw, host_w, wb, cudaMemcpyHostToDevice, st));
    w = ts.own_qw;
  }
  e->dyn[term].pts = ts.own_pts; e->dyn[term].qw = w; e->dyn[term].n = n;
  retile(e);
  return 0;
}

int pinn_set_global_count(pinn_handle e, int32_t term, int64_t n_global) {
  if (check_term(e, term, "pinn_set_global_count")) return 1;
  if (n_global <= 0) return fail("pinn_set_global_count: n_global must be positive");
  if (term == e->plan.prob.func_term && n_global != e->dyn[term].n)
    return fail("pinn_set_global_count: term %d is a functional term: g(sum) is not the sum of the ranks' g, so its whole "
                "node set stays on one rank (0 points on the others) and its global count is the local count %lld", term,
                (long long)e->dyn[term].n);
  e->term[term].n_global = n_global; e->term[term].n_global_set = true;
  return 0;
}

// scale_k (so that L_k = scale_k * sum_p qw r^2) and the loss weights w_k
static int prepare_scales(pinn_engine* e, const double* host_weights, double* seed, ScaleW& sw) {
  for (int t = 0; t < e->n_terms; ++t) {
    double sc;
    if (e->plan.term[t].reduction == PINN_REDUCE_MEAN) {
      long long ng = e->term[t].n_global_set ? e->term[t].n_global : e->dyn[t].n;
      if (ng <= 0) return fail("pinn_loss_grad: term %d has no points (pinn_set_points was not called or n == 0)", t);
      sc = 1.0 / (double)ng;
    } else {
      sc = e->plan.term[t].scale;
    }
    double w = host_weights ? host_weights[t] : 1.0;
    sw.scale[t] = sc;
    sw.w[t] = w;
    seed[t] = sc * w;
  }
  return 0;
}

// launch the fused kernel of the handle's mode over tiles [tile_begin, tile_end); c.tail.state != null attaches the
// in-kernel tail (gradient reduction / optimizer / peer allreduce) and makes the launch cooperative
static int launch_fused(pinn_engine* e, const LaunchCall& c, int grid, cudaStream_t st) {
  const Plan& p = e->plan;
  if (ffma_kernel_mode(e->mode)) {
    FfmaArgs a = with_call(p.ffma, e, c);
    a.n_tiles = e->total_tiles;
    for (int j = 0; j < p.prob.n_fixed; ++j)
      if (!e->fixed_ptr[j])
        return fail("pinn: fixed network %d has no parameters (call pinn_set_fixed_params or pinn_set_fixed_params_host "
                    "first)", j);
    CUDA_TRY(ffma_launch(e->dtype, p.bufs_smem, p.integ, p.prob.n_fixed > 0, p.prob.func_term >= 0,
                         e->mode == PINN_MODE_TC_F64, a, grid, p.smem, st));
    return 0;
  }
  if (p.wide) {
    TwPackArgs pk = p.pack;
    pk.theta = (const float*)c.theta; pk.counter_init = c.tile_begin + grid;
    CUDA_TRY(p.x256 ? tx_pack_launch(pk, st) : tw_pack_launch(pk, st));
    e->launches += 1;
    CUDA_TRY(p.x256 ? tx_launch(with_call(p.tw, e, c), grid, p.smem, st) : tw_launch(with_call(p.tw, e, c), grid, p.smem, st));
    return 0;
  }
  CUDA_TRY(tc_launch(with_call(p.tc, e, c), grid, p.smem, st));
  return 0;
}

}  // extern "C"

bool pinn::any_sampler(const pinn_engine* e) {
  for (int t = 0; t < e->n_terms; ++t) if (e->term[t].sampler_on) return true;
  return false;
}

// tail arguments of one step
static void fill_tail(pinn_engine* e, TailArgs& t, const ScaleW& sw, void* out_grad, void* out_terms, void* out_total,
                      bool adam, bool multi) {
  memset(&t, 0, sizeof t);
  t.state = e->d_state; t.out_grad = out_grad; t.out_terms = out_terms; t.out_total = out_total;
  if (adam) {
    t.adam_theta = e->d_theta; t.adam_m = e->adam_m; t.adam_v = e->adam_v;
    t.adam_lr = e->adam_lr; t.adam_b1 = e->adam_b1; t.adam_b2 = e->adam_b2; t.adam_eps = e->adam_eps;
    t.bump_draw = any_sampler(e) ? 1 : 0;
  }
  t.timeout_ns = e->tail_timeout_ns;
  t.nranks = multi ? e->nranks : 1; t.rank = multi ? e->rank : 0;
  t.recv_words = e->recv_words;
#ifdef PINN_DEBUG
  t.dbg = e->tail_dbg;
#endif
  if (multi)
    for (int r = 0; r < e->nranks; ++r) t.peer_recv[r] = e->peer_base[r];
  t.sw = sw;
}

// One evaluation of the hot path on stream st: fused kernel + tail and whatever follows it on this configuration.
//   single GPU, or peer memory mapped:  ONE launch (tail reduces, sums over the peers, writes / applies Adam)
//   multi-GPU without peer memory:      fused kernel (tail reduces into `packed`) -> ncclAllReduce -> finish_kernel
int pinn::eval_step(pinn_engine* e, const void* theta, const double* host_weights, void* out_grad, void* out_terms,
                     void* out_total, bool adam, cudaStream_t st) {
  const bool want_grad = adam || out_grad != nullptr;
  LaunchCall c = {};
  c.theta = theta; c.tile_end = e->total_tiles; c.mode = want_grad ? 0 : 1;
  ScaleW sw = {};
  if (prepare_scales(e, host_weights, c.seed, sw)) return 1;
  const bool multi = e->nranks > 1;
  int grid = std::min(e->num_sms, e->total_tiles);
  if (multi && e->p2p) grid = e->num_sms;       // the same slice partition of theta on every rank
  if (grid < 1) grid = 1;                       // a rank whose shard is empty still takes part in the reduction
  if (grid > kTailSlots) return fail("pinn_loss_grad: %d CTAs exceed the %d tail slots", grid, kTailSlots);
  if (e->timing) CUDA_TRY(cudaEventRecord(e->ev0, st));
  const long long ng = want_grad ? e->n_theta : 0;
  const bool nccl = multi && !e->p2p;
  if (!nccl) {
    fill_tail(e, c.tail, sw, out_grad, out_terms, out_total, adam, multi);
  } else {
    if (adam)
      return fail("pinn_adam_iterate: the multi-GPU device loop needs the peer-memory allreduce (%s)",
                  e->p2p_why[0] ? e->p2p_why : "not available");
    void* pk_terms = (char*)e->packed + (size_t)ng * e->es;
    fill_tail(e, c.tail, sw, want_grad ? e->packed : nullptr, pk_terms, nullptr, false, false);
  }
  if (launch_fused(e, c, grid, st)) return 1;
  if (e->timing) CUDA_TRY(cudaEventRecord(e->ev1, st));
  e->launches += 1;
  if (nccl) {
    // packed = [grad (n_theta, zero-length when no gradient is wanted) | term losses]: one allreduce
    ncclResult_t r = g_nccl.AllReduce(e->packed, e->packed, (size_t)ng + (size_t)e->n_terms,
                                      e->dtype == PINN_F64 ? ncclFloat64 : ncclFloat32, ncclSumOp, e->comm, st);
    if (r != 0) return fail("ncclAllReduce failed: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?");
    e->launches += 1;
    CUDA_TRY(finish_launch(e->dtype, e->packed, ng, e->n_terms, sw, out_grad, out_terms, out_total, st));
    e->launches += 1;
  }
  if (e->timing) {
    CUDA_TRY(cudaEventSynchronize(e->ev1));
    CUDA_TRY(cudaEventElapsedTime(&e->last_ms, e->ev0, e->ev1));
  }
  return 0;
}

extern "C" {

int pinn_loss_grad(pinn_handle e, const void* dev_theta, const double* host_weights, void* dev_grad,
                   void* dev_term_losses, void* dev_total, void* stream) {
  if (!e) return fail("pinn_loss_grad: null handle");
  if (!dev_theta || !dev_term_losses || !dev_total) return fail("pinn_loss_grad: null theta/term_losses/total");
  CUDA_TRY(cudaSetDevice(e->device));
  for (int t = 0; t < e->n_terms; ++t)
    if (e->dyn[t].n <= 0 && !(e->nranks > 1 && (e->term[t].n_global_set || t == e->plan.prob.func_term)))
      return fail("pinn_loss_grad: term %d has no points (call pinn_set_points first)", t);
  if (e->total_tiles <= 0 && e->nranks <= 1) return fail("pinn_loss_grad: no collocation points");
  return eval_step(e, dev_theta, host_weights, dev_grad, dev_term_losses, dev_total, false, (cudaStream_t)stream);
}

int pinn_loss_grad_host(pinn_handle e, const void* host_theta, const double* host_weights, void* host_grad,
                        void* host_term_losses, void* host_total) {
  if (!e) return fail("pinn_loss_grad_host: null handle");
  if (!host_theta || !host_total) return fail("pinn_loss_grad_host: null theta/total");
  CUDA_TRY(cudaSetDevice(e->device));
  cudaStream_t st = e->own_stream;
  const size_t tb = (size_t)e->n_theta * e->es;
  memcpy(e->h_pin_in, host_theta, tb);
  CUDA_TRY(cudaMemcpyAsync(e->d_theta, e->h_pin_in, tb, cudaMemcpyHostToDevice, st));
  char* hout = (char*)e->h_pin_out;
  if (e->zero_copy_out && (e->nranks <= 1 || e->p2p)) {
    // the kernel tail writes the gradient and the losses straight into the pinned host buffer (mapped into the device
    // address space): no device-to-host copies after the launch, just the stream synchronisation
    if (pinn_loss_grad(e, e->d_theta, host_weights, host_grad ? (void*)hout : nullptr, hout + tb,
                       hout + tb + (size_t)e->n_terms * e->es, st))
      return 1;
  } else {
    char* dout = (char*)e->d_out;
    if (pinn_loss_grad(e, e->d_theta, host_weights, host_grad ? e->d_grad : nullptr, dout,
                       dout + (size_t)e->n_terms * e->es, st))
      return 1;
    if (host_grad) CUDA_TRY(cudaMemcpyAsync(hout, e->d_grad, tb, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(hout + tb, e->d_out, ((size_t)e->n_terms + 1) * e->es, cudaMemcpyDeviceToHost, st));
  }
  CUDA_TRY(cudaStreamSynchronize(st));
  if (host_grad) memcpy(host_grad, hout, tb);
  if (host_term_losses) memcpy(host_term_losses, hout + tb, (size_t)e->n_terms * e->es);
  memcpy(host_total, hout + tb + (size_t)e->n_terms * e->es, e->es);
  return 0;
}

int pinn_adam_begin(pinn_handle e, const void* host_theta0, double lr, double beta1, double beta2, double eps) {
  if (!e) return fail("pinn_adam_begin: null handle");
  if (!host_theta0) return fail("pinn_adam_begin: null theta");
  CUDA_TRY(cudaSetDevice(e->device));
  const size_t tb = (size_t)e->n_theta * e->es;
  if (!e->adam_m) { if (dev_alloc(&e->adam_m, tb, e) || dev_alloc(&e->adam_v, tb, e)) return 1; }
  CUDA_TRY(cudaMemsetAsync(e->adam_m, 0, tb, e->own_stream));
  CUDA_TRY(cudaMemsetAsync(e->adam_v, 0, tb, e->own_stream));
  CUDA_TRY(cudaMemsetAsync(&e->d_state->adam_t, 0, sizeof(unsigned long long), e->own_stream));
  CUDA_TRY(cudaMemcpyAsync(e->d_theta, host_theta0, tb, cudaMemcpyHostToDevice, e->own_stream));
  CUDA_TRY(cudaStreamSynchronize(e->own_stream));
  e->adam_lr = lr; e->adam_b1 = beta1; e->adam_b2 = beta2; e->adam_eps = eps; e->adam_ready = true;
  return 0;
}

// one iteration of the device-resident loop: fresh points for the sampled terms, then the fused step with Adam in its tail
static int enqueue_adam_iteration(pinn_engine* e, const double* host_weights, cudaStream_t st) {
  char* dout = (char*)e->d_out;
  // draw = host counter + 1 + device counter; the tail advances the device counter, so graph replays resample
  for (int t = 0; t < e->n_terms; ++t)
    if (e->term[t].sampler_on && draw_term(e, t, e->sampler_draw + 1, &e->d_state->draw, st)) return 1;
  return eval_step(e, e->d_theta, host_weights, nullptr, dout, dout + (size_t)e->n_terms * e->es, true, st);
}

static unsigned long long fnv1a(const void* p, size_t n, unsigned long long h) {
  const unsigned char* b = (const unsigned char*)p;
  for (size_t i = 0; i < n; ++i) { h ^= b[i]; h *= 1099511628211ull; }
  return h;
}

int pinn_adam_iterate(pinn_handle e, int32_t n_steps, const double* host_weights, void* host_total, void* host_term_losses) {
  if (!e) return fail("pinn_adam_iterate: null handle");
  if (!e->adam_ready) return fail("pinn_adam_iterate: call pinn_adam_begin first");
  if (n_steps < 1) return fail("pinn_adam_iterate: n_steps must be >= 1");
  CUDA_TRY(cudaSetDevice(e->device));
  if (e->total_tiles <= 0 && e->nranks <= 1) return fail("pinn_adam_iterate: no collocation points");
  cudaStream_t st = e->own_stream;
  const char* ng = getenv("PINN_B200_NO_GRAPH");
  const bool use_graph = (e->nranks <= 1 || e->p2p) && !e->timing && !(ng && ng[0] == '1');
  if (use_graph) {
    // the n_steps iterations are captured once into a CUDA graph (sampler draws + ONE fused launch per iteration) and
    // replayed while the launch arguments stay the same: step counter, bias correction and draw counter live on the device
    unsigned long long key = 1469598103934665603ull;
    key = fnv1a(&n_steps, sizeof n_steps, key);
    double w[PINN_MAX_TERMS];
    for (int t = 0; t < PINN_MAX_TERMS; ++t) w[t] = (host_weights && t < e->n_terms) ? host_weights[t] : 1.0;
    key = fnv1a(w, sizeof w, key);
    key = fnv1a(e->dyn, sizeof e->dyn, key);
    for (const TermState& ts : e->term) key = fnv1a(&ts.n_global, sizeof ts.n_global, key);
    const double hp[4] = {e->adam_lr, e->adam_b1, e->adam_b2, e->adam_eps};
    key = fnv1a(hp, sizeof hp, key);
    key = fnv1a(&e->sampler_draw, sizeof e->sampler_draw, key);
    if (!e->adam_graph || e->adam_graph_key != key) {
      if (e->adam_graph) { cudaGraphExecDestroy(e->adam_graph); e->adam_graph = nullptr; }
      cudaGraph_t g = nullptr;
      CUDA_TRY(cudaStreamBeginCapture(st, cudaStreamCaptureModeRelaxed));
      int rc = 0;
      const long long l0 = e->launches;
      for (int it = 0; it < n_steps && !rc; ++it) rc = enqueue_adam_iteration(e, host_weights, st);
      cudaError_t ce = cudaStreamEndCapture(st, &g);
      e->launches = l0;
      if (rc) { if (g) cudaGraphDestroy(g); return 1; }
      if (ce != cudaSuccess) return fail("pinn_adam_iterate: graph capture failed: %s", cudaGetErrorString(ce));
      ce = cudaGraphInstantiate(&e->adam_graph, g, 0);
      cudaGraphDestroy(g);
      if (ce != cudaSuccess) { e->adam_graph = nullptr; return fail("pinn_adam_iterate: graph instantiation failed: %s", cudaGetErrorString(ce)); }
      e->adam_graph_key = key;
    }
    CUDA_TRY(cudaGraphLaunch(e->adam_graph, st));
    long long per_it = 1 + (e->plan.wide ? 1 : 0);
    for (int t = 0; t < e->n_terms; ++t) per_it += e->term[t].sampler_on ? 1 : 0;
    e->launches += per_it * n_steps;
  } else {
    for (int it = 0; it < n_steps; ++it)
      if (enqueue_adam_iteration(e, host_weights, st)) return 1;
  }
  char* hout = (char*)e->h_pin_out;
  CUDA_TRY(cudaMemcpyAsync(hout, e->d_out, ((size_t)e->n_terms + 1) * e->es, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  if (host_term_losses) memcpy(host_term_losses, hout, (size_t)e->n_terms * e->es);
  if (host_total) memcpy(host_total, hout + (size_t)e->n_terms * e->es, e->es);
  return 0;
}

int pinn_adam_theta(pinn_handle e, void* host_theta_out) {
  if (!e || !host_theta_out) return fail("pinn_adam_theta: null handle / output");
  if (!e->adam_ready) return fail("pinn_adam_theta: call pinn_adam_begin first");
  CUDA_TRY(cudaSetDevice(e->device));
  CUDA_TRY(cudaMemcpyAsync(host_theta_out, e->d_theta, (size_t)e->n_theta * e->es, cudaMemcpyDeviceToHost, e->own_stream));
  CUDA_TRY(cudaStreamSynchronize(e->own_stream));
  return 0;
}

int pinn_term_residual(pinn_handle e, int32_t term, const void* dev_theta, void* dev_r, void* stream) {
  if (check_term(e, term, "pinn_term_residual")) return 1;
  if (!dev_theta || !dev_r) return fail("pinn_term_residual: null theta/output");
  if (e->dyn[term].n <= 0) return fail("pinn_term_residual: term %d has no points", term);
  CUDA_TRY(cudaSetDevice(e->device));
  LaunchCall c = {};
  c.theta = dev_theta; c.mode = 2; c.resid_out = dev_r;
  c.tile_begin = e->dyn[term].tile0;
  c.tile_end = e->dyn[term].tile0 + e->dyn[term].n_tiles;
  const int grid = std::min(e->num_sms, e->dyn[term].n_tiles);
  if (launch_fused(e, c, grid, (cudaStream_t)stream)) return 1;
  e->launches += 1;
  return 0;
}

int pinn_term_residual_host(pinn_handle e, int32_t term, const void* host_theta, void* host_r) {
  if (check_term(e, term, "pinn_term_residual_host")) return 1;
  if (!host_theta || !host_r) return fail("pinn_term_residual_host: null theta/output");
  CUDA_TRY(cudaSetDevice(e->device));
  cudaStream_t st = e->own_stream;
  const size_t tb = (size_t)e->n_theta * e->es;
  CUDA_TRY(cudaMemcpyAsync(e->d_theta, host_theta, tb, cudaMemcpyHostToDevice, st));
  void* dr = nullptr;
  size_t rb = (size_t)e->dyn[term].n * e->es;
  CUDA_TRY(cudaMalloc(&dr, rb ? rb : 16));
  int rc = pinn_term_residual(e, term, e->d_theta, dr, st);
  if (!rc) {
    cudaError_t err = cudaMemcpyAsync(host_r, dr, rb, cudaMemcpyDeviceToHost, st);
    if (err == cudaSuccess) err = cudaStreamSynchronize(st);
    if (err != cudaSuccess) rc = fail("pinn_term_residual_host: %s", cudaGetErrorString(err));
  }
  cudaFree(dr);
  return rc;
}

}  // extern "C"

// effective draw index = draw + *draw_dev (the device counter is advanced by the tail of the device-resident loop)
int pinn::draw_term(pinn_engine* e, int term, unsigned long long draw, const unsigned long long* draw_dev, cudaStream_t st) {
  const int dim = e->plan.prob.terms[term].dim;
  TermState& ts = e->term[term];
  const long long n = ts.sampler_n;
  if (grow(&ts.own_pts, &ts.own_pts_cap, (size_t)n * dim * e->es, e)) return 1;
  const unsigned long long key = ts.sampler_seed + 0x9E3779B97F4A7C15ull * (unsigned long long)(term + 1);
  if (ts.sampler_kind == PINN_SAMPLER_KKL)   // keyed on the seed alone: the KKL terms of one seed share their draw
    CUDA_TRY(sample_kkl_launch(e->dtype, ts.own_pts, ts.kkl_times, ts.kkl_sub, dim - 1, ts.sampler_lb[0], ts.sampler_ub[0],
                               (ts.kkl_flags & PINN_KKL_STRONG) != 0, ts.sampler_seed ^ 0xD6E8FEB86659FD93ull, draw,
                               draw_dev, st));
  else if (ts.sampler_kind == PINN_SAMPLER_LHS)
    CUDA_TRY(sample_lhs_launch(e->dtype, ts.own_pts, n, dim, ts.sampler_lb, ts.sampler_ub, key, draw, draw_dev, st));
  else
    CUDA_TRY(sample_uniform_launch(e->dtype, ts.own_pts, n, dim, ts.sampler_lb, ts.sampler_ub, key, draw, draw_dev, st));
  e->launches += 1;
  e->dyn[term].pts = ts.own_pts; e->dyn[term].qw = nullptr; e->dyn[term].n = n;
  return 0;
}

extern "C" {

int pinn_set_sampler_ex(pinn_handle e, int32_t term, int32_t kind, int64_t n, const double* host_lb, const double* host_ub,
                        uint64_t seed, void* stream) {
  if (check_term(e, term, "pinn_set_sampler")) return 1;
  if (kind != PINN_SAMPLER_UNIFORM && kind != PINN_SAMPLER_LHS) return fail("pinn_set_sampler: unknown sampler kind %d", kind);
  if (n > 0x7fffffffLL) return fail("pinn_set_sampler: at most 2^31 - 1 points per term");
  if (n < 1) return fail("pinn_set_sampler: term %d needs at least one point", term);
  if (!host_lb || !host_ub) return fail("pinn_set_sampler: null bounds");
  if (e->plan.term[term].reduction == PINN_REDUCE_WSUM)
    return fail("pinn_set_sampler: term %d is a weighted-sum (quadrature) term; the uniform sampler serves mean(abs2) terms", term);
  if (term == e->plan.prob.func_term)
    return fail("pinn_set_sampler: term %d is a functional term; its nodes are fixed (pinn_set_points)", term);
  CUDA_TRY(cudaSetDevice(e->device));
  const int dim = e->plan.prob.terms[term].dim;
  TermState& ts = e->term[term];
  for (int r = 0; r < dim; ++r) {
    if (!(host_lb[r] <= host_ub[r])) return fail("pinn_set_sampler: term %d row %d has lb > ub", term, r);
    ts.sampler_lb[r] = host_lb[r]; ts.sampler_ub[r] = host_ub[r];
  }
  ts.sampler_on = true; ts.sampler_kind = kind; ts.sampler_seed = seed; ts.sampler_n = n;
  if (draw_term(e, term, e->sampler_draw, &e->d_state->draw, (cudaStream_t)stream)) return 1;
  retile(e);
  return 0;
}

int pinn_set_sampler_kkl(pinn_handle e, int32_t term, int64_t n_times, int32_t sub_batch, int32_t n_z, double t_lb,
                         double t_ub, uint32_t flags, uint64_t seed, void* stream) {
  if (check_term(e, term, "pinn_set_sampler_kkl")) return 1;
  if (n_times < 1 || sub_batch < 1)
    return fail("pinn_set_sampler_kkl: term %d needs at least one time and one sample (n_times=%lld, sub_batch=%d)", term,
                (long long)n_times, sub_batch);
  if (n_times * (long long)sub_batch > 0x7fffffffLL)
    return fail("pinn_set_sampler_kkl: at most 2^31 - 1 points per term (n_times * sub_batch)");
  if (n_z < 0 || 1 + n_z != e->plan.prob.terms[term].dim)
    return fail("pinn_set_sampler_kkl: term %d has %d point rows; the KKL sampler fills 1 + n_z = %d (t, z_1..z_n_z)", term,
                e->plan.prob.terms[term].dim, 1 + n_z);
  if (flags & ~(uint32_t)PINN_KKL_STRONG) return fail("pinn_set_sampler_kkl: unknown flags 0x%x", flags);
  if (!(t_lb <= t_ub)) return fail("pinn_set_sampler_kkl: term %d has t_lb > t_ub", term);
  if (e->plan.term[term].reduction == PINN_REDUCE_WSUM)
    return fail("pinn_set_sampler_kkl: term %d is a weighted-sum (quadrature) term; the KKL sampler serves mean(abs2) terms", term);
  if (term == e->plan.prob.func_term)
    return fail("pinn_set_sampler_kkl: term %d is a functional term; its nodes are fixed (pinn_set_points)", term);
  CUDA_TRY(cudaSetDevice(e->device));
  TermState& ts = e->term[term];
  ts.sampler_lb[0] = t_lb; ts.sampler_ub[0] = t_ub;
  ts.kkl_times = n_times; ts.kkl_sub = sub_batch; ts.kkl_flags = (int)flags;
  ts.sampler_on = true; ts.sampler_kind = PINN_SAMPLER_KKL; ts.sampler_seed = seed; ts.sampler_n = n_times * sub_batch;
  if (draw_term(e, term, e->sampler_draw, &e->d_state->draw, (cudaStream_t)stream)) return 1;
  retile(e);
  return 0;
}

int pinn_set_sampler(pinn_handle e, int32_t term, int64_t n, const double* host_lb, const double* host_ub, uint64_t seed,
                     void* stream) {
  return pinn_set_sampler_ex(e, term, PINN_SAMPLER_UNIFORM, n, host_lb, host_ub, seed, stream);
}

int pinn_resample(pinn_handle e, void* stream) {
  if (!e) return fail("pinn_resample: null handle");
  CUDA_TRY(cudaSetDevice(e->device));
  e->sampler_draw += 1;
  for (int t = 0; t < e->n_terms; ++t)
    if (e->term[t].sampler_on && draw_term(e, t, e->sampler_draw, &e->d_state->draw, (cudaStream_t)stream)) return 1;
  retile(e);
  return 0;
}

int pinn_get_points_host(pinn_handle e, int32_t term, void* host_pts) {
  if (check_term(e, term, "pinn_get_points_host")) return 1;
  if (!host_pts) return fail("pinn_get_points_host: null output");
  CUDA_TRY(cudaSetDevice(e->device));
  const size_t bytes = (size_t)e->dyn[term].n * e->plan.prob.terms[term].dim * e->es;
  CUDA_TRY(cudaDeviceSynchronize());
  if (bytes) CUDA_TRY(cudaMemcpy(host_pts, e->dyn[term].pts, bytes, cudaMemcpyDeviceToHost));
  return 0;
}

int pinn_term_grad_stats(pinn_handle e, int32_t term, const void* dev_theta, double* host_max_abs, double* host_mean_abs,
                         void* stream) {
  if (check_term(e, term, "pinn_term_grad_stats")) return 1;
  if (!dev_theta || !host_max_abs || !host_mean_abs) return fail("pinn_term_grad_stats: null theta/output");
  if (term == e->plan.prob.func_term)
    return fail("pinn_term_grad_stats: term %d is a functional term; its gradient is not a per-term loss gradient of the "
                "adaptive reweighting", term);
  CUDA_TRY(cudaSetDevice(e->device));
  cudaStream_t st = (cudaStream_t)stream;
  double w[PINN_MAX_TERMS];
  for (int t = 0; t < PINN_MAX_TERMS; ++t) w[t] = (t == term) ? 1.0 : 0.0;
  char* dout = (char*)e->d_out;
  // gradient of the single unweighted term loss L_term (other terms enter with weight 0)
  if (pinn_loss_grad(e, dev_theta, w, e->d_grad, dout, dout + (size_t)e->n_terms * e->es, st)) return 1;
  double* dstats = (double*)e->packed;       // >= 16 bytes, free after pinn_loss_grad returned its results
  CUDA_TRY(grad_stats_launch(e->dtype, e->d_grad, e->n_theta, dstats, st));
  e->launches += 1;
  double hs[2];
  CUDA_TRY(cudaMemcpyAsync(hs, dstats, sizeof hs, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  *host_max_abs = hs[0];
  *host_mean_abs = hs[1];
  return 0;
}

int pinn_term_grad_stats_host(pinn_handle e, int32_t term, const void* host_theta, double* host_max_abs,
                              double* host_mean_abs) {
  if (check_term(e, term, "pinn_term_grad_stats_host")) return 1;
  if (!host_theta) return fail("pinn_term_grad_stats_host: null theta");
  CUDA_TRY(cudaSetDevice(e->device));
  CUDA_TRY(cudaMemcpyAsync(e->d_theta, host_theta, (size_t)e->n_theta * e->es, cudaMemcpyHostToDevice, e->own_stream));
  return pinn_term_grad_stats(e, term, e->d_theta, host_max_abs, host_mean_abs, e->own_stream);
}

int pinn_comm_unique_id(void* out) {
  if (!out) return fail("pinn_comm_unique_id: null output");
  if (!load_nccl()) return fail("pinn_comm_unique_id: libnccl.so.2 could not be loaded: %s", dlerror());
  ncclUniqueId id;
  ncclResult_t r = g_nccl.GetUniqueId(&id);
  if (r != 0) return fail("ncclGetUniqueId failed: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?");
  memcpy(out, &id, sizeof id);
  return 0;
}

// Map every rank's receive region ([2 parities][nranks][n_theta words + term words] slots of {32-bit word, step flag})
// into this process so the fused kernel's tail can push its reduced gradient slices straight into the peers' memory over
// NVLink and add what the peers pushed (tail.cuh).  Every rank runs the same two
// collectives (handle allgather, agreement allreduce) whatever its local outcome; on any failure all ranks fall back to
// ncclAllReduce together and p2p_why says why.
struct PeerRec {
  cudaIpcMemHandle_t handle;
  char bus[32];
  int ok;
  int pad;
};

static int setup_p2p(pinn_engine* e) {
  e->p2p = false;
  int ok = 1;
  auto why = [&](const char* msg) { if (!e->p2p_why[0]) snprintf(e->p2p_why, sizeof e->p2p_why, "%s", msg); ok = 0; };
  if (!g_nccl.AllGather) { why("ncclAllGather not found"); return 0; }        // same library on every rank: uniform exit
  const char* no = getenv("PINN_B200_NO_P2P");
  if (no && no[0] == '1') why("disabled by PINN_B200_NO_P2P=1");
  if (e->nranks > kMaxRanks) why("more ranks than one NVSwitch domain (8)");
  if (e->num_sms > kTailSlots) why("more SMs than tail slots");
  e->recv_words = e->n_theta * (long long)(e->es / 4) + 2 * PINN_MAX_TERMS;
  const size_t total = (size_t)2 * (size_t)e->nranks * (size_t)e->recv_words * 8;
  PeerRec mine;
  memset(&mine, 0, sizeof mine);
  if (ok) {
    if (cudaMalloc(&e->sym, total) != cudaSuccess) { e->sym = nullptr; why("cudaMalloc of the symmetric region failed"); }
    else {
      e->ws_bytes += (long long)total;
      if (cudaMemset(e->sym, 0, total) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) why("symmetric region init failed");
      else if (cudaIpcGetMemHandle(&mine.handle, e->sym) != cudaSuccess) why("cudaIpcGetMemHandle failed");
      else if (cudaDeviceGetPCIBusId(mine.bus, sizeof mine.bus, e->device) != cudaSuccess) why("cudaDeviceGetPCIBusId failed");
    }
    cudaGetLastError();
  }
  mine.ok = ok;
  PeerRec* d_recs = nullptr;
  std::vector<PeerRec> recs((size_t)e->nranks);
  CUDA_TRY(cudaMalloc((void**)&d_recs, sizeof(PeerRec) * e->nranks));
  CUDA_TRY(cudaMemcpy(d_recs + e->rank, &mine, sizeof mine, cudaMemcpyHostToDevice));
  ncclResult_t r = g_nccl.AllGather(d_recs + e->rank, d_recs, sizeof(PeerRec), ncclInt8, e->comm, (cudaStream_t)0);
  if (r != 0) { cudaFree(d_recs); return fail("ncclAllGather failed: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?"); }
  CUDA_TRY(cudaStreamSynchronize((cudaStream_t)0));
  CUDA_TRY(cudaMemcpy(recs.data(), d_recs, sizeof(PeerRec) * e->nranks, cudaMemcpyDeviceToHost));
  for (int q = 0; q < e->nranks; ++q) if (!recs[q].ok) why("a peer rank could not export its symmetric region");
  if (ok) {
    for (int q = 0; q < e->nranks && ok; ++q) {
      if (q == e->rank) { e->peer_base[q] = e->sym; continue; }
      int pdev = -1, can = 0;
      if (cudaDeviceGetByPCIBusId(&pdev, recs[q].bus) != cudaSuccess) { why("a peer GPU is not visible to this process"); break; }
      if (cudaDeviceCanAccessPeer(&can, e->device, pdev) != cudaSuccess || !can) { why("no peer access between the GPUs"); break; }
      void* ptr = nullptr;
      if (cudaIpcOpenMemHandle(&ptr, recs[q].handle, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
        why("cudaIpcOpenMemHandle failed (ranks in one process, or IPC unavailable)");
        break;
      }
      e->peer_base[q] = ptr;
    }
    cudaGetLastError();
  }
  // agreement: the peer path is used only if every rank mapped every peer
  int* d_ok = (int*)d_recs;
  CUDA_TRY(cudaMemcpy(d_ok, &ok, sizeof(int), cudaMemcpyHostToDevice));
  r = g_nccl.AllReduce(d_ok, d_ok, 1, ncclInt32, ncclMinOp, e->comm, (cudaStream_t)0);
  if (r != 0) { cudaFree(d_recs); return fail("ncclAllReduce failed: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?"); }
  CUDA_TRY(cudaStreamSynchronize((cudaStream_t)0));
  int all_ok = 0;
  CUDA_TRY(cudaMemcpy(&all_ok, d_ok, sizeof(int), cudaMemcpyDeviceToHost));
  cudaFree(d_recs);
  if (!all_ok && ok) why("a peer rank could not map the symmetric regions");
  if (!all_ok) {
    for (int q = 0; q < e->nranks; ++q)
      if (q != e->rank && e->peer_base[q]) { cudaIpcCloseMemHandle(e->peer_base[q]); }
    memset(e->peer_base, 0, sizeof e->peer_base);
    cudaGetLastError();
    return 0;
  }
  e->p2p = true;
  return 0;
}

int pinn_comm_init(pinn_handle e, const void* uid, int32_t rank, int32_t nranks) {
  if (!e) return fail("pinn_comm_init: null handle");
  if (!uid) return fail("pinn_comm_init: null unique id");
  if (nranks < 1 || rank < 0 || rank >= nranks) return fail("pinn_comm_init: bad rank %d / nranks %d", rank, nranks);
  if (e->comm) return fail("pinn_comm_init: the handle already has a communicator");
  if (!load_nccl()) return fail("pinn_comm_init: libnccl.so.2 could not be loaded: %s", dlerror());
  CUDA_TRY(cudaSetDevice(e->device));
  ncclUniqueId id;
  memcpy(&id, uid, sizeof id);
  ncclResult_t r = g_nccl.CommInitRank(&e->comm, nranks, id, rank);
  if (r != 0) return fail("ncclCommInitRank failed: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?");
  e->rank = rank; e->nranks = nranks;
  if (nranks > 1 && setup_p2p(e)) return 1;
  return 0;
}

// which gradient-sum path pinn_loss_grad uses at nranks > 1: *fused_p2p = 1 when the sum runs inside the fused kernel over
// peer memory, 0 when it falls back to ncclAllReduce (reason, if any, in the returned string; valid until the next call)
const char* pinn_comm_info(pinn_handle e, int32_t* fused_p2p) {
  if (fused_p2p) *fused_p2p = (e && e->p2p) ? 1 : 0;
  return e ? e->p2p_why : "";
}

#ifdef PINN_DEBUG
// diagnostic (not part of the drop-in ABI): enable phase timestamps of CTA 0 in the tensor-core kernel and
// read them back (2000 x int64: [0,1000) phase marks id << 48 | clock, [1000,2000) per-CTA
// {globaltimer start, end, cycles, smid}); host_out == NULL only enables.
int pinn_debug_tc_timeline(pinn_handle e, long long* host_out) {
  if (!e) return fail("pinn_debug_tc_timeline: null handle");
  CUDA_TRY(cudaSetDevice(e->device));
  if (!e->tc_dbg) {
    CUDA_TRY(cudaMalloc((void**)&e->tc_dbg, 2000 * sizeof(long long)));
    CUDA_TRY(cudaMemset(e->tc_dbg, 0, 2000 * sizeof(long long)));
    e->plan.tc.dbg = e->plan.tw.dbg = e->tc_dbg;
  }
  if (host_out) {
    CUDA_TRY(cudaDeviceSynchronize());
    CUDA_TRY(cudaMemcpy(host_out, e->tc_dbg, 2000 * sizeof(long long), cudaMemcpyDeviceToHost));
  }
  return 0;
}

// diagnostic: enable (host_out == NULL) / read back the tail's per-CTA globaltimer marks of the last launch:
// kTailSlots x {tail entry, grid barrier passed, slice reduced (+ pushed), peers' slices added}
extern "C" int pinn_debug_tail_marks(pinn_handle e, long long* host_out) {
  if (!e) return fail("pinn_debug_tail_marks: null handle");
  CUDA_TRY(cudaSetDevice(e->device));
  if (!e->tail_dbg) {
    CUDA_TRY(cudaMalloc((void**)&e->tail_dbg, kTailSlots * 4 * sizeof(long long)));
    CUDA_TRY(cudaMemset(e->tail_dbg, 0, kTailSlots * 4 * sizeof(long long)));
  }
  if (host_out) {
    CUDA_TRY(cudaDeviceSynchronize());
    CUDA_TRY(cudaMemcpy(host_out, e->tail_dbg, kTailSlots * 4 * sizeof(long long), cudaMemcpyDeviceToHost));
  }
  return 0;
}
#endif

int64_t pinn_launch_count(pinn_handle e) { return e ? e->launches : 0; }
int pinn_set_timing(pinn_handle e, int32_t enable) {
  if (!e) return fail("pinn_set_timing: null handle");
  e->timing = enable != 0;
  return 0;
}
double pinn_last_kernel_ms(pinn_handle e) { return e ? (double)e->last_ms : 0.0; }
int64_t pinn_workspace_bytes(pinn_handle e) { return e ? e->ws_bytes : 0; }
double pinn_flops_per_eval(pinn_handle e) {
  if (!e) return 0.0;
  double f = 0;
  for (int t = 0; t < e->n_terms; ++t) f += e->plan.term[t].flops_per_point * (double)e->dyn[t].n;
  return f;
}

}  // extern "C"
