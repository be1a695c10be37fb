// pinn_abi.cu -- host side of the C ABI declared in include/pinn_b200.h: descriptor
// validation and lowering to the device representation, workspace ownership, kernel
// launch sequencing, host-buffer staging and the optional NCCL gradient allreduce.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <stdarg.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "dev_types.h"
#include "tc_types.h"

namespace pinn {
size_t ffma_smem_bytes(int dtype, long long buf_elems, int w_area, bool bufs_smem);
cudaError_t ffma_launch(int dtype, bool bufs_smem, const FfmaArgs& a, int grid, size_t smem, cudaStream_t st);
cudaError_t grad_stats_launch(int dtype, const void* grad, long long n, double* out2, cudaStream_t st);
cudaError_t sample_uniform_launch(int dtype, void* pts, long long n, int dim, const double* lb, const double* ub,
                                  unsigned long long seed, unsigned long long draw, const unsigned long long* draw_dev,
                                  cudaStream_t st);
cudaError_t sample_lhs_launch(int dtype, void* pts, long long n, int dim, const double* lb, const double* ub,
                              unsigned long long seed, unsigned long long draw, const unsigned long long* draw_dev,
                              cudaStream_t st);
cudaError_t finish_launch(int dtype, const void* packed, long long n_grad, int n_terms, const ScaleW& scale_w, void* out_grad,
                          void* out_terms, void* out_total, cudaStream_t st);
}  // namespace pinn

using namespace pinn;

// ---- minimal NCCL binding (resolved at run time so single-GPU use has no dependency) ----
typedef struct ncclComm* ncclComm_t;
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

static thread_local std::string g_err;
static int fail(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_err = buf;
  return 1;
}
#define CUDA_TRY(expr)                                                                  \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess) return fail("%s failed: %s", #expr, cudaGetErrorString(_e)); \
  } while (0)

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

struct pinn_engine {
  int dtype = 0, mode = 0, device = 0;
  size_t es = 4;
  DevProblem* hprob = nullptr;   // host copy (heap: ~250 KB)
  DevProblem* dprob = nullptr;   // device copy
  int n_terms = 0;
  long long n_theta = 0, partial_stride = 0;
  double term_scale[PINN_MAX_TERMS];     // WSUM scale (MEAN: 1/n_global at launch time)
  int reduction[PINN_MAX_TERMS];
  long long n_global[PINN_MAX_TERMS];
  bool n_global_set[PINN_MAX_TERMS];
  double flops_per_point[PINN_MAX_TERMS];
  TermDyn dyn[PINN_MAX_TERMS];
  int total_tiles = 0;
  // launch geometry
  int num_sms = 0;
  size_t smem = 0;
  bool bufs_smem = true;
  int weights_resident = 0;
  int w_area = 0, ldc = 0;
  long long buf_elems = 0, stash_per_cta = 0;
  // tensor-core path geometry
  int tile_pts = kTilePts;
  // (tc_off_P / _misc / _ones, tc_mx_*, tc_stash_per_cta and tc_net_ak serve both tensor-core kernels)
  int tc_split = 0, tc_tl_max = 0, tc_off_P = 0, tc_off_Q = 0, tc_off_misc = 0, tc_off_ones = 0, tc_mx_dim = 1, tc_mx_taps = 1;
  int tc_net_ak[PINN_MAX_NETS];  // 1: every hidden activation of the network is tanh (fast path), 0: generic
  TcNetSmem tc_nets[PINN_MAX_NETS];
  long long tc_stash_per_cta = 0;
  long long* tc_dbg = nullptr;   // device buffer for pinn_debug_tc_timeline
  long long* tail_dbg = nullptr; // device buffer for pinn_debug_tail_marks (PINN_DEBUG builds)
  // wide tensor path (128-wide layers): streamed weights, fp32 pre-activation stash
  bool tw = false;
  int tw_off_S = 0, tw_off_nets = 0, tw_off_fp[PINN_MAX_NETS], tw_wimg[PINN_MAX_NETS];
  int tw_n_images = 0;
  unsigned char tw_img_net[kTwMaxImages], tw_img_layer[kTwMaxImages];
  long long tw_zstash_per_cta = 0;
  void* tw_wpack = nullptr;
  int* tw_counter = nullptr;
  void* tw_zstash = nullptr;
  float* tc_acc = nullptr;       // tensor-core paths: per-CTA fp32 accumulator regions (tc_prims.cuh)
  // workspaces (device)
  void* partial = nullptr;
  double* term_sums = nullptr;
  void* stash = nullptr;
  void* gbufs = nullptr;
  void* packed = nullptr;        // [n_theta + n_terms] allreduce buffer
  long long ws_bytes = 0;
  // engine-owned point copies
  void* own_pts[PINN_MAX_TERMS];
  size_t own_pts_cap[PINN_MAX_TERMS];
  void* own_qw[PINN_MAX_TERMS];
  size_t own_qw_cap[PINN_MAX_TERMS];
  // host staging for the *_host entry points
  void* d_theta = nullptr;
  void* d_grad = nullptr;
  void* d_out = nullptr;         // [n_terms + 1] term losses then total
  void* h_pin_in = nullptr;      // pinned theta
  void* h_pin_out = nullptr;     // pinned grad + losses
  cudaStream_t own_stream = nullptr;
  bool zero_copy_out = false;    // h_pin_out is addressable from the device (kernel tail writes results to the host directly)
  // device-resident Adam state
  void* adam_m = nullptr;
  void* adam_v = nullptr;
  double adam_lr = 1e-3, adam_b1 = 0.9, adam_b2 = 0.999, adam_eps = 1e-8;
  bool adam_ready = false;
  // device-side samplers (StochasticTraining): per term box, seed, point count; draw counter shared by all terms
  bool sampler_on[PINN_MAX_TERMS];
  int sampler_kind[PINN_MAX_TERMS];
  double sampler_lb[PINN_MAX_TERMS][PINN_MAX_DIM], sampler_ub[PINN_MAX_TERMS][PINN_MAX_DIM];
  unsigned long long sampler_seed[PINN_MAX_TERMS];
  long long sampler_n[PINN_MAX_TERMS];
  unsigned long long sampler_draw = 0;
  // fused kernel tail (tail.cuh): device-resident barrier / step state
  TailState* d_state = nullptr;
  unsigned long long tail_timeout_ns = 20ull * 1000000000ull;
  // captured iteration graph of the device-resident Adam loop
  cudaGraphExec_t adam_graph = nullptr;
  int adam_graph_n = 0;
  unsigned long long adam_graph_key = 0;
  // comm
  ncclComm_t comm = nullptr;
  int rank = 0, nranks = 1;
  // peer-memory allreduce (NVLink): receive region [2 parities][nranks][recv_words] of 8-byte {word, flag} slots,
  // mapped from every rank
  bool p2p = false;
  void* sym = nullptr;
  long long recv_words = 0;
  void* peer_base[kMaxRanks];
  char p2p_why[160];
  // introspection
  long long launches = 0;
  bool timing = false;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  float last_ms = 0.f;
};

static int dev_alloc(void** p, size_t bytes, pinn_engine* e) {
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
    e->dyn[t].n_tiles = (int)((e->dyn[t].n + e->tile_pts - 1) / e->tile_pts);
    t0 += e->dyn[t].n_tiles;
  }
  e->total_tiles = t0;
}

// ---- descriptor validation + lowering -----------------------------------------------------------
static int lower_problem(const pinn_problem_desc* d, pinn_engine* e) {
  if (!d) return fail("pinn_create: null descriptor");
  if (d->abi_version != PINN_ABI_VERSION)
    return fail("pinn_create: descriptor abi_version %d, library %d", d->abi_version, PINN_ABI_VERSION);
  if (d->dtype != PINN_F32 && d->dtype != PINN_F64) return fail("pinn_create: unknown dtype %d", d->dtype);
  if (d->mode < PINN_MODE_FFMA || d->mode > PINN_MODE_TC_SPLIT) return fail("pinn_create: unknown mode %d", d->mode);
  if (d->n_nets < 1 || d->n_nets > PINN_MAX_NETS) return fail("pinn_create: n_nets=%d out of range [1,%d]", d->n_nets, PINN_MAX_NETS);
  if (d->n_terms < 1 || d->n_terms > PINN_MAX_TERMS)
    return fail("pinn_create: n_terms=%d out of range [1,%d]", d->n_terms, PINN_MAX_TERMS);
  if (d->n_params < 0 || d->n_params > PINN_MAX_PARAMS)
    return fail("pinn_create: n_params=%d out of range [0,%d]", d->n_params, PINN_MAX_PARAMS);
  if (!d->nets || !d->terms) return fail("pinn_create: null nets/terms");
  if (d->n_theta <= 0) return fail("pinn_create: n_theta must be positive");

  DevProblem& P = *e->hprob;
  memset(&P, 0, sizeof(DevProblem));
  P.n_nets = d->n_nets; P.n_terms = d->n_terms; P.n_params = d->n_params;
  P.param_off = d->param_offset; P.n_theta = d->n_theta;
  if (d->n_params > 0 && (d->param_offset < 0 || d->param_offset + d->n_params > d->n_theta))
    return fail("pinn_create: theta.p block [%lld,+%d) outside theta (n_theta=%lld)", (long long)d->param_offset,
                d->n_params, (long long)d->n_theta);

  int max_w8 = 8;
  long long resident = 0;
  for (int k = 0; k < d->n_nets; ++k) {
    const pinn_net_desc& nd = d->nets[k];
    DevNet& n = P.nets[k];
    if (nd.n_layers < 1 || nd.n_layers > PINN_MAX_LAYERS)
      return fail("pinn_create: net %d has %d layers (supported 1..%d)", k, nd.n_layers, PINN_MAX_LAYERS);
    if (!nd.dims || !nd.acts) return fail("pinn_create: net %d null dims/acts", k);
    n.n_layers = nd.n_layers;
    long long off = nd.theta_offset;
    if (off < 0) return fail("pinn_create: net %d negative theta_offset", k);
    for (int l = 0; l <= nd.n_layers; ++l) {
      if (nd.dims[l] < 1) return fail("pinn_create: net %d dims[%d]=%d must be >= 1", k, l, nd.dims[l]);
      n.dims[l] = nd.dims[l];
      max_w8 = std::max(max_w8, (nd.dims[l] + 7) & ~7);
    }
    if (n.dims[0] > PINN_MAX_IN) return fail("pinn_create: net %d input dimension %d > %d", k, n.dims[0], PINN_MAX_IN);
    for (int l = 0; l < nd.n_layers; ++l) {
      if (nd.acts[l] < PINN_ACT_IDENTITY || nd.acts[l] > PINN_ACT_SWISH)
        return fail("pinn_create: net %d layer %d unknown activation %d", k, l, nd.acts[l]);
      n.acts[l] = nd.acts[l];
      n.w_off[l] = off; off += (long long)n.dims[l] * n.dims[l + 1];
      n.b_off[l] = off; off += n.dims[l + 1];
      int in8 = (n.dims[l] + 7) & ~7, out8 = (n.dims[l + 1] + 7) & ~7;
      n.ws_off[l] = (int)resident; resident += (long long)in8 * out8;
      n.bs_off[l] = (int)resident; resident += out8;
    }
    if (off > d->n_theta)
      return fail("pinn_create: net %d parameters [%lld,%lld) exceed n_theta=%lld", k, (long long)nd.theta_offset, off,
                  (long long)d->n_theta);
    n.max_width8 = max_w8;
  }

  int maxC = 1;
  long long stash_max = 0;
  for (int t = 0; t < d->n_terms; ++t) {
    const pinn_term_desc& td = d->terms[t];
    DevTerm& T = P.terms[t];
    if (td.dim < 1 || td.dim > PINN_MAX_DIM) return fail("pinn_create: term %d dim=%d out of range [1,%d]", t, td.dim, PINN_MAX_DIM);
    if (td.n_taps < 1)
      return fail("pinn_create: term %d has no network taps (an equation such as 0 ~ 0 cannot be trained on)", t);
    if (td.n_taps > PINN_MAX_TAPS) return fail("pinn_create: term %d has %d taps (max %d)", t, td.n_taps, PINN_MAX_TAPS);
    if (td.n_instr < 1 || td.n_instr > PINN_MAX_INSTR)
      return fail("pinn_create: term %d program length %d out of range [1,%d]", t, td.n_instr, PINN_MAX_INSTR);
    if (!td.taps || !td.prog || !td.net_rows) return fail("pinn_create: term %d null taps/prog/net_rows", t);
    if (td.reduction != PINN_REDUCE_MEAN && td.reduction != PINN_REDUCE_WSUM)
      return fail("pinn_create: term %d unknown reduction %d", t, td.reduction);
    T.dim = td.dim; T.n_taps = td.n_taps; T.n_instr = td.n_instr;
    T.weighted = td.reduction == PINN_REDUCE_WSUM;
    e->reduction[t] = td.reduction;
    e->term_scale[t] = td.reduction == PINN_REDUCE_WSUM ? td.scale : 1.0;

    // slots: networks in order of first use
    int slot_of[PINN_MAX_NETS];
    for (int k = 0; k < PINN_MAX_NETS; ++k) slot_of[k] = -1;
    T.n_used = 0;
    for (int i = 0; i < td.n_taps; ++i) {
      const pinn_tap_desc& tp = td.taps[i];
      if (tp.net < 0 || tp.net >= d->n_nets) return fail("pinn_create: term %d tap %d names network %d", t, i, tp.net);
      if (slot_of[tp.net] < 0) {
        slot_of[tp.net] = T.n_used;
        T.used_net[T.n_used] = tp.net;
        DevChan& ch = T.chan[T.n_used];
        ch.C = 1; ch.n1 = 0; ch.n2 = 0; ch.n3 = 0;
        const int din = P.nets[tp.net].dims[0];
        for (int j = 0; j < din; ++j) {
          int r = td.net_rows[tp.net * PINN_MAX_IN + j];
          if (r < 0 || r >= td.dim)
            return fail("pinn_create: term %d network %d input %d maps to point row %d (dim=%d)", t, tp.net, j, r, td.dim);
          ch.rows[j] = r;
        }
        ++T.n_used;
      }
    }
    // channels
    for (int pass = 1; pass <= 2; ++pass) {
      for (int i = 0; i < td.n_taps; ++i) {
        const pinn_tap_desc& tp = td.taps[i];
        const int din = P.nets[tp.net].dims[0];
        DevChan& ch = T.chan[slot_of[tp.net]];
        if (tp.order < 0 || tp.order > 3)
          return fail("pinn_create: term %d tap %d has derivative order %d; orders 0..3 are supported (order 4 and mixed "
                      "third derivatives are not)", t, i, tp.order);
        if (tp.order == 3 && !(tp.dir[0] == tp.dir[1] && tp.dir[1] == tp.dir[2]))
          return fail("pinn_create: term %d tap %d is a mixed third derivative; only pure third derivatives d^3/dx_i^3 are "
                      "supported", t, i);
        if (tp.out < 0 || tp.out >= P.nets[tp.net].dims[P.nets[tp.net].n_layers])
          return fail("pinn_create: term %d tap %d output component %d out of range", t, i, tp.out);
        for (int q = 0; q < tp.order; ++q)
          if (tp.dir[q] < 0 || tp.dir[q] >= din)
            return fail("pinn_create: term %d tap %d direction %d out of range for a %d-input network", t, i, tp.dir[q], din);
        if (pass == 1) {
          // first-derivative channels needed directly or as intermediates of second derivatives
          for (int q = 0; q < tp.order; ++q) {
            int found = -1;
            for (int j = 0; j < ch.n1; ++j) if (ch.dir1[j] == tp.dir[q]) found = j;
            if (found < 0) ch.dir1[ch.n1++] = tp.dir[q];
          }
        } else if (tp.order >= 2) {
          // order 3 (pure) needs the pure second derivative along the same direction as an intermediate
          int a = -1, b = -1;
          for (int j = 0; j < ch.n1; ++j) { if (ch.dir1[j] == tp.dir[0]) a = j; if (ch.dir1[j] == tp.dir[1]) b = j; }
          if (a > b) std::swap(a, b);
          int found = -1;
          for (int s = 0; s < ch.n2; ++s) if (ch.s_a[s] == a && ch.s_b[s] == b) found = s;
          if (found < 0) {
            if (1 + ch.n1 + ch.n2 + ch.n3 >= PINN_MAX_CH)
              return fail("pinn_create: term %d network %d needs more than %d channels", t, tp.net, PINN_MAX_CH);
            ch.s_a[ch.n2] = a; ch.s_b[ch.n2] = b; ++ch.n2;
          }
          if (tp.order == 3) {
            int ft = -1;
            for (int q = 0; q < ch.n3; ++q) if (ch.t_a[q] == a) ft = q;
            if (ft < 0) {
              if (1 + ch.n1 + ch.n2 + ch.n3 >= PINN_MAX_CH)
                return fail("pinn_create: term %d network %d needs more than %d channels", t, tp.net, PINN_MAX_CH);
              ch.t_a[ch.n3++] = a;
            }
          }
        }
      }
    }
    // canonical channel order: directions that carry a pure second derivative come first, so that
    // (when every second-derivative channel is pure) channel n1+1+s is d2/d(dir1[s])^2
    for (int s = 0; s < T.n_used; ++s) {
      DevChan& ch = T.chan[s];
      int order[PINN_MAX_IN], inv[PINN_MAX_IN], n = 0;
      bool used[PINN_MAX_IN] = {false};
      for (int q = 0; q < ch.n2; ++q)
        if (ch.s_a[q] == ch.s_b[q] && !used[ch.s_a[q]]) { order[n++] = ch.s_a[q]; used[ch.s_a[q]] = true; }
      const int npure = n;
      for (int j = 0; j < ch.n1; ++j) if (!used[j]) order[n++] = j;
      int nd[PINN_MAX_IN];
      for (int i = 0; i < ch.n1; ++i) { nd[i] = ch.dir1[order[i]]; inv[order[i]] = i; }
      for (int i = 0; i < ch.n1; ++i) ch.dir1[i] = nd[i];
      for (int q = 0; q < ch.n2; ++q) {
        int a = inv[ch.s_a[q]], b = inv[ch.s_b[q]];
        if (a > b) std::swap(a, b);
        ch.s_a[q] = a; ch.s_b[q] = b;
      }
      ch.pure = (npure == ch.n2) ? 1 : 0;
      if (ch.pure) for (int q = 0; q < ch.n2; ++q) ch.s_a[q] = ch.s_b[q] = q;
      for (int q = 0; q < ch.n3; ++q) {
        ch.t_a[q] = inv[ch.t_a[q]];
        ch.t_s[q] = -1;
        for (int q2 = 0; q2 < ch.n2; ++q2) if (ch.s_a[q2] == ch.t_a[q] && ch.s_b[q2] == ch.t_a[q]) ch.t_s[q] = q2;
      }
    }
    long long stash = 0;
    for (int s = 0; s < T.n_used; ++s) {
      DevChan& ch = T.chan[s];
      ch.C = 1 + ch.n1 + ch.n2 + ch.n3;
      if (ch.C > PINN_MAX_CH) return fail("pinn_create: term %d needs %d channels (max %d)", t, ch.C, PINN_MAX_CH);
      maxC = std::max(maxC, ch.C);
      const DevNet& n = P.nets[T.used_net[s]];
      for (int l = 0; l < n.n_layers; ++l) {
        ch.stash_off[l] = (int)stash;
        stash += (long long)ch.C * n.dims[l + 1] * kTilePts;
      }
    }
    stash_max = std::max(stash_max, stash);
    // tap -> (slot, channel)
    for (int i = 0; i < td.n_taps; ++i) {
      const pinn_tap_desc& tp = td.taps[i];
      const DevChan& ch = T.chan[slot_of[tp.net]];
      T.tap_slot[i] = slot_of[tp.net];
      T.tap_out[i] = tp.out;
      if (tp.order == 0) T.tap_ch[i] = 0;
      else if (tp.order == 1) {
        int j = 0; while (ch.dir1[j] != tp.dir[0]) ++j;
        T.tap_ch[i] = 1 + j;
      } else if (tp.order == 2) {
        int a = -1, b = -1;
        for (int j = 0; j < ch.n1; ++j) { if (ch.dir1[j] == tp.dir[0]) a = j; if (ch.dir1[j] == tp.dir[1]) b = j; }
        if (a > b) std::swap(a, b);
        int s = 0; while (!(ch.s_a[s] == a && ch.s_b[s] == b)) ++s;
        T.tap_ch[i] = 1 + ch.n1 + s;
      } else {
        int a = 0; while (ch.dir1[a] != tp.dir[0]) ++a;
        int q = 0; while (ch.t_a[q] != a) ++q;
        T.tap_ch[i] = 1 + ch.n1 + ch.n2 + q;
      }
    }
    // program
    bool any_tap = false;
    for (int i = 0; i < td.n_instr; ++i) {
      const pinn_instr& in = td.prog[i];
      DevInstr& o = T.prog[i];
      o.op = in.op; o.a = in.a; o.b = in.b; o.pad = 0; o.imm = in.imm;
      auto val_ok = [&](int v) { return v >= 0 && v < i; };
      switch (in.op) {
        case PINN_OP_CONST: break;
        case PINN_OP_COORD:
          if (in.a < 0 || in.a >= td.dim) return fail("pinn_create: term %d instr %d COORD row %d out of range", t, i, in.a);
          break;
        case PINN_OP_TAP:
          if (in.a < 0 || in.a >= td.n_taps) return fail("pinn_create: term %d instr %d TAP %d out of range", t, i, in.a);
          any_tap = true;
          break;
        case PINN_OP_PARAM:
          if (in.a < 0 || in.a >= d->n_params) return fail("pinn_create: term %d instr %d PARAM %d out of range", t, i, in.a);
          break;
        case PINN_OP_ADD: case PINN_OP_SUB: case PINN_OP_MUL: case PINN_OP_DIV: case PINN_OP_POW:
          if (!val_ok(in.a) || !val_ok(in.b)) return fail("pinn_create: term %d instr %d operand out of range", t, i);
          break;
        case PINN_OP_NEG: case PINN_OP_POWI: case PINN_OP_SIN: case PINN_OP_COS: case PINN_OP_EXP:
        case PINN_OP_LOG: case PINN_OP_TANH: case PINN_OP_SQRT: case PINN_OP_ABS:
          if (!val_ok(in.a)) return fail("pinn_create: term %d instr %d operand out of range", t, i);
          break;
        default:
          return fail("pinn_create: term %d instr %d unknown opcode %d", t, i, in.op);
      }
    }
    if (!any_tap)
      return fail("pinn_create: term %d residual program never reads a tap (nothing depends on theta)", t);
    // algorithmic flops per point: 6 * sum_nets C * S
    double f = 0;
    for (int s = 0; s < T.n_used; ++s) {
      const DevNet& n = P.nets[T.used_net[s]];
      double S = 0;
      for (int l = 0; l < n.n_layers; ++l) S += (double)n.dims[l] * n.dims[l + 1];
      f += 6.0 * T.chan[s].C * S;
    }
    e->flops_per_point[t] = f;
  }

  // ---- launch geometry -------------------------------------------------------------------------
  const int TP = kTilePts + (int)(16 / e->es);
  e->ldc = max_w8 * TP;
  e->buf_elems = (long long)maxC * e->ldc;
  e->stash_per_cta = (stash_max + 3) & ~3LL;
  const long long panel = (long long)(kWarps * 8) * max_w8 + kWarps * 8;   // 64 x max_width8 (+ bias)
  int max_smem = 0;
  cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, e->device);
  if (max_smem <= 0) max_smem = 227 * 1024;
  struct Opt { bool bufs; bool res; };
  const Opt opts[3] = {{true, true}, {true, false}, {false, false}};
  bool chosen = false;
  for (const Opt& o : opts) {
    long long wa = o.res ? resident : panel;
    wa = (wa + 3) & ~3LL;
    if (wa > (1LL << 30)) continue;
    size_t need = ffma_smem_bytes(e->dtype, e->buf_elems, (int)wa, o.bufs);
    if (need <= (size_t)max_smem) {
      e->bufs_smem = o.bufs; e->weights_resident = o.res ? 1 : 0; e->w_area = (int)wa; e->smem = need;
      chosen = true;
      break;
    }
  }
  if (d->mode == PINN_MODE_FFMA) {
    if (!chosen)
      return fail("pinn_create: a %d-wide layer panel does not fit in shared memory (%d bytes)", max_w8, max_smem);
    return 0;
  }

  // ---- tensor-core path: supported-shape check and shared-memory plan -----------------------------------
  if (d->dtype != PINN_F32) return fail("pinn_create: the tensor-core modes compute in bf16/fp32 and need dtype PINN_F32");
  for (int t = 0; t < d->n_terms; ++t)
    for (int s2 = 0; s2 < P.terms[t].n_used; ++s2)
      if (P.terms[t].chan[s2].n3 > 0)
        return fail("pinn_create(tc): term %d takes a third derivative; the tensor-core path propagates derivatives up to order 2 "
                    "(use PINN_MODE_FFMA)", t);
  e->tc_split = d->mode == PINN_MODE_TC_SPLIT ? 1 : 0;
  e->tile_pts = kTcPts;
  int tl_max = 0;
  bool wide = false;
  for (int k = 0; k < PINN_MAX_NETS; ++k) e->tc_net_ak[k] = 1;
  for (int k = 0; k < d->n_nets; ++k) {
    const DevNet& n = P.nets[k];
    for (int l = 0; l + 1 < n.n_layers; ++l)
      if (n.acts[l] != PINN_ACT_TANH) e->tc_net_ak[k] = 0;
    if (n.n_layers < 2) return fail("pinn_create(tc): net %d needs at least 2 Dense layers", k);
    if (n.dims[n.n_layers] != 1) return fail("pinn_create(tc): net %d must have a 1-dimensional output", k);
    if (n.acts[n.n_layers - 1] != PINN_ACT_IDENTITY)
      return fail("pinn_create(tc): net %d: the last layer must be linear (identity activation)", k);
    for (int l = 1; l < n.n_layers; ++l)
      if (n.dims[l] > 64) wide = true;
    if (n.n_layers - 2 > kTcMaxTL)
      return fail("pinn_create(tc): net %d has %d hidden->hidden layers (max %d)", k, n.n_layers - 2, kTcMaxTL);
    tl_max = std::max(tl_max, n.n_layers - 2);
  }
  for (int k = 0; k < d->n_nets; ++k) {
    const DevNet& n = P.nets[k];
    for (int l = 1; l < n.n_layers; ++l) {
      const int w = n.dims[l];
      if (!wide && (w % 16 != 0 || w < 16 || w > 64))
        return fail("pinn_create(tc): net %d hidden width %d unsupported by the tensor-core path (16, 32, 48, 64, or 64/128 "
                    "with PINN_MODE_TC_BF16; use PINN_MODE_FFMA for other shapes)", k, w);
      if (wide && w != 64 && w != 128)
        return fail("pinn_create(tc): net %d hidden width %d: networks with layers wider than 64 need every hidden width "
                    "to be 64 or 128 on the tensor-core path (use PINN_MODE_FFMA for other shapes)", k, w);
    }
    if (wide && n.n_layers < 3)
      return fail("pinn_create(tc): net %d: the 128-wide tensor-core path needs at least one hidden->hidden layer", k);
  }
  if (wide && d->mode != PINN_MODE_TC_BF16)
    return fail("pinn_create(tc): PINN_MODE_TC_SPLIT supports hidden widths up to 64; 128-wide layers run in "
                "PINN_MODE_TC_BF16 (or PINN_MODE_FFMA for fp32 accuracy)");
  e->tw = wide;
  if (wide) {
    // A network that needs more than kTwMaxC channels is evaluated in several passes ("slots") over the same weights,
    // each with the value channel and a subset of the derivative directions (first-fit over the directions, a
    // direction with a pure second derivative costs 2 channels).  The passes recompute the value channel; the
    // gradient contributions add up in the per-CTA partial.
    for (int t = 0; t < d->n_terms; ++t) {
      DevTerm& T = P.terms[t];
      bool need = false;
      for (int s2 = 0; s2 < T.n_used; ++s2) need = need || T.chan[s2].C > kTwMaxC;
      if (!need) continue;
      int n_new = 0, new_net[PINN_MAX_NETS], first_new[PINN_MAX_NETS];
      DevChan nch[PINN_MAX_NETS];
      int dir_slot[PINN_MAX_NETS][PINN_MAX_IN], dir_pos[PINN_MAX_NETS][PINN_MAX_IN];
      for (int s2 = 0; s2 < T.n_used; ++s2) {
        const DevChan& ch = T.chan[s2];
        first_new[s2] = n_new;
        if (ch.C <= kTwMaxC) {
          if (n_new >= PINN_MAX_NETS) return fail("pinn_create(tc): term %d needs more than %d network passes", t, PINN_MAX_NETS);
          for (int j = 0; j < ch.n1; ++j) { dir_slot[s2][j] = n_new; dir_pos[s2][j] = j; }
          new_net[n_new] = T.used_net[s2]; nch[n_new] = ch; ++n_new;
          continue;
        }
        if (!ch.pure)
          return fail("pinn_create(tc): term %d needs %d channels including mixed second derivatives; the 128-wide tensor-core "
                      "path splits only pure second derivatives into passes (use PINN_MODE_FFMA)", t, ch.C);
        bool placed[PINN_MAX_IN] = {false};
        int left = ch.n1;
        while (left > 0) {
          if (n_new >= PINN_MAX_NETS) return fail("pinn_create(tc): term %d needs more than %d network passes", t, PINN_MAX_NETS);
          DevChan g;
          memset(&g, 0, sizeof g);
          for (int j = 0; j < PINN_MAX_IN; ++j) g.rows[j] = ch.rows[j];
          int cost = 0;
          for (int j = 0; j < ch.n1; ++j) {          // pure directions (cost 2) come first in the canonical order
            const int cj = 1 + (j < ch.n2 ? 1 : 0);
            if (placed[j] || cost + cj > kTwMaxC - 1) continue;
            placed[j] = true; --left; cost += cj;
            dir_slot[s2][j] = n_new; dir_pos[s2][j] = g.n1;
            g.dir1[g.n1++] = ch.dir1[j];
            if (j < ch.n2) ++g.n2;
          }
          for (int q2 = 0; q2 < g.n2; ++q2) g.s_a[q2] = g.s_b[q2] = q2;
          g.pure = 1; g.C = 1 + g.n1 + g.n2;
          new_net[n_new] = T.used_net[s2]; nch[n_new] = g; ++n_new;
        }
      }
      for (int i = 0; i < T.n_taps; ++i) {
        const int os = T.tap_slot[i], tch = T.tap_ch[i];
        const DevChan& ch = T.chan[os];
        if (tch == 0) { T.tap_slot[i] = first_new[os]; T.tap_ch[i] = 0; }
        else if (tch <= ch.n1) { T.tap_slot[i] = dir_slot[os][tch - 1]; T.tap_ch[i] = 1 + dir_pos[os][tch - 1]; }
        else {
          const int q2 = tch - 1 - ch.n1;          // pure: second-derivative channel q2 belongs to direction q2
          const int ns = dir_slot[os][q2];
          T.tap_slot[i] = ns; T.tap_ch[i] = 1 + nch[ns].n1 + dir_pos[os][q2];
        }
      }
      T.n_used = n_new;
      for (int s2 = 0; s2 < n_new; ++s2) { T.used_net[s2] = new_net[s2]; T.chan[s2] = nch[s2]; }
    }
  }
  int n_used_max = 1;
  for (int t = 0; t < d->n_terms; ++t) {
    const DevTerm& T = P.terms[t];
    if (T.n_taps > kTcMaxTaps) return fail("pinn_create(tc): term %d has %d taps (tensor-core path: max %d)", t, T.n_taps, kTcMaxTaps);
    n_used_max = std::max(n_used_max, T.n_used);
    for (int s2 = 0; s2 < T.n_used; ++s2) {
      const DevChan& ch = T.chan[s2];
      const int key = ch.n1 * 8 + ch.n2;
      const int ok[] = {0, 8, 16, 24, 32, 9, 17, 25, 18};
      bool found = false;
      for (int v : ok) found = found || v == key;
      if (wide && (ch.C > kTwMaxC || key == 32))
        return fail("pinn_create(tc): term %d needs %d channels on a 128-wide network; the tensor-core path propagates at most "
                    "%d there (use PINN_MODE_FFMA)", t, ch.C, kTwMaxC);
      if (!found || ch.C > kTcMaxC)
        return fail("pinn_create(tc): term %d needs %d first + %d second derivative channels; the tensor-core path "
                    "propagates at most %d channels per network (use PINN_MODE_FFMA)", t, ch.n1, ch.n2, kTcMaxC);
    }
    for (int i = 0; i < T.n_taps; ++i)
      if (T.tap_out[i] != 0) return fail("pinn_create(tc): term %d tap %d: output component must be 0", t, i);
  }
  e->tc_tl_max = tl_max;
  e->tc_mx_dim = 1; e->tc_mx_taps = 1;
  for (int t = 0; t < d->n_terms; ++t) {
    e->tc_mx_dim = std::max(e->tc_mx_dim, (int)P.terms[t].dim);
    e->tc_mx_taps = std::max(e->tc_mx_taps, (int)P.terms[t].n_taps);
  }
  if (wide) {
    int maxCw = 1;
    for (int t = 0; t < d->n_terms; ++t)
      for (int s2 = 0; s2 < P.terms[t].n_used; ++s2) maxCw = std::max(maxCw, (int)P.terms[t].chan[s2].C);
    size_t o2 = 0;
    e->tc_off_P = (int)o2; o2 += (size_t)maxCw * kTwNB * kTileBytes;
    e->tw_off_S = (int)o2; o2 += (size_t)2 * kTwImgBytes;
    e->tc_off_ones = (int)o2; o2 += 1024;
    e->tw_n_images = 0;
    for (int k = 0; k < PINN_MAX_NETS; ++k) { e->tw_off_fp[k] = -1; e->tw_wimg[k] = 0; }
    for (int k = 0; k < d->n_nets; ++k) {
      e->tw_off_fp[k] = (int)o2;
      o2 += ((size_t)FpBlock<kTwW>::SIZE * 4 + 15) & ~size_t(15);
      e->tw_wimg[k] = e->tw_n_images;
      for (int l = 1; l <= P.nets[k].n_layers - 2; ++l) {
        e->tw_img_net[e->tw_n_images] = (unsigned char)k;
        e->tw_img_layer[e->tw_n_images] = (unsigned char)l;
        ++e->tw_n_images;
      }
    }
    e->tw_off_nets = (int)o2;
    o2 += ((size_t)d->n_nets * sizeof(DevNet) + 15) & ~size_t(15);
    e->tc_off_misc = (int)o2;
    o2 += tc_misc_bytes(e->tc_mx_dim, e->tc_mx_taps);
    if (o2 + 1024 > (size_t)max_smem)
      return fail("pinn_create(tc): the problem needs %zu bytes of shared memory per CTA (limit %d): too many networks "
                  "for the 128-wide tensor-core path", o2, max_smem);
    e->smem = o2;
    // per pass: inputs of the tl_max tensor layers + the last hidden activations (restored for multi-pass terms)
    e->tc_stash_per_cta = (long long)n_used_max * (tl_max + 1) * kTwMaxC * kTwNB * kTileBytes;
    e->tw_zstash_per_cta = (long long)n_used_max * tl_max * kTwMaxC * 64 * kTcPts * 2;      // floats
    return 0;
  }
  size_t off = 0;
  e->tc_off_P = (int)off; off += (size_t)maxC * kTileBytes;
  e->tc_off_Q = (int)off; off += (size_t)maxC * kTileBytes;
  for (int k = 0; k < PINN_MAX_NETS; ++k) {
    e->tc_nets[k].fp = -1;
    for (int l = 0; l < kTcMaxTL; ++l) e->tc_nets[k].w_hi[l] = e->tc_nets[k].w_lo[l] = 0;
  }
  for (int k = 0; k < d->n_nets; ++k) {
    const int TL = P.nets[k].n_layers - 2;
    for (int l = 0; l < TL; ++l) {
      e->tc_nets[k].w_hi[l] = (int)off; off += 8192;
      if (e->tc_split) { e->tc_nets[k].w_lo[l] = (int)off; off += 8192; }
      else e->tc_nets[k].w_lo[l] = e->tc_nets[k].w_hi[l];
    }
  }
  e->tc_off_ones = (int)off; off += 1024;      // 1024-aligned: P, Q and the weight tiles are multiples of 8 KB
  for (int k = 0; k < d->n_nets; ++k) {
    e->tc_nets[k].fp = (int)off;
    off += ((size_t)FpBlock<kTcW>::SIZE * 4 + 15) & ~size_t(15);
  }
  e->tc_off_misc = (int)off;
  off += tc_misc_bytes(e->tc_mx_dim, e->tc_mx_taps);
  if (off + 1024 > (size_t)max_smem)   // + the kernel's static shared memory
    return fail("pinn_create(tc): the problem needs %zu bytes of shared memory per CTA (limit %d): too many "
                "resident weight tiles / channels for the tensor-core path", off, max_smem);
  e->smem = off;
  e->tc_stash_per_cta = (long long)n_used_max * std::max(tl_max, 1) * kTcMaxC * kTileBytes;
  return 0;
}

extern "C" {

const char* pinn_last_error(void) { return g_err.c_str(); }
int pinn_abi_version(void) { return PINN_ABI_VERSION; }

int pinn_destroy(pinn_handle e) {
  if (!e) return 0;
  cudaSetDevice(e->device);
  if (e->adam_graph) cudaGraphExecDestroy(e->adam_graph);
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
  for (int t = 0; t < PINN_MAX_TERMS; ++t) {
    if (e->own_pts[t]) cudaFree(e->own_pts[t]);
    if (e->own_qw[t]) cudaFree(e->own_qw[t]);
  }
  if (e->h_pin_in) cudaFreeHost(e->h_pin_in);
  if (e->h_pin_out) cudaFreeHost(e->h_pin_out);
  if (e->own_stream) cudaStreamDestroy(e->own_stream);
  if (e->ev0) cudaEventDestroy(e->ev0);
  if (e->ev1) cudaEventDestroy(e->ev1);
  delete e->hprob;
  delete e;
  return 0;
}

int pinn_create(const pinn_problem_desc* d, pinn_handle* out) {
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
  memset(e->own_pts, 0, sizeof e->own_pts); memset(e->own_qw, 0, sizeof e->own_qw);
  memset(e->own_pts_cap, 0, sizeof e->own_pts_cap); memset(e->own_qw_cap, 0, sizeof e->own_qw_cap);
  memset(e->dyn, 0, sizeof e->dyn); memset(e->n_global_set, 0, sizeof e->n_global_set);
  memset(e->n_global, 0, sizeof e->n_global);
  memset(e->sampler_on, 0, sizeof e->sampler_on);
  memset(e->sampler_kind, 0, sizeof e->sampler_kind);
  memset(e->peer_base, 0, sizeof e->peer_base);
  e->p2p_why[0] = 0;
  e->hprob = new DevProblem();
  e->dtype = d->dtype; e->mode = d->mode; e->device = d->device;
  e->es = d->dtype == PINN_F64 ? 8 : 4;
  e->n_terms = d->n_terms; e->n_theta = d->n_theta;
  if (lower_problem(d, e)) { pinn_destroy(e); return 1; }
  cudaDeviceGetAttribute(&e->num_sms, cudaDevAttrMultiProcessorCount, e->device);
  if (e->num_sms <= 0) e->num_sms = 132;

#define TRY_OR_DESTROY(x) do { if (x) { pinn_destroy(e); return 1; } } while (0)
  TRY_OR_DESTROY(dev_alloc((void**)&e->dprob, sizeof(DevProblem), e));
  cudaError_t err = cudaMemcpy(e->dprob, e->hprob, sizeof(DevProblem), cudaMemcpyHostToDevice);
  if (err != cudaSuccess) { fail("pinn_create: upload failed: %s", cudaGetErrorString(err)); pinn_destroy(e); return 1; }
  const size_t g = (size_t)e->num_sms;
  e->partial_stride = (e->n_theta + 3) & ~3LL;
  TRY_OR_DESTROY(dev_alloc(&e->partial, g * (size_t)e->partial_stride * e->es, e));
  TRY_OR_DESTROY(dev_alloc((void**)&e->term_sums, g * PINN_MAX_TERMS * sizeof(double), e));
  if (e->mode == PINN_MODE_FFMA) {
    TRY_OR_DESTROY(dev_alloc(&e->stash, g * (size_t)e->stash_per_cta * e->es, e));
    if (!e->bufs_smem) TRY_OR_DESTROY(dev_alloc(&e->gbufs, g * 2 * (size_t)e->buf_elems * e->es, e));
  } else {
    TRY_OR_DESTROY(dev_alloc(&e->stash, g * (size_t)e->tc_stash_per_cta, e));
    TRY_OR_DESTROY(dev_alloc((void**)&e->tc_acc, g * (size_t)kAccCols * kAccRows * sizeof(float), e));
    if (e->tw) {
      TRY_OR_DESTROY(dev_alloc(&e->tw_zstash, g * (size_t)e->tw_zstash_per_cta * sizeof(float), e));
      TRY_OR_DESTROY(dev_alloc(&e->tw_wpack, (size_t)std::max(e->tw_n_images, 1) * kTwImgBytes, e));
      TRY_OR_DESTROY(dev_alloc((void**)&e->tw_counter, 64, e));
    }
  }
  TRY_OR_DESTROY(dev_alloc(&e->packed, ((size_t)e->n_theta + PINN_MAX_TERMS) * e->es, e));
  TRY_OR_DESTROY(dev_alloc((void**)&e->d_state, sizeof(TailState), e));
  err = cudaMemset(e->d_state, 0, sizeof(TailState));
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
  retile(e);
  *out = e;
  return 0;
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
  if (e->reduction[term] == PINN_REDUCE_WSUM && n > 0 && !dev_w)
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
  if (e->reduction[term] == PINN_REDUCE_WSUM && n > 0 && !host_w)
    return fail("pinn_set_points_host: term %d is a weighted-sum (quadrature) term and needs weights", term);
  CUDA_TRY(cudaSetDevice(e->device));
  const int dim = e->hprob->terms[term].dim;
  cudaStream_t st = (cudaStream_t)stream;
  size_t bytes = (size_t)n * dim * e->es;
  if (grow(&e->own_pts[term], &e->own_pts_cap[term], bytes, e)) return 1;
  if (bytes) CUDA_TRY(cudaMemcpyAsync(e->own_pts[term], host_pts, bytes, cudaMemcpyHostToDevice, st));
  const void* w = nullptr;
  if (host_w) {
    size_t wb = (size_t)n * e->es;
    if (grow(&e->own_qw[term], &e->own_qw_cap[term], wb, e)) return 1;
    if (wb) CUDA_TRY(cudaMemcpyAsync(e->own_qw[term], host_w, wb, cudaMemcpyHostToDevice, st));
    w = e->own_qw[term];
  }
  e->dyn[term].pts = e->own_pts[term]; e->dyn[term].qw = w; e->dyn[term].n = n;
  retile(e);
  return 0;
}

int pinn_set_global_count(pinn_handle e, int32_t term, int64_t n_global) {
  if (check_term(e, term, "pinn_set_global_count")) return 1;
  if (n_global <= 0) return fail("pinn_set_global_count: n_global must be positive");
  e->n_global[term] = n_global; e->n_global_set[term] = true;
  return 0;
}

// scale_k (so that L_k = scale_k * sum_p qw r^2) and the loss weights w_k
static int prepare_scales(pinn_engine* e, const double* host_weights, FfmaArgs& a, ScaleW& sw) {
  for (int t = 0; t < e->n_terms; ++t) {
    double sc;
    if (e->reduction[t] == PINN_REDUCE_MEAN) {
      long long ng = e->n_global_set[t] ? e->n_global[t] : e->dyn[t].n;
      if (ng <= 0) return fail("pinn_loss_grad: term %d has no points (pinn_set_points was not called or n == 0)", t);
      sc = 1.0 / (double)ng;
    } else {
      sc = e->term_scale[t];
    }
    double w = host_weights ? host_weights[t] : 1.0;
    sw.scale[t] = sc;
    sw.w[t] = w;
    a.seed[t] = sc * w;
  }
  return 0;
}

static void fill_args(pinn_engine* e, FfmaArgs& a, const void* theta, int mode) {
  a.prob = e->dprob; a.theta = theta; a.partial = e->partial; a.partial_stride = e->partial_stride; a.term_sums = e->term_sums; a.stash = e->stash;
  a.gbufs = e->gbufs; a.stash_per_cta = e->stash_per_cta; a.buf_elems = e->buf_elems; a.ldc = e->ldc;
  a.w_area = e->w_area; a.weights_resident = e->weights_resident; a.n_tiles = e->total_tiles;
  a.tile_begin = 0; a.tile_end = e->total_tiles; a.mode = mode; a.resid_out = nullptr;
  for (int t = 0; t < PINN_MAX_TERMS; ++t) a.dyn[t] = e->dyn[t];
}

// launch the fused kernel of the handle's mode over tiles [tile_begin, tile_end); a.tail.state != null attaches the
// in-kernel tail (gradient reduction / optimizer / peer allreduce) and makes the launch cooperative
static int launch_fused(pinn_engine* e, const FfmaArgs& a, int grid, cudaStream_t st) {
  if (e->mode == PINN_MODE_FFMA) {
    CUDA_TRY(ffma_launch(e->dtype, e->bufs_smem, a, grid, e->smem, st));
    return 0;
  }
  TcCommonArgs c;
  memset(&c, 0, sizeof c);
  c.prob = a.prob; c.theta = (const float*)a.theta; c.partial = (float*)a.partial; c.partial_stride = a.partial_stride; c.term_sums = a.term_sums;
  c.tl_max = std::max(e->tc_tl_max, 1);
  c.tile_begin = a.tile_begin; c.tile_end = a.tile_end; c.mode = a.mode; c.resid_out = (float*)a.resid_out; c.acc = e->tc_acc;
  c.dbg = e->tc_dbg;
  c.off_P = e->tc_off_P; c.off_misc = e->tc_off_misc; c.off_ones = e->tc_off_ones; c.mx_dim = e->tc_mx_dim; c.mx_taps = e->tc_mx_taps;
  memcpy(c.net_ak, e->tc_net_ak, sizeof c.net_ak);
  for (int k = 0; k < PINN_MAX_TERMS; ++k) { c.seed[k] = a.seed[k]; c.dyn[k] = a.dyn[k]; }
  c.tail = a.tail;
  if (e->tw) {
    TwPackArgs pk;
    memset(&pk, 0, sizeof pk);
    pk.prob = a.prob; pk.theta = (const float*)a.theta; pk.wpack = (uint8_t*)e->tw_wpack; pk.n_images = e->tw_n_images;
    pk.tile_counter = e->tw_counter; pk.counter_init = a.tile_begin + grid;
    memcpy(pk.img_net, e->tw_img_net, sizeof pk.img_net);
    memcpy(pk.img_layer, e->tw_img_layer, sizeof pk.img_layer);
    CUDA_TRY(tw_pack_launch(pk, st));
    e->launches += 1;
    TwArgs w;
    memset(&w, 0, sizeof w);
    static_cast<TcCommonArgs&>(w) = c;
    w.hstash = (uint8_t*)e->stash; w.hstash_per_cta = e->tc_stash_per_cta;
    w.zstash = (float*)e->tw_zstash; w.zstash_per_cta = e->tw_zstash_per_cta;
    w.wpack = (const uint8_t*)e->tw_wpack; w.tile_counter = e->tw_counter;
    w.off_S = e->tw_off_S; w.off_nets = e->tw_off_nets;
    memcpy(w.off_fp, e->tw_off_fp, sizeof w.off_fp);
    memcpy(w.wimg, e->tw_wimg, sizeof w.wimg);
    CUDA_TRY(tw_launch(w, grid, e->smem, st));
    return 0;
  }
  TcArgs t;
  memset(&t, 0, sizeof t);
  static_cast<TcCommonArgs&>(t) = c;
  t.stash = (uint8_t*)e->stash; t.stash_per_cta = e->tc_stash_per_cta; t.split = e->tc_split;
  t.off_Q = e->tc_off_Q;
  t.off_Q_bytes = e->tc_off_Q - e->tc_off_P;   // P and Q regions have the same size
  t.n_nets = e->hprob->n_nets; t.n_terms = e->n_terms; t.n_theta = e->n_theta;
  for (int k = 0; k < e->n_terms; ++k) t.term_dim[k] = (unsigned char)e->hprob->terms[k].dim;
  memcpy(t.nets, e->tc_nets, sizeof t.nets);
  CUDA_TRY(tc_launch(t, grid, e->smem, st));
  return 0;
}


static bool any_sampler(const pinn_engine* e) {
  for (int t = 0; t < e->n_terms; ++t) if (e->sampler_on[t]) return true;
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
static int eval_step(pinn_engine* e, const void* theta, const double* host_weights, void* out_grad, void* out_terms,
                     void* out_total, bool adam, cudaStream_t st) {
  const bool want_grad = adam || out_grad != nullptr;
  FfmaArgs a;
  memset(&a, 0, sizeof a);
  fill_args(e, a, theta, want_grad ? 0 : 1);
  ScaleW sw;
  memset(&sw, 0, sizeof sw);
  if (prepare_scales(e, host_weights, a, sw)) return 1;
  const bool multi = e->nranks > 1;
  int grid = std::min(e->num_sms, e->total_tiles);
  if (multi && e->p2p) grid = e->num_sms;       // the same slice partition of theta on every rank
  if (grid < 1) grid = 1;                       // a rank whose shard is empty still takes part in the reduction
  if (grid > kTailSlots) return fail("pinn_loss_grad: %d CTAs exceed the %d tail slots", grid, kTailSlots);
  if (e->timing) CUDA_TRY(cudaEventRecord(e->ev0, st));
  const long long ng = want_grad ? e->n_theta : 0;
  const bool nccl = multi && !e->p2p;
  if (!nccl) {
    fill_tail(e, a.tail, sw, out_grad, out_terms, out_total, adam, multi);
  } else {
    if (adam)
      return fail("pinn_adam_iterate: the multi-GPU device loop needs the peer-memory allreduce (%s)",
                  e->p2p_why[0] ? e->p2p_why : "not available");
    void* pk_terms = (char*)e->packed + (size_t)ng * e->es;
    fill_tail(e, a.tail, sw, want_grad ? e->packed : nullptr, pk_terms, nullptr, false, false);
  }
  if (launch_fused(e, a, grid, st)) return 1;
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

int pinn_loss_grad(pinn_handle e, const void* dev_theta, const double* host_weights, void* dev_grad,
                   void* dev_term_losses, void* dev_total, void* stream) {
  if (!e) return fail("pinn_loss_grad: null handle");
  if (!dev_theta || !dev_term_losses || !dev_total) return fail("pinn_loss_grad: null theta/term_losses/total");
  CUDA_TRY(cudaSetDevice(e->device));
  for (int t = 0; t < e->n_terms; ++t)
    if (e->dyn[t].n <= 0 && !(e->nranks > 1 && e->n_global_set[t]))
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

static int draw_term(pinn_engine* e, int term, unsigned long long draw, const unsigned long long* draw_dev, cudaStream_t st);

// one iteration of the device-resident loop: fresh points for the sampled terms, then the fused step with Adam in its tail
static int enqueue_adam_iteration(pinn_engine* e, const double* host_weights, cudaStream_t st) {
  char* dout = (char*)e->d_out;
  // draw = host counter + 1 + device counter; the tail advances the device counter, so graph replays resample
  for (int t = 0; t < e->n_terms; ++t)
    if (e->sampler_on[t] && draw_term(e, t, e->sampler_draw + 1, &e->d_state->draw, st)) return 1;
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
    key = fnv1a(e->n_global, sizeof e->n_global, key);
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
      e->adam_graph_key = key; e->adam_graph_n = n_steps;
    }
    CUDA_TRY(cudaGraphLaunch(e->adam_graph, st));
    long long per_it = 1 + (e->tw ? 1 : 0);
    for (int t = 0; t < e->n_terms; ++t) per_it += e->sampler_on[t] ? 1 : 0;
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
  FfmaArgs a;
  memset(&a, 0, sizeof a);
  fill_args(e, a, dev_theta, 2);
  a.tile_begin = e->dyn[term].tile0;
  a.tile_end = e->dyn[term].tile0 + e->dyn[term].n_tiles;
  a.resid_out = dev_r;
  const int grid = std::min(e->num_sms, e->dyn[term].n_tiles);
  if (launch_fused(e, a, grid, (cudaStream_t)stream)) return 1;
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

// effective draw index = draw + *draw_dev (the device counter is advanced by the tail of the device-resident loop)
static int draw_term(pinn_engine* e, int term, unsigned long long draw, const unsigned long long* draw_dev, cudaStream_t st) {
  const int dim = e->hprob->terms[term].dim;
  const long long n = e->sampler_n[term];
  if (grow(&e->own_pts[term], &e->own_pts_cap[term], (size_t)n * dim * e->es, e)) return 1;
  const unsigned long long key = e->sampler_seed[term] + 0x9E3779B97F4A7C15ull * (unsigned long long)(term + 1);
  if (e->sampler_kind[term] == PINN_SAMPLER_LHS)
    CUDA_TRY(sample_lhs_launch(e->dtype, e->own_pts[term], n, dim, e->sampler_lb[term], e->sampler_ub[term], key, draw, draw_dev, st));
  else
    CUDA_TRY(sample_uniform_launch(e->dtype, e->own_pts[term], n, dim, e->sampler_lb[term], e->sampler_ub[term], key, draw, draw_dev, st));
  e->launches += 1;
  e->dyn[term].pts = e->own_pts[term]; e->dyn[term].qw = nullptr; e->dyn[term].n = n;
  return 0;
}

int pinn_set_sampler_ex(pinn_handle e, int32_t term, int32_t kind, int64_t n, const double* host_lb, const double* host_ub,
                        uint64_t seed, void* stream) {
  if (check_term(e, term, "pinn_set_sampler")) return 1;
  if (kind != PINN_SAMPLER_UNIFORM && kind != PINN_SAMPLER_LHS) return fail("pinn_set_sampler: unknown sampler kind %d", kind);
  if (n > 0x7fffffffLL) return fail("pinn_set_sampler: at most 2^31 - 1 points per term");
  if (n < 1) return fail("pinn_set_sampler: term %d needs at least one point", term);
  if (!host_lb || !host_ub) return fail("pinn_set_sampler: null bounds");
  if (e->reduction[term] == PINN_REDUCE_WSUM)
    return fail("pinn_set_sampler: term %d is a weighted-sum (quadrature) term; the uniform sampler serves mean(abs2) terms", term);
  CUDA_TRY(cudaSetDevice(e->device));
  const int dim = e->hprob->terms[term].dim;
  for (int r = 0; r < dim; ++r) {
    if (!(host_lb[r] <= host_ub[r])) return fail("pinn_set_sampler: term %d row %d has lb > ub", term, r);
    e->sampler_lb[term][r] = host_lb[r]; e->sampler_ub[term][r] = host_ub[r];
  }
  e->sampler_on[term] = true; e->sampler_kind[term] = kind; e->sampler_seed[term] = seed; e->sampler_n[term] = n;
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
    if (e->sampler_on[t] && draw_term(e, t, e->sampler_draw, &e->d_state->draw, (cudaStream_t)stream)) return 1;
  retile(e);
  return 0;
}

int pinn_get_points_host(pinn_handle e, int32_t term, void* host_pts) {
  if (check_term(e, term, "pinn_get_points_host")) return 1;
  if (!host_pts) return fail("pinn_get_points_host: null output");
  CUDA_TRY(cudaSetDevice(e->device));
  const size_t bytes = (size_t)e->dyn[term].n * e->hprob->terms[term].dim * e->es;
  CUDA_TRY(cudaDeviceSynchronize());
  if (bytes) CUDA_TRY(cudaMemcpy(host_pts, e->dyn[term].pts, bytes, cudaMemcpyDeviceToHost));
  return 0;
}

int pinn_term_grad_stats(pinn_handle e, int32_t term, const void* dev_theta, double* host_max_abs, double* host_mean_abs,
                         void* stream) {
  if (check_term(e, term, "pinn_term_grad_stats")) return 1;
  if (!dev_theta || !host_max_abs || !host_mean_abs) return fail("pinn_term_grad_stats: null theta/output");
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
  }
  if (host_out) {
    CUDA_TRY(cudaDeviceSynchronize());
    CUDA_TRY(cudaMemcpy(host_out, e->tc_dbg, 2000 * sizeof(long long), cudaMemcpyDeviceToHost));
  }
  return 0;
}
#endif

#ifdef PINN_DEBUG
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
  for (int t = 0; t < e->n_terms; ++t) f += e->flops_per_point[t] * (double)e->dyn[t].n;
  return f;
}

}  // extern "C"
