// engine.h -- the handle behind pinn_handle and the host helpers the C-ABI translation units share (pinn_abi.cu, qn.cu,
// hmc.cu).
#pragma once
#include <cuda_runtime.h>

#include "plan.h"

#define CUDA_TRY(expr)                                                                  \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess) return fail("%s failed: %s", #expr, cudaGetErrorString(_e)); \
  } while (0)

typedef struct ncclComm* ncclComm_t;

namespace pinn {

// per-term host state that changes after pinn_create
struct TermState {
  long long n_global = 0; bool n_global_set = false;   // pinn_set_global_count: points over all ranks (MEAN scale)
  // device-side sampler (StochasticTraining): box, seed, point count; the draw counter is shared by all terms
  bool sampler_on = false; int sampler_kind = 0;
  double sampler_lb[PINN_MAX_DIM] = {}, sampler_ub[PINN_MAX_DIM] = {};
  unsigned long long sampler_seed = 0; long long sampler_n = 0;
  // PINN_SAMPLER_KKL (pinn_set_sampler_kkl): sampler_n = kkl_times * kkl_sub points, time bounds in sampler_lb/ub[0]
  long long kkl_times = 0; int kkl_sub = 0, kkl_flags = 0;
  void *own_pts = nullptr, *own_qw = nullptr;   // engine-owned point copies
  size_t own_pts_cap = 0, own_qw_cap = 0;
};

struct QnState;   // quasi-Newton driver state (qn.cu)
struct HmcState;  // HMC sampler state (hmc.cu)

}  // namespace pinn

struct pinn_engine {
  int dtype = 0, mode = 0, device = 0;
  size_t es = 4;
  pinn::Plan plan;               // what the handle keeps fixed: problem image, term values, launch-argument templates
  pinn::DevProblem* dprob = nullptr;   // device copy of plan.prob
  int n_terms = 0;
  long long n_theta = 0, partial_stride = 0;
  pinn::TermState term[PINN_MAX_TERMS];
  pinn::TermDyn dyn[PINN_MAX_TERMS] = {};
  // fixed networks: the parameters each launch reads (aliased or fixed_own), engine-owned copies of the *_host variant
  const void* fixed_ptr[PINN_MAX_FIXED_NETS] = {};
  void* fixed_own[PINN_MAX_FIXED_NETS] = {};
  int total_tiles = 0, num_sms = 0;
  long long *tc_dbg = nullptr, *tail_dbg = nullptr;   // pinn_debug_tc_timeline / pinn_debug_tail_marks buffers
  // wide tensor path (128-wide layers): streamed weights, fp32 pre-activation stash
  void *tw_wpack = nullptr, *tw_zstash = nullptr;
  int* tw_counter = nullptr;
  float* tc_acc = nullptr;       // tensor-core paths: per-CTA fp32 accumulator regions (tc_prims.cuh)
  // workspaces (device)
  void* partial = nullptr;
  double* term_sums = nullptr;
  void* stash = nullptr;
  void* gbufs = nullptr;
  void* packed = nullptr;        // [n_theta + n_terms] allreduce buffer
  long long ws_bytes = 0;
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
  unsigned long long sampler_draw = 0;
  // device-resident quasi-Newton state (pinn_qn_begin)
  pinn::QnState* qn = nullptr;
  // device-resident HMC sampler state (pinn_hmc_begin)
  pinn::HmcState* hmc = nullptr;
  // fused kernel tail (tail.cuh): device-resident barrier / step state
  pinn::TailState* d_state = nullptr;
  unsigned long long tail_timeout_ns = 20ull * 1000000000ull;
  // captured iteration graph of the device-resident Adam loop
  cudaGraphExec_t adam_graph = nullptr;
  unsigned long long adam_graph_key = 0;
  // comm
  ncclComm_t comm = nullptr;
  int rank = 0, nranks = 1;
  // peer-memory allreduce (NVLink): receive region [2 parities][nranks][recv_words] of 8-byte {word, flag} slots,
  // mapped from every rank
  bool p2p = false;
  void* sym = nullptr;
  long long recv_words = 0;
  void* peer_base[pinn::kMaxRanks] = {};
  char p2p_why[160] = {};
  // introspection
  long long launches = 0;
  bool timing = false;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  float last_ms = 0.f;
};

namespace pinn {
// cudaMalloc counted in the handle's workspace bytes
int dev_alloc(void** p, size_t bytes, pinn_engine* e);
bool any_sampler(const pinn_engine* e);
// One evaluation of the hot path on stream st (fused kernel + tail, plus the allreduce steps of the NCCL fallback).
int eval_step(pinn_engine* e, const void* theta, const double* host_weights, void* out_grad, void* out_terms,
              void* out_total, bool adam, cudaStream_t st);
// fresh points of a device-sampled term: draw index draw + *draw_dev (draw_dev nullable)
int draw_term(pinn_engine* e, int term, unsigned long long draw, const unsigned long long* draw_dev, cudaStream_t st);
// frees the quasi-Newton state (qn.cu); called by pinn_destroy and by a repeated pinn_qn_begin
void qn_release(pinn_engine* e);
// frees the HMC sampler state and its graph (hmc.cu); called by pinn_destroy and by a repeated pinn_hmc_begin
void hmc_release(pinn_engine* e);
}  // namespace pinn
