// dev_types.h -- device-side problem representation shared by the host ABI layer and
// the CUDA kernels.  Built once by pinn_create from pinn_problem_desc and uploaded to
// global memory; kernels read it through uniform (warp-wide identical) loads.
#pragma once
#include <stdint.h>
#include "../../include/pinn_b200.h"

namespace pinn {

constexpr int kTilePts = 32;     // collocation points per tile (= warp lanes) in the FFMA path
constexpr int kWarps = 8;        // warps per CTA in the FFMA path
constexpr int kThreads = kWarps * 32;

struct DevInstr {
  int op, a, b, pad;
  double imm;
};

struct DevNet {
  int n_layers;
  int dims[PINN_MAX_LAYERS + 1];
  int acts[PINN_MAX_LAYERS];
  long long w_off[PINN_MAX_LAYERS];  // theta offset of layer weight (out x in col-major)
  long long b_off[PINN_MAX_LAYERS];  // theta offset of layer bias
  int ws_off[PINN_MAX_LAYERS];       // offset (in scalars) of the layer's staged W^T in the smem weight area
  int bs_off[PINN_MAX_LAYERS];       // offset of the staged (zero padded) bias
  int max_width8;                    // max over dims, rounded up to 8
};

// channel structure of one (term, network) pair:
//   channel 0            value
//   channels 1..n1       first derivatives along dir1[i]
//   channels n1+1..      second derivatives d^2/(d dir1[s_a] d dir1[s_b])
//   channels n1+n2+1..   pure third derivatives d^3/(d dir1[t_a])^3 (t_s: the pure second-derivative channel along the same
//                        direction, which the chain rule of the third needs)
struct DevChan {
  int C, n1, n2, n3;
  int t_a[PINN_MAX_IN], t_s[PINN_MAX_IN];
  int dir1[PINN_MAX_IN];
  int s_a[PINN_MAX_CH], s_b[PINN_MAX_CH];   // indices into dir1[] (0-based)
  int rows[PINN_MAX_IN];                    // point row feeding network input j
  int stash_off[PINN_MAX_LAYERS];           // per-layer offset (scalars) inside the CTA stash
  int pure;                                 // every second-derivative channel s is d2/d(dir1[s])^2
};

struct DevTerm {
  int dim;
  int n_used;                       // networks tapped by this term
  int used_net[PINN_MAX_NETS];
  DevChan chan[PINN_MAX_NETS];      // indexed by slot 0..n_used-1
  int n_taps;
  int tap_slot[PINN_MAX_TAPS];
  int tap_ch[PINN_MAX_TAPS];
  int tap_out[PINN_MAX_TAPS];
  int n_instr;
  DevInstr prog[PINN_MAX_INSTR];
  int weighted;                     // PINN_REDUCE_WSUM
};

// per-term state that changes with pinn_set_points; travels in the kernel arguments
struct TermDyn {
  const void* pts;
  const void* qw;
  long long n;                      // local number of points
  int tile0;                        // first tile index of this term in the global enumeration
  int n_tiles;
};

// one integral term (pinn_integral_desc): the node-point geometry, the Gauss-Legendre table and the integrand, planned
// like a term over the node point (dim = owner dim + n_dims rows)
struct DevIntegral {
  int owner;                        // owner term
  int slot;                         // the owner reads the value as its tap n_taps + (index among its integrals)
  int n_dims, q;
  int row[2], lb_row[2], ub_row[2], inf_kind[2];
  double lb[2], ub[2], shift[2];
  double xi[PINN_MAX_QUAD], wq[PINN_MAX_QUAD];   // nodes and weights on [-1, 1]
  DevTerm body;
};

struct DevProblem {
  int n_nets, n_terms, n_params;
  long long param_off, n_theta;
  DevNet nets[PINN_MAX_NETS];
  DevTerm terms[PINN_MAX_TERMS];
  int n_integrals;
  DevIntegral integ[PINN_MAX_INTEGRALS];
  // fixed networks (pinn_create_ex2): a tap's network n_nets + j is fixed[j]; w_off / b_off index its own parameter
  // buffer fixed_params[j] (written by pinn_set_fixed_params: the kernel arguments of problems without fixed networks
  // stay as they were), not theta
  int n_fixed;
  DevNet fixed[PINN_MAX_FIXED_NETS];
  const void* fixed_params[PINN_MAX_FIXED_NETS];
  // functional term (PINN_REDUCE_*_OF_SUM): its index (-1: none) and 1 for g = (.)^2, 0 for g = |.|
  int func_term, func_square;
};

// per term scale (L_k = scale_k * sum_p qw_p r_p^2) and loss weight, passed by value
struct ScaleW {
  double scale[PINN_MAX_TERMS];
  double w[PINN_MAX_TERMS];
};

// ---- fused kernel tail (tail.cuh): grid barrier, slice reduction, one-shot peer allreduce, optimizer step ----------
constexpr int kMaxRanks = 8;       // GPUs of one NVSwitch domain that share the peer-memory allreduce
constexpr int kTailSlots = 256;    // per-slice flags per peer (>= CTAs per launch)

struct TailState {                 // device-resident, owned by the handle (zero-initialised)
  unsigned int count, gen;         // self-resetting generation barrier over the CTAs of one launch
  unsigned int step;               // launches with a tail so far (flag value / buffer parity of the peer allreduce)
  short func_term, func_square;    // DevProblem's functional term, for the tail of its kernel (written by pinn_create)
  unsigned long long adam_t;       // optimizer steps taken (bias correction)
  unsigned long long draw;         // sampler draw counter (advanced by the tail so captured graphs resample)
};

struct TailArgs {
  TailState* state;                // null: no tail (the launch only writes per-CTA partials)
  void* out_grad;                  // [n_theta] or null
  void* out_terms;                 // [n_terms] unweighted term losses
  void* out_total;                 // weighted total or null
  void* adam_theta;                // non-null: Adam step applied in place (theta, m, v)
  void* adam_m;
  void* adam_v;
  double adam_lr, adam_b1, adam_b2, adam_eps;
  unsigned long long timeout_ns;   // spin bound of the barriers (a lost peer traps instead of hanging)
  int bump_draw;                   // advance state->draw (device-side samplers present)
  int nranks, rank;
  long long recv_words;            // 8-byte slots per (parity, source rank) block: n_theta words + 2 per term loss
  long long* dbg;                  // -DPINN_DEBUG builds: 4 globaltimer marks per CTA (tail entry, barrier, pushed, done)
  void* peer_recv[kMaxRanks];      // receive region of every rank (peer-mapped): [2 parities][nranks][recv_words] slots
  ScaleW sw;
};

// kernel launch arguments (passed by value, < 4 KB)
struct FfmaArgs {
  const DevProblem* prob;
  const void* theta;
  void* partial;          // [grid][partial_stride] per-CTA gradient partials (scalar type); with a functional term the
                          // functional's own partials G [grid][partial_stride] follow them
  long long partial_stride;   // n_theta rounded up to 4 scalars (16-byte aligned rows for the vector loads of the tail)
  double* term_sums;      // [grid][PINN_MAX_TERMS] per-CTA sum_p qw_p r_p^2
  void* stash;            // [grid][stash_per_cta]
  void* gbufs;            // [grid][2*buf_elems] global fallback for the two activation buffers
  long long stash_per_cta;
  long long buf_elems;    // scalars per activation buffer = max C * max_width8 * TP
  int ldc;                // channel stride inside a buffer = max_width8 * TP
  int w_area;             // scalars in the smem weight area
  int weights_resident;   // all layers of all nets staged once per CTA
  int n_tiles;
  int tile_begin;         // restrict to [tile_begin, tile_end) (single-term residual mode)
  int tile_end;
  int mode;               // 0 loss+grad, 1 loss only, 2 residual out
  void* resid_out;        // mode 2: r[n] of the selected term
  double seed[PINN_MAX_TERMS];  // w_k * scale_k : d(total)/d(sum_p qw r^2) of each term
  TermDyn dyn[PINN_MAX_TERMS];
  TailArgs tail;
};
static_assert(sizeof(FfmaArgs) <= 4096, "FFMA kernel arguments must stay under 4 KB");

}  // namespace pinn
