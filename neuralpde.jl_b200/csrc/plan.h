// plan.h -- host planner: validates a pinn_problem_desc and lowers it to what a handle keeps fixed for its lifetime.
#pragma once
#include "dev_types.h"
#include "tc_types.h"

namespace pinn {
int fail(const char* fmt, ...);    // sets the message pinn_last_error returns; returns 1
const char* last_error();

struct TermPlan {
  int reduction;                   // PINN_REDUCE_*
  double scale;                    // WSUM / *_OF_SUM scale (MEAN: 1/n_global, formed at launch time)
  double flops_per_point;          // algorithmic: 6 * sum over the term's networks of C * sum_l dims[l] * dims[l+1]
};

struct Plan {
  DevProblem prob;                 // uploaded once by pinn_create
  TermPlan term[PINN_MAX_TERMS];
  int tile_pts;                    // points per tile of the mode's kernels
  size_t smem;                     // dynamic shared memory per CTA
  bool bufs_smem;                  // FFMA: the two activation buffers live in shared memory (else in gbufs)
  bool wide;                       // tensor-core modes: tw_pack + the 128-wide kernel run instead of the narrow one
  bool x256;                       // (with wide) a hidden width is 192 or 256: tx_pack + the 256-wide kernel run instead
  bool integ;                      // FFMA: the problem has integral terms (the kernel instantiation with node tiles runs)
  bool func;                       // FFMA: the problem has a functional term (its own kernel instantiation runs)
  long long fixed_len[PINN_MAX_FIXED_NETS];   // scalars of each fixed network's parameter buffer
  // launch-argument templates: the planner fills the layout, pinn_create the buffers, a launch the per-call fields
  FfmaArgs ffma; TcArgs tc; TwArgs tw; TwPackArgs pack;
};

// the modes that run ffma_loss_grad_kernel (CUDA-core FMA, or its DMMA instantiation for PINN_MODE_TC_F64)
inline bool ffma_kernel_mode(int mode) { return mode == PINN_MODE_FFMA || mode == PINN_MODE_TC_F64; }

// the q-point Gauss-Legendre rule on [-1, 1], nodes ascending
void gauss_legendre(int q, double* x, double* w);

// networks a tap may name: the trainable ones, then the fixed ones
constexpr int kMaxAllNets = PINN_MAX_NETS + PINN_MAX_FIXED_NETS;

// Pure host code (no CUDA runtime call); max_smem: the device's opt-in shared memory per block in bytes.
// integrals[n_integrals]: integral terms (pinn_create_ex), fixed[n_fixed]: fixed networks (pinn_create_ex2); none for
// pinn_create.
int plan_problem(const pinn_problem_desc* d, const pinn_integral_desc* integrals, int n_integrals,
                 const pinn_fixed_net_desc* fixed, int n_fixed, int max_smem, Plan& p);
}  // namespace pinn
