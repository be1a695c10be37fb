/*
 * pinn_b200.h -- C ABI of the H100-native PINN residual/loss engine.
 *
 * This is the drop-in boundary for NeuralPDE.jl's PhysicsInformedNN hot path
 * (SURVEY.md section 8(b), boundary B1).  The reference has no FFI of its own:
 * its extension point is the object `discretize` returns,
 *     OptimizationProblem(OptimizationFunction(full_loss_function, AutoZygote()), flat_init_params)
 *     (reference src/discretize.jl:776-780),
 * i.e. `f(theta, p)::Real` plus its reverse-mode gradient.  A Julia shim (see
 * INTEGRATION.md) lowers a `PINNRepresentation` to `pinn_problem_desc` once at
 * `discretize` time and then calls the entry points below through
 * `@ccall libpinn_b200.pinn_loss_grad(...)` with `CuPtr`s on CUDA.jl's task-local
 * stream.  All signatures are plain C: pointers, sizes, no torch / C++ types.
 *
 * Reference functions each entry point replaces (file:line in /root/reference):
 *   pinn_create            <- symbolic_discretize's closure construction
 *                             (src/discretize.jl:413-651), Phi (src/pinn_types.jl:79-90)
 *   pinn_create_ex         <- the same, with get_numeric_integral's integral terms
 *                             (src/discretize.jl:334-397, src/transform_inf_integral.jl)
 *   pinn_set_points[_host] <- train-set placement in get_loss_function
 *                             (src/training_strategies.jl:215-221 Grid, :271-282 Stochastic)
 *   pinn_loss_grad[_host]  <- full_loss_function(theta,p) (src/discretize.jl:567-598)
 *                             + Zygote gradient (src/discretize.jl:778)
 *                             + numeric_derivative (src/pinn_types.jl:445-482; replaced
 *                               by exact forward-mode taps, SURVEY Appendix B)
 *   pinn_term_residual     <- datafree_{pde,bc}_loss_functions[i](points, theta)
 *                             (src/pinn_types.jl:414-440; probe used by
 *                             test/Forward/forward__ode.jl:134-137)
 *   pinn_comm_init         <- (no counterpart: the reference is single-process)
 *
 * Conventions
 *   - Every function returns 0 on success, nonzero on error; the message is
 *     available from pinn_last_error() (thread-local).  No C++ exception crosses
 *     the ABI.
 *   - theta / grad use the reference's flat ComponentArray layout: per network,
 *     per Dense layer: weight (out x in, column-major) then bias (out); networks in
 *     depvar order; then the `p` block when param_estim=true
 *     (src/discretize.jl:451-465, src/pinn_types.jl:337-351).
 *   - Point sets are d x N column-major (one point = d contiguous scalars), the
 *     reference's train-set layout (src/discretize.jl:226-238).
 *   - Ownership: the caller owns theta / grad / output buffers and device point
 *     buffers passed to pinn_set_points (aliased, not copied, while the handle
 *     lives).  The engine owns its workspaces, host-staged copies and the NCCL
 *     communicator.
 *   - Threading: a handle is not thread-safe; one handle per GPU rank.  All
 *     device work is enqueued on the stream passed in; no hidden device
 *     synchronisation except in the *_host variants.
 */
#ifndef PINN_B200_H
#define PINN_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PINN_ABI_VERSION 2

/* hard limits (validated by pinn_create) */
#define PINN_MAX_LAYERS 16   /* Dense layers per network */
#define PINN_MAX_IN 8        /* network input dimension */
#define PINN_MAX_CH 10       /* propagated channels per (term, network): 1 + #first + #second + #third */
#define PINN_MAX_NETS 8
#define PINN_MAX_TAPS 32     /* taps per term */
#define PINN_MAX_INSTR 192   /* residual-program length per term */
#define PINN_MAX_TERMS 32
#define PINN_MAX_PARAMS 16   /* length of the theta.p block */
#define PINN_MAX_DIM 8       /* rows of a term's point matrix */

typedef struct pinn_engine* pinn_handle;

/* scalar type of theta / points / outputs (theta's eltype rules, src/eltype_matching.jl) */
enum { PINN_F32 = 0, PINN_F64 = 1 };

/* arithmetic mode of the layer contractions.
 * Shapes the tensor-core modes accept (anything else: pinn_create fails with a message, never a silent fallback):
 *   1-output networks, linear last layer, >= 2 Dense layers, PINN_F32, and either
 *     - every hidden width in {16, 32, 48, 64}, <= 6 taps per term and <= 5 propagated channels per (term, network)
 *                                                                                                    [both modes], or
 *     - every hidden width in {64, 128}, <= 6 taps per term, at least one hidden->hidden layer; terms that need more
 *       than 4 channels are evaluated in several passes over the same weights (pure second derivatives only)
 *                                                                                           [PINN_MODE_TC_BF16], or
 *     - a hidden width of 192 or 256 and every hidden width a multiple of 64 up to 256, up to PINN_MAX_TAPS taps per
 *       term (as far as shared memory allows), otherwise as the previous case                [PINN_MODE_TC_BF16]. */
enum {
  PINN_MODE_FFMA = 0,      /* CUDA-core FMA in the scalar type (parity mode, fp32 / fp64)   */
  PINN_MODE_TC_BF16 = 1,   /* wgmma, bf16 operands, fp32 accumulate                          */
  PINN_MODE_TC_SPLIT = 2,  /* wgmma, split-bf16 x2 (3 MMAs per product), fp32 accumulate     */
  PINN_MODE_TC_F64 = 3     /* DMMA (mma.sync m16n8k16 .f64), fp64 operands and accumulate    */
};
/* PINN_MODE_TC_F64 runs the kernel of PINN_MODE_FFMA with its three layer products (forward, input adjoint, weight
 * gradient) on the FP64 tensor cores; activations, derivative channels, the residual program and the tail are the FFMA
 * path's.  It needs PINN_F64 and accepts every shape, integral term, fixed network and functional term PINN_MODE_FFMA
 * accepts.  Results equal PINN_MODE_FFMA's up to the summation order of the layer products. */

/* activations (Lux Dense: act.(W*x .+ b)) */
enum {
  PINN_ACT_IDENTITY = 0,
  PINN_ACT_TANH = 1,
  PINN_ACT_SIGMOID = 2,
  PINN_ACT_SIN = 3,
  PINN_ACT_SOFTPLUS = 4,
  PINN_ACT_SWISH = 5,
  PINN_ACT_GELU = 6,       /* NNlib's gelu, tanh form: x/2 (1 + tanh(sqrt(2/pi) (x + 0.044715 x^3))); FFMA kernel
                            * (PINN_MODE_FFMA, PINN_MODE_TC_F64) only */
  PINN_ACT_LOGCOSH = 7,    /* NNlib's logcosh: x + softplus(-2x) - log 2; FFMA kernel (PINN_MODE_FFMA,
                            * PINN_MODE_TC_F64) only */
  PINN_ACT_COS = 8         /* cos x; FFMA kernel (PINN_MODE_FFMA, PINN_MODE_TC_F64) only */
};

/* residual-program opcodes.  The program is in SSA form: instruction i defines
 * value i; `a` / `b` name earlier values (or an index for the LOAD ops); the last
 * instruction's value is the residual r = lhs - rhs of the equation, i.e. what the
 * reference's generated function returns per point (src/symbolic_utilities.jl:360-370). */
enum {
  PINN_OP_CONST = 0,  /* imm                                                     */
  PINN_OP_COORD = 1,  /* row `a` of the term's point matrix (cord[[a],:])        */
  PINN_OP_TAP = 2,    /* tap `a` of the term (u(...) or a pure partial of it)    */
  PINN_OP_PARAM = 3,  /* theta.p[a]  (param_estim) -- differentiated             */
  PINN_OP_ADD = 4,
  PINN_OP_SUB = 5,
  PINN_OP_MUL = 6,
  PINN_OP_DIV = 7,
  PINN_OP_NEG = 8,
  PINN_OP_POW = 9,    /* v[a] ^ v[b]                                             */
  PINN_OP_POWI = 10,  /* v[a] ^ (int)imm                                         */
  PINN_OP_SIN = 11,
  PINN_OP_COS = 12,
  PINN_OP_EXP = 13,
  PINN_OP_LOG = 14,
  PINN_OP_TANH = 15,
  PINN_OP_SQRT = 16,
  PINN_OP_ABS = 17,
  PINN_OP_INTEGRAL = 18   /* value of integral `a` at the term's point (pinn_create_ex only) */
};

typedef struct {
  int32_t op;
  int32_t a;
  int32_t b;
  int32_t _pad;
  double imm;
} pinn_instr;

/* one Dense MLP (Lux.Chain of Dense layers), one per dependent variable */
typedef struct {
  int32_t n_layers;      /* number of Dense layers                         */
  const int32_t* dims;   /* n_layers+1 entries: in, hidden..., out         */
  const int32_t* acts;   /* n_layers entries: PINN_ACT_* of each layer      */
  int64_t theta_offset;  /* start of this network's block inside theta      */
} pinn_net_desc;

/* a tap = u_k or one pure partial derivative of it, as produced by
 * _transform_expression (src/symbolic_utilities.jl:150-201).  dir[] index the
 * network's own input vector (dict_interior_indvars), not the point rows. */
typedef struct {
  int32_t net;     /* network (depvar) index                               */
  int32_t out;     /* output component of the network (0 for 1-output nets) */
  int32_t order;   /* 0, 1, 2 (any pair of directions) or 3 (pure: d^3/dx_i^3, PINN_MODE_FFMA) */
  int32_t dir[4];  /* derivative directions, `order` entries used            */
} pinn_tap_desc;

/* The two *_OF_SUM reductions make a FUNCTIONAL term: its program yields a value v_p per point (not a residual to
 * square) and its loss is g(scale * sum_p w_p v_p), g = |.| or (.)^2, w_p the nullable weights of pinn_set_points (1
 * when none are given).  It is an integral constraint such as normalisation or a zero mean (reference
 * docs/src/tutorials/constraints.md, test/NNPDE2/additional_loss__fokker_planck.jl); for |.| the gradient uses
 * g'(0) = 0.  At most one functional term per problem, PINN_MODE_FFMA or PINN_MODE_TC_F64, no PINN_OP_INTEGRAL in its program.  Its
 * nodes are fixed: pinn_set_sampler*, pinn_term_grad_stats and the HMC entry points refuse it, and with several ranks
 * the whole node set goes to one rank (0 points elsewhere; pinn_set_global_count only accepts the local count),
 * because g(sum_r S_r) != sum_r g(S_r).  pinn_term_residual returns v_p. */
enum { PINN_REDUCE_MEAN = 0,          /* mean(abs2, r)            training_strategies.jl:220 */
       PINN_REDUCE_WSUM = 1,          /* scale * sum(w .* abs2(r)) fixed-node quadrature      */
       PINN_REDUCE_ABS_OF_SUM = 2,    /* abs(scale * sum(w .* v))  functional term            */
       PINN_REDUCE_SQUARE_OF_SUM = 3  /* abs2(scale * sum(w .* v)) functional term            */ };

typedef struct {
  int32_t dim;                 /* rows of the point matrix                              */
  int32_t n_taps;              /* 0: a parameter-only term, whose program must read PINN_OP_PARAM
                                  (PINN_MODE_FFMA / PINN_MODE_TC_F64; the FFMA kernel runs
                                  its program alone, no network pass)                   */
  const pinn_tap_desc* taps;
  const int32_t* net_rows;     /* [n_nets][PINN_MAX_IN]: point row feeding input j of
                                  network k (cord_k = vcat(...), discretize.jl:111-116);
                                  ignored for networks the term does not tap            */
  int32_t n_instr;
  const pinn_instr* prog;
  int32_t reduction;           /* PINN_REDUCE_*                                         */
  double scale;                /* PINN_REDUCE_WSUM / *_OF_SUM: multiplies the weighted sum */
} pinn_term_desc;

typedef struct {
  int32_t abi_version;         /* PINN_ABI_VERSION                                      */
  int32_t dtype;               /* PINN_F32 / PINN_F64                                   */
  int32_t mode;                /* PINN_MODE_*                                           */
  int32_t device;              /* CUDA device ordinal                                   */
  int32_t n_nets;
  const pinn_net_desc* nets;
  int32_t n_terms;             /* PDE terms then BC terms, in full_loss_function order   */
  const pinn_term_desc* terms;
  int32_t n_params;            /* length of theta.p (0 unless param_estim)               */
  int64_t param_offset;        /* start of theta.p inside theta                          */
  int64_t n_theta;             /* total length of theta                                  */
} pinn_problem_desc;

/* ---- integral terms (integro-differential equations) ----------------------------------------------------------
 * An integral over 1 or 2 of the owner term's coordinates, I(p) = int g(s) ds, evaluated per collocation point p of
 * the owner term -- the reference's get_numeric_integral (src/discretize.jl:334-397), which calls adaptive h-cubature
 * with reltol = abstol = 1e-3.  The engine uses a fixed Gauss-Legendre rule instead: q nodes per integrating dimension
 * (a tensor product for two), so the value is deterministic and its gradient is the exact gradient of the rule.
 * The quadrature runs in the variable t: t_k in [lb_k, ub_k] (a constant, or an owner point row such as a hoisted
 * coordinate expression), and the coordinate the integrand sees is x_k(t_k):
 *   PINN_INF_NONE   x = t
 *   PINN_INF_BOTH   x = t / (1 - t^2)             (-inf, inf)   (reference src/transform_inf_integral.jl)
 *   PINN_INF_UPPER  x = shift + t / (1 - t)       [a, inf)
 *   PINN_INF_LOWER  x = shift + t / (1 + t)       (-inf, b]
 * The Jacobian of the substitution is part of the integrand's program.  The integrand's point ("node point") has
 * dim(owner) + n_dims rows: the owner's rows with row[k] replaced by x_k, then t_0 (, t_1).  Its taps, net_rows and
 * program (COORD / TAP / PARAM / arithmetic; the last value is g) follow pinn_term_desc.  The owner's program reads
 * the integral with PINN_OP_INTEGRAL a.  Integral terms run on the FFMA path only. */
#define PINN_MAX_INTEGRALS 8   /* integrals per problem */
#define PINN_MAX_QUAD 64       /* Gauss-Legendre nodes per integrating dimension */
enum { PINN_INF_NONE = 0, PINN_INF_BOTH = 1, PINN_INF_UPPER = 2, PINN_INF_LOWER = 3 };
typedef struct {
  int32_t owner;               /* term whose program reads the integral                                  */
  int32_t n_dims;              /* integrating dimensions, 1 or 2                                          */
  int32_t q;                   /* Gauss-Legendre nodes per dimension, 1..PINN_MAX_QUAD                    */
  int32_t row[2];              /* owner point row of each integrating variable                           */
  int32_t lb_row[2], ub_row[2];   /* owner point row holding the bound (in t), or -1: the constant below   */
  double lb[2], ub[2];         /* constant bounds in t                                                   */
  int32_t inf_kind[2];         /* PINN_INF_*                                                             */
  double shift[2];             /* PINN_INF_UPPER / LOWER: the shift of the substitution                  */
  int32_t n_taps;
  const pinn_tap_desc* taps;
  const int32_t* net_rows;     /* [n_nets][PINN_MAX_IN]: node point row feeding input j of network k     */
  int32_t n_instr;
  const pinn_instr* prog;
} pinn_integral_desc;

/* ---- fixed networks (neural adapters, registered network functions) ------------------------------------------
 * A fixed network is a Dense MLP whose parameters are not trained: a teacher a neural adapter fits its student to
 * (reference src/neural_adapter.jl), or a trained network read through a registered function such as
 * `phi_bound(x, y) = first(phi(vcat(x, y), res.u))` with `@register_symbolic phi_bound(x, y)`.  Its shape rules and
 * activations are those of pinn_net_desc; its parameters live in their own buffer (flat Lux layout, the handle's dtype),
 * outside theta.  A tap names fixed network j as net = n_nets + j (values and derivatives as for trainable networks),
 * and a term's net_rows then has n_nets + n_fixed rows.  The forward pass runs in the fused kernel like any other tap;
 * nothing flows back into a fixed network, so the gradient has n_theta entries as before.  FFMA path only. */
#define PINN_MAX_FIXED_NETS 16
typedef struct {
  int32_t n_layers;      /* number of Dense layers                         */
  const int32_t* dims;   /* n_layers+1 entries: in, hidden..., out         */
  const int32_t* acts;   /* n_layers entries: PINN_ACT_* of each layer      */
} pinn_fixed_net_desc;

/* ---- lifecycle ---------------------------------------------------------------- */
int pinn_create(const pinn_problem_desc* desc, pinn_handle* out);
/* pinn_create with integral terms integrals[n_integrals] (0 <= n_integrals <= PINN_MAX_INTEGRALS; 0 is pinn_create) */
int pinn_create_ex(const pinn_problem_desc* desc, const pinn_integral_desc* integrals, int32_t n_integrals,
                   pinn_handle* out);
/* pinn_create_ex with fixed networks fixed[n_fixed] (0 <= n_fixed <= PINN_MAX_FIXED_NETS; 0 is pinn_create_ex).  Every
 * fixed network needs its parameters (pinn_set_fixed_params[_host]) before the first evaluation. */
int pinn_create_ex2(const pinn_problem_desc* desc, const pinn_integral_desc* integrals, int32_t n_integrals,
                    const pinn_fixed_net_desc* fixed, int32_t n_fixed, pinn_handle* out);
/* Parameters of fixed network j: alias a device buffer (owned by the caller while the handle uses it), or copy a host
 * buffer into engine memory (on `stream`).  Either may be called again between evaluations to re-point it: both first
 * wait for the device to finish the evaluations already enqueued, and the copy is complete when the call returns. */
int pinn_set_fixed_params(pinn_handle h, int32_t j, const void* dev_params);
int pinn_set_fixed_params_host(pinn_handle h, int32_t j, const void* host_params, void* stream);
int pinn_destroy(pinn_handle h);
const char* pinn_last_error(void);
int pinn_abi_version(void);

/* ---- point sets ---------------------------------------------------------------- */
/* Alias a device-resident d x n point matrix (and optional n quadrature weights).   */
int pinn_set_points(pinn_handle h, int32_t term, const void* dev_pts, int64_t n,
                    const void* dev_weights /* nullable */);
/* Copy a host d x n matrix into engine-owned device memory (Stochastic resampling:
 * host rand + upload every call, training_strategies.jl:277-281).  Async on `stream`. */
int pinn_set_points_host(pinn_handle h, int32_t term, const void* host_pts, int64_t n,
                         const void* host_weights /* nullable */, void* stream);
/* Number of points the mean is taken over when the term is sharded across ranks
 * (defaults to the local n). */
int pinn_set_global_count(pinn_handle h, int32_t term, int64_t n_global);

/* ---- the hot path --------------------------------------------------------------- */
/* loss and gradient of  sum_k w[k] * L_k(theta)  (discretize.jl:582-588).
 *   dev_theta       [n_theta]  device
 *   host_weights    [n_terms]  host doubles (adaptive-loss weights; NULL = all 1)
 *   dev_grad        [n_theta]  device, nullable (loss only)
 *   dev_term_losses [n_terms]  device: unweighted L_k (for logging / adaptive weights)
 *   dev_total       [1]        device
 * With a communicator attached, grad / losses are summed over ranks (one allreduce). */
int pinn_loss_grad(pinn_handle h, const void* dev_theta, const double* host_weights,
                   void* dev_grad, void* dev_term_losses, void* dev_total, void* stream);

/* Same, through HOST buffers: copies theta in, runs, copies grad / losses / total out
 * and synchronises.  This is the end-to-end call a CPU-resident optimizer makes. */
int pinn_loss_grad_host(pinn_handle h, const void* host_theta, const double* host_weights,
                        void* host_grad, void* host_term_losses, void* host_total);

/* residual vector r[n] of one term at its current point set (parity probe) */
int pinn_term_residual(pinn_handle h, int32_t term, const void* dev_theta, void* dev_r,
                       void* stream);
int pinn_term_residual_host(pinn_handle h, int32_t term, const void* host_theta, void* host_r);

/* ---- device-side StochasticTraining sampler (SURVEY section 8(f) item 1) -----------------------------------------
 * The reference draws `lb .+ (ub .- lb) .* rand(T, d, n)` on the host and uploads it on EVERY loss evaluation
 * (generate_random_points src/training_strategies.jl:242-245, get_loss_function :271-282).  pinn_set_sampler registers
 * a term's box (one [lb, ub] per point row) and point count and draws the first sample into engine-owned memory;
 * pinn_resample draws the next sample of every registered term (one small Philox4x32-10 kernel per term, counter =
 * (point, row group, draw), key = seed + term), so a training iteration has no host round trip.  pinn_adam_iterate
 * resamples before every step when samplers are registered.  pinn_get_points_host copies a term's current points out
 * (callbacks, tests).  The random stream necessarily differs from Julia's default RNG; the distribution is the same. */
int pinn_set_sampler(pinn_handle h, int32_t term, int64_t n, const double* host_lb, const double* host_ub, uint64_t seed,
                     void* stream);
/* QuasiRandomTraining on the device: kind = PINN_SAMPLER_LHS draws a Latin hypercube sample per call -- the reference's
 * default `sampling_alg = LatinHypercubeSample()` (src/training_strategies.jl:285-334; QuasiMonteCarlo.sample on the host
 * + upload per call, :365-389).  Each row's n strata hold exactly one point per draw: stratum index = a keyed Feistel
 * permutation of the point index, position inside the stratum uniform (Philox).  pinn_set_sampler == kind UNIFORM. */
enum { PINN_SAMPLER_UNIFORM = 0, PINN_SAMPLER_LHS = 1, PINN_SAMPLER_KKL = 2 };
int pinn_set_sampler_ex(pinn_handle h, int32_t term, int32_t kind, int64_t n, const double* host_lb, const double* host_ub,
                        uint64_t seed, void* stream);
/* NNSDE's StochasticTraining on the device (kind PINN_SAMPLER_KKL; pinn_set_sampler_ex does not take it): the points
 * (t, z_1..z_n_z) of a truncated Karhunen-Loeve (KKL) Wiener path, term dim = 1 + n_z.  Draw d (the host counter of
 * pinn_resample plus the device counter, as the other samplers) fills point p = i * sub_batch + s,
 * i < n_times, s < sub_batch:
 *   key   = seed ^ 0xD6E8FEB86659FD93 (k0 = low 32 bits, k1 = high; no term index: every KKL term of a handle
 *           registered with one seed sees the same draw);
 *   U(a, b) = ((a << 32 | b) >> 11) * 2^-53 in [0, 1) from two Philox4x32-10 words;
 *   row 0:   c = philox({i, 0xFFFFFFFF, d_lo, d_hi}),  t_i = t_lb + (t_ub - t_lb) * U(c0, c1)  (the same for all s);
 *   rows 1 + 2j, 2 + 2j (pair j < ceil(n_z / 2); the second only while 2 + 2j <= n_z):
 *            c = philox({q, j, d_lo, d_hi ^ 0x4B4B4C00}), q = p (weak) or q = s (flags & PINN_KKL_STRONG: a path's
 *            z is bit-identical at all its times),
 *            u1 = 1 - U(c0, c1) in (0, 1], u2 = U(c2, c3), r = sqrt(-2 log u1),
 *            z_{1+2j} = r cos(2 pi u2), z_{2+2j} = r sin(2 pi u2) (Box-Muller, N(0, 1)),
 * computed in float64 (2 pi = 6.283185307179586) and rounded to the engine dtype.  The term must be a MEAN term (as
 * for pinn_set_sampler); n_times * sub_batch <= 2^31 - 1. */
enum { PINN_KKL_STRONG = 1 };
int pinn_set_sampler_kkl(pinn_handle h, int32_t term, int64_t n_times, int32_t sub_batch, int32_t n_z, double t_lb,
                         double t_ub, uint32_t flags, uint64_t seed, void* stream);
int pinn_resample(pinn_handle h, void* stream);
int pinn_get_points_host(pinn_handle h, int32_t term, void* host_pts);

/* max |dL_term/dtheta_i| and mean |dL_term/dtheta_i| of ONE term's unweighted loss (the other terms enter with
 * weight 0): what GradientScaleAdaptiveLoss needs per reweighting (reference src/adaptive_losses.jl:115-123 calls
 * Zygote.gradient(pde_loss_function, theta) per term and takes maximum(abs, .) / mean(abs, .) on the host; SURVEY 8(f).2).
 * One fused evaluation + one reduction launch; only the two scalars cross to the host.  Synchronises the stream. */
int pinn_term_grad_stats(pinn_handle h, int32_t term, const void* dev_theta, double* host_max_abs,
                         double* host_mean_abs, void* stream);
int pinn_term_grad_stats_host(pinn_handle h, int32_t term, const void* host_theta, double* host_max_abs,
                              double* host_mean_abs);

/* ---- device-resident optimizer loop (SURVEY section 8(f) item 1) ------------------------------------ */
/* Adam (Optimisers.Adam semantics: m, v, bias-corrected step) applied in the TAIL of the fused kernel, right after
 * the in-kernel gradient reduction (and, at nranks > 1, the peer-memory sum): a training iteration is ONE launch
 * (+ one sampler launch per sampled term, + the weight-pack launch on the 128-wide path) with no host round trip.
 * theta, m, v, the step counter and the sampler draw counter live in engine-owned device memory, so
 * pinn_adam_iterate captures its n_steps iterations once into a CUDA graph and replays it while the arguments
 * stay the same (PINN_B200_NO_GRAPH=1 disables the capture).  Point sets: fixed (Grid / fixed-node quadrature /
 * non-resampled) or drawn by the device-side samplers.  Multi-GPU: every rank applies the identical update to its
 * replica (needs the peer-memory path, see pinn_comm_info).  The reference's per-iteration host loop
 * (Optimization.solve + Zygote + Optimisers.Adam) is what this replaces. */
int pinn_adam_begin(pinn_handle h, const void* host_theta0, double lr, double beta1, double beta2, double eps);
/* run n_steps iterations; host_total (nullable) receives the loss of the LAST evaluated theta,
 * host_term_losses (nullable) its per-term losses.  Synchronises at the end. */
int pinn_adam_iterate(pinn_handle h, int32_t n_steps, const double* host_weights, void* host_total,
                      void* host_term_losses);
int pinn_adam_theta(pinn_handle h, void* host_theta_out);

/* ---- device-resident quasi-Newton (BFGS / L-BFGS) ------------------------------------------------------------------
 * The reference's users finish most PINNs with Optim's quasi-Newton methods through OptimizationOptimJL, e.g.
 *   BFGS()                               test/NNPDE1/nnpde__pde_iii_3rd_order_ode.jl:126, every IntegroDiff/ test
 *   BFGS(linesearch = BackTracking())    test/NNPDE1/nnpde__pde_ii_2d_poisson.jl:85 (polish after Adam)
 *   BFGS(initial_stepnorm = 0.01)        test/NNPDE2/direct_function__approximation_of_function_1d.jl:36
 *   LBFGS()                              test/NNPDE2/additional_loss__fokker_planck.jl:71
 * The options restate Optim's documented defaults: alphaguess = InitialStatic (the first trial step of every line search
 * is alpha = 1), LBFGS m = 10 with scaleinvH0 (H0 = gamma I, gamma = s'y / y'y of the newest pair; the first step is
 * along -g), BFGS H0 = I or I * initial_stepnorm / ||g0||_inf, convergence at ||g||_inf <= 1e-8 (g_abstol).
 * Line searches (LineSearches.jl defaults): HagerZhang delta 0.1, sigma 0.9, epsilon 1e-6, midpoint bisection, gamma 0.66,
 * rho 5, psi3 0.1, 50 iterations; BackTracking c_1 1e-4, rho_hi 0.5, rho_lo 0.1, order 3, 1000 iterations.
 * A pair with s'y <= 0 is not stored (L-BFGS) / does not update H (BFGS); a direction that is not a descent direction
 * resets the history / H to the identity and steps along -g.
 *
 * theta, g, the direction, the L-BFGS pairs ([m+1][n_theta] ring) and BFGS's dense H (n_theta x n_theta) are float64 on
 * the device for both engine dtypes; the fused kernel sees theta rounded to the engine dtype.  The line search runs on
 * the host: each evaluation copies {phi, phi'} (16 bytes) back and synchronises once.  Every reduction has a fixed
 * order and a grid that depends on n_theta only, so two runs -- and all ranks of a multi-GPU handle -- are bit-identical.
 * With device samplers registered every evaluation draws fresh points first (as pinn_resample).  BFGS is refused for
 * n_theta > 16384 (H would exceed 2 GiB). */
enum { PINN_QN_LBFGS = 0, PINN_QN_BFGS = 1 };
enum { PINN_LS_HAGERZHANG = 0, PINN_LS_BACKTRACKING = 1 };
/* status after pinn_qn_iterate: still iterating, converged (||g||_inf <= 1e-8, or an accepted step left theta
 * unchanged), or the line search failed (theta stays at the last accepted point) */
enum { PINN_QN_RUNNING = 0, PINN_QN_CONVERGED = 1, PINN_QN_LS_FAILED = 2 };
typedef struct {
  int32_t kind;              /* PINN_QN_*                                                  */
  int32_t m;                 /* L-BFGS history length (Optim default 10), 1..32            */
  int32_t linesearch;        /* PINN_LS_*                                                  */
  int32_t _pad;
  double initial_stepnorm;   /* BFGS: H0 = I * initial_stepnorm / ||g0||_inf; <= 0: H0 = I */
} pinn_qn_options;
/* Start from host theta0 (engine dtype): allocates the state and evaluates loss and gradient at theta0.
 * host_weights [n_terms] (nullable) stay fixed for the whole run.  Synchronises. */
int pinn_qn_begin(pinn_handle h, const void* host_theta0, const pinn_qn_options* opts, const double* host_weights);
/* Run up to n_iters iterations (accepted steps); the state persists across calls, so callers may iterate one step at a
 * time.  Outputs (each nullable): loss at the current theta, ||g||_inf there, PINN_QN_* status, iterations and loss /
 * gradient evaluations since pinn_qn_begin (the one at theta0 included).  Once stopped, further calls do nothing. */
int pinn_qn_iterate(pinn_handle h, int32_t n_iters, double* host_f, double* host_gnorm_inf, int32_t* host_status,
                    int64_t* host_iters, int64_t* host_evals);
/* current theta rounded to the engine dtype */
int pinn_qn_theta(pinn_handle h, void* host_theta_out);

/* ---- device-resident HMC sampler (BayesianPINN posteriors) --------------------------------------------------------
 * Samples the log density l(theta) = sum_k w_k L_k(theta) + ll_const + log N(theta; prior_mean, prior_std^2 I), where
 * L_k are the engine's term losses and w_k the host weights (for a BayesianPINN: w_k = -W n_k / (2 sigma_k^2) and
 * ll_const the Gaussian normalisation, so that the first two parts are full_loss_function(theta, allstd)).  With
 * pinn_hmc_begin_ex the last entries of theta (an inverse problem's theta.p) carry their own priors instead.
 * Hamiltonian Monte Carlo with a fixed number of leapfrog steps and end-point Metropolis acceptance, with AdvancedHMC's
 * defaults: find_good_stepsize for the initial step size, Nesterov dual averaging of the step size (gamma 0.05, t0 10,
 * kappa 0.75) and Stan's windowed diagonal mass-matrix adaptation (buffers 75 / 25 / 50) over the first n_adapts
 * transitions.  theta, the momentum, the gradient, M^-1 and the adaptation state are float64 on the device for both
 * engine dtypes; the fused kernel sees theta rounded to the engine dtype.  One transition is a fixed launch sequence with
 * no host decision, captured once into a CUDA graph (PINN_B200_NO_GRAPH=1: enqueued directly).  Random numbers are
 * Philox4x32-10 draws keyed by (seed, transition, index, stream), so two runs with one seed are bit-identical.
 * Single-GPU handles (nranks == 1) with fixed point sets only, unless pinn_hmc_begin_ex2 asks for PINN_HMC_REDRAW. */
enum { PINN_HMC_ADAPT_NONE = 0, PINN_HMC_ADAPT_STAN = 1 };
enum { PINN_HMC_METRIC_UNIT = 0, PINN_HMC_METRIC_DIAG = 1 };
/* columns of one statistics row of pinn_hmc_iterate */
enum {
  PINN_HMC_STAT_STEP_SIZE = 0, PINN_HMC_STAT_ACCEPTANCE_RATE = 1, PINN_HMC_STAT_IS_ACCEPT = 2,
  PINN_HMC_STAT_LOG_DENSITY = 3, PINN_HMC_STAT_HAMILTONIAN_ENERGY = 4, PINN_HMC_STAT_HAMILTONIAN_ENERGY_ERROR = 5,
  PINN_HMC_STAT_NUMERICAL_ERROR = 6, PINN_HMC_STAT_IS_ADAPT = 7, PINN_HMC_N_STATS = 8
};
typedef struct {
  int32_t n_leapfrog;        /* leapfrog steps per transition (HMC(0.1, 30): 30), >= 1                     */
  int32_t adaptor;           /* PINN_HMC_ADAPT_*                                                          */
  int32_t metric;            /* PINN_HMC_METRIC_*                                                         */
  int32_t n_adapts;          /* transitions 1..n_adapts adapt (AdvancedHMC: min(draws / 10, 1000)), >= 0  */
  double target_accept;      /* dual-averaging target acceptance rate delta, in (0, 1)                    */
  double step_size;          /* initial step size; <= 0: find_good_stepsize                               */
  double prior_mean, prior_std;   /* Normal prior of every parameter; prior_std > 0                       */
  uint64_t seed;
} pinn_hmc_options;
/* Start a chain at host_theta0 (float64 [n_theta]): allocates the state, evaluates l and its gradient there and, when
 * opts->step_size <= 0, runs find_good_stepsize (one synchronisation per trial).  host_weights [n_terms] (nullable:
 * all 1) and ll_const stay fixed for the chain.  *step_size_out (nullable): the initial step size. */
int pinn_hmc_begin(pinn_handle h, const double* host_theta0, const pinn_hmc_options* opts, const double* host_weights,
                   double ll_const, double* step_size_out);
/* Per-entry priors of the last n_tail entries of theta (parameter estimation: theta.p), as Distributions.jl defines
 * them: Normal(mu = a, sigma = b), LogNormal(mu = a, sigma = b) (of log x; support x > 0) and Uniform(a, b) (support
 * a <= x <= b).  Entry j applies to theta[n_theta - n_tail + j]; the Normal(prior_mean, prior_std^2) prior of the options
 * then covers the first n_theta - n_tail entries only.  A tail entry outside its support makes l = -Inf: the trajectory
 * stops and the proposal is rejected with numerical_error = 1. */
enum { PINN_HMC_PRIOR_NORMAL = 0, PINN_HMC_PRIOR_LOGNORMAL = 1, PINN_HMC_PRIOR_UNIFORM = 2 };
typedef struct {
  int32_t kind;              /* PINN_HMC_PRIOR_*                                                           */
  double a, b;               /* (mu, sigma > 0) or Uniform's bounds a < b; finite                         */
} pinn_hmc_prior;
/* pinn_hmc_begin with tail priors tail[n_tail], 0 <= n_tail <= PINN_MAX_PARAMS and n_tail < n_theta; n_tail = 0 is
 * pinn_hmc_begin.  theta0's tail must lie in the priors' supports. */
int pinn_hmc_begin_ex(pinn_handle h, const double* host_theta0, const pinn_hmc_options* opts, const double* host_weights,
                      double ll_const, const pinn_hmc_prior* tail, int32_t n_tail, double* step_size_out);
/* pinn_hmc_begin_ex with two additions (tail_logabs = NULL and flags = 0 is pinn_hmc_begin_ex):
 * - tail_logabs[n_tail] (nullable, finite): l gains sum_j tail_logabs[j] * log|theta_tail_j| and its gradient
 *   tail_logabs[j] / theta_tail_j -- the normalisation -n log|sigma(p)| of a Gaussian likelihood whose sigma is a
 *   monomial in theta.p.  Where such an entry is 0 the value is not finite: the proposal is rejected (numerical_error = 1).
 * - PINN_HMC_REDRAW: the handle's device samplers (pinn_set_sampler*) draw fresh points before every evaluation of the
 *   chain -- theta0, every find_good_stepsize trial, every leapfrog step.  Evaluation j since this call (j = 0 at
 *   theta0) uses draw index j (the sampler's draw argument 0 plus j), counted on the device, whether or not a trajectory
 *   has stopped early.  Without the flag a handle with a device sampler is refused.  A rejected proposal returns to the
 *   previous state with its cached log density and gradient. */
enum { PINN_HMC_REDRAW = 1u };
int pinn_hmc_begin_ex2(pinn_handle h, const double* host_theta0, const pinn_hmc_options* opts, const double* host_weights,
                       double ll_const, const pinn_hmc_prior* tail, int32_t n_tail, const double* tail_logabs,
                       uint32_t flags, double* step_size_out);
/* Run n transitions: host_samples [n][n_theta] float64 (theta after each transition) and host_stats
 * [n][PINN_HMC_N_STATS] (each nullable).  The chain continues across calls. */
int pinn_hmc_iterate(pinn_handle h, int32_t n, double* host_samples, double* host_stats);
/* the chain's current theta (float64 [n_theta]) */
int pinn_hmc_theta(pinn_handle h, double* host_theta_out);

/* ---- multi-GPU -------------------------------------------------------------------- */
/* Attach an NCCL communicator built from a 128-byte ncclUniqueId that the caller
 * distributed (rank 0 obtains it from pinn_comm_unique_id). */
int pinn_comm_unique_id(void* out_128_bytes);
int pinn_comm_init(pinn_handle h, const void* unique_id_128_bytes, int32_t rank, int32_t nranks);
/* pinn_comm_init also maps every rank's symmetric gradient buffer into this process (CUDA IPC over NVLink peer
 * access, handles exchanged through the communicator).  When that succeeds on all ranks the sum over ranks runs INSIDE
 * the fused kernel: each CTA publishes its slice of the reduced gradient, signals per-slice flags in the peers'
 * memory and adds the peers' slices in rank order -- no ncclAllReduce, no extra launch, identical bits on every
 * rank.  Otherwise (GPUs without peer access, ranks that are threads of one process, PINN_B200_NO_P2P=1) the step is
 * fused kernel -> ncclAllReduce -> unpack.  pinn_comm_info reports which: *fused_p2p = 1 / 0, and returns the reason
 * for a fallback ("" when none).  All ranks must issue the same sequence of pinn_loss_grad / pinn_adam_iterate calls
 * (SPMD), and synchronise with each other before destroying their handles. */
const char* pinn_comm_info(pinn_handle h, int32_t* fused_p2p);

/* ---- introspection ------------------------------------------------------------------ */
/* kernels launched by this handle since creation (bench.py's gpu_launches) */
int64_t pinn_launch_count(pinn_handle h);
/* device time (ms) of the main fused kernel in the most recent pinn_loss_grad, measured
 * with CUDA events on the launching stream; requires pinn_set_timing(h, 1). Blocks. */
int pinn_set_timing(pinn_handle h, int32_t enable);
double pinn_last_kernel_ms(pinn_handle h);
/* bytes of device workspace owned by the handle */
int64_t pinn_workspace_bytes(pinn_handle h);
/* algorithmic FLOPs of one pinn_loss_grad at the current point sets:
 * 6 * sum_terms N * sum_nets C * S  (SURVEY section 8(d)); an integral adds 2 q^n_dims integrand evaluations per point
 * of its owner term; a fixed network counts its forward pass only, 2 * C * S */
double pinn_flops_per_eval(pinn_handle h);
/* the q-point Gauss-Legendre rule on [-1, 1] that integral terms use (nodes ascending): x[q], w[q]; 1 <= q <= 64.
 * Host only, no device needed. */
int pinn_quadrature_nodes(int32_t q, double* x, double* w);

#ifdef __cplusplus
}
#endif
#endif /* PINN_B200_H */
