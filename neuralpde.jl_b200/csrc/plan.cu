// plan.cu -- host planner (plan.h): descriptor validation, θ and channel layout, the tensor-core pass split and the
// shared-memory layouts of the fused kernels.  Each stage below does one step and reports errors through fail().
#include <stdarg.h>
#include <stdio.h>
#include <string.h>
#include <algorithm>
#include <string>
#include "plan.h"

namespace pinn {
size_t ffma_smem_bytes(int dtype, long long buf_elems, int w_area, bool bufs_smem, bool integ);   // ffma_launch.cu

static thread_local std::string g_err;
int fail(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
  g_err = buf;
  return 1;
}
const char* last_error() { return g_err.c_str(); }

namespace {
// ---- networks and θ layout ------------------------------------------------------------------------------------------
// one network's layer offsets (from off: θ, or a fixed network's own buffer) and the FFMA path's staged (8-padded) weight
// layout; returns the end offset, or -1 after fail()
long long plan_net(const char* what, int k, int n_layers, const int32_t* dims, const int32_t* acts, long long off,
                   DevNet& n, int& max_w8, long long& resident) {
  if (n_layers < 1 || n_layers > PINN_MAX_LAYERS)
    return fail("pinn_create: %s %d has %d layers (supported 1..%d)", what, k, n_layers, PINN_MAX_LAYERS), -1;
  if (!dims || !acts) return fail("pinn_create: %s %d null dims/acts", what, k), -1;
  n.n_layers = n_layers;
  for (int l = 0; l <= n_layers; ++l) {
    if (dims[l] < 1) return fail("pinn_create: %s %d dims[%d]=%d must be >= 1", what, k, l, dims[l]), -1;
    n.dims[l] = dims[l];
    max_w8 = std::max(max_w8, (dims[l] + 7) & ~7);
  }
  if (n.dims[0] > PINN_MAX_IN) return fail("pinn_create: %s %d input dimension %d > %d", what, k, n.dims[0], PINN_MAX_IN), -1;
  for (int l = 0; l < n_layers; ++l) {
    if (acts[l] < PINN_ACT_IDENTITY || acts[l] > PINN_ACT_COS)
      return fail("pinn_create: %s %d layer %d unknown activation %d", what, k, l, acts[l]), -1;
    n.acts[l] = acts[l];
    n.w_off[l] = off; off += (long long)n.dims[l] * n.dims[l + 1];
    n.b_off[l] = off; off += n.dims[l + 1];
    int in8 = (n.dims[l] + 7) & ~7, out8 = (n.dims[l + 1] + 7) & ~7;
    n.ws_off[l] = (int)resident; resident += (long long)in8 * out8;
    n.bs_off[l] = (int)resident; resident += out8;
  }
  n.max_width8 = max_w8;   // running maximum over the networks planned so far
  return off;
}

// the trainable networks (θ layout), then the fixed ones (each from offset 0 of its own buffer; *fixed_len: its length)
int plan_nets(const pinn_problem_desc* d, const pinn_fixed_net_desc* fixed, int n_fixed, DevProblem& P, int& max_w8,
              long long& resident, long long* fixed_len) {
  for (int k = 0; k < d->n_nets; ++k) {
    const pinn_net_desc& nd = d->nets[k];
    if (nd.theta_offset < 0) return fail("pinn_create: net %d negative theta_offset", k);
    const long long off = plan_net("net", k, nd.n_layers, nd.dims, nd.acts, nd.theta_offset, P.nets[k], max_w8, resident);
    if (off < 0) return 1;
    if (off > d->n_theta)
      return fail("pinn_create: net %d parameters [%lld,%lld) exceed n_theta=%lld", k, (long long)nd.theta_offset, off,
                  (long long)d->n_theta);
  }
  for (int j = 0; j < n_fixed; ++j) {
    fixed_len[j] = plan_net("fixed network", j, fixed[j].n_layers, fixed[j].dims, fixed[j].acts, 0, P.fixed[j], max_w8,
                            resident);
    if (fixed_len[j] < 0) return 1;
  }
  return 0;
}

// network k of a tap: trainable (k < n_nets) or fixed network k - n_nets
const DevNet& net_ref(const DevProblem& P, int k) { return k < P.n_nets ? P.nets[k] : P.fixed[k - P.n_nets]; }

// ---- per-term channel planning ---------------------------------------------------------------------------------------
// lookups in a slot's channel set (-1: absent): direction x in dir1, second derivative (a, b), third along dir1[a]
int find_dir(const DevChan& ch, int x) { for (int j = 0; j < ch.n1; ++j) if (ch.dir1[j] == x) return j; return -1; }
int find_pair(const DevChan& ch, int a, int b) { for (int s = 0; s < ch.n2; ++s) if (ch.s_a[s] == a && ch.s_b[s] == b) return s; return -1; }
int find_third(const DevChan& ch, int a) { for (int q = 0; q < ch.n3; ++q) if (ch.t_a[q] == a) return q; return -1; }
// dir1 indices (a <= b) of the two directions of a second derivative
void dir_pair(const DevChan& ch, const int* dir, int& a, int& b) {
  a = find_dir(ch, dir[0]); b = find_dir(ch, dir[1]);
  if (a > b) std::swap(a, b);
}
// room for one more derivative channel
int check_room(const DevChan& ch, const char* what, int t, int net) {
  if (1 + ch.n1 + ch.n2 + ch.n3 < PINN_MAX_CH) return 0;
  return fail("pinn_create: %s %d network %d needs more than %d channels", what, t, net, PINN_MAX_CH);
}

// slots (the networks the term taps, in order of first use, with the point rows feeding their inputs), then the
// derivative channels of every slot: first derivatives (needed directly or as intermediates), then second and pure
// third derivatives (order 3 needs the pure second derivative along the same direction as an intermediate)
// (what, t: "term" / "integral" and its index, for the messages)
int plan_channels(const pinn_problem_desc* d, const pinn_term_desc& td, const char* what, int t, const DevProblem& P,
                  DevTerm& T, int* slot_of) {
  const int n_all = d->n_nets + P.n_fixed;
  for (int k = 0; k < kMaxAllNets; ++k) slot_of[k] = -1;
  T.n_used = 0;
  for (int i = 0; i < td.n_taps; ++i) {
    const pinn_tap_desc& tp = td.taps[i];
    if (tp.net < 0 || tp.net >= n_all)
      return fail("pinn_create: %s %d tap %d names network %d (the problem has %d trainable and %d fixed networks)", what,
                  t, i, tp.net, d->n_nets, P.n_fixed);
    if (slot_of[tp.net] >= 0) continue;
    if (T.n_used == PINN_MAX_NETS)
      return fail("pinn_create: %s %d taps more than %d networks", what, t, PINN_MAX_NETS);
    slot_of[tp.net] = T.n_used;
    T.used_net[T.n_used] = tp.net;
    DevChan& ch = T.chan[T.n_used];   // zeroed with the plan: no derivative channels yet
    for (int j = 0; j < net_ref(P, tp.net).dims[0]; ++j) {
      int r = td.net_rows[tp.net * PINN_MAX_IN + j];
      if (r < 0 || r >= td.dim)
        return fail("pinn_create: %s %d network %d input %d maps to point row %d (dim=%d)", what, t, tp.net, j, r, td.dim);
      ch.rows[j] = r;
    }
    ++T.n_used;
  }
  for (int i = 0; i < td.n_taps; ++i) {
    const pinn_tap_desc& tp = td.taps[i];
    const DevNet& n = net_ref(P, tp.net);
    DevChan& ch = T.chan[slot_of[tp.net]];
    if (tp.order < 0 || tp.order > 3)
      return fail("pinn_create: %s %d tap %d has derivative order %d; orders 0..3 are supported (order 4 and mixed "
                  "third derivatives are not)", what, t, i, tp.order);
    if (tp.order == 3 && !(tp.dir[0] == tp.dir[1] && tp.dir[1] == tp.dir[2]))
      return fail("pinn_create: %s %d tap %d is a mixed third derivative; only pure third derivatives d^3/dx_i^3 are "
                  "supported", what, t, i);
    if (tp.out < 0 || tp.out >= n.dims[n.n_layers])
      return fail("pinn_create: %s %d tap %d output component %d out of range", what, t, i, tp.out);
    for (int q = 0; q < tp.order; ++q)
      if (tp.dir[q] < 0 || tp.dir[q] >= n.dims[0])
        return fail("pinn_create: %s %d tap %d direction %d out of range for a %d-input network", what, t, i, tp.dir[q],
                    n.dims[0]);
    for (int q = 0; q < tp.order; ++q)
      if (find_dir(ch, tp.dir[q]) < 0) ch.dir1[ch.n1++] = tp.dir[q];
  }
  for (int i = 0; i < td.n_taps; ++i) {
    const pinn_tap_desc& tp = td.taps[i];
    if (tp.order < 2) continue;
    DevChan& ch = T.chan[slot_of[tp.net]];
    int a, b;
    dir_pair(ch, tp.dir, a, b);
    if (find_pair(ch, a, b) < 0) {
      if (check_room(ch, what, t, tp.net)) return 1;
      ch.s_a[ch.n2] = a; ch.s_b[ch.n2] = b; ++ch.n2;
    }
    if (tp.order == 3 && find_third(ch, a) < 0) {
      if (check_room(ch, what, t, tp.net)) return 1;
      ch.t_a[ch.n3++] = a;
    }
  }
  return 0;
}

// canonical channel order: directions that carry a pure second derivative come first, so that (when every
// second-derivative channel is pure) channel n1+1+s is d2/d(dir1[s])^2
void canonical_order(DevChan& ch) {
  int order[PINN_MAX_IN], inv[PINN_MAX_IN] = {}, n = 0;
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
    ch.t_s[q] = find_pair(ch, ch.t_a[q], ch.t_a[q]);
  }
}

// ---- tap mapping and the residual program ----------------------------------------------------------------------------
// PINN_OP_INTEGRAL a (terms only) becomes a TAP of index n_taps + k, k = the rank of integral a among the term's
// integrals: the fused kernel stores the integral's value there
int plan_taps(const pinn_problem_desc* d, const pinn_term_desc& td, const char* what, int t, const int* slot_of,
              const pinn_integral_desc* integrals, int n_integrals, DevTerm& T) {
  for (int i = 0; i < td.n_taps; ++i) {
    const pinn_tap_desc& tp = td.taps[i];
    const DevChan& ch = T.chan[slot_of[tp.net]];
    int a, b;
    T.tap_slot[i] = slot_of[tp.net];
    T.tap_out[i] = tp.out;
    if (tp.order == 0) T.tap_ch[i] = 0;
    else if (tp.order == 1) T.tap_ch[i] = 1 + find_dir(ch, tp.dir[0]);
    else if (tp.order == 2) { dir_pair(ch, tp.dir, a, b); T.tap_ch[i] = 1 + ch.n1 + find_pair(ch, a, b); }
    else T.tap_ch[i] = 1 + ch.n1 + ch.n2 + find_third(ch, find_dir(ch, tp.dir[0]));
  }
  bool any_tap = false, any_param = false;
  const bool is_term = strcmp(what, "term") == 0;
  for (int i = 0; i < td.n_instr; ++i) {
    const pinn_instr& in = td.prog[i];
    DevInstr& o = T.prog[i];
    o.op = in.op; o.a = in.a; o.b = in.b; o.pad = 0; o.imm = in.imm;
    auto val_ok = [&](int v) { return v >= 0 && v < i; };
    switch (in.op) {
      case PINN_OP_CONST: break;
      case PINN_OP_COORD:
        if (in.a < 0 || in.a >= td.dim) return fail("pinn_create: %s %d instr %d COORD row %d out of range", what, t, i, in.a);
        break;
      case PINN_OP_TAP:
        if (in.a < 0 || in.a >= td.n_taps) return fail("pinn_create: %s %d instr %d TAP %d out of range", what, t, i, in.a);
        any_tap = true;
        break;
      case PINN_OP_PARAM:
        if (in.a < 0 || in.a >= d->n_params) return fail("pinn_create: %s %d instr %d PARAM %d out of range", what, t, i, in.a);
        any_param = true;
        break;
      case PINN_OP_INTEGRAL: {
        if (!is_term) return fail("pinn_create: integral %d instr %d: integrals nested in an integrand are not supported", t, i);
        if (n_integrals == 0)
          return fail("pinn_create: term %d instr %d reads an integral; integral terms are created with pinn_create_ex", t, i);
        if (in.a < 0 || in.a >= n_integrals) return fail("pinn_create: term %d instr %d INTEGRAL %d out of range", t, i, in.a);
        if (integrals[in.a].owner != t)
          return fail("pinn_create: term %d instr %d reads integral %d, which belongs to term %d", t, i, in.a,
                      integrals[in.a].owner);
        int k = 0;
        for (int j = 0; j < in.a; ++j) k += integrals[j].owner == t;
        o.op = PINN_OP_TAP; o.a = td.n_taps + k;
        any_tap = true;
      } break;
      case PINN_OP_ADD: case PINN_OP_SUB: case PINN_OP_MUL: case PINN_OP_DIV: case PINN_OP_POW:
        if (!val_ok(in.a) || !val_ok(in.b)) return fail("pinn_create: %s %d instr %d operand out of range", what, t, i);
        break;
      case PINN_OP_NEG: case PINN_OP_POWI: case PINN_OP_SIN: case PINN_OP_COS: case PINN_OP_EXP:
      case PINN_OP_LOG: case PINN_OP_TANH: case PINN_OP_SQRT: case PINN_OP_ABS:
        if (!val_ok(in.a)) return fail("pinn_create: %s %d instr %d operand out of range", what, t, i);
        break;
      default:
        return fail("pinn_create: %s %d instr %d unknown opcode %d", what, t, i, in.op);
    }
  }
  // a term without taps is a parameter-only term (plan_term): its program must read theta.p instead
  if (!any_tap && !(is_term && td.n_taps == 0 && any_param))
    return fail("pinn_create: %s %d %s program never reads a tap (nothing depends on theta)", what, t,
                is_term ? "residual" : "integrand");
  return 0;
}

// the networks of a term or an integrand: channels, the FFMA stash layout (stash_max: scalars per CTA), taps and program;
// *flops: algorithmic flops per point, 6 * sum_nets C * S
int plan_body(const pinn_problem_desc* d, const pinn_term_desc& td, const char* what, int t, DevProblem& P, DevTerm& T,
              const pinn_integral_desc* integrals, int n_integrals, int& max_c, long long& stash_max, double* flops) {
  if (td.n_taps > PINN_MAX_TAPS) return fail("pinn_create: %s %d has %d taps (max %d)", what, t, td.n_taps, PINN_MAX_TAPS);
  if (td.n_instr < 1 || td.n_instr > PINN_MAX_INSTR)
    return fail("pinn_create: %s %d program length %d out of range [1,%d]", what, t, td.n_instr, PINN_MAX_INSTR);
  if (!td.taps || !td.prog || !td.net_rows) return fail("pinn_create: %s %d null taps/prog/net_rows", what, t);
  T.dim = td.dim; T.n_taps = td.n_taps; T.n_instr = td.n_instr;
  int slot_of[kMaxAllNets];
  if (plan_channels(d, td, what, t, P, T, slot_of)) return 1;
  long long stash = 0;
  double f = 0;
  for (int s = 0; s < T.n_used; ++s) {
    DevChan& ch = T.chan[s];
    canonical_order(ch);
    ch.C = 1 + ch.n1 + ch.n2 + ch.n3;
    if (ch.C > PINN_MAX_CH) return fail("pinn_create: %s %d needs %d channels (max %d)", what, t, ch.C, PINN_MAX_CH);
    max_c = std::max(max_c, ch.C);
    const DevNet& n = net_ref(P, T.used_net[s]);
    const bool fixed = T.used_net[s] >= P.n_nets;   // forward only: no stash, no reverse sweep
    double S = 0;
    for (int l = 0; l < n.n_layers; ++l) {
      ch.stash_off[l] = (int)stash;
      if (!fixed) stash += (long long)ch.C * n.dims[l + 1] * kTilePts;
      S += (double)n.dims[l] * n.dims[l + 1];
    }
    f += (fixed ? 2.0 : 6.0) * ch.C * S;
  }
  stash_max = std::max(stash_max, stash);
  if (plan_taps(d, td, what, t, slot_of, integrals, n_integrals, T)) return 1;
  *flops = f;
  return 0;
}

// one term
int plan_term(const pinn_problem_desc* d, int t, const pinn_integral_desc* integrals, int n_integrals, DevProblem& P,
              TermPlan& tp, int& max_c, long long& stash_max) {
  const pinn_term_desc& td = d->terms[t];
  DevTerm& T = P.terms[t];
  int n_own = 0;
  for (int i = 0; i < n_integrals; ++i) n_own += integrals[i].owner == t;
  if (td.dim < 1 || td.dim > PINN_MAX_DIM) return fail("pinn_create: term %d dim=%d out of range [1,%d]", t, td.dim, PINN_MAX_DIM);
  // a term without taps or integrals is accepted when its program reads theta.p: a parameter-only term (such as an
  // Euler-Maruyama data loss), for which the FFMA kernel runs the residual program alone -- no network is staged,
  // propagated, stashed or swept back, and the adjoint reaches theta.p through the program's PARAM reads
  bool reads_param = false;
  for (int i = 0; i < td.n_instr && td.prog; ++i) reads_param = reads_param || td.prog[i].op == PINN_OP_PARAM;
  if (td.n_taps < 1 && n_own == 0 && !reads_param)
    return fail("pinn_create: term %d has no network taps (an equation such as 0 ~ 0 cannot be trained on)", t);
  if (td.n_taps + n_own > PINN_MAX_TAPS)
    return fail("pinn_create: term %d has %d taps and %d integrals (max %d together)", t, td.n_taps, n_own, PINN_MAX_TAPS);
  if (td.reduction < PINN_REDUCE_MEAN || td.reduction > PINN_REDUCE_SQUARE_OF_SUM)
    return fail("pinn_create: term %d unknown reduction %d", t, td.reduction);
  const bool func = td.reduction == PINN_REDUCE_ABS_OF_SUM || td.reduction == PINN_REDUCE_SQUARE_OF_SUM;
  if (func) {    // a functional term: g(scale * sum_p w_p v_p) (the kernel reads its nullable weights itself)
    if (!ffma_kernel_mode(d->mode))
      return fail("pinn_create: term %d is a functional term; functional terms run on the FFMA path (mode PINN_MODE_FFMA)", t);
    if (P.func_term >= 0)
      return fail("pinn_create: term %d is a second functional term (term %d is one); a problem has at most one", t,
                  P.func_term);
    if (n_own > 0)
      return fail("pinn_create: term %d is a functional term and owns integral terms; its program may not read "
                  "PINN_OP_INTEGRAL", t);
    for (int i = 0; i < td.n_instr && td.prog; ++i)
      if (td.prog[i].op == PINN_OP_INTEGRAL)
        return fail("pinn_create: term %d is a functional term and its program reads PINN_OP_INTEGRAL (instr %d); "
                    "integrals inside a functional term are not supported", t, i);
    P.func_term = t;
    P.func_square = td.reduction == PINN_REDUCE_SQUARE_OF_SUM ? 1 : 0;
  }
  T.weighted = td.reduction == PINN_REDUCE_WSUM;
  tp.reduction = td.reduction;
  tp.scale = td.reduction == PINN_REDUCE_MEAN ? 1.0 : td.scale;
  return plan_body(d, td, "term", t, P, T, integrals, n_integrals, max_c, stash_max, &tp.flops_per_point);
}

// ---- integral terms ---------------------------------------------------------------------------------------------------
}  // namespace

// q-point Gauss-Legendre rule on [-1, 1]: Newton's method on P_q from the Chebyshev-like first guess
void gauss_legendre(int q, double* x, double* w) {
  const double pi = 3.14159265358979323846;
  // P_q(z) and P_q'(z) by the three-term recurrence
  auto legendre = [q](double z, double& dp) {
    double p0 = 1.0, p1 = 0.0;
    for (int j = 1; j <= q; ++j) { const double p2 = p1; p1 = p0; p0 = ((2.0 * j - 1.0) * z * p1 - (j - 1.0) * p2) / j; }
    dp = q * (z * p0 - p1) / (z * z - 1.0);
    return p0;
  };
  for (int i = 0; i < q; ++i) {
    double z = cos(pi * (i + 0.75) / (q + 0.5)), dp = 1.0;
    for (int it = 0; it < 100; ++it) {
      const double dz = legendre(z, dp) / dp;
      z -= dz;
      if (fabs(dz) < 1e-16) break;
    }
    legendre(z, dp);              // the weight from the derivative at the converged node
    x[q - 1 - i] = z;             // ascending, as numpy.polynomial.legendre.leggauss
    w[q - 1 - i] = 2.0 / ((1.0 - z * z) * dp * dp);
  }
}

namespace {

// one integral: geometry, node table and the integrand (a term over the node point); *flops: per owner point
int plan_integral(const pinn_problem_desc* d, const pinn_integral_desc* integrals, int n_integrals, int i, DevProblem& P,
                  int& max_c, long long& stash_max, double* flops) {
  const pinn_integral_desc& id = integrals[i];
  DevIntegral& I = P.integ[i];
  if (id.owner < 0 || id.owner >= d->n_terms) return fail("pinn_create: integral %d owner term %d out of range", i, id.owner);
  const int odim = d->terms[id.owner].dim;
  if (id.n_dims < 1 || id.n_dims > 2)
    return fail("pinn_create: integral %d has %d integrating dimensions (supported 1 or 2)", i, id.n_dims);
  if (id.q < 1 || id.q > PINN_MAX_QUAD)
    return fail("pinn_create: integral %d has q=%d Gauss-Legendre nodes per dimension (supported 1..%d)", i, id.q, PINN_MAX_QUAD);
  I.owner = id.owner; I.n_dims = id.n_dims; I.q = id.q;
  for (int k = 0; k < 2; ++k) { I.row[k] = 0; I.lb_row[k] = I.ub_row[k] = -1; I.inf_kind[k] = PINN_INF_NONE; }
  for (int k = 0; k < id.n_dims; ++k) {
    if (id.row[k] < 0 || id.row[k] >= odim)
      return fail("pinn_create: integral %d integrating row %d out of range (owner dim=%d)", i, id.row[k], odim);
    if (id.lb_row[k] < -1 || id.lb_row[k] >= odim || id.ub_row[k] < -1 || id.ub_row[k] >= odim)
      return fail("pinn_create: integral %d bound row out of range (owner dim=%d)", i, odim);
    if (id.inf_kind[k] < PINN_INF_NONE || id.inf_kind[k] > PINN_INF_LOWER)
      return fail("pinn_create: integral %d unknown infinite-bound kind %d", i, id.inf_kind[k]);
    I.row[k] = id.row[k]; I.lb_row[k] = id.lb_row[k]; I.ub_row[k] = id.ub_row[k]; I.inf_kind[k] = id.inf_kind[k];
    I.lb[k] = id.lb[k]; I.ub[k] = id.ub[k]; I.shift[k] = id.shift[k];
  }
  if (id.n_dims == 2 && id.row[0] == id.row[1]) return fail("pinn_create: integral %d integrates row %d twice", i, id.row[0]);
  gauss_legendre(id.q, I.xi, I.wq);
  I.slot = d->terms[id.owner].n_taps;
  for (int j = 0; j < i; ++j) I.slot += integrals[j].owner == id.owner;
  pinn_term_desc td;
  memset(&td, 0, sizeof td);
  td.dim = odim + id.n_dims; td.n_taps = id.n_taps; td.taps = id.taps; td.net_rows = id.net_rows;
  td.n_instr = id.n_instr; td.prog = id.prog;
  if (td.n_taps < 1) return fail("pinn_create: integral %d has no network taps", i);
  double f = 0;
  if (plan_body(d, td, "integral", i, P, I.body, integrals, n_integrals, max_c, stash_max, &f)) return 1;
  double nodes = id.q;
  if (id.n_dims == 2) nodes *= id.q;
  *flops = 2.0 * nodes * f;     // the forward pass, and again in the reverse sweep (recomputed per node tile)
  return 0;
}

// ---- FFMA geometry: the first shared-memory option that fits ---------------------------------------------------------
int plan_ffma(int dtype, int max_w8, long long resident, int max_c, long long stash_max, int max_smem, Plan& p) {
  FfmaArgs& a = p.ffma;
  const int TP = kTilePts + 16 / (dtype == PINN_F64 ? 8 : 4);
  a.ldc = max_w8 * TP; a.buf_elems = (long long)max_c * a.ldc; a.stash_per_cta = (stash_max + 3) & ~3LL;
  const long long panel = (long long)(kWarps * 8) * max_w8 + kWarps * 8;   // 64 x max_width8 (+ bias)
  const struct { bool bufs, res; } opts[3] = {{true, true}, {true, false}, {false, false}};
  for (const auto& o : opts) {
    long long wa = o.res ? resident : panel;
    wa = (wa + 3) & ~3LL;
    if (wa > (1LL << 30)) continue;
    size_t need = ffma_smem_bytes(dtype, a.buf_elems, (int)wa, o.bufs, p.integ || p.func);   // FUNC runs with INTEG
    if (need <= (size_t)max_smem) {
      p.bufs_smem = o.bufs; a.weights_resident = o.res ? 1 : 0; a.w_area = (int)wa; p.smem = need;
      return 0;
    }
  }
  return fail("pinn_create: a %d-wide layer panel does not fit in shared memory (%d bytes)", max_w8, max_smem);
}

// ---- tensor-core support checks --------------------------------------------------------------------------------------
TcCommonArgs& tc_common(Plan& p) { return p.wide ? static_cast<TcCommonArgs&>(p.tw) : static_cast<TcCommonArgs&>(p.tc); }

// network shapes; sets p.wide, net_ak and tl_max (most tensor layers of a network)
int check_tc_nets(const pinn_problem_desc* d, const DevProblem& P, Plan& p, int& tl_max) {
  if (d->dtype != PINN_F32) return fail("pinn_create: the tensor-core modes compute in bf16/fp32 and need dtype PINN_F32");
  for (int t = 0; t < d->n_terms; ++t)
    for (int s = 0; s < P.terms[t].n_used; ++s)
      if (P.terms[t].chan[s].n3 > 0)
        return fail("pinn_create(tc): term %d takes a third derivative; the tensor-core path propagates derivatives up to order 2 "
                    "(use PINN_MODE_FFMA)", t);
  tl_max = 0;
  bool wide = false, x256 = false;
  for (int k = 0; k < d->n_nets; ++k) {
    const DevNet& n = P.nets[k];
    if (n.n_layers < 2) return fail("pinn_create(tc): net %d needs at least 2 Dense layers", k);
    if (n.dims[n.n_layers] != 1) return fail("pinn_create(tc): net %d must have a 1-dimensional output", k);
    if (n.acts[n.n_layers - 1] != PINN_ACT_IDENTITY)
      return fail("pinn_create(tc): net %d: the last layer must be linear (identity activation)", k);
    for (int l = 0; l < n.n_layers; ++l)
      if (n.acts[l] == PINN_ACT_GELU || n.acts[l] == PINN_ACT_LOGCOSH || n.acts[l] == PINN_ACT_COS)
        return fail("pinn_create(tc): net %d layer %d: %s layers run on the FFMA path (PINN_MODE_FFMA, or "
                    "PINN_MODE_TC_F64 for Float64)", k, l,
                    n.acts[l] == PINN_ACT_GELU ? "gelu" : n.acts[l] == PINN_ACT_LOGCOSH ? "logcosh" : "cos");
    for (int l = 1; l < n.n_layers; ++l) {
      if (n.dims[l] > 64) wide = true;
      if (n.dims[l] == 192 || n.dims[l] == 256) x256 = true;
    }
    if (n.n_layers - 2 > kTcMaxTL)
      return fail("pinn_create(tc): net %d has %d hidden->hidden layers (max %d)", k, n.n_layers - 2, kTcMaxTL);
    tl_max = std::max(tl_max, n.n_layers - 2);
  }
  if (x256) {     // the 256-wide kernel: every hidden width a multiple of 64 up to 256
    if (d->mode != PINN_MODE_TC_BF16)
      return fail("pinn_create(tc): PINN_MODE_TC_SPLIT supports hidden widths up to 64; 192- and 256-wide layers run in "
                  "PINN_MODE_TC_BF16 (or PINN_MODE_FFMA for fp32 accuracy)");
    for (int k = 0; k < d->n_nets; ++k) {
      const DevNet& n = P.nets[k];
      for (int l = 1; l < n.n_layers; ++l)
        if (n.dims[l] % 64 != 0 || n.dims[l] > kTxW)
          return fail("pinn_create(tc): net %d hidden width %d: networks with 192- or 256-wide layers need every hidden "
                      "width to be a multiple of 64 up to %d on the tensor-core path (use PINN_MODE_FFMA for other shapes)",
                      k, n.dims[l], kTxW);
      if (n.n_layers < 3)
        return fail("pinn_create(tc): net %d: the 256-wide tensor-core path needs at least one hidden->hidden layer", k);
    }
  }
  for (int k = 0; !x256 && k < d->n_nets; ++k) {
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
  p.wide = wide;
  p.x256 = x256;
  for (int k = 0; k < PINN_MAX_NETS; ++k)    // 1: every hidden activation is tanh (fast path), 0: generic
    tc_common(p).net_ak[k] = std::all_of(P.nets[k].acts, P.nets[k].acts + std::max(P.nets[k].n_layers - 1, 0),
                                         [](int act) { return act == PINN_ACT_TANH; });
  return 0;
}

// channel sets and taps of every (split) term; the most slots of a term and channels of a slot
// (max_taps: kTcMaxTaps, or kTxMaxTaps on the 256-wide kernel, whose misc region is sized for the problem's taps)
int check_tc_terms(const DevProblem& P, bool wide, int max_taps, int& n_used_max, int& max_c) {
  n_used_max = 1; max_c = 1;
  for (int t = 0; t < P.n_terms; ++t) {
    const DevTerm& T = P.terms[t];
    if (T.n_used == 0)
      return fail("pinn_create(tc): term %d reads no network (a parameter-only term); parameter-only terms run on the FFMA "
                  "path (PINN_MODE_FFMA, or PINN_MODE_TC_F64 for Float64)", t);
    if (T.n_taps > max_taps) return fail("pinn_create(tc): term %d has %d taps (tensor-core path: max %d)", t, T.n_taps, max_taps);
    n_used_max = std::max(n_used_max, T.n_used);
    for (int s = 0; s < T.n_used; ++s) {
      const DevChan& ch = T.chan[s];
      max_c = std::max(max_c, ch.C);
      const int key = ch.n1 * 8 + ch.n2;
      const int ok[] = {0, 8, 16, 24, 32, 9, 17, 25, 18};
      const bool found = std::find(ok, ok + 9, key) != ok + 9;
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
  return 0;
}

// ---- wide-path pass split --------------------------------------------------------------------------------------------
// A network that needs more than kTwMaxC channels is evaluated in several passes ("slots") over the same weights, each
// with the value channel and a subset of the derivative directions (first-fit over the directions, a direction with a
// pure second derivative costs 2 channels).  The passes recompute the value channel; the gradient contributions add up
// in the per-CTA partial.
int split_passes(int t, DevTerm& T) {
  if (std::none_of(T.chan, T.chan + T.n_used, [](const DevChan& ch) { return ch.C > kTwMaxC; })) return 0;
  int n_new = 0, new_net[PINN_MAX_NETS], first_new[PINN_MAX_NETS];
  DevChan nch[PINN_MAX_NETS];
  int dir_slot[PINN_MAX_NETS][PINN_MAX_IN], dir_pos[PINN_MAX_NETS][PINN_MAX_IN];
  auto too_many = [&]() { return fail("pinn_create(tc): term %d needs more than %d network passes", t, PINN_MAX_NETS); };
  for (int s = 0; s < T.n_used; ++s) {
    const DevChan& ch = T.chan[s];
    first_new[s] = n_new;
    if (ch.C <= kTwMaxC) {
      if (n_new >= PINN_MAX_NETS) return too_many();
      for (int j = 0; j < ch.n1; ++j) { dir_slot[s][j] = n_new; dir_pos[s][j] = j; }
      new_net[n_new] = T.used_net[s]; nch[n_new] = ch; ++n_new;
      continue;
    }
    if (!ch.pure)
      return fail("pinn_create(tc): term %d needs %d channels including mixed second derivatives; the 128-wide tensor-core "
                  "path splits only pure second derivatives into passes (use PINN_MODE_FFMA)", t, ch.C);
    bool placed[PINN_MAX_IN] = {false};
    int left = ch.n1;
    while (left > 0) {
      if (n_new >= PINN_MAX_NETS) return too_many();
      DevChan g;
      memset(&g, 0, sizeof g);
      for (int j = 0; j < PINN_MAX_IN; ++j) g.rows[j] = ch.rows[j];
      int cost = 0;
      for (int j = 0; j < ch.n1; ++j) {          // pure directions (cost 2) come first in the canonical order
        const int cj = 1 + (j < ch.n2 ? 1 : 0);
        if (placed[j] || cost + cj > kTwMaxC - 1) continue;
        placed[j] = true; --left; cost += cj;
        dir_slot[s][j] = n_new; dir_pos[s][j] = g.n1;
        g.dir1[g.n1++] = ch.dir1[j];
        if (j < ch.n2) ++g.n2;
      }
      for (int q = 0; q < g.n2; ++q) g.s_a[q] = g.s_b[q] = q;
      g.pure = 1; g.C = 1 + g.n1 + g.n2;
      new_net[n_new] = T.used_net[s]; nch[n_new] = g; ++n_new;
    }
  }
  for (int i = 0; i < T.n_taps; ++i) {
    const int os = T.tap_slot[i], tch = T.tap_ch[i];
    const DevChan& ch = T.chan[os];
    if (tch == 0) { T.tap_slot[i] = first_new[os]; T.tap_ch[i] = 0; }
    else if (tch <= ch.n1) { T.tap_slot[i] = dir_slot[os][tch - 1]; T.tap_ch[i] = 1 + dir_pos[os][tch - 1]; }
    else {
      const int q = tch - 1 - ch.n1;          // pure: second-derivative channel q belongs to direction q
      const int ns = dir_slot[os][q];
      T.tap_slot[i] = ns; T.tap_ch[i] = 1 + nch[ns].n1 + dir_pos[os][q];
    }
  }
  T.n_used = n_new;
  for (int s = 0; s < n_new; ++s) { T.used_net[s] = new_net[s]; T.chan[s] = nch[s]; }
  return 0;
}

// ---- tensor-core shared-memory layout --------------------------------------------------------------------------------
// P operand tiles, the kernel's own regions, the 1 KB ones atom, one fp32 parameter block per network, (wide: the DevNet
// copy,) the misc region; the kernel's static shared memory takes the last 1 KB of the limit
int plan_tc_smem(const DevProblem& P, int max_c, int max_smem, Plan& p) {
  TcCommonArgs& c = tc_common(p);
  size_t off = 0;
  auto take = [&](size_t bytes) { const int o = (int)off; off += bytes; return o; };
  for (int k = 0; k < PINN_MAX_NETS; ++k) p.tw.off_fp[k] = p.tc.nets[k].fp = -1;
  if (p.wide) {
    c.off_P = take((size_t)max_c * kTwNB * kTileBytes);
    p.tw.off_S = take((size_t)2 * kTwImgBytes);
  } else {
    // P also holds the reverse sweep's four 16 KB weight-gradient partials (tc_kernel.cu net_backward): four tiles at least
    c.off_P = take((size_t)std::max(max_c, 4) * kTileBytes);
    p.tc.off_Q = take((size_t)max_c * kTileBytes);
    p.tc.off_Q_bytes = max_c * kTileBytes;
    for (int k = 0; k < P.n_nets; ++k)
      for (int l = 0; l < P.nets[k].n_layers - 2; ++l) {
        TcNetSmem& n = p.tc.nets[k];
        n.w_hi[l] = take(8192);
        n.w_lo[l] = p.tc.split ? take(8192) : n.w_hi[l];
      }
  }
  c.off_ones = take(1024);      // 1024-aligned: the regions before it are multiples of 8 KB
  if (p.x256) {     // one fp32 block, staged for each pass
    p.tw.off_fp[0] = take(((size_t)FpBlock<kTxW>::SIZE * 4 + 15) & ~size_t(15));
  } else {
    const size_t fp_bytes = ((size_t)(p.wide ? FpBlock<kTwW>::SIZE : FpBlock<kTcW>::SIZE) * 4 + 15) & ~size_t(15);
    for (int k = 0; k < P.n_nets; ++k) (p.wide ? p.tw.off_fp[k] : p.tc.nets[k].fp) = take(fp_bytes);
  }
  if (p.wide) p.tw.off_nets = take(((size_t)P.n_nets * sizeof(DevNet) + 15) & ~size_t(15));
  c.off_misc = take(tc_misc_bytes(c.mx_dim, c.mx_taps));
  if (off + 1024 > (size_t)max_smem)
    return fail("pinn_create(tc): the problem needs %zu bytes of shared memory per CTA (limit %d): %s", off, max_smem,
                p.x256 ? "too many channels or taps for the 256-wide tensor-core path"
                : p.wide ? "too many networks for the 128-wide tensor-core path"
                         : "too many resident weight tiles / channels for the tensor-core path");
  p.smem = off;
  return 0;
}

int plan_tc(const pinn_problem_desc* d, int max_smem, Plan& p) {
  DevProblem& P = p.prob;
  int tl_max, n_used_max, max_c;
  if (check_tc_nets(d, P, p, tl_max)) return 1;
  for (int t = 0; p.wide && t < d->n_terms; ++t)
    if (split_passes(t, P.terms[t])) return 1;
  if (check_tc_terms(P, p.wide, p.x256 ? kTxMaxTaps : kTcMaxTaps, n_used_max, max_c)) return 1;
  TcCommonArgs& c = tc_common(p);
  c.tl_max = std::max(tl_max, 1);
  c.mx_dim = 1; c.mx_taps = 1;
  for (int t = 0; t < d->n_terms; ++t) { c.mx_dim = std::max(c.mx_dim, P.terms[t].dim); c.mx_taps = std::max(c.mx_taps, P.terms[t].n_taps); }
  p.tc.split = d->mode == PINN_MODE_TC_SPLIT ? 1 : 0;
  if (plan_tc_smem(P, max_c, max_smem, p)) return 1;
  if (p.x256) {
    // per channel of a pass and half tile: inputs of the tensor layers + the last hidden activations (4 tiles each), fp32
    // pre-activations; channels of the term with the most (sum over its passes of 2 C, tc_x256_kernel.cu tx_chan0)
    long long nch = 1;
    for (int t = 0; t < d->n_terms; ++t) {
      long long n = 0;
      for (int s = 0; s < P.terms[t].n_used; ++s) n += 2 * P.terms[t].chan[s].C;
      nch = std::max(nch, n);
    }
    p.tw.hstash_per_cta = nch * (c.tl_max + 1) * 4 * kTxTileBytes;
    p.tw.zstash_per_cta = nch * c.tl_max * kTxW * kTxPts;      // floats
  }
  if (p.wide && !p.x256) {
    // per pass: inputs of the tl_max tensor layers + the last hidden activations (restored for multi-pass terms)
    p.tw.hstash_per_cta = (long long)n_used_max * (tl_max + 1) * kTwMaxC * kTwNB * kTileBytes;
    p.tw.zstash_per_cta = (long long)n_used_max * tl_max * kTwMaxC * 64 * kTcPts * 2;      // floats
  }
  if (p.wide) {      // one packed weight image per tensor layer
    for (int k = 0; k < d->n_nets; ++k) {
      p.tw.wimg[k] = p.pack.n_images;
      for (int l = 1; l <= P.nets[k].n_layers - 2; ++l) {
        p.pack.img_net[p.pack.n_images] = (unsigned char)k;
        p.pack.img_layer[p.pack.n_images++] = (unsigned char)l;
      }
    }
    return 0;
  }
  TcArgs& a = p.tc;
  a.stash_per_cta = (long long)n_used_max * c.tl_max * kTcMaxC * kTileBytes;
  a.n_nets = d->n_nets; a.n_terms = d->n_terms; a.n_theta = d->n_theta;
  for (int t = 0; t < d->n_terms; ++t) a.term_dim[t] = (unsigned char)P.terms[t].dim;
  return 0;
}
}  // namespace

// validation of the descriptor header, then the stages above in order
int plan_problem(const pinn_problem_desc* d, const pinn_integral_desc* integrals, int n_integrals,
                 const pinn_fixed_net_desc* fixed, int n_fixed, int max_smem, Plan& p) {
  memset(&p, 0, sizeof p);
  if (!d) return fail("pinn_create: null descriptor");
  if (n_fixed < 0 || n_fixed > PINN_MAX_FIXED_NETS)
    return fail("pinn_create_ex2: n_fixed=%d out of range [0,%d]", n_fixed, PINN_MAX_FIXED_NETS);
  if (n_fixed > 0 && !fixed) return fail("pinn_create_ex2: null fixed networks");
  if (n_fixed > 0 && !ffma_kernel_mode(d->mode))
    return fail("pinn_create_ex2: fixed networks run on the FFMA path (mode PINN_MODE_FFMA); the tensor-core modes do not "
                "evaluate them");
  if (n_integrals < 0 || n_integrals > PINN_MAX_INTEGRALS)
    return fail("pinn_create_ex: n_integrals=%d out of range [0,%d]", n_integrals, PINN_MAX_INTEGRALS);
  if (n_integrals > 0 && !integrals) return fail("pinn_create_ex: null integrals");
  if (n_integrals > 0 && !ffma_kernel_mode(d->mode))
    return fail("pinn_create_ex: integral terms run on the FFMA path (mode PINN_MODE_FFMA); the tensor-core modes do not "
                "evaluate them");
  if (d->abi_version != PINN_ABI_VERSION)
    return fail("pinn_create: descriptor abi_version %d, library %d", d->abi_version, PINN_ABI_VERSION);
  if (d->dtype != PINN_F32 && d->dtype != PINN_F64) return fail("pinn_create: unknown dtype %d", d->dtype);
  if (d->mode < PINN_MODE_FFMA || d->mode > PINN_MODE_TC_F64) return fail("pinn_create: unknown mode %d", d->mode);
  if (d->mode == PINN_MODE_TC_F64 && d->dtype != PINN_F64)
    return fail("pinn_create: PINN_MODE_TC_F64 runs the layer products on the FP64 tensor cores and needs dtype PINN_F64 "
                "(use PINN_MODE_FFMA, PINN_MODE_TC_BF16 or PINN_MODE_TC_SPLIT for PINN_F32)");
  if (d->n_nets < 1 || d->n_nets > PINN_MAX_NETS) return fail("pinn_create: n_nets=%d out of range [1,%d]", d->n_nets, PINN_MAX_NETS);
  if (d->n_terms < 1 || d->n_terms > PINN_MAX_TERMS)
    return fail("pinn_create: n_terms=%d out of range [1,%d]", d->n_terms, PINN_MAX_TERMS);
  if (d->n_params < 0 || d->n_params > PINN_MAX_PARAMS)
    return fail("pinn_create: n_params=%d out of range [0,%d]", d->n_params, PINN_MAX_PARAMS);
  if (!d->nets || !d->terms) return fail("pinn_create: null nets/terms");
  if (d->n_theta <= 0) return fail("pinn_create: n_theta must be positive");
  if (d->n_params > 0 && (d->param_offset < 0 || d->param_offset + d->n_params > d->n_theta))
    return fail("pinn_create: theta.p block [%lld,+%d) outside theta (n_theta=%lld)", (long long)d->param_offset,
                d->n_params, (long long)d->n_theta);
  DevProblem& P = p.prob;
  P.n_nets = d->n_nets; P.n_terms = d->n_terms; P.n_params = d->n_params;
  P.param_off = d->param_offset; P.n_theta = d->n_theta; P.n_fixed = n_fixed;
  P.func_term = -1;
  int max_w8 = 8, max_c = 1;
  long long resident = 0, stash_max = 0;
  if (plan_nets(d, fixed, n_fixed, P, max_w8, resident, p.fixed_len)) return 1;
  for (int t = 0; t < d->n_terms; ++t)
    if (plan_term(d, t, integrals, n_integrals, P, p.term[t], max_c, stash_max)) return 1;
  P.n_integrals = n_integrals;
  p.integ = n_integrals > 0;
  p.func = P.func_term >= 0;
  for (int i = 0; i < n_integrals; ++i) {     // after the terms: the owners' dims and tap counts are validated
    double f = 0;
    if (plan_integral(d, integrals, n_integrals, i, P, max_c, stash_max, &f)) return 1;
    p.term[integrals[i].owner].flops_per_point += f;
  }
  p.tile_pts = ffma_kernel_mode(d->mode) ? kTilePts : kTcPts;
  if (ffma_kernel_mode(d->mode)) return plan_ffma(d->dtype, max_w8, resident, max_c, stash_max, max_smem, p);
  return plan_tc(d, max_smem, p);
}
}  // namespace pinn
