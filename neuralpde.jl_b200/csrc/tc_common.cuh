// tc_common.cuh -- device helpers shared by the tensor-core kernels (tc_kernel.cu: widths <= 64, all operands resident;
// tc_wide_kernel.cu: 128-wide layers, streamed weights): fp32x2 arithmetic, the forward-mode tap chain rule
// and its adjoint, accumulator loads, swizzled-tile stores and bf16 hi / lo splits, warp reduce-scatter, MMA chains, the
// common part of the CTA's shared constants, the steps of the tile driver both kernels share (CTA setup, parameter and
// point-tile staging, residual program, kernel end), the steps of the per-network passes they share (end of the forward,
// ubar gather, last-layer gradient, tensor-layer gradient flush, layer-0 gradient), dispatch macro.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "tc_types.h"
#include "ffma_kernel.cuh"   // act_eval, run_program, warp_sum
#include "tc_prims.cuh"
#include "tail.cuh"

namespace pinn {

// ---- small helpers ---------------------------------------------------------------------------------
constexpr int kNH = kTcThreads / 128;   // warps per 32-row quadrant of the accumulators: each takes 1/kNH of the columns
static_assert(kTcThreads == 512, "the MMA chains are spread over four warpgroups");
constexpr int GW = 4;                   // columns per epilogue granule
constexpr int GWB = 2;                  // granule of the layer-0 reverse epilogue of tc_kernel.cu (register-heaviest loop)

template <int N>
__device__ __forceinline__ float pick(const float* v, int idx) {
  float r = v[0];
#pragma unroll
  for (int i = 1; i < N; ++i) r = (idx == i) ? v[i] : r;
  return r;
}
template <int N>
__device__ __forceinline__ void add_at(float* v, int idx, float x) {
#pragma unroll
  for (int i = 0; i < N; ++i) v[i] += (idx == i) ? x : 0.f;
}

// activation value and first three derivatives.  AK = 1: tanh, 2: sigmoid (branch-free, built on
// ex2.approx + rcp.approx: absolute error ~1e-7, far below the bf16-split operand noise);
// AK = 0: any activation through the accurate generic evaluator (gelu, logcosh and cos excepted: check_tc_nets
// refuses them).
template <int AK>
__device__ __forceinline__ void act_eval_tc(int act, float z, float& a, float& d1, float& d2, float& d3) {
  if (AK == 1) {
    const float e = __expf(2.f * z);
    const float t = 1.f - __fdividef(2.f, e + 1.f);
    const float s = fmaf(-t, t, 1.f);
    a = t; d1 = s; d2 = -2.f * t * s; d3 = s * fmaf(6.f * t, t, -2.f);
  } else if (AK == 2) {
    const float g = __fdividef(1.f, 1.f + __expf(-z));
    const float g1 = g * (1.f - g);
    a = g; d1 = g1; d2 = g1 * fmaf(-2.f, g, 1.f); d3 = g1 * fmaf(-6.f, g1, 1.f);
  } else {
    act_eval<float, false>(act, z, a, d1, d2, d3);
  }
}
__device__ __forceinline__ int act_kind(int act) { return act == PINN_ACT_TANH ? 1 : (act == PINN_ACT_SIGMOID ? 2 : 0); }

__device__ __forceinline__ float lds_f32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts_v2(uint32_t addr, uint32_t x, uint32_t y) {
  asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ void sts_v4(uint32_t addr, uint32_t x, uint32_t y, uint32_t z, uint32_t w) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}

// bf16 (hi, lo) split of the pair (a, b): hi = tc::pack_bf16(a, b), lo = bf16x2_lo(a, b, hi) = bf16x2 of the residuals
// (a, b) - hi.  lo is a call of its own so that a lo that only one branch stores is computed on that branch alone.
__device__ __forceinline__ uint32_t bf16x2_lo(float a, float b, uint32_t hi) {
  return tc::pack_bf16(a - __uint_as_float(hi << 16), b - __uint_as_float(hi & 0xffff0000u));
}

// store 4 consecutive columns (half of a 16-byte chunk) of a row into a swizzled tile; with `split`
// also the bf16 residual v - bf16(v) into the lo tile
__device__ __forceinline__ void store_half(uint32_t tile_hi, uint32_t tile_lo, int row, int col0, const float (&v)[4],
                                           bool split) {
  const uint32_t off = tc::swz_chunk(row, col0 >> 3) + ((col0 & 4) << 1);
  const uint32_t hx = tc::pack_bf16(v[0], v[1]), hy = tc::pack_bf16(v[2], v[3]);
  sts_v2(tile_hi + off, hx, hy);
  if (split) sts_v2(tile_lo + off, bf16x2_lo(v[0], v[1], hx), bf16x2_lo(v[2], v[3], hy));
}

// accumulator loads: columns col .. col + n - 1 of row (base + lane), see tc::acc_row
__device__ __forceinline__ void acc_ld4(uint32_t aaddr, float (&v)[4]) {
  const float* r = tc::acc_row(aaddr);
#pragma unroll
  for (int i = 0; i < 4; ++i) v[i] = r[i * kAccRows];
}
__device__ __forceinline__ void acc_ld2(uint32_t aaddr, float (&v)[2]) {
  const float* r = tc::acc_row(aaddr);
  v[0] = r[0]; v[1] = r[kAccRows];
}
__device__ __forceinline__ void acc_ldg(uint32_t aaddr, float (&v)[4]) { acc_ld4(aaddr, v); }
__device__ __forceinline__ void acc_ldg(uint32_t aaddr, float (&v)[2]) { acc_ld2(aaddr, v); }

// 2-column variant of store_half
__device__ __forceinline__ void store_half(uint32_t tile_hi, uint32_t tile_lo, int row, int col0, const float (&v)[2],
                                           bool split) {
  const uint32_t off = tc::swz_chunk(row, col0 >> 3) + ((col0 & 6) << 1);
  const uint32_t hx = tc::pack_bf16(v[0], v[1]);
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(tile_hi + off), "r"(hx) : "memory");
  if (split) asm volatile("st.shared.b32 [%0], %1;" ::"r"(tile_lo + off), "r"(bf16x2_lo(v[0], v[1], hx)) : "memory");
}

// ---- fp32x2 arithmetic: two columns per value (component-wise fp32 instructions) ---------------
struct P2 { float2 v; };
__device__ __forceinline__ P2 mk2(float a, float b) { P2 r; r.v = make_float2(a, b); return r; }
__device__ __forceinline__ P2 splat2(float a) { return mk2(a, a); }
__device__ __forceinline__ P2 operator*(P2 a, P2 b) { return mk2(__fmul_rn(a.v.x, b.v.x), __fmul_rn(a.v.y, b.v.y)); }
__device__ __forceinline__ P2 operator+(P2 a, P2 b) { return mk2(__fadd_rn(a.v.x, b.v.x), __fadd_rn(a.v.y, b.v.y)); }
__device__ __forceinline__ P2 vfma(P2 a, P2 b, P2 c) { return mk2(__fmaf_rn(a.v.x, b.v.x, c.v.x), __fmaf_rn(a.v.y, b.v.y, c.v.y)); }
__device__ __forceinline__ float vfma(float a, float b, float c) { return fmaf(a, b, c); }
template <typename T> __device__ __forceinline__ T vsplat(float x);
template <> __device__ __forceinline__ float vsplat<float>(float x) { return x; }
template <> __device__ __forceinline__ P2 vsplat<P2>(float x) { return splat2(x); }
__device__ __forceinline__ float ex2_approx(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float rcp_approx(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

// tanh and its first three derivatives for two columns at once
__device__ __forceinline__ void tanh_eval2(P2 z, P2& a, P2& d1, P2& d2, P2& d3) {
  const P2 zz = z * splat2(2.8853900817779268f);                 // 2 * log2(e)
  const P2 den = mk2(ex2_approx(zz.v.x), ex2_approx(zz.v.y)) + splat2(1.f);
  const P2 r = mk2(rcp_approx(den.v.x), rcp_approx(den.v.y));
  const P2 t = vfma(r, splat2(-2.f), splat2(1.f));
  const P2 s = vfma(t * splat2(-1.f), t, splat2(1.f));
  a = t; d1 = s;
  d2 = (t * s) * splat2(-2.f);
  d3 = s * vfma(t * splat2(6.f), t, splat2(-2.f));
}

// channel bookkeeping of one (term, network): value + N1 first + N2 second derivative channels.
// PURE: second-derivative channel s is d2/dx_s^2 of first-derivative channel s (no index selects).
template <int N1, int N2>
struct Chan {
  int sa[N2 > 0 ? N2 : 1], sb[N2 > 0 ? N2 : 1];
};

template <typename T, int N>
__device__ __forceinline__ T pickT(const T* v, int idx) {
  T r = v[0];
#pragma unroll
  for (int i = 1; i < N; ++i) r = (idx == i) ? v[i] : r;
  return r;
}

// activation dispatch on the value type: packed tanh for P2, scalar evaluators otherwise
template <int AK>
__device__ __forceinline__ void act_any(int act, float z, float& a, float& d1, float& d2, float& d3) {
  act_eval_tc<AK>(act, z, a, d1, d2, d3);
}
template <int AK>
__device__ __forceinline__ void act_any(int act, P2 z, P2& a, P2& d1, P2& d2, P2& d3) {
  if (AK == 1) {
    tanh_eval2(z, a, d1, d2, d3);
  } else {
    float ax, d1x, d2x, d3x, ay, d1y, d2y, d3y;
    act_eval_tc<AK>(act, z.v.x, ax, d1x, d2x, d3x);
    act_eval_tc<AK>(act, z.v.y, ay, d1y, d2y, d3y);
    a = mk2(ax, ay); d1 = mk2(d1x, d1y); d2 = mk2(d2x, d2y); d3 = mk2(d3x, d3y);
  }
}

// post-activation channels from pre-activation channels (z[0] value, z[1..N1], z[1+N1..]); T = float or P2
template <int N1, int N2, bool PURE, int AK, typename T>
__device__ __forceinline__ void chain_fwd(int act, const Chan<N1, N2>& ch, const T* z, T* h) {
  constexpr int M1 = (N1 > 0) ? N1 : 1;
  T a, d1, d2, d3;
  act_any<AK>(act, z[0], a, d1, d2, d3);
  h[0] = a;
#pragma unroll
  for (int i = 0; i < N1; ++i) h[1 + i] = d1 * z[1 + i];
#pragma unroll
  for (int s = 0; s < N2; ++s) {
    const T za = PURE ? z[1 + (s < N1 ? s : 0)] : pickT<T, M1>(z + 1, ch.sa[s]);
    const T zb = PURE ? za : pickT<T, M1>(z + 1, ch.sb[s]);
    h[1 + N1 + s] = vfma(d1, z[1 + N1 + s], d2 * za * zb);
  }
}

// adjoints of pre-activations from adjoints of post-activations; T = float or P2
template <int N1, int N2, bool PURE, int AK, typename T>
__device__ __forceinline__ void chain_bwd(int act, const Chan<N1, N2>& ch, const T* z, const T* hb, T* zb) {
  constexpr int M1 = (N1 > 0) ? N1 : 1;
  T a, d1, d2, d3;
  act_any<AK>(act, z[0], a, d1, d2, d3);
  T acc0 = d1 * hb[0];
#pragma unroll
  for (int i = 0; i < N1; ++i) {
    acc0 = vfma(d2 * z[1 + i], hb[1 + i], acc0);
    zb[1 + i] = d1 * hb[1 + i];
  }
#pragma unroll
  for (int s = 0; s < N2; ++s) {
    const T g = hb[1 + N1 + s];
    if (PURE) {
      const int i = s < N1 ? s : 0;
      const T za = z[1 + i];
      acc0 = vfma(vfma(d2, z[1 + N1 + s], d3 * za * za), g, acc0);
      zb[1 + i] = vfma((d2 * za) * vsplat<T>(2.f), g, zb[1 + i]);
    } else {
      const T za = pickT<T, M1>(z + 1, ch.sa[s]), zbb = pickT<T, M1>(z + 1, ch.sb[s]);
      acc0 = vfma(vfma(d2, z[1 + N1 + s], d3 * za * zbb), g, acc0);
      const T ga = d2 * zbb * g, gb2 = d2 * za * g;
#pragma unroll
      for (int i = 0; i < M1; ++i) {
        if (ch.sa[s] == i) zb[1 + i] = zb[1 + i] + ga;
        if (ch.sb[s] == i) zb[1 + i] = zb[1 + i] + gb2;
      }
    }
    zb[1 + N1 + s] = d1 * g;
  }
  zb[0] = acc0;
}

// sum over the 32 lanes of the GW = 4 per-lane values of a granule with 6 shuffles.  Every lane receives the total of
// element reduceg_elem(lane); the lanes with reduceg_lead(lane) act on it.
__device__ __forceinline__ float warp_reduceg(const float (&v)[GW], int lane) {
  const bool up16 = (lane & 16) != 0;
  float a0 = (up16 ? v[2] : v[0]) + __shfl_xor_sync(0xffffffffu, up16 ? v[0] : v[2], 16);
  float a1 = (up16 ? v[3] : v[1]) + __shfl_xor_sync(0xffffffffu, up16 ? v[1] : v[3], 16);
  const bool up8 = (lane & 8) != 0;
  float r = (up8 ? a1 : a0) + __shfl_xor_sync(0xffffffffu, up8 ? a0 : a1, 8);
  r += __shfl_xor_sync(0xffffffffu, r, 4);
  r += __shfl_xor_sync(0xffffffffu, r, 2);
  r += __shfl_xor_sync(0xffffffffu, r, 1);
  return r;
}
__device__ __forceinline__ int reduceg_elem(int lane) { return ((lane >> 4) & 1) * 2 + ((lane >> 3) & 1); }
__device__ __forceinline__ bool reduceg_lead(int lane) { return (lane & 7) == 0; }

// phase timestamps for the timeline tool (scripts/tc_timeline.py): id in the high bits, clock in the low
// (only in -DPINN_DEBUG builds: libpinn_b200_debug.so; the product library carries no instrumentation)
template <typename CS>
__device__ __forceinline__ void dbg_mark(CS* cs, int id) {
#ifdef PINN_DEBUG
  if (cs->dbg && threadIdx.x == 0 && cs->dbg_n < 1000) {
    cs->dbg[cs->dbg_n++] = ((long long)id << 48) | (clock64() & 0xffffffffffffLL);
  }
#endif
}

// CTA-wide constants kept in shared memory so that the per-network passes (separate functions) do not drag a context
// struct through local memory: the fields both kernels use (each kernel's CtaShared / TwShared adds its own)
struct CtaBase {
  float* partial;          // this CTA's gradient partial
  long long* dbg;          // optional phase-timestamp buffer (CTA 0, thread 0)
  int dbg_n;
  int tl_max, off_P, off_misc, off_ones, mx_dim, mx_taps;
};
// thread 0: fill the common fields and write the start record of the phase timeline
__device__ __forceinline__ void cta_base_init(CtaBase& cs, const TcCommonArgs& a, float* partial) {
  cs.partial = partial;
  cs.tl_max = a.tl_max; cs.off_P = a.off_P; cs.off_misc = a.off_misc; cs.off_ones = a.off_ones;
  cs.mx_dim = a.mx_dim; cs.mx_taps = a.mx_taps;
#ifdef PINN_DEBUG
  cs.dbg = (blockIdx.x == 0) ? a.dbg : nullptr;
#else
  cs.dbg = nullptr;
#endif
  cs.dbg_n = 0;
  dbg_mark(&cs, 1);
}

struct Misc {   // carve-up of the misc region
  float *Xs, *taps, *tapbar, *scratch, *qws;
  double* tsum;
  uint64_t* bar_ld;
};
// mx_dim / mx_taps: largest point dimension / tap count over the problem's terms (the arrays are sized to them)
__device__ __forceinline__ Misc misc_of(uint8_t* m, int mx_dim, int mx_taps) {
  Misc r;
  r.Xs = reinterpret_cast<float*>(m);             m += mx_dim * kTcPts * 4;
  r.taps = reinterpret_cast<float*>(m);           m += mx_taps * kTcPts * 4;
  r.tapbar = reinterpret_cast<float*>(m);         m += mx_taps * kTcPts * 4;
  r.scratch = reinterpret_cast<float*>(m);        m += kTcMaxC * kTcPts * 4;
  r.qws = reinterpret_cast<float*>(m);            m += kTcPts * 4;
  r.tsum = reinterpret_cast<double*>(m);          m += PINN_MAX_TERMS * 8;
  r.bar_ld = reinterpret_cast<uint64_t*>(m);
  return r;
}

// descriptor fields a network pass needs, read once from global memory into registers
template <int N1, int N2>
struct PassInfo {
  int L, TL, d_in, n1w, nL;
  int dir1[N1 > 0 ? N1 : 1];
  Chan<N1, N2> ch;
};
template <int N1, int N2>
__device__ __forceinline__ void load_pass(PassInfo<N1, N2>& pi, const DevNet& net, const DevChan& dc) {
  pi.L = net.n_layers; pi.TL = pi.L - 2; pi.d_in = net.dims[0]; pi.n1w = net.dims[1]; pi.nL = net.dims[pi.L - 1];
#pragma unroll
  for (int j = 0; j < N1; ++j) pi.dir1[j] = dc.dir1[j];
#pragma unroll
  for (int s = 0; s < N2; ++s) { pi.ch.sa[s] = dc.s_a[s]; pi.ch.sb[s] = dc.s_b[s]; }
}

// first-layer pre-activations of neuron o (channel vector zz); fpa = shared-memory address of the FpBlock<W>
template <int W, int N1, int N2>
__device__ __forceinline__ void first_layer_elem(uint32_t fpa, const PassInfo<N1, N2>& pi, const float (&x)[PINN_MAX_IN],
                                                 int o, float* zz) {
  using F = FpBlock<W>;
  float s = lds_f32(fpa + (F::B1 + o) * 4);
  const uint32_t wa = fpa + (F::W1 + o * 8) * 4;
  if (pi.d_in <= 3) {            // common 1-D / 2-D / 3-D problems: no predicated tail
    s = fmaf(lds_f32(wa), x[0], s);
    if (pi.d_in >= 2) s = fmaf(lds_f32(wa + 4), x[1], s);
    if (pi.d_in == 3) s = fmaf(lds_f32(wa + 8), x[2], s);
  } else {
#pragma unroll
    for (int k = 0; k < PINN_MAX_IN; ++k)
      if (k < pi.d_in) s = fmaf(lds_f32(wa + k * 4), x[k], s);
  }
  zz[0] = s;
#pragma unroll
  for (int j = 0; j < N1; ++j) zz[1 + j] = lds_f32(fpa + (F::W1 + o * 8 + pi.dir1[j]) * 4);
#pragma unroll
  for (int j = 0; j < N2; ++j) zz[1 + N1 + j] = 0.f;
}

__device__ __forceinline__ void wait_bar(uint64_t* bar, uint32_t& phase) {
  tc::mbar_wait(bar, phase);
  phase ^= 1u;
}

// a chain of nk MMAs D[128 x N] (+)= A_k * B_k into accumulator column d; descriptors advance by a_step / b_step bytes per
// k-step.  CTA-collective: every thread calls it with the same arguments, and the two 64-row halves of D run on warpgroup
// pair {0, 1} or {2, 3}, chosen by the parity of the set bits of d / 16.  Chains into the same columns therefore run on one
// warpgroup in program order (an accumulating chain sees its predecessor's result without a barrier), and chains at any
// power-of-two column stride (64 per channel in tc_kernel.cu, 128 in tc_wide_kernel.cu) alternate between the two pairs.
// The second half reads rows 64..127 of a K-major A (+8 KB) or the next 64-column tile of an MN-major A (LBO); an MN-major
// A with LBO = 0 has 64 rows and only the first half runs.  Results are visible to the CTA after the next __syncthreads.
static __device__ __noinline__ void mma_chain(uint32_t d, uint64_t adesc, uint64_t bdesc, uint32_t a_step, uint32_t b_step, int nk,
                                          uint32_t idesc, uint32_t acc_first) {
  const int n = (int)(idesc & 0xffu), ta = (int)((idesc >> 8) & 1u), tb = (int)((idesc >> 9) & 1u);
  const uint32_t dcol = d & 0xffffu, j = dcol >> 4;
  const uint32_t lbo = (uint32_t)((adesc >> 16) & 0x3fffu) << 4;
  const int wg = (int)(threadIdx.x >> 7);
#pragma unroll 1
  for (int h = 0; h < 2; ++h) {
    if (h == 1 && ta && lbo == 0) break;
    if (wg != 2 * (__popc(j) & 1) + h) continue;
    const uint64_t a = adesc + ((h ? (ta ? lbo : 8192u) : 0u) >> 4);
    if (ta == 0 && tb == 0) tc::wg_chain_n<0, 0>(n, dcol, h, a, bdesc, a_step, b_step, nk, acc_first);
    else if (ta == 0) tc::wg_chain_n<0, 1>(n, dcol, h, a, bdesc, a_step, b_step, nk, acc_first);
    else if (tb == 0) tc::wg_chain_n<1, 0>(n, dcol, h, a, bdesc, a_step, b_step, nk, acc_first);
    else tc::wg_chain_n<1, 1>(n, dcol, h, a, bdesc, a_step, b_step, nk, acc_first);
  }
}

// thread identity inside the CTA
struct Tid {
  int tid, warp, lane, q, hh, p;
  uint32_t lane_addr;
};
__device__ __forceinline__ Tid tid_of() {
  Tid t;
  t.tid = threadIdx.x; t.warp = t.tid >> 5; t.lane = t.tid & 31; t.q = t.warp & 3; t.hh = t.warp >> 2;
  t.p = t.q * 32 + t.lane;
  t.lane_addr = (uint32_t)(t.q * 32) << 16;   // accumulator row base of the warp's quadrant
  return t;
}

// ---- steps of the tile driver that both tensor-core kernels share ----------------------------------------------------------
// (plain helpers: each kernel body keeps its own setup, tile loop and sweeps, and calls these where the steps coincide)

// zero the CTA's gradient partial (want_grad) and term sums, write the ones atom
__device__ __forceinline__ void cta_setup(const TcCommonArgs& a, const Misc& ms, float* partial, long long n_theta, bool want_grad) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x;
  if (want_grad) {
    const long long n4 = n_theta / 4;
    float4* p4 = reinterpret_cast<float4*>(partial);
    if ((reinterpret_cast<uintptr_t>(partial) & 15) == 0) {
      for (long long i = tid; i < n4; i += kTcThreads) p4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      for (long long i = n4 * 4 + tid; i < n_theta; i += kTcThreads) partial[i] = 0.f;
    } else {
      for (long long i = tid; i < n_theta; i += kTcThreads) partial[i] = 0.f;
    }
  }
  if (tid < PINN_MAX_TERMS) ms.tsum[tid] = 0.0;
  if (tid < 64) {      // ones atom: row r (128 B) holds bf16 1.0 in logical column 0 = 16-byte chunk (0 ^ r)
    const int r = tid >> 3, ch = tid & 7;
    *reinterpret_cast<uint4*>(smem + a.off_ones + r * 128 + ch * 16) = make_uint4(ch == r ? 0x00003f80u : 0u, 0u, 0u, 0u);
  }
}

// fp32 parameter block FpBlock<W> of one network: first layer, tensor-layer biases, last layer (CTA-wide: has a barrier)
template <int W>
__device__ __forceinline__ void stage_fp_block(float* fp, const DevNet& net, const float* theta) {
  using F = FpBlock<W>;
  const int tid = threadIdx.x, L = net.n_layers;
  for (int i = tid; i < F::SIZE; i += kTcThreads) fp[i] = 0.f;
  __syncthreads();
  const int n1w = net.dims[1], d_in = net.dims[0];
  const long long w0 = net.w_off[0], b0 = net.b_off[0];
  for (int i = tid; i < n1w * d_in; i += kTcThreads) {
    const int o = i % n1w, k = i / n1w;
    fp[F::W1 + o * 8 + k] = __ldg(&theta[w0 + i]);
  }
  for (int i = tid; i < n1w; i += kTcThreads) fp[F::B1 + i] = __ldg(&theta[b0 + i]);
  for (int i = tid; i < (L - 2) * W; i += kTcThreads) {
    const int l = 1 + i / W, o = i & (W - 1);
    if (o < net.dims[l + 1]) fp[F::BT + (l - 1) * W + o] = __ldg(&theta[net.b_off[l] + o]);
  }
  const int nL = net.dims[L - 1];
  const long long wl = net.w_off[L - 1], bl = net.b_off[L - 1];
  for (int i = tid; i < nL; i += kTcThreads) fp[F::WL + i] = __ldg(&theta[wl + i]);
  if (tid == 0) fp[F::BL] = __ldg(&theta[bl]);
}

// a point tile: its term, the index of its first point in the term, the term's point count
struct TileRef {
  int ti;
  long long p0, n_pts;
};

// find the term of `tile`, stage its points into ms.Xs ([row][point]) and quadrature weights into ms.qws, clear the tap
// adjoints.  ld_phase: parity of the collocation-tile barrier ms.bar_ld.  CTA-wide, ends with a barrier.
__device__ __forceinline__ TileRef stage_tile(const TcCommonArgs& a, const DevProblem& P, const Misc& ms, int tile,
                                              uint32_t& ld_phase) {
  const int tid = threadIdx.x;
  int ti = 0;
  while (ti + 1 < P.n_terms && tile >= a.dyn[ti + 1].tile0) ++ti;
  const DevTerm& tm = P.terms[ti];
  const long long p0 = (long long)(tile - a.dyn[ti].tile0) * kTcPts;
  const long long n_pts = a.dyn[ti].n;
  const float* pts = reinterpret_cast<const float*>(a.dyn[ti].pts);
  const float* qw = reinterpret_cast<const float*>(a.dyn[ti].qw);
  // warm L1 with the term header + residual program (read by every phase)
  if (tid < (int)((sizeof(DevTerm) + 127) / 128)) tc::prefetch_l1(reinterpret_cast<const char*>(&tm) + tid * 128);
  const int dim = tm.dim, n_taps = tm.n_taps, weighted = tm.weighted;
  // Collocation tile: one point = dim contiguous scalars (the reference's d x N train-set layout), so a full 128-point
  // tile is ONE contiguous block of dim x 512 bytes.  The TMA unit copies it into shared memory in a single bulk transfer
  // (cp.async.bulk + mbarrier transaction count; staged in the scratch array, free between tiles, kTcMaxC rows) and 128
  // threads transpose it to [row][point].  Partial last tiles (clamped rows) and callers' buffers that are not 16-byte
  // aligned take the per-element path.
  const float* tile_src = pts + p0 * dim;
  const bool bulk_tile = (p0 + kTcPts <= n_pts) && dim <= kTcMaxC && ((reinterpret_cast<uintptr_t>(tile_src) & 15) == 0);
  if (bulk_tile) {
    if (tid == 0) {
      tc::mbar_arrive_expect_tx(ms.bar_ld, (uint32_t)(dim * kTcPts * 4));
      tc::bulk_load(ms.scratch, tile_src, (uint32_t)(dim * kTcPts * 4), ms.bar_ld);
    }
    wait_bar(ms.bar_ld, ld_phase);
    if (tid < kTcPts)
      for (int r = 0; r < dim; ++r) ms.Xs[r * kTcPts + tid] = ms.scratch[tid * dim + r];
  } else {
    for (int i = tid; i < dim * kTcPts; i += kTcThreads) {
      int pp = i / dim, r = i - pp * dim;
      long long gp = p0 + pp;
      if (gp >= n_pts) gp = n_pts - 1;
      ms.Xs[r * kTcPts + pp] = pts[gp * dim + r];
    }
  }
  if (tid < kTcPts) {
    long long gp = p0 + tid;
    float w = 0.f;
    if (gp < n_pts) w = weighted ? qw[gp] : 1.f;
    ms.qws[tid] = w;
  }
  for (int i = tid; i < n_taps * kTcPts; i += kTcThreads) ms.tapbar[i] = 0.f;
  __syncthreads();
  return TileRef{ti, p0, n_pts};
}

// residual program of the tile (threads 0..127: one point each): loss partial into ms.tsum, the residual probe (mode 2)
// and, for a gradient, the tap adjoints scaled by the loss seed and the theta.p gradient.  The program text and the
// per-point value / adjoint arrays go to the idle shared memory [region, region + region_bytes) when they fit.
// CTA-wide, ends with a barrier.
__device__ __forceinline__ void residual_step(const TcCommonArgs& a, const DevProblem& P, const DevTerm& tm, const Misc& ms,
                                              const TileRef& tr, uint8_t* region, size_t region_bytes, float* partial,
                                              bool want_grad) {
  const int tid = threadIdx.x, lane = tid & 31;
  const int n_instr = tm.n_instr, n_taps = tm.n_taps;
  DevInstr* sprog = reinterpret_cast<DevInstr*>(region);
  float* sval = reinterpret_cast<float*>(region + 8192);
  const bool prog_sm = (size_t)8192 + (size_t)2 * n_instr * kTcPts * 4 <= region_bytes;
  if (prog_sm) {
    const int nw = n_instr * (int)(sizeof(DevInstr) / 4);
    const int* src = reinterpret_cast<const int*>(tm.prog);
    for (int i = tid; i < nw; i += kTcThreads) reinterpret_cast<int*>(sprog)[i] = __ldg(src + i);
    __syncthreads();
  }
  if (tid < kTcPts) {
    float pbar[PINN_MAX_PARAMS];
#pragma unroll
    for (int j = 0; j < PINN_MAX_PARAMS; ++j) pbar[j] = 0.f;
    float r;
    if (prog_sm) {
      r = run_program_t<float, kTcPts, true>(sprog, n_instr, a.theta + P.param_off, ms.Xs, ms.taps, ms.tapbar, pbar, tid,
                                             want_grad, sval, sval + n_instr * kTcPts);
    } else {
      r = run_program<float, kTcPts>(tm, a.theta + P.param_off, ms.Xs, ms.taps, ms.tapbar, pbar, tid, want_grad);
    }
    const float w = ms.qws[tid];
    double s = (double)w * (double)r * (double)r;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) atomicAdd(&ms.tsum[tr.ti], s);
    if (a.mode == 2) {
      long long gp = tr.p0 + tid;
      if (gp < tr.n_pts) a.resid_out[gp] = r;
    }
    if (want_grad) {
      const float g = (float)a.seed[tr.ti] * w * 2.f * r;
      for (int tt = 0; tt < n_taps; ++tt) ms.tapbar[tt * kTcPts + tid] *= g;
      const int n_params = P.n_params;
      for (int j = 0; j < n_params; ++j) {
        float v = warp_sum<float>(pbar[j] * g);
        if (lane == 0) atomicAdd(&partial[P.param_off + j], v);
      }
    }
  }
  __syncthreads();
}

// start clocks of the CTA's span record (PINN_DEBUG builds, written by cta_finish)
struct DbgSpan {
  long long c0;
  unsigned long long g0;
};
__device__ __forceinline__ DbgSpan dbg_span_begin(const long long* dbg) {
  DbgSpan s{0, 0};
#ifdef PINN_DEBUG
  if (dbg && threadIdx.x == 0) {
    s.c0 = clock64();
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(s.g0));
  }
#endif
  return s;
}

// end of the kernel: span record (PINN_DEBUG), per-CTA term sums, and the kernel tail (tail.cuh: gradient reduction,
// optimizer step, multi-GPU sum)
template <typename CS>
__device__ __forceinline__ void cta_finish(const TcCommonArgs& a, const CS& cs, const DbgSpan& span, const Misc& ms,
                                           const DevProblem& P, bool want_grad) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x;
#ifdef PINN_DEBUG
  if (tid == 0 && cs.dbg) cs.dbg[999] = cs.dbg_n;
  if (a.dbg && tid == 0 && blockIdx.x < 250) {
    unsigned long long g1;
    unsigned int smid;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(g1));
    asm volatile("mov.u32 %0, %smid;" : "=r"(smid));
    long long* rec = a.dbg + 1000 + 4 * blockIdx.x;
    rec[0] = (long long)span.g0; rec[1] = (long long)g1; rec[2] = clock64() - span.c0; rec[3] = smid;
  }
#endif
  if (tid < PINN_MAX_TERMS) a.term_sums[(long long)blockIdx.x * PINN_MAX_TERMS + tid] = ms.tsum[tid];
  if (a.tail.state)
    fused_tail<float, kTcThreads>(a.tail, a.partial, a.partial_stride, a.term_sums, P.n_theta, P.n_terms, want_grad ? 1 : 0,
                                  reinterpret_cast<float*>(smem + a.off_P));
}

// ---- steps of the per-network passes that both tensor-core kernels share --------------------------------------------------
// (what differs between the kernels comes in as arguments: shared-memory tile addresses and strides, descriptor LBOs,
// accumulator columns, and `rows`, the accumulator rows a flush reads = the kernel's widest layer)

// end of the forward: combine the per-warp last-layer dots u of every point through ms.scratch (zeroed when the pass
// began), add b_L (*bl) and write the taps the term reads from network slot `slot`.  CTA-wide.
template <int C, typename CS>
__device__ __forceinline__ void finish_forward(CS* cs, const DevTerm& tm, int slot, const Misc& ms, const float* bl, const Tid& t,
                                               const float (&u)[C]) {
  __syncthreads();
  dbg_mark(cs, 15);
#pragma unroll
  for (int c = 0; c < C; ++c) atomicAdd(&ms.scratch[c * kTcPts + t.p], u[c]);
  __syncthreads();
  if (t.hh == 0) {
    float s[C];
#pragma unroll
    for (int c = 0; c < C; ++c) s[c] = ms.scratch[c * kTcPts + t.p];
    s[0] += *bl;
    const int n_taps = tm.n_taps;
    for (int tt = 0; tt < n_taps; ++tt)
      if (tm.tap_slot[tt] == slot) {
        const int tch = tm.tap_ch[tt];
        float v = s[0];
#pragma unroll
        for (int c = 1; c < C; ++c) v = (tch == c) ? s[c] : v;
        ms.taps[tt * kTcPts + t.p] = v;
      }
  }
  __syncthreads();
  dbg_mark(cs, 16);
}

// adjoints of the network outputs per channel at point p (every thread of the point needs them)
template <int C>
__device__ __forceinline__ void gather_ubar(const DevTerm& tm, int slot, const Misc& ms, int p, float (&ub)[C]) {
#pragma unroll
  for (int c = 0; c < C; ++c) ub[c] = 0.f;
  const int n_taps = tm.n_taps;
  for (int tt = 0; tt < n_taps; ++tt)
    if (tm.tap_slot[tt] == slot) {
      const float g = ms.tapbar[tt * kTcPts + p];
      const int tch = tm.tap_ch[tt];
#pragma unroll
      for (int c = 0; c < C; ++c) ub[c] += (tch == c) ? g : 0.f;
    }
}

// last layer: bias gradient by warp sums; weight gradient  wbar_L[o] = sum_{c,p} ubar_c[p] H_c[p][o]  on the tensor core:
// D_c[o][0..15] = H_c^T U into accumulator columns acol + 16c, with U[p] = (hi, lo) bf16 pairs of ubar_0..ubar_(C-1)
// (columns 2c, 2c+1) written to the tile at u_tile.  H_c is the tile at h_tile + c * h_stride, read MN-major (h_lbo: the
// next 64 rows of M when the last hidden layer is wider than 64).  CTA-wide.
template <int C>
__device__ __forceinline__ void last_layer_grad(const Tid& t, const float (&ub)[C], int nL, float* gw, float* gb, uint32_t u_tile,
                                                uint32_t h_tile, uint32_t h_stride, uint32_t h_lbo, uint32_t acol, int rows) {
  if (t.hh == 0) {
    const float s = warp_sum<float>(ub[0]);
    if (t.lane == 0) atomicAdd(gb, s);
    uint32_t w[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) w[c] = 0u;
#pragma unroll
    for (int c = 0; c < C; ++c) {
      const uint32_t hi = tc::pack_bf16(ub[c], 0.f);   // upper halves bf16(0): hi | lo << 16 = (bf16 hi, bf16 lo) of ubar_c
      w[c] = hi | (bf16x2_lo(ub[c], 0.f, hi) << 16);
    }
    sts_v4(u_tile + tc::swz_chunk(t.p, 0), w[0], w[1], w[2], w[3]);
    sts_v4(u_tile + tc::swz_chunk(t.p, 1), w[4], w[5], w[6], w[7]);
  }
  tc::fence_async_smem();
  __syncthreads();
  {
    const uint32_t idesc = tc::make_idesc(16, 1, 1);
    const uint64_t db = tc::make_desc(u_tile, 0, 1024);
#pragma unroll 1
    for (int c = 0; c < C; ++c)
      mma_chain(acol + 16 * c, tc::make_desc(h_tile + c * h_stride, h_lbo, 1024), db, 2048, 2048, kTcPts / 16, idesc, 0);
  }
  __syncthreads();
  if (t.hh == 0 && t.q * 32 < rows) {
    const int o = t.q * 32 + t.lane;
    float acc = 0.f;
#pragma unroll
    for (int c = 0; c < C; ++c) {
      float v[2];
      acc_ld2(t.lane_addr + acol + 16 * c + 2 * c, v);
      acc += v[0] + v[1];
    }
    if (o < nL) atomicAdd(gw + o, acc);
  }
  __syncthreads();
}

// flush a tensor layer's gradient tile: accumulator row = output neuron o, columns wcol .. wcol + n_in - 1 = input
// neuron k of the weight gradient, column bcol = the bias gradient
__device__ __forceinline__ void flush_wgrad(const Tid& t, uint32_t wcol, uint32_t bcol, int rows, int n_in, int n_out, float* gw,
                                            float* gb) {
  if (t.q * 32 < rows) {
    const int o = t.q * 32 + t.lane;
    if (t.hh == 0) {
      float v[2];
      acc_ld2(t.lane_addr + bcol, v);
      if (o < n_out) atomicAdd(gb + o, v[0]);
    }
    const int part = n_in / kNH;
#pragma unroll 1
    for (int k0 = t.hh * part; k0 < (t.hh + 1) * part; k0 += 4) {
      float v[4];
      acc_ld4(t.lane_addr + wcol + k0, v);
      if (o < n_out) {
#pragma unroll
        for (int i = 0; i < 4; ++i) atomicAdd(gw + o + (long long)n_out * (k0 + i), v[i]);
      }
    }
  }
}

// layer-0 weight / bias gradient as one MMA chain over K = the 128 points:
//   D[o][0..15] = Zbar_0^T [x | 1] + sum_j Zbar_(1+j)^T E_(dir1[j]),  Wbar_0[o][k] = D[o][k],  bbar_0[o] = D[o][8].
// coord_tiles writes the B tiles (rows = points, 16 columns used), kTileBytes apart from b_tile (threads 0..127):
//   tile 0: bf16 hi of (x_0..x_7) in columns 0..7, 1.0 in column 8;  tile 1+j: 1.0 in column dir1[j];
//   tile 1+N1: bf16 lo of x (x_lo: when the kernel has a spare tile for it)
// coord_row writes row `row` of those tiles (the point with coordinates x)
template <int N1>
__device__ __forceinline__ void coord_row(uint32_t b_tile, int row, const float (&x)[PINN_MAX_IN],
                                          const int (&dir1)[N1 > 0 ? N1 : 1], bool x_lo) {
  uint32_t hi[4], lo[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    hi[k] = tc::pack_bf16(x[2 * k], x[2 * k + 1]);
    lo[k] = bf16x2_lo(x[2 * k], x[2 * k + 1], hi[k]);
  }
  const uint32_t c0a = b_tile + tc::swz_chunk(row, 0), c1a = b_tile + tc::swz_chunk(row, 1);
  sts_v4(c0a, hi[0], hi[1], hi[2], hi[3]);
  sts_v4(c1a, 0x00003f80u, 0u, 0u, 0u);
  if (x_lo) {
    sts_v4(c0a + (1 + N1) * kTileBytes, lo[0], lo[1], lo[2], lo[3]);
    sts_v4(c1a + (1 + N1) * kTileBytes, 0u, 0u, 0u, 0u);
  }
#pragma unroll
  for (int j = 0; j < N1; ++j) {
    const int d = dir1[j];
    uint32_t w[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) w[k] = (d == 2 * k) ? 0x00003f80u : ((d == 2 * k + 1) ? 0x3f800000u : 0u);
    sts_v4(c0a + (1 + j) * kTileBytes, w[0], w[1], w[2], w[3]);
    sts_v4(c1a + (1 + j) * kTileBytes, 0u, 0u, 0u, 0u);
  }
}
template <int N1>
__device__ __forceinline__ void coord_tiles(const Tid& t, uint32_t b_tile, const float (&x)[PINN_MAX_IN],
                                            const int (&dir1)[N1 > 0 ? N1 : 1], bool x_lo) {
  if (t.tid >= kTcPts) return;
  coord_row<N1>(b_tile, t.p, x, dir1, x_lo);
}
// the MMA chains against the coord_tiles at b_tile and the flush into W_0 / b_0.  Zbar_c is the tile at z_tile + c * z_stride,
// read MN-major (z_lbo: the next 64 rows of M when the first layer is wider than 64).  Publishes the tiles itself; CTA-wide.
template <int N1>
__device__ __forceinline__ void layer0_grad(const Tid& t, uint32_t z_tile, uint32_t z_stride, uint32_t z_lbo, uint32_t b_tile,
                                            bool x_lo, uint32_t acol, int rows, int n1w, int d_in, float* gw0, float* gb0) {
  tc::fence_async_smem();
  __syncthreads();
  {
    const uint32_t idesc = tc::make_idesc(16, 1, 1);
    const uint64_t a0 = tc::make_desc(z_tile, z_lbo, 1024);
    mma_chain(acol, a0, tc::make_desc(b_tile, 0, 1024), 2048, 2048, kTcPts / 16, idesc, 0);
    if (x_lo) mma_chain(acol, a0, tc::make_desc(b_tile + (1 + N1) * kTileBytes, 0, 1024), 2048, 2048, kTcPts / 16, idesc, 1);
#pragma unroll 1
    for (int j = 0; j < N1; ++j)
      mma_chain(acol, tc::make_desc(z_tile + (1 + j) * z_stride, z_lbo, 1024), tc::make_desc(b_tile + (1 + j) * kTileBytes, 0, 1024),
                2048, 2048, kTcPts / 16, idesc, 1);
  }
  __syncthreads();
  if (t.hh == 0 && t.q * 32 < rows) {
    const int o = t.q * 32 + t.lane;
    float v[16];
    tc::acc_ld16(t.lane_addr + acol, v);
    if (o < n1w) {
#pragma unroll
      for (int k = 0; k < PINN_MAX_IN; ++k)
        if (k < d_in) atomicAdd(gw0 + o + (long long)n1w * k, v[k]);
      atomicAdd(gb0 + o, v[8]);
    }
  }
}

// channel structure <A1, A2, PU> of PINN_TC_DISPATCH; not instantiated when it has more than maxc channels
#define PINN_TC_CASE(maxc, a1, a2, pu, CALL)                                                  \
  {                                                                                           \
    constexpr int A1 = a1, A2 = a2;                                                           \
    constexpr bool PU = pu;                                                                   \
    if constexpr (1 + A1 + A2 <= (maxc)) {                                                    \
      if (_ak == 1) { constexpr int AK = 1; CALL; } else { constexpr int AK = 0; CALL; }     \
    }                                                                                         \
  }                                                                                           \
  break
// maxc: the kernel's channel limit; ak = 1 when every hidden layer of the network is tanh (fast branch-free activation), else 0
#define PINN_TC_DISPATCH(maxc, n1, n2, pure, ak, CALL)                                        \
  do {                                                                                        \
    const int _ak = (ak);                                                                     \
    const int _key = ((n1) * 8 + (n2)) * 2 + ((pure) ? 1 : 0);                                \
    switch (_key) {                                                                           \
      case (0 * 8 + 0) * 2: case (0 * 8 + 0) * 2 + 1: PINN_TC_CASE(maxc, 0, 0, true, CALL);   \
      case (1 * 8 + 0) * 2: case (1 * 8 + 0) * 2 + 1: PINN_TC_CASE(maxc, 1, 0, true, CALL);   \
      case (2 * 8 + 0) * 2: case (2 * 8 + 0) * 2 + 1: PINN_TC_CASE(maxc, 2, 0, true, CALL);   \
      case (3 * 8 + 0) * 2: case (3 * 8 + 0) * 2 + 1: PINN_TC_CASE(maxc, 3, 0, true, CALL);   \
      case (4 * 8 + 0) * 2: case (4 * 8 + 0) * 2 + 1: PINN_TC_CASE(maxc, 4, 0, true, CALL);   \
      case (1 * 8 + 1) * 2: case (1 * 8 + 1) * 2 + 1: PINN_TC_CASE(maxc, 1, 1, true, CALL);   \
      case (2 * 8 + 1) * 2 + 1: PINN_TC_CASE(maxc, 2, 1, true, CALL);                         \
      case (2 * 8 + 1) * 2: PINN_TC_CASE(maxc, 2, 1, false, CALL);                            \
      case (3 * 8 + 1) * 2 + 1: PINN_TC_CASE(maxc, 3, 1, true, CALL);                         \
      case (3 * 8 + 1) * 2: PINN_TC_CASE(maxc, 3, 1, false, CALL);                            \
      case (2 * 8 + 2) * 2 + 1: PINN_TC_CASE(maxc, 2, 2, true, CALL);                         \
      case (2 * 8 + 2) * 2: PINN_TC_CASE(maxc, 2, 2, false, CALL);                            \
      default: break;                                                                         \
    }                                                                                         \
  } while (0)

}  // namespace pinn
