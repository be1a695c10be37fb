// ffma_kernel.cuh -- fused PINN loss+gradient kernel, CUDA-core FMA path (parity mode).
//
// One persistent CTA per SM walks tiles of 32 collocation points (lane == point).  For a
// tile it runs, entirely on chip except for the layer stash:
//   1. MLP forward of every network the term taps, propagating the value channel plus
//      the first/second-derivative channels exactly (forward-mode "taps", SURVEY App. B)
//      -- replaces Phi (reference src/pinn_types.jl:79-90) and numeric_derivative
//      (src/pinn_types.jl:445-482);
//   2. the term's residual program r = lhs - rhs per point and its reverse sweep
//      -- replaces the RuntimeGeneratedFunction body (src/discretize.jl:28-175);
//   3. sum_p qw_p r_p^2 (mean(abs2, .), src/training_strategies.jl:220);
//   4. the reverse sweep through every network, accumulating d(total)/d(theta) into a
//      per-CTA partial (no atomics; reduced in fixed order by the kernel tail, tail.cuh,
//      so the gradient is deterministic) -- replaces the Zygote pullback (src/discretize.jl:778).
//
// Data layout: activation buffers are [channel][neuron][point] with the point index
// fastest and a row stride of TP = 32 + 16/sizeof(real) scalars, which makes both the
// lane==point accesses (forward / dgrad) and the 16-byte vector accesses with
// lane==neuron (wgrad) bank-conflict free.  Staged weights are W^T[k][o] = theta's own
// column-major out x in block, so no transpose is needed.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include "dev_types.h"
#include "tail.cuh"

namespace pinn {

template <typename real> struct VecOf;
template <> struct VecOf<float> { using type = float4; static constexpr int N = 4; };
template <> struct VecOf<double> { using type = double2; static constexpr int N = 2; };

template <typename real> __device__ __forceinline__ real vget(const typename VecOf<real>::type& v, int i);
template <> __device__ __forceinline__ float vget<float>(const float4& v, int i) {
  return i == 0 ? v.x : (i == 1 ? v.y : (i == 2 ? v.z : v.w));
}
template <> __device__ __forceinline__ double vget<double>(const double2& v, int i) {
  return i == 0 ? v.x : v.y;
}

template <typename real> __device__ __forceinline__ real rfma(real a, real b, real c);
template <> __device__ __forceinline__ float rfma<float>(float a, float b, float c) { return fmaf(a, b, c); }
template <> __device__ __forceinline__ double rfma<double>(double a, double b, double c) { return fma(a, b, c); }

// ---- math in the scalar type (accurate libm versions: this is the parity path) -----------
__device__ __forceinline__ float m_tanh(float x) { return tanhf(x); }
__device__ __forceinline__ double m_tanh(double x) { return tanh(x); }
__device__ __forceinline__ float m_exp(float x) { return expf(x); }
__device__ __forceinline__ double m_exp(double x) { return exp(x); }
__device__ __forceinline__ float m_log(float x) { return logf(x); }
__device__ __forceinline__ double m_log(double x) { return log(x); }
__device__ __forceinline__ float m_log1p(float x) { return log1pf(x); }
__device__ __forceinline__ double m_log1p(double x) { return log1p(x); }
__device__ __forceinline__ float m_sin(float x) { return sinf(x); }
__device__ __forceinline__ double m_sin(double x) { return sin(x); }
__device__ __forceinline__ float m_cos(float x) { return cosf(x); }
__device__ __forceinline__ double m_cos(double x) { return cos(x); }
__device__ __forceinline__ float m_sqrt(float x) { return sqrtf(x); }
__device__ __forceinline__ double m_sqrt(double x) { return sqrt(x); }
__device__ __forceinline__ float m_pow(float x, float y) { return powf(x, y); }
__device__ __forceinline__ double m_pow(double x, double y) { return pow(x, y); }
__device__ __forceinline__ float m_abs(float x) { return fabsf(x); }
__device__ __forceinline__ double m_abs(double x) { return fabs(x); }

template <typename real>
__device__ __forceinline__ real m_sigmoid(real z) {
  // stable for both signs
  if (z >= real(0)) {
    real e = m_exp(-z);
    return real(1) / (real(1) + e);
  }
  real e = m_exp(z);
  return e / (real(1) + e);
}

// NNlib's gelu, the tanh form z/2 (1 + T), T = tanh(u), u = c (z + k z^3), and its first four derivatives: T's
// z-derivatives by Faa di Bruno from tanh's u-derivatives t1..t4 and u1 = c (1 + 3k z^2), u2 = 6ck z, u3 = 6ck (u4 = 0)
template <typename real>
__device__ __forceinline__ void gelu_eval4(real z, real& a, real& d1, real& d2, real& d3, real& d4) {
  const real c = real(0.79788456080286535588), k = real(0.044715);
  const real z2 = z * z;
  real t = m_tanh(c * (z + k * z2 * z));
  real t1 = real(1) - t * t, t2 = real(-2) * t * t1, t3 = t1 * (real(6) * t * t - real(2));
  real t4 = real(8) * t * t1 * (real(2) - real(3) * t * t);
  real u1 = c * (real(1) + real(3) * k * z2), u2 = real(6) * c * k * z, u3 = real(6) * c * k;
  real T1 = t1 * u1, T2 = t2 * u1 * u1 + t1 * u2;
  real T3 = t3 * u1 * u1 * u1 + real(3) * t2 * u1 * u2 + t1 * u3;
  real T4 = t4 * u1 * u1 * u1 * u1 + real(6) * t3 * u1 * u1 * u2 + t2 * (real(3) * u2 * u2 + real(4) * u1 * u3);
  a = real(0.5) * z * (real(1) + t);
  d1 = real(0.5) * (real(1) + t + z * T1);
  d2 = real(0.5) * (real(2) * T1 + z * T2);
  d3 = real(0.5) * (real(3) * T2 + z * T3);
  d4 = real(0.5) * (real(4) * T3 + z * T4);
}

// NNlib's logcosh, z + softplus(-2z) - log 2, evaluated as |z| + log1p(exp(-2|z|)) - log 2 so that it neither
// overflows nor cancels for large |z|.  Its derivatives are tanh's shifted by one: t, 1 - t^2, -2t(1 - t^2), ...
template <typename real>
__device__ __forceinline__ void logcosh_eval4(real z, real& a, real& d1, real& d2, real& d3, real& d4) {
  const real az = m_abs(z);
  const real t = m_tanh(z), s = real(1) - t * t;
  a = az + m_log1p(m_exp(real(-2) * az)) - real(0.69314718055994530942);
  d1 = t; d2 = s; d3 = real(-2) * t * s; d4 = s * (real(6) * t * t - real(2));
}

// activation value and its first four derivatives at z (the fourth enters the reverse sweep through third-derivative taps).
// kFfmaOnly = false (the tensor-core kernels, which refuse gelu, logcosh and cos layers) leaves those three out, so their
// code stays as it was
template <typename real, bool kFfmaOnly = true>
__device__ __forceinline__ void act_eval4(int act, real z, real& a, real& d1, real& d2, real& d3, real& d4) {
  if constexpr (kFfmaOnly) {
    if (act >= PINN_ACT_GELU) {     // one compare on the common path, as with gelu alone
      if (act == PINN_ACT_GELU) {
        gelu_eval4<real>(z, a, d1, d2, d3, d4);
      } else if (act == PINN_ACT_LOGCOSH) {
        logcosh_eval4<real>(z, a, d1, d2, d3, d4);
      } else {
        const real s = m_sin(z), c = m_cos(z);
        a = c; d1 = -s; d2 = -c; d3 = s; d4 = c;
      }
      return;
    }
  }
  switch (act) {
    case PINN_ACT_TANH: {
      real t = m_tanh(z);
      real s = real(1) - t * t;
      a = t; d1 = s; d2 = real(-2) * t * s; d3 = s * (real(6) * t * t - real(2));
      d4 = real(8) * t * s * (real(2) - real(3) * t * t);
    } break;
    case PINN_ACT_SIGMOID: {
      real g = m_sigmoid(z);
      real g1 = g * (real(1) - g);
      real q = real(1) - real(2) * g;
      real g2 = g1 * q;
      real g3 = g2 * q - real(2) * g1 * g1;
      a = g; d1 = g1; d2 = g2; d3 = g3; d4 = g3 * q - real(6) * g1 * g2;
    } break;
    case PINN_ACT_SIN: {
      real s = m_sin(z), c = m_cos(z);
      a = s; d1 = c; d2 = -s; d3 = -c; d4 = s;
    } break;
    case PINN_ACT_SOFTPLUS: {
      real g = m_sigmoid(z);
      real g1 = g * (real(1) - g);
      real q = real(1) - real(2) * g;
      real g2 = g1 * q;
      a = (z > real(0)) ? z + m_log1p(m_exp(-z)) : m_log1p(m_exp(z));
      d1 = g; d2 = g1; d3 = g2; d4 = g2 * q - real(2) * g1 * g1;
    } break;
    case PINN_ACT_SWISH: {
      real g = m_sigmoid(z);
      real g1 = g * (real(1) - g);
      real q = real(1) - real(2) * g;
      real g2 = g1 * q;
      real g3 = g2 * q - real(2) * g1 * g1;
      real g4 = g3 * q - real(6) * g1 * g2;
      a = z * g; d1 = g + z * g1; d2 = real(2) * g1 + z * g2; d3 = real(3) * g2 + z * g3; d4 = real(4) * g3 + z * g4;
    } break;
    default:
      a = z; d1 = real(1); d2 = real(0); d3 = real(0); d4 = real(0);
  }
}
template <typename real, bool kFfmaOnly = true>
__device__ __forceinline__ void act_eval(int act, real z, real& a, real& d1, real& d2, real& d3) {
  real d4;
  act_eval4<real, kFfmaOnly>(act, z, a, d1, d2, d3, d4);
}

template <typename real> struct Cfg {
  static constexpr int VEC = VecOf<real>::N;
  static constexpr int TP = kTilePts + VEC;   // padded row stride (scalars)
};

// ------------------------------------------------------------------------------------------
// One block of 8 output neurons [ob, ob+8):
//   z[c][o][p] = sum_k W^T[k][o] * h[c][k][p] (+ bias on the value channel)
// lane == point.  Wt_blk points at W^T[0][ob] with row stride ldw (zero padded columns),
// bias_blk at bias[ob].
template <typename real, int C>
__device__ __forceinline__ void gemm_fwd_block(const real* Hin, real* Zout, const real* Wt_blk, const real* bias_blk,
                                               int n_in, int n_out, int ob, int ldw, int ldc, int lane) {
  using V = typename VecOf<real>::type;
  constexpr int VEC = VecOf<real>::N;
  constexpr int TP = Cfg<real>::TP;
  real acc[C][8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    acc[0][j] = bias_blk[j];
#pragma unroll
    for (int c = 1; c < C; ++c) acc[c][j] = real(0);
  }
#pragma unroll 2
  for (int k = 0; k < n_in; ++k) {
    real hv[C];
#pragma unroll
    for (int c = 0; c < C; ++c) hv[c] = Hin[c * ldc + k * TP + lane];
    real wv[8];
#pragma unroll
    for (int v = 0; v < 8 / VEC; ++v) {
      V w = *reinterpret_cast<const V*>(&Wt_blk[k * ldw + v * VEC]);
#pragma unroll
      for (int i = 0; i < VEC; ++i) wv[v * VEC + i] = vget<real>(w, i);
    }
#pragma unroll
    for (int c = 0; c < C; ++c)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[c][j] = rfma<real>(hv[c], wv[j], acc[c][j]);
  }
#pragma unroll
  for (int j = 0; j < 8; ++j)
    if (ob + j < n_out) {
#pragma unroll
      for (int c = 0; c < C; ++c) Zout[c * ldc + (ob + j) * TP + lane] = acc[c][j];
    }
}

// One block of 8 input neurons [kb, kb+8):
//   hbar_in[c][k][p] = sum_o zbar[c][o][p] * W^T[k][o]
// lane == point.  Wt_rows points at W^T[kb][0] with row stride ldw; columns >= n_out are zero.
template <typename real, int C>
__device__ __forceinline__ void gemm_dgrad_block(const real* Zbar, real* Hout, const real* Wt_rows, int n_in,
                                                 int n_out, int kb, int ldw, int ldc, int lane) {
  using V = typename VecOf<real>::type;
  constexpr int VEC = VecOf<real>::N;
  constexpr int TP = Cfg<real>::TP;
  const int n_outv = (n_out + VEC - 1) / VEC * VEC;
  real acc[C][8];
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int c = 0; c < C; ++c) acc[c][j] = real(0);
  for (int o = 0; o < n_outv; o += VEC) {
    V w[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) w[j] = *reinterpret_cast<const V*>(&Wt_rows[j * ldw + o]);
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      real zv[C];
#pragma unroll
      for (int c = 0; c < C; ++c) zv[c] = Zbar[c * ldc + (o + i) * TP + lane];
#pragma unroll
      for (int c = 0; c < C; ++c)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[c][j] = rfma<real>(zv[c], vget<real>(w[j], i), acc[c][j]);
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j)
    if (kb + j < n_in) {
#pragma unroll
      for (int c = 0; c < C; ++c) Hout[c * ldc + (kb + j) * TP + lane] = acc[c][j];
    }
}

// gW[o + n_out*k] += sum_{c,p} zbar[c][o][p] * h[c][k][p];  gb[o] += sum_p zbar[0][o][p]
// lane == output neuron, warp == block of 8 input neurons; 16-byte vectors along p.
// gW/gb point into this CTA's private gradient partial: plain read-modify-write.
template <typename real, int C>
__device__ __forceinline__ void gemm_wgrad(const real* Zbar, const real* H, real* gW, real* gb, int n_in,
                                           int n_out, int ldc, int warp, int lane) {
  using V = typename VecOf<real>::type;
  constexpr int VEC = VecOf<real>::N;
  constexpr int TP = Cfg<real>::TP;
  for (int ob = 0; ob < n_out; ob += 32) {
    const int o = ob + lane;
    const bool ovalid = o < n_out;
    const int oc = ovalid ? o : n_out - 1;
    for (int kb = warp * 8; kb < n_in; kb += kWarps * 8) {
      real acc[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = real(0);
#pragma unroll
      for (int c = 0; c < C; ++c) {
#pragma unroll 2
        for (int p = 0; p < kTilePts; p += VEC) {
          V zv = *reinterpret_cast<const V*>(&Zbar[c * ldc + oc * TP + p]);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            V hv = *reinterpret_cast<const V*>(&H[c * ldc + (kb + j) * TP + p]);
#pragma unroll
            for (int i = 0; i < VEC; ++i) acc[j] = rfma<real>(vget<real>(zv, i), vget<real>(hv, i), acc[j]);
          }
        }
      }
      if (ovalid) {
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (kb + j < n_in) gW[o + (long long)n_out * (kb + j)] += acc[j];
      }
    }
    if (warp == 0 && ovalid) {
      real s = real(0);
      for (int p = 0; p < kTilePts; p += VEC) {
        V zv = *reinterpret_cast<const V*>(&Zbar[oc * TP + p]);
#pragma unroll
        for (int i = 0; i < VEC; ++i) s += vget<real>(zv, i);
      }
      gb[o] += s;
    }
  }
}

// ---- the same three products on the FP64 tensor cores (PINN_MODE_TC_F64, double only) ----------------------------------
// mma.sync m16n8k16 .f64 (DMMA.16x8x16, sm_90).  Fragments of lane = 4 g + t: A a[i] at (row g + 8 (i&1), col t + 4 (i>>1)),
// B b[i] at (k t + 4 i, n g), C/D d[i] at (row g + 8 (i>>1), col 2 t + (i&1)).  Accumulators stay in registers; the
// fragments are read straight from the activation buffers and the staged weight panels.  Rows or k beyond a layer's
// width read as zero, so a partial k step adds exact zeros.  The products are calls, not inlined: inlined at every call
// site and channel count, the global-buffer units with integral terms take cicc longer than 20 minutes to compile.
__device__ __forceinline__ void dmma16816(double (&d)[4], const double (&a)[8], const double (&b)[4]) {
  asm("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
      "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
      : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
        "d"(b[2]), "d"(b[3]));
}

// Point of fragment row r (0..15) of m-tile mt, lane group g: the bits of g are spread so that the 16 lanes of a
// half-warp hit 16 distinct 8-byte bank pairs at the fp64 row stride TP = 34 (t * TP + dmma_pt(...) covers 0..15 mod 16).
__device__ __forceinline__ int dmma_pt(int g, int h, int mt) {
  return (g & 1) | ((g >> 2) << 1) | (h << 2) | (((g >> 1) & 1) << 3) | (mt << 4);
}

// gemm_fwd_block on DMMA: M = the 32 points (2 m-tiles, rows permuted by dmma_pt), N = the warp's 8 output neurons, K = n_in
template <int C>
__device__ __noinline__ void gemm_fwd_block_dmma(const double* Hin, double* Zout, const double* Wt_blk,
                                                    const double* bias_blk, int n_in, int n_out, int ob, int ldw, int ldc,
                                                    int lane) {
  constexpr int TP = Cfg<double>::TP;
  const int g = lane >> 2, t = lane & 3;
  double acc[C][2][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      acc[0][mt][i] = bias_blk[2 * t + (i & 1)];
#pragma unroll
      for (int c = 1; c < C; ++c) acc[c][mt][i] = 0.0;
    }
  int pa[2][2];   // points of this lane's A rows
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) pa[mt][h] = dmma_pt(g, h, mt);
  auto step = [&](int k0, bool tail) {
    double b[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int k = k0 + t + 4 * i;
      b[i] = (!tail || k < n_in) ? Wt_blk[k * ldw + g] : 0.0;
    }
#pragma unroll
    for (int c = 0; c < C; ++c)
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        double a[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int k = k0 + t + 4 * (i >> 1);
          a[i] = (!tail || k < n_in) ? Hin[c * ldc + k * TP + pa[mt][i & 1]] : 0.0;
        }
        dmma16816(acc[c][mt], a, b);
      }
  };
  int k0 = 0;
#pragma unroll 1
  for (; k0 + 16 <= n_in; k0 += 16) step(k0, false);
  if (k0 < n_in) step(k0, true);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int o = ob + 2 * t + (i & 1);
    if (o < n_out)
#pragma unroll
      for (int c = 0; c < C; ++c)
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) Zout[c * ldc + o * TP + pa[mt][i >> 1]] = acc[c][mt][i];
  }
}

// gemm_dgrad_block on DMMA: M = the 32 points, N = the warp's 8 input neurons, K = n_out
template <int C>
__device__ __noinline__ void gemm_dgrad_block_dmma(const double* Zbar, double* Hout, const double* Wt_rows, int n_in,
                                                      int n_out, int kb, int ldw, int ldc, int lane) {
  constexpr int TP = Cfg<double>::TP;
  const int g = lane >> 2, t = lane & 3;
  double acc[C][2][4];
#pragma unroll
  for (int c = 0; c < C; ++c)
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[c][mt][i] = 0.0;
  int pa[2][2];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) pa[mt][h] = dmma_pt(g, h, mt);
  auto step = [&](int o0, bool tail) {
    double b[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int o = o0 + t + 4 * i;
      b[i] = (!tail || o < n_out) ? Wt_rows[g * ldw + o] : 0.0;
    }
#pragma unroll
    for (int c = 0; c < C; ++c)
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        double a[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int o = o0 + t + 4 * (i >> 1);
          a[i] = (!tail || o < n_out) ? Zbar[c * ldc + o * TP + pa[mt][i & 1]] : 0.0;
        }
        dmma16816(acc[c][mt], a, b);
      }
  };
  int o0 = 0;
#pragma unroll 1
  for (; o0 + 16 <= n_out; o0 += 16) step(o0, false);
  if (o0 < n_out) step(o0, true);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int k = kb + 2 * t + (i & 1);
    if (k < n_in)
#pragma unroll
      for (int c = 0; c < C; ++c)
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) Hout[c * ldc + k * TP + pa[mt][i >> 1]] = acc[c][mt][i];
  }
}

// gemm_wgrad on DMMA: per (block of 32 outputs, warp's block of 8 inputs) M = the 32 outputs, N = the 8 inputs,
// K = C x 32 points (k permuted within each 16 so that both operands' loads are free of bank conflicts).  Every gW
// element has one owning lane (plain read-modify-write); the bias sum is gemm_wgrad's.
template <int C>
__device__ __noinline__ void gemm_wgrad_dmma(const double* Zbar, const double* H, double* gW, double* gb, int n_in,
                                                int n_out, int ldc, int warp, int lane) {
  constexpr int TP = Cfg<double>::TP;
  const int g = lane >> 2, t = lane & 3;
  int pk[4];   // point offset of k = t + 4 i within a 16-point step
#pragma unroll
  for (int i = 0; i < 4; ++i) pk[i] = (t & 1) | (i << 1) | ((t >> 1) << 3);
  for (int ob = 0; ob < n_out; ob += 32) {
    int orow[2][2];   // A rows (outputs), clamped into the layer
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int h = 0; h < 2; ++h) orow[mt][h] = min(ob + 16 * mt + 8 * h + g, n_out - 1);
    for (int kb = warp * 8; kb < n_in; kb += kWarps * 8) {
      double acc[2][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[mt][i] = 0.0;
#pragma unroll
      for (int c = 0; c < C; ++c)
#pragma unroll
        for (int p0 = 0; p0 < kTilePts; p0 += 16) {
          double b[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) b[i] = H[c * ldc + (kb + g) * TP + p0 + pk[i]];
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) {
            double a[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) a[i] = Zbar[c * ldc + orow[mt][i & 1] * TP + p0 + pk[i >> 1]];
            dmma16816(acc[mt], a, b);
          }
        }
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int o = ob + 16 * mt + 8 * (i >> 1) + g, k = kb + 2 * t + (i & 1);
          if (o < n_out && k < n_in) gW[o + (long long)n_out * k] += acc[mt][i];
        }
    }
    if (warp == 0 && ob + lane < n_out) {
      const int o = ob + lane;
      double s = 0.0;
      for (int p = 0; p < kTilePts; p += 2) {
        double2 zv = *reinterpret_cast<const double2*>(&Zbar[o * TP + p]);
        s += zv.x;
        s += zv.y;
      }
      gb[o] += s;
    }
  }
}

// the layer products of the kernel instantiation: CUDA-core FMA, or DMMA (DMMA: double only)
template <typename real, int C, bool DMMA>
__device__ __forceinline__ void gemm_fwd(const real* Hin, real* Zout, const real* Wt_blk, const real* bias_blk, int n_in,
                                         int n_out, int ob, int ldw, int ldc, int lane) {
  if constexpr (DMMA) gemm_fwd_block_dmma<C>(Hin, Zout, Wt_blk, bias_blk, n_in, n_out, ob, ldw, ldc, lane);
  else gemm_fwd_block<real, C>(Hin, Zout, Wt_blk, bias_blk, n_in, n_out, ob, ldw, ldc, lane);
}
template <typename real, int C, bool DMMA>
__device__ __forceinline__ void gemm_dgrad(const real* Zbar, real* Hout, const real* Wt_rows, int n_in, int n_out, int kb,
                                           int ldw, int ldc, int lane) {
  if constexpr (DMMA) gemm_dgrad_block_dmma<C>(Zbar, Hout, Wt_rows, n_in, n_out, kb, ldw, ldc, lane);
  else gemm_dgrad_block<real, C>(Zbar, Hout, Wt_rows, n_in, n_out, kb, ldw, ldc, lane);
}
template <typename real, int C, bool DMMA>
__device__ __forceinline__ void gemm_wgrad_any(const real* Zbar, const real* H, real* gW, real* gb, int n_in, int n_out,
                                               int ldc, int warp, int lane) {
  if constexpr (DMMA) gemm_wgrad_dmma<C>(Zbar, H, gW, gb, n_in, n_out, ldc, warp, lane);
  else gemm_wgrad<real, C>(Zbar, H, gW, gb, n_in, n_out, ldc, warp, lane);
}

#define PINN_DISPATCH_C(Cval, CALL)                                                   \
  switch (Cval) {                                                                     \
    case 1: { constexpr int CC = 1; CALL; } break;                                    \
    case 2: { constexpr int CC = 2; CALL; } break;                                    \
    case 3: { constexpr int CC = 3; CALL; } break;                                    \
    case 4: { constexpr int CC = 4; CALL; } break;                                    \
    case 5: { constexpr int CC = 5; CALL; } break;                                    \
    case 6: { constexpr int CC = 6; CALL; } break;                                    \
    case 7: { constexpr int CC = 7; CALL; } break;                                    \
    case 8: { constexpr int CC = 8; CALL; } break;                                    \
    case 9: { constexpr int CC = 9; CALL; } break;                                    \
    default: { constexpr int CC = 10; CALL; } break;                                  \
  }

// stage rows [k0, k0+nk) x columns [o0, o0+no) of a layer's W^T (zero padded outside the
// layer) into dst[nk][no], and bias[o0, o0+no) into bdst (if non-null)
template <typename real>
__device__ __forceinline__ void stage_panel(const real* __restrict__ theta, const DevNet& net, int l, int k0, int nk,
                                            int o0, int no, real* dst, real* bdst, int tid) {
  const int n_in = net.dims[l], n_out = net.dims[l + 1];
  const real* W = theta + net.w_off[l];
  for (int i = tid; i < nk * no; i += kThreads) {
    int kk = i / no, oo = i - kk * no;
    int k = k0 + kk, o = o0 + oo;
    dst[i] = (k < n_in && o < n_out) ? __ldg(&W[(long long)k * n_out + o]) : real(0);
  }
  if (bdst) {
    const real* B = theta + net.b_off[l];
    for (int i = tid; i < no; i += kThreads) bdst[i] = (o0 + i < n_out) ? __ldg(&B[o0 + i]) : real(0);
  }
}

// write the input channels of a network: value = selected coordinate rows, first-derivative
// seeds are one-hot, second-derivative seeds are zero.
template <typename real>
__device__ __forceinline__ void init_inputs(real* H, const real* Xs, const DevChan& ch, int n_in, int ldc, int tid) {
  constexpr int TP = Cfg<real>::TP;
  const int C = ch.C;
  for (int i = tid; i < C * n_in * kTilePts; i += kThreads) {
    int p = i & (kTilePts - 1);
    int rest = i / kTilePts;
    int k = rest % n_in;
    int c = rest / n_in;
    real v;
    if (c == 0) v = Xs[ch.rows[k] * kTilePts + p];
    else if (c <= ch.n1) v = (ch.dir1[c - 1] == k) ? real(1) : real(0);
    else v = real(0);
    H[c * ldc + k * TP + p] = v;
  }
}

// in-place activation of pre-activations Z (all channels), also saving Z into the stash
template <typename real>
__device__ __forceinline__ void elementwise_fwd(real* Z, real* stash, const DevChan& ch, int act, int n_out, int ldc,
                                                int warp, int lane, bool save) {
  constexpr int TP = Cfg<real>::TP;
  const int C = ch.C, n1 = ch.n1, n2 = ch.n2;
  for (int o = warp; o < n_out; o += kWarps) {
    const int idx = o * TP + lane;
    if (save)
      for (int c = 0; c < C; ++c) stash[(c * n_out + o) * kTilePts + lane] = Z[c * ldc + idx];
    real a, d1, d2, d3;
    act_eval<real>(act, Z[idx], a, d1, d2, d3);
    for (int q = 0; q < ch.n3; ++q) {       // pure third derivatives first: they read the pre-activations of the lower orders
      real z1 = Z[(1 + ch.t_a[q]) * ldc + idx];
      real z2 = Z[(n1 + 1 + ch.t_s[q]) * ldc + idx];
      real z3 = Z[(n1 + n2 + 1 + q) * ldc + idx];
      Z[(n1 + n2 + 1 + q) * ldc + idx] = d1 * z3 + real(3) * d2 * z1 * z2 + d3 * z1 * z1 * z1;
    }
    for (int s = 0; s < n2; ++s) {
      real zs = Z[(n1 + 1 + s) * ldc + idx];
      real za = Z[(1 + ch.s_a[s]) * ldc + idx];
      real zb = Z[(1 + ch.s_b[s]) * ldc + idx];
      Z[(n1 + 1 + s) * ldc + idx] = d1 * zs + d2 * za * zb;
    }
    for (int i = 0; i < n1; ++i) Z[(1 + i) * ldc + idx] = d1 * Z[(1 + i) * ldc + idx];
    Z[idx] = a;
  }
}

// in place: adjoints of post-activations -> adjoints of pre-activations, using stashed Z
template <typename real>
__device__ __forceinline__ void elementwise_bwd(real* B, const real* stash, const DevChan& ch, int act, int n_out,
                                                int ldc, int warp, int lane) {
  constexpr int TP = Cfg<real>::TP;
  const int n1 = ch.n1, n2 = ch.n2;
  for (int o = warp; o < n_out; o += kWarps) {
    const int idx = o * TP + lane;
    const int sidx = o * kTilePts + lane;
    const int cs = n_out * kTilePts;  // channel stride in the stash
    real a, d1, d2, d3, d4;
    act_eval4<real>(act, stash[sidx], a, d1, d2, d3, d4);
    real acc0 = d1 * B[idx];
    for (int i = 0; i < n1; ++i) {
      real zi = stash[(1 + i) * cs + sidx];
      real hb = B[(1 + i) * ldc + idx];
      acc0 += d2 * zi * hb;
      B[(1 + i) * ldc + idx] = d1 * hb;
    }
    for (int s = 0; s < n2; ++s) {
      const int ca = 1 + ch.s_a[s], cb = 1 + ch.s_b[s], cq = n1 + 1 + s;
      real zs = stash[cq * cs + sidx];
      real za = stash[ca * cs + sidx];
      real zb = stash[cb * cs + sidx];
      real hb = B[cq * ldc + idx];
      acc0 += (d2 * zs + d3 * za * zb) * hb;
      B[ca * ldc + idx] += d2 * zb * hb;
      B[cb * ldc + idx] += d2 * za * hb;
      B[cq * ldc + idx] = d1 * hb;
    }
    for (int q = 0; q < ch.n3; ++q) {       // h3 = d1 z3 + 3 d2 z1 z2 + d3 z1^3
      const int c1 = 1 + ch.t_a[q], c2 = n1 + 1 + ch.t_s[q], c3 = n1 + n2 + 1 + q;
      real z1 = stash[c1 * cs + sidx], z2 = stash[c2 * cs + sidx], z3 = stash[c3 * cs + sidx];
      real hb = B[c3 * ldc + idx];
      acc0 += (d2 * z3 + real(3) * d3 * z1 * z2 + d4 * z1 * z1 * z1) * hb;
      B[c1 * ldc + idx] += real(3) * (d2 * z2 + d3 * z1 * z1) * hb;
      B[c2 * ldc + idx] += real(3) * d2 * z1 * hb;
      B[c3 * ldc + idx] = d1 * hb;
    }
    B[idx] = acc0;
  }
}

// rebuild post-activation channels of a hidden layer from its stashed pre-activations
template <typename real>
__device__ __forceinline__ void rebuild_h(real* H, const real* stash, const DevChan& ch, int act, int n, int ldc,
                                          int warp, int lane) {
  constexpr int TP = Cfg<real>::TP;
  const int n1 = ch.n1, n2 = ch.n2;
  const int cs = n * kTilePts;
  for (int k = warp; k < n; k += kWarps) {
    const int idx = k * TP + lane;
    const int sidx = k * kTilePts + lane;
    real a, d1, d2, d3;
    act_eval<real>(act, stash[sidx], a, d1, d2, d3);
    H[idx] = a;
    for (int i = 0; i < n1; ++i) H[(1 + i) * ldc + idx] = d1 * stash[(1 + i) * cs + sidx];
    for (int s = 0; s < n2; ++s) {
      real zs = stash[(n1 + 1 + s) * cs + sidx];
      real za = stash[(1 + ch.s_a[s]) * cs + sidx];
      real zb = stash[(1 + ch.s_b[s]) * cs + sidx];
      H[(n1 + 1 + s) * ldc + idx] = d1 * zs + d2 * za * zb;
    }
    for (int q = 0; q < ch.n3; ++q) {
      real z1 = stash[(1 + ch.t_a[q]) * cs + sidx], z2 = stash[(n1 + 1 + ch.t_s[q]) * cs + sidx];
      real z3 = stash[(n1 + n2 + 1 + q) * cs + sidx];
      H[(n1 + n2 + 1 + q) * ldc + idx] = d1 * z3 + real(3) * d2 * z1 * z2 + d3 * z1 * z1 * z1;
    }
  }
}

// residual program: forward values and reverse adjoints, one point per lane (warp 0 only)
// STRIDE = points per tile in the Xs / taps / tapbar arrays ([index][point])
// SM: the program text and the per-point value / adjoint arrays live in shared memory (sprog, sval, sadj:
// [instr][point]) instead of global / local memory.
template <typename real, int STRIDE, bool SM>
__device__ __noinline__ real run_program_t(const DevInstr* prog, int n, const real* theta_p, const real* Xs, const real* taps,
                                            real* tapbar, real* pbar, int lane, bool want_adjoint, real* sval, real* sadj) {
  real lval[SM ? 1 : PINN_MAX_INSTR];
  real ladj[SM ? 1 : PINN_MAX_INSTR];
  real* val = SM ? (sval + lane) : lval;
  real* adj = SM ? (sadj + lane) : ladj;
  constexpr int VS = SM ? STRIDE : 1;
#define PV(i) val[(i) * VS]
#define PA(i) adj[(i) * VS]
  for (int i = 0; i < n; ++i) {
    const DevInstr& in = prog[i];
    real v;
    switch (in.op) {
      case PINN_OP_CONST: v = real(in.imm); break;
      case PINN_OP_COORD: v = Xs[in.a * STRIDE + lane]; break;
      case PINN_OP_TAP: v = taps[in.a * STRIDE + lane]; break;
      case PINN_OP_PARAM: v = theta_p[in.a]; break;
      case PINN_OP_ADD: v = PV(in.a) + PV(in.b); break;
      case PINN_OP_SUB: v = PV(in.a) - PV(in.b); break;
      case PINN_OP_MUL: v = PV(in.a) * PV(in.b); break;
      case PINN_OP_DIV: v = PV(in.a) / PV(in.b); break;
      case PINN_OP_NEG: v = -PV(in.a); break;
      case PINN_OP_POW: v = m_pow(PV(in.a), PV(in.b)); break;
      case PINN_OP_POWI: {
        int e = (int)in.imm;
        real b = PV(in.a), r = real(1);
        int ae = e < 0 ? -e : e;
        while (ae) { if (ae & 1) r *= b; b *= b; ae >>= 1; }
        v = e < 0 ? real(1) / r : r;
      } break;
      case PINN_OP_SIN: v = m_sin(PV(in.a)); break;
      case PINN_OP_COS: v = m_cos(PV(in.a)); break;
      case PINN_OP_EXP: v = m_exp(PV(in.a)); break;
      case PINN_OP_LOG: v = m_log(PV(in.a)); break;
      case PINN_OP_TANH: v = m_tanh(PV(in.a)); break;
      case PINN_OP_SQRT: v = m_sqrt(PV(in.a)); break;
      case PINN_OP_ABS: v = m_abs(PV(in.a)); break;
      default: v = real(0);
    }
    PV(i) = v;
  }
  const real r = PV(n - 1);
  if (!want_adjoint) return r;

  for (int i = 0; i < n; ++i) PA(i) = real(0);
  PA(n - 1) = real(1);
  for (int i = n - 1; i >= 0; --i) {
    const DevInstr& in = prog[i];
    const real g = PA(i);
    switch (in.op) {
      case PINN_OP_TAP: tapbar[in.a * STRIDE + lane] += g; break;
      case PINN_OP_PARAM: pbar[in.a] += g; break;
      case PINN_OP_ADD: PA(in.a) += g; PA(in.b) += g; break;
      case PINN_OP_SUB: PA(in.a) += g; PA(in.b) -= g; break;
      case PINN_OP_MUL: PA(in.a) += g * PV(in.b); PA(in.b) += g * PV(in.a); break;
      case PINN_OP_DIV: {
        real inv = real(1) / PV(in.b);
        PA(in.a) += g * inv;
        PA(in.b) -= g * PV(i) * inv;
      } break;
      case PINN_OP_NEG: PA(in.a) -= g; break;
      case PINN_OP_POW: {
        real x = PV(in.a), y = PV(in.b);
        PA(in.a) += g * y * m_pow(x, y - real(1));
        if (x > real(0)) PA(in.b) += g * PV(i) * m_log(x);
      } break;
      case PINN_OP_POWI: {
        int e = (int)in.imm;
        if (e != 0) {
          real b = PV(in.a), rr = real(1);
          int e1 = e - 1;
          int ae = e1 < 0 ? -e1 : e1;
          real bb = b;
          while (ae) { if (ae & 1) rr *= bb; bb *= bb; ae >>= 1; }
          if (e1 < 0) rr = real(1) / rr;
          PA(in.a) += g * real(e) * rr;
        }
      } break;
      case PINN_OP_SIN: PA(in.a) += g * m_cos(PV(in.a)); break;
      case PINN_OP_COS: PA(in.a) -= g * m_sin(PV(in.a)); break;
      case PINN_OP_EXP: PA(in.a) += g * PV(i); break;
      case PINN_OP_LOG: PA(in.a) += g / PV(in.a); break;
      case PINN_OP_TANH: PA(in.a) += g * (real(1) - PV(i) * PV(i)); break;
      case PINN_OP_SQRT: PA(in.a) += g * real(0.5) / PV(i); break;
      case PINN_OP_ABS: PA(in.a) += (PV(in.a) >= real(0)) ? g : -g; break;
      default: break;
    }
  }
  return r;
#undef PV
#undef PA
}

// STRIDE = points per tile in the Xs / taps / tapbar arrays ([index][point]); program read from the term
template <typename real, int STRIDE>
__device__ __forceinline__ real run_program(const DevTerm& tm, const real* theta_p, const real* Xs, const real* taps,
                                            real* tapbar, real* pbar, int lane, bool want_adjoint) {
  return run_program_t<real, STRIDE, false>(tm.prog, tm.n_instr, theta_p, Xs, taps, tapbar, pbar, lane, want_adjoint,
                                            (real*)nullptr, (real*)nullptr);
}

template <typename real>
__device__ __forceinline__ real warp_sum(real v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- fixed networks (pinn_create_ex2): network index n_nets + j is fixed network j -------------------------------------
// FIXED: the instantiation for problems with fixed networks; without it these compile to the old reads
template <bool FIXED>
__device__ __forceinline__ bool is_fixed(const DevProblem& P, int k) {
  if constexpr (FIXED) return k >= P.n_nets;
  return false;
}
template <bool FIXED>
__device__ __forceinline__ const DevNet& net_of(const DevProblem& P, int k) {
  if constexpr (FIXED)
    if (k >= P.n_nets) return P.fixed[k - P.n_nets];
  return P.nets[k];
}
template <typename real>
__device__ __forceinline__ const real* fixed_params(const DevProblem& P, int k) {
  return reinterpret_cast<const real*>(P.fixed_params[k - P.n_nets]);
}

// ------------------------------------------------------------------------------------------
// forward through every network term tm taps, at the point tile X ([row][point]): the outputs land in taps; save:
// keep the pre-activations in the stash for the reverse sweep
template <typename real, bool FIXED, bool DMMA>
__device__ __forceinline__ void forward_nets(const FfmaArgs& args, const DevProblem& P, const DevTerm& tm,
                                             const real* __restrict__ theta, const real* X, real* bufA, real* bufB,
                                             real* wsm, real* stash, real* taps, bool save, int ldc, int tid, int warp,
                                             int lane) {
  constexpr int TP = Cfg<real>::TP;
  for (int slot = 0; slot < tm.n_used; ++slot) {
    const int k = tm.used_net[slot];
    const DevNet& net = net_of<FIXED>(P, k);
    const bool fixed = is_fixed<FIXED>(P, k);
    const real* src = fixed ? fixed_params<real>(P, k) : theta;   // a fixed network saves nothing to the stash
    const DevChan& ch = tm.chan[slot];
    const int C = ch.C;
    real* H = bufA;
    real* Z = bufB;
    init_inputs<real>(H, X, ch, net.dims[0], ldc, tid);
    for (int l = 0; l < net.n_layers; ++l) {
      const int n_in = net.dims[l], n_out = net.dims[l + 1];
      const int n_in8 = (n_in + 7) & ~7, n_out8 = (n_out + 7) & ~7;
      if (args.weights_resident) {
        const real* Wt = wsm + net.ws_off[l];
        const real* bs = wsm + net.bs_off[l];
        __syncthreads();   // layer inputs visible
        for (int ob = warp * 8; ob < n_out8; ob += kWarps * 8) {
          PINN_DISPATCH_C(C, (gemm_fwd<real, CC, DMMA>(H, Z, Wt + ob, bs + ob, n_in, n_out, ob, n_out8, ldc, lane)));
        }
        __syncthreads();
      } else {
        constexpr int PW = kWarps * 8;   // panel of 64 output neurons
        for (int pb = 0; pb < n_out8; pb += PW) {
          stage_panel<real>(src, net, l, 0, n_in8, pb, PW, wsm, wsm + n_in8 * PW, tid);
          __syncthreads();   // panel (and, first time, layer inputs) visible
          const int ob = pb + warp * 8;
          if (ob < n_out8) {
            PINN_DISPATCH_C(C, (gemm_fwd<real, CC, DMMA>(H, Z, wsm + warp * 8, wsm + n_in8 * PW + warp * 8, n_in,
                                                         n_out, ob, PW, ldc, lane)));
          }
          __syncthreads();   // panel consumed
        }
      }
      elementwise_fwd<real>(Z, stash + ch.stash_off[l], ch, net.acts[l], n_out, ldc, warp, lane, save && !fixed);
      real* t = H; H = Z; Z = t;
      // the next layer's __syncthreads (or the one below) orders these writes
    }
    __syncthreads();
    // network outputs -> taps
    for (int i = tid; i < tm.n_taps * kTilePts; i += kThreads) {
      int t = i / kTilePts, p = i - t * kTilePts;
      if (tm.tap_slot[t] == slot) taps[i] = H[tm.tap_ch[t] * ldc + tm.tap_out[t] * TP + p];
    }
    __syncthreads();
  }
}

// reverse sweep through every network term tm taps, from the tap adjoints tapbar, into this CTA's gradient partial
// (fixed networks are skipped: their tap adjoints reach nothing trainable)
template <typename real, bool FIXED, bool DMMA>
__device__ __forceinline__ void reverse_nets(const FfmaArgs& args, const DevProblem& P, const DevTerm& tm,
                                             const real* __restrict__ theta, const real* X, real* bufA, real* bufB,
                                             real* wsm, const real* stash, const real* tapbar, real* partial, int ldc,
                                             int tid, int warp, int lane) {
  constexpr int TP = Cfg<real>::TP;
  for (int slot = 0; slot < tm.n_used; ++slot) {
    if (is_fixed<FIXED>(P, tm.used_net[slot])) continue;   // uniform over the CTA
    const DevNet& net = P.nets[tm.used_net[slot]];
    const DevChan& ch = tm.chan[slot];
    const int C = ch.C;
    const int L = net.n_layers;
    real* B = bufA;   // adjoints
    real* H = bufB;   // rebuilt layer inputs
    // seed: adjoint of the network outputs
    {
      const int n_out = net.dims[L];
      for (int i = tid; i < C * n_out * kTilePts; i += kThreads) {
        int p = i & (kTilePts - 1);
        int rest = i / kTilePts;
        int o = rest % n_out, c = rest / n_out;
        B[c * ldc + o * TP + p] = real(0);
      }
      __syncthreads();
      // several taps may name the same (channel, out) element: one thread per point accumulates
      if (tid < kTilePts) {
        for (int t = 0; t < tm.n_taps; ++t)
          if (tm.tap_slot[t] == slot)
            B[tm.tap_ch[t] * ldc + tm.tap_out[t] * TP + tid] += tapbar[t * kTilePts + tid];
      }
      __syncthreads();
    }
    for (int l = L - 1; l >= 0; --l) {
      const int n_in = net.dims[l], n_out = net.dims[l + 1];
      const int n_in8 = (n_in + 7) & ~7, n_out8 = (n_out + 7) & ~7;
      elementwise_bwd<real>(B, stash + ch.stash_off[l], ch, net.acts[l], n_out, ldc, warp, lane);
      if (l == 0) init_inputs<real>(H, X, ch, n_in, ldc, tid);
      else rebuild_h<real>(H, stash + ch.stash_off[l - 1], ch, net.acts[l - 1], n_in, ldc, warp, lane);
      __syncthreads();
      PINN_DISPATCH_C(C, (gemm_wgrad_any<real, CC, DMMA>(B, H, partial + net.w_off[l], partial + net.b_off[l], n_in,
                                               n_out, ldc, warp, lane)));
      if (l > 0) {
        __syncthreads();   // wgrad finished reading H before dgrad overwrites it
        if (args.weights_resident) {
          const real* Wt = wsm + net.ws_off[l];
          for (int kb = warp * 8; kb < n_in8; kb += kWarps * 8) {
            PINN_DISPATCH_C(C, (gemm_dgrad<real, CC, DMMA>(B, H, Wt + kb * n_out8, n_in, n_out, kb, n_out8, ldc,
                                                           lane)));
          }
        } else {
          constexpr int PW = kWarps * 8;   // panel of 64 input neurons
          for (int pb = 0; pb < n_in8; pb += PW) {
            stage_panel<real>(theta, net, l, pb, PW, 0, n_out8, wsm, (real*)nullptr, tid);
            __syncthreads();
            const int kb = pb + warp * 8;
            if (kb < n_in8) {
              PINN_DISPATCH_C(C, (gemm_dgrad<real, CC, DMMA>(B, H, wsm + warp * 8 * n_out8, n_in, n_out, kb,
                                                             n_out8, ldc, lane)));
            }
            __syncthreads();
          }
        }
        real* t = B; B = H; H = t;
      }
      __syncthreads();
    }
  }
}

// ---- integral terms (pinn_create_ex) -----------------------------------------------------------------------------------
// The owner tile's 32 points (lane == point) and node j of integral I give one more tile of 32 node points, lane ==
// owner point: no cross-lane reduction, no grid barrier, no extra launch.  The forward pass runs every node tile and
// accumulates I_p = sum_j w_j(p) g_j(p) in a register of warp 0; the reverse pass recomputes each node tile and sweeps it
// back with the seed dtotal/dI_p * w_j(p).

// node j of integral I for this lane's owner point: writes the node point (the owner's rows with the integrating rows
// replaced by x_k(t_k), then the t_k) into Xn and returns the node weight w_j(p) = prod_k (hi_k - lo_k) / 2 * wq[j_k]
template <typename real>
__device__ __forceinline__ real node_tile(const DevIntegral& I, int dim, int j, const real* Xs, real* Xn, int lane) {
  for (int r = 0; r < dim; ++r) Xn[r * kTilePts + lane] = Xs[r * kTilePts + lane];
  real w = real(1);
  for (int k = 0; k < I.n_dims; ++k, j /= I.q) {
    const int jk = j % I.q;
    const real lo = I.lb_row[k] >= 0 ? Xs[I.lb_row[k] * kTilePts + lane] : real(I.lb[k]);
    const real hi = I.ub_row[k] >= 0 ? Xs[I.ub_row[k] * kTilePts + lane] : real(I.ub[k]);
    const real h = real(0.5) * (hi - lo);
    const real t = lo + h * (real(1) + real(I.xi[jk]));
    real x = t;
    if (I.inf_kind[k] == PINN_INF_BOTH) x = t / (real(1) - t * t);
    else if (I.inf_kind[k] == PINN_INF_UPPER) x = real(I.shift[k]) + t / (real(1) - t);
    else if (I.inf_kind[k] == PINN_INF_LOWER) x = real(I.shift[k]) + t / (real(1) + t);
    Xn[I.row[k] * kTilePts + lane] = x;
    Xn[(dim + k) * kTilePts + lane] = t;
    w *= h * real(I.wq[jk]);
  }
  return w;
}

inline __device__ int node_count(const DevIntegral& I) { return I.n_dims == 2 ? I.q * I.q : I.q; }

// values of term ti's integrals at the owner tile Xs: ival[k][p] for its k-th integral
template <typename real, bool FIXED, bool DMMA>
__device__ __forceinline__ void integrals_forward(const FfmaArgs& args, const DevProblem& P, int ti,
                                                  const real* __restrict__ theta, const real* Xs, real* Xn, real* ival,
                                                  real* bufA, real* bufB, real* wsm, real* stash, real* taps, int tid,
                                                  int warp, int lane) {
  int k = 0;
  for (int i = 0; i < P.n_integrals; ++i) {
    const DevIntegral& I = P.integ[i];
    if (I.owner != ti) continue;
    real acc = real(0), wj = real(0);
    for (int j = 0; j < node_count(I); ++j) {
      if (warp == 0) wj = node_tile<real>(I, P.terms[ti].dim, j, Xs, Xn, lane);
      __syncthreads();
      forward_nets<real, FIXED, DMMA>(args, P, I.body, theta, Xn, bufA, bufB, wsm, stash, taps, false, args.ldc, tid, warp, lane);
      if (warp == 0)
        acc += wj * run_program<real, kTilePts>(I.body, theta + P.param_off, Xn, taps, (real*)nullptr, (real*)nullptr,
                                                lane, false);
    }
    if (warp == 0) ival[k * kTilePts + lane] = acc;
    ++k;
  }
}

// gradient of term ti's integrals, given ibar[k][p] = dtotal / dI_p of its k-th integral
template <typename real, bool FIXED, bool DMMA>
__device__ __forceinline__ void integrals_reverse(const FfmaArgs& args, const DevProblem& P, int ti,
                                                  const real* __restrict__ theta, const real* Xs, real* Xn,
                                                  const real* ibar, real* bufA, real* bufB, real* wsm, real* stash,
                                                  real* taps, real* tapbar, real* partial, int tid, int warp, int lane) {
  int k = 0;
  for (int i = 0; i < P.n_integrals; ++i) {
    const DevIntegral& I = P.integ[i];
    if (I.owner != ti) continue;
    const DevTerm& body = I.body;
    real wj = real(0);
    for (int j = 0; j < node_count(I); ++j) {
      if (warp == 0) wj = node_tile<real>(I, P.terms[ti].dim, j, Xs, Xn, lane);
      __syncthreads();
      forward_nets<real, FIXED, DMMA>(args, P, body, theta, Xn, bufA, bufB, wsm, stash, taps, true, args.ldc, tid, warp, lane);
      if (warp == 0) {
        real pbar[PINN_MAX_PARAMS];
#pragma unroll
        for (int q = 0; q < PINN_MAX_PARAMS; ++q) pbar[q] = real(0);
        for (int t = 0; t < body.n_taps; ++t) tapbar[t * kTilePts + lane] = real(0);
        run_program<real, kTilePts>(body, theta + P.param_off, Xn, taps, tapbar, pbar, lane, true);
        const real sd = ibar[k * kTilePts + lane] * wj;
        for (int t = 0; t < body.n_taps; ++t) tapbar[t * kTilePts + lane] *= sd;
        for (int q = 0; q < P.n_params; ++q) {
          real v = warp_sum<real>(pbar[q] * sd);
          if (lane == 0) partial[P.param_off + q] += v;
        }
      }
      __syncthreads();
      reverse_nets<real, FIXED, DMMA>(args, P, body, theta, Xn, bufA, bufB, wsm, stash, tapbar, partial, args.ldc, tid, warp, lane);
    }
    ++k;
  }
}

// ------------------------------------------------------------------------------------------
// INTEG: the problem has integral terms (pinn_create_ex); FIXED: it has fixed networks (pinn_create_ex2), instantiated
// with INTEG = true only.  <false, false> is the kernel without either, <true, false> the integral kernel as it was.
// FUNC: the problem has a functional term (PINN_REDUCE_*_OF_SUM), instantiated with INTEG = FIXED = true only.  Its
// tiles add sum_p w_p v_p to the term sum and sweep back the seed w_p into this CTA's row of the second partial G (after
// the ordinary partials of the launch); the tail scales G by g'(S) once S is known.
// DMMA: PINN_MODE_TC_F64, double only: the three layer products run on the FP64 tensor cores (gemm_*_dmma); everything
// else is the FMA instantiation's.
template <typename real, bool BUFS_SMEM, bool INTEG, bool FIXED, bool FUNC, bool DMMA>
__global__ void __launch_bounds__(kThreads, 1) ffma_loss_grad_kernel(const FfmaArgs args) {
  static_assert(!DMMA || sizeof(real) == 8, "the DMMA layer products are fp64");
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const DevProblem& P = *args.prob;
  const real* __restrict__ theta = reinterpret_cast<const real*>(args.theta);
  const int ldc = args.ldc;

  // ---- carve shared memory --------------------------------------------------------------
  real* sm = reinterpret_cast<real*>(smem_raw);
  real *bufA, *bufB;
  if (BUFS_SMEM) {
    bufA = sm; sm += args.buf_elems;
    bufB = sm; sm += args.buf_elems;
  } else {
    real* g = reinterpret_cast<real*>(args.gbufs) + (long long)blockIdx.x * 2 * args.buf_elems;
    bufA = g; bufB = g + args.buf_elems;
  }
  real* wsm = sm; sm += args.w_area;
  real* Xs = sm; sm += PINN_MAX_DIM * kTilePts;
  real* taps = sm; sm += PINN_MAX_TAPS * kTilePts;
  real* tapbar = sm; sm += PINN_MAX_TAPS * kTilePts;
  real* rres = sm; sm += kTilePts;      // residual per point
  real* qws = sm; sm += kTilePts;       // quadrature weight per point (0 for padded lanes)
  double* tsum = reinterpret_cast<double*>(sm);  // [PINN_MAX_TERMS], 8-byte aligned by construction
  real* Xn = reinterpret_cast<real*>(tsum + PINN_MAX_TERMS);   // integral terms: node-point tile
  real* ival = Xn + (PINN_MAX_DIM + 2) * kTilePts;              // integral terms: the term's integrals, then their adjoints

  real* partial = reinterpret_cast<real*>(args.partial) + (long long)blockIdx.x * args.partial_stride;
  real* stash = reinterpret_cast<real*>(args.stash) + (long long)blockIdx.x * args.stash_per_cta;
  const bool want_grad = (args.mode == 0);
  real* gpart = partial;   // FUNC: this CTA's row of G
  if constexpr (FUNC)
    gpart = reinterpret_cast<real*>(args.partial) + ((long long)gridDim.x + blockIdx.x) * args.partial_stride;

  // ---- per-CTA init ------------------------------------------------------------------------
  for (long long i = tid; i < 2 * args.buf_elems; i += kThreads) {
    if (i < args.buf_elems) bufA[i] = real(0); else bufB[i - args.buf_elems] = real(0);
  }
  if (want_grad)
    for (long long i = tid; i < P.n_theta; i += kThreads) partial[i] = real(0);
  if constexpr (FUNC)
    if (want_grad)
      for (long long i = tid; i < P.n_theta; i += kThreads) gpart[i] = real(0);
  if (tid < PINN_MAX_TERMS) tsum[tid] = 0.0;
  if (args.weights_resident) {
    for (int k = 0; k < P.n_nets; ++k)
      for (int l = 0; l < P.nets[k].n_layers; ++l)
        stage_panel<real>(theta, P.nets[k], l, 0, (P.nets[k].dims[l] + 7) & ~7, 0, (P.nets[k].dims[l + 1] + 7) & ~7,
                          wsm + P.nets[k].ws_off[l], wsm + P.nets[k].bs_off[l], tid);
    if constexpr (FIXED)
      for (int j = 0; j < P.n_fixed; ++j) {
        const DevNet& f = P.fixed[j];
        for (int l = 0; l < f.n_layers; ++l)
          stage_panel<real>(reinterpret_cast<const real*>(P.fixed_params[j]), f, l, 0, (f.dims[l] + 7) & ~7, 0,
                            (f.dims[l + 1] + 7) & ~7, wsm + f.ws_off[l], wsm + f.bs_off[l], tid);
      }
  }
  __syncthreads();

  for (int tile = args.tile_begin + blockIdx.x; tile < args.tile_end; tile += gridDim.x) {
    // ---- locate the term (uniform) ------------------------------------------------------
    int ti = 0;
    while (ti + 1 < P.n_terms && tile >= args.dyn[ti + 1].tile0) ++ti;
    const DevTerm& tm = P.terms[ti];
    const long long p0 = (long long)(tile - args.dyn[ti].tile0) * kTilePts;
    const long long n_pts = args.dyn[ti].n;
    const real* pts = reinterpret_cast<const real*>(args.dyn[ti].pts);
    const real* qw = reinterpret_cast<const real*>(args.dyn[ti].qw);
    bool func = false;                 // the functional term (uniform)
    if constexpr (FUNC) func = ti == P.func_term;

    // ---- load the point tile ---------------------------------------------------------------
    for (int i = tid; i < tm.dim * kTilePts; i += kThreads) {
      int p = i / tm.dim, r = i - p * tm.dim;
      long long gp = p0 + p;
      if (gp >= n_pts) gp = n_pts - 1;
      Xs[r * kTilePts + p] = pts[gp * tm.dim + r];
    }
    if (tid < kTilePts) {
      long long gp = p0 + tid;
      real w = real(0);
      if (gp < n_pts) w = tm.weighted ? qw[gp] : real(1);
      if constexpr (FUNC)
        if (func && gp < n_pts && qw) w = qw[gp];   // nullable weights: 1 when none are given
      qws[tid] = w;
    }
    for (int i = tid; i < tm.n_taps * kTilePts; i += kThreads) tapbar[i] = real(0);
    __syncthreads();

    int n_int = 0;   // integrals of this term (uniform)
    if constexpr (INTEG) {
      for (int i = 0; i < P.n_integrals; ++i) n_int += P.integ[i].owner == ti;
      if (n_int) integrals_forward<real, FIXED, DMMA>(args, P, ti, theta, Xs, Xn, ival, bufA, bufB, wsm, stash, taps, tid, warp, lane);
    }

    // ---- forward through every tapped network ------------------------------------------------
    forward_nets<real, FIXED, DMMA>(args, P, tm, theta, Xs, bufA, bufB, wsm, stash, taps, want_grad, ldc, tid, warp, lane);

    // ---- residual, loss partial, tap adjoints (warp 0, lane == point) --------------------------
    if (warp == 0) {
      real pbar[PINN_MAX_PARAMS];
#pragma unroll
      for (int j = 0; j < PINN_MAX_PARAMS; ++j) pbar[j] = real(0);
      if constexpr (INTEG)
        for (int k = 0; k < n_int; ++k) {   // the program reads integral k as tap n_taps + k
          taps[(tm.n_taps + k) * kTilePts + lane] = ival[k * kTilePts + lane];
          tapbar[(tm.n_taps + k) * kTilePts + lane] = real(0);
        }
      const real r = run_program<real, kTilePts>(tm, theta + P.param_off, Xs, taps, tapbar, pbar, lane, want_grad);
      const real w = qws[lane];
      rres[lane] = r;
      double s = (double)w * (double)r * (double)r;
      if constexpr (FUNC)
        if (func) s = (double)w * (double)r;     // sum_p w_p v_p
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) tsum[ti] += s;
      if (args.mode == 2) {
        long long gp = p0 + lane;
        if (gp < n_pts) reinterpret_cast<real*>(args.resid_out)[gp] = r;
      }
      if (want_grad) {
        real g = real(args.seed[ti]) * w * real(2) * r;   // d total / d r_p
        real* dst = partial;
        if constexpr (FUNC)
          if (func) { g = w; dst = gpart; }           // d S / d v_p, into G
        for (int t = 0; t < tm.n_taps; ++t) tapbar[t * kTilePts + lane] *= g;
        if constexpr (INTEG)
          for (int k = 0; k < n_int; ++k) ival[k * kTilePts + lane] = tapbar[(tm.n_taps + k) * kTilePts + lane] * g;
        for (int j = 0; j < P.n_params; ++j) {
          real v = warp_sum<real>(pbar[j] * g);
          if (lane == 0) dst[P.param_off + j] += v;
        }
      }
    }
    __syncthreads();

    // ---- reverse sweep through every tapped network -----------------------------------------------
    if (want_grad)
      reverse_nets<real, FIXED, DMMA>(args, P, tm, theta, Xs, bufA, bufB, wsm, stash, tapbar, func ? gpart : partial, ldc, tid,
                                warp, lane);
    if constexpr (INTEG)
      if (want_grad && n_int)
        integrals_reverse<real, FIXED, DMMA>(args, P, ti, theta, Xs, Xn, ival, bufA, bufB, wsm, stash, taps, tapbar, partial, tid, warp,
                                lane);
  }

  __syncthreads();
  if (tid < PINN_MAX_TERMS) args.term_sums[(long long)blockIdx.x * PINN_MAX_TERMS + tid] = tsum[tid];
  // gradient reduction, optimizer step and the multi-GPU sum in the kernel tail (tail.cuh)
  if (args.tail.state)
    fused_tail<real, kThreads, FUNC>(args.tail, reinterpret_cast<const real*>(args.partial), args.partial_stride, args.term_sums,
                               P.n_theta, P.n_terms, want_grad ? 1 : 0, taps);
}


}  // namespace pinn
