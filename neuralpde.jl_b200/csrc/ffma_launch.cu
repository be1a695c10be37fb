// ffma_launch.cu -- host-callable launchers of the FFMA path, finish_kernel (unpacks the NCCL fallback's
// allreduced [grad | term losses]), the gradient statistics kernel and the device-side point samplers.
#include <cuda_runtime.h>
#include "dev_types.h"
#include "philox.cuh"

namespace pinn {

// after the allreduce of packed = [grad | term losses]: copy the gradient out and form total = sum_k w_k L_k
template <typename real>
__global__ void finish_kernel(const real* __restrict__ packed, long long n_grad, int n_terms, const ScaleW sw, real* out_grad,
                              real* out_terms, real* out_total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (out_grad && i < n_grad) out_grad[i] = packed[i];
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    const real* packed_terms = packed + n_grad;
    double tot = 0.0;
    for (int k = 0; k < n_terms; ++k) {
      double Lk = (double)packed_terms[k];
      out_terms[k] = real(Lk);
      tot += Lk * sw.w[k];
    }
    *out_total = real(tot);
  }
}

// ---- host-callable launchers -------------------------------------------------------------------
// integ: after the term sums, the node-point tile ((PINN_MAX_DIM + 2) rows) and one row per integral of the term
size_t ffma_smem_bytes(int dtype, long long buf_elems, int w_area, bool bufs_smem, bool integ) {
  size_t es = dtype == PINN_F64 ? 8 : 4;
  size_t n = (bufs_smem ? 2 * (size_t)buf_elems : 0) + (size_t)w_area + PINN_MAX_DIM * kTilePts +
             2 * PINN_MAX_TAPS * kTilePts + 2 * kTilePts;
  size_t bytes = n * es;
  bytes = (bytes + 7) & ~size_t(7);
  bytes += PINN_MAX_TERMS * sizeof(double);
  if (integ) bytes += (size_t)(PINN_MAX_DIM + 2 + PINN_MAX_INTEGRALS) * kTilePts * es;
  return bytes;
}

cudaError_t ffma_launch_float_smem(const FfmaArgs& a, int grid, size_t smem, cudaStream_t st);
cudaError_t ffma_launch_float_gmem(const FfmaArgs& a, int grid, size_t smem, cudaStream_t st);
cudaError_t ffma_launch_double_smem(const FfmaArgs& a, int grid, size_t smem, cudaStream_t st);
cudaError_t ffma_launch_double_gmem(const FfmaArgs& a, int grid, size_t smem, cudaStream_t st);
cudaError_t ffma_launch_float_smem_integ(const FfmaArgs& a, int grid, size_t smem, cudaStream_t st);
cudaError_t ffma_launch_float_gmem_integ(const FfmaArgs& a, int grid, size_t smem, cudaStream_t st);
cudaError_t ffma_launch_double_smem_integ(const FfmaArgs& a, int grid, size_t smem, cudaStream_t st);
cudaError_t ffma_launch_double_gmem_integ(const FfmaArgs& a, int grid, size_t smem, cudaStream_t st);
cudaError_t ffma_launch_float_smem_fixed(const FfmaArgs& a, int grid, size_t smem, cudaStream_t st);
cudaError_t ffma_launch_float_gmem_fixed(const FfmaArgs& a, int grid, size_t smem, cudaStream_t st);
cudaError_t ffma_launch_double_smem_fixed(const FfmaArgs& a, int grid, size_t smem, cudaStream_t st);
cudaError_t ffma_launch_double_gmem_fixed(const FfmaArgs& a, int grid, size_t smem, cudaStream_t st);
cudaError_t ffma_launch_float_smem_func(const FfmaArgs& a, int grid, size_t smem, cudaStream_t st);
cudaError_t ffma_launch_float_gmem_func(const FfmaArgs& a, int grid, size_t smem, cudaStream_t st);
cudaError_t ffma_launch_double_smem_func(const FfmaArgs& a, int grid, size_t smem, cudaStream_t st);
cudaError_t ffma_launch_double_gmem_func(const FfmaArgs& a, int grid, size_t smem, cudaStream_t st);
cudaError_t ffma_launch_double_dmma_smem(const FfmaArgs& a, int grid, size_t smem, cudaStream_t st);
cudaError_t ffma_launch_double_dmma_gmem(const FfmaArgs& a, int grid, size_t smem, cudaStream_t st);
cudaError_t ffma_launch_double_dmma_smem_integ(const FfmaArgs& a, int grid, size_t smem, cudaStream_t st);
cudaError_t ffma_launch_double_dmma_gmem_integ(const FfmaArgs& a, int grid, size_t smem, cudaStream_t st);
cudaError_t ffma_launch_double_dmma_smem_fixed(const FfmaArgs& a, int grid, size_t smem, cudaStream_t st);
cudaError_t ffma_launch_double_dmma_gmem_fixed(const FfmaArgs& a, int grid, size_t smem, cudaStream_t st);
cudaError_t ffma_launch_double_dmma_smem_func(const FfmaArgs& a, int grid, size_t smem, cudaStream_t st);
cudaError_t ffma_launch_double_dmma_gmem_func(const FfmaArgs& a, int grid, size_t smem, cudaStream_t st);

// integ: the instantiation that evaluates integral terms on node tiles; fixed: the one that also evaluates fixed networks;
// func: the one that also evaluates a functional term; dmma: the fp64 one with its layer products on DMMA
// (PINN_MODE_TC_F64; the planner admits it with PINN_F64 only)
cudaError_t ffma_launch(int dtype, bool bufs_smem, bool integ, bool fixed, bool func, bool dmma, const FfmaArgs& a,
                        int grid, size_t smem, cudaStream_t st) {
  const bool f64 = dtype == PINN_F64;
  if (dmma) {
    if (!f64) return cudaErrorInvalidValue;
    if (func) return bufs_smem ? ffma_launch_double_dmma_smem_func(a, grid, smem, st) : ffma_launch_double_dmma_gmem_func(a, grid, smem, st);
    if (fixed) return bufs_smem ? ffma_launch_double_dmma_smem_fixed(a, grid, smem, st) : ffma_launch_double_dmma_gmem_fixed(a, grid, smem, st);
    if (integ) return bufs_smem ? ffma_launch_double_dmma_smem_integ(a, grid, smem, st) : ffma_launch_double_dmma_gmem_integ(a, grid, smem, st);
    return bufs_smem ? ffma_launch_double_dmma_smem(a, grid, smem, st) : ffma_launch_double_dmma_gmem(a, grid, smem, st);
  }
  if (func) {
    if (f64) return bufs_smem ? ffma_launch_double_smem_func(a, grid, smem, st) : ffma_launch_double_gmem_func(a, grid, smem, st);
    return bufs_smem ? ffma_launch_float_smem_func(a, grid, smem, st) : ffma_launch_float_gmem_func(a, grid, smem, st);
  }
  if (fixed) {
    if (f64) return bufs_smem ? ffma_launch_double_smem_fixed(a, grid, smem, st) : ffma_launch_double_gmem_fixed(a, grid, smem, st);
    return bufs_smem ? ffma_launch_float_smem_fixed(a, grid, smem, st) : ffma_launch_float_gmem_fixed(a, grid, smem, st);
  }
  if (integ) {
    if (f64) return bufs_smem ? ffma_launch_double_smem_integ(a, grid, smem, st) : ffma_launch_double_gmem_integ(a, grid, smem, st);
    return bufs_smem ? ffma_launch_float_smem_integ(a, grid, smem, st) : ffma_launch_float_gmem_integ(a, grid, smem, st);
  }
  if (f64) return bufs_smem ? ffma_launch_double_smem(a, grid, smem, st) : ffma_launch_double_gmem(a, grid, smem, st);
  return bufs_smem ? ffma_launch_float_smem(a, grid, smem, st) : ffma_launch_float_gmem(a, grid, smem, st);
}

cudaError_t finish_launch(int dtype, const void* packed, long long n_grad, int n_terms, const ScaleW& scale_w, void* out_grad,
                          void* out_terms, void* out_total, cudaStream_t st) {
  int blocks = (int)((n_grad + 255) / 256);
  if (blocks < 1) blocks = 1;
  if (dtype == PINN_F64)
    finish_kernel<double><<<blocks, 256, 0, st>>>((const double*)packed, n_grad, n_terms, scale_w, (double*)out_grad,
                                                   (double*)out_terms, (double*)out_total);
  else
    finish_kernel<float><<<blocks, 256, 0, st>>>((const float*)packed, n_grad, n_terms, scale_w, (float*)out_grad,
                                                  (float*)out_terms, (float*)out_total);
  return cudaGetLastError();
}

// max |g_i| and sum |g_i| of a gradient vector (one block; the vectors are at most a few MB)
template <typename real>
__global__ void __launch_bounds__(1024) grad_stats_kernel(const real* g, long long n, double* out) {
  __shared__ double smax[32], ssum[32];
  double mx = 0.0, sm = 0.0;
  for (long long i = threadIdx.x; i < n; i += 1024) {
    const double a = fabs((double)g[i]);
    mx = a > mx ? a : mx;
    sm += a;
  }
  for (int o = 16; o > 0; o >>= 1) {
    const double m2 = __shfl_xor_sync(0xffffffffu, mx, o);
    mx = m2 > mx ? m2 : mx;
    sm += __shfl_xor_sync(0xffffffffu, sm, o);
  }
  if ((threadIdx.x & 31) == 0) { smax[threadIdx.x >> 5] = mx; ssum[threadIdx.x >> 5] = sm; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double m = 0.0, t = 0.0;
    for (int w = 0; w < 32; ++w) { m = smax[w] > m ? smax[w] : m; t += ssum[w]; }     // fixed order: reproducible
    out[0] = m;
    out[1] = n > 0 ? t / (double)n : 0.0;
  }
}

// ---- device-side StochasticTraining sampler ---------------------------------------------------------------------------
// Philox4x32-10 (philox.cuh): counter = (point index, group of 4 rows, draw), key = seed.  One thread per point
// writes its `dim` coordinates lb_r + (ub_r - lb_r) * u, u uniform in [0, 1) from the high 24 (float) / 53 (double) bits.

struct SampleBox { double lb[PINN_MAX_DIM], ub[PINN_MAX_DIM]; };

template <typename real>
__global__ void __launch_bounds__(256) sample_uniform_kernel(real* pts, long long n, int dim, SampleBox box,
                                                              unsigned long long seed, unsigned long long draw,
                                                              const unsigned long long* draw_dev) {
  const long long p = (long long)blockIdx.x * 256 + threadIdx.x;
  if (p >= n) return;
  if (draw_dev) draw += *draw_dev;       // device-side counter advanced by the fused kernel's tail (graph replays)
  for (int r0 = 0; r0 < dim; r0 += (sizeof(real) == 8 ? 2 : 4)) {
    uint32_t c[4] = {(uint32_t)p, (uint32_t)(p >> 32), (uint32_t)r0 ^ ((uint32_t)draw << 8), (uint32_t)(draw >> 24)};
    philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
    if (sizeof(real) == 8) {
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int r = r0 + j;
        if (r < dim) {
          const unsigned long long bits = ((unsigned long long)c[2 * j] << 32) | c[2 * j + 1];
          const double u = (double)(bits >> 11) * (1.0 / 9007199254740992.0);
          pts[p * dim + r] = (real)(box.lb[r] + (box.ub[r] - box.lb[r]) * u);
        }
      }
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int r = r0 + j;
        if (r < dim) {
          const float u = (float)(c[j] >> 8) * (1.0f / 16777216.0f);
          pts[p * dim + r] = (real)(box.lb[r] + (box.ub[r] - box.lb[r]) * (double)u);
        }
      }
    }
  }
}

// ---- device-side Latin hypercube sampler (QuasiRandomTraining's default sampling_alg = LatinHypercubeSample()) -----------
// Row r of point i is lb_r + (ub_r - lb_r) * (pi_r(i) + u) / n with pi_r a keyed permutation of [0, n) and u uniform in
// [0, 1): each of the n strata of every row holds exactly one point per draw.  pi_r is a 4-round Feistel network over
// ceil(log2 n) bits (each round XORs one half with a hash of the other: a bijection) with cycle walking back into [0, n):
// stateless, O(1) per point, no sort and no shuffle buffer.
__device__ __forceinline__ uint32_t mix32(uint32_t x) {
  x ^= x >> 16; x *= 0x85EBCA6Bu; x ^= x >> 13; x *= 0xC2B2AE35u; x ^= x >> 16;
  return x;
}
__device__ __forceinline__ uint32_t feistel_perm(uint32_t i, uint32_t n, uint32_t bits, uint32_t k0, uint32_t k1) {
  const uint32_t hb = bits >> 1, ob = bits - hb;
  const uint32_t ma = (1u << hb) - 1u, mb = (1u << ob) - 1u;      // bits >= 2 here
  uint32_t x = i;
  do {
    uint32_t a = x & ma, b = x >> hb;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      a ^= mix32(b + k0 + 0x9E3779B9u * (uint32_t)(2 * r + 1)) & ma;
      b ^= mix32(a + k1 + 0x9E3779B9u * (uint32_t)(2 * r + 2)) & mb;
    }
    x = (b << hb) | a;
  } while (x >= n);
  return x;
}

template <typename real>
__global__ void __launch_bounds__(256) sample_lhs_kernel(real* pts, long long n, int dim, SampleBox box, unsigned long long seed,
                                                          unsigned long long draw, const unsigned long long* draw_dev) {
  const long long p = (long long)blockIdx.x * 256 + threadIdx.x;
  if (p >= n) return;
  if (draw_dev) draw += *draw_dev;
  uint32_t bits = 2;
  while ((1ull << bits) < (unsigned long long)n) ++bits;
  for (int r = 0; r < dim; ++r) {
    // per (row, draw) permutation key and per (point, row, draw) jitter from Philox
    uint32_t kc[4] = {(uint32_t)r, (uint32_t)draw, (uint32_t)(draw >> 32), 0x4C48535Fu};
    philox4x32_10(kc, (uint32_t)seed, (uint32_t)(seed >> 32));
    uint32_t c[4] = {(uint32_t)p, (uint32_t)(p >> 32), (uint32_t)r ^ ((uint32_t)draw << 8), (uint32_t)(draw >> 24) ^ 0x80000000u};
    philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
    const double u = (double)((((unsigned long long)c[0] << 32) | c[1]) >> 11) * (1.0 / 9007199254740992.0);
    double x;
    if (n == 1) {
      x = u;
    } else {
      const uint32_t j = feistel_perm((uint32_t)p, (uint32_t)n, bits, kc[0], kc[1]);
      x = ((double)j + u) / (double)n;
    }
    pts[p * dim + r] = (real)(box.lb[r] + (box.ub[r] - box.lb[r]) * x);
  }
}

cudaError_t sample_lhs_launch(int dtype, void* pts, long long n, int dim, const double* lb, const double* ub,
                              unsigned long long seed, unsigned long long draw, const unsigned long long* draw_dev,
                              cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  SampleBox box;
  for (int r = 0; r < PINN_MAX_DIM; ++r) { box.lb[r] = r < dim ? lb[r] : 0.0; box.ub[r] = r < dim ? ub[r] : 0.0; }
  const int blocks = (int)((n + 255) / 256);
  if (dtype == PINN_F64) sample_lhs_kernel<double><<<blocks, 256, 0, st>>>((double*)pts, n, dim, box, seed, draw, draw_dev);
  else sample_lhs_kernel<float><<<blocks, 256, 0, st>>>((float*)pts, n, dim, box, seed, draw, draw_dev);
  return cudaGetLastError();
}

cudaError_t sample_uniform_launch(int dtype, void* pts, long long n, int dim, const double* lb, const double* ub,
                                  unsigned long long seed, unsigned long long draw, const unsigned long long* draw_dev,
                                  cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  SampleBox box;
  for (int r = 0; r < PINN_MAX_DIM; ++r) { box.lb[r] = r < dim ? lb[r] : 0.0; box.ub[r] = r < dim ? ub[r] : 0.0; }
  const int blocks = (int)((n + 255) / 256);
  if (dtype == PINN_F64) sample_uniform_kernel<double><<<blocks, 256, 0, st>>>((double*)pts, n, dim, box, seed, draw, draw_dev);
  else sample_uniform_kernel<float><<<blocks, 256, 0, st>>>((float*)pts, n, dim, box, seed, draw, draw_dev);
  return cudaGetLastError();
}

// ---- device-side KKL path sampler (NNSDE's StochasticTraining; the formula is in include/pinn_b200.h) -------------------
__device__ __forceinline__ double u53(uint32_t a, uint32_t b) {
  return (double)((((unsigned long long)a << 32) | b) >> 11) * (1.0 / 9007199254740992.0);
}

template <typename real>
__global__ void __launch_bounds__(256) sample_kkl_kernel(real* pts, long long n, int sub, int n_z, double t_lb, double t_ub,
                                                         bool strong, unsigned long long seed, unsigned long long draw,
                                                         const unsigned long long* draw_dev) {
  const long long p = (long long)blockIdx.x * 256 + threadIdx.x;
  if (p >= n) return;
  if (draw_dev) draw += *draw_dev;
  const int dim = 1 + n_z;
  const uint32_t i = (uint32_t)(p / sub), s = (uint32_t)(p - (long long)i * sub);
  const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32), d0 = (uint32_t)draw, d1 = (uint32_t)(draw >> 32);
  uint32_t c[4] = {i, 0xFFFFFFFFu, d0, d1};
  philox4x32_10(c, k0, k1);
  pts[p * dim] = (real)(t_lb + (t_ub - t_lb) * u53(c[0], c[1]));
  const uint32_t q = strong ? s : (uint32_t)p;
  for (int j = 0; 2 * j < n_z; ++j) {
    uint32_t z[4] = {q, (uint32_t)j, d0, d1 ^ 0x4B4B4C00u};
    philox4x32_10(z, k0, k1);
    const double u1 = 1.0 - u53(z[0], z[1]), u2 = u53(z[2], z[3]);
    const double r = sqrt(-2.0 * log(u1));
    double sn, cs;
    sincos(6.283185307179586 * u2, &sn, &cs);
    pts[p * dim + 1 + 2 * j] = (real)(r * cs);
    if (2 + 2 * j <= n_z) pts[p * dim + 2 + 2 * j] = (real)(r * sn);
  }
}

cudaError_t sample_kkl_launch(int dtype, void* pts, long long n_times, int sub, int n_z, double t_lb, double t_ub,
                              bool strong, unsigned long long seed, unsigned long long draw,
                              const unsigned long long* draw_dev, cudaStream_t st) {
  const long long n = n_times * sub;
  if (n <= 0) return cudaSuccess;
  const int blocks = (int)((n + 255) / 256);
  if (dtype == PINN_F64)
    sample_kkl_kernel<double><<<blocks, 256, 0, st>>>((double*)pts, n, sub, n_z, t_lb, t_ub, strong, seed, draw, draw_dev);
  else
    sample_kkl_kernel<float><<<blocks, 256, 0, st>>>((float*)pts, n, sub, n_z, t_lb, t_ub, strong, seed, draw, draw_dev);
  return cudaGetLastError();
}

cudaError_t grad_stats_launch(int dtype, const void* grad, long long n, double* out2, cudaStream_t st) {
  if (dtype == PINN_F64) grad_stats_kernel<double><<<1, 1024, 0, st>>>((const double*)grad, n, out2);
  else grad_stats_kernel<float><<<1, 1024, 0, st>>>((const float*)grad, n, out2);
  return cudaGetLastError();
}

}  // namespace pinn
