// reduce.cuh -- the fixed-order block reduction of the float64 drivers (qn.cu, hmc.cu).  Warp shuffles in a fixed
// pattern, then thread 0 adds the warps in order: the result depends on the block size only, so runs are bit-identical.
#pragma once

namespace pinn {

__device__ __forceinline__ double nan_max(double a, double b) { return (isnan(a) || a >= b) ? a : b; }

// sum (or NaN-propagating max) over the block; the result is valid in thread 0.  Callers that reduce twice in one
// kernel separate the calls with __syncthreads(): the warp partials live in one shared array.
template <int kThreads, bool kMax>
__device__ double block_reduce(double v) {
  __shared__ double warp_part[kThreads / 32];
  for (int o = 16; o; o >>= 1) {
    const double u = __shfl_xor_sync(0xffffffffu, v, o);
    v = kMax ? nan_max(v, u) : v + u;
  }
  if ((threadIdx.x & 31) == 0) warp_part[threadIdx.x >> 5] = v;
  __syncthreads();
  double r = warp_part[0];
  if (threadIdx.x == 0)
    for (int w = 1; w < kThreads / 32; ++w) r = kMax ? nan_max(r, warp_part[w]) : r + warp_part[w];
  return r;
}

}  // namespace pinn
