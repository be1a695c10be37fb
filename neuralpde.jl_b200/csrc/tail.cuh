// tail.cuh -- the tail every fused loss+gradient kernel ends with: the gradient reduction, the optimizer step and the
// multi-GPU sum run INSIDE the fused kernel instead of in follow-up launches (reference: the Zygote gradient returned to
// Optimization.jl, src/discretize.jl:778, followed by Optimisers.Adam on the host; there is no multi-GPU counterpart).
//
//   1. grid barrier        all CTAs of the launch are co-resident (grid <= SM count, cooperative launch); a
//                          self-resetting generation barrier in global memory, so CUDA-graph replays need no host state
//   2. slice reduction     CTA b sums gradient entries [b*S, (b+1)*S) over the per-CTA partials in a FIXED order
//                          (bitwise reproducible for a given grid); CTA 0 turns the per-CTA term sums into losses
//   3. one-shot allreduce  (nranks > 1) every reduced entry is PUSHED into each peer's receive buffer over NVLink as one
//                          8-byte store {32 data bits, step flag} (the word and its flag arrive together: no fence, no
//                          separate flag, no read round trip); the CTA that owns the same slice on the peer polls its
//                          local slots until the flag carries this step, and adds the N values in rank order --
//                          one NVLink hop, no extra launch, identical bits on every rank
//   4. consume             write the gradient, or apply Adam in place (theta, m, v resident on the device; bias
//                          correction from a device-side step counter, so a captured graph can be replayed)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include "dev_types.h"

namespace pinn {

// launch `kernel` with the cooperative attribute when it ends with the grid-wide tail (a.tail.state set: all CTAs must be
// co-resident).  The dynamic shared-memory limit is raised once per kernel, device and size instead of on every launch
// (host time of the per-step call path): each kernel has its own instantiation and so its own cache.
template <auto kernel, typename A>
static cudaError_t launch_fused_kernel(const A& a, int grid, int threads, size_t smem, cudaStream_t st) {
  static size_t granted[64] = {0};   // bytes already granted on device d
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= 64 || granted[dev] < smem) {
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < 64) granted[dev] = smem;
  }
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof cfg);
  cfg.gridDim = dim3((unsigned)grid); cfg.blockDim = dim3((unsigned)threads); cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeCooperative;
  at[0].val.cooperative = a.tail.state != nullptr ? 1 : 0;
  cfg.attrs = at; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, a);
}

__device__ __forceinline__ unsigned int ld_acquire_gpu(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// one receive slot = {32 data bits, step flag}: a single aligned 8-byte access, so the word never arrives without its flag
__device__ __forceinline__ void st_slot(uint2* p, unsigned int bits, unsigned int flag) {
  asm volatile("st.relaxed.sys.global.v2.u32 [%0], {%1, %2};" ::"l"(p), "r"(bits), "r"(flag) : "memory");
}
__device__ __forceinline__ uint2 ld_slot(const uint2* p) {
  uint2 v;
  asm volatile("ld.relaxed.sys.global.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned int atom_add_acq_rel_gpu(unsigned int* p, unsigned int v) {
  unsigned int old;
  asm volatile("atom.add.acq_rel.gpu.global.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
  return old;
}
__device__ __forceinline__ void red_add_release_gpu(unsigned int* p, unsigned int v) {
  asm volatile("red.add.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long tail_now_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

// spin until pred() holds; a protocol failure (lost peer, CTAs not co-resident) traps after timeout_ns instead of hanging
template <typename Pred>
__device__ __forceinline__ void tail_spin(Pred pred, unsigned long long timeout_ns) {
  unsigned long long t0 = 0;
  for (unsigned int it = 0;; ++it) {
    if (pred()) return;
    if ((it & 1023u) == 1023u) {
      const unsigned long long t = tail_now_ns();
      if (t0 == 0) t0 = t;
      else if (t - t0 > timeout_ns) __trap();
    }
  }
}

template <typename real> struct Vec16;
template <> struct Vec16<float> { typedef float4 type; };
template <> struct Vec16<double> { typedef double2 type; };

// NT = threads per CTA.  red: NT * (16 / sizeof(real)) scalars of 16-byte aligned shared memory.  partial:
// [gridDim.x][stride] (stride a multiple of 4 scalars); term_sums: [gridDim.x][PINN_MAX_TERMS] (this CTA's row already
// written).  Must be called by every thread of every CTA of the launch.
// FUNC: the problem has a functional term f (PINN_REDUCE_*_OF_SUM; st->func_term): its loss is L_f = g(scale_f S_f),
// S_f = sum_b term_sums[b][f], and the functional's own partials G [gridDim.x][stride] follow `partial`.  Every slice
// CTA forms S_f in the term CTA's order, kappa = w_f g'(scale_f S_f) scale_f, and reduces sum_b partial + kappa sum_b G
// (both in the fixed order): the chain rule of g(S) needs S before any point's contribution can be scaled.
template <typename real, int NT, bool FUNC = false>
__device__ __noinline__ void fused_tail(const TailArgs& ta, const real* partial, long long stride, const double* term_sums,
                                        long long n_theta, int n_terms, int want_grad, real* red) {
  constexpr int V = 16 / (int)sizeof(real);   // scalars per 16-byte load: the reduction is bound by bytes in flight
  constexpr int EW = 32 * V;                  // gradient entries per pass (one warp of 16-byte vectors)
  constexpr int NG = NT / 32;                 // partial-row groups summed concurrently (one warp each)
  typedef typename Vec16<real>::type vec_t;
  __shared__ unsigned int s_step;
  __shared__ unsigned long long s_t;
  TailState* st = ta.state;
  const int tid = threadIdx.x, nb = gridDim.x, bid = blockIdx.x;

#ifdef PINN_DEBUG
#define TAIL_MARK(k) do { if (ta.dbg && tid == 0) ta.dbg[(size_t)bid * 4 + (k)] = (long long)tail_now_ns(); } while (0)
#else
#define TAIL_MARK(k) do { } while (0)
#endif
  // ---- 1. grid barrier ----------------------------------------------------------------------------------------------
  __syncthreads();
  TAIL_MARK(0);
  if (tid == 0) {
    const unsigned int step = *reinterpret_cast<volatile unsigned int*>(&st->step);
    const unsigned long long t_adam = *reinterpret_cast<volatile unsigned long long*>(&st->adam_t) + 1ull;
    const unsigned int gen = *reinterpret_cast<volatile unsigned int*>(&st->gen);
    s_step = step;
    s_t = t_adam;
    // arrive with acq_rel (orders this CTA's partials, made visible to this thread by the barrier above, before the
    // count; the last arriver acquires everyone's), release the generation: no separate fences on the critical path
    if (atom_add_acq_rel_gpu(&st->count, 1u) == (unsigned int)(nb - 1)) {
      st->count = 0u;
      st->step = step + 1u;
      if (ta.adam_theta && want_grad) st->adam_t = t_adam;
      if (ta.bump_draw) st->draw = st->draw + 1ull;
      red_add_release_gpu(&st->gen, 1u);
    } else {
      tail_spin([&] { return ld_acquire_gpu(&st->gen) != gen; }, ta.timeout_ns);
    }
  }
  __syncthreads();
  TAIL_MARK(1);
  const unsigned int step1 = s_step + 1u;          // flag value of this step (0 = never written)
  const bool multi = ta.nranks > 1;
  constexpr int W = (int)sizeof(real) / 4;         // 32-bit words per scalar
  // receive slots of (parity, source rank) on rank q: recv[q] + ((parity * nranks + src) * recv_words + word), 8 bytes each
  const size_t par_off = (size_t)(s_step & 1u) * (size_t)ta.nranks;
  auto push = [&](long long word, unsigned int bits) {          // this rank's word -> the same slot on every rank (self included)
#pragma unroll
    for (int q = 0; q < kMaxRanks; ++q)
      if (q < ta.nranks)
        st_slot(reinterpret_cast<uint2*>(ta.peer_recv[q]) + (par_off + (size_t)ta.rank) * (size_t)ta.recv_words + word, bits, step1);
  };
  auto pull = [&](int src, long long word) -> unsigned int {    // poll the local slot until the source's word of THIS step is there
    const uint2* slot = reinterpret_cast<const uint2*>(ta.peer_recv[ta.rank]) + (par_off + (size_t)src) * (size_t)ta.recv_words + word;
    uint2 v = ld_slot(slot);
    if (v.y != step1) tail_spin([&] { v = ld_slot(slot); return v.y == step1; }, ta.timeout_ns);
    return v.x;
  };

  // ---- 2. term losses (one warp per term): L_k = scale_k * sum_b term_sums[b][k], fixed order.  The LAST CTA does this and
  // takes no gradient slice (when there is more than one CTA), so the term path runs beside the slice path, not in front of it
  const int term_cta = nb - 1;
  const int nbs = nb > 1 ? nb - 1 : 1;              // CTAs that own gradient slices
  if (bid == term_cta) {
    double* sL = reinterpret_cast<double*>(red);          // n_terms doubles (<= 32 * 8 bytes: fits NT scalars)
    const int warp = tid >> 5, lane = tid & 31;
    for (int k = warp; k < n_terms; k += NT / 32) {
      double v[(kTailSlots + 31) / 32];
#pragma unroll
      for (int j = 0; j < (kTailSlots + 31) / 32; ++j) {
        const int b = lane + 32 * j;
        v[j] = (b < nb) ? __ldcg(&term_sums[(long long)b * PINN_MAX_TERMS + k]) : 0.0;
      }
      double s = 0.0;
#pragma unroll
      for (int j = 0; j < (kTailSlots + 31) / 32; ++j) s += v[j];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) {
        sL[k] = s * ta.sw.scale[k];
        if constexpr (FUNC)
          if (k == st->func_term) sL[k] = st->func_square ? sL[k] * sL[k] : fabs(sL[k]);
      }
    }
    __syncthreads();
    if (tid == 0) {
      double tot = 0.0;
      for (int k = 0; k < n_terms; ++k) {
        const double Lk = sL[k];
        tot += Lk * ta.sw.w[k];
        if (multi) {                                   // term losses travel as two words each behind the gradient
          const unsigned long long bits = (unsigned long long)__double_as_longlong(Lk);
          push(n_theta * W + 2 * k, (unsigned int)bits);
          push(n_theta * W + 2 * k + 1, (unsigned int)(bits >> 32));
        } else {
          reinterpret_cast<real*>(ta.out_terms)[k] = real(Lk);
        }
      }
      if (!multi && ta.out_total) *reinterpret_cast<real*>(ta.out_total) = real(tot);
    }
    __syncthreads();
  }

  // Adam coefficients (device-side step counter: graph replays advance it)
  double lr_t = 0.0, eps_t = 0.0;
  const bool adam = ta.adam_theta != nullptr && want_grad;
  if (adam) {
    const double t = (double)s_t;
    const double c1 = 1.0 - pow(ta.adam_b1, t), c2 = sqrt(1.0 - pow(ta.adam_b2, t));
    lr_t = ta.adam_lr * c2 / c1;                    // lr * sqrt(1 - beta2^t) / (1 - beta1^t)
    eps_t = ta.adam_eps * c2;
  }
  auto consume = [&](long long i, real g) {
    if (adam) {
      real* th = reinterpret_cast<real*>(ta.adam_theta);
      real* m = reinterpret_cast<real*>(ta.adam_m);
      real* v = reinterpret_cast<real*>(ta.adam_v);
      const double gd = (double)g;
      const double mi = ta.adam_b1 * (double)m[i] + (1.0 - ta.adam_b1) * gd;
      const double vi = ta.adam_b2 * (double)v[i] + (1.0 - ta.adam_b2) * gd * gd;
      m[i] = real(mi); v[i] = real(vi);
      th[i] = real((double)th[i] - lr_t * mi / (sqrt(vi) + eps_t));
      if (ta.out_grad) reinterpret_cast<real*>(ta.out_grad)[i] = g;
    } else {
      reinterpret_cast<real*>(ta.out_grad)[i] = g;
    }
  };

  // ---- 3. slice reduction over the per-CTA partials ----------------------------------------------------------------------
  // warp g adds rows g, g + NG, ... of a 32-vector-wide window (16-byte L2 loads, all in flight at once), the NG row
  // groups are then combined through shared memory in group order: a fixed summation order for a given grid
  long long S = (n_theta + nbs - 1) / nbs;
  S = (S + V - 1) / V * V;
  const bool slice_cta = bid < nbs;
  const long long i0 = slice_cta ? (long long)bid * S : n_theta;
  const long long i1 = (i0 + S < n_theta) ? i0 + S : n_theta;
  const int lane = tid & 31, g = tid >> 5;
  real kappa = real(0);                            // FUNC: d total / d S_f
  if constexpr (FUNC) {
    __shared__ double s_kappa;
    if (want_grad && tid < 32) {                   // S_f exactly as the term CTA sums it
      const int f = st->func_term;
      double v[(kTailSlots + 31) / 32];
#pragma unroll
      for (int j = 0; j < (kTailSlots + 31) / 32; ++j) {
        const int b = lane + 32 * j;
        v[j] = (b < nb) ? __ldcg(&term_sums[(long long)b * PINN_MAX_TERMS + f]) : 0.0;
      }
      double s = 0.0;
#pragma unroll
      for (int j = 0; j < (kTailSlots + 31) / 32; ++j) s += v[j];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) {
        const double x = s * ta.sw.scale[f];
        const double dg = st->func_square ? 2.0 * x : (x > 0.0 ? 1.0 : (x < 0.0 ? -1.0 : 0.0));   // sign(0) = 0
        s_kappa = ta.sw.w[f] * dg * ta.sw.scale[f];
      }
    }
    __syncthreads();
    kappa = real(s_kappa);
  }
  if (want_grad) {
    for (long long base = i0; base < i1; base += EW) {
      const long long i = base + (long long)V * lane;
      real tf = real(0);                           // FUNC: kappa * sum_b G[b][i], reduced like the partials below
      if constexpr (FUNC) {
        real acc[V];
#pragma unroll
        for (int j = 0; j < V; ++j) acc[j] = real(0);
        if (i < i1) {
          const real* col = partial + (long long)nb * stride + i;
#pragma unroll 8
          for (int b = g; b < nb; b += NG) {
            const vec_t v = __ldcg(reinterpret_cast<const vec_t*>(col + (long long)b * stride));
            const real* pv = reinterpret_cast<const real*>(&v);
#pragma unroll
            for (int j = 0; j < V; ++j) acc[j] += pv[j];
          }
        }
        *reinterpret_cast<vec_t*>(red + (size_t)(g * 32 + lane) * V) = *reinterpret_cast<vec_t*>(acc);
        __syncthreads();
        if (tid < EW && base + tid < i1) {
          tf = red[tid];
#pragma unroll
          for (int k = 1; k < NG; ++k) tf += red[k * EW + tid];
          tf *= kappa;
        }
        __syncthreads();
      }
      real acc[V];
#pragma unroll
      for (int j = 0; j < V; ++j) acc[j] = real(0);
      if (i < i1) {
        const real* col = partial + i;
#pragma unroll 8
        for (int b = g; b < nb; b += NG) {
          const vec_t v = __ldcg(reinterpret_cast<const vec_t*>(col + (long long)b * stride));
          const real* pv = reinterpret_cast<const real*>(&v);
#pragma unroll
          for (int j = 0; j < V; ++j) acc[j] += pv[j];
        }
      }
      *reinterpret_cast<vec_t*>(red + (size_t)(g * 32 + lane) * V) = *reinterpret_cast<vec_t*>(acc);
      __syncthreads();
      if (tid < EW && base + tid < i1) {
        real t = red[tid];
#pragma unroll
        for (int k = 1; k < NG; ++k) t += red[k * EW + tid];
        if constexpr (FUNC) t += tf;
        if (multi) {
          if (W == 1) {
            push(base + tid, (unsigned int)__float_as_uint((float)t));
          } else {
            const unsigned long long bits = (unsigned long long)__double_as_longlong((double)t);
            push(2 * (base + tid), (unsigned int)bits);
            push(2 * (base + tid) + 1, (unsigned int)(bits >> 32));
          }
        } else {
          consume(base + tid, t);
        }
      }
      __syncthreads();
    }
  }
  TAIL_MARK(2);
  if (!multi) return;

  // ---- 4. receive: the same slice of every rank (own included), added in rank order -----------------------------------------
  // every poll is an L2 round trip: the slots of all ranks are read TOGETHER first, only the ones whose flag is not there
  // yet are polled again (reading them one after the other cost ~0.5 us per rank and word on the critical path)
  auto slot_of = [&](int src, long long word) {
    return reinterpret_cast<const uint2*>(ta.peer_recv[ta.rank]) + (par_off + (size_t)src) * (size_t)ta.recv_words + word;
  };
  if (want_grad) {
    for (long long i = i0 + tid; i < i1; i += NT) {
      uint2 v[kMaxRanks][W];
#pragma unroll
      for (int r = 0; r < kMaxRanks; ++r)
        if (r < ta.nranks) {
#pragma unroll
          for (int w = 0; w < W; ++w) v[r][w] = ld_slot(slot_of(r, W * i + w));
        }
      real t = real(0);
#pragma unroll
      for (int r = 0; r < kMaxRanks; ++r)
        if (r < ta.nranks) {
#pragma unroll
          for (int w = 0; w < W; ++w)
            if (v[r][w].y != step1) v[r][w].x = pull(r, W * i + w);
          if (W == 1) t += (real)__uint_as_float(v[r][0].x);
          else t += (real)__longlong_as_double((long long)((unsigned long long)v[r][0].x | ((unsigned long long)v[r][W - 1].x << 32)));
        }
      consume(i, t);
    }
  }
  if (bid == term_cta) {
    // term losses: one thread per (term, rank, word), then thread 0 adds them in rank order
    unsigned int* sw = reinterpret_cast<unsigned int*>(red);           // n_terms * nranks * 2 words <= 512 <= NT * V
    const int n_words = n_terms * ta.nranks * 2;
    __syncthreads();
    for (int j = tid; j < n_words; j += NT) {
      const int k = j / (ta.nranks * 2), r = (j / 2) % ta.nranks, w = j & 1;
      sw[j] = pull(r, n_theta * W + 2 * k + w);
    }
    __syncthreads();
    if (tid == 0) {
      double tot = 0.0;
      for (int k = 0; k < n_terms; ++k) {
        double Lk = 0.0;
        for (int r = 0; r < ta.nranks; ++r) {
          const unsigned long long lo = sw[(k * ta.nranks + r) * 2], hi = sw[(k * ta.nranks + r) * 2 + 1];
          Lk += __longlong_as_double((long long)(lo | (hi << 32)));
        }
        reinterpret_cast<real*>(ta.out_terms)[k] = real(Lk);
        tot += Lk * ta.sw.w[k];
      }
      if (ta.out_total) *reinterpret_cast<real*>(ta.out_total) = real(tot);
    }
  }
  __syncthreads();
  TAIL_MARK(3);
}

}  // namespace pinn
