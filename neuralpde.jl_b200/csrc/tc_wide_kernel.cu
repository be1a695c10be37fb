// tc_wide_kernel.cu -- fused PINN loss+gradient kernel, tensor-core path for 128-wide layers (sm_90a wgmma, bf16 operands).
//
// Same decomposition as tc_kernel.cu (one CTA of 512 threads per 128-point tile, a point is a row of the accumulator
// region and of every operand tile, derivative channels share the weight operand), re-planned for hidden widths 64 / 128 where
// neither the weights of all layers nor two generations of activations fit in shared memory:
//
//   * an activation set is C channels x 2 tiles (128 points x 64 bf16, 128-byte swizzle) = C x 32 KB in region P;
//     the accumulator region holds C x 128 columns (C <= 4), so the epilogue of a layer overwrites its own input in place;
//   * weights are packed once per step by tw_pack_kernel into bf16 swizzled images (32 KB per layer) and streamed
//     through two 32 KB buffers S0 / S1 with cp.async.bulk + mbarrier, prefetched one layer ahead;
//   * the forward sweep stashes every tensor layer's input tiles (bf16, for wgrad) and biased pre-activations
//     (fp32, point-fastest so that a warp writes / reads 256 contiguous bytes) to a per-CTA global buffer (L2);
//     the reverse sweep reads the pre-activations straight into registers -- no recompute, no accumulator columns for it;
//   * reverse, per tensor layer:  Zbar tiles -> P;  wgrad  Wbar_l = sum_c Zbar_c^T H_c  with H_c streamed through
//     S0 / S1 per channel;  then dgrad  Hbar_c = Zbar_c W_l  with W_l in the buffer wgrad released first.
//     MN-major operands whose M / N extent is 128 span two tiles through the descriptor's leading-dimension byte
//     offset.
//
// Replaces the same reference functions as the other paths (Phi src/pinn_types.jl:79-90, numeric_derivative
// :445-482, the generated residual and mean(abs2) src/training_strategies.jl:215-221, Zygote gradient
// src/discretize.jl:778).
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include "tc_common.cuh"

namespace pinn {

constexpr uint32_t TB = kTileBytes;
using Fp = FpBlock<kTwW>;   // fp32 parameter block of a network

struct TwShared : CtaBase {
  int off_S, off_nets;
  uint8_t* hstash;
  float* zstash;
  const uint8_t* wpack;
  int off_fp[PINN_MAX_NETS], wimg[PINN_MAX_NETS];
  int next_tile;                     // dynamic scheduler: tile claimed for the next iteration
  uint32_t ph_ld[2];                 // phases of the streaming barriers (flipped by thread 0 after a CTA-wide wait)
  uint64_t bar_ld[2];                // S0 / S1: bytes landed
};

struct LoopW {
  uint32_t fp;            // shared-memory address of the network's fp32 parameter block
  uint32_t bt;            // shared-memory address of the current tensor layer's bias
  uint32_t tP;            // shared-memory address of the operand tiles (channel c, column block kb: (c*2+kb)*TB)
  uint32_t taddr;         // accumulator address of the warp's row quadrant
  int act, p, g0, g1, flag;
  // ng granules of the layer, spread over the kNH warps of the thread's row quadrant
  __device__ __forceinline__ LoopW(uint32_t fp_, uint32_t bt_, uint32_t tP_, const Tid& t, int act_, int ng, int flag_)
      : fp(fp_), bt(bt_), tP(tP_), taddr(t.lane_addr), act(act_), p(t.p), g0(t.hh * (ng / kNH)), g1((t.hh + 1) * (ng / kNH)),
        flag(flag_) {}
};

__device__ __forceinline__ uint32_t tile_of(uint32_t tP, int c, int col) { return tP + (uint32_t)(c * 2 + (col >> 6)) * TB; }

// layer 0 forward: coordinates -> H^0 tiles
template <int N1, int N2, bool PURE, int AK>
__device__ __forceinline__ void tw_l0_fwd_loop(const LoopW lc, const PassInfo<N1, N2> pi, const float* xp) {
  constexpr int C = 1 + N1 + N2;
  float x[PINN_MAX_IN];
#pragma unroll
  for (int k = 0; k < PINN_MAX_IN; ++k) x[k] = xp[k];
#pragma unroll 1
  for (int g = lc.g0; g < lc.g1; ++g) {
    float h[C][4];
#pragma unroll
    for (int i = 0; i < 4; i += 2) {
      float za[C], zb2[C];
      first_layer_elem<kTwW>(lc.fp, pi, x, g * 4 + i, za);
      first_layer_elem<kTwW>(lc.fp, pi, x, g * 4 + i + 1, zb2);
      P2 zz[C], hv[C];
#pragma unroll
      for (int c = 0; c < C; ++c) zz[c] = mk2(za[c], zb2[c]);
      chain_fwd<N1, N2, PURE, AK, P2>(lc.act, pi.ch, zz, hv);
#pragma unroll
      for (int c = 0; c < C; ++c) { h[c][i] = hv[c].v.x; h[c][i + 1] = hv[c].v.y; }
    }
    const int col = g * 4;
#pragma unroll
    for (int c = 0; c < C; ++c) store_half(tile_of(lc.tP, c, col), 0u, lc.p, col & 63, h[c], false);
  }
}

// tensor layer forward epilogue: accumulators -> bias + activation chain -> next operand tiles (in place),
// biased pre-activations -> fp32 stash (zst != nullptr), last-layer dot products (flag)
template <int N1, int N2, bool PURE, int AK>
__device__ __forceinline__ void tw_fwd_loop(const LoopW lc, const Chan<N1, N2> ch, float* up, float2* zst) {
  constexpr int C = 1 + N1 + N2;
  float u[C];
#pragma unroll
  for (int c = 0; c < C; ++c) u[c] = up[c];
#pragma unroll 1
  for (int g = lc.g0; g < lc.g1; ++g) {
    float z[C][4];
#pragma unroll
    for (int c = 0; c < C; ++c) acc_ld4(lc.taddr + c * kTwW + g * 4, z[c]);
    const int col = g * 4;
#pragma unroll
    for (int i = 0; i < 4; i += 2) {
      P2 zz[C], hv[C];
      zz[0] = mk2(z[0][i] + lds_f32(lc.bt + (col + i) * 4), z[0][i + 1] + lds_f32(lc.bt + (col + i + 1) * 4));
#pragma unroll
      for (int c = 1; c < C; ++c) zz[c] = mk2(z[c][i], z[c][i + 1]);
      if (zst) {
#pragma unroll
        for (int c = 0; c < C; ++c) zst[(c * 64 + ((col + i) >> 1)) * kTcPts] = zz[c].v;
      }
      chain_fwd<N1, N2, PURE, AK, P2>(lc.act, ch, zz, hv);
#pragma unroll
      for (int c = 0; c < C; ++c) { z[c][i] = hv[c].v.x; z[c][i + 1] = hv[c].v.y; }
      if (lc.flag) {
        const float w0 = lds_f32(lc.fp + (Fp::WL + col + i) * 4), w1 = lds_f32(lc.fp + (Fp::WL + col + i + 1) * 4);
#pragma unroll
        for (int c = 0; c < C; ++c) u[c] = fmaf(w1, hv[c].v.y, fmaf(w0, hv[c].v.x, u[c]));
      }
    }
#pragma unroll
    for (int c = 0; c < C; ++c) store_half(tile_of(lc.tP, c, col), 0u, lc.p, col & 63, z[c], false);
  }
#pragma unroll
  for (int c = 0; c < C; ++c) up[c] = u[c];
}

// tensor layer reverse epilogue: stashed pre-activations and output adjoints (columns X, or w_last * ubar for the last
// hidden layer: flag) -> Zbar tiles in P (the bias gradient is a column sum of Zbar_0, taken by an MMA chain against
// the ones atom).  The stash is read from HBM more often than from L2 (132 CTAs x 1.5 MB in flight > the 50 MB L2); the
// next granule's loads are in flight while the current one is processed.
template <int N1, int N2, bool PURE, int AK>
__device__ __forceinline__ void tw_bwd_loop(const LoopW lc, const Chan<N1, N2> ch, const float* ubp, const float2* zst) {
  constexpr int C = 1 + N1 + N2;
  float ub[C];
#pragma unroll
  for (int c = 0; c < C; ++c) ub[c] = ubp[c];
  float2 za[C][2], zb[C][2];
  auto load = [&](float2 (&zz)[C][2], int g) {
#pragma unroll
    for (int c = 0; c < C; ++c) {
      zz[c][0] = zst[(c * 64 + 2 * g) * kTcPts];
      zz[c][1] = zst[(c * 64 + 2 * g + 1) * kTcPts];
    }
  };
  auto process = [&](const float2 (&zc)[C][2], int g) {
    const int ocol = g * 4;
    float hb[C][4];
    if (!lc.flag) {
#pragma unroll
      for (int c = 0; c < C; ++c) acc_ld4(lc.taddr + c * kTwW + ocol, hb[c]);
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float wl = lds_f32(lc.fp + (Fp::WL + ocol + i) * 4);
#pragma unroll
        for (int c = 0; c < C; ++c) hb[c][i] = wl * ub[c];
      }
    }
#pragma unroll
    for (int i = 0; i < 4; i += 2) {
      P2 zz[C], hv[C], zv[C];
#pragma unroll
      for (int c = 0; c < C; ++c) { zz[c].v = zc[c][i >> 1]; hv[c] = mk2(hb[c][i], hb[c][i + 1]); }
      chain_bwd<N1, N2, PURE, AK, P2>(lc.act, ch, zz, hv, zv);
#pragma unroll
      for (int c = 0; c < C; ++c) { hb[c][i] = zv[c].v.x; hb[c][i + 1] = zv[c].v.y; }
    }
#pragma unroll
    for (int c = 0; c < C; ++c) store_half(tile_of(lc.tP, c, ocol), 0u, lc.p, ocol & 63, hb[c], false);
  };
  load(zb, lc.g0);
#pragma unroll 1
  for (int g = lc.g0; g < lc.g1; ++g) {
#pragma unroll
    for (int c = 0; c < C; ++c) { za[c][0] = zb[c][0]; za[c][1] = zb[c][1]; }
    if (g + 1 < lc.g1) load(zb, g + 1);
    process(za, g);
  }
}

// layer 0 reverse: adjoints of H^0 (columns X) -> Zbar^0 tiles of the value + first-derivative channels in P
template <int N1, int N2, bool PURE, int AK>
__device__ __forceinline__ void tw_l0_bwd_store_loop(const LoopW lc, const PassInfo<N1, N2> pi, const float* xp) {
  constexpr int C = 1 + N1 + N2;
  float x[PINN_MAX_IN];
#pragma unroll
  for (int k = 0; k < PINN_MAX_IN; ++k) x[k] = xp[k];
#pragma unroll 1
  for (int g = lc.g0; g < lc.g1; ++g) {
    const int col = g * 2;
    float hb[C][2];
#pragma unroll
    for (int c = 0; c < C; ++c) acc_ld2(lc.taddr + c * kTwW + col, hb[c]);
    float za[C], zb2[C];
    first_layer_elem<kTwW>(lc.fp, pi, x, col, za);
    first_layer_elem<kTwW>(lc.fp, pi, x, col + 1, zb2);
    P2 zz[C], hv[C], zv[C];
#pragma unroll
    for (int c = 0; c < C; ++c) { zz[c] = mk2(za[c], zb2[c]); hv[c] = mk2(hb[c][0], hb[c][1]); }
    chain_bwd<N1, N2, PURE, AK, P2>(lc.act, pi.ch, zz, hv, zv);
#pragma unroll
    for (int c = 0; c <= N1; ++c) {
      const float o2[2] = {zv[c].v.x, zv[c].v.y};
      store_half(tile_of(lc.tP, c, col), 0u, lc.p, col & 63, o2, false);
    }
  }
}

// ---- streaming helpers: thread 0 issues the bulk loads, every thread waits for them -----------------------------------
__device__ __forceinline__ void tw_load(TwShared* cs, int b, uint32_t dst, const uint8_t* src, int n_tiles) {
  tc::mbar_arrive_expect_tx(&cs->bar_ld[b], (uint32_t)n_tiles * TB);
  for (int i = 0; i < n_tiles; ++i)
    tc::bulk_load_u(dst + (uint32_t)i * TB, src + (size_t)i * TB, TB, tc::smem_u32(&cs->bar_ld[b]));
}
// CTA-wide: the next read of cs->ph_ld[b] must follow another __syncthreads
__device__ __forceinline__ void tw_wait_ld(TwShared* cs, int b) {
  const uint32_t ph = cs->ph_ld[b];
  tc::mbar_wait(&cs->bar_ld[b], ph);
  __syncthreads();
  if (threadIdx.x == 0) cs->ph_ld[b] = ph ^ 1u;
}

// ---------------------------------------------------------------------------------------------------------------------
// forward of one network for the current tile
template <int N1, int N2, bool PURE, int AK>
__device__ __noinline__ void tw_net_forward(TwShared* cs, const DevProblem* Pp, const DevTerm* tmp, int slot, int want_grad) {
  extern __shared__ __align__(1024) uint8_t smem[];
  constexpr int C = 1 + N1 + N2;
  const DevTerm& tm = *tmp;
  const int net_id = tm.used_net[slot];
  const DevNet& net = reinterpret_cast<const DevNet*>(smem + cs->off_nets)[net_id];
  const DevChan& dc = tm.chan[slot];
  const float* fp = reinterpret_cast<const float*>(smem + cs->off_fp[net_id]);
  uint8_t* tP = smem + cs->off_P;
  uint8_t* tS = smem + cs->off_S;
  const Misc ms = misc_of(smem + cs->off_misc, cs->mx_dim, cs->mx_taps);
  const uint32_t accm = 0;   // accumulator address of row 0, column 0
  PassInfo<N1, N2> pi;
  load_pass<N1, N2>(pi, net, dc);
  const int TL = pi.TL;
  const Tid t = tid_of();
  const int tid = t.tid, p = t.p;
  float x[PINN_MAX_IN];
#pragma unroll
  for (int k = 0; k < PINN_MAX_IN; ++k) x[k] = (k < pi.d_in) ? ms.Xs[dc.rows[k] * kTcPts + p] : 0.f;
  uint8_t* hst = cs->hstash + (size_t)slot * (cs->tl_max + 1) * kTwMaxC * 2 * TB;
  float* zst = cs->zstash + (size_t)slot * cs->tl_max * kTwMaxC * 64 * kTcPts * 2;
  const uint8_t* wimg = cs->wpack + (size_t)cs->wimg[net_id] * kTwImgBytes;

  dbg_mark(cs, 10);
  float u[C];
#pragma unroll
  for (int c = 0; c < C; ++c) u[c] = 0.f;
  if (tid < C * kTcPts / 4) reinterpret_cast<float4*>(ms.scratch)[tid] = make_float4(0.f, 0.f, 0.f, 0.f);
  // first tensor layer's weights stream in behind the layer-0 epilogue (buffer S[1])
  if (tid == 0) {
    tc::fence_async_smem();
    tw_load(cs, 1, tc::smem_u32(tS) + kTwImgBytes, wimg, (net.dims[1] + 63) >> 6);
  }
  const uint32_t sfp = tc::smem_u32(fp);
  tw_l0_fwd_loop<N1, N2, PURE, AK>(LoopW(sfp, sfp, tc::smem_u32(tP), t, net.acts[0], pi.n1w / 4, 0), pi, x);
  for (int l = 1; l <= TL; ++l) {
    const int n_in = net.dims[l], n_out = net.dims[l + 1];
    tc::fence_async_smem();
    __syncthreads();
    dbg_mark(cs, 11);
    const uint32_t sP = tc::smem_u32(tP), sS = tc::smem_u32(tS);
    const int nb_in = (n_in + 63) >> 6;
    if (tid == 0) {
      if (want_grad) {
        uint8_t* h = hst + (size_t)(l - 1) * kTwMaxC * 2 * TB;
        for (int c = 0; c < C; ++c)
          for (int kb = 0; kb < nb_in; ++kb) tc::bulk_store(h + (size_t)(c * 2 + kb) * TB, tP + (c * 2 + kb) * TB, TB);
        tc::bulk_commit();
      }
      if (l < TL)     // next layer's weights -> the other buffer (its last readers, layer l-1's MMAs, have retired)
        tw_load(cs, (l + 1) & 1, sS + ((l + 1) & 1) * kTwImgBytes, wimg + (size_t)l * kTwImgBytes, (net.dims[l + 1] + 63) >> 6);
    }
    tw_wait_ld(cs, l & 1);
    {
      const uint32_t idesc = tc::make_idesc(n_out, 0, 0);
      const uint32_t wbuf = sS + (l & 1) * kTwImgBytes;
#pragma unroll 1
      for (int c = 0; c < C; ++c) {
#pragma unroll 1
        for (int kb = 0; kb < nb_in; ++kb) {
          const int nk = ((n_in - kb * 64) < 64 ? (n_in - kb * 64) : 64) >> 4;
          mma_chain(accm + c * kTwW, tc::make_desc(sP + (c * 2 + kb) * TB, 0, 1024), tc::make_desc(wbuf + kb * TB, 0, 1024), 32, 32,
                    nk, idesc, kb > 0 ? 1u : 0u);
        }
      }
    }
    dbg_mark(cs, 12);
    __syncthreads();
    dbg_mark(cs, 13);
    if (want_grad && tid == 0) tc::bulk_wait_read0();   // stash copies have finished reading P
    __syncthreads();
    dbg_mark(cs, 14);
    const LoopW lc(sfp, sfp + (Fp::BT + (l - 1) * 128) * 4, sP, t, net.acts[l], n_out / 4, l == TL);
    float2* zl = want_grad ? reinterpret_cast<float2*>(zst + (size_t)(l - 1) * kTwMaxC * 64 * kTcPts * 2) + p : nullptr;
    tw_fwd_loop<N1, N2, PURE, AK>(lc, pi.ch, u, zl);
  }
  // ---- last layer (n -> 1, identity): combine the column parts of every point ---------------------------------
  if (want_grad && tm.n_used > 1) {
    // several passes share P: keep this pass's last hidden activations for its reverse sweep
    tc::fence_async_smem();
    __syncthreads();
    if (tid == 0) {
      uint8_t* h = hst + (size_t)TL * kTwMaxC * 2 * TB;
      const int nb = (pi.nL + 63) >> 6;
      for (int c = 0; c < C; ++c)
        for (int kb = 0; kb < nb; ++kb) tc::bulk_store(h + (size_t)(c * 2 + kb) * TB, tP + (c * 2 + kb) * TB, TB);
      tc::bulk_commit();
      tc::bulk_wait_read0();
    }
  }
  finish_forward<C>(cs, tm, slot, ms, fp + Fp::BL, t, u);
}

// reverse sweep of one network for the current tile (P still holds the last hidden activations)
template <int N1, int N2, bool PURE, int AK>
__device__ __noinline__ void tw_net_backward(TwShared* cs, const DevProblem* Pp, const DevTerm* tmp, int slot) {
  extern __shared__ __align__(1024) uint8_t smem[];
  constexpr int C = 1 + N1 + N2;
  constexpr uint32_t WG = (C <= 3) ? 384u : 0u;       // accumulator column of the weight gradient
  constexpr uint32_t BC = (C <= 2) ? 256u : 128u;     // accumulator column of the bias-gradient column sums (16 columns)
  // dgrad channels whose accumulator columns hold the weight / bias gradient until it is flushed: issued after the flush
  constexpr uint32_t DEFER = (C == 4) ? 0x3u : ((C == 3) ? 0x2u : 0x0u);
  const DevTerm& tm = *tmp;
  const int net_id = tm.used_net[slot];
  const DevNet& net = reinterpret_cast<const DevNet*>(smem + cs->off_nets)[net_id];
  const DevChan& dc = tm.chan[slot];
  const float* fp = reinterpret_cast<const float*>(smem + cs->off_fp[net_id]);
  uint8_t* tP = smem + cs->off_P;
  uint8_t* tS = smem + cs->off_S;
  const Misc ms = misc_of(smem + cs->off_misc, cs->mx_dim, cs->mx_taps);
  const uint32_t accm = 0;   // accumulator address of row 0, column 0
  float* partial = cs->partial;
  PassInfo<N1, N2> pi;
  load_pass<N1, N2>(pi, net, dc);
  const int L = pi.L, TL = pi.TL;
  const Tid t = tid_of();
  const int tid = t.tid, p = t.p;
  float x[PINN_MAX_IN];
#pragma unroll
  for (int k = 0; k < PINN_MAX_IN; ++k) x[k] = (k < pi.d_in) ? ms.Xs[dc.rows[k] * kTcPts + p] : 0.f;
  uint8_t* hst = cs->hstash + (size_t)slot * (cs->tl_max + 1) * kTwMaxC * 2 * TB;
  const float* zst = cs->zstash + (size_t)slot * cs->tl_max * kTwMaxC * 64 * kTcPts * 2;
  const uint8_t* wimg = cs->wpack + (size_t)cs->wimg[net_id] * kTwImgBytes;
  const uint32_t sfp = tc::smem_u32(fp);

  dbg_mark(cs, 20);
  if (tm.n_used > 1) {
    // restore this pass's last hidden activations into P
    if (tid == 0) {
      const uint8_t* h = hst + (size_t)TL * kTwMaxC * 2 * TB;
      const int nb = (pi.nL + 63) >> 6;
      tc::fence_async_smem();
      tc::mbar_arrive_expect_tx(&cs->bar_ld[0], (uint32_t)(C * nb) * TB);
      for (int c = 0; c < C; ++c)
        for (int kb = 0; kb < nb; ++kb) tc::bulk_load(tP + (c * 2 + kb) * TB, h + (size_t)(c * 2 + kb) * TB, TB, &cs->bar_ld[0]);
    }
    tw_wait_ld(cs, 0);
    __syncthreads();
  }
  float ub[C];
  gather_ubar<C>(tm, slot, ms, p, ub);
  // ---- last layer: the ubar tile goes to S0, the products into accumulator columns 0 .. 16C ---------------------------------
  last_layer_grad<C>(t, ub, pi.nL, partial + net.w_off[L - 1], partial + net.b_off[L - 1], tc::smem_u32(tS), tc::smem_u32(tP),
                     2 * TB, pi.nL > 64 ? TB : 0u, accm, kTwW);

  // ---- tensor layers, last to first ------------------------------------------------------------------------------------
  for (int l = TL; l >= 1; --l) {
    const int n_in = net.dims[l], n_out = net.dims[l + 1];
    float* gb = partial + net.b_off[l];
    float* gw = partial + net.w_off[l];
    dbg_mark(cs, 21);
    // this layer's input tiles of channels 0 and 1 stream into S0 / S1 behind the epilogue
    if (tid == 0) {
      const uint8_t* h = hst + (size_t)(l - 1) * kTwMaxC * 2 * TB;
      const int nb = (n_in + 63) >> 6;
      tc::fence_async_smem();
      tw_load(cs, 0, tc::smem_u32(tS), h, nb);
      if (C > 1) tw_load(cs, 1, tc::smem_u32(tS) + kTwImgBytes, h + 2 * TB, nb);
    }
    {
      const LoopW lc(sfp, sfp, tc::smem_u32(tP), t, net.acts[l], n_out / 4, l == TL);
      const float2* zl = reinterpret_cast<const float2*>(zst + (size_t)(l - 1) * kTwMaxC * 64 * kTcPts * 2) + p;
      tw_bwd_loop<N1, N2, PURE, AK>(lc, pi.ch, ub, zl);
    }
    tc::fence_async_smem();
    __syncthreads();
    dbg_mark(cs, 26);
    // wgrad: Wbar_l[o][k] = sum_c sum_p Zbar_c[p][o] H_c[p][k]  -> accumulator columns WG .. WG + n_in (row = o)
    const uint32_t sP = tc::smem_u32(tP), sS = tc::smem_u32(tS);
    {
      const int nb_in = (n_in + 63) >> 6;
      const uint32_t iwg = tc::make_idesc(n_in, 1, 1);
      const uint32_t a_lbo = (n_out > 64) ? TB : 0u;      // rows >= 64 of M: the next tile (n_out = 128)
      const uint8_t* h = hst + (size_t)(l - 1) * kTwMaxC * 2 * TB;
      if (C == 1 && tid == 0) tw_load(cs, 1, sS + kTwImgBytes, wimg + (size_t)(l - 1) * kTwImgBytes, nb_in);
#pragma unroll 1
      for (int c = 0; c < C; ++c) {
        const int b = c & 1;
        tw_wait_ld(cs, b);
        mma_chain(accm + WG, tc::make_desc(sP + (c * 2) * TB, a_lbo, 1024), tc::make_desc(sS + b * kTwImgBytes, TB, 1024),
                  2048, 2048, kTcPts / 16, iwg, c > 0 ? 1u : 0u);
        __syncthreads();      // S[b] has been read
        if (tid == 0) {
          if (c + 2 < C) tw_load(cs, b, sS + b * kTwImgBytes, h + (size_t)(c + 2) * 2 * TB, nb_in);
          else if (c == C - 2)   // W_l for dgrad goes into the buffer wgrad releases first
            tw_load(cs, b, sS + b * kTwImgBytes, wimg + (size_t)(l - 1) * kTwImgBytes, nb_in);
        }
      }
      // bias gradient: bbar_l[o] = sum_p Zbar_0[p][o]  (B = the constant ones atom: SBO = 0, no k advance)
      mma_chain(accm + BC, tc::make_desc(sP, a_lbo, 1024), tc::make_desc(tc::smem_u32(smem + cs->off_ones), 0, 0), 2048, 0,
                kTcPts / 16, tc::make_idesc(16, 1, 1), 0);
    }
    dbg_mark(cs, 27);
    __syncthreads();
    dbg_mark(cs, 28);
    // dgrad: Hbar_c[p][k] = sum_o Zbar_c[p][o] W_l[o][k] -> X (channel c at column c*128); W_l sits in S[C & 1]
    const int wb = C & 1;
    tw_wait_ld(cs, wb);
    const int nb_out = (n_out + 63) >> 6;
    const uint32_t idg = tc::make_idesc(n_in, 0, 1);
    const uint32_t wbuf = sS + wb * kTwImgBytes;
#pragma unroll 1
    for (int c = C - 1; c >= 0; --c) {
      if ((DEFER >> c) & 1u) continue;
#pragma unroll 1
      for (int ob = 0; ob < nb_out; ++ob) {
        const int nk = ((n_out - ob * 64) < 64 ? (n_out - ob * 64) : 64) >> 4;
        mma_chain(accm + c * kTwW, tc::make_desc(sP + (c * 2 + ob) * TB, 0, 1024), tc::make_desc(wbuf + ob * 8192, TB, 1024),
                  32, 2048, nk, idg, ob > 0 ? 1u : 0u);
      }
    }
    flush_wgrad(t, accm + WG, accm + BC, kTwW, n_in, n_out, gw, gb);
    if (DEFER != 0) {
      // the remaining channels' adjoints land on the columns the weight / bias gradient just left
      __syncthreads();
#pragma unroll 1
      for (int c = C - 1; c >= 0; --c) {
        if (!((DEFER >> c) & 1u)) continue;
#pragma unroll 1
        for (int ob = 0; ob < nb_out; ++ob) {
          const int nk = ((n_out - ob * 64) < 64 ? (n_out - ob * 64) : 64) >> 4;
          mma_chain(accm + c * kTwW, tc::make_desc(sP + (c * 2 + ob) * TB, 0, 1024), tc::make_desc(wbuf + ob * 8192, TB, 1024),
                    32, 2048, nk, idg, ob > 0 ? 1u : 0u);
        }
      }
    }
    __syncthreads();
    dbg_mark(cs, 29);
  }

  // ---- layer 0 reverse: Zbar^0 tiles, then  D[o][0..15] = Zbar_0^T [x | 1] + sum_j Zbar_(1+j)^T E_(dir1[j]) -----------------
  {
    float* gb0 = partial + net.b_off[0];
    float* gw0 = partial + net.w_off[0];
    constexpr bool kLo = (2 + N1) <= 4;         // a spare tile for the bf16 residual of the coordinates
    const uint32_t sP = tc::smem_u32(tP), sS = tc::smem_u32(tS);
    coord_tiles<N1>(t, sS, x, pi.dir1, kLo);
    tw_l0_bwd_store_loop<N1, N2, PURE, AK>(LoopW(sfp, sfp, sP, t, net.acts[0], pi.n1w / 2, 0), pi, x);
    layer0_grad<N1>(t, sP, 2 * TB, pi.n1w > 64 ? TB : 0u, sS, kLo, accm + WG, kTwW, pi.n1w, pi.d_in, gw0, gb0);
  }
  __syncthreads();
  dbg_mark(cs, 30);
}


// ---- weight packing: theta (fp32, out x in column-major) -> bf16 swizzled images [kb][128 rows o][64 k] ---------------
__global__ void __launch_bounds__(256) tw_pack_kernel(const TwPackArgs a) {
  const int img = blockIdx.x >> 3;
  const int idx = (blockIdx.x & 7) * 256 + threadIdx.x;     // 2048 16-byte chunks per image
  if (blockIdx.x == 0 && threadIdx.x == 0) *a.tile_counter = a.counter_init;
  if (img >= a.n_images) return;
  const DevNet& net = a.prob->nets[a.img_net[img]];
  const int l = a.img_layer[img];
  const int n_in = net.dims[l], n_out = net.dims[l + 1];
  const long long woff = net.w_off[l];
  const int kb = idx >> 10, o = (idx >> 3) & 127, kc = idx & 7;
  float w[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int k = kb * 64 + kc * 8 + e;
    w[e] = (o < n_out && k < n_in) ? __ldg(&a.theta[woff + o + (long long)n_out * k]) : 0.f;
  }
  uint4 h;
  h.x = tc::pack_bf16(w[0], w[1]); h.y = tc::pack_bf16(w[2], w[3]);
  h.z = tc::pack_bf16(w[4], w[5]); h.w = tc::pack_bf16(w[6], w[7]);
  *reinterpret_cast<uint4*>(a.wpack + (size_t)img * kTwImgBytes + (size_t)kb * TB + tc::swz_chunk(o, kc)) = h;
}

__global__ void __launch_bounds__(kTcThreads, 1) tw_loss_grad_kernel(const __grid_constant__ TwArgs args) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ TwShared cs;
  const int tid = threadIdx.x;
  const DevProblem* Pp = args.prob;
  const DevProblem& P = *Pp;
  const Misc ms = misc_of(smem + args.off_misc, args.mx_dim, args.mx_taps);
  float* partial = args.partial + (long long)blockIdx.x * args.partial_stride;
  const bool want_grad = (args.mode == 0);
  const float* theta = args.theta;
  const DbgSpan span = dbg_span_begin(args.dbg);

  // ---- per-CTA setup --------------------------------------------------------------------------------------------------------
  if (tid == 0) {
    tc::mbar_init(ms.bar_ld, 1);            // collocation-tile bulk loads (own barrier: the weight stream uses cs.bar_ld[])
    for (int b = 0; b < 2; ++b) {
      tc::mbar_init(&cs.bar_ld[b], 1);
      cs.ph_ld[b] = 0;
    }
    tc::fence_barrier_init();
    cs.off_S = args.off_S; cs.off_nets = args.off_nets;
    cs.hstash = args.hstash + (long long)blockIdx.x * args.hstash_per_cta;
    cs.zstash = args.zstash + (long long)blockIdx.x * args.zstash_per_cta;
    cs.wpack = args.wpack;
    for (int k = 0; k < PINN_MAX_NETS; ++k) { cs.off_fp[k] = args.off_fp[k]; cs.wimg[k] = args.wimg[k]; }
    cta_base_init(cs, args, partial);
  }
  if (tid == 0) tc::s_acc = args.acc + (size_t)blockIdx.x * kAccCols * kAccRows;
  cta_setup(args, ms, partial, P.n_theta, want_grad);
  {      // network descriptors: every layer of every sweep reads widths / offsets / activations
    const int nw = P.n_nets * (int)(sizeof(DevNet) / 4);
    const int* src = reinterpret_cast<const int*>(&P.nets[0]);
    int* dst = reinterpret_cast<int*>(smem + args.off_nets);
    for (int i = tid; i < nw; i += kTcThreads) dst[i] = __ldg(src + i);
  }
  // fp32 blocks of the first / last layers and the tensor-layer biases
  for (int kn = 0; kn < P.n_nets; ++kn)
    if (args.off_fp[kn] >= 0) stage_fp_block<kTwW>(reinterpret_cast<float*>(smem + args.off_fp[kn]), P.nets[kn], theta);
  tc::fence_async_smem();
  __syncthreads();
  dbg_mark(&cs, 2);
  uint32_t tile_ld_phase = 0;      // parity of the collocation-tile barrier (ms.bar_ld)

  // tiles are claimed dynamically after the first one (heavy PDE tiles come first in the enumeration, cheap boundary
  // tiles last): a static round-robin leaves the CTAs that drew an extra PDE tile 20 % behind the rest
  for (int tile = args.tile_begin + blockIdx.x; tile < args.tile_end;) {
    const TileRef tr = stage_tile(args, P, ms, tile, tile_ld_phase);
    const DevTerm* tmp = &P.terms[tr.ti];
    const DevTerm& tm = *tmp;
    const int n_used = tm.n_used;
    dbg_mark(&cs, 3);

    for (int slot = 0; slot < n_used; ++slot) {
      const int k1 = tm.chan[slot].n1, k2 = tm.chan[slot].n2, pu = tm.chan[slot].pure;
      const int ak = args.net_ak[tm.used_net[slot]];
      PINN_TC_DISPATCH(kTwMaxC, k1, k2, pu, ak, (tw_net_forward<A1, A2, PU, AK>(&cs, Pp, tmp, slot, want_grad ? 1 : 0)));
    }

    dbg_mark(&cs, 4);
    // S0 / S1 are idle between the sweeps
    residual_step(args, P, tm, ms, tr, smem + args.off_S, (size_t)(2 * kTwImgBytes), partial, want_grad);

    dbg_mark(&cs, 5);
    if (want_grad) {
      if (tid == 0) tc::bulk_wait0();             // operand-tile stash writes of this tile are complete before reloads
      __threadfence_block();
      __syncthreads();
      dbg_mark(&cs, 6);
      for (int slot = n_used - 1; slot >= 0; --slot) {
        const int k1 = tm.chan[slot].n1, k2 = tm.chan[slot].n2, pu = tm.chan[slot].pure;
        const int ak = args.net_ak[tm.used_net[slot]];
        PINN_TC_DISPATCH(kTwMaxC, k1, k2, pu, ak, (tw_net_backward<A1, A2, PU, AK>(&cs, Pp, tmp, slot)));
      }
    }
    // claim the next tile only now: claiming a tile ahead would hand the last cheap tiles to CTAs that still owe a heavy one
    if (tid == 0) cs.next_tile = atomicAdd(args.tile_counter, 1);
    __syncthreads();
    tile = cs.next_tile;
  }

  __syncthreads();
  dbg_mark(&cs, 7);
  cta_finish(args, cs, span, ms, P, want_grad);
}

// ---- host side ------------------------------------------------------------------------------------------------------------------
cudaError_t tw_pack_launch(const TwPackArgs& a, cudaStream_t st) {
  tw_pack_kernel<<<(a.n_images > 0 ? a.n_images : 1) * 8, 256, 0, st>>>(a);
  return cudaGetLastError();
}

cudaError_t tw_launch(const TwArgs& a, int grid, size_t smem, cudaStream_t st) {
  return launch_fused_kernel<tw_loss_grad_kernel>(a, grid, kTcThreads, smem, st);
}

}  // namespace pinn
