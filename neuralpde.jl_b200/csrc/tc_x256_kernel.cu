// tc_x256_kernel.cu -- fused PINN loss+gradient kernel, tensor-core path for hidden widths that are multiples of 64 up to
// 256 (sm_90a wgmma, bf16 operands).
//
// Same tile driver as tc_wide_kernel.cu (128-point tiles, dynamic tile claims, the shared residual step and kernel end),
// but every network pass runs on the two 64-point halves of a tile in turn.  At 64 points a 256-wide buffer is the size
// the wide kernel's 128-wide buffers have at 128 points:
//
//   * an activation set is C channels x 4 tiles (64 points x 64 bf16, 128-byte swizzle) = C x 32 KB in region P (C <= 4);
//   * the accumulator region [512 cols][128 rows] is used as two 64-row banks: channel c owns bank c >> 1, columns
//     (c & 1) * 256 .. + 255, so that C x 256 columns of 64 rows fit; a weight gradient (up to 256 x 256) fills both
//     banks and is flushed before the dgrad reuses them;
//   * weights are packed once per step by tx_pack_kernel into 128 KB images [kb][o / 128][128 rows o][64 k] and streamed
//     through two 32 KB buffers S0 / S1: the forward takes one K-chunk (64 k, every o) at a time, the dgrad one output
//     chunk (64 o, every k: four 8 KB row ranges), both prefetched one chunk ahead;
//   * with M = 64 an MMA chain is one warpgroup's M extent: the forward and dgrad split N into 64-column blocks (block j
//     on warpgroup j), the wgrad splits M (64-row block j of W-bar on warpgroup j);
//   * the forward stashes every tensor layer's input tiles (bf16) and pre-activations (fp32) per half, and the last
//     hidden activations, which the reverse sweep restores into P; the stash holds the channels of the problem's largest
//     term, pass by pass.
// Rounding is the wide kernel's: weights, activation tiles, Zbar tiles, (hi, lo) ubar of the last layer and the
// coordinates' (hi, lo) in the layer-0 gradient, so tests/tc_model.py's tw_bf16 mode models this kernel as well.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include "tc_common.cuh"

namespace pinn {

constexpr uint32_t TB = kTileBytes;      // 128-row block of a packed image
constexpr uint32_t HB = kTxTileBytes;    // 64-row operand tile
constexpr uint32_t SB = 4 * HB;          // one stream buffer, one channel of activations
using Fx = FpBlock<kTxW>;

struct TxShared : CtaBase {
  int off_S, off_nets, off_fp;
  int fp_net;                        // network whose fp32 block is staged at off_fp (-1: none)
  const float* theta;
  uint8_t* hstash;
  float* zstash;
  int nch;                           // channels per layer of the stash: the most (pass, half) channels of a term
  const uint8_t* wpack;
  int wimg[PINN_MAX_NETS];
  int next_tile;
  uint32_t ph_ld[2];
  uint64_t bar_ld[2];
};

// thread identity inside a half tile: point row r (0..63: warp parity and lane), column eighth `part` (warp / 2)
struct Tx {
  int tid, lane, r, rb, part, p;     // rb: accumulator row base of the warp; p: the point in the 128-point tile
};
__device__ __forceinline__ Tx tx_of(int half) {
  Tx t;
  t.tid = threadIdx.x; t.lane = t.tid & 31;
  const int w = t.tid >> 5;
  t.rb = (w & 1) * 32; t.r = t.rb + t.lane; t.part = w >> 1; t.p = half * kTxPts + t.r;
  return t;
}
// accumulator address of channel c, column col, rows from `row` (bank c >> 1)
__device__ __forceinline__ uint32_t xacc(int c, int row, int col) {
  return ((uint32_t)(64 * (c >> 1) + row) << 16) | (uint32_t)((c & 1) * kTxW + col);
}
// accumulator value of block j (64 rows of bank j >> 1, columns from (j & 1) * 256), row o & 63, column col
__device__ __forceinline__ float xacc_at(int j, int o, int col) {
  return tc::s_acc[(size_t)((j & 1) * kTxW + col) * kAccRows + 64 * (j >> 1) + (o & 63)];
}

// an MMA chain D[64 x N] (+)= A_k * B_k on warpgroup wg into rows [64 bank, 64 bank + 64) at column dcol.  Chains into
// the same columns are issued on the same warpgroup, so they run in program order; results are visible to the CTA after
// the next __syncthreads.
template <int N, int TA, int TB_>
static __device__ __noinline__ void x_chain(int wg, int bank, uint32_t dcol, uint64_t a, uint64_t b, uint32_t a_step,
                                            uint32_t b_step, int nk, uint32_t acc_first) {
  if ((int)(threadIdx.x >> 7) == wg) tc::wg_chain<N, TA, TB_>(dcol, bank, a, b, a_step, b_step, nk, acc_first);
}
// descriptor of a 64-row operand tile; every operand here is one tile wide in M / N, so no leading-dimension offset
__device__ __forceinline__ uint64_t xdesc(uint32_t addr) { return tc::make_desc(addr, 0, 1024); }

__device__ __forceinline__ uint32_t tile_x(uint32_t sP, int c, int col) { return sP + (uint32_t)(c * 4 + (col >> 6)) * HB; }

// ---- streaming: thread 0 issues the bulk loads, every thread waits for them ----------------------------------------------
__device__ __forceinline__ void tx_load(TxShared* cs, int b, uint32_t dst, const uint8_t* src, uint32_t bytes) {
  tc::mbar_arrive_expect_tx(&cs->bar_ld[b], bytes);
  tc::bulk_load_u(dst, src, bytes, tc::smem_u32(&cs->bar_ld[b]));
}
// dgrad chunk j of a layer image: rows o in [64 j, 64 j + 64) of every 64-column block kq of k, one 8 KB tile each
__device__ __forceinline__ void tx_load_rows(TxShared* cs, int b, uint32_t dst, const uint8_t* img, int j, int nkq) {
  tc::mbar_arrive_expect_tx(&cs->bar_ld[b], (uint32_t)nkq * HB);
  for (int kq = 0; kq < nkq; ++kq)
    tc::bulk_load_u(dst + (uint32_t)kq * HB, img + (size_t)(kq * 2 + (j >> 1)) * TB + (size_t)(j & 1) * HB, HB,
                    tc::smem_u32(&cs->bar_ld[b]));
}
// CTA-wide: the next read of cs->ph_ld[b] must follow another __syncthreads
__device__ __forceinline__ void tx_wait_ld(TxShared* cs, int b) {
  const uint32_t ph = cs->ph_ld[b];
  tc::mbar_wait(&cs->bar_ld[b], ph);
  __syncthreads();
  if (threadIdx.x == 0) cs->ph_ld[b] = ph ^ 1u;
}

// the network's fp32 block (first / last layer, tensor-layer biases) in the one staging area; CTA-wide
__device__ __forceinline__ void tx_stage_fp(TxShared* cs, const DevNet& net, int net_id) {
  extern __shared__ __align__(1024) uint8_t smem[];
  if (cs->fp_net == net_id) return;
  __syncthreads();
  stage_fp_block<kTxW>(reinterpret_cast<float*>(smem + cs->off_fp), net, cs->theta);
  __syncthreads();
  if (threadIdx.x == 0) cs->fp_net = net_id;
  __syncthreads();
}

// The stash is [layer][channel]: bf16 operand tiles [tl_max + 1][nch][4 tiles], fp32 pre-activations
// [tl_max][nch][128][64] float2.  The channels of a term are numbered pass by pass, both halves of a pass in turn, so a
// CTA keeps only as many as the problem's largest term has (sum over its passes of 2 C).
__device__ __forceinline__ int tx_chan0(const DevTerm& tm, int slot, int half) {
  int c0 = 0;
  for (int s = 0; s < slot; ++s) c0 += 2 * tm.chan[s].C;
  return c0 + half * tm.chan[slot].C;
}
__device__ __forceinline__ uint8_t* tx_hst(const TxShared* cs, int l, int ch) {
  return cs->hstash + ((size_t)l * cs->nch + ch) * SB;
}
__device__ __forceinline__ float2* tx_zst(const TxShared* cs, int l, int ch) {
  return reinterpret_cast<float2*>(cs->zstash) + ((size_t)l * cs->nch + ch) * 128 * kTxPts;
}

// ---- epilogues (one point per thread, an eighth of the columns) ---------------------------------------------------------
// layer 0 forward: coordinates -> H^0 tiles
template <int N1, int N2, bool PURE, int AK>
__device__ __forceinline__ void tx_l0_fwd_loop(const Tx& t, uint32_t sfp, uint32_t sP, int act, int n1w,
                                               const PassInfo<N1, N2>& pi, const float (&x)[PINN_MAX_IN]) {
  constexpr int C = 1 + N1 + N2;
  const int ng = n1w >> 5;
#pragma unroll 1
  for (int g = t.part * ng; g < (t.part + 1) * ng; ++g) {
    float h[C][4];
#pragma unroll
    for (int i = 0; i < 4; i += 2) {
      float za[C], zb2[C];
      first_layer_elem<kTxW>(sfp, pi, x, g * 4 + i, za);
      first_layer_elem<kTxW>(sfp, pi, x, g * 4 + i + 1, zb2);
      P2 zz[C], hv[C];
#pragma unroll
      for (int c = 0; c < C; ++c) zz[c] = mk2(za[c], zb2[c]);
      chain_fwd<N1, N2, PURE, AK, P2>(act, pi.ch, zz, hv);
#pragma unroll
      for (int c = 0; c < C; ++c) { h[c][i] = hv[c].v.x; h[c][i + 1] = hv[c].v.y; }
    }
    const int col = g * 4;
#pragma unroll
    for (int c = 0; c < C; ++c) store_half(tile_x(sP, c, col), 0u, t.r, col & 63, h[c], false);
  }
}

// tensor layer forward: accumulators -> bias + activation chain -> next operand tiles (in place), pre-activations ->
// stash (zst, this thread's row), last-layer dot products (flag)
template <int N1, int N2, bool PURE, int AK>
__device__ __forceinline__ void tx_fwd_loop(const Tx& t, uint32_t sfp, uint32_t bt, uint32_t sP, int act, int n_out, int flag,
                                            const Chan<N1, N2>& ch, float (&u)[1 + N1 + N2], float2* zst) {
  constexpr int C = 1 + N1 + N2;
  const int ng = n_out >> 5;
#pragma unroll 1
  for (int g = t.part * ng; g < (t.part + 1) * ng; ++g) {
    const int col = g * 4;
    float z[C][4];
#pragma unroll
    for (int c = 0; c < C; ++c) acc_ld4(xacc(c, t.rb, col), z[c]);
#pragma unroll
    for (int i = 0; i < 4; i += 2) {
      P2 zz[C], hv[C];
      zz[0] = mk2(z[0][i] + lds_f32(bt + (col + i) * 4), z[0][i + 1] + lds_f32(bt + (col + i + 1) * 4));
#pragma unroll
      for (int c = 1; c < C; ++c) zz[c] = mk2(z[c][i], z[c][i + 1]);
      if (zst) {
#pragma unroll
        for (int c = 0; c < C; ++c) zst[(c * 128 + ((col + i) >> 1)) * kTxPts] = zz[c].v;
      }
      chain_fwd<N1, N2, PURE, AK, P2>(act, ch, zz, hv);
#pragma unroll
      for (int c = 0; c < C; ++c) { z[c][i] = hv[c].v.x; z[c][i + 1] = hv[c].v.y; }
      if (flag) {
        const float w0 = lds_f32(sfp + (Fx::WL + col + i) * 4), w1 = lds_f32(sfp + (Fx::WL + col + i + 1) * 4);
#pragma unroll
        for (int c = 0; c < C; ++c) u[c] = fmaf(w1, hv[c].v.y, fmaf(w0, hv[c].v.x, u[c]));
      }
    }
#pragma unroll
    for (int c = 0; c < C; ++c) store_half(tile_x(sP, c, col), 0u, t.r, col & 63, z[c], false);
  }
}

// tensor layer reverse: stashed pre-activations and output adjoints (accumulators, or w_last * ubar for the last hidden
// layer: flag) -> Zbar tiles in P
template <int N1, int N2, bool PURE, int AK>
__device__ __forceinline__ void tx_bwd_loop(const Tx& t, uint32_t sfp, uint32_t sP, int act, int n_out, int flag,
                                            const Chan<N1, N2>& ch, const float (&ub)[1 + N1 + N2], const float2* zst) {
  constexpr int C = 1 + N1 + N2;
  const int ng = n_out >> 5;
#pragma unroll 1
  for (int g = t.part * ng; g < (t.part + 1) * ng; ++g) {
    const int col = g * 4;
    float hb[C][4];
    float2 zc[C][2];
#pragma unroll
    for (int c = 0; c < C; ++c) {
      zc[c][0] = zst[(c * 128 + 2 * g) * kTxPts];
      zc[c][1] = zst[(c * 128 + 2 * g + 1) * kTxPts];
    }
    if (!flag) {
#pragma unroll
      for (int c = 0; c < C; ++c) acc_ld4(xacc(c, t.rb, col), hb[c]);
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float wl = lds_f32(sfp + (Fx::WL + col + i) * 4);
#pragma unroll
        for (int c = 0; c < C; ++c) hb[c][i] = wl * ub[c];
      }
    }
#pragma unroll
    for (int i = 0; i < 4; i += 2) {
      P2 zz[C], hv[C], zv[C];
#pragma unroll
      for (int c = 0; c < C; ++c) { zz[c].v = zc[c][i >> 1]; hv[c] = mk2(hb[c][i], hb[c][i + 1]); }
      chain_bwd<N1, N2, PURE, AK, P2>(act, ch, zz, hv, zv);
#pragma unroll
      for (int c = 0; c < C; ++c) { hb[c][i] = zv[c].v.x; hb[c][i + 1] = zv[c].v.y; }
    }
#pragma unroll
    for (int c = 0; c < C; ++c) store_half(tile_x(sP, c, col), 0u, t.r, col & 63, hb[c], false);
  }
}

// layer 0 reverse: adjoints of H^0 (accumulators) -> Zbar^0 tiles of the value + first-derivative channels in P
template <int N1, int N2, bool PURE, int AK>
__device__ __forceinline__ void tx_l0_bwd_loop(const Tx& t, uint32_t sfp, uint32_t sP, int act, int n1w,
                                               const PassInfo<N1, N2>& pi, const float (&x)[PINN_MAX_IN]) {
  constexpr int C = 1 + N1 + N2;
  const int ng = n1w >> 4;
#pragma unroll 1
  for (int g = t.part * ng; g < (t.part + 1) * ng; ++g) {
    const int col = g * 2;
    float hb[C][2];
#pragma unroll
    for (int c = 0; c < C; ++c) acc_ld2(xacc(c, t.rb, col), hb[c]);
    float za[C], zb2[C];
    first_layer_elem<kTxW>(sfp, pi, x, col, za);
    first_layer_elem<kTxW>(sfp, pi, x, col + 1, zb2);
    P2 zz[C], hv[C], zv[C];
#pragma unroll
    for (int c = 0; c < C; ++c) { zz[c] = mk2(za[c], zb2[c]); hv[c] = mk2(hb[c][0], hb[c][1]); }
    chain_bwd<N1, N2, PURE, AK, P2>(act, pi.ch, zz, hv, zv);
#pragma unroll
    for (int c = 0; c <= N1; ++c) {
      const float o2[2] = {zv[c].v.x, zv[c].v.y};
      store_half(tile_x(sP, c, col), 0u, t.r, col & 63, o2, false);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// forward of one network on one half tile
template <int N1, int N2, bool PURE, int AK>
__device__ __noinline__ void tx_net_forward(TxShared* cs, const DevTerm* tmp, int slot, int half, int want_grad) {
  extern __shared__ __align__(1024) uint8_t smem[];
  constexpr int C = 1 + N1 + N2;
  const DevTerm& tm = *tmp;
  const int net_id = tm.used_net[slot];
  const DevNet& net = reinterpret_cast<const DevNet*>(smem + cs->off_nets)[net_id];
  const DevChan& dc = tm.chan[slot];
  tx_stage_fp(cs, net, net_id);
  const float* fp = reinterpret_cast<const float*>(smem + cs->off_fp);
  const Misc ms = misc_of(smem + cs->off_misc, cs->mx_dim, cs->mx_taps);
  PassInfo<N1, N2> pi;
  load_pass<N1, N2>(pi, net, dc);
  const int TL = pi.TL;
  const Tx t = tx_of(half);
  const int tid = t.tid;
  float x[PINN_MAX_IN];
#pragma unroll
  for (int k = 0; k < PINN_MAX_IN; ++k) x[k] = (k < pi.d_in) ? ms.Xs[dc.rows[k] * kTcPts + t.p] : 0.f;
  const int ch0 = tx_chan0(tm, slot, half);
  const uint8_t* wimg = cs->wpack + (size_t)cs->wimg[net_id] * kTxImgBytes;
  const uint32_t sP = tc::smem_u32(smem + cs->off_P), sS = tc::smem_u32(smem + cs->off_S), sfp = tc::smem_u32(fp);
  uint8_t* tP = smem + cs->off_P;

  dbg_mark(cs, 10);
  float u[C];
#pragma unroll
  for (int c = 0; c < C; ++c) u[c] = 0.f;
  if (tid < C * kTxPts) ms.scratch[(tid / kTxPts) * kTcPts + half * kTxPts + (tid % kTxPts)] = 0.f;
  // weight K-chunk q of the pass (layer l, columns 64 kb ..) streams into buffer q & 1, one chunk ahead; the 128-row
  // halves of o beyond the layer's width are not loaded
  auto chunk_bytes = [&](int l) { return (uint32_t)((net.dims[l + 1] + 127) >> 7) * TB; };
  if (tid == 0) {
    tc::fence_async_smem();
    tx_load(cs, 0, sS, wimg, chunk_bytes(1));
  }
  tx_l0_fwd_loop<N1, N2, PURE, AK>(t, sfp, sP, net.acts[0], pi.n1w, pi, x);
  int q = 0;
  for (int l = 1; l <= TL; ++l) {
    const int n_in = net.dims[l], n_out = net.dims[l + 1];
    const int nb_in = n_in >> 6, nj = n_out >> 6;
    tc::fence_async_smem();
    __syncthreads();
    dbg_mark(cs, 11);
    if (want_grad && tid == 0) {
      for (int c = 0; c < C; ++c) tc::bulk_store(tx_hst(cs, l - 1, ch0 + c), tP + c * SB, (uint32_t)nb_in * HB);
      tc::bulk_commit();
    }
#pragma unroll 1
    for (int kb = 0; kb < nb_in; ++kb, ++q) {
      if (tid == 0) {
        const int nb = (q + 1) & 1;
        if (kb + 1 < nb_in)
          tx_load(cs, nb, sS + nb * SB, wimg + (size_t)(l - 1) * kTxImgBytes + (size_t)(kb + 1) * 2 * TB, chunk_bytes(l));
        else if (l < TL)
          tx_load(cs, nb, sS + nb * SB, wimg + (size_t)l * kTxImgBytes, chunk_bytes(l + 1));
      }
      tx_wait_ld(cs, q & 1);
      const uint32_t wb = sS + (q & 1) * SB;
#pragma unroll 1
      for (int c = 0; c < C; ++c)
#pragma unroll 1
        for (int j = 0; j < nj; ++j)
          x_chain<64, 0, 0>(j, c >> 1, (c & 1) * kTxW + j * 64, xdesc(sP + (c * 4 + kb) * HB),
                            xdesc(wb + (j >> 1) * TB + (j & 1) * HB), 32, 32, 4, kb > 0 ? 1u : 0u);
      __syncthreads();     // buffer q & 1 has been read
    }
    dbg_mark(cs, 12);
    if (want_grad && tid == 0) tc::bulk_wait_read0();   // stash copies have finished reading P
    __syncthreads();
    dbg_mark(cs, 14);
    float2* zl = want_grad ? tx_zst(cs, l - 1, ch0) + t.r : nullptr;
    tx_fwd_loop<N1, N2, PURE, AK>(t, sfp, sfp + (Fx::BT + (l - 1) * kTxW) * 4, sP, net.acts[l], n_out, l == TL, pi.ch, u, zl);
  }
  if (want_grad) {
    // the halves and passes share P: keep this pass's last hidden activations for its reverse sweep
    tc::fence_async_smem();
    __syncthreads();
    if (tid == 0) {
      for (int c = 0; c < C; ++c) tc::bulk_store(tx_hst(cs, TL, ch0 + c), tP + c * SB, (uint32_t)(pi.nL >> 6) * HB);
      tc::bulk_commit();
      tc::bulk_wait_read0();
    }
  }
  Tid ft;
  ft.tid = tid; ft.lane = t.lane; ft.p = t.p; ft.hh = t.part;
  finish_forward<C>(cs, tm, slot, ms, fp + Fx::BL, ft, u);
}

// reverse sweep of one network on one half tile
template <int N1, int N2, bool PURE, int AK>
__device__ __noinline__ void tx_net_backward(TxShared* cs, const DevTerm* tmp, int slot, int half) {
  extern __shared__ __align__(1024) uint8_t smem[];
  constexpr int C = 1 + N1 + N2;
  const DevTerm& tm = *tmp;
  const int net_id = tm.used_net[slot];
  const DevNet& net = reinterpret_cast<const DevNet*>(smem + cs->off_nets)[net_id];
  const DevChan& dc = tm.chan[slot];
  tx_stage_fp(cs, net, net_id);
  const float* fp = reinterpret_cast<const float*>(smem + cs->off_fp);
  const Misc ms = misc_of(smem + cs->off_misc, cs->mx_dim, cs->mx_taps);
  float* partial = cs->partial;
  PassInfo<N1, N2> pi;
  load_pass<N1, N2>(pi, net, dc);
  const int L = pi.L, TL = pi.TL;
  const Tx t = tx_of(half);
  const int tid = t.tid;
  float x[PINN_MAX_IN];
#pragma unroll
  for (int k = 0; k < PINN_MAX_IN; ++k) x[k] = (k < pi.d_in) ? ms.Xs[dc.rows[k] * kTcPts + t.p] : 0.f;
  const int ch0 = tx_chan0(tm, slot, half);
  const uint8_t* wimg = cs->wpack + (size_t)cs->wimg[net_id] * kTxImgBytes;
  const uint32_t sP = tc::smem_u32(smem + cs->off_P), sS = tc::smem_u32(smem + cs->off_S), sfp = tc::smem_u32(fp);

  dbg_mark(cs, 20);
  // restore this pass's last hidden activations into P
  if (tid == 0) {
    tc::fence_async_smem();
    tc::mbar_arrive_expect_tx(&cs->bar_ld[0], (uint32_t)(C * (pi.nL >> 6)) * HB);
    for (int c = 0; c < C; ++c)
      tc::bulk_load_u(sP + c * SB, tx_hst(cs, TL, ch0 + c), (uint32_t)(pi.nL >> 6) * HB, tc::smem_u32(&cs->bar_ld[0]));
  }
  tx_wait_ld(cs, 0);
  __syncthreads();
  float ub[C];
  gather_ubar<C>(tm, slot, ms, t.p, ub);

  // ---- last layer: bias by warp sums; wbar_L[o] = sum_c H_c^T (ubar_c hi, lo) with the ubar tile in S0 -------------------
  {
    float* gw = partial + net.w_off[L - 1];
    if (t.part == 0) {
      const float s = warp_sum<float>(ub[0]);
      if (t.lane == 0) atomicAdd(partial + net.b_off[L - 1], s);
      uint32_t w[8];
#pragma unroll
      for (int c = 0; c < 8; ++c) w[c] = 0u;
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const uint32_t hi = tc::pack_bf16(ub[c], 0.f);
        w[c] = hi | (bf16x2_lo(ub[c], 0.f, hi) << 16);
      }
      sts_v4(sS + tc::swz_chunk(t.r, 0), w[0], w[1], w[2], w[3]);
      sts_v4(sS + tc::swz_chunk(t.r, 1), w[4], w[5], w[6], w[7]);
    }
    tc::fence_async_smem();
    __syncthreads();
#pragma unroll 1
    for (int j = 0; j < (pi.nL >> 6); ++j)
#pragma unroll 1
      for (int c = 0; c < C; ++c)
        x_chain<16, 1, 1>(j, j >> 1, (j & 1) * kTxW + 16 * c, xdesc(sP + (c * 4 + j) * HB), tc::make_desc(sS, 0, 1024), 2048,
                          2048, kTxPts / 16, 0);
    __syncthreads();
    if (tid < pi.nL) {
      float acc = 0.f;
#pragma unroll
      for (int c = 0; c < C; ++c) acc += xacc_at(tid >> 6, tid, 16 * c + 2 * c) + xacc_at(tid >> 6, tid, 16 * c + 2 * c + 1);
      atomicAdd(gw + tid, acc);
    }
    __syncthreads();
  }

  // ---- tensor layers, last to first ------------------------------------------------------------------------------------
  for (int l = TL; l >= 1; --l) {
    const int n_in = net.dims[l], n_out = net.dims[l + 1];
    const int nkq = n_in >> 6, nj = n_out >> 6;
    float* gb = partial + net.b_off[l];
    float* gw = partial + net.w_off[l];
    const uint8_t* h = tx_hst(cs, l - 1, ch0);      // channel c at h + c * SB
    const uint8_t* img = wimg + (size_t)(l - 1) * kTxImgBytes;
    dbg_mark(cs, 21);
    // this layer's input tiles of channels 0 and 1 stream into S0 / S1 behind the epilogue
    if (tid == 0) {
      tc::fence_async_smem();
      tx_load(cs, 0, sS, h, (uint32_t)nkq * HB);
      if (C > 1) tx_load(cs, 1, sS + SB, h + SB, (uint32_t)nkq * HB);
    }
    tx_bwd_loop<N1, N2, PURE, AK>(t, sfp, sP, net.acts[l], n_out, l == TL, pi.ch, ub, tx_zst(cs, l - 1, ch0) + t.r);
    tc::fence_async_smem();
    __syncthreads();
    dbg_mark(cs, 26);
    // wgrad: Wbar_l[o][k] = sum_c sum_p Zbar_c[p][o] H_c[p][k]; o-block j on warpgroup j -> accumulator block j
#pragma unroll 1
    for (int c = 0; c < C; ++c) {
      const int b = c & 1;
      tx_wait_ld(cs, b);
#pragma unroll 1
      for (int j = 0; j < nj; ++j)
#pragma unroll 1
        for (int kq = 0; kq < nkq; ++kq)
          x_chain<64, 1, 1>(j, j >> 1, (j & 1) * kTxW + kq * 64, xdesc(sP + (c * 4 + j) * HB), xdesc(sS + b * SB + kq * HB),
                            2048, 2048, kTxPts / 16, c > 0 ? 1u : 0u);
      __syncthreads();      // S[b] has been read
      if (tid == 0 && c + 2 < C) tx_load(cs, b, sS + b * SB, h + (size_t)(c + 2) * SB, (uint32_t)nkq * HB);
    }
    // the first dgrad chunk of W_l streams in behind the flush
    if (tid == 0) tx_load_rows(cs, 0, sS, img, 0, nkq);
    {   // flush: warp w takes the 32 rows (w & 7) of o and half (w >> 3) of the columns k
      const int w = tid >> 5, rg = w & 7, o = rg * 32 + t.lane, j = o >> 6;
      if (rg * 32 < n_out) {
        const int half_k = n_in >> 1;
#pragma unroll 1
        for (int k0 = (w >> 3) * half_k; k0 < ((w >> 3) + 1) * half_k; k0 += 4) {
          float v[4];
          acc_ld4(((uint32_t)(64 * (j >> 1) + (rg & 1) * 32) << 16) | (uint32_t)((j & 1) * kTxW + k0), v);
#pragma unroll
          for (int i = 0; i < 4; ++i) atomicAdd(gw + o + (long long)n_out * (k0 + i), v[i]);
        }
      }
    }
    __syncthreads();
    // bias gradient: bbar_l[o] = sum_p Zbar_0[p][o]  (B = the constant ones atom: SBO = 0, no k advance)
#pragma unroll 1
    for (int j = 0; j < nj; ++j)
      x_chain<16, 1, 1>(j, j >> 1, (j & 1) * kTxW, xdesc(sP + j * HB), tc::make_desc(tc::smem_u32(smem + cs->off_ones), 0, 0),
                        2048, 0, kTxPts / 16, 0);
    __syncthreads();
    if (tid < n_out) atomicAdd(gb + tid, xacc_at(tid >> 6, tid, 0));
    __syncthreads();
    dbg_mark(cs, 28);
    // dgrad: Hbar_c[p][k] = sum_o Zbar_c[p][o] W_l[o][k], K = o in chunks of 64 rows (prefetched one ahead), k-block kq on
    // warpgroup kq -> channel c's accumulator columns
#pragma unroll 1
    for (int j = 0; j < nj; ++j) {
      if (tid == 0 && j + 1 < nj) tx_load_rows(cs, (j + 1) & 1, sS + ((j + 1) & 1) * SB, img, j + 1, nkq);
      tx_wait_ld(cs, j & 1);
      const uint32_t wb = sS + (j & 1) * SB;
#pragma unroll 1
      for (int c = 0; c < C; ++c)
#pragma unroll 1
        for (int kq = 0; kq < nkq; ++kq)
          x_chain<64, 0, 1>(kq, c >> 1, (c & 1) * kTxW + kq * 64, xdesc(sP + (c * 4 + j) * HB), xdesc(wb + kq * HB), 32, 2048,
                            4, j > 0 ? 1u : 0u);
      __syncthreads();
    }
    dbg_mark(cs, 29);
  }

  // ---- layer 0 reverse: Zbar^0 tiles, then  D[o][0..15] = Zbar_0^T [x | 1] + sum_j Zbar_(1+j)^T E_(dir1[j]) -----------------
  {
    float* gb0 = partial + net.b_off[0];
    float* gw0 = partial + net.w_off[0];
    constexpr bool kLo = (2 + N1) <= 4;         // a spare tile for the bf16 residual of the coordinates
    Tid ct;                                     // coord_tiles: threads 0..63 write rows 0..63
    ct.tid = tid < kTxPts ? tid : kTcPts; ct.p = tid & (kTxPts - 1);
    coord_tiles<N1>(ct, sS, x, pi.dir1, kLo);
    tx_l0_bwd_loop<N1, N2, PURE, AK>(t, sfp, sP, net.acts[0], pi.n1w, pi, x);
    tc::fence_async_smem();
    __syncthreads();
#pragma unroll 1
    for (int j = 0; j < (pi.n1w >> 6); ++j) {
      const uint32_t dcol = (j & 1) * kTxW;
      x_chain<16, 1, 1>(j, j >> 1, dcol, xdesc(sP + j * HB), tc::make_desc(sS, 0, 1024), 2048, 2048, kTxPts / 16, 0);
      if (kLo)
        x_chain<16, 1, 1>(j, j >> 1, dcol, xdesc(sP + j * HB), tc::make_desc(sS + (1 + N1) * kTileBytes, 0, 1024), 2048, 2048,
                          kTxPts / 16, 1);
#pragma unroll 1
      for (int jj = 0; jj < N1; ++jj)
        x_chain<16, 1, 1>(j, j >> 1, dcol, xdesc(sP + ((1 + jj) * 4 + j) * HB), tc::make_desc(sS + (1 + jj) * kTileBytes, 0, 1024),
                          2048, 2048, kTxPts / 16, 1);
    }
    __syncthreads();
    if (tid < pi.n1w) {
#pragma unroll
      for (int k = 0; k < PINN_MAX_IN; ++k)
        if (k < pi.d_in) atomicAdd(gw0 + tid + (long long)pi.n1w * k, xacc_at(tid >> 6, tid, k));
      atomicAdd(gb0 + tid, xacc_at(tid >> 6, tid, 8));
    }
  }
  __syncthreads();
  dbg_mark(cs, 30);
}

// ---- weight packing: theta (fp32, out x in column-major) -> bf16 swizzled images [kb][o / 128][128 rows][64 k] ----------
__global__ void __launch_bounds__(256) tx_pack_kernel(const TwPackArgs a) {
  const int img = blockIdx.x >> 5;
  const int idx = (blockIdx.x & 31) * 256 + threadIdx.x;     // 8192 16-byte chunks per image
  if (blockIdx.x == 0 && threadIdx.x == 0) *a.tile_counter = a.counter_init;
  if (img >= a.n_images) return;
  const DevNet& net = a.prob->nets[a.img_net[img]];
  const int l = a.img_layer[img];
  const int n_in = net.dims[l], n_out = net.dims[l + 1];
  const long long woff = net.w_off[l];
  const int blk = idx >> 10, row = (idx >> 3) & 127, kc = idx & 7;
  const int kb = blk >> 1, o = (blk & 1) * 128 + row;
  float w[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int k = kb * 64 + kc * 8 + e;
    w[e] = (o < n_out && k < n_in) ? __ldg(&a.theta[woff + o + (long long)n_out * k]) : 0.f;
  }
  uint4 h;
  h.x = tc::pack_bf16(w[0], w[1]); h.y = tc::pack_bf16(w[2], w[3]);
  h.z = tc::pack_bf16(w[4], w[5]); h.w = tc::pack_bf16(w[6], w[7]);
  *reinterpret_cast<uint4*>(a.wpack + (size_t)img * kTxImgBytes + (size_t)blk * TB + tc::swz_chunk(row, kc)) = h;
}

__global__ void __launch_bounds__(kTcThreads, 1) tx_loss_grad_kernel(const __grid_constant__ TwArgs args) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ TxShared cs;
  const int tid = threadIdx.x;
  const DevProblem* Pp = args.prob;
  const DevProblem& P = *Pp;
  const Misc ms = misc_of(smem + args.off_misc, args.mx_dim, args.mx_taps);
  float* partial = args.partial + (long long)blockIdx.x * args.partial_stride;
  const bool want_grad = (args.mode == 0);
  const DbgSpan span = dbg_span_begin(args.dbg);

  // ---- per-CTA setup --------------------------------------------------------------------------------------------------------
  if (tid == 0) {
    tc::mbar_init(ms.bar_ld, 1);            // collocation-tile bulk loads (own barrier: the weight stream uses cs.bar_ld[])
    for (int b = 0; b < 2; ++b) {
      tc::mbar_init(&cs.bar_ld[b], 1);
      cs.ph_ld[b] = 0;
    }
    tc::fence_barrier_init();
    cs.off_S = args.off_S; cs.off_nets = args.off_nets; cs.off_fp = args.off_fp[0]; cs.fp_net = -1;
    cs.theta = args.theta;
    cs.hstash = args.hstash + (long long)blockIdx.x * args.hstash_per_cta;
    cs.zstash = args.zstash + (long long)blockIdx.x * args.zstash_per_cta;
    cs.nch = (int)(args.hstash_per_cta / ((long long)(args.tl_max + 1) * SB));
    cs.wpack = args.wpack;
    for (int k = 0; k < PINN_MAX_NETS; ++k) cs.wimg[k] = args.wimg[k];
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
  tc::fence_async_smem();
  __syncthreads();
  dbg_mark(&cs, 2);
  uint32_t tile_ld_phase = 0;      // parity of the collocation-tile barrier (ms.bar_ld)

  for (int tile = args.tile_begin + blockIdx.x; tile < args.tile_end;) {
    const TileRef tr = stage_tile(args, P, ms, tile, tile_ld_phase);
    const DevTerm* tmp = &P.terms[tr.ti];
    const DevTerm& tm = *tmp;
    const int n_used = tm.n_used;
    dbg_mark(&cs, 3);

    for (int slot = 0; slot < n_used; ++slot) {
      const int k1 = tm.chan[slot].n1, k2 = tm.chan[slot].n2, pu = tm.chan[slot].pure;
      const int ak = args.net_ak[tm.used_net[slot]];
      for (int half = 0; half < 2; ++half)
        PINN_TC_DISPATCH(kTwMaxC, k1, k2, pu, ak, (tx_net_forward<A1, A2, PU, AK>(&cs, tmp, slot, half, want_grad ? 1 : 0)));
    }

    dbg_mark(&cs, 4);
    // S0 / S1 are idle between the sweeps
    residual_step(args, P, tm, ms, tr, smem + args.off_S, (size_t)(2 * SB), partial, want_grad);

    dbg_mark(&cs, 5);
    if (want_grad) {
      if (tid == 0) tc::bulk_wait0();             // operand-tile stash writes of this tile are complete before reloads
      __threadfence_block();
      __syncthreads();
      dbg_mark(&cs, 6);
      for (int slot = n_used - 1; slot >= 0; --slot) {
        const int k1 = tm.chan[slot].n1, k2 = tm.chan[slot].n2, pu = tm.chan[slot].pure;
        const int ak = args.net_ak[tm.used_net[slot]];
        for (int half = 0; half < 2; ++half)
          PINN_TC_DISPATCH(kTwMaxC, k1, k2, pu, ak, (tx_net_backward<A1, A2, PU, AK>(&cs, tmp, slot, half)));
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
cudaError_t tx_pack_launch(const TwPackArgs& a, cudaStream_t st) {
  tx_pack_kernel<<<(a.n_images > 0 ? a.n_images : 1) * 32, 256, 0, st>>>(a);
  return cudaGetLastError();
}

cudaError_t tx_launch(const TwArgs& a, int grid, size_t smem, cudaStream_t st) {
  return launch_fused_kernel<tx_loss_grad_kernel>(a, grid, kTcThreads, smem, st);
}

}  // namespace pinn
