// tc_kernel.cu -- fused PINN loss+gradient kernel, tensor-core path (sm_90a, wgmma).
//
// One CTA (512 threads = 4 warpgroups) owns a tile of 128 collocation points; a point is a row
// of every operand tile.  The hidden->hidden Dense
// layers run on the tensor cores (wgmma, bf16 operands from 128B-swizzled shared-memory tiles,
// fp32 accumulators); every derivative channel (value, d/dx_i, d2/dx_i dx_j) is its own
// 128-row M block that shares the same weight operand.  The epilogue (bias + activation +
// forward-mode tap chain rule, or its reverse) runs on the CUDA cores and re-packs the result as
// the next GEMM's bf16 operand tile straight from the wgmma register fragments (each warpgroup
// owns a 64-row x 32-column block of every channel).  The reverse sweep runs the tensor layers and layer 0 of the tile as
// two 64-point halves, one after the other, so that its MMAs stay in registers and the input adjoints handed to the next
// layer down stay in shared memory; the per-warpgroup gradient partials go through shared memory too.  Only the last
// layer's small gradient chains (last_layer_grad) still use the accumulator region of tc_prims.cuh.
//
//   forward, per tensor layer l :  D_c[128 x n_out] = H_c[128 x n_in] * W_l^T        (A, B K-major)
//   backward, per half and tensor layer l:  Z_c   (recompute, 16 columns per warpgroup) = H_c * W_l^T
//                                  Hbar_c^T[n_in x 64] = W_l^T * Zbar_c^T             (A MN-major; 16 points per warpgroup)
//                                  Wbar_l^T[n_in x n_out] = sum_c H_c^T * Zbar_c       (A, B MN-major; 16 points per warpgroup)
//                                  bbar_l[n_out]        = Zbar_0^T * 1                  (B = constant ones atom)
//   last layer                  :  wbar_L[n]            = sum_c H_c^T * ubar_c          (B = (hi, lo) pairs of ubar)
//   layer 0, per half           :  [Wbar_0 | bbar_0]^T  = Zbar^0_0^T [x | 1] + sum_j Zbar^0_(1+j)^T E_dir(j)
//
// The first (d -> n) and last (n -> 1) layers are tiny and stay on the CUDA cores inside the
// same epilogues.  Arithmetic modes: PINN_MODE_TC_BF16 (one MMA per product) and
// PINN_MODE_TC_SPLIT (forward operands split into bf16 hi + lo, three MMAs per product,
// which restores ~fp32 accuracy of the loss; the reverse sweep uses the hi parts).
//
// Replaces the same reference functions as the FFMA path (see ffma_kernel.cuh).
#include "tc_common.cuh"

namespace pinn {

using Fp = FpBlock<kTcW>;   // fp32 parameter block of a network

struct CtaShared : CtaBase {
  int split, off_Q;
  uint8_t* stash;
  TcNetSmem nets[PINN_MAX_NETS];
};

// ---- granule loops (4 columns x all channels per step), specialised on the activation kind -------------
// (inlined into the per-network passes; a noinline callee only gets the ABI scratch registers and spills)
struct LoopCtx {
  uint32_t fp;            // shared-memory address of the network's fp32 parameter block
  uint32_t bt;            // shared-memory address of the current tensor layer's bias
  uint32_t tP;            // shared-memory address of the hi operand tiles
  uint32_t tQ;            // shared-memory address of the lo operand tiles (forward split)
  float* gb;              // bias gradient of the current layer (CTA partial)
  float* gw;              // weight gradient of the first layer (CTA partial)
  int act, split, p, lane, g0, g1, flag;
  // ng granules of the layer, spread over the kNH warps of the thread's row quadrant
  __device__ __forceinline__ LoopCtx(uint32_t fp_, uint32_t bt_, uint32_t tP_, uint32_t tQ_, const Tid& t, int act_, int ng,
                                     int flag_, int split_ = 0, float* gb_ = nullptr, float* gw_ = nullptr)
      : fp(fp_), bt(bt_), tP(tP_), tQ(tQ_), gb(gb_), gw(gw_), act(act_), split(split_), p(t.p), lane(t.lane),
        g0(t.hh * (ng / kNH)), g1((t.hh + 1) * (ng / kNH)), flag(flag_) {}
};

// layer 0 forward: coordinates -> H^0 tiles (+ last-layer dot when there is no tensor layer: flag)
template <int N1, int N2, bool PURE, int AK>
__device__ __forceinline__ void l0_fwd_loop(const LoopCtx lc, const PassInfo<N1, N2> pi, const float* xp, float* up) {
  constexpr int C = 1 + N1 + N2;
  float x[PINN_MAX_IN], u[C];
#pragma unroll
  for (int k = 0; k < PINN_MAX_IN; ++k) x[k] = xp[k];
#pragma unroll
  for (int c = 0; c < C; ++c) u[c] = up[c];
#pragma unroll 1
  for (int g = lc.g0; g < lc.g1; ++g) {
    float h[C][GW];
#pragma unroll
    for (int i = 0; i < GW; i += 2) {
      float za[C], zb2[C];
      first_layer_elem<kTcW>(lc.fp, pi, x, g * GW + i, za);
      first_layer_elem<kTcW>(lc.fp, pi, x, g * GW + i + 1, zb2);
      P2 zz[C], hv[C];
#pragma unroll
      for (int c = 0; c < C; ++c) zz[c] = mk2(za[c], zb2[c]);
      chain_fwd<N1, N2, PURE, AK, P2>(lc.act, pi.ch, zz, hv);
#pragma unroll
      for (int c = 0; c < C; ++c) { h[c][i] = hv[c].v.x; h[c][i + 1] = hv[c].v.y; }
      if (lc.flag) {
        const float w0 = lds_f32(lc.fp + (Fp::WL + g * GW + i) * 4), w1 = lds_f32(lc.fp + (Fp::WL + g * GW + i + 1) * 4);
#pragma unroll
        for (int c = 0; c < C; ++c) u[c] = fmaf(w1, hv[c].v.y, fmaf(w0, hv[c].v.x, u[c]));
      }
    }
#pragma unroll
    for (int c = 0; c < C; ++c) store_half(lc.tP + c * kTileBytes, lc.tQ + c * kTileBytes, lc.p, g * GW, h[c], lc.split != 0);
  }
#pragma unroll
  for (int c = 0; c < C; ++c) up[c] = u[c];
}

// ---- register-resident forward of a tensor layer --------------------------------------------------------------------------
// Warpgroup wg owns the block rows [64 h, 64 h + 64) x columns [32 j, 32 j + 32) of the layer output, h = wg & 1,
// j = wg >> 1, for every channel: d[c] holds the m64n32k16 fragment of channel c (layout: tc::wg_chain).
// All four warpgroups issue the same instruction sequence, so the MMAs of a layer are spread evenly and stay in registers
// until the epilogue has consumed them.
// The block is 32 columns wide whatever the layer width: the weight tiles are zero beyond n_out, so a narrower layer
// gets zero pre-activations in the columns it does not have, and nothing reads them.  NK = n_in / 16 k-steps and the
// product count are compile-time, so the MMAs of the layer are one straight-line sequence (ptxas serializes wgmmas
// whose accumulators are carried around a loop).
template <int C, int NK, bool SPLIT>
__device__ __forceinline__ void fwd_mma(float (&d)[C][16], uint32_t sP, uint32_t sQ, uint32_t whi, uint32_t wlo) {
  const int wg = threadIdx.x >> 7;
  const uint32_t aoff = (wg & 1) * 8192u, boff = (wg >> 1) * 32u * 128u;
  const uint64_t dwhi = tc::make_desc(whi + boff, 0, 1024), dwlo = tc::make_desc(wlo + boff, 0, 1024);
  tc::wgmma_fence();
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const uint64_t dahi = tc::make_desc(sP + c * kTileBytes + aoff, 0, 1024);
    const uint64_t dalo = tc::make_desc(sQ + c * kTileBytes + aoff, 0, 1024);
    // the split products hi*hi, hi*lo, lo*hi accumulate into the same registers, in this order
#pragma unroll
    for (int pr = 0; pr < (SPLIT ? 3 : 1); ++pr) {
      const uint64_t a = (pr == 2) ? dalo : dahi, b = (pr == 1) ? dwlo : dwhi;
#pragma unroll
      for (int k = 0; k < NK; ++k)   // k-steps of 16 columns = 32 bytes = 2 descriptor units in both K-major operands
        tc::wgmma_n32<0, 0>(d[c], a + 2 * k, b + 2 * k, (pr | k) ? 1u : 0u);
    }
  }
  tc::wgmma_commit();
  tc::wgmma_wait0();
}
template <int C>
__device__ __forceinline__ void fwd_mma_any(float (&d)[C][16], uint32_t sP, uint32_t sQ, uint32_t whi, uint32_t wlo, int nk,
                                            bool split) {
  switch (nk * 2 + (split ? 1 : 0)) {   // pinn_create admits widths 16, 32, 48, 64 for this kernel
    case 2: fwd_mma<C, 1, false>(d, sP, sQ, whi, wlo); break;
    case 3: fwd_mma<C, 1, true>(d, sP, sQ, whi, wlo); break;
    case 4: fwd_mma<C, 2, false>(d, sP, sQ, whi, wlo); break;
    case 5: fwd_mma<C, 2, true>(d, sP, sQ, whi, wlo); break;
    case 6: fwd_mma<C, 3, false>(d, sP, sQ, whi, wlo); break;
    case 7: fwd_mma<C, 3, true>(d, sP, sQ, whi, wlo); break;
    case 8: fwd_mma<C, 4, false>(d, sP, sQ, whi, wlo); break;
    default: fwd_mma<C, 4, true>(d, sP, sQ, whi, wlo); break;
  }
}

// tensor layer forward epilogue on the fragments of fwd_mma: bias + activation chain -> next operand tiles (hi in P,
// lo in Q); for the last hidden layer (flag) the last-layer dot products of the block's rows are summed over the quad
// of lanes that share a row and added to ms.scratch (two column warpgroups per row)
template <int N1, int N2, bool PURE, int AK, int C>
__device__ __forceinline__ void tl_fwd_frag(const float (&d)[C][16], const LoopCtx lc, const Chan<N1, N2> ch, float* scratch) {
  const int wg = threadIdx.x >> 7, w = (threadIdx.x >> 5) & 3;
  const int row0 = 64 * (wg & 1) + 16 * w + (lc.lane >> 2);
  const int col0 = 32 * (wg >> 1) + 2 * (lc.lane & 3);
  float u[2][C];
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int c = 0; c < C; ++c) u[r][c] = 0.f;
#pragma unroll
  for (int i = 0; i < 16; i += 2) {
    const int rh = (i >> 1) & 1;
    const int row = row0 + 8 * rh, col = col0 + 8 * (i >> 2);
    P2 zz[C], hv[C];
    zz[0] = mk2(d[0][i] + lds_f32(lc.bt + col * 4), d[0][i + 1] + lds_f32(lc.bt + (col + 1) * 4));
#pragma unroll
    for (int c = 1; c < C; ++c) zz[c] = mk2(d[c][i], d[c][i + 1]);
    chain_fwd<N1, N2, PURE, AK, P2>(lc.act, ch, zz, hv);
    const uint32_t off = tc::swz_off(row, col);
#pragma unroll
    for (int c = 0; c < C; ++c) {
      const uint32_t hx = tc::pack_bf16(hv[c].v.x, hv[c].v.y);
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(lc.tP + c * kTileBytes + off), "r"(hx) : "memory");
      if (lc.split)
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(lc.tQ + c * kTileBytes + off), "r"(bf16x2_lo(hv[c].v.x, hv[c].v.y, hx))
                     : "memory");
    }
    if (lc.flag) {
      const float w0 = lds_f32(lc.fp + (Fp::WL + col) * 4), w1 = lds_f32(lc.fp + (Fp::WL + col + 1) * 4);
#pragma unroll
      for (int c = 0; c < C; ++c) u[rh][c] = fmaf(w1, hv[c].v.y, fmaf(w0, hv[c].v.x, u[rh][c]));
    }
  }
  if (lc.flag) {
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
      for (int c = 0; c < C; ++c) {
        float s = u[r][c];
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        s += __shfl_xor_sync(0xffffffffu, s, 2);
        if ((lc.lane & 3) == 0) atomicAdd(&scratch[c * kTcPts + row0 + 8 * r], s);
      }
  }
}

// ---- register-resident reverse of a tensor layer, one 64-point half of the tile at a time --------------------------------------
// The reverse sweep runs the tensor layers of the tile as two independent halves (points 64 h .. 64 h + 63), each through
// every tensor layer before the next starts, so that the input adjoints of a layer fit in shared memory: per channel c, Q holds the
// tile pair at Q + c * kTileBytes = the half's reloaded input rows H_c (8 KB, 64 rows) followed by its Zbar_c (8 KB), and P
// holds the half's Hbar in fp32 (C x 16 KB, layout hb_idx).  Every warpgroup takes 16 points or 16 columns of the half:
//   recompute: Z_c[p][o]  = sum_k H_c[p][k] W_l[o][k]           A = H_c K-major (the 64 rows), B = W_l K-major (16 columns)
//   dgrad    : Hbar_c^T[k][p] = sum_o W_l[o][k] Zbar_c[p][o]     A = W_l MN-major (M = the 64 input columns), B = Zbar_c K-major
//   wgrad    : Wbar_l^T[k][o] = sum_c sum_p H_c[p][k] Zbar_c[p][o]   A = H_c MN-major, B = Zbar_c MN-major; partial over 16 points
//   bias     : bbar_l[o] = sum_p Zbar_0[p][o]                    A = Zbar_0 MN-major, B = the constant ones atom
// Each is one straight-line sequence with one commit / wait, on all four warpgroups (NK, NKO = k-steps: compile-time).
constexpr uint32_t kHalfBytes = kTileBytes / 2;

// recompute of the half: warpgroup wg owns its 64 rows x columns [16 wg, 16 wg + 16) for every channel (m64n16 fragments,
// layout: tc::wg_chain); the k order of fwd_mma, so Z is the forward's to the bit
template <int C, int NK>
__device__ __forceinline__ void rec_mma(float (&d)[C][8], uint32_t sQ, uint32_t whi) {
  const uint64_t dw = tc::make_desc(whi + (threadIdx.x >> 7) * 16u * 128u, 0, 1024);
  tc::wgmma_fence();
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const uint64_t da = tc::make_desc(sQ + c * kTileBytes, 0, 1024);
#pragma unroll
    for (int k = 0; k < NK; ++k) tc::wgmma_n16<0, 0>(d[c], da + 2 * k, dw + 2 * k, k ? 1u : 0u);
  }
  tc::wgmma_commit();
  tc::wgmma_wait0();
}
template <int C>
__device__ __forceinline__ void rec_mma_any(float (&d)[C][8], uint32_t sQ, uint32_t whi, int nk) {
  switch (nk) {
    case 1: rec_mma<C, 1>(d, sQ, whi); break;
    case 2: rec_mma<C, 2>(d, sQ, whi); break;
    case 3: rec_mma<C, 3>(d, sQ, whi); break;
    default: rec_mma<C, 4>(d, sQ, whi); break;
  }
}
template <int C, int NKO>
__device__ __forceinline__ void dgrad_mma(float (&d)[C][8], uint32_t sQ, uint32_t whi) {
  const uint32_t poff = kHalfBytes + (threadIdx.x >> 7) * 16u * 128u;
  const uint64_t dw = tc::make_desc(whi, 0, 1024);
  tc::wgmma_fence();
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const uint64_t dz = tc::make_desc(sQ + c * kTileBytes + poff, 0, 1024);
#pragma unroll
    for (int k = 0; k < NKO; ++k)   // k-step of 16 output neurons: 16 rows (2048 bytes) of W, 32 bytes of the Zbar rows
      tc::wgmma_n16<1, 0>(d[c], dw + 128 * k, dz + 2 * k, k ? 1u : 0u);
  }
  tc::wgmma_commit();
  tc::wgmma_wait0();
}
template <int C>
__device__ __forceinline__ void dgrad_mma_any(float (&d)[C][8], uint32_t sQ, uint32_t whi, int nko) {
  switch (nko) {
    case 1: dgrad_mma<C, 1>(d, sQ, whi); break;
    case 2: dgrad_mma<C, 2>(d, sQ, whi); break;
    case 3: dgrad_mma<C, 3>(d, sQ, whi); break;
    default: dgrad_mma<C, 4>(d, sQ, whi); break;
  }
}
template <int C>
__device__ __forceinline__ void wgrad_mma(float (&dw)[32], float (&db)[8], uint32_t sQ, uint32_t s_ones) {
  const uint32_t poff = (threadIdx.x >> 7) * 16u * 128u;
  const uint64_t d1 = tc::make_desc(s_ones, 0, 0);   // SBO = 0: every 8-point group of K reads the same ones atom
  tc::wgmma_fence();
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const uint64_t dh = tc::make_desc(sQ + c * kTileBytes + poff, 0, 1024);
    const uint64_t dz = tc::make_desc(sQ + c * kTileBytes + kHalfBytes + poff, 0, 1024);
    tc::wgmma_n64<1, 1>(dw, dh, dz, c ? 1u : 0u);
  }
  tc::wgmma_n16<1, 1>(db, tc::make_desc(sQ + kHalfBytes + poff, 0, 1024), d1, 0u);
  tc::wgmma_commit();
  tc::wgmma_wait0();
}

// layer-0 weight / bias gradient of the half, 16 points (one k-step) per warpgroup, as one m64n16 fragment (row = neuron o
// of the first layer, column = input k, 8 = the bias): D = Zbar^0_0^T [x_hi | 1] (+ Zbar^0_0^T [x_lo | 0]) +
// sum_j Zbar^0_(1+j)^T E_dir(j), in layer0_grad's product order.  Per channel tile of Q: the Zbar half holds Zbar^0_c
// (c <= N1, MN-major, M = the 64 neurons), the H half the coordinate tile of the same index (coord_row; the x_lo tile at
// 1 + N1 when N2 > 0).
template <int N1, int N2>
__device__ __forceinline__ void l0_mma(float (&d)[8], uint32_t sQ) {
  const uint32_t poff = (threadIdx.x >> 7) * 16u * 128u;
  const uint64_t dz0 = tc::make_desc(sQ + kHalfBytes + poff, 0, 1024);
  tc::wgmma_fence();
  tc::wgmma_n16<1, 1>(d, dz0, tc::make_desc(sQ + poff, 0, 1024), 0u);
  if (N2 > 0) tc::wgmma_n16<1, 1>(d, dz0, tc::make_desc(sQ + (1 + N1) * kTileBytes + poff, 0, 1024), 1u);
#pragma unroll
  for (int j = 0; j < N1; ++j)
    tc::wgmma_n16<1, 1>(d, tc::make_desc(sQ + (1 + j) * kTileBytes + kHalfBytes + poff, 0, 1024),
                        tc::make_desc(sQ + (1 + j) * kTileBytes + poff, 0, 1024), 1u);
  tc::wgmma_commit();
  tc::wgmma_wait0();
}

// Hbar of the half in P: element (channel c, input column k, point p of the half) at hb_idx.  The point index is XORed in its
// bits 3-4 with two bits of k, so that the dgrad fragment stores (8-byte pairs of points, rows k of a quad) and the epilogue
// loads (8 consecutive points x 4 columns k = 8 m + 2 j (+1)) both touch 32 distinct banks.
__device__ __forceinline__ int hb_idx(int c, int k, int p) { return (c * 64 + k) * 64 + (p ^ ((((k >> 1) ^ k) & 3) << 3)); }

// store the dgrad fragments (rows = input column k, columns = the warpgroup's 16 points) as the half's Hbar
template <int C>
__device__ __forceinline__ void hbar_store(float* hbar, const float (&d)[C][8]) {
  const int wg = threadIdx.x >> 7, w = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
#pragma unroll
  for (int c = 0; c < C; ++c)
#pragma unroll
    for (int i = 0; i < 8; i += 2) {
      const int k = 16 * w + (lane >> 2) + 8 * ((i >> 1) & 1), p = 16 * wg + 8 * (i >> 2) + 2 * (lane & 3);
      *reinterpret_cast<float2*>(hbar + hb_idx(c, k, p)) = make_float2(d[c][i], d[c][i + 1]);
    }
}

// store the m64nNk16 fragment d of this warpgroup (layout: tc::wg_chain) as rows of a row-major fp32 array: element
// (row r, column n) at base[r * ld + n].  The lanes of a pair swap half of their values so that each holds four
// consecutive columns of one row: one 16-byte store per 8-column block, and a quad writes 32 contiguous bytes of two rows.
template <int NF>
__device__ __forceinline__ void frag_store_rows(float* base, int ld, const float (&d)[NF]) {
  const int w = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const bool odd = (lane & 1) != 0;
  float* row = base + (16 * w + (lane >> 2) + (odd ? 8 : 0)) * ld + 4 * ((lane >> 1) & 1);
#pragma unroll
  for (int j = 0; j < NF / 4; ++j) {
    const float r0 = __shfl_xor_sync(0xffffffffu, odd ? d[4 * j] : d[4 * j + 2], 1);
    const float r1 = __shfl_xor_sync(0xffffffffu, odd ? d[4 * j + 1] : d[4 * j + 3], 1);
    *reinterpret_cast<float4*>(row + 8 * j) =
        odd ? make_float4(r0, r1, d[4 * j + 2], d[4 * j + 3]) : make_float4(d[4 * j], d[4 * j + 1], r0, r1);
  }
}

// tensor layer backward epilogue of half h on the fragments of rec_mma: bias + adjoint chain -> Zbar tiles (bf16 hi) in Q.
// The output adjoints come from the half's Hbar in P (the dgrad of the layer above), or for the last hidden layer (flag) are
// w_last[column] * ubar_c[point], with ubar_c[point] at ubs[c * kTcPts + point].  Columns beyond n_out get Zbar = 0 (zero
// weights, bias and adjoints).
template <int N1, int N2, bool PURE, int AK, int C>
__device__ __forceinline__ void tl_bwd_frag(const float (&d)[C][8], const LoopCtx lc, const Chan<N1, N2> ch, const float* ubs,
                                            const float* hbar, int h) {
  const int wg = threadIdx.x >> 7, w = (threadIdx.x >> 5) & 3;
  const int row0 = 16 * w + (lc.lane >> 2);
  const int col0 = 16 * wg + 2 * (lc.lane & 3);
#pragma unroll
  for (int i = 0; i < 8; i += 2) {
    const int row = row0 + 8 * ((i >> 1) & 1), col = col0 + 8 * (i >> 2);
    P2 zz[C], hv[C], zv[C];
    zz[0] = mk2(d[0][i] + lds_f32(lc.bt + col * 4), d[0][i + 1] + lds_f32(lc.bt + (col + 1) * 4));
#pragma unroll
    for (int c = 1; c < C; ++c) zz[c] = mk2(d[c][i], d[c][i + 1]);
    if (lc.flag) {
      const float w0 = lds_f32(lc.fp + (Fp::WL + col) * 4), w1 = lds_f32(lc.fp + (Fp::WL + col + 1) * 4);
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const float u = ubs[c * kTcPts + 64 * h + row];
        hv[c] = mk2(w0 * u, w1 * u);
      }
    } else {
#pragma unroll
      for (int c = 0; c < C; ++c) hv[c] = mk2(hbar[hb_idx(c, col, row)], hbar[hb_idx(c, col + 1, row)]);
    }
    chain_bwd<N1, N2, PURE, AK, P2>(lc.act, ch, zz, hv, zv);
    const uint32_t off = kHalfBytes + tc::swz_off(row, col);
#pragma unroll
    for (int c = 0; c < C; ++c)
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(lc.tQ + c * kTileBytes + off), "r"(tc::pack_bf16(zv[c].v.x, zv[c].v.y))
                   : "memory");
  }
}

// layer 0 backward of a half, tensor-core variant: the half's Hbar^0 in P (layout hb_idx) -> Zbar^0 (value + first-derivative
// channels; bf16 hi) in the Zbar half of Q's channel tiles, row = point of the half.  The thread takes point lc.p of the half
// and granules [lc.g0, lc.g1).  The weight / bias gradient is then one small MMA against the augmented coordinate tiles
// (l0_mma), so no cross-lane reductions are needed here.
template <int N1, int N2, bool PURE, int AK>
__device__ __forceinline__ void l0_bwd_store_loop(const LoopCtx lc, const PassInfo<N1, N2> pi, const float (&x)[PINN_MAX_IN],
                                                  const float* hbar) {
  constexpr int C = 1 + N1 + N2;
#pragma unroll 1
  for (int g = lc.g0; g < lc.g1; ++g) {
    float hb[C][GWB];
#pragma unroll
    for (int c = 0; c < C; ++c)
#pragma unroll
      for (int i = 0; i < GWB; ++i) hb[c][i] = hbar[hb_idx(c, g * GWB + i, lc.p)];
#pragma unroll
    for (int i = 0; i < GWB; i += 2) {
      float za[C], zb2[C];
      first_layer_elem<kTcW>(lc.fp, pi, x, g * GWB + i, za);
      first_layer_elem<kTcW>(lc.fp, pi, x, g * GWB + i + 1, zb2);
      P2 zz[C], hv[C], zv[C];
#pragma unroll
      for (int c = 0; c < C; ++c) { zz[c] = mk2(za[c], zb2[c]); hv[c] = mk2(hb[c][i], hb[c][i + 1]); }
      chain_bwd<N1, N2, PURE, AK, P2>(lc.act, pi.ch, zz, hv, zv);
#pragma unroll
      for (int c = 0; c <= N1; ++c) { hb[c][i] = zv[c].v.x; hb[c][i + 1] = zv[c].v.y; }
    }
#pragma unroll
    for (int c = 0; c <= N1; ++c) store_half(lc.tQ + c * kTileBytes + kHalfBytes, lc.tQ, lc.p, g * GWB, hb[c], false);
  }
}

// layer 0 backward of a network without tensor layers: adjoints of H^0 (w_last * ubar) -> first-layer weight / bias gradient
template <int N1, int N2, bool PURE, int AK>
__device__ __forceinline__ void l0_bwd_loop(const LoopCtx lc, const PassInfo<N1, N2> pi, const float* xp, const float* ubp) {
  constexpr int C = 1 + N1 + N2;
  float x[PINN_MAX_IN], ub[C];
#pragma unroll
  for (int k = 0; k < PINN_MAX_IN; ++k) x[k] = xp[k];
#pragma unroll
  for (int c = 0; c < C; ++c) ub[c] = ubp[c];
  const int re = reduceg_elem(lc.lane);
  const bool rlead = reduceg_lead(lc.lane);
  const int n1w = pi.n1w;
#pragma unroll 1
  for (int g = lc.g0; g < lc.g1; ++g) {
    float hb[C][GW];
#pragma unroll
    for (int i = 0; i < GW; ++i) {
      const float wl = lds_f32(lc.fp + (Fp::WL + g * GW + i) * 4);
#pragma unroll
      for (int c = 0; c < C; ++c) hb[c][i] = wl * ub[c];
    }
    float zv0[GW], zvd[N1 > 0 ? N1 : 1][GW];
#pragma unroll
    for (int i = 0; i < GW; ++i) {
      // scalar here: the packed form raises the register pressure of this loop past the 128-register budget
      float zz[C], hv[C], zv[C];
      first_layer_elem<kTcW>(lc.fp, pi, x, g * GW + i, zz);
#pragma unroll
      for (int c = 0; c < C; ++c) hv[c] = hb[c][i];
      chain_bwd<N1, N2, PURE, AK, float>(lc.act, pi.ch, zz, hv, zv);
      zv0[i] = zv[0];
#pragma unroll
      for (int jd = 0; jd < N1; ++jd) zvd[jd][i] = zv[1 + jd];
    }
    // Wbar_0[o][k] = sum_p zbar_0 x_k + zbar_(channel of direction k);  bbar_0[o] = sum_p zbar_0
    const float bs = warp_reduceg(zv0, lc.lane);
    if (rlead) atomicAdd(lc.gb + g * GW + re, bs);
#pragma unroll
    for (int k = 0; k < PINN_MAX_IN; ++k) {
      if (k < pi.d_in) {
        float gk[GW];
#pragma unroll
        for (int i = 0; i < GW; ++i) {
          float gg = zv0[i] * x[k];
#pragma unroll
          for (int jd = 0; jd < N1; ++jd) gg += (pi.dir1[jd] == k) ? zvd[jd][i] : 0.f;
          gk[i] = gg;
        }
        const float gs = warp_reduceg(gk, lc.lane);
        if (rlead) atomicAdd(lc.gw + g * GW + re + (long long)n1w * k, gs);
      }
    }
  }
}

// layer 0 of the reverse sweep for half h (points 64 h .. 64 h + 63) of a network with tensor layers, on the half's Hbar^0 in
// P (layout hb_idx): the augmented-coordinate tiles go to the H halves of Q (no layer below reloads it) -> barrier -> Zbar^0 by
// the CUDA cores into the Zbar halves of Q -> barrier -> l0_mma, whose per-warpgroup fragments go to P -> barrier -> each
// element of W_0 / b_0 is summed in warpgroup order by one thread, which adds it to the CTA partial (as for the tensor layers).
// A call of its own: inlined into net_backward, the step faulted on the H100 when CUDA 12.9 built it with every dispatch
// instantiation in the unit (built for fewer instantiations, the same code ran correctly).  CTA-wide.
template <int N1, int N2, bool PURE, int AK>
__device__ __noinline__ void l0_half(uint32_t fpa, uint8_t* tP, uint8_t* tQ, int act0, const PassInfo<N1, N2> pi, const float* xs,
                                     const int* rows, int h, float* gw0, float* gb0) {
  const Tid t = tid_of();
  const int tid = t.tid, wg = tid >> 7;
  const uint32_t sP = tc::smem_u32(tP), sQ = tc::smem_u32(tQ);
  const float* hbar = reinterpret_cast<const float*>(tP);     // [c][k][point] (hb_idx)
  float* lpart = reinterpret_cast<float*>(tP);                // [wg][o][16] (column k of W_0, 8 = b_0)
  {
    // the thread's point of the half, and an eighth of the layer's granules (n1w is a multiple of 16)
    const int pl = 32 * (t.warp & 1) + t.lane, ng = pi.n1w / (8 * GWB);
    float x[PINN_MAX_IN];
#pragma unroll
    for (int k = 0; k < PINN_MAX_IN; ++k) x[k] = (k < pi.d_in) ? xs[rows[k] * kTcPts + 64 * h + pl] : 0.f;
    // coordinate tiles 0 .. N1 (and 1 + N1, the lo of x, when N2 > 0: C >= 2 + N1 tiles) in the H halves of Q
    if (tid < 64) coord_row<N1>(sQ, pl, x, pi.dir1, N2 > 0);
    __syncthreads();   // Hbar^0 of the half is in P
    LoopCtx lc(fpa, fpa, sP, sQ, t, act0, 0, 0);
    lc.p = pl;
    lc.g0 = (t.warp >> 1) * ng;
    lc.g1 = lc.g0 + ng;
    l0_bwd_store_loop<N1, N2, PURE, AK>(lc, pi, x, hbar);
  }
  tc::fence_async_smem();   // Zbar^0 and the coordinate tiles (generic-proxy stores to Q) -> l0_mma
  __syncthreads();
  {
    float d[8];
    l0_mma<N1, N2>(d, sQ);
    frag_store_rows(lpart + wg * 64 * 16, 16, d);   // Zbar^0 has read Hbar^0 in P
  }
  __syncthreads();
  const int n1w = pi.n1w, d_in = pi.d_in;
#pragma unroll 1
  for (int e = tid; e < 64 * 16; e += kTcThreads) {
    const int o = e >> 4, k = e & 15;
    if (o < n1w && (k < d_in || k == 8)) {
      float* g = (k == 8) ? gb0 + o : gw0 + o + (long long)n1w * k;
      *g += ((lpart[e] + lpart[1024 + e]) + lpart[2048 + e]) + lpart[3072 + e];
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// forward of one network for the current tile, channel structure <N1, N2, PURE>.
// `phase` bit 1 = parity of the bulk-load barrier (bit 0 unused); returned updated.
template <int N1, int N2, bool PURE, int AK>
__device__ __noinline__ uint32_t net_forward(CtaShared* cs, const DevProblem* Pp, const DevTerm* tmp, int slot,
                                             int want_grad, uint32_t phase) {
  extern __shared__ __align__(1024) uint8_t smem[];
  constexpr int C = 1 + N1 + N2;
  const DevTerm& tm = *tmp;
  const int net_id = tm.used_net[slot];
  const DevNet& net = Pp->nets[net_id];
  const DevChan& dc = tm.chan[slot];
  const TcNetSmem ns = cs->nets[net_id];
  const float* fp = reinterpret_cast<const float*>(smem + ns.fp);
  uint8_t* tP = smem + cs->off_P;
  uint8_t* tQ = smem + cs->off_Q;
  const Misc ms = misc_of(smem + cs->off_misc, cs->mx_dim, cs->mx_taps);
  const bool split = cs->split != 0;
  PassInfo<N1, N2> pi;
  load_pass<N1, N2>(pi, net, dc);
  const int TL = pi.TL;
  const Tid t = tid_of();
  const int tid = t.tid, p = t.p;
  float x[PINN_MAX_IN];
#pragma unroll
  for (int k = 0; k < PINN_MAX_IN; ++k) x[k] = (k < pi.d_in) ? ms.Xs[dc.rows[k] * kTcPts + p] : 0.f;
  uint8_t* stash_slot = cs->stash + (size_t)slot * cs->tl_max * kTcMaxC * kTileBytes;

  dbg_mark(cs, 10);
  float u[C];                                   // last-layer partial dot products of this thread
#pragma unroll
  for (int c = 0; c < C; ++c) u[c] = 0.f;
  // the cross-warp combination of u goes through shared-memory atomics (finish_forward)
  if (tid < C * kTcPts / 4) reinterpret_cast<float4*>(ms.scratch)[tid] = make_float4(0.f, 0.f, 0.f, 0.f);
  {
    // ---- layer 0 on the CUDA cores ------------------------------------------------------------------
    const LoopCtx lc(tc::smem_u32(fp), tc::smem_u32(fp), tc::smem_u32(tP), tc::smem_u32(tQ), t, net.acts[0], pi.n1w / GW, TL == 0, split);
    l0_fwd_loop<N1, N2, PURE, AK>(lc, pi, x, u);
  }
  // ---- tensor layers -------------------------------------------------------------------------------------
  for (int l = 1; l <= TL; ++l) {
    const int n_in = net.dims[l], n_out = net.dims[l + 1];
    const int act = net.acts[l];
    tc::fence_async_smem();
    __syncthreads();
    dbg_mark(cs, 11);
    if (want_grad && tid == 0) {
      // stash this layer's input tiles for the reverse sweep (the bulk copies read P while the MMAs run)
      for (int c = 0; c < C; ++c)
        tc::bulk_store(stash_slot + (size_t)(l - 1) * kTcMaxC * kTileBytes + (size_t)c * kTileBytes, tP + c * kTileBytes, kTileBytes);
      tc::bulk_commit();
    }
    float d[C][16];
    {
      const uint32_t sP = tc::smem_u32(tP), sQ = tc::smem_u32(tQ);
      const uint32_t whi = tc::smem_u32(smem + ns.w_hi[l - 1]), wlo = tc::smem_u32(smem + ns.w_lo[l - 1]);
      const int nk = n_in / 16;
      fwd_mma_any<C>(d, sP, sQ, whi, wlo, nk, split);
    }
    dbg_mark(cs, 13);
    // the epilogue overwrites rows of P / Q that the other warpgroup of the row half, and the stash copies, may still read
    if (want_grad && tid == 0) tc::bulk_wait_read0();   // stash copies have finished reading P (same thread issued them)
    __syncthreads();
    dbg_mark(cs, 14);
    const LoopCtx lc(tc::smem_u32(fp), tc::smem_u32(fp) + (Fp::BT + (l - 1) * 64) * 4, tc::smem_u32(tP), tc::smem_u32(tQ), t, act, 0, l == TL, split);
    tl_fwd_frag<N1, N2, PURE, AK, C>(d, lc, pi.ch, ms.scratch);
  }
  // ---- last layer (n -> 1, identity): combine the column parts of every point ---------------------------------
  finish_forward<C>(cs, tm, slot, ms, fp + Fp::BL, t, u);
  return phase;
}

// reverse sweep of one network for the current tile
template <int N1, int N2, bool PURE, int AK>
__device__ __noinline__ uint32_t net_backward(CtaShared* cs, const DevProblem* Pp, const DevTerm* tmp, int slot,
                                              uint32_t phase) {
  extern __shared__ __align__(1024) uint8_t smem[];
  constexpr int C = 1 + N1 + N2;
  const DevTerm& tm = *tmp;
  const int net_id = tm.used_net[slot];
  const DevNet& net = Pp->nets[net_id];
  const DevChan& dc = tm.chan[slot];
  const TcNetSmem ns = cs->nets[net_id];
  const float* fp = reinterpret_cast<const float*>(smem + ns.fp);
  uint8_t* tP = smem + cs->off_P;
  uint8_t* tQ = smem + cs->off_Q;
  const Misc ms = misc_of(smem + cs->off_misc, cs->mx_dim, cs->mx_taps);
  float* partial = cs->partial;
  PassInfo<N1, N2> pi;
  load_pass<N1, N2>(pi, net, dc);
  const int L = pi.L, TL = pi.TL;
  const Tid t = tid_of();
  const int tid = t.tid, p = t.p, wg = tid >> 7;
  uint32_t ld_phase = (phase >> 1) & 1u;
  uint8_t* stash_slot = cs->stash + (size_t)slot * cs->tl_max * kTcMaxC * kTileBytes;
  const uint32_t sP = tc::smem_u32(tP), sQ = tc::smem_u32(tQ);

  dbg_mark(cs, 20);
  float ub[C];
  gather_ubar<C>(tm, slot, ms, p, ub);
  // the last hidden layer's epilogue reads ubar by fragment row (published by the barriers of last_layer_grad)
  if (t.hh == 0) {
#pragma unroll
    for (int c = 0; c < C; ++c) ms.scratch[c * kTcPts + p] = ub[c];
  }
  // ---- last layer: the ubar tile goes to Q, the products into accumulator columns Y ----------------------------------------
  last_layer_grad<C>(t, ub, pi.nL, partial + net.w_off[L - 1], partial + net.b_off[L - 1], sQ, sP, kTileBytes, 0u, TM_Y, kTcW);

  const int act0 = net.acts[0];
  float* gb0 = partial + net.b_off[0];
  float* gw0 = partial + net.w_off[0];
  if (TL == 0) {
    // ---- no tensor layer: layer 0 on the CUDA cores (warp reduce-scatter + atomics) -----------------------------------------
    __syncthreads();
    dbg_mark(cs, 29);
    float x[PINN_MAX_IN];
#pragma unroll
    for (int k = 0; k < PINN_MAX_IN; ++k) x[k] = (k < pi.d_in) ? ms.Xs[dc.rows[k] * kTcPts + p] : 0.f;
    const LoopCtx lc(tc::smem_u32(fp), tc::smem_u32(fp), sP, sQ, t, act0, pi.n1w / GW, 1, 0, gb0, gw0);
    l0_bwd_loop<N1, N2, PURE, AK>(lc, pi, x, ub);
  }

  // ---- tensor layers, last to first, then layer 0: one 64-point half of the tile after the other -------------------------------
  // Per layer: the stash reload of the half's H^{l-1} in Q has landed -> recompute -> barrier (the half's Hbar^l in P is
  // complete) -> Zbar epilogue into Q -> barrier -> wgrad, whose four per-warpgroup partials of Wbar_l^T go to the first four
  // tiles of P (plan.cu gives P at least four: every epilogue has read Hbar^l), then dgrad, whose fragments stay in registers
  // -> barrier (every MMA has read Q) -> the bias partials go to the Zbar half of Q's first tile and the reload of H^{l-2}
  // to Q -> barrier -> each gradient element is summed in warpgroup order by one thread, which adds it to the CTA partial
  // (half 0 before half 1, so the result does not depend on scheduling) -> barrier -> the dgrad fragments become Hbar^{l-1}
  // in P.  Generic-proxy stores to P and Q after async-proxy reads that have completed need no proxy fence; the fence before
  // the MMAs orders the Zbar stores before them.
  // Then layer 0 of the half (l0_half).
  float* hbar = reinterpret_cast<float*>(tP);                 // [c][k][point] (hb_idx), C x 16 KB
  float* wpart = reinterpret_cast<float*>(tP);                // [wg][k][o] (4 x 64 x 64)
  float* bpart = reinterpret_cast<float*>(tQ + kHalfBytes);   // [wg][o]
#pragma unroll 1
  for (int h = 0; h < (TL > 0 ? 2 : 0); ++h) {
    for (int l = TL; l >= 1; --l) {
      const int n_in = net.dims[l], n_out = net.dims[l + 1];
      const int act = net.acts[l];
      float* gb = partial + net.b_off[l];
      float* gw = partial + net.w_off[l];
      const float* bt = fp + Fp::BT + (l - 1) * 64;
      const uint32_t whi = tc::smem_u32(smem + ns.w_hi[l - 1]);
      dbg_mark(cs, 21);
      if (tid == 0 && l == TL) {
        // reload the half's rows of this layer's input tiles H^{l-1} (bf16 hi) from the stash into Q: the MMAs that read Q
        // before (last_layer_grad's ubar tile, the previous half's l0_mma) have been waited for.  The layers below are
        // reloaded by the layer above them.
        const uint8_t* src = stash_slot + (size_t)(l - 1) * kTcMaxC * kTileBytes + h * kHalfBytes;
        tc::mbar_arrive_expect_tx(ms.bar_ld, C * kHalfBytes);
        for (int c = 0; c < C; ++c) tc::bulk_load(tQ + c * kTileBytes, src + (size_t)c * kTileBytes, kHalfBytes, ms.bar_ld);
      }
      wait_bar(ms.bar_ld, ld_phase);
      dbg_mark(cs, 22);
      {
        float d[C][8];
        rec_mma_any<C>(d, sQ, whi, n_in / 16);
        __syncthreads();
        dbg_mark(cs, 24);
        const LoopCtx lc(tc::smem_u32(fp), tc::smem_u32(bt), sP, sQ, t, act, 0, l == TL);
        tl_bwd_frag<N1, N2, PURE, AK, C>(d, lc, pi.ch, ms.scratch, hbar, h);
      }
      tc::fence_async_smem();   // Zbar (generic-proxy stores to Q) -> the dgrad / wgrad MMAs (async proxy)
      __syncthreads();
      dbg_mark(cs, 26);
      float db0, db2;
      {
        float dw[32], db[8];
        wgrad_mma<C>(dw, db, sQ, tc::smem_u32(smem + cs->off_ones));
        frag_store_rows(wpart + wg * 64 * 64, 64, dw);
        db0 = db[0]; db2 = db[2];   // column 0 of the bias product: rows 16 w + lane / 4 (+ 8) of lanes 0, 4, ..., 28
      }
      float d[C][8];
      dgrad_mma_any<C>(d, sQ, whi, n_out / 16);
      __syncthreads();
      dbg_mark(cs, 27);
      if (tid == 0 && l > 1) {
        // the half's input tiles H^{l-2} of the next layer down travel into Q while the gradient sum below runs
        const uint8_t* src = stash_slot + (size_t)(l - 2) * kTcMaxC * kTileBytes + h * kHalfBytes;
        tc::mbar_arrive_expect_tx(ms.bar_ld, C * kHalfBytes);
        for (int c = 0; c < C; ++c) tc::bulk_load(tQ + c * kTileBytes, src + (size_t)c * kTileBytes, kHalfBytes, ms.bar_ld);
      }
      if ((t.lane & 3) == 0) {
        const int o = 16 * (t.warp & 3) + (t.lane >> 2);
        bpart[wg * 64 + o] = db0;
        bpart[wg * 64 + o + 8] = db2;
      }
      __syncthreads();
      dbg_mark(cs, 28);
      // owner-thread read-add-write: element (k, o) belongs to one thread in both halves and in every tile
      if ((reinterpret_cast<uintptr_t>(gw) & 15) == 0) {   // n_out is a multiple of 16: four columns o per float4
        const float4* wp4 = reinterpret_cast<const float4*>(wpart);
#pragma unroll 1
        for (int e = tid; e < 64 * 16; e += kTcThreads) {
          const int k = e >> 4, o = (e & 15) * 4;
          if (k < n_in && o < n_out) {
            const float4 a = wp4[e], b = wp4[1024 + e], c = wp4[2048 + e], q = wp4[3072 + e];
            float4* g = reinterpret_cast<float4*>(gw + o + (long long)n_out * k);
            float4 v = *g;
            v.x += ((a.x + b.x) + c.x) + q.x;
            v.y += ((a.y + b.y) + c.y) + q.y;
            v.z += ((a.z + b.z) + c.z) + q.z;
            v.w += ((a.w + b.w) + c.w) + q.w;
            *g = v;
          }
        }
      } else {
#pragma unroll 1
        for (int e = tid; e < 64 * 64; e += kTcThreads) {
          const int k = e >> 6, o = e & 63;
          if (k < n_in && o < n_out) gw[o + (long long)n_out * k] += ((wpart[e] + wpart[4096 + e]) + wpart[8192 + e]) + wpart[12288 + e];
        }
      }
      if (tid < n_out) gb[tid] += ((bpart[tid] + bpart[64 + tid]) + bpart[128 + tid]) + bpart[192 + tid];
      __syncthreads();   // the sum has read P
      hbar_store<C>(hbar, d);
    }
    // ---- layer 0 of the half -------------------------------------------------------------------------------------------------
    dbg_mark(cs, 29);
    l0_half<N1, N2, PURE, AK>(tc::smem_u32(fp), tP, tQ, act0, pi, ms.Xs, dc.rows, h, gw0, gb0);
    // the next half's first P store (the top layer's wgrad partials) follows two barriers: the sum above has read P by then
  }

  __syncthreads();
  dbg_mark(cs, 30);
  return (ld_phase << 1) | (phase & 1u);
}


__global__ void __launch_bounds__(kTcThreads, 1) tc_loss_grad_kernel(const __grid_constant__ TcArgs args) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ CtaShared cs;
  const int tid = threadIdx.x;
  const DevProblem* Pp = args.prob;
  const DevProblem& P = *Pp;
  const Misc ms = misc_of(smem + args.off_misc, args.mx_dim, args.mx_taps);
  float* partial = args.partial + (long long)blockIdx.x * args.partial_stride;
  const bool want_grad = (args.mode == 0);
  const float* theta = args.theta;
  const DbgSpan span = dbg_span_begin(args.dbg);

  // ---- per-CTA setup --------------------------------------------------------------------------------------------------------
  // The step usually starts with everything cold in L2 (the caller's other work evicted it).  Pull what the serial setup
  // code is about to read -- theta (tens of KB), the network / term descriptors and this CTA's first point tile -- into L2
  // right away, from counts that travel in the launch arguments: the dependent loads below then pay L2 latency, not a chain
  // of HBM round trips.
  for (long long i = (long long)tid * 32; i < args.n_theta; i += (long long)kTcThreads * 32) tc::prefetch_l2(theta + i);
  {
    const char* nets0 = reinterpret_cast<const char*>(&Pp->nets[0]);
    const char* terms0 = reinterpret_cast<const char*>(&Pp->terms[0]);
    const int nb_nets = args.n_nets * (int)sizeof(DevNet), nb_terms = args.n_terms * (int)sizeof(DevTerm);
    if (tid == 0) tc::prefetch_l2(Pp);
    for (int o = tid * 128; o < nb_nets; o += kTcThreads * 128) tc::prefetch_l2(nets0 + o);
    for (int o = tid * 128; o < nb_terms; o += kTcThreads * 128) tc::prefetch_l2(terms0 + o);
    const int tile = args.tile_begin + (int)blockIdx.x;
    if (tile < args.tile_end && tid < 32) {
      int ti = 0;
      while (ti + 1 < args.n_terms && tile >= args.dyn[ti + 1].tile0) ++ti;
      const long long p0 = (long long)(tile - args.dyn[ti].tile0) * kTcPts;
      const long long row_bytes = 4ll * args.term_dim[ti];
      const long long off = p0 * row_bytes + (long long)tid * 128;
      if (off < args.dyn[ti].n * row_bytes) tc::prefetch_l2(reinterpret_cast<const char*>(args.dyn[ti].pts) + off);
    }
  }
  if (tid == 0) {
    tc::mbar_init(ms.bar_ld, 1);
    tc::fence_barrier_init();
    cs.split = args.split; cs.off_Q = args.off_Q;
    cs.stash = args.stash + (long long)blockIdx.x * args.stash_per_cta;
    for (int k = 0; k < PINN_MAX_NETS; ++k) cs.nets[k] = args.nets[k];
    cta_base_init(cs, args, partial);
  }
  if (tid == 0) tc::s_acc = args.acc + (size_t)blockIdx.x * kAccCols * kAccRows;
  cta_setup(args, ms, partial, P.n_theta, want_grad);
  // stage weights: fp32 blocks of the first / last layers, bf16 hi / lo operand tiles of the tensor layers
  for (int kn = 0; kn < P.n_nets; ++kn) {
    const DevNet& net = P.nets[kn];
    const TcNetSmem& ns = args.nets[kn];
    if (ns.fp < 0) continue;
    stage_fp_block<kTcW>(reinterpret_cast<float*>(smem + ns.fp), net, theta);
    const int L = net.n_layers;
    // thread <-> (layer, row o, chunk of 8 k).  All global loads of all layers are issued before the first conversion
    // (fully unrolled, predicated on the layer count): one memory round trip instead of one per layer -- the step
    // starts with theta cold in L2 when the caller's other work has evicted it
    {
      constexpr int kItMax = kTcMaxTL * 512 / kTcThreads;
      const int n_items = (L - 2) * 512;
      float w[kItMax][8];
#pragma unroll
      for (int it = 0; it < kItMax; ++it) {
        const int i = tid + it * kTcThreads;
        if (i < n_items) {
          const int l = 1 + i / 512, r = i & 511;
          const int o = r & 63, kc = r >> 6;
          const int n_in = net.dims[l], n_out = net.dims[l + 1];
          const long long woff = net.w_off[l];
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            const int k = kc * 8 + e;
            w[it][e] = (o < n_out && k < n_in) ? __ldg(&theta[woff + o + (long long)n_out * k]) : 0.f;
          }
        }
      }
#pragma unroll
      for (int it = 0; it < kItMax; ++it) {
        const int i = tid + it * kTcThreads;
        if (i < n_items) {
          const int l = 1 + i / 512, r = i & 511;
          const int o = r & 63, kc = r >> 6;
          uint8_t* thi = smem + ns.w_hi[l - 1];
          uint8_t* tlo = smem + ns.w_lo[l - 1];
          const float* v = w[it];
          uint32_t h[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) h[e] = tc::pack_bf16(v[2 * e], v[2 * e + 1]);
          *reinterpret_cast<uint4*>(thi + tc::swz_chunk(o, kc)) = make_uint4(h[0], h[1], h[2], h[3]);
          if (args.split)
            *reinterpret_cast<uint4*>(tlo + tc::swz_chunk(o, kc)) = make_uint4(
                bf16x2_lo(v[0], v[1], h[0]), bf16x2_lo(v[2], v[3], h[1]), bf16x2_lo(v[4], v[5], h[2]), bf16x2_lo(v[6], v[7], h[3]));
        }
      }
    }
  }
  tc::fence_async_smem();
  __syncthreads();
  dbg_mark(&cs, 2);
  uint32_t phase = 0;

  for (int tile = args.tile_begin + blockIdx.x; tile < args.tile_end; tile += gridDim.x) {
    // warm L1 with the network descriptors (read by every phase)
    if (tid >= 128 && tid < 128 + (int)((sizeof(DevNet) * PINN_MAX_NETS + 127) / 128))
      tc::prefetch_l1(reinterpret_cast<const char*>(&P.nets[0]) + (tid - 128) * 128);
    uint32_t ldp = (phase >> 1) & 1u;
    const TileRef tr = stage_tile(args, P, ms, tile, ldp);
    phase = (phase & 1u) | (ldp << 1);
    const DevTerm* tmp = &P.terms[tr.ti];
    const DevTerm& tm = *tmp;
    const int n_used = tm.n_used;
    dbg_mark(&cs, 3);

    for (int slot = 0; slot < n_used; ++slot) {
      const int k1 = tm.chan[slot].n1, k2 = tm.chan[slot].n2, pu = tm.chan[slot].pure;
      const int ak = args.net_ak[tm.used_net[slot]];
      PINN_TC_DISPATCH(kTcMaxC, k1, k2, pu, ak, (phase = net_forward<A1, A2, PU, AK>(&cs, Pp, tmp, slot, want_grad ? 1 : 0, phase)));
    }

    dbg_mark(&cs, 4);
    // the lo-tile region Q is free between the forward and the reverse sweep
    residual_step(args, P, tm, ms, tr, smem + args.off_Q, (size_t)args.off_Q_bytes, partial, want_grad);

    dbg_mark(&cs, 5);
    if (want_grad) {
      if (tid == 0) tc::bulk_wait0();             // stash writes of this tile are complete before reloads
      __syncthreads();
      dbg_mark(&cs, 6);
      for (int slot = n_used - 1; slot >= 0; --slot) {
        const int k1 = tm.chan[slot].n1, k2 = tm.chan[slot].n2, pu = tm.chan[slot].pure;
        const int ak = args.net_ak[tm.used_net[slot]];
        if (n_used > 1) {
          // P must hold this slot's last hidden activations again: recompute its forward
          PINN_TC_DISPATCH(kTcMaxC, k1, k2, pu, ak, (phase = net_forward<A1, A2, PU, AK>(&cs, Pp, tmp, slot, 0, phase)));
        }
        PINN_TC_DISPATCH(kTcMaxC, k1, k2, pu, ak, (phase = net_backward<A1, A2, PU, AK>(&cs, Pp, tmp, slot, phase)));
      }
    }
  }

  __syncthreads();
  dbg_mark(&cs, 7);
  cta_finish(args, cs, span, ms, P, want_grad);
}

// ---- host side ------------------------------------------------------------------------------------------------------------------
size_t tc_misc_bytes(int mx_dim, int mx_taps) {
  return (size_t)mx_dim * kTcPts * 4 + 2 * (size_t)mx_taps * kTcPts * 4 + (size_t)kTcMaxC * kTcPts * 4 + kTcPts * 4 +
         PINN_MAX_TERMS * 8 + 16 + 16;
}

cudaError_t tc_launch(const TcArgs& a, int grid, size_t smem, cudaStream_t st) {
  return launch_fused_kernel<tc_loss_grad_kernel>(a, grid, kTcThreads, smem, st);
}

}  // namespace pinn
