// tc_types.h -- constants and launch arguments of the tensor-core path, shared by the kernel and
// the host ABI layer.
#pragma once
#include <stdint.h>
#include "dev_types.h"

namespace pinn {

constexpr int kTcPts = 128;
constexpr int kTcThreads = 512;
constexpr int kTcMaxC = 5;
constexpr int kTcMaxTaps = 6;
constexpr int kTcMaxTL = 6;            // tensor (hidden->hidden) layers per network
constexpr int kTileBytes = 16384;      // 128 rows x 128 bytes
constexpr int kAccRows = 128;          // accumulator region of a CTA: [kAccCols][kAccRows] fp32 (tc_prims.cuh)
constexpr int kAccCols = 512;
constexpr int kTcW = 64;               // accumulator column stride of a channel = widest supported layer (tc_kernel.cu)
// fp32 parameter block per network (floats), for a layer stride W (kTcW or kTwW)
template <int W>
struct FpBlock {
  static constexpr int W1 = 0;                   // [W][8] first-layer weight, W1[o*8 + k]
  static constexpr int B1 = 8 * W;               // [W]
  static constexpr int BT = 9 * W;               // [kTcMaxTL][W] tensor-layer biases
  static constexpr int WL = BT + kTcMaxTL * W;   // [W] last-layer weight
  static constexpr int BL = WL + W;              // [1]
  static constexpr int SIZE = BL + 4;
};
// accumulator-region columns (tc_prims.cuh)
constexpr uint32_t TM_X = 0;           // [c][64]: adjoints of a tensor layer's input (reverse hand-off, row = point)
constexpr uint32_t TM_Y = 320;         // last-layer / layer-0 gradient chains

struct TcNetSmem {
  int w_hi[kTcMaxTL];   // byte offsets of the bf16 weight tiles
  int w_lo[kTcMaxTL];
  int fp;               // byte offset of the fp32 parameter block
};

// launch arguments both tensor-core kernels take (TcArgs and TwArgs add their own)
struct TcCommonArgs {
  const DevProblem* prob;
  const float* theta;
  float* partial;         // [grid][partial_stride]
  long long partial_stride;
  double* term_sums;      // [grid][PINN_MAX_TERMS]
  int tl_max;             // max tensor layers over networks (stash indexing)
  int tile_begin, tile_end;
  int mode;               // 0 loss+grad, 1 loss only, 2 residual out
  float* resid_out;
  float* acc;             // [grid][kAccCols * kAccRows] fp32 accumulator regions
  long long* dbg;         // optional: 1000 x int64 phase timestamps of CTA 0 (pinn_debug_tc_timeline)
  int off_P, off_misc;    // byte offsets into dynamic shared memory
  int off_ones;           // 1 KB constant atom: bf16 1.0 in column 0 of 8 swizzled rows (bias gradient by MMA)
  int mx_dim, mx_taps;    // sizes of the per-tile coordinate / tap arrays in the misc region
  int net_ak[PINN_MAX_NETS];   // 1: every hidden activation is tanh (fast path), 0: generic
  double seed[PINN_MAX_TERMS];
  TermDyn dyn[PINN_MAX_TERMS];
  TailArgs tail;
};

struct TcArgs : TcCommonArgs {
  uint8_t* stash;         // [grid][stash_per_cta] operand-tile images of every tensor layer's input
  long long stash_per_cta;
  int split;              // forward hi/lo split
  int off_Q;              // byte offset of the lo operand tiles in dynamic shared memory
  int off_Q_bytes;        // size of the Q tile region
  int n_nets, n_terms;    // copies of the descriptor's counts (so the kernel can prefetch it before its first read)
  long long n_theta;
  unsigned char term_dim[PINN_MAX_TERMS];   // rows per point of every term (first-tile prefetch)
  TcNetSmem nets[PINN_MAX_NETS];
};


// ---- wide path (tc_wide_kernel.cu): hidden widths 64 / 128, bf16 operands, weights streamed per layer ---------------
constexpr int kTwMaxC = 4;             // channels per network: C x 128 accumulator columns
constexpr int kTwW = 128;              // accumulator column stride of a channel = widest supported layer
constexpr int kTwNB = 2;               // 64-column operand tiles per channel
constexpr int kTwImgBytes = kTwNB * kTileBytes;   // packed bf16 image of one tensor layer's weight: [kb][128 rows o][64 k]
constexpr int kTwMaxImages = PINN_MAX_NETS * kTcMaxTL;

struct TwArgs : TcCommonArgs {
  uint8_t* hstash;         // [grid][hstash_per_cta] bf16 operand tiles: input of tensor layer l, [slot][l-1][c][kb]
  long long hstash_per_cta;
  float* zstash;           // [grid][zstash_per_cta floats] fp32 pre-activations, [slot][l-1][c][col/2][point] float2
  long long zstash_per_cta;
  const uint8_t* wpack;    // packed weight images, kTwImgBytes each
  int wimg[PINN_MAX_NETS]; // image index of a network's first tensor layer
  int off_S;               // byte offset of the weight stream buffers S0 / S1 (2 x 32 KB; P holds C x 2 tiles)
  int off_nets;            // shared-memory copy of the DevNet descriptors (read every layer)
  int* tile_counter;       // dynamic tile scheduler: next unclaimed tile (reset by tw_pack_kernel)
  int off_fp[PINN_MAX_NETS];   // fp32 parameter block per network (-1: unused)
};

struct TwPackArgs {
  const DevProblem* prob;
  const float* theta;
  uint8_t* wpack;
  int n_images;
  int* tile_counter;       // reset to counter_init for the fused kernel that follows
  int counter_init;
  unsigned char img_net[kTwMaxImages], img_layer[kTwMaxImages];
};

cudaError_t tw_pack_launch(const TwPackArgs& a, cudaStream_t st);
cudaError_t tw_launch(const TwArgs& a, int grid, size_t smem, cudaStream_t st);

// ---- 256-wide path (tc_x256_kernel.cu): hidden widths multiples of 64 up to 256, each 128-point tile as two 64-point
// halves.  Launch arguments are TwArgs / TwPackArgs; off_fp[0] is the one fp32 parameter block, staged per pass.
constexpr int kTxW = 256;              // accumulator column stride of a channel = widest supported layer
constexpr int kTxPts = 64;             // points per half tile = rows of an operand tile
constexpr int kTxTileBytes = kTxPts * 128;        // operand tile: 64 rows x 64 bf16
constexpr int kTxImgBytes = 8 * kTileBytes;       // packed bf16 image of one tensor layer: [kb][128-row half of o][128 rows][64 k]
constexpr int kTxMaxTaps = PINN_MAX_TAPS;         // the misc region is sized per problem (the other kernels keep kTcMaxTaps)

cudaError_t tx_pack_launch(const TwPackArgs& a, cudaStream_t st);
cudaError_t tx_launch(const TwArgs& a, int grid, size_t smem, cudaStream_t st);

size_t tc_misc_bytes(int mx_dim, int mx_taps);
cudaError_t tc_launch(const TcArgs& a, int grid, size_t smem, cudaStream_t st);

}  // namespace pinn
