// Shared definitions: packed-weight layout, kernel parameter blocks, launch helpers.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace nrn {

// ------------------------------------------------------------------------------------------
// Geometry of the fused field kernels
// ------------------------------------------------------------------------------------------
constexpr int kTileM = 128;                 // points per tile = 2 warpgroups x wgmma M (64)
constexpr int kChunkBytes = kTileM * 16;    // one 8-column chunk of a 128-row activation image
constexpr int kHBytes = 32 * kChunkBytes;   // 256-wide hidden activations, 64 KB
constexpr int kEBytes = 8 * kChunkBytes;    // 64-wide positional embedding, 16 KB
constexpr int kSlotBytes = kHBytes + kEBytes;
constexpr int kRingStageBytes = 32768;      // one weight slab: 256 rows x 64 K-columns fp16
constexpr int kRingStages = 4;
constexpr int kFwdThreads = 384;            // 2 consumer warpgroups (MMA + epilogue), 1 producer warpgroup (one thread streams)
constexpr int kProducerRegs = 40, kConsumerRegs = 232;   // setmaxnreg budgets: 128 x (40 + 2 x 232) <= 64K

// ------------------------------------------------------------------------------------------
// Packed NeRF weights (fp16, chunk-major images in streaming order), see pack.cu
//   L0   : [ 8 chunks][256 rows][8]  K = 63 (+1 zero pad)                 32 KB   (1 slab)
//   L1-4 : [32 chunks][256 rows][8]                                       128 KB  (4 slabs each)
//   L5   : [40 chunks][256 rows][8]  K = 64 (embedding, padded) + 256     160 KB  (5 slabs)
//   L6-7 : [32 chunks][256 rows][8]                                       128 KB  (4 slabs each)
//   head : [32 chunks][ 16 rows][8]  N = out_ch (<= 16, zero padded)      8 KB    (1 slab)
// followed by fp32 biases: [8][256] + [16]
// ------------------------------------------------------------------------------------------
constexpr int kNerfL0Bytes = 8 * 256 * 16;
constexpr int kNerfLBytes = 32 * 256 * 16;
constexpr int kNerfL5Bytes = 40 * 256 * 16;
constexpr int kNerfHeadBytes = 32 * 16 * 16;
constexpr int kNerfWBytes = kNerfL0Bytes + 6 * kNerfLBytes + kNerfL5Bytes + kNerfHeadBytes;  // 991,232
constexpr int kNerfBiasFloats = 8 * 256 + 16;
constexpr int kNerfTOffset = kNerfWBytes + kNerfBiasFloats * 4;   // transposed images (DGRAD) follow the biases

// Packed ray-bender weights (fp16): offset MLP and rigidity MLP fused block-diagonally.
//   B0: N=96 K=48  rows 0-63 offset L0 (cols: xyz_hi 0-2, xyz_lo 3-5, latent 6-37), rows 64-95 rigidity L0
//   B1: N=96 K=96  rows 0-63 offset L1 (cols 0-63),   rows 64-95 rigidity L1 (cols 64-95)
//   B2: N=80 K=96  rows 0-63 offset L2 (cols 0-63),   row 64 rigidity L2 (cols 64-95)
//   B3: N=64 K=64  offset L3
//   B4: N=16 K=64  rows 0-2 offset L4 (no bias)
// followed by fp32 biases: [96] [96] [80] [64]
constexpr int kBendB0Bytes = 6 * 96 * 16;
constexpr int kBendB1Bytes = 12 * 96 * 16;
constexpr int kBendB2Bytes = 12 * 80 * 16;
constexpr int kBendB3Bytes = 8 * 64 * 16;
constexpr int kBendB4Bytes = 8 * 16 * 16;
constexpr int kBendWBytes = kBendB0Bytes + kBendB1Bytes + kBendB2Bytes + kBendB3Bytes + kBendB4Bytes;  // 53,248
constexpr int kBendBiasFloats = 96 + 96 + 80 + 64;
constexpr int kBendTOffset = kBendWBytes + kBendBiasFloats * 4;
constexpr int kLatent = 32;

// ------------------------------------------------------------------------------------------
// Training stash (forward -> backward), per 128-point tile, fp16 chunk-major tile images:
//   E  (positional encoding of the bent point, 64 cols; the pad column 63 holds 1.0 so that the
//       WGRAD of L0 / L5 yields the bias gradient in that column)
//   H1..H8 (post-ReLU activations), bender input and hidden activations.
// Gradient stash (DGRAD -> WGRAD), same format: d_raw, dY7..dY0, bender dY's.
// ------------------------------------------------------------------------------------------
constexpr int kStE = 0;
constexpr int kStH = kStE + kEBytes;                       // H_l at kStH + (l-1)*kHBytes, l = 1..8
constexpr int kStBin = kStH + 8 * kHBytes;                 // bender input, 6 chunks
constexpr int kStHb1 = kStBin + 6 * kChunkBytes;           // 12 chunks
constexpr int kStHb2 = kStHb1 + 12 * kChunkBytes;          // 12 chunks
constexpr int kStHb3 = kStHb2 + 12 * kChunkBytes;          // 8 chunks
constexpr int kStHb4 = kStHb3 + 8 * kChunkBytes;           // 8 chunks
constexpr int kStashTileBytes = kStHb4 + 8 * kChunkBytes;  // 634,880

constexpr int kGsRaw = 0;                                  // d_raw, 2 chunks (16 cols)
constexpr int kGsY = kGsRaw + 2 * kChunkBytes;             // dY_l at kGsY + l*kHBytes, l = 0..7
constexpr int kGsYb4 = kGsY + 8 * kHBytes;                 // 2 chunks (d unmasked offsets)
constexpr int kGsYb3 = kGsYb4 + 2 * kChunkBytes;           // 8 chunks
constexpr int kGsYb2 = kGsYb3 + 8 * kChunkBytes;           // 10 chunks (64 + rigidity pre-activation + pad)
constexpr int kGsYb1 = kGsYb2 + 10 * kChunkBytes;          // 12 chunks
constexpr int kGsYb0 = kGsYb1 + 12 * kChunkBytes;          // 12 chunks
constexpr int kGradTileBytes = kGsYb0 + 12 * kChunkBytes;  // 618,496
// compact stashes of the divergence regulariser (div.cu): only the bender images, same relative order
constexpr int kTanTileBytes = kStashTileBytes - kStBin;    // 94,208: [e | t1 s1 | t2 s2 | t3 | t4]
constexpr int kAdjTileBytes = kGradTileBytes - kGsYb4;     // 90,112: adjoints of the tangent chain

// ------------------------------------------------------------------------------------------
// Transposed weight images for DGRAD (dX = dY . W: B operand = W^T, rows = input features,
// K = output features), fp16, in the order field_bwd.cu streams them (pack.cu):
//   head^T [2 chunks][256][8] | L7^T L6^T [32][256][8] | L5e^T [32][64][8] | L5h^T L4^T..L1^T | L0^T [32][64][8]
//   bender: B4^T [2][64][8] | B3^T [8][64][8] | B2^T [10][96][8] | B1^T [12][96][8] | B0^T [12][48][8]
// ------------------------------------------------------------------------------------------
constexpr int kNerfTHeadBytes = 2 * 256 * 16;
constexpr int kNerfTEBytes = 32 * 64 * 16;
constexpr int kNerfTWBytes = kNerfTHeadBytes + 7 * kNerfLBytes + 2 * kNerfTEBytes;
constexpr int kBendTB4Bytes = 2 * 64 * 16;
constexpr int kBendTB3Bytes = 8 * 64 * 16;
constexpr int kBendTB2Bytes = 10 * 96 * 16;
constexpr int kBendTB1Bytes = 12 * 96 * 16;
constexpr int kBendTB0Bytes = 12 * 48 * 16;
constexpr int kBendTWBytes = kBendTB4Bytes + kBendTB3Bytes + kBendTB2Bytes + kBendTB1Bytes + kBendTB0Bytes;
constexpr int kNerfPackedBytes = kNerfTOffset + kNerfTWBytes;
constexpr int kBendPackedBytes = kBendTOffset + kBendTWBytes;

struct FieldBwdParams {
  long long P;
  int n_tiles, S, n_rays, out_ch;
  const float* d_raw;          // [P][out_ch] upstream gradient of the raw field output
  const float* amax;           // device scalar: max |d_raw| (loss-scale source) or null (scale 1)
  const uint8_t* stash;        // forward stash   [n_tiles even][kStashTileBytes]
  uint8_t* gstash;             // gradient stash  [n_tiles even][kGradTileBytes]
  const uint8_t* nerf_wT;
  const uint8_t* bend_wT;
  const float* unmasked;       // [P][3] forward details (bender only)
  const float* rigidity;       // [P]
  const float* d_unmasked_up;  // [P][3] upstream gradient from the offsets regulariser, or null
  const float* d_rigid_up;     // [P]    upstream gradient from the rigidity regulariser, or null
  float cutoff, scaling;
  int use_cutoff, use_scaling;
  float* d_latents;            // [n_rays][32] fp32, zero-initialised, accumulated with atomics
  int* err;
};

// ------------------------------------------------------------------------------------------
// Kernel parameter blocks
// ------------------------------------------------------------------------------------------
struct FieldFwdParams {
  const float* rays;      // [N][8]  o(3) d(3) near far
  const float* z_vals;    // [N][S]
  const float* pts;       // point mode (rays == null): [N][pts_stride] xyz first, S == 1
  long long pts_stride;
  const float* latents;   // [N][32] (row stride latent_stride floats; 0 = one latent for all rays)
  long long latent_stride;
  int n_rays, S;
  long long P;            // n_rays * S
  int n_tiles;
  const uint8_t* nerf_w;
  const float* nerf_bias;
  const uint8_t* bend_w;
  const float* bend_bias;
  float cutoff, scaling, removal;
  int use_cutoff, use_scaling, use_removal;
  int out_ch;
  float* raw;             // [P][out_ch]
  float* d_init;          // [P][3] or null
  float* d_bent;          // [P][3] or null
  float* d_unmasked;      // [P][3] or null
  float* d_masked;        // [P][3] or null
  float* d_rigid;         // [P]    or null
  uint8_t* stash;         // training stash [n_tiles rounded up to even][kStashTileBytes] or null
  int* err;               // device error word (0 = ok)
};

}  // namespace nrn
