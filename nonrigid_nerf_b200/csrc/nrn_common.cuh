// Shared definitions: the layout of the fused field path, kernel parameter blocks.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace nrn {

// ------------------------------------------------------------------------------------------
// Layout of the fused field path: the shapes of the weight images (pack.cu), the GEMM steps of the forward, DGRAD and
// divergence kernels, the stash, gradient-stash and ReLU-mask images of a tile, and the flat gradient buffers.  Every
// kernel, the packer and the C ABI read these; a new layer is one entry here.
// ------------------------------------------------------------------------------------------
constexpr int kTileM = 128;                 // points per tile = 2 warpgroups x wgmma M (64)
constexpr int kChunkBytes = kTileM * 16;    // one 8-column chunk of a 128-row activation image
constexpr int kRingStageBytes = 32768;      // one weight slab: 256 rows x 64 K-columns fp16
constexpr int kFwdThreads = 384;            // 2 consumer warpgroups (MMA + epilogue), 1 producer warpgroup (one thread streams)
constexpr int kProducerRegs = 40, kConsumerRegs = 232;   // setmaxnreg budgets: 128 x (40 + 2 x 232) <= 64K
constexpr int kLatent = 32;

// A packed weight image: `rows` output features (the MMA's N) x `chunks` 8-column K chunks, fp16, chunk-major
// ([chunk][row][8]); t(): its transpose W^T (DGRAD).
struct WImage {
  int rows, chunks;
  __host__ __device__ constexpr int bytes() const { return rows * chunks * 16; }
  __host__ __device__ constexpr WImage t() const { return {8 * chunks, rows / 8}; }
};

// Forward steps in streaming order: the ray bender's B0..B4 (offset and rigidity MLPs fused block-diagonally, its own
// packed block), then NeRF L0..L7 and the head.  The A operand of a step is the image the step before wrote.
namespace fwd {
enum Id : int { B0, B1, B2, B3, B4, L0, L1, L2, L3, L4, L5, L6, L7, Head, kCount };
__host__ __device__ constexpr WImage image(int s) {
  switch (s) {
    case B0: return {96, 6};      // rows 0-63 offset L0, 64-95 rigidity L0; K = xyz_hi(3) xyz_lo(3) latent(32) 0(10)
    case B1: return {96, 12};     // offset L1 (64 x 64) | rigidity L1 (32 x 32)
    case B2: return {80, 12};     // offset L2 (64 x 64) | rigidity output (row 64, cols 64-95)
    case B3: return {64, 8};
    case B4: return {16, 8};      // offsets: rows 0-2, no bias
    case L0: return {256, 8};     // K = 63 (+1 zero pad column)
    case L5: return {256, 40};    // skip connection: K = embedding (64) + 256
    case Head: return {16, 32};   // N = out_ch (<= 16, zero padded)
    default: return {256, 32};    // L1-L4, L6, L7
  }
}
}  // namespace fwd

// DGRAD steps in streaming order; step X^T's image is the transpose of forward step X's (L5 in two parts).
namespace dgrad {
enum Id : int { HeadT, L7T, L6T, L5eT, L5hT, L4T, L3T, L2T, L1T, L0T, B4T, B3T, B2T, B1T, B0T, kCount };
// the forward step whose weights step s applies transposed
__host__ __device__ constexpr int forward_of(int s) {
  const int f[kCount] = {fwd::Head, fwd::L7, fwd::L6, fwd::L5, fwd::L5, fwd::L4, fwd::L3, fwd::L2, fwd::L1, fwd::L0,
                         fwd::B4, fwd::B3, fwd::B2, fwd::B1, fwd::B0};
  return f[s];
}
__host__ __device__ constexpr WImage image(int s) {
  const WImage w = fwd::image(forward_of(s));
  const int e = fwd::image(fwd::L0).chunks;   // L5's first chunks multiply the embedding (L5e^T), the rest h (L5h^T)
  return s == L5eT ? WImage{w.rows, e}.t() : s == L5hT ? WImage{w.rows, w.chunks - e}.t() : w.t();
}
}  // namespace dgrad

// Shape of one GEMM step of the field kernels: its weight image goes through the ring in `nslabs` slabs of `slab_bytes`
// (as many chunks as fit one ring stage), k16 MMAs of K = 16 per slab.
struct Step { uint32_t N, nslabs, slab_bytes, k16; };
__host__ __device__ constexpr Step make_step(WImage w) {
  const int per_slab = w.chunks < kRingStageBytes / (16 * w.rows) ? w.chunks : kRingStageBytes / (16 * w.rows);
  return {(uint32_t)w.rows, (uint32_t)(w.chunks / per_slab), (uint32_t)(per_slab * w.rows * 16), (uint32_t)(per_slab / 2)};
}
__host__ __device__ constexpr bool operator==(Step a, Step b) {
  return a.N == b.N && a.nslabs == b.nslabs && a.slab_bytes == b.slab_bytes && a.k16 == b.k16;
}
// w_off: byte offset of a step's weight image in its module's packed block (bender: B*, NeRF: the rest); b_off: float
// offset of its bias (one per image row) in the module's biases.
namespace fwd {
__host__ __device__ constexpr Step step(int s) { return make_step(image(s)); }
__host__ __device__ constexpr int w_off(int s) { int o = 0; for (int i = s < L0 ? B0 : L0; i < s; ++i) o += image(i).bytes(); return o; }
__host__ __device__ constexpr int b_off(int s) { int o = 0; for (int i = s < L0 ? B0 : L0; i < s; ++i) o += image(i).rows; return o; }
}  // namespace fwd
namespace dgrad {
__host__ __device__ constexpr Step step(int s) { return make_step(image(s)); }
__host__ __device__ constexpr int w_off(int s) { int o = 0; for (int i = s < B4T ? HeadT : B4T; i < s; ++i) o += image(i).bytes(); return o; }
}  // namespace dgrad

// Packed NeRF weights: forward images L0..head | fp32 biases (one per image row) | transposed images head^T..L0^T
constexpr int kNerfWBytes = fwd::w_off(fwd::Head) + fwd::image(fwd::Head).bytes();
constexpr int kNerfBiasFloats = fwd::b_off(fwd::Head) + fwd::image(fwd::Head).rows;
constexpr int kNerfTOffset = kNerfWBytes + kNerfBiasFloats * 4;
constexpr int kNerfTWBytes = dgrad::w_off(dgrad::L0T) + dgrad::image(dgrad::L0T).bytes();
constexpr int kNerfPackedBytes = kNerfTOffset + kNerfTWBytes;
// Packed ray-bender weights: forward images B0..B4 | fp32 biases of B0..B3 | transposed images B4^T..B0^T | residuals
// for the divergence kernels (div.cu): fp16((w - fp16(w)) * kBendLoScale) of every weight w of those images, so that
// fp16(w) + lo / kBendLoScale carries w to about 22 bits and the tangent / adjoint chains run at fp32 accuracy on fp16.
constexpr int kBendWBytes = fwd::w_off(fwd::B4) + fwd::image(fwd::B4).bytes();
constexpr int kBendBiasFloats = fwd::b_off(fwd::B4);
constexpr int kBendTOffset = kBendWBytes + kBendBiasFloats * 4;
constexpr int kBendTWBytes = dgrad::w_off(dgrad::B0T) + dgrad::image(dgrad::B0T).bytes();
constexpr float kBendLoScale = 2048.f;
constexpr int kBendLoOffset = kBendTOffset + kBendTWBytes;   // residuals of B0..B4
constexpr int kBendTLoOffset = kBendLoOffset + kBendWBytes;  // residuals of B4^T..B0^T
constexpr int kBendPackedBytes = kBendTLoOffset + kBendTWBytes;
static_assert(kNerfWBytes == 991232 && kNerfTWBytes == 991232 && kBendWBytes == 53248 && kBendTWBytes == 53248, "weight images");
static_assert(kNerfBiasFloats == 8 * 256 + 16 && kBendBiasFloats == 96 + 96 + 80 + 64, "biases");

// View-dependent head of NeRF(use_viewdirs=True), forward only.  The trunk runs L0..L7 and the Head step unchanged, the
// head image holding alpha_linear in row 3 (rows 0-2 zero), so the Head step yields alpha in column 3.  Then, in streaming
// order after Head: feature_linear (no ReLU), views_linears.0 split at input column 256 into its direction-encoding columns
// (ViewsE, K = 27 padded to 32, A from shared memory) and its feature columns (ViewsF, A = the feature fragments), both
// into one N = 128 accumulator, and rgb_linear (N = 3 padded to 16).  Step ids continue the forward table; the images are
// a packed block of their own: forward images Feature..Rgb | fp32 biases (feature 256 | views 128 | rgb 16).
namespace views {
enum Id : int { Feature = fwd::kCount, ViewsE, ViewsF, Rgb, kEnd };
constexpr int kDirCols = 27;   // direction encoding: d, then sin(2^k d), cos(2^k d) for k = 0..3
__host__ __device__ constexpr WImage image(int s) {
  switch (s) {
    case Feature: return {256, 32};
    case ViewsE: return {128, 4};
    case ViewsF: return {128, 32};
    default: return {16, 16};     // Rgb
  }
}
__host__ __device__ constexpr Step step(int s) { return make_step(image(s)); }
__host__ __device__ constexpr int w_off(int s) { int o = 0; for (int i = Feature; i < s; ++i) o += image(i).bytes(); return o; }
// ViewsE and ViewsF share the views layer's bias (stored once, at ViewsF's offset)
__host__ __device__ constexpr int b_off(int s) { int o = 0; for (int i = Feature; i < s; ++i) o += i == ViewsE ? 0 : image(i).rows; return o; }
}  // namespace views
constexpr int kViewsWBytes = views::w_off(views::kEnd);
constexpr int kViewsBiasFloats = views::b_off(views::kEnd);
constexpr int kViewsPackedBytes = kViewsWBytes + kViewsBiasFloats * 4;
static_assert(views::b_off(views::ViewsE) == 256 && views::b_off(views::ViewsF) == 256 && views::b_off(views::Rgb) == 384, "view biases");
static_assert(kViewsWBytes == 208896 && kViewsPackedBytes == 210496, "view-head images");
// Training the view-dependent head without a bender: the DGRAD steps in front of the trunk's, step ids continuing the DGRAD
// table.  Rgb^T (A = d_raw, K = 16: rgb_linear has zero column 3, so alpha's channel drops out) -> dhv; ViewsF^T (A = dYv)
// -> dF; Feature^T (A = dF) -> dh8, to which head^T of the NeRF pack adds alpha's term (its column 3 is alpha_linear,
// the rest zero).  ViewsE^T is not needed: without a bender the direction gradient has no consumer.  The images are a
// packed block of their own (nrn_pack_views_t): Rgb^T | ViewsF^T | Feature^T.
namespace vdgrad {
enum Id : int { RgbT = dgrad::kCount, ViewsFT, FeatureT, kEnd };
__host__ __device__ constexpr int forward_of(int s) { return s == RgbT ? views::Rgb : s == ViewsFT ? views::ViewsF : views::Feature; }
__host__ __device__ constexpr WImage image(int s) { return views::image(forward_of(s)).t(); }
__host__ __device__ constexpr Step step(int s) { return make_step(image(s)); }
__host__ __device__ constexpr int w_off(int s) { int o = 0; for (int i = RgbT; i < s; ++i) o += image(i).bytes(); return o; }
}  // namespace vdgrad
constexpr int kViewsTWBytes = vdgrad::w_off(vdgrad::kEnd);
static_assert(vdgrad::image(vdgrad::RgbT).rows == 128 && vdgrad::image(vdgrad::RgbT).chunks == 2 &&
              vdgrad::image(vdgrad::ViewsFT).rows == 256 && vdgrad::image(vdgrad::ViewsFT).chunks == 16 &&
              vdgrad::image(vdgrad::FeatureT).rows == 256 && vdgrad::image(vdgrad::FeatureT).chunks == 32, "view-head transposed images");
static_assert(kViewsTWBytes == 200704, "view-head transposed block");

// A tile image of the stashes: `chunks` 8-column chunks of 128 rows (fp16, chunk-major) at byte `off` of the tile.
struct Image {
  int off, chunks;
  __host__ __device__ constexpr int end() const { return off + chunks * kChunkBytes; }
  __host__ __device__ constexpr Image next(int c) const { return {end(), c}; }   // the image behind this one
};
constexpr int kHChunks = fwd::image(fwd::L1).chunks;                 // 256-wide hidden activations
constexpr int kHBytes = kHChunks * kChunkBytes;                         // 64 KB
constexpr int kEBytes = fwd::image(fwd::L0).chunks * kChunkBytes;   // 64-wide positional embedding, 16 KB

// Training stash (forward -> DGRAD, WGRAD), per tile: every image is the A operand of the forward step it feeds.
//   E: positional encoding of the bent point; the pad column 63 holds 1.0, so that the WGRAD of L0 / L5 yields the bias
//   gradient in that column.  H_l: post-ReLU activations (l = 1..8).  Bin: bender input.  Hb1..Hb4: bender hidden.
constexpr Image kStE{0, fwd::image(fwd::L0).chunks};
constexpr int kStH = kStE.end();                           // H_l at kStH + (l - 1) * kHBytes
__host__ __device__ constexpr Image st_h(int l) { return {kStH + (l - 1) * kHBytes, kHChunks}; }
constexpr Image kStBin{kStH + 8 * kHBytes, fwd::image(fwd::B0).chunks};
constexpr Image kStHb1 = kStBin.next(fwd::image(fwd::B1).chunks);
constexpr Image kStHb2 = kStHb1.next(fwd::image(fwd::B2).chunks);
constexpr Image kStHb3 = kStHb2.next(fwd::image(fwd::B3).chunks);
constexpr Image kStHb4 = kStHb3.next(fwd::image(fwd::B4).chunks);
constexpr int kStashTileBytes = kStHb4.end();
// Gradient stash (DGRAD -> WGRAD), per tile: every image is the A operand of the DGRAD step it feeds.  d_raw, dY_l
// (pre-activation gradient of L_l), dYb4 (d unmasked offsets) .. dYb0; dYb2 = [64 offset | rigidity pre-activation | pad].
constexpr Image kGsRaw{0, dgrad::image(dgrad::HeadT).chunks};
constexpr int kGsY = kGsRaw.end();                         // dY_l at kGsY + l * kHBytes, kHChunks each
constexpr Image kGsYb4{kGsY + 8 * kHBytes, dgrad::image(dgrad::B4T).chunks};
constexpr Image kGsYb3 = kGsYb4.next(dgrad::image(dgrad::B3T).chunks);
constexpr Image kGsYb2 = kGsYb3.next(dgrad::image(dgrad::B2T).chunks);
constexpr Image kGsYb1 = kGsYb2.next(dgrad::image(dgrad::B1T).chunks);
constexpr Image kGsYb0 = kGsYb1.next(dgrad::image(dgrad::B0T).chunks);
constexpr int kGradTileBytes = kGsYb0.end();
// Compact stashes of the divergence regulariser (div.cu): only the bender images, in the same order.  Tangent stash
// [e | t1 s1 | t2 s2 | t3 | t4] = the forward stash from kStBin on; adjoint stash = the gradient stash from kGsYb4 on.
constexpr int kTanTileBytes = kStashTileBytes - kStBin.off;
constexpr int kAdjTileBytes = kGradTileBytes - kGsYb4.off;
__host__ __device__ constexpr Image tan_image(Image st) { return {st.off - kStBin.off, st.chunks}; }
__host__ __device__ constexpr Image adj_image(Image gs) { return {gs.off - kGsYb4.off, gs.chunks}; }

// ReLU masks (forward -> DGRAD and the divergence kernels), per tile: one bit per element of H1..H8 and Hb1..Hb4, in the
// wgmma accumulator's order (field_mma.cuh: ReluMask); images of more than 128 columns take 32 B per row, others 16 B.
struct MaskImage {
  int off, cols;
  __host__ __device__ constexpr int end() const { return off + kTileM * (cols > 128 ? 32 : 16); }
  __host__ __device__ constexpr MaskImage next(int c) const { return {end(), c}; }
};
constexpr int kMaskHCols = 8 * kHChunks;
constexpr int kMaskHBytes = MaskImage{0, kMaskHCols}.end();  // 4 KB
constexpr int kMkH = 0;                                      // H_l at kMkH + (l - 1) * kMaskHBytes
constexpr MaskImage kMkHb1 = MaskImage{kMkH + 7 * kMaskHBytes, kMaskHCols}.next(8 * kStHb1.chunks);
constexpr MaskImage kMkHb2 = kMkHb1.next(8 * kStHb2.chunks);
constexpr MaskImage kMkHb3 = kMkHb2.next(8 * kStHb3.chunks);
constexpr MaskImage kMkHb4 = kMkHb3.next(8 * kStHb4.chunks);
constexpr int kMaskTileBytes = kMkHb4.end();
static_assert(kStashTileBytes == 634880 && kGradTileBytes == 618496 && kMaskTileBytes == 40960, "stash tiles");
static_assert(kTanTileBytes == 94208 && kAdjTileBytes == 90112, "divergence stash tiles");
// Training the view-dependent head (no bender), buffers of their own next to the trunk's:
//   view stash, per tile: Dir (direction encoding, 27 columns + 5 zero), F (feature_linear output), Hv (post-ReLU
//   views_linears.0 output); Dir and F are adjacent, the B operand [Dir | F] of views_linears.0's WGRAD.
//   view gradient stash, per tile: dYv (pre-activation gradient of views_linears.0), dF (gradient of the feature).
//   Hv mask, per tile: the ReLU mask bits of Hv (ReluMask<128>: 16 B per row).
constexpr Image kVsDir{0, views::image(views::ViewsE).chunks};
constexpr Image kVsF = kVsDir.next(views::image(views::Feature).rows / 8);
constexpr Image kVsHv = kVsF.next(views::image(views::ViewsF).rows / 8);
constexpr int kVStashTileBytes = kVsHv.end();
constexpr Image kVgYv{0, views::image(views::ViewsF).rows / 8};
constexpr Image kVgF = kVgYv.next(views::image(views::Feature).rows / 8);
constexpr int kVGradTileBytes = kVgF.end();
constexpr MaskImage kMkHv{0, views::image(views::ViewsF).rows};
constexpr int kHvMaskTileBytes = kMkHv.end();
static_assert(kVsDir.chunks == 4 && kVsF.chunks == 32 && kVsHv.chunks == 16 && kVgYv.chunks == 16 && kVgF.chunks == 32, "view stash images");
static_assert(kVStashTileBytes == 106496 && kVGradTileBytes == 98304 && kHvMaskTileBytes == 2048, "view stash tiles");

// Flat gradient buffers, in the reference's parameter order and shapes ([out][in] weights, then the bias):
//   NeRF   : W0[256][63] b0 W1[256][256] b1 ... W5[256][63 + 256] b5 ... W7 b7 Wout[out_ch][256] bout
//   bender : net_w0[64][35] net_b0 net_w1 net_b1 net_w2 net_b2 net_w3 net_b3 net_w4[3][64]
//            rig_w0[32][3] rig_b0 rig_w1[32][32] rig_b1 rig_w2[1][32] rig_b2
constexpr int kPeCols = 63;   // positional encoding of xyz, 10 octaves
__host__ __device__ constexpr int nerf_in(int l) { return l == 0 ? kPeCols : l == 5 ? kPeCols + 256 : 256; }
__host__ __device__ constexpr int nerf_grad_floats(int out_ch) { int n = out_ch * 257; for (int l = 0; l < 8; ++l) n += 256 * (nerf_in(l) + 1); return n; }
namespace bparam {
enum Id : int { NetW0, NetB0, NetW1, NetB1, NetW2, NetB2, NetW3, NetB3, NetW4, RigW0, RigB0, RigW1, RigB1, RigW2, RigB2, kCount };
constexpr int kShape[kCount][2] = {{64, 3 + kLatent}, {64, 1}, {64, 64}, {64, 1}, {64, 64}, {64, 1}, {64, 64}, {64, 1}, {3, 64},
                                   {32, 3}, {32, 1}, {32, 32}, {32, 1}, {1, 32}, {1, 1}};   // [rows, cols]
__host__ __device__ constexpr int floats(int i) { return kShape[i][0] * kShape[i][1]; }
__host__ __device__ constexpr int total() { int n = 0; for (int i = 0; i < kCount; ++i) n += floats(i); return n; }
}  // namespace bparam
static_assert(nerf_grad_floats(4) == 494084 && nerf_grad_floats(5) == 494341 && bparam::total() == 16193, "gradient buffers");
// Time-conditioned baseline (NeRF(time_conditioned_baseline=True), no bender): L0 reads [PE(63) | z(32)] and L5
// [PE(63) | z(32) | h(256)], so its flat buffer has W0[256][95] and W5[256][351].  The latent z is the same for every
// sample of a ray, so the kernels keep the geometry above and fold W_l[:, 63:95] . z + b_l into one fp32 bias row per ray
// and layer (L0, L5): the "ray bias" [rays][2][256].
__host__ __device__ constexpr int nerf_tc_grad_floats(int out_ch) { return nerf_grad_floats(out_ch) + 2 * 256 * kLatent; }
static_assert(nerf_tc_grad_floats(5) == 510725, "time-conditioned gradient buffer");
// View-dependent head (NeRF(use_viewdirs=True), module parameter order): the trunk W0 b0 .. W7 b7, then the head block
//   views_linears.0 W[128][256 + 27] b, feature_linear W[256][256] b, alpha_linear W[1][256] b, rgb_linear W[3][128] b
namespace vparam {
enum Id : int { ViewsW, ViewsB, FeatureW, FeatureB, AlphaW, AlphaB, RgbW, RgbB, kCount };
constexpr int kShape[kCount][2] = {{128, 256 + views::kDirCols}, {128, 1}, {256, 256}, {256, 1}, {1, 256}, {1, 1}, {3, 128}, {3, 1}};
__host__ __device__ constexpr int floats(int i) { return kShape[i][0] * kShape[i][1]; }
__host__ __device__ constexpr int total() { int n = 0; for (int i = 0; i < kCount; ++i) n += floats(i); return n; }
}  // namespace vparam
constexpr int kViewsTrunkFloats = nerf_grad_floats(4) - 4 * 257;
__host__ __device__ constexpr int nerf_views_grad_floats() { return kViewsTrunkFloats + vparam::total(); }
static_assert(kViewsTrunkFloats == 493056 && vparam::total() == 102788 && nerf_views_grad_floats() == 595844, "view-head gradient buffer");

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
  const uint8_t* relu_mask;    // ReLU masks of the forward call [n_tiles even][kMaskTileBytes]
};

// The point gradient d raw[3] / d x (field_bwd_grad_kernel), next to a FieldBwdParams: grad [P][3] out; the test-time
// object removal zeroes raw[3], and so the gradient, where rigidity >= removal (use_removal)
struct PointGradParams {
  float* grad;
  float removal;
  int use_removal;
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
  uint8_t* relu_mask;     // training only (with stash): ReLU masks [n_tiles rounded up to even][kMaskTileBytes]
  const float* ray_bias;  // time-conditioned kernels only: [ray][2][256] biases of L0 / L5 (stride ray_bias_stride floats,
  long long ray_bias_stride;   // 0 = one row for every ray); the other kernels ignore both
};

// View-dependent head (field_fwd.cu: the bend pass and the view-head kernel), next to a FieldFwdParams
struct ViewParams {
  const uint8_t* w;            // nrn_pack_views images ...
  const float* bias;           // ... and biases
  const float* viewdirs;       // no bender: normalised view directions, one row per ray (ray mode) or point (point mode)
  long long viewdirs_stride;   // floats between rows
  float4* ws;                  // bend workspace [P]: bent xyz and rigidity of every point (bend pass out, view head in)
};
// Training the view-dependent head (no bender), next to a FieldFwdParams and a ViewParams
struct ViewTrainParams {
  uint8_t* vstash;             // view stash [n_tiles even][kVStashTileBytes]
  uint8_t* hv_mask;            // ReLU masks of Hv [n_tiles even][kHvMaskTileBytes]
};
// Its DGRAD, next to a FieldBwdParams
struct ViewBwdParams {
  const uint8_t* wT;           // nrn_pack_views_t images
  const uint8_t* hv_mask;      // the forward's Hv masks
  uint8_t* vgstash;            // view gradient stash [n_tiles even][kVGradTileBytes]
};

// Time-conditioned backward: the per-ray sums s_l[ray] = sum over the ray's samples of dY_l (l = L0, L5), d z and the
// latent columns of dW0 / dW5 (field_bwd.cu).
struct TcBwdParams {
  const uint8_t* gstash;       // gradient stash written by DGRAD
  const float* amax;           // loss-scale source of that DGRAD run
  long long P;
  int S, n_rays;
  const float* latents;        // [n_rays][32], row stride latent_stride floats (0 = one row for all)
  long long latent_stride;
  const float* w0;             // fp32 W0 [256][95]
  const float* w5;             // fp32 W5 [256][351]
  float* sums;                 // workspace [n_rays][2][256]
  float* d_latents;            // out [n_rays][32]
  float* dw_lat;               // out [2][256][32]: dW0[:, 63:95], dW5[:, 63:95]
};

}  // namespace nrn
