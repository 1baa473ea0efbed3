// LPIPS v0.1 with the AlexNet backbone (lpips.LPIPS(net='alex'), eval mode), the perceptual score
// free_viewpoint_rendering.py:788-849 keeps per frame: layer geometry, the packed weight block, the workspace layout and
// the launchers of lpips.cu.
//
// Activations are fp16 NHWC images, one per stage and image: the scaled input (3 channels padded to 8), then
// conv1 | pool1 | conv2 | pool2 | conv3 | conv4 | conv5.  The five convolution outputs (after ReLU) are the taps.
//
// Workspace of one call (nrn_lpips_workspace_bytes): the derived mask (H * W bytes, rounded up to 256), then frames in
// chunks of Fc.  A chunk of Fc frames holds its 2 Fc images (ground truth first, then renders) at every stage, each stage
// one 256-byte aligned buffer, then the distance partials [5][Fc][max blocks] fp64 and right after them the saturation
// words [2 Fc] u32 (bit l: conv l + 1 clamped an output of the image above 65504; zeroed per chunk).
// lpips_frame_bytes(H, W) bounds one frame's share of that, so a workspace of mask + Fc * lpips_frame_bytes(H, W) bytes
// holds a chunk of Fc frames.  The default chunk is as many frames as fit kLpipsChunkBudget (at least one, at most the
// call's frames and kLpipsMaxChunk).
//
// Spatial maps (nrn_lpips_maps) use the same layout and add, right after the chunk's Fc * lpips_frame_bytes(H, W) bytes,
// its tap maps: per tap l a 256-byte aligned buffer [Fc][h_l][w_l] fp32 of the per-pixel distances the distance kernel
// sums.  lpips_map_frame_bytes(H, W) bounds one frame's share of both, and sizes the chunks of a map call.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stddef.h>
#include <stdint.h>

namespace nrn {

constexpr int kLpipsTaps = 5;
constexpr int kLpipsMinSide = 31;                       // the smallest H and W for which every tap has a pixel
constexpr int kLpipsMaxSide = 16384;
constexpr size_t kLpipsChunkBudget = 256ull << 20;      // default bytes of one chunk's activations
constexpr int kLpipsMaxChunk = 4096;                    // frames per chunk at most (the distance grid's y extent)
constexpr int kLpipsSlabChunks = 8;                     // K columns per weight slab / A stage: 8 chunks of 8 channels
constexpr float kLpipsHalfMax = 65504.f;                // the largest fp16: a convolution output above it is clamped

// One convolution as the kernels run it: cin is the channel count of its NHWC input (conv1: 3 padded to 8), cin_real
// that of the weight tensor; the output channels go in `split` launches-worth of N = cout / split columns.
struct LpipsConv {
  int cin_real, cin, cout, ks, stride, pad, split;
  __host__ __device__ constexpr int n() const { return cout / split; }
  __host__ __device__ constexpr int k_chunks() const { return ks * ks * cin / 8; }   // K = [ky][kx][cin], 8 per chunk
  __host__ __device__ constexpr int slabs() const { return (k_chunks() + kLpipsSlabChunks - 1) / kLpipsSlabChunks; }
  __host__ __device__ constexpr int slab_bytes() const { return n() * kLpipsSlabChunks * 16; }
  // packed fp16 B image: [split][slabs * 8 chunks][n][8], zero past k_chunks()
  __host__ __device__ constexpr int w_bytes() const { return split * slabs() * slab_bytes(); }
};
constexpr LpipsConv kLpipsConv[kLpipsTaps] = {
    {3, 8, 64, 11, 4, 2, 1}, {64, 64, 192, 5, 1, 2, 1}, {192, 192, 384, 3, 1, 1, 2}, {384, 384, 256, 3, 1, 1, 1}, {256, 256, 256, 3, 1, 1, 1}};

// Packed weight block (nrn_lpips_pack): the five B images, then fp32 biases (cout per layer), tap weights (cout per
// layer), shift[3], scale[3].
constexpr size_t lpips_w_off(int l) { size_t o = 0; for (int i = 0; i < l; ++i) o += kLpipsConv[i].w_bytes(); return o; }
constexpr int lpips_c_off(int l) { int o = 0; for (int i = 0; i < l; ++i) o += kLpipsConv[i].cout; return o; }
constexpr int kLpipsChannels = lpips_c_off(kLpipsTaps);
constexpr size_t kLpipsFloatOff = lpips_w_off(kLpipsTaps);
constexpr size_t kLpipsBiasOff = kLpipsFloatOff;                                  // floats at byte kLpipsBiasOff
constexpr size_t kLpipsLinOff = kLpipsBiasOff + kLpipsChannels * 4;
constexpr size_t kLpipsShiftOff = kLpipsLinOff + kLpipsChannels * 4;
constexpr size_t kLpipsScaleOff = kLpipsShiftOff + 12;
constexpr size_t kLpipsPackedBytes = kLpipsScaleOff + 12;
static_assert(kLpipsChannels == 1152 && lpips_w_off(kLpipsTaps) == 131072 + 614400 + 1327104 + 1769472 + 1179648, "LPIPS packed block");

// Spatial sizes of the 8 stages: 0 input, 1 conv1, 2 pool1, 3 conv2, 4 pool2, 5 conv3, 6 conv4, 7 conv5
constexpr int kLpipsStages = 8;
constexpr int kLpipsStageChannels[kLpipsStages] = {8, 64, 64, 192, 192, 384, 256, 256};
constexpr int kLpipsTapStage[kLpipsTaps] = {1, 3, 5, 6, 7};
constexpr int kLpipsDistPixels = 256;                   // pixels per block of the distance kernel
struct LpipsDims {
  int h[kLpipsStages], w[kLpipsStages];
  long long px(int s) const { return static_cast<long long>(h[s]) * w[s]; }
  long long image_bytes(int s) const { return px(s) * kLpipsStageChannels[s] * 2; }
  int dist_blocks(int tap) const { return static_cast<int>((px(kLpipsTapStage[tap]) + kLpipsDistPixels - 1) / kLpipsDistPixels); }
};
LpipsDims lpips_dims(int H, int W);
size_t lpips_mask_bytes(int H, int W);
size_t lpips_frame_bytes(int H, int W);

// A chunk's buffers in the workspace
struct LpipsChunk {
  int fc;                          // frames; images 0..fc-1 ground truth, fc..2fc-1 renders
  __half* act[kLpipsStages];       // [2 fc][h][w][channels]
  double* partials;                // [5][fc][max dist blocks]
  unsigned* sat;                   // [2 fc] saturation words, after the partials
  int max_blocks;
};
LpipsChunk lpips_chunk(void* ws, int fc, int H, int W);

// Spatial maps: a frame's bytes with its tap maps, and tap l's map [fc][h_l][w_l] fp32 of a chunk of fc frames
size_t lpips_map_frame_bytes(int H, int W);
float* lpips_tap_map(void* ws, int fc, int H, int W, int tap);

// The per-pixel map of a chunk of fc frames of H x W from its tap maps (lpips.LPIPS(net='alex', spatial=True)): per tap
// the bilinear upsample (align_corners=False) to H x W, NaN from the first tap whose convolution clamped an output of
// the frame on, and their sum in tap order.  Outputs point at the chunk's first frame; layer_maps, error_image may be null.
struct LpipsUpsampleParams {
  const float* tap[kLpipsTaps];    // [fc][h_l][w_l]
  int h[kLpipsTaps], w[kLpipsTaps];
  float scale_y[kLpipsTaps], scale_x[kLpipsTaps];   // (float)h_l / H, (float)w_l / W
  const unsigned* sat;             // [2 fc] the chunk's saturation words
  int fc, H, W;
  float* map;                      // [fc][H][W]
  float* layer_maps;               // [fc][5][H][W]
  uint8_t* error_image;            // [fc][H][W][3] to8b(jet(clip(map, 0, 1)))
};

struct LpipsPackSources {
  const float* conv_w[kLpipsTaps];   // OIHW
  const float* conv_b[kLpipsTaps];
  const float* lin[kLpipsTaps];      // [cout]
  const float* shift;                // [3]
  const float* scale;                // [3]
};
cudaError_t launch_lpips_pack(const LpipsPackSources& s, uint8_t* packed, cudaStream_t st);
cudaError_t launch_lpips_input(const float* gt, const float* gen, const uint8_t* mask, const uint8_t* packed, int fc, int H, int W,
                               __half* out, cudaStream_t st);
cudaError_t launch_lpips_conv(int layer, const LpipsDims& d, const __half* in, __half* out, const uint8_t* packed, int n_images,
                              int num_sms, int* err, unsigned* sat, cudaStream_t st);
cudaError_t launch_lpips_pool(const __half* in, __half* out, int n_images, int hin, int win, int hout, int wout, int channels,
                              cudaStream_t st);
cudaError_t launch_lpips_distance(int tap, const LpipsDims& d, const LpipsChunk& c, const uint8_t* packed, cudaStream_t st);
cudaError_t launch_lpips_reduce(const LpipsDims& d, const LpipsChunk& c, float* lpips, float* per_layer, cudaStream_t st);
// The distances of launch_lpips_distance that also stores each tap pixel's distance into tap_map [fc][h_l][w_l]
cudaError_t launch_lpips_distance_map(int tap, const LpipsDims& d, const LpipsChunk& c, const uint8_t* packed, float* tap_map,
                                      cudaStream_t st);
cudaError_t launch_lpips_upsample(const LpipsUpsampleParams& p, cudaStream_t st);

}  // namespace nrn
