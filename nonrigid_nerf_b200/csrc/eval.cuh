// Parameter blocks and launchers of the evaluation / visualisation kernels (eval.cu): PSNR and SSIM scores with their
// error images, disparity images, and the background-stability map of free_viewpoint_rendering.py.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace nrn {

constexpr int kEvalTileW = 32;   // SSIM output tile (pixels); the window reaches 5 pixels past it on every side
constexpr int kEvalTileH = 8;

struct ImageScoreParams {
  const float* gt;          // [F][H][W][3]
  const float* gen;         // [F][H][W][3]
  const uint8_t* mask;      // [H][W], nonzero = pixel zeroed in both images (may point into the workspace)
  int F, H, W;
  float* psnr;              // [F]
  float* ssim;              // [F]
  float* ssim_map;          // [F][H][W][3] or null
  uint8_t* error_rgb;       // [F][H][W][3] or null
  uint8_t* error_ssim;      // [F][H][W][3] or null
  double* partials;         // [F][tiles per frame][2] workspace: (squared-error sum, cropped SSIM sum) per tile
};

// Number of SSIM tiles of one frame and the workspace layout: partials first, then the derived mask (H * W bytes)
long long eval_tiles_per_frame(int H, int W);
size_t eval_partials_bytes(int F, int H, int W);

// The tables of matplotlib's cm.jet (256 entries, built from its segment data): colour values (float64) and to8b of them
void jet_table(double* rgb, uint8_t* rgb8);

cudaError_t launch_frame_mask(const float* gt, int H, int W, uint8_t* mask, cudaStream_t st);
cudaError_t launch_image_scores(const ImageScoreParams& p, cudaStream_t st);
cudaError_t launch_score_reduce(const ImageScoreParams& p, cudaStream_t st);
cudaError_t launch_disparity_images(const float* disp, int F, int H, int W, float* jet, float* phong, cudaStream_t st);
cudaError_t launch_frame_std(const float* rgbs, int F, int H, int W, float* std_out, float* image, cudaStream_t st);

}  // namespace nrn
