// Parameter blocks and launchers of the evaluation / visualisation kernels (eval.cu): PSNR and SSIM scores with their
// error images, disparity images, and the background-stability map of free_viewpoint_rendering.py.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace nrn {

// uint8(255 * clip(v, 0, 1)) as numpy's .astype("uint8") truncates it (to8b); NaN (clip keeps it) maps to index 0, what
// the float -> uint8 cast gives on x86 hosts
__device__ __forceinline__ int lut_index(float v) {
  if (!(v == v)) return 0;
  return static_cast<int>(__fmul_rn(255.f, fminf(fmaxf(v, 0.f), 1.f)));
}
__device__ __forceinline__ int lut_index(double v) {
  if (!(v == v)) return 0;
  return static_cast<int>(255.0 * fmin(fmax(v, 0.0), 1.0));
}

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

// The saved 8-bit images of F frames of H x W pixels; an output is written only when its pointer is not null
struct FrameImageParams {
  const float* rgb;                 // [F][H][W][3]
  const float* disp;                // [F][H][W]
  const float* surface_pts;         // [F][H * W][3]
  const float* surface_rigidity;    // [F][H * W]
  double min_point[3], max_point[3];
  int F, H, W;
  const float* disp_max;            // [F] np.max of each disparity frame (launch_disp_max)
  uint8_t* out_rgb;                 // [F][H][W][3] to8b(rgb)
  uint8_t* out_disp;                // [F][H][W]    to8b(disp / frame max)
  uint8_t* out_disp_video;          // [F][H][W]    to8b(disp / stack max)
  uint8_t* out_disp_jet;            // [F][H][W][3] to8b(jet(disp / frame max))
  uint8_t* out_disp_phong;          // [F][H][W][3] to8b(phong(disp / frame max))
  uint8_t* out_correspondences;     // [F][H][W][3]
  uint8_t* out_rigidity;            // [F][H][W]    to8b(rigidity)
  uint8_t* out_rigidity_jet;        // [F][H][W][3] to8b(jet(rigidity))
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
cudaError_t launch_disp_max(const float* disp, int F, int H, int W, float* disp_max, cudaStream_t st);
cudaError_t launch_frame_images(const FrameImageParams& p, cudaStream_t st);

}  // namespace nrn
