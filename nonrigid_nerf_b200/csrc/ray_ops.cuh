// Parameter blocks and launchers of the per-ray kernels (ray_ops.cu).
#pragma once
#include <cuda_runtime.h>

namespace nrn {

struct CompositeParams {
  const float* raw;     // [n][S][C]
  const float* z;       // [n][S]
  const float* rays_d;  // row stride rays_d_stride floats (8 when pointing into the [n][8] ray table)
  int rays_d_stride;
  const float* noise;   // [n][S] additive sigma noise (already scaled) or null
  int n, S, C, white_bkgd;
  float* rgb;           // [n][3]
  float* disp;          // [n]
  float* acc;           // [n]
  float* depth;         // [n] or null
  float* weights;       // [n][S] or null
  float* alpha;         // [n][S] or null
  // importance resampling (n_imp == 0: off)
  int n_imp;
  const float* u;       // [n][n_imp] or null (deterministic linspace)
  float* z_out;         // [n][S + n_imp]
  float* z_std;         // [n] or null
};

struct CompositeBwdParams {
  const float* raw;
  const float* z;
  const float* rays_d;
  int rays_d_stride;
  const float* noise;
  int n, S, C, white_bkgd;
  const float* d_rgb;   // [n][3]
  const float* d_acc;   // [n] or null
  float* d_raw;         // [n][S][C]
};

// |d| of a ray direction, as compositing scales the sample distances by it (train.py:748)
__device__ __forceinline__ float ray_dnorm(float dx, float dy, float dz) { return sqrtf(dx * dx + dy * dy + dz * dz); }

// The opacity of a sample (raw2outputs, train.py:740-761): 1 - exp(-relu(sigma) * gap * |d|), where sigma is the raw
// sigma plus the sample's noise (already scaled by raw_noise_std) when there is noise, and gap = z[i + 1] - z[i], or 1e10
// for the last sample (:743-748).  composite_kernel and the early-termination pass (occupancy.cu) share it, so the
// transmittance that decides termination is made of the very alphas compositing uses.  It takes values, not pointers:
// the loads stay in the callers, which keeps composite_kernel's code as it was.
__device__ __forceinline__ float composite_alpha(float sigma, float gap, float dnorm) {
  const float dist = gap * dnorm;
  return 1.0f - expf(-fmaxf(sigma, 0.f) * dist);
}

cudaError_t launch_sample_coarse(const float* rays, const float* t_rand, int n, int S, int lindisp, float* z_out,
                                 cudaStream_t st);
cudaError_t launch_composite(const CompositeParams& p, cudaStream_t st);
cudaError_t launch_sample_pdf(const float* bins, const float* weights, const float* u, int n, int nb, int n_samp,
                              float* out, cudaStream_t st);
cudaError_t launch_composite_bwd(const CompositeBwdParams& p, cudaStream_t st);
cudaError_t launch_get_rays(const float* c2w, const float* K, int H, int W, float* rays_o, float* rays_d, cudaStream_t st);
cudaError_t launch_ray_batch(const long long* pix, int n, const float* poses, const float* K, const int* image_to_view,
                             const float* images, int H, int W, float* rays_o, float* rays_d, float* target, cudaStream_t st);
cudaError_t launch_pack_rays(const float* o, const float* d, float near, float far, int n, float* rays, cudaStream_t st);
cudaError_t launch_median_index(const float* w, int n, int S, long long* idx, cudaStream_t st);

}  // namespace nrn
