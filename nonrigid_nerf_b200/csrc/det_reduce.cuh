// Fixed-order per-ray reductions of deterministic mode (det_reduce.cu).
#pragma once
#include <cuda_runtime.h>

namespace nrn {
// d_latents [n_rays][32] = per-ray sums of field_bwd_det_kernel's latent rows [n_rays * S][32]
cudaError_t launch_latent_reduce(const float* rows, float* d_latents, int n_rays, int S, cudaStream_t st);
// loss [n_rays] = per-ray sums of div_fwd_det_kernel's loss rows [n_rays * S]
cudaError_t launch_div_loss_reduce(const float* rows, float* loss, int n_rays, int S, cudaStream_t st);
}  // namespace nrn
