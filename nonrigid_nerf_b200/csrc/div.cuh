// Parameter block and launchers of the divergence-regulariser kernels (div.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace nrn {

struct DivParams {
  long long P;               // coarse sample points = n_rays * S
  int S, n_rays;
  const uint8_t* relu_mask;  // ReLU mask bits of the coarse field pass [tiles][kMaskTileBytes]
  const uint8_t* bender;     // packed bender weights (ops.pack_bender): B0..B4 images, transposed images at kBendTOffset
  const float* e;            // [P][3]  Hutchinson probe vectors ~ N(0, I)
  const float* unmasked;     // [P][3]  coarse unmasked offsets
  const float* rigidity;     // [P]     coarse rigidity mask
  const float* w;            // [P]     loss weights 1 - exp(-relu(alpha)) (detached) -- or alpha itself:
  int w_is_alpha;            //         1 = `w` holds opacity_alpha, the kernels apply 1 - exp(-relu(.)) (train.py:267)
  uint8_t* tan;              // tangent stash  [tiles][kTanTileBytes]
  float* d;                  // [P] divergence estimate, and the scalars the backward needs:
  float* adot;               // [P] alpha = e . tau_off
  float* beta;               // [P] beta  = e . off
  float* tauc;               // [P] tangent of the rigidity pre-activation
  float* loss;               // [n_rays] (zero-initialised) mean_s(w d^2)
  // backward
  const float* G;            // [P] dL/dd
  const float* amax;         // device scalar max|G| (loss scale source)
  uint8_t* adj;              // adjoint stash [tiles][kAdjTileBytes]
  float* d_unmasked;         // [P][3] out
  float* d_rigid;            // [P]    out
  int* err;                  // device error word (0 = ok)
};

cudaError_t launch_div_fwd(const DivParams& p, int num_sms, cudaStream_t st);
cudaError_t launch_div_bwd(const DivParams& p, int num_sms, cudaStream_t st);
// launch_div_bwd leaving the points of held-out rays (held [n_rays] bytes, nonzero = held out) out of the adjoint stash
cudaError_t launch_div_bwd_held(const DivParams& p, const uint8_t* held, int num_sms, cudaStream_t st);
// deterministic mode: per-point loss rows [P] instead of atomics into p.loss (launch_div_loss_reduce then writes p.loss)
cudaError_t launch_div_fwd_det(const DivParams& p, float* loss_rows, int num_sms, cudaStream_t st);
// G[pt] = g_ray[pt / S] * 2 * w * d / S (the gradient of mean_s(w d^2)) and amax = max|G| in one pass
cudaError_t launch_div_G(const DivParams& p, const float* g_ray, float* G, float* amax, cudaStream_t st);

}  // namespace nrn
