// The inverse of the ray bender: canonical points into every frame by Newton iteration (deform.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace nrn {

struct DeformParams {
  const float* points;         // [P][3] canonical points c
  long long P;
  const float* latents;        // [F][32], row stride latent_stride floats
  long long latent_stride;
  int F;
  const uint8_t* bender;       // nrn_pack_bender output
  int use_cutoff, use_scaling;
  float cutoff, scaling;
  int iterations;              // Newton steps, 1..64
  float tol;                   // |b(x) - c|_2 <= tol: converged (and frozen)
  float* out;                  // [F][P][3]
  float* residual;             // [F][P] or null
  uint8_t* converged;          // [F][P] or null
  float* rigidity;             // [F][P] or null
  int* err;                    // device error word
};

constexpr int kDeformMaxIterations = 64;
// J is treated as singular when |det J| <= kDeformSingular * |J e_0| |J e_1| |J e_2| (Hadamard's bound of |det J|)
constexpr float kDeformSingular = 1e-6f;

cudaError_t launch_deform(const DeformParams& p, int num_sms, cudaStream_t st);

}  // namespace nrn
