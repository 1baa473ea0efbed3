// Parameter block and launchers of the weight-gradient kernels (wgrad.cu) and small utilities.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace nrn {

constexpr int kWgScratchFloats = 256 * 256 + 256;  // per-CTA partial: dW tile [256][256] + bias [256]
constexpr int kWgMaxCtas = 192;

struct WgradParams {
  const uint8_t* stash;    // forward activation stash
  const uint8_t* gstash;   // gradient stash written by DGRAD
  float* scratch;          // [kWgMaxCtas][kWgScratchFloats]: one partial per (job, split)
  const float* amax;       // loss-scale source (see field_bwd.cu) or null
  int n_tiles;
  int compact;             // 1: stashes hold only the bender images (divergence regulariser), bender jobs only
  long long stash_tile_bytes, gstash_tile_bytes;   // filled in by launch_wgrad
  int n_jobs;
  int job_ids[16];
  int splits[16];          // scratch partials (tile ranges) per job
  int halves[16];          // CTAs per split: 2 for a NeRF layer's 256-row dW, else 1
  int* err;
};

// Destination of the reduced gradients.  nerf: pts_linears part (nerf_n - out_ch * 257 floats) then, at `nerf_head` when
// given (else directly behind), the output_linear part.  acc_* : add to the destination instead of overwriting it.
struct WgradDst {
  float* nerf;
  float* nerf_head;
  float* bend;
  int nerf_n, bend_n;
  int acc_nerf, acc_bend;
};
cudaError_t launch_wgrad(WgradParams p, bool has_bender, int num_sms, const WgradDst& dst, int out_ch, cudaStream_t st);
// amax[0] = max |x[i]| over n floats (device scalar, overwritten)
cudaError_t launch_absmax(const float* x, long long n, float* amax, cudaStream_t st, bool accumulate = false);

}  // namespace nrn
