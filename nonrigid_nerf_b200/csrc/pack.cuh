// Source-pointer tables for the weight packers (pack.cu).
#pragma once
#include <cuda_runtime.h>

namespace nrn {

struct NerfSrc {
  const float* w[9];  // pts_linears.0-7.weight, output_linear.weight
  const float* b[9];  // pts_linears.0-7.bias,   output_linear.bias
};
struct BenderSrc {
  const float* net_w[5];  // ray_bending.network.0-4.weight
  const float* net_b[4];  // ray_bending.network.0-3.bias (layer 4 has none)
  const float* rig_w[3];  // ray_bending.rigidity_network.0-2.weight
  const float* rig_b[3];  // ray_bending.rigidity_network.0-2.bias
};

struct ViewsSrc {
  const float* w[3];  // feature_linear.weight [256][256], views_linears.0.weight [128][256 + 27], rgb_linear.weight [3][128]
  const float* b[3];  // their biases
};

cudaError_t launch_pack_nerf(const NerfSrc& src, int in_ch, int out_ch, void* packed, cudaStream_t st);
cudaError_t launch_pack_bender(const BenderSrc& src, void* packed, cudaStream_t st);
cudaError_t launch_pack_views(const ViewsSrc& src, void* packed, cudaStream_t st);
cudaError_t launch_pack_views_t(const ViewsSrc& src, void* packed, cudaStream_t st);   // weights only (src.b not read)

}  // namespace nrn
