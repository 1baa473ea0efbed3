// Baked canonical radiance grids: the fp16 plane store of a bake, and the grid lookup of a render pass without a ray
// bender (with one, field_fwd.cu's field_baked_kernel does the lookup in the bend pass's epilogue).  baked.cuh has the rules.
#include "baked.cuh"

namespace nrn {
namespace {

constexpr int kBakedThreads = 256;

__global__ void __launch_bounds__(kBakedThreads) baked_plane_kernel(const float* __restrict__ raw, long long n, int out_ch,
                                                                    uint2* __restrict__ plane) {
  for (long long q = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; q < n; q += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float* r = raw + q * out_ch;
    const __half2 h01 = __halves2half2(baked_half(__ldg(r + 0)), baked_half(__ldg(r + 1)));
    const __half2 h23 = __halves2half2(baked_half(__ldg(r + 2)), baked_half(__ldg(r + 3)));
    plane[q] = make_uint2(*reinterpret_cast<const uint32_t*>(&h01), *reinterpret_cast<const uint32_t*>(&h23));
  }
}

__global__ void __launch_bounds__(kBakedThreads) baked_rays_kernel(const BakedGrid g, const float* __restrict__ rays,
                                                                   const float* __restrict__ z_vals, int S, long long P,
                                                                   float* __restrict__ raw, int out_ch) {
  for (long long q = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; q < P; q += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float z = __ldg(z_vals + q);
    const float* r = rays + (q / S) * 8;
    float x[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) x[d] = __fadd_rn(__ldg(r + d), __fmul_rn(__ldg(r + 3 + d), z));   // multiply, then add
    baked_raw(g, x, false, raw, q, out_ch);
  }
}

unsigned blocks_for(long long n) {
  const long long nb = (n + kBakedThreads - 1) / kBakedThreads;
  return static_cast<unsigned>(nb < (1 << 20) ? nb : (1 << 20));
}

}  // namespace

cudaError_t launch_baked_plane(const float* raw, long long n, int out_ch, uint2* plane, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  baked_plane_kernel<<<blocks_for(n), kBakedThreads, 0, st>>>(raw, n, out_ch, plane);
  return cudaGetLastError();
}

cudaError_t launch_baked_rays(const BakedGrid& g, const float* rays, const float* z_vals, int S, long long P, float* raw, int out_ch,
                              cudaStream_t st) {
  if (P <= 0) return cudaSuccess;
  baked_rays_kernel<<<blocks_for(P), kBakedThreads, 0, st>>>(g, rays, z_vals, S, P, raw, out_ch);
  return cudaGetLastError();
}

}  // namespace nrn
