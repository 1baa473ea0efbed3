// Small utility kernels.
#include "wgrad.cuh"

namespace nrn {

namespace {
__global__ void absmax_kernel(const float* __restrict__ x, long long n, int row_len, int cols, float* __restrict__ amax) {
  float m = 0.f;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    if (row_len > 1 && i % row_len >= cols) continue;
    const float v = fabsf(x[i]);
    if (v < 3.0e38f) m = fmaxf(m, v);   // ignore inf / nan: the scale must stay finite
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  // non-negative floats order like their bit patterns
  if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<int*>(amax), __float_as_int(m));
}
}  // namespace

cudaError_t launch_absmax(const float* x, long long n, float* amax, cudaStream_t st, bool accumulate, int row_len, int cols) {
  if (!accumulate) {
    cudaError_t e = cudaMemsetAsync(amax, 0, sizeof(float), st);
    if (e != cudaSuccess) return e;
  }
  if (n <= 0 || !x) return cudaSuccess;
  long long blocks = (n + 1023) / 1024;
  if (blocks > 1184) blocks = 1184;
  absmax_kernel<<<static_cast<unsigned>(blocks), 256, 0, st>>>(x, n, row_len, cols, amax);
  return cudaGetLastError();
}

}  // namespace nrn
