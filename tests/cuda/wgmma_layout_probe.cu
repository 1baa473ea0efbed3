// Known-answer test of the wgmma operand layouts the library relies on (nonrigid_nerf_b200/csrc/sm90_ptx.cuh):
//   * K-major A and B from chunk-major images, A starting at row 64 of a 128-row image (the second consumer
//     warpgroup of the field kernels), K advanced by two chunks per k16 step (field_mma.cuh);
//   * MN-major (transposed) A and B from 128-point images, K advanced by 16 points per step (wgrad.cu);
// for every N the kernels use.  Small integer operands make the fp32 results exact, so any layout error shows.
// Exit status 0 and "all ok" when every element matches.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "sm90_ptx.cuh"

using namespace nrn;

namespace {

constexpr int kRows = 128;                 // rows (points) of an activation image
constexpr int kChunk = kRows * 16;         // bytes of one 8-column chunk of such an image

template <int N, int MN>
__global__ void __launch_bounds__(128, 1) probe_kernel(const uint4* a_img, int a_bytes, const uint4* b_img, int b_bytes, float* d) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* as = smem;
  uint8_t* bs = smem + ((a_bytes + 1023) / 1024) * 1024;
  for (int i = threadIdx.x; i < a_bytes / 16; i += blockDim.x) reinterpret_cast<uint4*>(as)[i] = a_img[i];
  for (int i = threadIdx.x; i < b_bytes / 16; i += blockDim.x) reinterpret_cast<uint4*>(bs)[i] = b_img[i];
  fence_proxy_async_smem();
  __syncthreads();

  float acc[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
  acc_fence(acc);
  wgmma_fence();
  if (MN == 0) {
    // A: rows 64..127 of a 128-row, K = 32 image; B: N rows x K = 32
    const uint64_t adesc = gmma_desc(smem_u32(as) + 64 * 16, kChunk, 128);
    const uint64_t bdesc = gmma_desc(smem_u32(bs), N * 16, 128);
    for (int k = 0; k < 2; ++k)
      wgmma<N, 0, 0>(acc, gmma_desc_advance(adesc, k * 2 * kChunk), gmma_desc_advance(bdesc, k * 2 * N * 16), k ? 1u : 0u);
  } else {
    // A: 64 features x 128 points, B: N features x 128 points, both stored [feature chunk][point][8]
    const uint64_t adesc = gmma_desc(smem_u32(as), 128, kChunk);
    const uint64_t bdesc = gmma_desc(smem_u32(bs), 128, kChunk);
    for (int k = 0; k < kRows / 16; ++k)
      wgmma<N, 1, 1>(acc, gmma_desc_advance(adesc, k * 256), gmma_desc_advance(bdesc, k * 256), k ? 1u : 0u);
  }
  wgmma_commit();
  wgmma_wait<0>();
  acc_fence(acc);
  const int r0 = (threadIdx.x >> 5) * 16 + ((threadIdx.x & 31) >> 2), q = threadIdx.x & 3;
#pragma unroll
  for (int j = 0; j < N / 8; ++j)
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int c = 0; c < 2; ++c) d[(r0 + 8 * i) * N + 8 * j + 2 * q + c] = acc[4 * j + 2 * i + c];
}

#define CK(x)                                                                             \
  do {                                                                                    \
    cudaError_t e_ = (x);                                                                 \
    if (e_ != cudaSuccess) {                                                              \
      std::printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
      std::exit(2);                                                                       \
    }                                                                                     \
  } while (0)

// logical operand values: small integers, exact in fp16 and in fp32 sums
float a_val(int r, int k) { return static_cast<float>((r * 3 + k * 5) % 7 - 3); }
float b_val(int n, int k) { return static_cast<float>((n * 5 + k * 3 + 1) % 5 - 2); }

template <int N, int MN>
int run() {
  // images in the chunk-major layout: element (row, col) of an R-row image at half index (col/8)*R*8 + row*8 + col%8
  std::vector<__half> a, b;
  std::vector<float> ref(64 * N, 0.f);
  if (MN == 0) {
    const int K = 32;
    a.assign(kRows * K, __float2half(0.f));
    b.assign(N * K, __float2half(0.f));
    for (int r = 0; r < kRows; ++r)
      for (int k = 0; k < K; ++k) a[(k / 8) * kRows * 8 + r * 8 + k % 8] = __float2half(a_val(r, k));
    for (int n = 0; n < N; ++n)
      for (int k = 0; k < K; ++k) b[(k / 8) * N * 8 + n * 8 + k % 8] = __float2half(b_val(n, k));
    for (int m = 0; m < 64; ++m)
      for (int n = 0; n < N; ++n)
        for (int k = 0; k < K; ++k) ref[m * N + n] += a_val(64 + m, k) * b_val(n, k);
  } else {
    a.assign(64 * kRows, __float2half(0.f));
    b.assign(N * kRows, __float2half(0.f));
    for (int p = 0; p < kRows; ++p) {
      for (int m = 0; m < 64; ++m) a[(m / 8) * kRows * 8 + p * 8 + m % 8] = __float2half(a_val(m, p));
      for (int n = 0; n < N; ++n) b[(n / 8) * kRows * 8 + p * 8 + n % 8] = __float2half(b_val(n, p));
    }
    for (int m = 0; m < 64; ++m)
      for (int n = 0; n < N; ++n)
        for (int p = 0; p < kRows; ++p) ref[m * N + n] += a_val(m, p) * b_val(n, p);
  }
  const int a_bytes = static_cast<int>(a.size() * 2), b_bytes = static_cast<int>(b.size() * 2);
  uint4 *da, *db;
  float* dd;
  CK(cudaMalloc(&da, a_bytes));
  CK(cudaMalloc(&db, b_bytes));
  CK(cudaMalloc(&dd, 64 * N * sizeof(float)));
  CK(cudaMemcpy(da, a.data(), a_bytes, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(db, b.data(), b_bytes, cudaMemcpyHostToDevice));
  CK(cudaMemset(dd, 0xff, 64 * N * sizeof(float)));
  const int smem = ((a_bytes + 1023) / 1024) * 1024 + b_bytes;
  CK(cudaFuncSetAttribute(probe_kernel<N, MN>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  probe_kernel<N, MN><<<1, 128, smem>>>(da, a_bytes, db, b_bytes, dd);
  CK(cudaGetLastError());
  CK(cudaDeviceSynchronize());
  std::vector<float> out(64 * N);
  CK(cudaMemcpy(out.data(), dd, out.size() * sizeof(float), cudaMemcpyDeviceToHost));
  CK(cudaFree(da));
  CK(cudaFree(db));
  CK(cudaFree(dd));
  int bad = 0;
  for (int i = 0; i < 64 * N; ++i) bad += out[i] != ref[i];
  std::printf("%s N=%3d: %s (%d of %d elements differ)\n", MN ? "MN-major" : "K-major ", N, bad ? "MISMATCH" : "ok", bad, 64 * N);
  return bad;
}

}  // namespace

int main() {
  int bad = 0;
  bad += run<16, 0>() + run<48, 0>() + run<64, 0>() + run<80, 0>() + run<96, 0>() + run<256, 0>();
  bad += run<48, 1>() + run<64, 1>() + run<96, 1>() + run<256, 1>();
  std::printf(bad ? "FAILED\n" : "all ok\n");
  return bad ? 1 : 0;
}
