// Known-answer test of the register-A (RS) wgmma form the field kernels chain their trunk layers with
// (nonrigid_nerf_b200/csrc/sm90_ptx.cuh: wgmma_rs, frag_pair): a 64 x 256 accumulator is packed to fp16 A fragments
// with frag_pair and multiplied by B through the RS MMA; the same fp16 values, written to a chunk-major image in shared
// memory, go through the shared-memory (SS) MMA.  Both results must equal each other bit for bit and the exact product,
// for every N the kernels run in RS form.  Small integer operands make every fp16 value and fp32 sum exact.
// Exit status 0 and "all ok" when every element matches.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "sm90_ptx.cuh"

using namespace nrn;

namespace {

constexpr int kM = 64;               // rows of one warpgroup's MMA
constexpr int kChunk = kM * 16;      // bytes of one 8-column chunk of a 64-row image
constexpr int kK0 = 32;              // K of the first product
constexpr int kN0 = 256;             // its N = K of the second product

// RS: the second product takes A from the fragments, else from the image
template <int N, bool RS>
__global__ void __launch_bounds__(128, 1) rs_probe_kernel(const uint4* x_img, const uint4* w0_img, const uint4* b_img, float* out) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* xs = smem;                               // 64 x 32
  uint8_t* w0s = xs + kK0 / 8 * kChunk;             // 256 x 32
  uint8_t* bs = w0s + kK0 / 8 * kN0 * 16;           // N x 256
  uint8_t* hs = bs + kN0 / 8 * N * 16;              // 64 x 256: the fp16 image of the first product
  for (int i = threadIdx.x; i < kK0 / 8 * kM; i += blockDim.x) reinterpret_cast<uint4*>(xs)[i] = x_img[i];
  for (int i = threadIdx.x; i < kK0 / 8 * kN0; i += blockDim.x) reinterpret_cast<uint4*>(w0s)[i] = w0_img[i];
  for (int i = threadIdx.x; i < kN0 / 8 * N; i += blockDim.x) reinterpret_cast<uint4*>(bs)[i] = b_img[i];
  fence_proxy_async_smem();
  __syncthreads();

  // first product (SS), then its fp16 pairs -> A fragments and -> the chunk-major image
  float h[kN0 / 2];
#pragma unroll
  for (int i = 0; i < kN0 / 2; ++i) h[i] = 0.f;
  acc_fence(h);
  wgmma_fence();
  const uint64_t xdesc = gmma_desc(smem_u32(xs), kChunk, 128), w0desc = gmma_desc(smem_u32(w0s), kN0 * 16, 128);
  for (int k = 0; k < kK0 / 16; ++k)
    wgmma<kN0, 0, 0>(h, gmma_desc_advance(xdesc, k * 2 * kChunk), gmma_desc_advance(w0desc, k * 2 * kN0 * 16), k ? 1u : 0u);
  wgmma_commit();
  wgmma_wait<0>();
  acc_fence(h);
  const int r0 = (threadIdx.x >> 5) * 16 + ((threadIdx.x & 31) >> 2), q = threadIdx.x & 3;
  uint32_t a[kN0 / 16][4];
#pragma unroll
  for (int j = 0; j < kN0 / 8; ++j)
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const uint32_t h2 = pack_h2_sat(h[4 * j + 2 * i], h[4 * j + 2 * i + 1]);
      frag_pair(a, j, i) = h2;
      *reinterpret_cast<uint32_t*>(hs + j * kChunk + (r0 + 8 * i) * 16 + 4 * q) = h2;
    }
  fence_proxy_async_smem();
  __syncthreads();

  const uint64_t bdesc = gmma_desc(smem_u32(bs), N * 16, 128);
  float d[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
  acc_fence(d);
  frag_fence(a);
  wgmma_fence();
  if constexpr (RS) {
#pragma unroll
    for (int k = 0; k < kN0 / 16; ++k) wgmma_rs<N, 0>(d, a[k], gmma_desc_advance(bdesc, k * 2 * N * 16), k ? 1u : 0u);
  } else {
    const uint64_t hdesc = gmma_desc(smem_u32(hs), kChunk, 128);
    for (int k = 0; k < kN0 / 16; ++k)
      wgmma<N, 0, 0>(d, gmma_desc_advance(hdesc, k * 2 * kChunk), gmma_desc_advance(bdesc, k * 2 * N * 16), k ? 1u : 0u);
  }
  wgmma_commit();
  wgmma_wait<0>();
  acc_fence(d);
  frag_fence(a);
#pragma unroll
  for (int j = 0; j < N / 8; ++j)
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int c = 0; c < 2; ++c) out[(r0 + 8 * i) * N + 8 * j + 2 * q + c] = d[4 * j + 2 * i + c];
}

#define CK(x)                                                                             \
  do {                                                                                    \
    cudaError_t e_ = (x);                                                                 \
    if (e_ != cudaSuccess) {                                                              \
      std::printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
      std::exit(2);                                                                       \
    }                                                                                     \
  } while (0)

float x_val(int r, int k) { return static_cast<float>((r * 3 + k * 5) % 7 - 3); }
float w0_val(int n, int k) { return static_cast<float>((n * 5 + k * 3 + 1) % 5 - 2); }
float b_val(int n, int k) { return static_cast<float>((n * 7 + k * 2 + 3) % 5 - 2); }

// chunk-major image of an R x K matrix: element (r, k) at half index (k / 8) R 8 + 8 r + k % 8
template <typename F>
std::vector<__half> image(int rows, int cols, F f) {
  std::vector<__half> v(rows * cols);
  for (int r = 0; r < rows; ++r)
    for (int k = 0; k < cols; ++k) v[(k / 8) * rows * 8 + r * 8 + k % 8] = __float2half(f(r, k));
  return v;
}

template <int N>
int run() {
  const std::vector<__half> x = image(kM, kK0, x_val), w0 = image(kN0, kK0, w0_val), b = image(N, kN0, b_val);
  std::vector<float> h(kM * kN0, 0.f), ref(kM * N, 0.f);
  for (int m = 0; m < kM; ++m)
    for (int n = 0; n < kN0; ++n)
      for (int k = 0; k < kK0; ++k) h[m * kN0 + n] += x_val(m, k) * w0_val(n, k);
  for (int m = 0; m < kM; ++m)
    for (int n = 0; n < N; ++n)
      for (int k = 0; k < kN0; ++k) ref[m * N + n] += h[m * kN0 + k] * b_val(n, k);
  uint4 *dx, *dw0, *db;
  float *drs, *dss;
  CK(cudaMalloc(&dx, x.size() * 2));
  CK(cudaMalloc(&dw0, w0.size() * 2));
  CK(cudaMalloc(&db, b.size() * 2));
  CK(cudaMalloc(&drs, kM * N * sizeof(float)));
  CK(cudaMalloc(&dss, kM * N * sizeof(float)));
  CK(cudaMemcpy(dx, x.data(), x.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dw0, w0.data(), w0.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(db, b.data(), b.size() * 2, cudaMemcpyHostToDevice));
  CK(cudaMemset(drs, 0xff, kM * N * sizeof(float)));
  CK(cudaMemset(dss, 0xff, kM * N * sizeof(float)));
  const int smem = static_cast<int>((x.size() + w0.size() + b.size()) * 2) + kN0 / 8 * kChunk;
  CK(cudaFuncSetAttribute(rs_probe_kernel<N, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  CK(cudaFuncSetAttribute(rs_probe_kernel<N, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  rs_probe_kernel<N, true><<<1, 128, smem>>>(dx, dw0, db, drs);
  rs_probe_kernel<N, false><<<1, 128, smem>>>(dx, dw0, db, dss);
  CK(cudaGetLastError());
  CK(cudaDeviceSynchronize());
  std::vector<float> rs(kM * N), ss(kM * N);
  CK(cudaMemcpy(rs.data(), drs, rs.size() * sizeof(float), cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(ss.data(), dss, ss.size() * sizeof(float), cudaMemcpyDeviceToHost));
  CK(cudaFree(dx));
  CK(cudaFree(dw0));
  CK(cudaFree(db));
  CK(cudaFree(drs));
  CK(cudaFree(dss));
  int bad_rs = 0, bad_ss = 0;
  for (int i = 0; i < kM * N; ++i) {
    bad_rs += rs[i] != ref[i] || rs[i] != ss[i];
    bad_ss += ss[i] != ref[i];
  }
  std::printf("RS N=%3d: %s (%d of %d elements differ from SS or exact; SS vs exact: %d)\n", N,
              bad_rs || bad_ss ? "MISMATCH" : "ok", bad_rs, kM * N, bad_ss);
  return bad_rs + bad_ss;
}

}  // namespace

int main() {
  const int bad = run<16>() + run<256>();
  std::printf(bad ? "FAILED\n" : "all ok\n");
  return bad ? 1 : 0;
}
