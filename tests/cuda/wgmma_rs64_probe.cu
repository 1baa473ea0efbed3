// Known-answer test of the register-A (RS) wgmma at N = 64 (nonrigid_nerf_b200/csrc/sm90_ptx.cuh: wgmma_m64n64_rs), the
// form DGRAD runs L5e^T and L0^T in, and of the skip layer's pattern: one set of A fragments feeds an N = 64 MMA and then,
// unchanged, an N = 256 MMA (L5e^T, then L5h^T, on dY5).  A 64 x 256 accumulator is packed to fp16 A fragments with
// frag_pair; the same fp16 values, written to a chunk-major image in shared memory, go through the shared-memory (SS) MMA.
// Both products of the RS kernel must equal those of the SS kernel bit for bit and the exact product.  Small integer
// operands make every fp16 value and fp32 sum exact.  Exit status 0 and "all ok" when every element matches.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "sm90_ptx.cuh"

using namespace nrn;

namespace {

constexpr int kM = 64;               // rows of one warpgroup's MMA
constexpr int kChunk = kM * 16;      // bytes of one 8-column chunk of a 64-row image
constexpr int kK0 = 32;              // K of the first product
constexpr int kN0 = 256;             // its N = K of the two products that follow
constexpr int kN1 = 64;              // first consumer of the fragments (L5e^T, L0^T)
constexpr int kN2 = 256;             // second consumer of the same fragments (L5h^T)

// out[M x N] of a product, in the accumulator layout of sm90_ptx.cuh
template <int N>
__device__ void store_acc(const float (&d)[N / 2], float* out) {
  const int r0 = (threadIdx.x >> 5) * 16 + ((threadIdx.x & 31) >> 2), q = threadIdx.x & 3;
#pragma unroll
  for (int j = 0; j < N / 8; ++j)
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int c = 0; c < 2; ++c) out[(r0 + 8 * i) * N + 8 * j + 2 * q + c] = d[4 * j + 2 * i + c];
}

// d = H . B^T over K = kN0 with A from the fragments a (RS) or from the image at hs (SS); one commit group
template <int N, bool RS>
__device__ void product(float (&d)[N / 2], uint32_t (&a)[kN0 / 16][4], uint32_t hs, uint32_t bs) {
  const uint64_t bdesc = gmma_desc(bs, N * 16, 128);
#pragma unroll
  for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
  acc_fence(d);
  frag_fence(a);
  wgmma_fence();
  if constexpr (RS) {
#pragma unroll
    for (int k = 0; k < kN0 / 16; ++k) wgmma_rs<N, 0>(d, a[k], gmma_desc_advance(bdesc, k * 2 * N * 16), k ? 1u : 0u);
  } else {
    const uint64_t hdesc = gmma_desc(hs, kChunk, 128);
    for (int k = 0; k < kN0 / 16; ++k)
      wgmma<N, 0, 0>(d, gmma_desc_advance(hdesc, k * 2 * kChunk), gmma_desc_advance(bdesc, k * 2 * N * 16), k ? 1u : 0u);
  }
  wgmma_commit();
  wgmma_wait<0>();
  acc_fence(d);
  frag_fence(a);
}

// RS: both products take A from the same fragments, else from the image
template <bool RS>
__global__ void __launch_bounds__(128, 1) rs64_probe_kernel(const uint4* x_img, const uint4* w0_img, const uint4* b1_img,
                                                            const uint4* b2_img, float* out1, float* out2) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* xs = smem;                               // 64 x 32
  uint8_t* w0s = xs + kK0 / 8 * kChunk;             // 256 x 32
  uint8_t* b1s = w0s + kK0 / 8 * kN0 * 16;          // 64 x 256
  uint8_t* b2s = b1s + kN0 / 8 * kN1 * 16;          // 256 x 256
  uint8_t* hs = b2s + kN0 / 8 * kN2 * 16;           // 64 x 256: the fp16 image of the first product
  for (int i = threadIdx.x; i < kK0 / 8 * kM; i += blockDim.x) reinterpret_cast<uint4*>(xs)[i] = x_img[i];
  for (int i = threadIdx.x; i < kK0 / 8 * kN0; i += blockDim.x) reinterpret_cast<uint4*>(w0s)[i] = w0_img[i];
  for (int i = threadIdx.x; i < kN0 / 8 * kN1; i += blockDim.x) reinterpret_cast<uint4*>(b1s)[i] = b1_img[i];
  for (int i = threadIdx.x; i < kN0 / 8 * kN2; i += blockDim.x) reinterpret_cast<uint4*>(b2s)[i] = b2_img[i];
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

  {
    float d1[kN1 / 2];
    product<kN1, RS>(d1, a, smem_u32(hs), smem_u32(b1s));
    store_acc<kN1>(d1, out1);
  }
  float d2[kN2 / 2];
  product<kN2, RS>(d2, a, smem_u32(hs), smem_u32(b2s));
  store_acc<kN2>(d2, out2);
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
float b1_val(int n, int k) { return static_cast<float>((n * 7 + k * 2 + 3) % 5 - 2); }
float b2_val(int n, int k) { return static_cast<float>((n * 3 + k * 7 + 2) % 5 - 2); }

// chunk-major image of an R x K matrix: element (r, k) at half index (k / 8) R 8 + 8 r + k % 8
template <typename F>
std::vector<__half> image(int rows, int cols, F f) {
  std::vector<__half> v(rows * cols);
  for (int r = 0; r < rows; ++r)
    for (int k = 0; k < cols; ++k) v[(k / 8) * rows * 8 + r * 8 + k % 8] = __float2half(f(r, k));
  return v;
}

template <typename T>
T* to_device(const std::vector<T>& v) {
  T* d;
  CK(cudaMalloc(&d, v.size() * sizeof(T)));
  CK(cudaMemcpy(d, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
  return d;
}

std::vector<float> to_host(const float* d, size_t n) {
  std::vector<float> v(n);
  CK(cudaMemcpy(v.data(), d, n * sizeof(float), cudaMemcpyDeviceToHost));
  return v;
}

int compare(const char* what, const std::vector<float>& rs, const std::vector<float>& ss, const std::vector<float>& ref) {
  int bad_rs = 0, bad_ss = 0;
  for (size_t i = 0; i < ref.size(); ++i) {
    bad_rs += rs[i] != ref[i] || rs[i] != ss[i];
    bad_ss += ss[i] != ref[i];
  }
  std::printf("%s: %s (%d of %zu elements differ from SS or exact; SS vs exact: %d)\n", what,
              bad_rs || bad_ss ? "MISMATCH" : "ok", bad_rs, ref.size(), bad_ss);
  return bad_rs + bad_ss;
}

}  // namespace

int main() {
  const std::vector<__half> x = image(kM, kK0, x_val), w0 = image(kN0, kK0, w0_val), b1 = image(kN1, kN0, b1_val),
                            b2 = image(kN2, kN0, b2_val);
  std::vector<float> h(kM * kN0, 0.f), ref1(kM * kN1, 0.f), ref2(kM * kN2, 0.f);
  for (int m = 0; m < kM; ++m)
    for (int n = 0; n < kN0; ++n)
      for (int k = 0; k < kK0; ++k) h[m * kN0 + n] += x_val(m, k) * w0_val(n, k);
  for (int m = 0; m < kM; ++m)
    for (int k = 0; k < kN0; ++k) {
      for (int n = 0; n < kN1; ++n) ref1[m * kN1 + n] += h[m * kN0 + k] * b1_val(n, k);
      for (int n = 0; n < kN2; ++n) ref2[m * kN2 + n] += h[m * kN0 + k] * b2_val(n, k);
    }
  uint4 *dx = reinterpret_cast<uint4*>(to_device(x)), *dw0 = reinterpret_cast<uint4*>(to_device(w0)),
        *db1 = reinterpret_cast<uint4*>(to_device(b1)), *db2 = reinterpret_cast<uint4*>(to_device(b2));
  float* dout[4];
  const size_t n_out[4] = {kM * kN1, kM * kN2, kM * kN1, kM * kN2};   // RS N = 64, RS N = 256, SS N = 64, SS N = 256
  for (int i = 0; i < 4; ++i) {
    CK(cudaMalloc(&dout[i], n_out[i] * sizeof(float)));
    CK(cudaMemset(dout[i], 0xff, n_out[i] * sizeof(float)));
  }
  const int smem = static_cast<int>((x.size() + w0.size() + b1.size() + b2.size()) * 2) + kN0 / 8 * kChunk;
  CK(cudaFuncSetAttribute(rs64_probe_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  CK(cudaFuncSetAttribute(rs64_probe_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  rs64_probe_kernel<true><<<1, 128, smem>>>(dx, dw0, db1, db2, dout[0], dout[1]);
  rs64_probe_kernel<false><<<1, 128, smem>>>(dx, dw0, db1, db2, dout[2], dout[3]);
  CK(cudaGetLastError());
  CK(cudaDeviceSynchronize());
  std::vector<float> out[4];
  for (int i = 0; i < 4; ++i) out[i] = to_host(dout[i], n_out[i]);
  CK(cudaFree(dx));
  CK(cudaFree(dw0));
  CK(cudaFree(db1));
  CK(cudaFree(db2));
  for (int i = 0; i < 4; ++i) CK(cudaFree(dout[i]));
  const int bad = compare("RS N= 64", out[0], out[2], ref1) + compare("RS N=256 on the same fragments after N=64", out[1], out[3], ref2);
  std::printf(bad ? "FAILED\n" : "all ok\n");
  return bad ? 1 : 0;
}
