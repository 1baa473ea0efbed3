// Weight packing of the view-dependent head's transposed images, for the DGRAD of its training (field_bwd.cu:
// field_bwd_views_kernel); layout in nrn_common.cuh (vdgrad::).  A translation unit of its own beside pack.cu.
#include <cuda_fp16.h>
#include "nrn_common.cuh"
#include "pack.cuh"

namespace nrn {

namespace {

constexpr int kPackThreads = 256;

// image element index -> (chunk column k, row r) for an image with R rows (as pack.cu)
__device__ __forceinline__ void decode(int idx, int R, int& k, int& r) {
  const int c = idx / (R * 8);
  const int rem = idx - c * R * 8;
  r = rem >> 3;
  k = c * 8 + (rem & 7);
}

// Transposed images of the view-dependent head for its DGRAD (layout in nrn_common.cuh, vdgrad::): Rgb^T (rows = 128
// hidden, K = 3 rgb channels padded to 16), ViewsF^T (rows = 256 feature inputs, K = 128 outputs), Feature^T.
__global__ void __launch_bounds__(kPackThreads) pack_views_t_kernel(ViewsSrc src, __half* __restrict__ w) {
  using namespace vdgrad;
  constexpr WImage wr = image(RgbT), wv = image(ViewsFT), wf = image(FeatureT);
  constexpr int nr = wr.bytes() / 2, nv = wv.bytes() / 2;
  constexpr int ldv = 256 + views::kDirCols;
  int i = blockIdx.x * kPackThreads + threadIdx.x, k, r;
  if (i >= kViewsTWBytes / 2) return;
  const int idx = i;
  float v = 0.f;
  if (i < nr) {                            // Rgb^T
    decode(i, wr.rows, k, r);
    v = k < 3 ? src.w[2][k * 128 + r] : 0.f;
  } else if ((i -= nr) < nv) {             // ViewsF^T: the feature columns of views_linears.0
    decode(i, wv.rows, k, r);
    v = src.w[1][k * ldv + r];
  } else {                                 // Feature^T
    i -= nv;
    decode(i, wf.rows, k, r);
    v = src.w[0][k * 256 + r];
  }
  w[idx] = __float2half_rn(v);
}

}  // namespace

cudaError_t launch_pack_views_t(const ViewsSrc& src, void* packed, cudaStream_t st) {
  pack_views_t_kernel<<<(kViewsTWBytes / 2 + kPackThreads - 1) / kPackThreads, kPackThreads, 0, st>>>(src, reinterpret_cast<__half*>(packed));
  return cudaGetLastError();
}

}  // namespace nrn
