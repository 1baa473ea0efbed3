// Weight packing: fp32 nn.Linear tensors ([out][in] row-major, the reference's checkpoint layout,
// run_nerf_helpers.py:218-238 and :411-482) -> fp16 "chunk-major" wgmma operand images laid out in the
// exact order the fused kernels stream them (layout table in nrn_common.cuh).
// Re-run after every optimizer step / load_state_dict (1.07 M parameters: a few microseconds); forward and
// transposed (DGRAD) images of a module are written by ONE launch.
#include <cuda_fp16.h>
#include "nrn_common.cuh"
#include "pack.cuh"

namespace nrn {

namespace {

// image element index -> (chunk, row, e) for an image with R rows
__device__ __forceinline__ void decode(int idx, int R, int& k, int& r) {
  const int c = idx / (R * 8);
  const int rem = idx - c * R * 8;
  r = rem >> 3;
  k = c * 8 + (rem & 7);
}

// TC (time-conditioned baseline, in_ch = 63 + 32): W0 / W5 carry the latent columns 63-94 behind the embedding; they are
// skipped (they enter the kernels as a per-ray bias), so the images are the same as for in_ch = 63.
template <bool TC>
__device__ __forceinline__ void pack_nerf_elem(const int idx, const NerfSrc& src, int in_ch, int out_ch, __half* __restrict__ w, float* __restrict__ bias) {
  const int pe = TC ? kPeCols : in_ch;   // embedding columns
  constexpr WImage w0 = fwd::image(fwd::L0), wl = fwd::image(fwd::L1), w5 = fwd::image(fwd::L5), wh = fwd::image(fwd::Head);
  constexpr int n0 = w0.bytes() / 2, nl = wl.bytes() / 2, n5 = w5.bytes() / 2;
  if (idx < kNerfWBytes / 2) {
    int i = idx, k, r;
    float v = 0.f;
    if (i < n0) {  // L0: K = in_ch (63) padded to 64
      decode(i, w0.rows, k, r);
      v = k < pe ? src.w[0][r * in_ch + k] : 0.f;
    } else if ((i -= n0) < 4 * nl) {  // L1..L4
      const int L = 1 + i / nl;
      decode(i % nl, wl.rows, k, r);
      v = src.w[L][r * 256 + k];
    } else if ((i -= 4 * nl) < n5) {  // L5: [embedding(in_ch) pad | h(256)]
      decode(i, w5.rows, k, r);
      const int ld = in_ch + 256;
      if (k < 8 * w0.chunks) v = k < pe ? src.w[5][r * ld + k] : 0.f;
      else v = src.w[5][r * ld + in_ch + (k - 8 * w0.chunks)];
    } else if ((i -= n5) < 2 * nl) {  // L6, L7
      const int L = 6 + i / nl;
      decode(i % nl, wl.rows, k, r);
      v = src.w[L][r * 256 + k];
    } else {  // head, N padded to 16
      i -= 2 * nl;
      decode(i, wh.rows, k, r);
      v = r < out_ch ? src.w[8][r * 256 + k] : 0.f;
    }
    w[idx] = __float2half_rn(v);
  }
  if (idx < kNerfBiasFloats) {
    float b;
    constexpr int bh = fwd::b_off(fwd::Head);
    if (idx < bh) b = src.b[idx >> 8][idx & 255];
    else b = (idx - bh) < out_ch ? src.b[8][idx - bh] : 0.f;
    bias[idx] = b;
  }
}

// fp16 residual of a weight, scaled into fp16's normal range (nrn_common.cuh: kBendLoScale)
__device__ __forceinline__ __half lo_half(float v) { return __float2half_rn((v - __half2float(__float2half_rn(v))) * kBendLoScale); }

__device__ __forceinline__ void pack_bender_elem(const int idx, const BenderSrc& src, __half* __restrict__ w, float* __restrict__ bias,
                                                 __half* __restrict__ wlo) {
  constexpr WImage w0 = fwd::image(fwd::B0), w1 = fwd::image(fwd::B1), w2 = fwd::image(fwd::B2), w3 = fwd::image(fwd::B3), w4 = fwd::image(fwd::B4);
  constexpr int n0 = w0.bytes() / 2, n1 = w1.bytes() / 2, n2 = w2.bytes() / 2, n3 = w3.bytes() / 2;
  constexpr int ld0 = 3 + kLatent;
  if (idx < kBendWBytes / 2) {
    int i = idx, k, r;
    float v = 0.f;
    if (i < n0) {  // B0: K = [xyz_hi xyz_lo latent pad] = 48
      decode(i, w0.rows, k, r);
      if (r < 64) {
        if (k < 3) v = src.net_w[0][r * ld0 + k];
        else if (k < 6) v = src.net_w[0][r * ld0 + (k - 3)];
        else if (k < 6 + kLatent) v = src.net_w[0][r * ld0 + 3 + (k - 6)];
      } else {
        if (k < 3) v = src.rig_w[0][(r - 64) * 3 + k];
        else if (k < 6) v = src.rig_w[0][(r - 64) * 3 + (k - 3)];
      }
    } else if ((i -= n0) < n1) {  // B1: block diagonal 64x64 + 32x32
      decode(i, w1.rows, k, r);
      if (r < 64) { if (k < 64) v = src.net_w[1][r * 64 + k]; }
      else { if (k >= 64) v = src.rig_w[1][(r - 64) * 32 + (k - 64)]; }
    } else if ((i -= n1) < n2) {  // B2: offset L2 + rigidity output row
      decode(i, w2.rows, k, r);
      if (r < 64) { if (k < 64) v = src.net_w[2][r * 64 + k]; }
      else if (r == 64) { if (k >= 64) v = src.rig_w[2][k - 64]; }
    } else if ((i -= n2) < n3) {  // B3
      decode(i, w3.rows, k, r);
      v = src.net_w[3][r * 64 + k];
    } else {  // B4: 3 output rows, no bias
      i -= n3;
      decode(i, w4.rows, k, r);
      if (r < 3) v = src.net_w[4][r * 64 + k];
    }
    w[idx] = __float2half_rn(v);
    wlo[idx] = lo_half(v);
  }
  if (idx < kBendBiasFloats) {
    float b = 0.f;
    constexpr int b1 = fwd::b_off(fwd::B1), b2 = fwd::b_off(fwd::B2), b3 = fwd::b_off(fwd::B3);
    if (idx < b1) b = idx < 64 ? src.net_b[0][idx] : src.rig_b[0][idx - 64];
    else if (idx < b2) { const int j = idx - b1; b = j < 64 ? src.net_b[1][j] : src.rig_b[1][j - 64]; }
    else if (idx < b3) { const int j = idx - b2; b = j < 64 ? src.net_b[2][j] : (j == 64 ? src.rig_b[2][0] : 0.f); }
    else b = src.net_b[3][idx - b3];
    bias[idx] = b;
  }
}

// ---- transposed images for DGRAD: W^T (rows = input features, K = output features), layout in nrn_common.cuh ----
// r = input feature, k = output feature
template <bool TC>
__device__ __forceinline__ void pack_nerf_t_elem(const int idx, const NerfSrc& src, int in_ch, int out_ch, __half* __restrict__ w) {
  if (idx >= kNerfTWBytes / 2) return;
  const int pe = TC ? kPeCols : in_ch;
  constexpr WImage wh = dgrad::image(dgrad::HeadT), wl = dgrad::image(dgrad::L7T), we = dgrad::image(dgrad::L5eT), w0 = dgrad::image(dgrad::L0T);
  constexpr int nh = wh.bytes() / 2, nl = wl.bytes() / 2, ne = we.bytes() / 2;
  int i = idx, k, r;
  float v = 0.f;
  const int ld5 = in_ch + 256;
  if (i < nh) {                           // head^T: K = out_ch padded to 16
    decode(i, wh.rows, k, r);
    v = k < out_ch ? src.w[8][k * 256 + r] : 0.f;
  } else if ((i -= nh) < 2 * nl) {        // L7^T, L6^T
    const int L = 7 - i / nl;
    decode(i % nl, wl.rows, k, r);
    v = src.w[L][k * 256 + r];
  } else if ((i -= 2 * nl) < ne) {        // L5e^T: rows = embedding inputs (in_ch, padded to 64)
    decode(i, we.rows, k, r);
    v = r < pe ? src.w[5][k * ld5 + r] : 0.f;
  } else if ((i -= ne) < nl) {            // L5h^T
    decode(i, wl.rows, k, r);
    v = src.w[5][k * ld5 + in_ch + r];
  } else if ((i -= nl) < 4 * nl) {        // L4^T .. L1^T
    const int L = 4 - i / nl;
    decode(i % nl, wl.rows, k, r);
    v = src.w[L][k * 256 + r];
  } else {                                // L0^T
    i -= 4 * nl;
    decode(i, w0.rows, k, r);
    v = r < pe ? src.w[0][k * in_ch + r] : 0.f;
  }
  w[idx] = __float2half_rn(v);
}

__device__ __forceinline__ void pack_bender_t_elem(const int idx, const BenderSrc& src, __half* __restrict__ w, __half* __restrict__ wlo) {
  if (idx >= kBendTWBytes / 2) return;
  using namespace dgrad;
  constexpr WImage w4 = image(B4T), w3 = image(B3T), w2 = image(B2T), w1 = image(B1T), w0 = image(B0T);
  constexpr int n4 = w4.bytes() / 2, n3 = w3.bytes() / 2, n2 = w2.bytes() / 2, n1 = w1.bytes() / 2;
  constexpr int ld0 = 3 + kLatent;
  int i = idx, k, r;
  float v = 0.f;
  if (i < n4) {                           // B4^T: rows = 64 hidden, K = 3 outputs (padded to 16)
    decode(i, w4.rows, k, r);
    v = k < 3 ? src.net_w[4][k * 64 + r] : 0.f;
  } else if ((i -= n4) < n3) {            // B3^T
    decode(i, w3.rows, k, r);
    v = src.net_w[3][k * 64 + r];
  } else if ((i -= n3) < n2) {            // B2^T: rows = 96 inputs, K = 80 outputs (64 offset, 1 rigidity, pad)
    decode(i, w2.rows, k, r);
    if (r < 64) { if (k < 64) v = src.net_w[2][k * 64 + r]; }
    else { if (k == 64) v = src.rig_w[2][r - 64]; }
  } else if ((i -= n2) < n1) {            // B1^T: block diagonal
    decode(i, w1.rows, k, r);
    if (r < 64) { if (k < 64) v = src.net_w[1][k * 64 + r]; }
    else { if (k >= 64) v = src.rig_w[1][(k - 64) * 32 + (r - 64)]; }
  } else {                                // B0^T: rows = 48 inputs [xyz_hi xyz_lo latent pad], K = 96 outputs
    i -= n1;
    decode(i, w0.rows, k, r);
    if (r >= 6 && r < 6 + kLatent) { if (k < 64) v = src.net_w[0][k * ld0 + 3 + (r - 6)]; }
    else if (r < 3) v = k < 64 ? src.net_w[0][k * ld0 + r] : src.rig_w[0][(k - 64) * 3 + r];
  }
  w[idx] = __float2half_rn(v);
  wlo[idx] = lo_half(v);
}


// one launch per module: the first blocks write the forward images (+ biases), the rest the transposed images
constexpr int kPackThreads = 256;
__global__ void __launch_bounds__(kPackThreads) pack_nerf_kernel(NerfSrc src, int in_ch, int out_ch, __half* __restrict__ w,
                                                                 float* __restrict__ bias, __half* __restrict__ wt) {
  constexpr int nb_fwd = (kNerfWBytes / 2 + kPackThreads - 1) / kPackThreads;
  if (blockIdx.x < nb_fwd) pack_nerf_elem<false>(blockIdx.x * kPackThreads + threadIdx.x, src, in_ch, out_ch, w, bias);
  else pack_nerf_t_elem<false>((blockIdx.x - nb_fwd) * kPackThreads + threadIdx.x, src, in_ch, out_ch, wt);
}
__global__ void __launch_bounds__(kPackThreads) pack_nerf_tc_kernel(NerfSrc src, int out_ch, __half* __restrict__ w,
                                                                    float* __restrict__ bias, __half* __restrict__ wt) {
  constexpr int nb_fwd = (kNerfWBytes / 2 + kPackThreads - 1) / kPackThreads;
  constexpr int in_ch = kPeCols + kLatent;
  if (blockIdx.x < nb_fwd) pack_nerf_elem<true>(blockIdx.x * kPackThreads + threadIdx.x, src, in_ch, out_ch, w, bias);
  else pack_nerf_t_elem<true>((blockIdx.x - nb_fwd) * kPackThreads + threadIdx.x, src, in_ch, out_ch, wt);
}
__global__ void __launch_bounds__(kPackThreads) pack_bender_kernel(BenderSrc src, __half* __restrict__ w, float* __restrict__ bias,
                                                                   __half* __restrict__ wt, __half* __restrict__ wlo,
                                                                   __half* __restrict__ wtlo) {
  constexpr int nb_fwd = (kBendWBytes / 2 + kPackThreads - 1) / kPackThreads;
  if (blockIdx.x < nb_fwd) pack_bender_elem(blockIdx.x * kPackThreads + threadIdx.x, src, w, bias, wlo);
  else pack_bender_t_elem((blockIdx.x - nb_fwd) * kPackThreads + threadIdx.x, src, wt, wtlo);
}

// View-dependent head (layout in nrn_common.cuh, views::): feature_linear; views_linears.0 split at input column 256
// into its direction-encoding columns (ViewsE, K = 27 padded to 32) and its feature columns (ViewsF); rgb_linear (N = 3
// padded to 16).  Forward images only.
__global__ void __launch_bounds__(kPackThreads) pack_views_kernel(ViewsSrc src, __half* __restrict__ w, float* __restrict__ bias) {
  using namespace views;
  constexpr WImage wf = image(Feature), we = image(ViewsE), wv = image(ViewsF), wr = image(Rgb);
  constexpr int nf = wf.bytes() / 2, ne = we.bytes() / 2, nv = wv.bytes() / 2;
  constexpr int ldv = 256 + kDirCols;   // views_linears.0: [feature(256) | direction encoding(27)] inputs
  const int idx = blockIdx.x * kPackThreads + threadIdx.x;
  if (idx < kViewsWBytes / 2) {
    int i = idx, k, r;
    float v = 0.f;
    if (i < nf) {                          // Feature
      decode(i, wf.rows, k, r);
      v = src.w[0][r * 256 + k];
    } else if ((i -= nf) < ne) {           // ViewsE: K = direction encoding, padded to 32
      decode(i, we.rows, k, r);
      v = k < kDirCols ? src.w[1][r * ldv + 256 + k] : 0.f;
    } else if ((i -= ne) < nv) {           // ViewsF: K = feature
      decode(i, wv.rows, k, r);
      v = src.w[1][r * ldv + k];
    } else {                               // Rgb: N = 3 padded to 16
      i -= nv;
      decode(i, wr.rows, k, r);
      v = r < 3 ? src.w[2][r * 128 + k] : 0.f;
    }
    w[idx] = __float2half_rn(v);
  }
  if (idx < kViewsBiasFloats) {
    constexpr int bv = b_off(ViewsF), br = b_off(Rgb);
    bias[idx] = idx < bv ? src.b[0][idx] : idx < br ? src.b[1][idx - bv] : (idx - br < 3 ? src.b[2][idx - br] : 0.f);
  }
}

}  // namespace

cudaError_t launch_pack_views(const ViewsSrc& src, void* packed, cudaStream_t st) {
  uint8_t* base = reinterpret_cast<uint8_t*>(packed);
  const int nb = (kViewsWBytes / 2 + kPackThreads - 1) / kPackThreads;
  pack_views_kernel<<<nb, kPackThreads, 0, st>>>(src, reinterpret_cast<__half*>(base), reinterpret_cast<float*>(base + kViewsWBytes));
  return cudaGetLastError();
}

// packed = [forward images | biases | transposed images] (+ the bender's residual images; offsets in nrn_common.cuh)
cudaError_t launch_pack_nerf(const NerfSrc& src, int in_ch, int out_ch, void* packed, cudaStream_t st) {
  uint8_t* base = reinterpret_cast<uint8_t*>(packed);
  const int nb = (kNerfWBytes / 2 + kPackThreads - 1) / kPackThreads + (kNerfTWBytes / 2 + kPackThreads - 1) / kPackThreads;
  if (in_ch == kPeCols + kLatent)   // time-conditioned baseline: [embedding | latent] inputs
    pack_nerf_tc_kernel<<<nb, kPackThreads, 0, st>>>(src, out_ch, reinterpret_cast<__half*>(base), reinterpret_cast<float*>(base + kNerfWBytes),
                                                     reinterpret_cast<__half*>(base + kNerfTOffset));
  else
    pack_nerf_kernel<<<nb, kPackThreads, 0, st>>>(src, in_ch, out_ch, reinterpret_cast<__half*>(base),
                                                 reinterpret_cast<float*>(base + kNerfWBytes), reinterpret_cast<__half*>(base + kNerfTOffset));
  return cudaGetLastError();
}
cudaError_t launch_pack_bender(const BenderSrc& src, void* packed, cudaStream_t st) {
  uint8_t* base = reinterpret_cast<uint8_t*>(packed);
  const int nb = (kBendWBytes / 2 + kPackThreads - 1) / kPackThreads + (kBendTWBytes / 2 + kPackThreads - 1) / kPackThreads;
  pack_bender_kernel<<<nb, kPackThreads, 0, st>>>(src, reinterpret_cast<__half*>(base), reinterpret_cast<float*>(base + kBendWBytes),
                                                 reinterpret_cast<__half*>(base + kBendTOffset), reinterpret_cast<__half*>(base + kBendLoOffset),
                                                 reinterpret_cast<__half*>(base + kBendTLoOffset));
  return cudaGetLastError();
}

}  // namespace nrn
