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

__device__ __forceinline__ void pack_nerf_elem(const int idx, const NerfSrc& src, int in_ch, int out_ch, __half* __restrict__ w, float* __restrict__ bias) {
  constexpr int n0 = kNerfL0Bytes / 2, nl = kNerfLBytes / 2, n5 = kNerfL5Bytes / 2, nh = kNerfHeadBytes / 2;
  if (idx < kNerfWBytes / 2) {
    int i = idx, k, r;
    float v = 0.f;
    if (i < n0) {  // L0: K = in_ch (63) padded to 64
      decode(i, 256, k, r);
      v = k < in_ch ? src.w[0][r * in_ch + k] : 0.f;
    } else if ((i -= n0) < 4 * nl) {  // L1..L4
      const int L = 1 + i / nl;
      decode(i % nl, 256, k, r);
      v = src.w[L][r * 256 + k];
    } else if ((i -= 4 * nl) < n5) {  // L5: [embedding(in_ch) pad | h(256)]
      decode(i, 256, k, r);
      const int ld = in_ch + 256;
      if (k < 64) v = k < in_ch ? src.w[5][r * ld + k] : 0.f;
      else v = src.w[5][r * ld + in_ch + (k - 64)];
    } else if ((i -= n5) < 2 * nl) {  // L6, L7
      const int L = 6 + i / nl;
      decode(i % nl, 256, k, r);
      v = src.w[L][r * 256 + k];
    } else {  // head, N padded to 16
      i -= 2 * nl;
      decode(i, 16, k, r);
      v = r < out_ch ? src.w[8][r * 256 + k] : 0.f;
    }
    w[idx] = __float2half_rn(v);
  }
  if (idx < kNerfBiasFloats) {
    float b;
    if (idx < 2048) b = src.b[idx >> 8][idx & 255];
    else b = (idx - 2048) < out_ch ? src.b[8][idx - 2048] : 0.f;
    bias[idx] = b;
  }
  (void)nh;
}

__device__ __forceinline__ void pack_bender_elem(const int idx, const BenderSrc& src, __half* __restrict__ w, float* __restrict__ bias) {
  constexpr int n0 = kBendB0Bytes / 2, n1 = kBendB1Bytes / 2, n2 = kBendB2Bytes / 2, n3 = kBendB3Bytes / 2;
  constexpr int ld0 = 3 + kLatent;
  if (idx < kBendWBytes / 2) {
    int i = idx, k, r;
    float v = 0.f;
    if (i < n0) {  // B0: K = [xyz_hi xyz_lo latent pad] = 48
      decode(i, 96, k, r);
      if (r < 64) {
        if (k < 3) v = src.net_w[0][r * ld0 + k];
        else if (k < 6) v = src.net_w[0][r * ld0 + (k - 3)];
        else if (k < 6 + kLatent) v = src.net_w[0][r * ld0 + 3 + (k - 6)];
      } else {
        if (k < 3) v = src.rig_w[0][(r - 64) * 3 + k];
        else if (k < 6) v = src.rig_w[0][(r - 64) * 3 + (k - 3)];
      }
    } else if ((i -= n0) < n1) {  // B1: block diagonal 64x64 + 32x32
      decode(i, 96, k, r);
      if (r < 64) { if (k < 64) v = src.net_w[1][r * 64 + k]; }
      else { if (k >= 64) v = src.rig_w[1][(r - 64) * 32 + (k - 64)]; }
    } else if ((i -= n1) < n2) {  // B2: offset L2 + rigidity output row
      decode(i, 80, k, r);
      if (r < 64) { if (k < 64) v = src.net_w[2][r * 64 + k]; }
      else if (r == 64) { if (k >= 64) v = src.rig_w[2][k - 64]; }
    } else if ((i -= n2) < n3) {  // B3
      decode(i, 64, k, r);
      v = src.net_w[3][r * 64 + k];
    } else {  // B4: 3 output rows, no bias
      i -= n3;
      decode(i, 16, k, r);
      if (r < 3) v = src.net_w[4][r * 64 + k];
    }
    w[idx] = __float2half_rn(v);
  }
  if (idx < kBendBiasFloats) {
    float b = 0.f;
    if (idx < 96) b = idx < 64 ? src.net_b[0][idx] : src.rig_b[0][idx - 64];
    else if (idx < 192) { const int j = idx - 96; b = j < 64 ? src.net_b[1][j] : src.rig_b[1][j - 64]; }
    else if (idx < 272) { const int j = idx - 192; b = j < 64 ? src.net_b[2][j] : (j == 64 ? src.rig_b[2][0] : 0.f); }
    else b = src.net_b[3][idx - 272];
    bias[idx] = b;
  }
}

// ---- transposed images for DGRAD: W^T (rows = input features, K = output features), layout in nrn_common.cuh ----
// r = input feature, k = output feature
__device__ __forceinline__ void pack_nerf_t_elem(const int idx, const NerfSrc& src, int in_ch, int out_ch, __half* __restrict__ w) {
  if (idx >= kNerfTWBytes / 2) return;
  constexpr int nh = kNerfTHeadBytes / 2, nl = kNerfLBytes / 2, ne = kNerfTEBytes / 2;
  int i = idx, k, r;
  float v = 0.f;
  const int ld5 = in_ch + 256;
  if (i < nh) {                           // head^T: K = out_ch padded to 16
    decode(i, 256, k, r);
    v = k < out_ch ? src.w[8][k * 256 + r] : 0.f;
  } else if ((i -= nh) < 2 * nl) {        // L7^T, L6^T
    const int L = 7 - i / nl;
    decode(i % nl, 256, k, r);
    v = src.w[L][k * 256 + r];
  } else if ((i -= 2 * nl) < ne) {        // L5e^T: rows = embedding inputs (in_ch, padded to 64)
    decode(i, 64, k, r);
    v = r < in_ch ? src.w[5][k * ld5 + r] : 0.f;
  } else if ((i -= ne) < nl) {            // L5h^T
    decode(i, 256, k, r);
    v = src.w[5][k * ld5 + in_ch + r];
  } else if ((i -= nl) < 4 * nl) {        // L4^T .. L1^T
    const int L = 4 - i / nl;
    decode(i % nl, 256, k, r);
    v = src.w[L][k * 256 + r];
  } else {                                // L0^T
    i -= 4 * nl;
    decode(i, 64, k, r);
    v = r < in_ch ? src.w[0][k * in_ch + r] : 0.f;
  }
  w[idx] = __float2half_rn(v);
}

__device__ __forceinline__ void pack_bender_t_elem(const int idx, const BenderSrc& src, __half* __restrict__ w) {
  if (idx >= kBendTWBytes / 2) return;
  constexpr int n4 = kBendTB4Bytes / 2, n3 = kBendTB3Bytes / 2, n2 = kBendTB2Bytes / 2, n1 = kBendTB1Bytes / 2;
  constexpr int ld0 = 3 + kLatent;
  int i = idx, k, r;
  float v = 0.f;
  if (i < n4) {                           // B4^T: rows = 64 hidden, K = 3 outputs (padded to 16)
    decode(i, 64, k, r);
    v = k < 3 ? src.net_w[4][k * 64 + r] : 0.f;
  } else if ((i -= n4) < n3) {            // B3^T
    decode(i, 64, k, r);
    v = src.net_w[3][k * 64 + r];
  } else if ((i -= n3) < n2) {            // B2^T: rows = 96 inputs, K = 80 outputs (64 offset, 1 rigidity, pad)
    decode(i, 96, k, r);
    if (r < 64) { if (k < 64) v = src.net_w[2][k * 64 + r]; }
    else { if (k == 64) v = src.rig_w[2][r - 64]; }
  } else if ((i -= n2) < n1) {            // B1^T: block diagonal
    decode(i, 96, k, r);
    if (r < 64) { if (k < 64) v = src.net_w[1][k * 64 + r]; }
    else { if (k >= 64) v = src.rig_w[1][(k - 64) * 32 + (r - 64)]; }
  } else {                                // B0^T: rows = 48 inputs [xyz_hi xyz_lo latent pad], K = 96 outputs
    i -= n1;
    decode(i, 48, k, r);
    if (r >= 6 && r < 6 + kLatent) { if (k < 64) v = src.net_w[0][k * ld0 + 3 + (r - 6)]; }
    else if (r < 3) v = k < 64 ? src.net_w[0][k * ld0 + r] : src.rig_w[0][(k - 64) * 3 + r];
  }
  w[idx] = __float2half_rn(v);
}


// one launch per module: the first blocks write the forward images (+ biases), the rest the transposed images
constexpr int kPackThreads = 256;
__global__ void __launch_bounds__(kPackThreads) pack_nerf_kernel(NerfSrc src, int in_ch, int out_ch, __half* __restrict__ w,
                                                                 float* __restrict__ bias, __half* __restrict__ wt) {
  constexpr int nb_fwd = (kNerfWBytes / 2 + kPackThreads - 1) / kPackThreads;
  if (blockIdx.x < nb_fwd) pack_nerf_elem(blockIdx.x * kPackThreads + threadIdx.x, src, in_ch, out_ch, w, bias);
  else pack_nerf_t_elem((blockIdx.x - nb_fwd) * kPackThreads + threadIdx.x, src, in_ch, out_ch, wt);
}
__global__ void __launch_bounds__(kPackThreads) pack_bender_kernel(BenderSrc src, __half* __restrict__ w, float* __restrict__ bias,
                                                                   __half* __restrict__ wt) {
  constexpr int nb_fwd = (kBendWBytes / 2 + kPackThreads - 1) / kPackThreads;
  if (blockIdx.x < nb_fwd) pack_bender_elem(blockIdx.x * kPackThreads + threadIdx.x, src, w, bias);
  else pack_bender_t_elem((blockIdx.x - nb_fwd) * kPackThreads + threadIdx.x, src, wt);
}

}  // namespace

// packed = [forward images | biases | transposed images] (offsets in nrn_common.cuh)
cudaError_t launch_pack_nerf(const NerfSrc& src, int in_ch, int out_ch, void* packed, cudaStream_t st) {
  uint8_t* base = reinterpret_cast<uint8_t*>(packed);
  const int nb = (kNerfWBytes / 2 + kPackThreads - 1) / kPackThreads + (kNerfTWBytes / 2 + kPackThreads - 1) / kPackThreads;
  pack_nerf_kernel<<<nb, kPackThreads, 0, st>>>(src, in_ch, out_ch, reinterpret_cast<__half*>(base),
                                               reinterpret_cast<float*>(base + kNerfWBytes), reinterpret_cast<__half*>(base + kNerfTOffset));
  return cudaGetLastError();
}
cudaError_t launch_pack_bender(const BenderSrc& src, void* packed, cudaStream_t st) {
  uint8_t* base = reinterpret_cast<uint8_t*>(packed);
  const int nb = (kBendWBytes / 2 + kPackThreads - 1) / kPackThreads + (kBendTWBytes / 2 + kPackThreads - 1) / kPackThreads;
  pack_bender_kernel<<<nb, kPackThreads, 0, st>>>(src, reinterpret_cast<__half*>(base), reinterpret_cast<float*>(base + kBendWBytes),
                                                 reinterpret_cast<__half*>(base + kBendTOffset));
  return cudaGetLastError();
}

}  // namespace nrn
