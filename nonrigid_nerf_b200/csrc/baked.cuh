// Baked canonical radiance grids (baked.cu, field_fwd.cu's field_baked_kernel): the fp16 store of a bake's planes and the
// trilinear lookup a render pass runs in place of the NeRF trunk for samples inside the grid's box.  Baked per-frame
// deformation grids store the ray bender's (offset, rigidity) the same way and are looked up by the same rule.
//
// A grid has n[0] x n[1] x n[2] vertices over [lo, hi]; vertex (i, j, k) holds the 4 raw channels of the canonical model at
// the mesh grid's point (i, j, k) (mesh.cu's grid_coord), as fp16 at vox[(k * ny + j) * nx + i]: one 8-byte load per corner.
// Every floating-point step of the lookup is an explicit _rn intrinsic, so tests/baked_reference.py restates it in numpy fp32
// bit for bit.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace nrn {

constexpr int kBakedMinSide = 2;
constexpr int kBakedMaxSide = 1024;   // vertices per axis

struct BakedGrid {
  const uint2* vox;   // [nz][ny][nx] x 4 fp16
  int n[3];           // vertices per axis
  float lo[3], hi[3];
  float scale[3];     // fl((n - 1) / fl(hi - lo)), computed on the host
};

// fp32 -> fp16, round to nearest even; finite values beyond fp16's range saturate to +-65504, inf and NaN stay non-finite
__device__ __forceinline__ __half baked_half(float v) {
  return __float2half_rn(isfinite(v) ? fminf(fmaxf(v, -65504.f), 65504.f) : v);
}

__device__ __forceinline__ float baked_lerp(float a, float b, float t) { return __fadd_rn(a, __fmul_rn(t, __fsub_rn(b, a))); }

// A point is looked up when every coordinate is finite and lo <= x <= hi.  Then per axis u = fl(fl(x - lo) * scale),
// i = min(floor(u), n - 2), f = fl(u - i), and the 8 corners are blended along x, then y, then z, each step a + f (b - a).
// Returns false (o untouched) for any other point: the trunk evaluates it.
__device__ __forceinline__ bool baked_lookup(const BakedGrid& g, const float (&x)[3], float (&o)[4]) {
  int c[3];
  float f[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    if (!(x[d] >= g.lo[d] && x[d] <= g.hi[d])) return false;
    const float u = __fmul_rn(__fsub_rn(x[d], g.lo[d]), g.scale[d]);
    c[d] = min(static_cast<int>(floorf(u)), g.n[d] - 2);
    f[d] = __fsub_rn(u, static_cast<float>(c[d]));
  }
  const long long sy = g.n[0], sz = static_cast<long long>(g.n[0]) * g.n[1];
  const uint2* b = g.vox + c[2] * sz + c[1] * sy + c[0];
  float yz[4][4];   // [dz * 2 + dy][channel]: the x-blends
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const uint2* r = b + (q >> 1) * sz + (q & 1) * sy;
    const uint2 v0 = __ldg(r), v1 = __ldg(r + 1);
    const float2 a01 = __half22float2(*reinterpret_cast<const __half2*>(&v0.x)), a23 = __half22float2(*reinterpret_cast<const __half2*>(&v0.y));
    const float2 b01 = __half22float2(*reinterpret_cast<const __half2*>(&v1.x)), b23 = __half22float2(*reinterpret_cast<const __half2*>(&v1.y));
    yz[q][0] = baked_lerp(a01.x, b01.x, f[0]);
    yz[q][1] = baked_lerp(a01.y, b01.y, f[0]);
    yz[q][2] = baked_lerp(a23.x, b23.x, f[0]);
    yz[q][3] = baked_lerp(a23.y, b23.y, f[0]);
  }
#pragma unroll
  for (int ch = 0; ch < 4; ++ch) o[ch] = baked_lerp(baked_lerp(yz[0][ch], yz[1][ch], f[1]), baked_lerp(yz[2][ch], yz[3][ch], f[1]), f[2]);
  return true;
}

// raw of point pt from the grid when it is inside the box (alpha zeroed like the fused kernel's test-time object removal
// where removed; channel 4 of a 5-channel raw, which compositing does not read, is 0).  Points outside are left alone.
__device__ __forceinline__ void baked_raw(const BakedGrid& g, const float (&x)[3], bool removed, float* __restrict__ raw, long long pt,
                                          int out_ch) {
  float o[4];
  if (!baked_lookup(g, x, o)) return;
  if (removed) o[3] *= 0.f;
  float* dst = raw + pt * out_ch;
  dst[0] = o[0]; dst[1] = o[1]; dst[2] = o[2]; dst[3] = o[3];
  if (out_ch == 5) dst[4] = 0.f;
}

// plane [n] x 4 fp16 <- baked_half of raw [n][out_ch] channels 0..3
cudaError_t launch_baked_plane(const float* raw, long long n, int out_ch, uint2* plane, cudaStream_t st);
// Without a bender: raw of every sample of rays x z inside the grid's box, at rays_o + rays_d * z (the field kernel's rounding)
cudaError_t launch_baked_rays(const BakedGrid& g, const float* rays, const float* z_vals, int S, long long P, float* raw, int out_ch,
                              cudaStream_t st);

// ---- baked per-frame deformation grids (c_abi.cu: nrn_field_forward_deformed) ----
// One frame's grid is a BakedGrid whose 4 channels are the bender's unmasked offset o (0..2) and rigidity r (3), looked up
// with baked_lookup.  A ray is DEFORMED when every one of its samples x = o + d z is finite and inside the grid's box; then
// per sample r~ = (use_cutoff && r <= cutoff) ? 0 : r, m = fl(r~ o), m = fl(m s) with scaling, c = fl(x + m).  Any other ray
// FALLS BACK: the bend pass bends it exactly, so its samples come out as the baked pass without a deformation grid.

// The per-sample outputs of a deformed pass: the bend workspace (c, r~) as the bend pass writes it, raw of the samples whose
// c the radiance grid looks up, and the details (each may be null)
struct DeformOut {
  float4* ws;
  float* raw;
  int out_ch;
  float* d_init;
  float* d_bent;
  float* d_unmasked;
  float* d_masked;
  float* d_rigid;
};

struct DeformKnobs {
  int use_cutoff, use_scaling, use_removal;
  float cutoff, scaling, removal;
};

// The fallback rays, compacted in ascending order: their count K (device memory), their indices, and their rays [K][8],
// depths [K][S] and latent rows [K][32] gathered for the bend pass
struct DeformFallback {
  uint8_t* flag;           // [n_rays] 1: the ray falls back
  int32_t* block_counts;   // ceil(n_rays / kOccTile) + 1
  int32_t* count;
  int32_t* idx;
  float* rays;
  float* z_vals;
  float* latents;
};

// plane [n] x 4 fp16 <- baked_half of (offsets [n][3], rigidity [n])
cudaError_t launch_deform_plane(const float* offsets, const float* rigidity, long long n, uint2* plane, cudaStream_t st);
// A warp per ray: the vote, and for a deformed ray every sample's c and r~ -> o.ws, the details, and raw where rg looks c up
cudaError_t launch_deform_rays(const BakedGrid& dg, const BakedGrid& rg, const DeformKnobs& k, const float* rays, const float* z_vals,
                               int n_rays, int S, const DeformOut& o, uint8_t* fallback, cudaStream_t st);
// The fallback rays in ascending order (count, indices), and their rays, depths and latent rows gathered
cudaError_t launch_deform_fallback(const DeformFallback& f, const float* rays, const float* z_vals, const float* latents,
                                   long long latent_stride, int n_rays, int S, int num_sms, cudaStream_t st);
// The bend pass's outputs over the gathered rays (bend workspace bw, details of `from`) back to the fallback rays' samples of
// `to`, and raw where rg looks their bent points up (the object removal as the bend pass with the lookup applies it)
cudaError_t launch_deform_scatter(const BakedGrid& rg, const DeformKnobs& k, const DeformFallback& f, const float4* bw, const DeformOut& from,
                                  int n_rays, int S, const DeformOut& to, int num_sms, cudaStream_t st);

}  // namespace nrn
