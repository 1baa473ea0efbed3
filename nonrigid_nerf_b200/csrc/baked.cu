// Baked canonical radiance grids: the fp16 plane store of a bake, and the grid lookup of a render pass without a ray
// bender (with one, field_fwd.cu's field_baked_kernel does the lookup in the bend pass's epilogue).  baked.cuh has the rules.
//
// Baked per-frame deformation grids: the fp16 plane store of their bake, and the kernels of a render pass that looks each
// sample's bend up in place of the ray-bender MLP (c_abi.cu: nrn_field_forward_deformed): the per-ray vote and lookup, the
// compaction and gather of the rays that fall back to the exact bender, and the scatter of what the bend pass made of them.
#include <cub/block/block_scan.cuh>
#include "baked.cuh"
#include "occupancy.cuh"

namespace nrn {
namespace {

constexpr int kBakedThreads = 256;
constexpr int kLatentRow = 32;   // floats per gathered latent row

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

// ---- baked per-frame deformation grids ----
__global__ void __launch_bounds__(kBakedThreads) deform_plane_kernel(const float* __restrict__ offsets, const float* __restrict__ rigidity,
                                                                     long long n, uint2* __restrict__ plane) {
  for (long long q = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; q < n; q += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float* o = offsets + q * 3;
    const __half2 h01 = __halves2half2(baked_half(__ldg(o + 0)), baked_half(__ldg(o + 1)));
    const __half2 h23 = __halves2half2(baked_half(__ldg(o + 2)), baked_half(__ldg(rigidity + q)));
    plane[q] = make_uint2(*reinterpret_cast<const uint32_t*>(&h01), *reinterpret_cast<const uint32_t*>(&h23));
  }
}

__device__ __forceinline__ void store3(float* d, long long pt, float a, float b, float c) {
  if (d) { d[pt * 3 + 0] = a; d[pt * 3 + 1] = b; d[pt * 3 + 2] = c; }
}

// A warp per ray.  Lanes take samples s = lane, lane + 32, ...; the ray is deformed when every lane's samples are inside
// the deformation grid's box (a vote), and only then are its samples written.
__global__ void __launch_bounds__(kBakedThreads) deform_rays_kernel(const BakedGrid dg, const BakedGrid rg, const DeformKnobs k,
                                                                    const float* __restrict__ rays, const float* __restrict__ z_vals,
                                                                    int n_rays, int S, const DeformOut o, uint8_t* __restrict__ fallback) {
  constexpr int kWarps = kBakedThreads / 32;
  const int lane = threadIdx.x & 31;
  for (long long ray = blockIdx.x * static_cast<long long>(kWarps) + (threadIdx.x >> 5); ray < n_rays;
       ray += static_cast<long long>(gridDim.x) * kWarps) {
    const float* r = rays + ray * 8;
    const float ro[3] = {__ldg(r + 0), __ldg(r + 1), __ldg(r + 2)}, rd[3] = {__ldg(r + 3), __ldg(r + 4), __ldg(r + 5)};
    const long long base = ray * S;
    bool inside = true;
    for (int s = lane; s < S; s += 32) {
      const float z = __ldg(z_vals + base + s);
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        const float x = __fadd_rn(ro[d], __fmul_rn(rd[d], z));   // multiply, then add
        inside &= x >= dg.lo[d] && x <= dg.hi[d];
      }
    }
    const bool falls_back = !__all_sync(0xffffffffu, inside);
    if (lane == 0) fallback[ray] = falls_back ? 1 : 0;
    if (falls_back) continue;
    for (int s = lane; s < S; s += 32) {
      const long long pt = base + s;
      const float z = __ldg(z_vals + pt);
      float x[3], v[4], m[3], c[3];
#pragma unroll
      for (int d = 0; d < 3; ++d) x[d] = __fadd_rn(ro[d], __fmul_rn(rd[d], z));
      baked_lookup(dg, x, v);   // inside, by the vote
      const float rt = k.use_cutoff && v[3] <= k.cutoff ? 0.f : v[3];
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        m[d] = __fmul_rn(rt, v[d]);
        if (k.use_scaling) m[d] = __fmul_rn(m[d], k.scaling);
        c[d] = __fadd_rn(x[d], m[d]);
      }
      o.ws[pt] = make_float4(c[0], c[1], c[2], rt);
      store3(o.d_init, pt, x[0], x[1], x[2]);
      store3(o.d_bent, pt, c[0], c[1], c[2]);
      store3(o.d_unmasked, pt, v[0], v[1], v[2]);
      store3(o.d_masked, pt, m[0], m[1], m[2]);
      if (o.d_rigid) o.d_rigid[pt] = rt;
      baked_raw(rg, c, k.use_removal && rt >= k.removal, o.raw, pt, o.out_ch);
    }
  }
}

// The fixed-order compaction of the fallback flags (occupancy.cu's block scan): per-block counts, one scan, per-block writes
__global__ void __launch_bounds__(kOccTile) deform_count_kernel(const uint8_t* __restrict__ flag, int n, int32_t* __restrict__ block_counts) {
  const long long i = static_cast<long long>(blockIdx.x) * kOccTile + threadIdx.x;
  const int cnt = __syncthreads_count(i < n && __ldg(flag + i));
  if (threadIdx.x == 0) block_counts[blockIdx.x] = cnt;
}

__global__ void __launch_bounds__(kOccTile) deform_write_kernel(const uint8_t* __restrict__ flag, int n, const int32_t* __restrict__ block_counts,
                                                                int32_t* __restrict__ idx) {
  using Scan = cub::BlockScan<int, kOccTile>;
  __shared__ typename Scan::TempStorage tmp;
  const long long i = static_cast<long long>(blockIdx.x) * kOccTile + threadIdx.x;
  const bool keep = i < n && __ldg(flag + i);
  int rank;
  Scan(tmp).ExclusiveSum(keep ? 1 : 0, rank);
  if (keep) idx[__ldg(block_counts + blockIdx.x) + rank] = static_cast<int32_t>(i);
}

// rays [K][8], depths [K][S] and latent rows [K][32] of the K fallback rays, K read on the device
__global__ void __launch_bounds__(kBakedThreads) deform_gather_kernel(const DeformFallback f, const float* __restrict__ rays,
                                                                      const float* __restrict__ z_vals, const float* __restrict__ latents,
                                                                      long long latent_stride, int S) {
  const long long K = __ldg(f.count);
  const long long q0 = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x, step = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long q = q0; q < K * S; q += step) {
    const long long j = q / S;
    f.z_vals[q] = __ldg(z_vals + static_cast<long long>(__ldg(f.idx + j)) * S + (q - j * S));
  }
  for (long long q = q0; q < K * 8; q += step) f.rays[q] = __ldg(rays + static_cast<long long>(__ldg(f.idx + q / 8)) * 8 + q % 8);
  for (long long q = q0; q < K * kLatentRow; q += step)
    f.latents[q] = __ldg(latents + static_cast<long long>(__ldg(f.idx + q / kLatentRow)) * latent_stride + q % kLatentRow);
}

__device__ __forceinline__ void copy3(const float* s, float* d, long long q, long long pt) {
  if (d) { d[pt * 3 + 0] = __ldg(s + q * 3 + 0); d[pt * 3 + 1] = __ldg(s + q * 3 + 1); d[pt * 3 + 2] = __ldg(s + q * 3 + 2); }
}

__global__ void __launch_bounds__(kBakedThreads) deform_scatter_kernel(const BakedGrid rg, const DeformKnobs k, const DeformFallback f,
                                                                       const float4* __restrict__ bw, const DeformOut from, int S,
                                                                       const DeformOut to) {
  const long long K = __ldg(f.count);
  for (long long q = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; q < K * S; q += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long j = q / S;
    const long long pt = static_cast<long long>(__ldg(f.idx + j)) * S + (q - j * S);
    const float4 w = __ldg(bw + q);
    to.ws[pt] = w;
    copy3(from.d_init, to.d_init, q, pt);
    copy3(from.d_bent, to.d_bent, q, pt);
    copy3(from.d_unmasked, to.d_unmasked, q, pt);
    copy3(from.d_masked, to.d_masked, q, pt);
    if (to.d_rigid) to.d_rigid[pt] = __ldg(from.d_rigid + q);
    const float x[3] = {w.x, w.y, w.z};
    baked_raw(rg, x, k.use_removal && w.w >= k.removal, to.raw, pt, to.out_ch);
  }
}

// Blocks of a grid-stride launch over at most n items whose count is read on the device
unsigned capped_blocks(long long n, int num_sms) {
  const long long nb = (n + kBakedThreads - 1) / kBakedThreads, cap = static_cast<long long>(num_sms) * 16;
  return static_cast<unsigned>(nb < 1 ? 1 : nb < cap ? nb : cap);
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

cudaError_t launch_deform_plane(const float* offsets, const float* rigidity, long long n, uint2* plane, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  deform_plane_kernel<<<blocks_for(n), kBakedThreads, 0, st>>>(offsets, rigidity, n, plane);
  return cudaGetLastError();
}

cudaError_t launch_deform_rays(const BakedGrid& dg, const BakedGrid& rg, const DeformKnobs& k, const float* rays, const float* z_vals,
                               int n_rays, int S, const DeformOut& o, uint8_t* fallback, cudaStream_t st) {
  if (n_rays <= 0) return cudaSuccess;
  constexpr int kWarps = kBakedThreads / 32;
  const long long nb = (n_rays + kWarps - 1) / kWarps;
  deform_rays_kernel<<<static_cast<unsigned>(nb < (1 << 20) ? nb : (1 << 20)), kBakedThreads, 0, st>>>(dg, rg, k, rays, z_vals, n_rays, S, o,
                                                                                                       fallback);
  return cudaGetLastError();
}

cudaError_t launch_deform_fallback(const DeformFallback& f, const float* rays, const float* z_vals, const float* latents,
                                   long long latent_stride, int n_rays, int S, int num_sms, cudaStream_t st) {
  const unsigned nb = static_cast<unsigned>((static_cast<long long>(n_rays) + kOccTile - 1) / kOccTile);
  if (nb > 0) deform_count_kernel<<<nb, kOccTile, 0, st>>>(f.flag, n_rays, f.block_counts);
  cudaError_t e = launch_occupancy_scan(f.block_counts, static_cast<int>(nb), f.count, st);
  if (e != cudaSuccess) return e;
  if (nb == 0) return cudaGetLastError();
  deform_write_kernel<<<nb, kOccTile, 0, st>>>(f.flag, n_rays, f.block_counts, f.idx);
  deform_gather_kernel<<<capped_blocks(static_cast<long long>(n_rays) * (S > kLatentRow ? S : kLatentRow), num_sms), kBakedThreads, 0, st>>>(
      f, rays, z_vals, latents, latent_stride, S);
  return cudaGetLastError();
}

cudaError_t launch_deform_scatter(const BakedGrid& rg, const DeformKnobs& k, const DeformFallback& f, const float4* bw, const DeformOut& from,
                                  int n_rays, int S, const DeformOut& to, int num_sms, cudaStream_t st) {
  if (n_rays <= 0) return cudaSuccess;
  deform_scatter_kernel<<<capped_blocks(static_cast<long long>(n_rays) * S, num_sms), kBakedThreads, 0, st>>>(rg, k, f, bw, from, S, to);
  return cudaGetLastError();
}

}  // namespace nrn
