// Occupancy grid of the canonical volume, and the kernels of a render pass that skips the NeRF trunk for samples that bend
// into empty cells (c_abi.cu: nrn_field_forward_occupancy).
//
// Build: a cell is occupied when any of its 8 corner densities is > threshold or NaN; the occupied set is dilated by d
// cells in the Chebyshev sense (three separable passes, one per axis) and packed to bits, 32 cells per word.
//
// Pass: after the bend pass (or, without a bender, from the rays and depths), each point is looked up in the grid.  Points
// outside the box or with a non-finite coordinate are kept.  The kept points are compacted in ascending point order by a
// fixed block scan (per-block counts, one scan of the counts, per-block writes: no atomics decide the order), with K
// written to device memory; the point-mode trunk runs on them reading K from there, and the scatter writes their raw to
// the pass's [N, S, C] output, which is zero everywhere else.  Every floating-point step of the lookup is an explicit _rn
// intrinsic, so a numpy restatement in fp32 reproduces it (tests/occupancy_reference.py).
//
// Early termination (c_abi.cu: nrn_field_forward_terminate) runs the same steps in rounds over segments of the samples:
// the lookup of a round covers only its segment's slots and keeps those of rays still alive (and, with a grid, those the
// grid keeps), through the same count / write bodies as the lookup above; after the trunk and the scatter, a per-ray
// kernel multiplies the ray's transmittance by the segment's (1 - alpha + 1e-10) and marks the ray dead below the
// threshold.
#include <cub/block/block_scan.cuh>
#include "occupancy.cuh"
#include "ray_ops.cuh"

namespace nrn {
namespace {

constexpr int kOccThreads = 256;

__global__ void __launch_bounds__(kOccThreads) occ_corner_kernel(const float* __restrict__ sigma, int nx, int ny, int nz, float t,
                                                                 uint8_t* __restrict__ occ) {
  const long long n = static_cast<long long>(nx) * ny * nz;
  const long long c = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (c >= n) return;
  const int i = static_cast<int>(c % nx), j = static_cast<int>((c / nx) % ny), k = static_cast<int>(c / (static_cast<long long>(nx) * ny));
  const long long vx = nx + 1, vxy = vx * (ny + 1);
  const float* s = sigma + k * vxy + j * vx + i;
  bool o = false;
#pragma unroll
  for (int q = 0; q < 8; ++q) o |= !(__ldg(s + ((q >> 2) & 1) * vxy + ((q >> 1) & 1) * vx + (q & 1)) <= t);   // NaN is occupied
  occ[c] = o ? 1 : 0;
}

// out[c] = OR of in over the cells within d of c along `axis` (0 = x, 1 = y, 2 = z)
__global__ void __launch_bounds__(kOccThreads) occ_dilate_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int nx, int ny,
                                                                 int nz, int axis, int d) {
  const long long n = static_cast<long long>(nx) * ny * nz;
  const long long c = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (c >= n) return;
  const long long stride = axis == 0 ? 1 : axis == 1 ? nx : static_cast<long long>(nx) * ny;
  const int len = axis == 0 ? nx : axis == 1 ? ny : nz;
  const int a = static_cast<int>((c / stride) % len);
  const int a0 = max(a - d, 0), a1 = min(a + d, len - 1);
  uint8_t o = 0;
  for (int b = a0; b <= a1 && !o; ++b) o = __ldg(in + c + (b - a) * stride);
  out[c] = o;
}

// 32 consecutive cells -> one word (cell c at bit c % 32)
__global__ void __launch_bounds__(kOccThreads) occ_pack_kernel(const uint8_t* __restrict__ occ, long long n, uint32_t* __restrict__ bits) {
  const long long c = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const unsigned w = __ballot_sync(0xffffffffu, c < n && __ldg(occ + c) != 0);
  if ((threadIdx.x & 31) == 0 && c < n) bits[c >> 5] = w;
}

__device__ __forceinline__ void occ_point(const OccPoints& s, long long i, float (&x)[3]) {
  if (s.ws) {
    const float4 q = __ldg(s.ws + i);
    x[0] = q.x; x[1] = q.y; x[2] = q.z;
  } else if (s.pts) {
    const float* q = s.pts + i * s.pts_stride;
    x[0] = __ldg(q + 0); x[1] = __ldg(q + 1); x[2] = __ldg(q + 2);
  } else {   // pts = rays_o + rays_d * z, multiply then add like the field kernel
    const float z = __ldg(s.z_vals + i);
    const float* r = s.rays + (i / s.S) * 8;
#pragma unroll
    for (int d = 0; d < 3; ++d) x[d] = __fadd_rn(__ldg(r + d), __fmul_rn(__ldg(r + 3 + d), z));
  }
}

// Kept: outside the box, non-finite, or in an occupied cell
__device__ __forceinline__ bool occ_keep(const OccGrid& g, const float (&x)[3]) {
  const int n[3] = {g.nx, g.ny, g.nz};
  int c[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    if (!(x[d] >= g.lo[d] && x[d] <= g.hi[d])) return true;
    c[d] = min(static_cast<int>(floorf(__fmul_rn(__fsub_rn(x[d], g.lo[d]), g.scale[d]))), n[d] - 1);
  }
  const long long cell = (static_cast<long long>(c[2]) * g.ny + c[1]) * g.nx + c[0];
  return (__ldg(g.bits + (cell >> 5)) >> (cell & 31)) & 1u;
}

// Lookup slot q of a segment: the sample's index in the pass, and whether its ray is still alive
__device__ __forceinline__ long long occ_seg_sample(const OccPoints& s, const OccSegment& seg, long long q, bool* alive) {
  const long long ray = q / seg.len;
  const int j = seg.s0 + static_cast<int>(q - ray * seg.len);
  *alive = j < __ldg(seg.term + ray);
  return ray * s.S + j;
}

// The count step of the lookup, over every point of s (kSeg = false) or over the slots of one segment of an
// early-terminating pass (kSeg = true: kept while the ray is alive, and by the grid when seg.use_grid)
template <bool kSeg>
__device__ __forceinline__ void occ_count_body(const OccGrid& g, const OccPoints& s, const OccSegment& seg, int32_t* __restrict__ block_counts) {
  const long long i = static_cast<long long>(blockIdx.x) * kOccTile + threadIdx.x;
  bool keep = false;
  if constexpr (kSeg) {
    if (i < seg.P) {
      const long long k = occ_seg_sample(s, seg, i, &keep);
      if (keep && seg.use_grid) {
        float x[3];
        occ_point(s, k, x);
        keep = occ_keep(g, x);
      }
    }
  } else if (i < s.P) {
    float x[3];
    occ_point(s, i, x);
    keep = occ_keep(g, x);
  }
  const int cnt = __syncthreads_count(keep);
  if (threadIdx.x == 0) block_counts[blockIdx.x] = cnt;
}

__global__ void __launch_bounds__(kOccTile) occ_count_kernel(const OccGrid g, const OccPoints s, int32_t* __restrict__ block_counts) {
  occ_count_body<false>(g, s, OccSegment{}, block_counts);
}
__global__ void __launch_bounds__(kOccTile) occ_count_seg_kernel(const OccGrid g, const OccPoints s, const OccSegment seg,
                                                                 int32_t* __restrict__ block_counts) {
  occ_count_body<true>(g, s, seg, block_counts);
}

// One block: the exclusive scan of the n block counts in place, the total -> counts[n] and *count
__global__ void __launch_bounds__(kOccTile) occ_scan_kernel(int32_t* __restrict__ counts, int n, int32_t* __restrict__ count) {
  using Scan = cub::BlockScan<int, kOccTile>;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < n; base += kOccTile) {
    const int i = base + threadIdx.x;
    const int v = i < n ? counts[i] : 0;
    int ex, tot;
    Scan(tmp).ExclusiveSum(v, ex, tot);
    const int c0 = carry;
    if (i < n) counts[i] = c0 + ex;
    __syncthreads();   // every thread has read carry and tmp
    if (threadIdx.x == 0) carry = c0 + tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    counts[n] = carry;
    *count = carry;
  }
}

__global__ void __launch_bounds__(kOccTile) occ_write_kernel(const OccGrid g, const OccPoints s, const OccCompact c) {
  using Scan = cub::BlockScan<int, kOccTile>;
  __shared__ typename Scan::TempStorage tmp;
  const long long i = static_cast<long long>(blockIdx.x) * kOccTile + threadIdx.x;
  float x[3] = {0.f, 0.f, 0.f};
  bool keep = false;
  if (i < s.P) {
    occ_point(s, i, x);
    keep = occ_keep(g, x);
    if (c.d_init) { c.d_init[i * 3 + 0] = x[0]; c.d_init[i * 3 + 1] = x[1]; c.d_init[i * 3 + 2] = x[2]; }
    if (c.d_bent) { c.d_bent[i * 3 + 0] = x[0]; c.d_bent[i * 3 + 1] = x[1]; c.d_bent[i * 3 + 2] = x[2]; }
  }
  int rank;
  Scan(tmp).ExclusiveSum(keep ? 1 : 0, rank);
  if (keep) {
    const long long o = static_cast<long long>(__ldg(c.block_counts + blockIdx.x)) + rank;
    c.kept_xyz[o * 3 + 0] = x[0]; c.kept_xyz[o * 3 + 1] = x[1]; c.kept_xyz[o * 3 + 2] = x[2];
    c.kept_idx[o] = static_cast<int32_t>(i);
  }
}

// occ_write_kernel over the slots of one segment.  It is a kernel of its own rather than a second instance of a shared
// body: folding occ_write_kernel into a template body reorders two of its instructions, and its SASS is kept as it was.
// The steps it shares with occ_write_kernel are occ_point, occ_keep and the block scan's write-out, in the same order.
__global__ void __launch_bounds__(kOccTile) occ_write_seg_kernel(const OccGrid g, const OccPoints s, const OccSegment seg, const OccCompact c) {
  using Scan = cub::BlockScan<int, kOccTile>;
  __shared__ typename Scan::TempStorage tmp;
  const long long q = static_cast<long long>(blockIdx.x) * kOccTile + threadIdx.x;
  long long i = 0;
  float x[3] = {0.f, 0.f, 0.f};
  bool keep = false;
  if (q < seg.P) {
    bool alive;
    i = occ_seg_sample(s, seg, q, &alive);
    occ_point(s, i, x);
    keep = alive && (!seg.use_grid || occ_keep(g, x));
    if (c.d_init) { c.d_init[i * 3 + 0] = x[0]; c.d_init[i * 3 + 1] = x[1]; c.d_init[i * 3 + 2] = x[2]; }
    if (c.d_bent) { c.d_bent[i * 3 + 0] = x[0]; c.d_bent[i * 3 + 1] = x[1]; c.d_bent[i * 3 + 2] = x[2]; }
  }
  int rank;
  Scan(tmp).ExclusiveSum(keep ? 1 : 0, rank);
  if (keep) {
    const long long o = static_cast<long long>(__ldg(c.block_counts + blockIdx.x)) + rank;
    c.kept_xyz[o * 3 + 0] = x[0]; c.kept_xyz[o * 3 + 1] = x[1]; c.kept_xyz[o * 3 + 2] = x[2];
    c.kept_idx[o] = static_cast<int32_t>(i);
  }
}

__global__ void __launch_bounds__(kOccThreads) occ_scatter_kernel(const float* __restrict__ craw, const int32_t* __restrict__ idx,
                                                                  const int32_t* __restrict__ count, int out_ch, const float4* __restrict__ ws,
                                                                  int use_removal, float removal, float* __restrict__ raw) {
  const long long K = __ldg(count);
  for (long long k = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; k < K; k += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long p = __ldg(idx + k);
    float o[5];
#pragma unroll
    for (int ch = 0; ch < 5; ++ch) o[ch] = ch < out_ch ? __ldg(craw + k * out_ch + ch) : 0.f;
    // test-time non-rigid object removal (run_nerf_helpers.py:309-310), as the fused kernel applies it
    if (ws && use_removal && __ldg(ws + p).w >= removal) o[3] *= 0.f;
#pragma unroll
    for (int ch = 0; ch < 5; ++ch)
      if (ch < out_ch) raw[p * out_ch + ch] = o[ch];
  }
}

__global__ void __launch_bounds__(kOccThreads) term_init_kernel(const TermPass t) {
  const int ray = blockIdx.x * blockDim.x + threadIdx.x;
  if (ray >= t.n) return;
  t.T[ray] = 1.0f;
  t.term[ray] = t.S;
}

// One thread per ray: T <- T * (1 - alpha + 1e-10) over the segment's samples in order, one rounded multiply each, alpha
// from composite_alpha on the raw the round wrote (a sample not evaluated has raw 0, so its factor is exactly 1).  The ray
// dies when T < threshold (never for a NaN T, nor for threshold 0).
__global__ void __launch_bounds__(kOccThreads) term_transmittance_kernel(const TermPass t, int s0, int len) {
  const int ray = blockIdx.x * blockDim.x + threadIdx.x;
  if (ray >= t.n || t.term[ray] < t.S) return;
  const float* d = t.rays + static_cast<long long>(ray) * 8 + 3;
  const float dnorm = ray_dnorm(__ldg(d + 0), __ldg(d + 1), __ldg(d + 2));
  const long long base = static_cast<long long>(ray) * t.S;
  const float* z = t.z + base;
  float T = t.T[ray];
  for (int i = s0; i < s0 + len; ++i) {
    const float zi = __ldg(z + i);
    const float gap = i + 1 < t.S ? __ldg(z + i + 1) - zi : 1e10f;   // as composite_kernel
    float sigma = t.raw[(base + i) * t.out_ch + 3];
    if (t.noise) sigma += __ldg(t.noise + base + i);
    const float alpha = composite_alpha(sigma, gap, dnorm);
    T = __fmul_rn(T, 1.0f - alpha + 1e-10f);
  }
  t.T[ray] = T;
  if (T < t.threshold) t.term[ray] = s0 + len;
}

unsigned blocks_for(long long n, int per_block) { return static_cast<unsigned>((n + per_block - 1) / per_block); }

}  // namespace

cudaError_t launch_occupancy_build(const float* sigma, int nx, int ny, int nz, float threshold, int dilation, uint8_t* ws,
                                   uint32_t* bits, cudaStream_t st) {
  const long long n = static_cast<long long>(nx) * ny * nz;
  const unsigned nb = blocks_for(n, kOccThreads);
  uint8_t* a = ws;
  uint8_t* b = ws + n;
  occ_corner_kernel<<<nb, kOccThreads, 0, st>>>(sigma, nx, ny, nz, threshold, a);
  if (dilation > 0) {
    for (int axis = 0; axis < 3; ++axis) {
      occ_dilate_kernel<<<nb, kOccThreads, 0, st>>>(a, b, nx, ny, nz, axis, dilation);
      uint8_t* t = a; a = b; b = t;
    }
  }
  occ_pack_kernel<<<nb, kOccThreads, 0, st>>>(a, n, bits);
  return cudaGetLastError();
}

cudaError_t launch_occupancy_compact(const OccGrid& g, const OccPoints& pts, const OccCompact& c, cudaStream_t st) {
  const unsigned nb = blocks_for(pts.P, kOccTile);
  if (nb > 0) occ_count_kernel<<<nb, kOccTile, 0, st>>>(g, pts, c.block_counts);
  occ_scan_kernel<<<1, kOccTile, 0, st>>>(c.block_counts, static_cast<int>(nb), c.count);
  if (nb > 0) occ_write_kernel<<<nb, kOccTile, 0, st>>>(g, pts, c);
  return cudaGetLastError();
}

// max_kept bounds the count the kernel reads from device memory: it sizes the grid
cudaError_t launch_occupancy_scatter(const float* compact_raw, const int32_t* kept_idx, const int32_t* count, long long max_kept, int out_ch,
                                     const float4* ws, int use_removal, float removal, float* raw, int num_sms, cudaStream_t st) {
  const long long cap = static_cast<long long>(num_sms) * 16;
  const long long nb = blocks_for(max_kept, kOccThreads);
  occ_scatter_kernel<<<static_cast<unsigned>(nb < cap ? nb : cap), kOccThreads, 0, st>>>(compact_raw, kept_idx, count, out_ch, ws, use_removal,
                                                                                        removal, raw);
  return cudaGetLastError();
}

cudaError_t launch_occupancy_scan(int32_t* counts, int n, int32_t* count, cudaStream_t st) {
  occ_scan_kernel<<<1, kOccTile, 0, st>>>(counts, n, count);
  return cudaGetLastError();
}

cudaError_t launch_termination_init(const TermPass& t, cudaStream_t st) {
  term_init_kernel<<<blocks_for(t.n, kOccThreads), kOccThreads, 0, st>>>(t);
  return cudaGetLastError();
}

cudaError_t launch_termination_compact(const OccGrid& g, const OccPoints& pts, const OccSegment& seg, const OccCompact& c, cudaStream_t st) {
  const unsigned nb = blocks_for(seg.P, kOccTile);
  if (nb > 0) occ_count_seg_kernel<<<nb, kOccTile, 0, st>>>(g, pts, seg, c.block_counts);
  occ_scan_kernel<<<1, kOccTile, 0, st>>>(c.block_counts, static_cast<int>(nb), c.count);
  if (nb > 0) occ_write_seg_kernel<<<nb, kOccTile, 0, st>>>(g, pts, seg, c);
  return cudaGetLastError();
}

cudaError_t launch_termination_transmittance(const TermPass& t, int s0, int len, cudaStream_t st) {
  term_transmittance_kernel<<<blocks_for(t.n, kOccThreads), kOccThreads, 0, st>>>(t, s0, len);
  return cudaGetLastError();
}

}  // namespace nrn
