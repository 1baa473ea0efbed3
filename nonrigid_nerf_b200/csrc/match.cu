// Exact nearest canonical surface points between rendered frames (correspondence.py).  Per frame of a stack: the bounding
// box of its valid points (order-key atomics), points per cell of an n^3 uniform grid over that box, an exclusive scan of
// the counts, and a scatter of the points into cell order.  Each query pixel then searches rings of cells around its own
// cell until no unsearched cell can hold a point as close as the best one found (or within max_distance).
//
// The distance is d2 = (dx*dx + dy*dy) + dz*dz with every step an explicit _rn intrinsic, and the best point is the
// smallest (d2, index) pair.  The result is that of a brute-force search, whatever order the scatter left the points of a
// cell in, so it is the same on every run and in a CUDA graph.  The grid geometry is fp64; the termination bound is
// widened so that neither its rounding nor that of d2 can skip the true nearest point.
#include <cub/block/block_scan.cuh>
#include "match.cuh"

namespace nrn {
namespace {

constexpr int kThreads = 256;
constexpr int kScanThreads = 1024;
constexpr int kScanItems = 8;

size_t align256(size_t b) { return (b + 255) & ~static_cast<size_t>(255); }

// A float's order key: signed int comparison of keys is float comparison (finite values)
__device__ __forceinline__ int order_key(float f) {
  const int i = __float_as_int(f);
  return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float key_float(int k) { return __int_as_float(k >= 0 ? k : k ^ 0x7fffffff); }

__device__ __forceinline__ bool finite3(float x, float y, float z) {
  return isfinite(x) && isfinite(y) && isfinite(z);
}

// The grid of one frame, from its bounding-box keys
struct CellGrid {
  double lo[3], hi[3], inv[3];
  int na[3];     // cells on each axis: n, or 1 where the box is flat
  bool empty;    // no valid point
};

__device__ __forceinline__ CellGrid cell_grid(const int32_t* bbox, int n) {
  CellGrid g;
  g.empty = bbox[0] > bbox[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double lo = key_float(bbox[a]), hi = key_float(bbox[3 + a]);
    const double ext = hi - lo;
    g.lo[a] = lo;
    g.hi[a] = hi;
    g.inv[a] = ext > 0.0 ? n / ext : 0.0;
    g.na[a] = ext > 0.0 ? n : 1;
  }
  return g;
}

// The cell of coordinate p on axis a; monotone in p, so every point of a cell above (below) a face lies above (below) it
__device__ __forceinline__ int cell_axis(const CellGrid& g, int a, float p) {
  double v = (static_cast<double>(p) - g.lo[a]) * g.inv[a];
  v = fmin(fmax(v, 0.0), static_cast<double>(g.na[a] - 1));
  return static_cast<int>(v);
}

__device__ __forceinline__ float dist2(float qx, float qy, float qz, float px, float py, float pz) {
  const float dx = __fsub_rn(px, qx), dy = __fsub_rn(py, qy), dz = __fsub_rn(pz, qz);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// Every point the search skips lies in a cell outside the searched box [bl, bh]: beyond one of the box's open faces on
// some axis a, and inside the frame's bounding box on the other two.  The bound is the smallest squared distance from q to
// such a region, so a query outside the bounding box (a point that left the frame) stops as soon as the rings reach past
// its nearest point instead of when they have grown as far as it is from the box.  A face's coordinate is widened by far
// more than the fp64 rounding of the cell assignment and of the face itself; the squared bound is shrunk by far more than
// the relative rounding of d2 (5 * 2^-24) plus the subnormal spacing.
__device__ __forceinline__ double unsearched_bound2(const CellGrid& g, const int bl[3], const int bh[3], const float q[3], bool* all) {
  double out2[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double o = fmax(fmax(g.lo[a] - q[a], q[a] - g.hi[a]), 0.0);
    out2[a] = o * o;
  }
  double lb2 = INFINITY;
  *all = true;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double rest = out2[(a + 1) % 3] + out2[(a + 2) % 3];
    if (bh[a] < g.na[a] - 1) {
      const double face = g.lo[a] + (bh[a] + 1) / g.inv[a];
      const double d = fmax(face - 1e-12 * (fabs(g.lo[a]) + fabs(face)) - q[a], 0.0);
      lb2 = fmin(lb2, d * d + rest);
      *all = false;
    }
    if (bl[a] > 0) {
      const double face = g.lo[a] + bl[a] / g.inv[a];
      const double d = fmax(q[a] - (face + 1e-12 * (fabs(g.lo[a]) + fabs(face))), 0.0);
      lb2 = fmin(lb2, d * d + rest);
      *all = false;
    }
  }
  return lb2 * (1.0 - 1e-6) - 1e-44;
}

__device__ __forceinline__ void scan_points(const float4* __restrict__ pts, int s, int e, const float q[3], float& best_d2, int& best_i) {
  for (int k = s; k < e; ++k) {
    const float4 p = pts[k];
    const float d2 = dist2(q[0], q[1], q[2], p.x, p.y, p.z);
    const int i = __float_as_int(p.w);
    if (d2 < best_d2 || (d2 == best_d2 && i < best_i)) {
      best_d2 = d2;
      best_i = i;
    }
  }
}

// The index of frame f's nearest valid point to q within max_d2, or -1; *d2_out its d2
__device__ int nearest(const MatchCloud& c, int f, const float q[3], float max_d2, float* d2_out) {
  const CellGrid g = cell_grid(c.bbox + 8LL * f, c.n);
  if (g.empty) return -1;
  const long long C = static_cast<long long>(c.n) * c.n * c.n;
  const int32_t* __restrict__ start = c.start + f * (C + 1);
  const float4* __restrict__ pts = c.sorted + f * c.N;
  int cc[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) cc[a] = cell_axis(g, a, q[a]);
  float best_d2 = INFINITY;
  int best_i = 0x7fffffff;
  for (int r = 0;; ++r) {
    int bl[3], bh[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      bl[a] = max(cc[a] - r, 0);
      bh[a] = min(cc[a] + r, g.na[a] - 1);
    }
    for (int z = bl[2]; z <= bh[2]; ++z) {
      for (int y = bl[1]; y <= bh[1]; ++y) {
        const long long row = (static_cast<long long>(z) * c.n + y) * c.n;
        if (abs(z - cc[2]) == r || abs(y - cc[1]) == r) {          // a whole row of the shell: its points are contiguous
          scan_points(pts, start[row + bl[0]], start[row + bh[0] + 1], q, best_d2, best_i);
        } else {
          if (cc[0] - r >= 0) scan_points(pts, start[row + cc[0] - r], start[row + cc[0] - r + 1], q, best_d2, best_i);
          if (cc[0] + r <= g.na[0] - 1) scan_points(pts, start[row + cc[0] + r], start[row + cc[0] + r + 1], q, best_d2, best_i);
        }
      }
    }
    bool all;
    const double bound = unsearched_bound2(g, bl, bh, q, &all);
    if (all || bound > static_cast<double>(fminf(best_d2, max_d2))) break;
  }
  *d2_out = best_d2;
  return best_i != 0x7fffffff && best_d2 <= max_d2 ? best_i : -1;
}

__device__ __forceinline__ bool point_valid(const MatchCloud& c, int f, long long i, float q[3]) {
  const long long at = f * c.N + i;
  q[0] = c.pts[3 * at];
  q[1] = c.pts[3 * at + 1];
  q[2] = c.pts[3 * at + 2];
  return (!c.mask || c.mask[at]) && finite3(q[0], q[1], q[2]);
}

__global__ void match_init_kernel(MatchCloud c) {
  const long long C = static_cast<long long>(c.n) * c.n * c.n;
  const long long total = c.F * C;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x)
    c.count[i] = 0;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < 8LL * c.F; i += static_cast<long long>(gridDim.x) * blockDim.x)
    c.bbox[i] = (i & 7) < 3 ? 0x7fffffff : ((i & 7) < 6 ? static_cast<int>(0x80000000u) : 0);
}

__global__ void __launch_bounds__(kThreads) match_bbox_kernel(MatchCloud c) {
  const int f = blockIdx.y;
  int mn[3] = {0x7fffffff, 0x7fffffff, 0x7fffffff}, mx[3] = {static_cast<int>(0x80000000u), static_cast<int>(0x80000000u), static_cast<int>(0x80000000u)};
  for (long long i = blockIdx.x * static_cast<long long>(kThreads) + threadIdx.x; i < c.N; i += static_cast<long long>(gridDim.x) * kThreads) {
    float p[3];
    if (!point_valid(c, f, i, p)) continue;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const int k = order_key(p[a]);
      mn[a] = min(mn[a], k);
      mx[a] = max(mx[a], k);
    }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    mn[a] = __reduce_min_sync(0xffffffffu, mn[a]);
    mx[a] = __reduce_max_sync(0xffffffffu, mx[a]);
  }
  if ((threadIdx.x & 31) == 0 && mn[0] <= mx[0]) {
    int32_t* b = c.bbox + 8LL * f;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      atomicMin(b + a, mn[a]);
      atomicMax(b + 3 + a, mx[a]);
    }
  }
}

__device__ __forceinline__ long long cell_of(const CellGrid& g, int n, const float p[3]) {
  return (static_cast<long long>(cell_axis(g, 2, p[2])) * n + cell_axis(g, 1, p[1])) * n + cell_axis(g, 0, p[0]);
}

__global__ void __launch_bounds__(kThreads) match_count_kernel(MatchCloud c) {
  const int f = blockIdx.y;
  const long long i = blockIdx.x * static_cast<long long>(kThreads) + threadIdx.x;
  float p[3];
  if (i >= c.N || !point_valid(c, f, i, p)) return;
  const CellGrid g = cell_grid(c.bbox + 8LL * f, c.n);
  const long long C = static_cast<long long>(c.n) * c.n * c.n;
  atomicAdd(c.count + f * C + cell_of(g, c.n, p), 1);
}

// One block per frame: start = exclusive scan of count (C + 1 entries, the total last); count is zeroed for the scatter
__global__ void __launch_bounds__(kScanThreads) match_scan_kernel(MatchCloud c) {
  using Scan = cub::BlockScan<int, kScanThreads>;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ int carry;
  const int f = blockIdx.x;
  const long long C = static_cast<long long>(c.n) * c.n * c.n;
  int32_t* count = c.count + f * C;
  int32_t* start = c.start + f * (C + 1);
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  constexpr long long tile = static_cast<long long>(kScanThreads) * kScanItems;
  for (long long t0 = 0; t0 < C; t0 += tile) {
    int v[kScanItems];
    int sum = 0;
    const long long base = t0 + static_cast<long long>(threadIdx.x) * kScanItems;
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) {
      v[k] = base + k < C ? count[base + k] : 0;
      sum += v[k];
    }
    int excl, total;
    Scan(tmp).ExclusiveSum(sum, excl, total);
    excl += carry;
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) {
      if (base + k < C) {
        start[base + k] = excl;
        count[base + k] = 0;
      }
      excl += v[k];
    }
    __syncthreads();
    if (threadIdx.x == 0) carry += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) start[C] = carry;
}

__global__ void __launch_bounds__(kThreads) match_scatter_kernel(MatchCloud c) {
  const int f = blockIdx.y;
  const long long i = blockIdx.x * static_cast<long long>(kThreads) + threadIdx.x;
  float p[3];
  if (i >= c.N || !point_valid(c, f, i, p)) return;
  const CellGrid g = cell_grid(c.bbox + 8LL * f, c.n);
  const long long C = static_cast<long long>(c.n) * c.n * c.n;
  const long long cell = f * C + cell_of(g, c.n, p);
  const int slot = c.start[f * (C + 1) + (cell - f * C)] + atomicAdd(c.count + cell, 1);
  c.sorted[f * c.N + slot] = make_float4(p[0], p[1], p[2], __int_as_float(static_cast<int>(i)));
}

__global__ void __launch_bounds__(kThreads) match_query_kernel(MatchQueryParams p) {
  const long long total = static_cast<long long>(p.F) * p.q.N;
  const long long gi = blockIdx.x * static_cast<long long>(kThreads) + threadIdx.x;
  if (gi >= total) return;
  const int f = static_cast<int>(gi / p.q.N);
  const long long pix = gi - static_cast<long long>(f) * p.q.N;
  const int qf = p.q.F == 1 ? 0 : f, tf = p.t.F == 1 ? 0 : f;
  float q[3], d2 = INFINITY;
  int j = -1;
  if (point_valid(p.q, qf, pix, q)) j = nearest(p.t, tf, q, p.max_d2, &d2);
  const float xq = static_cast<float>(pix % p.Wq), yq = static_cast<float>(pix / p.Wq);
  p.index[gi] = j;
  if (j < 0) {
    p.distance[gi] = INFINITY;
    p.flow[2 * gi] = NAN;
    p.flow[2 * gi + 1] = NAN;
    if (p.consistent) p.consistent[gi] = 0;
    return;
  }
  p.distance[gi] = __fsqrt_rn(d2);
  p.flow[2 * gi] = __fsub_rn(static_cast<float>(j % p.Wt), xq);
  p.flow[2 * gi + 1] = __fsub_rn(static_cast<float>(j / p.Wt), yq);
  if (p.consistent) {
    // the matched target point against the query frame: back where it started, within the tolerance?
    float t[3], back_d2;
    point_valid(p.t, tf, j, t);
    const int k = nearest(p.q, qf, t, p.max_d2, &back_d2);
    bool ok = false;
    if (k >= 0) {
      const float dx = __fsub_rn(static_cast<float>(k % p.Wq), xq), dy = __fsub_rn(static_cast<float>(k / p.Wq), yq);
      ok = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)) <= p.rt_tol2;
    }
    p.consistent[gi] = ok ? 1 : 0;
  }
}

unsigned blocks_for(long long n) { return static_cast<unsigned>((n + kThreads - 1) / kThreads); }

}  // namespace

int match_cells_per_axis(long long N) {
  const long long cells = N / 2 > 1 ? N / 2 : 1;
  int n = 1;
  while (static_cast<long long>(n + 1) * (n + 1) * (n + 1) <= cells) ++n;
  return n;
}

static size_t cloud_sections(int F, long long N, size_t* off) {
  const long long n = match_cells_per_axis(N), C = n * n * n;
  size_t at = 0;
  off[0] = at; at += align256(static_cast<size_t>(F) * 8 * sizeof(int32_t));
  off[1] = at; at += align256(static_cast<size_t>(F) * C * sizeof(int32_t));
  off[2] = at; at += align256(static_cast<size_t>(F) * (C + 1) * sizeof(int32_t));
  off[3] = at; at += align256(static_cast<size_t>(F) * N * sizeof(float4));
  return at;
}

size_t match_cloud_bytes(int F, long long N) {
  size_t off[4];
  return cloud_sections(F, N, off);
}

MatchCloud match_cloud(void* ws, const float* pts, const uint8_t* mask, int F, long long N) {
  size_t off[4];
  cloud_sections(F, N, off);
  uint8_t* b = static_cast<uint8_t*>(ws);
  MatchCloud c;
  c.pts = pts; c.mask = mask; c.F = F; c.N = N; c.n = match_cells_per_axis(N);
  c.bbox = reinterpret_cast<int32_t*>(b + off[0]);
  c.count = reinterpret_cast<int32_t*>(b + off[1]);
  c.start = reinterpret_cast<int32_t*>(b + off[2]);
  c.sorted = reinterpret_cast<float4*>(b + off[3]);
  return c;
}

cudaError_t launch_match_build(const MatchCloud& c, int num_sms, cudaStream_t st) {
  const long long C = static_cast<long long>(c.n) * c.n * c.n;
  const long long init = c.F * C > 8LL * c.F ? c.F * C : 8LL * c.F;
  const long long init_blocks = (init + kThreads - 1) / kThreads;
  match_init_kernel<<<static_cast<unsigned>(init_blocks < 4LL * num_sms ? init_blocks : 4LL * num_sms), kThreads, 0, st>>>(c);
  const unsigned nb = blocks_for(c.N);
  // the box: a few blocks per frame, each reducing a strided share before one atomic per warp
  const unsigned bb = nb < 16u ? nb : 16u;
  match_bbox_kernel<<<dim3(bb, c.F), kThreads, 0, st>>>(c);
  match_count_kernel<<<dim3(nb, c.F), kThreads, 0, st>>>(c);
  match_scan_kernel<<<c.F, kScanThreads, 0, st>>>(c);
  match_scatter_kernel<<<dim3(nb, c.F), kThreads, 0, st>>>(c);
  return cudaGetLastError();
}

cudaError_t launch_match_query(const MatchQueryParams& p, cudaStream_t st) {
  match_query_kernel<<<blocks_for(static_cast<long long>(p.F) * p.q.N), kThreads, 0, st>>>(p);
  return cudaGetLastError();
}

}  // namespace nrn
