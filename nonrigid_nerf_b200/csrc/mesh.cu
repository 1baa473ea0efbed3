// Marching cubes over a density grid that is processed one z-slab at a time (geometry.py): grid points of a plane for the
// point-mode field pass, the density relu(raw[3]), per-plane edge and per-cell case counts, their exclusive scans, and the
// compacted vertices and faces.  Vertices are ordered by edge key (k, j, i, axis), faces by cell (k, j, i) and then by
// table order, so the mesh is the same on every run.  Offsets within one plane are int32 (the plane size is bounded,
// kMeshMaxPlane); the plane bases and every global index are 64-bit until they are stored.
//
// Every floating-point step is an explicit _rn intrinsic, so no multiply-add is contracted and a numpy restatement in
// fp32 reproduces the vertices bit for bit (tests/mesh_reference.py).
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>
#include "eval.cuh"
#include "mesh.cuh"

namespace nrn {
namespace {

// ---- the cube table, built by construction ----------------------------------------------------------------------------
// Corner c sits at offset (c & 1, (c >> 1) & 1, (c >> 2) & 1) in (x, y, z); the case index is sum occupied(c) << c.  Edge
// e = 4 * axis + r runs along `axis` from its lower corner, whose offsets on the other two axes (in increasing axis order)
// are r & 1 and r >> 1.  On each face the crossed edges are joined by segments: two crossed edges give one segment, four (an
// ambiguous face) give two, each cutting off one occupied corner.  A segment P -> Q is oriented so that an occupied corner C
// it separates lies to its right seen from outside the cell, ((Q - P) x (C - P)) . n_out < 0 with P, Q the edge midpoints.
// The segments chain into closed loops, taken in order of their lowest edge and fanned from it, which gives triangles whose
// normals point out of the occupied region.  Each face's choice depends on its four corners alone, so cells sharing the face
// agree and the surface has no cracks.
constexpr int corner_coord(int c, int a) { return (c >> a) & 1; }
constexpr int edge_axis(int e) { return e >> 2; }
constexpr int edge_lo(int e) {
  const int axis = e >> 2, r = e & 3, a1 = axis == 0 ? 1 : 0, a2 = axis == 2 ? 1 : 2;
  return ((r & 1) << a1) | ((r >> 1) << a2);
}
constexpr int edge_hi(int e) { return edge_lo(e) | (1 << edge_axis(e)); }
constexpr int mid2(int e, int a) { return 2 * corner_coord(edge_lo(e), a) + (a == edge_axis(e) ? 1 : 0); }

struct CubeTable {
  int8_t count[256];
  int8_t edges[256][kMeshMaxTris][3];
  bool ok;   // every crossed edge starts exactly one segment and no case needs more than kMeshMaxTris triangles
};

constexpr CubeTable make_cube_table() {
  CubeTable t{};
  t.ok = true;
  for (int cs = 0; cs < 256; ++cs) {
    int next[12] = {-1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1};
    for (int axis = 0; axis < 3; ++axis)
      for (int side = 0; side < 2; ++side) {
        int crossed[4] = {}, nc = 0;
        for (int e = 0; e < 12; ++e)
          if (edge_axis(e) != axis && corner_coord(edge_lo(e), axis) == side &&
              ((cs >> edge_lo(e)) & 1) != ((cs >> edge_hi(e)) & 1))
            crossed[nc++] = e;
        int seg[2][3] = {}, ns = 0;   // (P, Q, corner C)
        for (int c = 0; c < 8; ++c) {
          if (corner_coord(c, axis) != side || !((cs >> c) & 1)) continue;
          if (nc == 2 && ns == 0) {
            seg[ns][0] = crossed[0]; seg[ns][1] = crossed[1]; seg[ns][2] = c; ++ns;
          } else if (nc == 4) {
            int m = 0;
            for (int i = 0; i < 4; ++i)
              if (edge_lo(crossed[i]) == c || edge_hi(crossed[i]) == c) seg[ns][m++] = crossed[i];
            seg[ns][2] = c; ++ns;
          }
        }
        for (int s = 0; s < ns; ++s) {
          int p = seg[s][0], q = seg[s][1];
          const int c = seg[s][2], a1 = (axis + 1) % 3, a2 = (axis + 2) % 3;
          const int u1 = mid2(q, a1) - mid2(p, a1), u2 = mid2(q, a2) - mid2(p, a2);
          const int v1 = 2 * corner_coord(c, a1) - mid2(p, a1), v2 = 2 * corner_coord(c, a2) - mid2(p, a2);
          if ((u1 * v2 - u2 * v1) * (2 * side - 1) > 0) { const int x = p; p = q; q = x; }
          if (next[p] != -1) t.ok = false;
          next[p] = q;
        }
      }
    bool seen[12] = {};
    int nt = 0;
    for (int start = 0; start < 12; ++start) {
      if (next[start] < 0 || seen[start]) continue;
      int loop[12] = {}, len = 0;
      for (int e = start; !seen[e]; e = next[e]) {
        if (e < 0) { t.ok = false; break; }
        seen[e] = true;
        loop[len++] = e;
        if (next[e] < 0) { t.ok = false; break; }
      }
      for (int i = 1; i + 1 < len; ++i) {
        if (nt == kMeshMaxTris) { t.ok = false; break; }
        t.edges[cs][nt][0] = static_cast<int8_t>(loop[0]);
        t.edges[cs][nt][1] = static_cast<int8_t>(loop[i]);
        t.edges[cs][nt][2] = static_cast<int8_t>(loop[i + 1]);
        ++nt;
      }
    }
    for (int i = nt; i < kMeshMaxTris; ++i) t.edges[cs][i][0] = t.edges[cs][i][1] = t.edges[cs][i][2] = -1;
    t.count[cs] = static_cast<int8_t>(nt);
  }
  return t;
}
constexpr CubeTable kCube = make_cube_table();
static_assert(kCube.ok, "cube table: a crossed edge without exactly one outgoing segment, or more than kMeshMaxTris triangles");
static_assert(kCube.count[0] == 0 && kCube.count[255] == 0 && kCube.count[1] == 1, "cube table: trivial cases");

struct CubeDeviceTable {
  int8_t count[256];
  int8_t edges[256][kMeshMaxTris][3];
};
constexpr CubeDeviceTable make_cube_device_table() {
  CubeDeviceTable d{};
  for (int c = 0; c < 256; ++c) {
    d.count[c] = kCube.count[c];
    for (int i = 0; i < kMeshMaxTris; ++i)
      for (int v = 0; v < 3; ++v) d.edges[c][i][v] = kCube.edges[c][i][v];
  }
  return d;
}
__constant__ CubeDeviceTable c_cube = make_cube_device_table();

// (axis, dx, dy, dz) of each edge's lower corner, packed: the faces kernel's lookups
constexpr int edge_code(int e) {
  return edge_axis(e) | (corner_coord(edge_lo(e), 0) << 2) | (corner_coord(edge_lo(e), 1) << 3) | (corner_coord(edge_lo(e), 2) << 4);
}
__constant__ int8_t c_edge_code[12] = {edge_code(0), edge_code(1), edge_code(2), edge_code(3), edge_code(4), edge_code(5),
                                       edge_code(6), edge_code(7), edge_code(8), edge_code(9), edge_code(10), edge_code(11)};

// ---- grid and density ---------------------------------------------------------------------------------------------------
// x_i = lo + (hi - lo) * (i / (n - 1)), each operation rounded in fp32, and x_{n-1} = hi exactly
__device__ __forceinline__ float grid_coord(const MeshGrid& g, int a, int i) {
  if (i == g.n[a] - 1) return g.hi[a];
  return __fadd_rn(g.lo[a], __fmul_rn(__fsub_rn(g.hi[a], g.lo[a]), __fdiv_rn(static_cast<float>(i), static_cast<float>(g.n[a] - 1))));
}

__global__ void mesh_grid_points_kernel(MeshGrid g, int k, float* __restrict__ pts) {
  const long long n = static_cast<long long>(g.n[0]) * g.n[1];
  const float z = grid_coord(g, 2, k);
  for (long long q = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; q < n; q += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int i = static_cast<int>(q % g.n[0]), j = static_cast<int>(q / g.n[0]);
    pts[q * 3 + 0] = grid_coord(g, 0, i);
    pts[q * 3 + 1] = grid_coord(g, 1, j);
    pts[q * 3 + 2] = z;
  }
}

// relu(raw[3]) as torch.relu computes it: NaN stays NaN
__global__ void mesh_sigma_kernel(const float* __restrict__ raw, long long n, int out_ch, float* __restrict__ sigma) {
  for (long long q = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; q < n; q += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float v = __ldg(raw + q * out_ch + 3);
    sigma[q] = v != v ? v : fmaxf(v, 0.f);
  }
}

// ---- counts -------------------------------------------------------------------------------------------------------------
// Occupied: sigma > threshold (NaN is not).  Per point of plane k the edges to +x, +y and (with plane k + 1) +z that have
// exactly one occupied end; per cell between the planes its case index and triangle count.  The entry past the end of each
// count array is zeroed, so that the in-place exclusive scan leaves the plane's total there.
__global__ void mesh_count_kernel(int nx, int ny, const float* __restrict__ s0, const float* __restrict__ s1, float t, MeshPlaneState s) {
  const long long n = static_cast<long long>(nx) * ny, ncell = static_cast<long long>(nx - 1) * (ny - 1);
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const long long first = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (first == 0) {
    s.voff[n] = 0;
    if (s1) s.toff[ncell] = 0;
  }
  for (long long q = first; q < n; q += stride) {
    const int i = static_cast<int>(q % nx), j = static_cast<int>(q / nx);
    const bool o = __ldg(s0 + q) > t;
    int m = 0;
    if (i + 1 < nx && o != (__ldg(s0 + q + 1) > t)) m |= 1;
    if (j + 1 < ny && o != (__ldg(s0 + q + nx) > t)) m |= 2;
    if (s1 && o != (__ldg(s1 + q) > t)) m |= 4;
    s.emask[q] = static_cast<uint8_t>(m);
    s.voff[q] = __popc(m);
    if (s1 && i + 1 < nx && j + 1 < ny) {
      const float* pl[2] = {s0, s1};
      int cs = 0;
#pragma unroll
      for (int c = 0; c < 8; ++c)
        cs |= (__ldg(pl[c >> 2] + q + (c & 1) + ((c >> 1) & 1) * static_cast<long long>(nx)) > t) << c;
      const long long cell = static_cast<long long>(j) * (nx - 1) + i;
      s.ccase[cell] = static_cast<uint8_t>(cs);
      s.toff[cell] = c_cube.count[cs];
    }
  }
}

// ---- exclusive scan of int32 counts, in place: block sums, a scan of the sums in one block, then each block's scan -------
constexpr int kScanThreads = 256, kScanItems = 4, kScanTile = kScanThreads * kScanItems;

__global__ void __launch_bounds__(kScanThreads) mesh_scan_sums_kernel(const int32_t* __restrict__ data, long long n, int32_t* __restrict__ partials) {
  using Reduce = cub::BlockReduce<int32_t, kScanThreads>;
  __shared__ typename Reduce::TempStorage tmp;
  const long long base = static_cast<long long>(blockIdx.x) * kScanTile;
  int32_t v = 0;
#pragma unroll
  for (int i = 0; i < kScanItems; ++i) {
    const long long q = base + threadIdx.x * kScanItems + i;
    if (q < n) v += data[q];
  }
  const int32_t sum = Reduce(tmp).Sum(v);
  if (threadIdx.x == 0) partials[blockIdx.x] = sum;
}

__global__ void __launch_bounds__(kScanThreads) mesh_scan_partials_kernel(int32_t* __restrict__ partials, int nb) {
  using Scan = cub::BlockScan<int32_t, kScanThreads>;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ int32_t carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < nb; base += kScanTile) {
    int32_t v[kScanItems];
#pragma unroll
    for (int i = 0; i < kScanItems; ++i) {
      const int q = base + threadIdx.x * kScanItems + i;
      v[i] = q < nb ? partials[q] : 0;
    }
    int32_t total;
    Scan(tmp).ExclusiveSum(v, v, total);
    const int32_t c = carry;
#pragma unroll
    for (int i = 0; i < kScanItems; ++i) {
      const int q = base + threadIdx.x * kScanItems + i;
      if (q < nb) partials[q] = v[i] + c;
    }
    __syncthreads();
    if (threadIdx.x == 0) carry = c + total;
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kScanThreads) mesh_scan_apply_kernel(int32_t* __restrict__ data, long long n, const int32_t* __restrict__ partials) {
  using Scan = cub::BlockScan<int32_t, kScanThreads>;
  __shared__ typename Scan::TempStorage tmp;
  const long long base = static_cast<long long>(blockIdx.x) * kScanTile;
  int32_t v[kScanItems];
#pragma unroll
  for (int i = 0; i < kScanItems; ++i) {
    const long long q = base + threadIdx.x * kScanItems + i;
    v[i] = q < n ? data[q] : 0;
  }
  Scan(tmp).ExclusiveSum(v, v);
  const int32_t off = partials[blockIdx.x];
#pragma unroll
  for (int i = 0; i < kScanItems; ++i) {
    const long long q = base + threadIdx.x * kScanItems + i;
    if (q < n) data[q] = v[i] + off;
  }
}

// ---- emission -----------------------------------------------------------------------------------------------------------
// The vertex of each crossed edge owned by plane k, at p_a + ((t - s_a) / (s_b - s_a)) * (p_b - p_a) per component, from its
// lower end a; NaN densities count as 0 here
__device__ __forceinline__ float nan_to_zero(float v) { return v != v ? 0.f : v; }

__global__ void mesh_vertices_kernel(MeshGrid g, int k, const float* __restrict__ s0, const float* __restrict__ s1, float t,
                                     MeshPlaneState s, long long vbase, float* __restrict__ vertices) {
  const int nx = g.n[0];
  const long long n = static_cast<long long>(nx) * g.n[1];
  for (long long q = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; q < n; q += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int m = s.emask[q];
    if (!m) continue;
    const int i = static_cast<int>(q % nx), j = static_cast<int>(q / nx);
    const float pa[3] = {grid_coord(g, 0, i), grid_coord(g, 1, j), grid_coord(g, 2, k)};
    const float sa = nan_to_zero(__ldg(s0 + q));
    long long v = vbase + s.voff[q];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (!((m >> a) & 1)) continue;
      const float sb = nan_to_zero(a == 0 ? __ldg(s0 + q + 1) : a == 1 ? __ldg(s0 + q + nx) : __ldg(s1 + q));
      const float pb[3] = {a == 0 ? grid_coord(g, 0, i + 1) : pa[0], a == 1 ? grid_coord(g, 1, j + 1) : pa[1],
                           a == 2 ? grid_coord(g, 2, k + 1) : pa[2]};
      const float w = __fdiv_rn(__fsub_rn(t, sa), __fsub_rn(sb, sa));
#pragma unroll
      for (int c = 0; c < 3; ++c) vertices[v * 3 + c] = __fadd_rn(pa[c], __fmul_rn(w, __fsub_rn(pb[c], pa[c])));
      ++v;
    }
  }
}

// The faces of the cell layer between the planes of `lower` and `upper`, as the global ids of their edges' vertices
__global__ void mesh_faces_kernel(int nx, int ny, MeshPlaneState lower, MeshPlaneState upper, long long vbase_lower,
                                  long long vbase_upper, long long tbase, int32_t* __restrict__ faces) {
  const long long ncell = static_cast<long long>(nx - 1) * (ny - 1);
  for (long long cell = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; cell < ncell; cell += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int cs = lower.ccase[cell];
    const int nt = c_cube.count[cs];
    if (!nt) continue;
    const int i = static_cast<int>(cell % (nx - 1)), j = static_cast<int>(cell / (nx - 1));
    long long f = tbase + lower.toff[cell];
    for (int tr = 0; tr < nt; ++tr, ++f)
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const int code = c_edge_code[c_cube.edges[cs][tr][c]];
        const int a = code & 3;
        const long long q = static_cast<long long>(j + ((code >> 3) & 1)) * nx + i + ((code >> 2) & 1);
        const MeshPlaneState& p = (code >> 4) ? upper : lower;
        const long long vb = (code >> 4) ? vbase_upper : vbase_lower;
        faces[f * 3 + c] = static_cast<int32_t>(vb + p.voff[q] + __popc(p.emask[q] & ((1 << a) - 1)));
      }
  }
}

// to8b(sigmoid(raw[0:3])), the sigmoid as raw2outputs computes it
__global__ void mesh_colors_kernel(const float* __restrict__ raw, long long n, int out_ch, uint8_t* __restrict__ colors) {
  for (long long q = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; q < n * 3; q += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long v = q / 3;
    const int c = static_cast<int>(q - v * 3);
    colors[q] = static_cast<uint8_t>(lut_index(1.0f / (1.0f + expf(-__ldg(raw + v * out_ch + c)))));
  }
}

constexpr int kThreads = 256;
unsigned grid_for(long long n) {
  const long long b = (n + kThreads - 1) / kThreads;
  return static_cast<unsigned>(b < 65535 * 16 ? (b > 0 ? b : 1) : 65535 * 16);
}

size_t align256(size_t b) { return (b + 255) & ~static_cast<size_t>(255); }
size_t plane_state_bytes(int nx, int ny) {
  const size_t n = static_cast<size_t>(nx) * ny, nc = static_cast<size_t>(nx - 1) * (ny - 1);
  return align256(n) + align256(4 * (n + 1)) + align256(nc) + align256(4 * (nc + 1));
}
long long scan_blocks(long long n) { return (n + kScanTile - 1) / kScanTile; }

}  // namespace

size_t mesh_workspace_bytes(int nx, int ny) {
  return kMeshSlots * plane_state_bytes(nx, ny) + align256(4 * static_cast<size_t>(scan_blocks(static_cast<long long>(nx) * ny + 1)));
}

MeshPlaneState mesh_plane_state(void* ws, int nx, int ny, int slot) {
  const size_t n = static_cast<size_t>(nx) * ny, nc = static_cast<size_t>(nx - 1) * (ny - 1);
  uint8_t* b = static_cast<uint8_t*>(ws) + slot * plane_state_bytes(nx, ny);
  MeshPlaneState s;
  s.emask = b;                                        b += align256(n);
  s.voff = reinterpret_cast<int32_t*>(b);             b += align256(4 * (n + 1));
  s.ccase = b;                                        b += align256(nc);
  s.toff = reinterpret_cast<int32_t*>(b);
  return s;
}

int32_t* mesh_scan_partials(void* ws, int nx, int ny) {
  return reinterpret_cast<int32_t*>(static_cast<uint8_t*>(ws) + kMeshSlots * plane_state_bytes(nx, ny));
}

void mesh_cube_table(int32_t* counts, int8_t* edges) {
  for (int c = 0; c < 256; ++c) {
    if (counts) counts[c] = kCube.count[c];
    if (edges)
      for (int i = 0; i < kMeshMaxTris; ++i)
        for (int v = 0; v < 3; ++v) edges[(c * kMeshMaxTris + i) * 3 + v] = kCube.edges[c][i][v];
  }
}

cudaError_t launch_mesh_grid_points(const MeshGrid& g, int k, float* points, cudaStream_t st) {
  mesh_grid_points_kernel<<<grid_for(static_cast<long long>(g.n[0]) * g.n[1]), kThreads, 0, st>>>(g, k, points);
  return cudaGetLastError();
}

cudaError_t launch_mesh_sigma(const float* raw, long long n, int out_ch, float* sigma, cudaStream_t st) {
  mesh_sigma_kernel<<<grid_for(n), kThreads, 0, st>>>(raw, n, out_ch, sigma);
  return cudaGetLastError();
}

cudaError_t launch_mesh_count(const MeshGrid& g, const float* s0, const float* s1, float threshold, const MeshPlaneState& s,
                              cudaStream_t st) {
  mesh_count_kernel<<<grid_for(static_cast<long long>(g.n[0]) * g.n[1]), kThreads, 0, st>>>(g.n[0], g.n[1], s0, s1, threshold, s);
  return cudaGetLastError();
}

cudaError_t launch_mesh_scan(int32_t* data, long long n, int32_t* partials, cudaStream_t st) {
  const long long nb = scan_blocks(n);
  mesh_scan_sums_kernel<<<static_cast<unsigned>(nb), kScanThreads, 0, st>>>(data, n, partials);
  mesh_scan_partials_kernel<<<1, kScanThreads, 0, st>>>(partials, static_cast<int>(nb));
  mesh_scan_apply_kernel<<<static_cast<unsigned>(nb), kScanThreads, 0, st>>>(data, n, partials);
  return cudaGetLastError();
}

cudaError_t launch_mesh_vertices(const MeshGrid& g, int k, const float* s0, const float* s1, float threshold,
                                 const MeshPlaneState& s, long long vbase, float* vertices, cudaStream_t st) {
  mesh_vertices_kernel<<<grid_for(static_cast<long long>(g.n[0]) * g.n[1]), kThreads, 0, st>>>(g, k, s0, s1, threshold, s, vbase, vertices);
  return cudaGetLastError();
}

cudaError_t launch_mesh_faces(const MeshGrid& g, const MeshPlaneState& lower, const MeshPlaneState& upper, long long vbase_lower,
                              long long vbase_upper, long long tbase, int32_t* faces, cudaStream_t st) {
  mesh_faces_kernel<<<grid_for(static_cast<long long>(g.n[0] - 1) * (g.n[1] - 1)), kThreads, 0, st>>>(
      g.n[0], g.n[1], lower, upper, vbase_lower, vbase_upper, tbase, faces);
  return cudaGetLastError();
}

cudaError_t launch_mesh_colors(const float* raw, long long n, int out_ch, uint8_t* colors, cudaStream_t st) {
  mesh_colors_kernel<<<grid_for(n * 3), kThreads, 0, st>>>(raw, n, out_ch, colors);
  return cudaGetLastError();
}

}  // namespace nrn
