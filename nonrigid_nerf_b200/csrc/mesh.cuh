// Parameter blocks and launchers of the marching-cubes kernels (mesh.cu): grid points of one z-plane, the density of a
// point-mode field pass, per-slab edge / cell counts with their exclusive scans, the compacted vertices and faces, and
// vertex colours.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace nrn {

constexpr int kMeshMaxTris = 5;            // triangles of one cell at most (checked where the table is built)
constexpr int kMeshSlots = 3;              // per-plane states kept: plane k - 1 and k for the faces, k + 1 counted ahead
constexpr long long kMeshMaxPlane = 1LL << 28;   // nx * ny at most: 3 vertices per point and 5 faces per cell stay in int32
constexpr int kMeshMaxAxis = 1 << 24;      // points per axis at most: the index i is exact in fp32

// The grid of nx x ny x nz points between min and max (fp32)
struct MeshGrid {
  float lo[3], hi[3];
  int n[3];
};

// The workspace of nx x ny planes (nrn_mesh_workspace_bytes): kMeshSlots per-plane states, then the scan partials
struct MeshPlaneState {
  uint8_t* emask;    // [ny * nx]           bit a: the edge to +axis a crosses the surface
  int32_t* voff;     // [ny * nx + 1]       vertex counts, scanned in place to offsets within the plane (total last)
  uint8_t* ccase;    // [(ny-1) * (nx-1)]   case index of each cell of the layer above the plane
  int32_t* toff;     // [(ny-1) * (nx-1) + 1] triangle counts, scanned in place (total last)
};
size_t mesh_workspace_bytes(int nx, int ny);
MeshPlaneState mesh_plane_state(void* ws, int nx, int ny, int slot);
int32_t* mesh_scan_partials(void* ws, int nx, int ny);

// Host copy of the cube table: triangle count of each case, and its triangles' edges ([256][kMeshMaxTris][3], -1 padded)
void mesh_cube_table(int32_t* counts, int8_t* edges);

cudaError_t launch_mesh_grid_points(const MeshGrid& g, int k, float* points, cudaStream_t st);
cudaError_t launch_mesh_sigma(const float* raw, long long n, int out_ch, float* sigma, cudaStream_t st);
cudaError_t launch_mesh_count(const MeshGrid& g, const float* s0, const float* s1, float threshold, const MeshPlaneState& s,
                              cudaStream_t st);
cudaError_t launch_mesh_scan(int32_t* data, long long n, int32_t* partials, cudaStream_t st);
cudaError_t launch_mesh_vertices(const MeshGrid& g, int k, const float* s0, const float* s1, float threshold,
                                 const MeshPlaneState& s, long long vbase, float* vertices, cudaStream_t st);
cudaError_t launch_mesh_faces(const MeshGrid& g, const MeshPlaneState& lower, const MeshPlaneState& upper, long long vbase_lower,
                              long long vbase_upper, long long tbase, int32_t* faces, cudaStream_t st);
cudaError_t launch_mesh_colors(const float* raw, long long n, int out_ch, uint8_t* colors, cudaStream_t st);

}  // namespace nrn
