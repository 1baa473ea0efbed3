// Parameter blocks and launchers of the correspondence kernels (match.cu): a uniform grid over the canonical surface
// points of every frame of a stack, and the exact nearest-neighbour search of query pixels against it.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace nrn {

constexpr long long kMatchMaxPoints = 0x7fffffffLL;   // points of one frame at most: a point index is an int32
constexpr int kMatchMaxSide = 1 << 24;                // frame height and width at most: pixel coordinates are exact in fp32
constexpr int kMatchMaxFrames = 65535;                // frames of one stack at most (the frame is the build grid's y)

// The points of F frames of N points each and the grid built over each frame (the workspace of nrn_match).  The grid of a
// frame has n x n x n cells over the bounding box of its valid points (n from N alone, match_cells_per_axis); an axis on
// which the box is flat keeps one layer of cells.
struct MatchCloud {
  const float* pts;      // [F][N][3]
  const uint8_t* mask;   // [F][N], nonzero = a surface point, or null (all valid); non-finite points are never valid
  int F;
  long long N;
  int n;                 // cells per axis; C = n^3 per frame
  int32_t* bbox;         // [F][8]      order keys of the valid points' minimum (x, y, z) and maximum (x, y, z)
  int32_t* count;        // [F][C]      points per cell, then the scatter's fill cursor
  int32_t* start;        // [F][C + 1]  exclusive scan of the counts: the first sorted point of each cell
  float4* sorted;        // [F][N]      valid points in cell order: (x, y, z, index bits)
};
int match_cells_per_axis(long long N);
size_t match_cloud_bytes(int F, long long N);
MatchCloud match_cloud(void* ws, const float* pts, const uint8_t* mask, int F, long long N);

// F frame pairs: query frame (Fq == 1 ? 0 : f) against target frame (Ft == 1 ? 0 : f)
struct MatchQueryParams {
  MatchCloud q;          // the query frames; their grids are read only for the round trip
  MatchCloud t;          // the target frames and their grids
  int F, Wq, Wt;
  float max_d2;          // fl(max_distance * max_distance)
  int round_trip;
  float rt_tol2;         // fl(round_trip_pixels * round_trip_pixels)
  int32_t* index;        // [F][Nq]
  float* distance;       // [F][Nq]
  float* flow;           // [F][Nq][2]
  uint8_t* consistent;   // [F][Nq] or null
};

cudaError_t launch_match_build(const MatchCloud& c, int num_sms, cudaStream_t st);
cudaError_t launch_match_query(const MatchQueryParams& p, cudaStream_t st);

}  // namespace nrn
