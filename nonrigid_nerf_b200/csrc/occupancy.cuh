// Parameter blocks and launchers of the occupancy-grid kernels (occupancy.cu): building the bit grid from a density grid,
// looking up sample points in it and compacting the kept ones, and scattering the trunk's outputs back to every sample.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace nrn {

constexpr long long kOccMaxPoints = 0x7fffffffLL;   // points of one pass at most: a kept index is an int32
constexpr int kOccMaxSide = 1 << 12;                // cells per axis at most
constexpr int kOccMaxDilation = 1 << 12;
constexpr int kOccTile = 1024;                      // points per block of the lookup and compaction

// nx * ny * nz cells over [lo, hi]; cell (i, j, k) is bit c % 32 of word c / 32, c = (k * ny + j) * nx + i.  A point inside
// the box falls into cell min(floor(fl(fl(x - lo) * scale)), n - 1) per axis, scale = fl(n / fl(hi - lo)).
struct OccGrid {
  const uint32_t* bits;
  int nx, ny, nz;
  float lo[3], hi[3], scale[3];
};

// Where a pass's sample points come from: the bend workspace (bent xyz, rigidity), given points [P][stride], or the rays
// and depths (pts = o + d * z, the field kernel's rounding)
struct OccPoints {
  const float4* ws;
  const float* pts;
  long long pts_stride;
  const float* rays;
  const float* z_vals;
  int S;
  long long P;
};

// The lookup's outputs: kept points' xyz [K][3] and indices [K] in ascending order, K -> *count.  block_counts holds
// ceil(P / kOccTile) + 1 ints.  d_init / d_bent (rays and depths only, may be null): every point's xyz, the details the
// fused kernel writes without a bender.
struct OccCompact {
  float* kept_xyz;
  int32_t* kept_idx;
  int32_t* count;
  int32_t* block_counts;
  float* d_init;
  float* d_bent;
};

cudaError_t launch_occupancy_build(const float* sigma, int nx, int ny, int nz, float threshold, int dilation, uint8_t* ws,
                                   uint32_t* bits, cudaStream_t st);
cudaError_t launch_occupancy_compact(const OccGrid& g, const OccPoints& pts, const OccCompact& c, cudaStream_t st);
// raw [P][out_ch] (zeroed first) <- compact_raw [K][out_ch] at the kept indices; with ws and use_removal, alpha *= 0 where
// the point's rigidity >= removal (the fused kernel's test-time object removal)
cudaError_t launch_occupancy_scatter(const float* compact_raw, const int32_t* kept_idx, const int32_t* count, long long P, int out_ch,
                                     const float4* ws, int use_removal, float removal, float* raw, int num_sms, cudaStream_t st);

}  // namespace nrn
