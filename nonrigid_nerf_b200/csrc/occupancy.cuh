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

// Samples per segment of an early-terminating render pass (nrn_field_forward_terminate): round r evaluates samples
// [r K, min((r + 1) K, S)) of the rays still alive.  Chosen by measurement (DESIGN.md); a build may override it with
// -DNRN_TERM_SEGMENT=K to repeat that measurement.
#ifndef NRN_TERM_SEGMENT
#define NRN_TERM_SEGMENT 16
#endif
constexpr int kTermSegment = NRN_TERM_SEGMENT;
static_assert(kTermSegment >= 1, "NRN_TERM_SEGMENT must be positive");

// One round of an early-terminating pass: lookup slot q (0 <= q < P = n_rays * len) is sample s0 + q % len of ray q / len.
// A slot is kept while its ray is alive (its sample index < term[ray]; term holds S until the ray dies) and, when
// use_grid is set, the grid keeps its point.
struct OccSegment {
  int s0, len;
  long long P;
  const int32_t* term;
  int use_grid;
};

// The state of an early-terminating pass: per ray the transmittance T and termination_index (term), and what the alphas
// of the round's samples are made of (the field's raw after the scatter, the depths, the ray directions, the noise)
struct TermPass {
  const float* raw;     // [n][S][out_ch]
  const float* z;       // [n][S]
  const float* rays;    // [n][8]
  const float* noise;   // [n][S] or null
  int n, S, out_ch;
  float threshold;
  float* T;             // [n]
  int32_t* term;        // [n]
};

cudaError_t launch_occupancy_build(const float* sigma, int nx, int ny, int nz, float threshold, int dilation, uint8_t* ws,
                                   uint32_t* bits, cudaStream_t st);
cudaError_t launch_occupancy_compact(const OccGrid& g, const OccPoints& pts, const OccCompact& c, cudaStream_t st);
// raw[kept_idx[k]] <- compact_raw [k][out_ch] for k < K = *count <= max_kept; raw elsewhere is left as it is (a pass zeroes
// it first).  With ws and use_removal, alpha *= 0 where the point's rigidity >= removal (the fused kernel's test-time object
// removal).
cudaError_t launch_occupancy_scatter(const float* compact_raw, const int32_t* kept_idx, const int32_t* count, long long max_kept, int out_ch,
                                     const float4* ws, int use_removal, float removal, float* raw, int num_sms, cudaStream_t st);
// The exclusive scan of n per-block counts in place (one block), the total -> counts[n] and *count: the middle step of the
// compaction above, for other per-block counts (baked.cu's fallback rays)
cudaError_t launch_occupancy_scan(int32_t* counts, int n, int32_t* count, cudaStream_t st);

// Early termination (nrn_field_forward_terminate).  init: T = 1 and term = S for every ray.  compact: the lookup and
// compaction of one segment's slots (kept indices are the samples' indices in the pass, so launch_occupancy_scatter takes
// them as they are).  transmittance: every alive ray multiplies T by (1 - alpha + 1e-10) over samples [s0, s0 + len), in
// order, and dies (term = s0 + len) when T < threshold.
cudaError_t launch_termination_init(const TermPass& t, cudaStream_t st);
cudaError_t launch_termination_compact(const OccGrid& g, const OccPoints& pts, const OccSegment& seg, const OccCompact& c, cudaStream_t st);
cudaError_t launch_termination_transmittance(const TermPass& t, int s0, int len, cudaStream_t st);

}  // namespace nrn
