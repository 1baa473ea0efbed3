// Weight gradients (WGRAD) of the fused field:  dW_l[out][in] = sum_p dY_l[p][out] * X_l[p][in],
// db_l[out] = sum_p dY_l[p][out]  -- what torch.autograd accumulates into the .grad of
// NeRF.pts_linears / output_linear (run_nerf_helpers.py:218-238) and ray_bending.network /
// rigidity_network (run_nerf_helpers.py:411-482).
//
// Both operands are the fp16 chunk-major tile images written by the forward (activation stash) and
// DGRAD (gradient stash) kernels; read MN-major they are exactly the transposed operands WGRAD needs
// (sm90_ptx.cuh: transposed wgmma), so no transpose pass exists.  The contraction runs over points (K = 128 per tile).
//
// Decomposition: a fixed list of jobs; a job is a set of up to three "sub-MMAs" over one gradient image block (A)
// and one activation image block (B) per tile (jobs 0-9: one NeRF layer; jobs 10-11: the five small ray-bender
// layers, grouped so that their images are one contiguous range of each stash).  The fp32 accumulators live in
// registers: a consumer warpgroup holds at most 64 x 256 of them, so a CTA (two consumer warpgroups) covers 128 rows
// of dW and a NeRF layer's 256-row dW is split over two CTAs ("halves").  The two halves of a split are the two CTAs
// of one cluster: each fetches its own A block (different gradient columns) and half of the shared B block, which TMA
// multicasts into both CTAs, so every activation block leaves L2 once per cluster.  A pipeline stage holds one
// tile's A block followed by its B block (at most 48 chunks, 96 KB); the 192 KB ring has 2 such stages, or 4 for
// the 48 KB tiles of the L5e / L0 jobs, so the next tile's operands are in flight while the current tile's MMAs and
// bias sums run.  A stage that received multicast data is refilled only after the consumers of BOTH CTAs released
// it (each consumer warp arrives on its own and on the partner's empty barrier).  Every job is
// split over contiguous tile ranges ("split-K") proportionally to its bytes; partial sums go to a scratch buffer
// and a second kernel reduces them in a fixed order (deterministic) while un-padding / un-permuting
// into the reference's parameter layout and dividing out the loss scale.
// The kernel is HBM-bound (each stash byte feeds 256 MACs): while the MMAs of a stage run, the consumer warps
// compute the bias gradient from the same shared-memory stage.
//
// Compact mode (WgradParams.compact): the same two bender jobs over the tangent / adjoint stashes of
// the divergence regulariser (div.cu), which hold only the bender images.
#include "nrn_common.cuh"
#include "sm90_ptx.cuh"
#include "wgrad.cuh"

namespace nrn {

namespace {

constexpr int kRingBytes = 96 * kChunkBytes;       // operand ring: 96 chunk images (128 points x 8 features each)
constexpr int kMaxStages = 4;
constexpr uint32_t kPieceBytes = 16384;            // size of one bulk copy
constexpr int kWgThreads = 384;                    // 2 consumer warpgroups (MMA, bias sums, drain), producer warpgroup

// One 64-row M tile of a sub-MMA, issued by one warpgroup: dW rows [m0, m0 + 64) of the sub.
struct Unit {
  int a_chunk, b_chunk;  // operand chunk offsets inside the A / B stage
  int dst, ld;           // scratch partial: row r of the tile goes to part[dst + r * ld + column]
  int rows;              // valid rows of the tile (the rest belong to padding or to the next sub)
};
struct Job {
  int a_off, a_chunks;   // contiguous range of the gradient stash tile (bytes, chunks)
  int b_off, b_chunks;   // contiguous range of the activation stash tile
  int bias;              // compute column sums over all A chunks
  int bias_off;          // column of the first A chunk in the job's bias partial
  Unit u[2];             // the units of the calling consumer warpgroup
};

// job ids: 0 head, 1..7 = L1..L7 (input h_l), 8 L5e, 9 L0, 10 = {B4,B3,B2}, 11 = {B1,B0}; half: rows [128 half, +128)
// of a NeRF layer's dW; g: the calling consumer warpgroup (0 or 1; the producer passes 0).  Built per warpgroup so that
// the units are selected by branches, not by a runtime array index, and the Job stays in registers.
// Scratch partial layout: NeRF jobs [256 rows][256]; bender jobs [sub][128 rows][128].
// The bender jobs read adjacent images of both stashes: A = dYb4 dYb3 dYb2 (job 10), dYb1 dYb0 (job 11); B = Hb2 Hb3
// Hb4 (job 10), bender input and Hb1 (job 11).
__host__ __device__ constexpr Image span(Image first, Image last) { return {first.off, (last.end() - first.off) / kChunkBytes}; }
__host__ __device__ constexpr int chunk_in(Image im, Image first) { return (im.off - first.off) / kChunkBytes; }
constexpr Image kJ10A = span(kGsYb4, kGsYb2), kJ10B = span(kStHb2, kStHb4), kJ11A = span(kGsYb1, kGsYb0), kJ11B = span(kStBin, kStHb1);

__device__ __forceinline__ Job job_desc(int j, int half, int g, int compact) {
  Job jb{};
  if (j <= 9) {
    int a_off, a_cols, b_off, b_cols, bias = 1;
    if (j == 0) { a_off = kGsRaw.off; a_cols = 8 * kGsRaw.chunks; b_off = kStH + 7 * kHBytes; b_cols = 8 * kHChunks; }
    else if (j == 8) { a_off = kGsY + 5 * kHBytes; a_cols = 8 * kHChunks; b_off = kStE.off; b_cols = 8 * kStE.chunks; bias = 0; }
    else if (j == 9) { a_off = kGsY; a_cols = 8 * kHChunks; b_off = kStE.off; b_cols = 8 * kStE.chunks; }
    else { a_off = kGsY + j * kHBytes; a_cols = 8 * kHChunks; b_off = kStH + (j - 1) * kHBytes; b_cols = 8 * kHChunks; }
    jb.a_off = a_off + half * 16 * kChunkBytes; jb.a_chunks = min(a_cols / 8 - 16 * half, 16);
    jb.b_off = b_off; jb.b_chunks = b_cols / 8;
    jb.bias = bias; jb.bias_off = half * 128;
    const int m0 = half * 128 + g * 64;
    jb.u[0] = {8 * g, 0, m0 * 256, 256, max(min(a_cols - m0, 64), 0)};
    return jb;
  }
  // in compact mode the stashes hold only the bender images
  const int ga = compact ? kGsYb4.off : 0, sa = compact ? kStBin.off : 0;
  if (j == 10) {
    jb.a_off = kJ10A.off - ga; jb.a_chunks = kJ10A.chunks;
    jb.b_off = kJ10B.off - sa; jb.b_chunks = kJ10B.chunks;
    if (g == 0) {
      jb.u[0] = {chunk_in(kGsYb4, kJ10A), chunk_in(kStHb4, kJ10B), 0, 128, 8 * kGsYb4.chunks};           // dYb4 x Hb4
      jb.u[1] = {chunk_in(kGsYb3, kJ10A), chunk_in(kStHb3, kJ10B), 16384, 128, 8 * kGsYb3.chunks};       // dYb3 x Hb3
    } else {
      jb.u[0] = {chunk_in(kGsYb2, kJ10A), chunk_in(kStHb2, kJ10B), 2 * 16384, 128, 64};                  // dYb2 x Hb2, rows 0-63
      jb.u[1] = {chunk_in(kGsYb2, kJ10A) + 8, chunk_in(kStHb2, kJ10B), 2 * 16384 + 64 * 128, 128, 8 * kGsYb2.chunks - 64};  // rows 64-
    }
  } else {
    jb.a_off = kJ11A.off - ga; jb.a_chunks = kJ11A.chunks;
    jb.b_off = kJ11B.off - sa; jb.b_chunks = kJ11B.chunks;
    if (g == 0) {
      jb.u[0] = {chunk_in(kGsYb1, kJ11A), chunk_in(kStHb1, kJ11B), 0, 128, 64};                          // dYb1 x Hb1, rows 0-63
      jb.u[1] = {chunk_in(kGsYb1, kJ11A) + 8, chunk_in(kStHb1, kJ11B), 64 * 128, 128, 8 * kGsYb1.chunks - 64};  // rows 64-
    } else {
      jb.u[0] = {chunk_in(kGsYb0, kJ11A), chunk_in(kStBin, kJ11B), 16384, 128, 64};                      // dYb0 x input, rows 0-63
      jb.u[1] = {chunk_in(kGsYb0, kJ11A) + 8, chunk_in(kStBin, kJ11B), 16384 + 64 * 128, 128, 8 * kGsYb0.chunks - 64};  // rows 64-
    }
  }
  jb.bias = compact ? 0 : 1;   // the tangent chain of the divergence term has no bias
  return jb;
}

// View-dependent head (training without a bender, wgrad_views_kernel): the trunk's jobs 0-9 (job 0's row 3 is
// alpha_linear), then 12 = feature_linear (A = dF, B = H8; two halves like a NeRF layer), 13 and 15 = views_linears.0's
// feature and direction columns (A = dYv, B = F / Dir of the view stash: 48 and 20 chunks a stage, so that the ring
// holds two and four stages), 14 = rgb_linear (A = d_raw, B = Hv).
// Scratch partial layout: job 12 [256 rows][256]; job 13 [128 rows][256] (+ the bias); job 15 [128 rows][32]; job 14
// [16 rows][128].
constexpr int kJobFeature = 12, kJobViewsF = 13, kJobRgb = 14, kJobViewsE = 15;
__device__ __forceinline__ Job views_job_desc(int j, int half, int g) {
  if (j <= 9) return job_desc(j, half, g, 0);
  Job jb{};
  jb.bias = 1;
  if (j == kJobFeature) {
    jb.a_off = kVgF.off + half * 16 * kChunkBytes; jb.a_chunks = 16;
    jb.b_off = kStH + 7 * kHBytes; jb.b_chunks = kHChunks;
    jb.bias_off = half * 128;
    const int m0 = half * 128 + g * 64;
    jb.u[0] = {8 * g, 0, m0 * 256, 256, 64};
  } else if (j == kJobViewsF || j == kJobViewsE) {
    const Image b = j == kJobViewsF ? kVsF : kVsDir;
    jb.a_off = kVgYv.off; jb.a_chunks = kVgYv.chunks;
    jb.b_off = b.off; jb.b_chunks = b.chunks;
    jb.bias = j == kJobViewsF;   // the bias gradient once
    jb.u[0] = {8 * g, 0, g * 64 * 8 * b.chunks, 8 * b.chunks, 64};
  } else {
    jb.a_off = kGsRaw.off; jb.a_chunks = kGsRaw.chunks;
    jb.b_off = kVsHv.off; jb.b_chunks = kVsHv.chunks;
    jb.u[0] = {0, 0, 0, 8 * kVsHv.chunks, g == 0 ? 8 * kGsRaw.chunks : 0};
  }
  return jb;
}

struct Shared {
  uint64_t full[kMaxStages];
  uint64_t empty[kMaxStages];
  int abort_flag;
};

// Operand ring: stage s holds one tile's A block at smem + s * stage_bytes and its B block right behind it.
struct Ring {
  uint8_t* smem;
  int stage_bytes, n_stages;
  bool paired;
  uint32_t partner_empty;   // shared::cluster address of the partner CTA's empty[0] (paired CTAs)
};

// which (job, split, half) does this CTA own, and which scratch partial is the split's?  job_ids[] / splits[] /
// halves[] come from the host (WgradParams); the halves of one split are the two CTAs of one cluster.
__device__ __forceinline__ bool locate(const WgradParams& p, int cta, int& job, int& split, int& nsplit, int& half, int& halves,
                                       int& part) {
  int base = 0, pbase = 0;
  for (int j = 0; j < p.n_jobs; ++j) {
    const int n = p.splits[j] * p.halves[j];
    if (cta < base + n) {
      job = p.job_ids[j]; split = (cta - base) / p.halves[j]; half = (cta - base) % p.halves[j]; nsplit = p.splits[j];
      halves = p.halves[j];
      part = pbase + split;
      return true;
    }
    base += n;
    pbase += p.splits[j];
  }
  return false;
}

template <int N, int NR>
__device__ __forceinline__ void unit_mma(float (&acc)[NR], const Unit& u, uint32_t a0, uint32_t b0, int it) {
  // MN-major: SBO = stride between 8-feature chunks, LBO = stride between 8-point groups
  const uint64_t adesc = gmma_desc(a0 + u.a_chunk * kChunkBytes, 128, kChunkBytes);
  const uint64_t bdesc = gmma_desc(b0 + u.b_chunk * kChunkBytes, 128, kChunkBytes);
#pragma unroll
  for (int k = 0; k < kTileM / 16; ++k)
    wgmma<N, 1, 1>(acc, gmma_desc_advance(adesc, k * 256), gmma_desc_advance(bdesc, k * 256), (it | k) ? 1u : 0u);
}

template <int NR>
__device__ __forceinline__ void unit_drain(const float (&acc)[NR], const Unit& u, float* part) {
  const int r0 = ((threadIdx.x >> 5) & 3) * 16 + ((threadIdx.x & 31) >> 2), q = threadIdx.x & 3;  // sm90_ptx.cuh
#pragma unroll
  for (int j = 0; j < NR / 4; ++j)
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = r0 + 8 * i;
      if (r < u.rows) *reinterpret_cast<float2*>(part + u.dst + r * u.ld + 8 * j + 2 * q) = make_float2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]);
    }
}

// One consumer warpgroup: its units' MMAs over every tile of the split (accumulators in registers), the bias column
// sums of its warps' A chunks, then the drain into the scratch partial.  N0 / N1 = 0: no such unit.
template <int N0, int N1>
__device__ __forceinline__ void consume(const Job& jb, const Unit& u0, const Unit& u1, const Ring& R, Shared* sh, const Waiter& W,
                                        int n_tiles_local, float* part, bool have) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float acc0[N0 > 0 ? N0 / 2 : 1];
  float acc1[N1 > 0 ? N1 / 2 : 1];
  // the first MMA overwrites the accumulators; defined inputs keep ptxas from spilling and serialising the wgmma chain
#pragma unroll
  for (int i = 0; i < (N0 > 0 ? N0 / 2 : 1); ++i) acc0[i] = 0.f;
#pragma unroll
  for (int i = 0; i < (N1 > 0 ? N1 / 2 : 1); ++i) acc1[i] = 0.f;
  float bias_acc = 0.f;
  uint32_t stage = 0, phase = 0;
  for (int it = 0; it < n_tiles_local; ++it) {
    W.wait(&sh->full[stage], phase, 201);
    const uint8_t* st_a = R.smem + stage * R.stage_bytes;
    const uint32_t a0 = smem_u32(st_a), b0 = a0 + jb.a_chunks * kChunkBytes;
    if constexpr (N0 > 0) {
      acc_fence(acc0);
      acc_fence(acc1);
      wgmma_fence();
      unit_mma<N0>(acc0, u0, a0, b0, it);
      if constexpr (N1 > 0) unit_mma<N1>(acc1, u1, a0, b0, it);
      wgmma_commit();
    }
    // db[feature] = sum over points of dY: warp w owns chunks 4w .. 4w+3 of the A block; lane l reads rows l, l+32,
    // l+64, l+96 of each chunk (consecutive lanes = consecutive 16-byte rows: conflict-free), keeps 4 x 8 partial
    // sums and a warp transpose-reduce leaves the total of (chunk 4w + L/8, feature L%8) in lane L.
    if (jb.bias) {
      float s[32];
#pragma unroll
      for (int cc = 0; cc < 4; ++cc) {
        const int c = warp * 4 + cc;
        const uint8_t* src = st_a + c * kChunkBytes + lane * 16;
        float t8[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (c < jb.a_chunks) {        // chunks beyond the A block belong to the B block
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            const uint4 w = *reinterpret_cast<const uint4*>(src + r * 512);
            const uint32_t wv[4] = {w.x, w.y, w.z, w.w};   // unpacked by value: no address of a local, no stack frame
#pragma unroll
            for (int qq = 0; qq < 4; ++qq) {
              t8[2 * qq] += h_lo(wv[qq]);
              t8[2 * qq + 1] += h_hi(wv[qq]);
            }
          }
        }
#pragma unroll
        for (int qq = 0; qq < 8; ++qq) s[cc * 8 + qq] = t8[qq];
      }
      bias_acc += warp_transpose_reduce(s, lane);
    }
    if constexpr (N0 > 0) {
      wgmma_wait<0>();
      acc_fence(acc0);
      acc_fence(acc1);
    }
    __syncwarp();
    if (lane == 0) {
      mbar_arrive(&sh->empty[stage]);
      if (R.paired) mbar_arrive_cluster(R.partner_empty + stage * static_cast<uint32_t>(sizeof(uint64_t)));
    }
    if (++stage == R.n_stages) { stage = 0; phase ^= 1u; }
  }
  if (!have || n_tiles_local == 0) return;
  if (jb.bias && (warp * 4 + (lane >> 3)) < jb.a_chunks) part[65536 + jb.bias_off + warp * 32 + lane] = bias_acc;
  if constexpr (N0 > 0) unit_drain(acc0, u0, part);
  if constexpr (N1 > 0) unit_drain(acc1, u1, part);
}

// VIEWS: the view-dependent head's job set (views_job_desc), whose jobs 12-15 read A and B blocks from the view stashes
template <bool VIEWS>
__device__ __forceinline__ void wgrad_body(const WgradParams& p, const WgradViewParams& v) {
  extern __shared__ __align__(1024) uint8_t smem[];
  Shared* sh = reinterpret_cast<Shared*>(smem + kRingBytes);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  int job_id = 0, split = 0, nsplit = 1, half = 0, halves = 1, part_idx = 0;
  const bool have = locate(p, blockIdx.x, job_id, split, nsplit, half, halves, part_idx);
  const Job jb = VIEWS ? views_job_desc(job_id, half, (warp >> 2) & 1) : job_desc(job_id, half, (warp >> 2) & 1, p.compact);
  // contiguous tile range of this split
  const int per = (p.n_tiles + nsplit - 1) / nsplit;
  const int t_begin = have ? min(split * per, p.n_tiles) : 0;
  const int t_end = have ? min(t_begin + per, p.n_tiles) : 0;
  const int n_local = t_end - t_begin;
  // the two halves of a NeRF-layer split share their B blocks with the other CTA of the cluster; every other CTA
  // (head, bender jobs, an idle CTA) works alone and shares only the cluster barriers with its neighbour
  const bool paired = have && halves == 2;
  const uint32_t rank = cluster_ctarank(), partner = rank ^ 1u;
  // both halves of a split have the same A and B block sizes, hence the same stage layout
  const int stage_bytes = (jb.a_chunks + jb.b_chunks) * kChunkBytes;
  const int n_stages = min(kMaxStages, kRingBytes / stage_bytes);

  if (threadIdx.x == 0) {
    for (int i = 0; i < n_stages; ++i) {
      mbar_init(&sh->full[i], 1);
      mbar_init(&sh->empty[i], paired ? 16 : 8);   // one arrival per consumer warp of every CTA that reads the stage
    }
    sh->abort_flag = 0;
    fence_mbar_init();
  }
  // the partner's barriers are initialised before any multicast data or remote arrival can reach them
  cluster_sync();
  const Waiter W{&sh->abort_flag, p.err, paired, paired ? mapa_shared(&sh->abort_flag, partner) : 0u};
  const Ring R{smem, stage_bytes, n_stages, paired, paired ? mapa_shared(&sh->empty[0], partner) : 0u};

  if (warp >= 8) {
    setmaxnreg_dec<kProducerRegs>();
    // ===================== producer: one tile's A and B blocks per stage, 16 KB bulk copies =====================
    if (warp == 8 && lane == 0) {
      const uint32_t a_bytes = static_cast<uint32_t>(jb.a_chunks) * kChunkBytes, b_bytes = static_cast<uint32_t>(jb.b_chunks) * kChunkBytes;
      // paired: this CTA fetches its own A block and its half of the B block, the latter multicast into both CTAs
      const uint32_t b_begin = paired ? rank * (b_bytes / 2) : 0u, b_end = paired ? b_begin + b_bytes / 2 : b_bytes;
      // the stashes the job's A and B blocks come from
      const uint8_t* a_base = p.gstash;
      const uint8_t* b_base = p.stash;
      long long a_tile = p.gstash_tile_bytes, b_tile = p.stash_tile_bytes;
      if constexpr (VIEWS) {
        if (job_id == kJobFeature || job_id == kJobViewsF || job_id == kJobViewsE) { a_base = v.vgstash; a_tile = kVGradTileBytes; }
        if (job_id == kJobViewsF || job_id == kJobViewsE || job_id == kJobRgb) { b_base = v.vstash; b_tile = kVStashTileBytes; }
      }
      uint32_t stage = 0, phase = 0;
      for (int it = 0; it < n_local; ++it) {
        const long long tile = t_begin + it;
        const uint8_t* a_src = a_base + tile * a_tile + jb.a_off;
        const uint8_t* b_src = b_base + tile * b_tile + jb.b_off;
        W.wait(&sh->empty[stage], phase ^ 1u, 101);
        mbar_arrive_expect_tx(&sh->full[stage], a_bytes + b_bytes);   // the partner delivers the other half of B
        uint8_t* dst = smem + stage * stage_bytes;
        for (uint32_t o = 0; o < a_bytes; o += kPieceBytes)
          tma_bulk_g2s(dst + o, a_src + o, a_bytes - o < kPieceBytes ? a_bytes - o : kPieceBytes, &sh->full[stage]);
        dst += a_bytes;
        for (uint32_t o = b_begin; o < b_end; o += kPieceBytes) {
          const uint32_t n = b_end - o < kPieceBytes ? b_end - o : kPieceBytes;
          if (paired) tma_bulk_g2s_multicast(dst + o, b_src + o, n, &sh->full[stage], 0x3);
          else tma_bulk_g2s(dst + o, b_src + o, n, &sh->full[stage]);
        }
        if (++stage == n_stages) { stage = 0; phase ^= 1u; }
      }
    }
  } else {
    setmaxnreg_inc<kConsumerRegs>();
    const int g = warp >> 2;
    float* part = p.scratch + static_cast<size_t>(part_idx) * kWgScratchFloats;
    const Unit& u0 = jb.u[0];
    const Unit& u1 = jb.u[1];
    if (VIEWS && job_id == kJobViewsF) {
      consume<8 * kVsF.chunks, 0>(jb, u0, u1, R, sh, W, n_local, part, have);
    } else if (VIEWS && job_id == kJobViewsE) {
      consume<8 * kVsDir.chunks, 0>(jb, u0, u1, R, sh, W, n_local, part, have);
    } else if (VIEWS && job_id == kJobRgb) {
      if (u0.rows > 0) consume<8 * kVsHv.chunks, 0>(jb, u0, u1, R, sh, W, n_local, part, have);
      else consume<0, 0>(jb, u0, u1, R, sh, W, n_local, part, have);
    } else if (VIEWS || job_id <= 9) {   // the trunk's jobs 0-9 and feature_linear (a NeRF layer's shape)
      const bool mine = u0.rows > 0;
      // N = columns of the job's activation image
      if (job_id == 8 || job_id == 9) {
        if (mine) consume<8 * kStE.chunks, 0>(jb, u0, u1, R, sh, W, n_local, part, have);
        else consume<0, 0>(jb, u0, u1, R, sh, W, n_local, part, have);
      } else {
        if (mine) consume<8 * kHChunks, 0>(jb, u0, u1, R, sh, W, n_local, part, have);
        else consume<0, 0>(jb, u0, u1, R, sh, W, n_local, part, have);
      }
    } else if (job_id == 10) {
      if (g == 0) consume<8 * kStHb4.chunks, 8 * kStHb3.chunks>(jb, u0, u1, R, sh, W, n_local, part, have);
      else consume<8 * kStHb2.chunks, 8 * kStHb2.chunks>(jb, u0, u1, R, sh, W, n_local, part, have);
    } else {
      if (g == 0) consume<8 * kStHb1.chunks, 8 * kStHb1.chunks>(jb, u0, u1, R, sh, W, n_local, part, have);
      else consume<8 * kStBin.chunks, 8 * kStBin.chunks>(jb, u0, u1, R, sh, W, n_local, part, have);
    }
  }
  // No CTA leaves while its partner may still arrive on its barriers or write its abort flag.  Multicast data has
  // landed: each CTA's consumers waited for every tile's full barrier.  Every thread gets here after a finite number of
  // bounded waits (an abort reaches the partner through its abort flag), so this barrier cannot hang.
  __syncwarp();
  cluster_sync();
}

}  // namespace

__global__ void __launch_bounds__(kWgThreads, 1) wgrad_kernel(const WgradParams p) { wgrad_body<false>(p, WgradViewParams{}); }
__global__ void __launch_bounds__(kWgThreads, 1) wgrad_views_kernel(const WgradParams p, const WgradViewParams v) {
  wgrad_body<true>(p, v);
}


// ------------------------------------------------------------------------------------------------
// Deterministic reduction of the split partials into the reference's parameter layout.
// One thread per destination element of the flat gradient buffers (their shapes: nrn_common.cuh).
// ------------------------------------------------------------------------------------------------
namespace {

struct Src {
  int job;   // job id
  int off;   // float offset inside the job's partial (weights) or bias index (bias == 1)
  int off2;  // second weight element to add (>= 0) or -1
  int bias;
};

__device__ __forceinline__ Src nerf_w(int job, int m, int n) { return {job, m * 256 + n, -1, 0}; }
__device__ __forceinline__ Src nerf_b(int job, int m) { return {job, m, -1, 1}; }
__device__ __forceinline__ Src bend_w(int job, int sub, int m, int n, int n2 = -1) {
  return {job, sub * 16384 + m * 128 + n, n2 >= 0 ? sub * 16384 + m * 128 + n2 : -1, 0};
}

// TC (time-conditioned baseline): W0 [256][63 + 32], W5 [256][63 + 32 + 256]; the latent columns come from
// tc_dw_lat_kernel (field_bwd.cu) as Src{kLatJob, index into its [2][256][32] output}.
constexpr int kLatJob = -1;
template <bool TC = false>
__device__ __forceinline__ Src nerf_src(int idx, int out_ch, bool& ok) {
  ok = true;
  constexpr int lat = TC ? kLatent : 0;
  constexpr int in0 = nerf_in(0) + lat, in5 = nerf_in(5) + lat;   // L0: the embedding (| z); L5: [embedding (| z) | h]
  constexpr int pe = nerf_in(0);
  const int sz0 = 256 * in0 + 256, szl = 256 * 256 + 256, sz5 = 256 * in5 + 256;
  if (idx < sz0) {
    if (idx < 256 * in0) {
      if constexpr (TC) {
        const int m = idx / in0, k = idx % in0;
        if (k >= pe) return {kLatJob, m * kLatent + (k - pe), -1, 0};
      }
      return nerf_w(9, idx / in0, idx % in0);
    }
    return nerf_b(9, idx - 256 * in0);
  }
  idx -= sz0;
  for (int l = 1; l < 8; ++l) {
    const int sz = l == 5 ? sz5 : szl;
    if (idx < sz) {
      if (l == 5) {
        if (idx < 256 * in5) {
          const int m = idx / in5, k = idx % in5;
          if constexpr (TC) {
            if (k >= pe && k < pe + lat) return {kLatJob, (256 + m) * kLatent + (k - pe), -1, 0};
          }
          return k < pe ? nerf_w(8, m, k) : nerf_w(5, m, k - (pe + lat));
        }
        return nerf_b(5, idx - 256 * in5);
      }
      if (idx < 65536) return nerf_w(l, idx >> 8, idx & 255);
      return nerf_b(l, idx - 65536);
    }
    idx -= sz;
  }
  if (idx < out_ch * 256) {
    const int m = idx >> 8;
    ok = m < 4;   // output channel 4 never reaches the loss: zero gradient (SURVEY.md 7.3-6)
    return nerf_w(0, m, idx & 255);
  }
  idx -= out_ch * 256;
  ok = idx < 4;
  return nerf_b(0, idx);
}

// Bias index of the bender jobs = column inside the job's concatenated A images: job 10 dYb4 | dYb3 | dYb2, job 11
// dYb1 | dYb0 (rigidity columns from 64 on).  Sub-MMAs: job 10 0 = B4, 1 = B3, 2 = B2; job 11 0 = B1, 1 = B0.
__device__ __forceinline__ Src bender_src(int idx, bool& ok) {
  using namespace bparam;
  constexpr int c_yb3 = 8 * chunk_in(kGsYb3, kJ10A), c_yb2 = 8 * chunk_in(kGsYb2, kJ10A), c_yb1 = 8 * chunk_in(kGsYb1, kJ11A),
                c_yb0 = 8 * chunk_in(kGsYb0, kJ11A);
  constexpr int n_w0 = floats(NetW0), n_b = floats(NetB0), n_w = floats(NetW1), n_w4 = floats(NetW4), n_rw0 = floats(RigW0),
                n_rb = floats(RigB0), n_rw1 = floats(RigW1), n_rw2 = floats(RigW2), k0 = kShape[NetW0][1];
  ok = true;
  if (idx < n_w0) {  // net_w0: xyz columns collect the hi and lo operand columns
    const int m = idx / k0, k = idx % k0;
    return k < 3 ? bend_w(11, 1, m, k, k + 3) : bend_w(11, 1, m, 6 + (k - 3));
  }
  idx -= n_w0;
  if (idx < n_b) return {11, c_yb0 + idx, -1, 1};                                 // net_b0
  idx -= n_b;
  if (idx < n_w) return bend_w(11, 0, idx >> 6, idx & 63);                        // net_w1
  idx -= n_w;
  if (idx < n_b) return {11, c_yb1 + idx, -1, 1};                                 // net_b1
  idx -= n_b;
  if (idx < n_w) return bend_w(10, 2, idx >> 6, idx & 63);                        // net_w2
  idx -= n_w;
  if (idx < n_b) return {10, c_yb2 + idx, -1, 1};                                 // net_b2
  idx -= n_b;
  if (idx < n_w) return bend_w(10, 1, idx >> 6, idx & 63);                        // net_w3
  idx -= n_w;
  if (idx < n_b) return {10, c_yb3 + idx, -1, 1};                                 // net_b3
  idx -= n_b;
  if (idx < n_w4) return bend_w(10, 0, idx >> 6, idx & 63);                       // net_w4
  idx -= n_w4;
  if (idx < n_rw0) return bend_w(11, 1, 64 + idx / 3, idx % 3, idx % 3 + 3);      // rig_w0
  idx -= n_rw0;
  if (idx < n_rb) return {11, c_yb0 + 64 + idx, -1, 1};                           // rig_b0
  idx -= n_rb;
  if (idx < n_rw1) return bend_w(11, 0, 64 + (idx >> 5), 64 + (idx & 31));        // rig_w1
  idx -= n_rw1;
  if (idx < n_rb) return {11, c_yb1 + 64 + idx, -1, 1};                           // rig_b1
  idx -= n_rb;
  if (idx < n_rw2) return bend_w(10, 2, 64, 64 + idx);                            // rig_w2
  idx -= n_rw2;
  return {10, c_yb2 + 64, -1, 1};                                                 // rig_b2
}

// View-dependent head: the trunk as nerf_src (jobs 1-9), then the head block in module order (nrn_common.cuh: vparam)
__device__ __forceinline__ Src views_src(int idx) {
  bool ok;
  if (idx < kViewsTrunkFloats) return nerf_src<false>(idx, 4, ok);
  idx -= kViewsTrunkFloats;
  using namespace vparam;
  constexpr int kIn = kShape[ViewsW][1], kDir = 8 * kVsDir.chunks;
  if (idx < floats(ViewsW)) {   // [feature | direction encoding] inputs: the feature job's and the direction job's partials
    const int m = idx / kIn, k = idx % kIn;
    return k < 256 ? Src{kJobViewsF, m * 256 + k, -1, 0} : Src{kJobViewsE, m * kDir + (k - 256), -1, 0};
  }
  idx -= floats(ViewsW);
  if (idx < floats(ViewsB)) return {kJobViewsF, idx, -1, 1};
  idx -= floats(ViewsB);
  if (idx < floats(FeatureW)) return nerf_w(kJobFeature, idx >> 8, idx & 255);
  idx -= floats(FeatureW);
  if (idx < floats(FeatureB)) return nerf_b(kJobFeature, idx);
  idx -= floats(FeatureB);
  if (idx < floats(AlphaW)) return nerf_w(0, 3, idx);   // the head job's row 3
  idx -= floats(AlphaW);
  if (idx < floats(AlphaB)) return nerf_b(0, 3);
  idx -= floats(AlphaB);
  if (idx < floats(RgbW)) return {kJobRgb, (idx >> 7) * 128 + (idx & 127), -1, 0};
  return {kJobRgb, idx - floats(RgbW), -1, 1};
}

}  // namespace

// The fixed-order sum over the split partials of job s.job (split 0, 1, 2, ...): deterministic gradients
__device__ __forceinline__ float split_sum(const WgradParams& p, const Src& s) {
  float sum = 0.f;
  int base = 0, slot = -1;
  for (int j = 0; j < p.n_jobs; ++j) {
    if (p.job_ids[j] == s.job) { slot = j; break; }
    base += p.splits[j];
  }
  if (slot >= 0) {
    const int nsplit = p.splits[slot];
    const int per = (p.n_tiles + nsplit - 1) / nsplit;
    const int n_valid = min(nsplit, (p.n_tiles + per - 1) / per);   // splits beyond that owned no tiles: scratch unwritten
    const float* __restrict__ src = p.scratch + static_cast<size_t>(base) * kWgScratchFloats + (s.bias ? 65536 + s.off : s.off);
    const bool has2 = !s.bias && s.off2 >= 0;
    const int d2 = has2 ? s.off2 - s.off : 0;
    // fixed summation order (split 0, 1, 2, ...) = deterministic gradients; the loads of 8 splits are in flight together
    int sp = 0;
    for (; sp + 8 <= n_valid; sp += 8) {
      float a[8], b[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float* q = src + static_cast<size_t>(sp + i) * kWgScratchFloats;
        a[i] = __ldg(q);
        b[i] = has2 ? __ldg(q + d2) : 0.f;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        sum += a[i];
        if (has2) sum += b[i];
      }
    }
    for (; sp < n_valid; ++sp) {
      const float* q = src + static_cast<size_t>(sp) * kWgScratchFloats;
      sum += __ldg(q);
      if (has2) sum += __ldg(q + d2);
    }
  }
  return sum;
}

template <bool TC>
__device__ __forceinline__ void wgrad_reduce(const WgradParams p, const WgradDst dst, int out_ch, const float* dw_lat) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int nerf_n = dst.nerf_n, bend_n = dst.bend_n;
  if (idx >= nerf_n + bend_n) return;
  bool ok;
  const Src s = idx < nerf_n ? nerf_src<TC>(idx, out_ch, ok) : bender_src(idx - nerf_n, ok);
  const float scale = loss_scale(p.amax);
  float sum = 0.f;
  const bool lat = TC && s.job == kLatJob;   // tc_dw_lat_kernel's sums: already divided by the loss scale
  if (ok && !lat && !(s.bias && p.compact)) sum = split_sum(p, s);
  const float v = lat ? __ldg(dw_lat + s.off) : sum / scale;
  float* out;
  bool acc;
  if (idx < nerf_n) {
    const int n_pts = nerf_n - out_ch * 257;
    out = (idx >= n_pts && dst.nerf_head) ? dst.nerf_head + (idx - n_pts) : dst.nerf + idx;
    acc = dst.acc_nerf != 0;
  } else {
    out = dst.bend + (idx - nerf_n);
    acc = dst.acc_bend != 0;
  }
  *out = acc ? *out + v : v;
}


__global__ void wgrad_reduce_kernel(const WgradParams p, const WgradDst dst, int out_ch) { wgrad_reduce<false>(p, dst, out_ch, nullptr); }
__global__ void wgrad_reduce_tc_kernel(const WgradParams p, const WgradDst dst, int out_ch, const float* dw_lat) {
  wgrad_reduce<true>(p, dst, out_ch, dw_lat);
}
// The view-dependent head's flat layout (nerf_views_grad_floats): dst.nerf the trunk, dst.nerf_head (or behind it) the
// head block; dst.nerf_n is the whole count
__global__ void wgrad_views_reduce_kernel(const WgradParams p, const WgradDst dst) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= dst.nerf_n) return;
  const float v = split_sum(p, views_src(idx)) / loss_scale(p.amax);
  float* out = (idx >= kViewsTrunkFloats && dst.nerf_head) ? dst.nerf_head + (idx - kViewsTrunkFloats) : dst.nerf + idx;
  *out = dst.acc_nerf ? *out + v : v;
}

// ------------------------------------------------------------------------------------------------
namespace {
// Relative cost of one tile of every job's CTAs, by job id = 2 KB chunks a CTA receives (a NeRF layer's half: 16 gradient
// chunks + the activation block; feature_linear's half likewise; views_linears.0's feature columns 16 + 32, its direction
// columns 16 + 4, both one MMA over a double-buffered ring).  The head job, rgb_linear (2 + 16) and the three-MMA bender
// job stream a little slower per byte, hence their surcharge.  The plan decides how the fp32 partial sums associate:
// changing a weight changes the gradients' last bits.
constexpr int kJobCost[16] = {46, 48, 48, 48, 48, 48, 48, 48, 16 + 8 + 8, 16 + 8 + 8, 54, 24 + 18, 48, 48, 24, 20};
// CTAs per split: a NeRF layer's and feature_linear's 256-row dW take two; the head's 16-row dW, the bender jobs and the
// other view-head jobs fit one CTA
constexpr int job_halves(int j) { return (j >= 1 && j <= 9) || j == kJobFeature ? 2 : 1; }

// Plans how the jobs jobs[0, n) split their tiles over the CTAs, writes the plan into p and launches `kernel`
// (wgrad_kernel or wgrad_views_kernel).
template <typename... Args>
cudaError_t launch_jobs(void (*kernel)(WgradParams, Args...), int* s_max_clusters, WgradParams& p, const int* jobs, int n,
                        int num_sms, cudaStream_t st, Args... args) {
  // Launched in clusters of 2 CTAs (the two halves of a NeRF-layer split).  A cluster lives inside one GPC, so the
  // CTAs that can run at once are the resident clusters x 2, which can be fewer than the SMs.
  const size_t smem = kRingBytes + sizeof(Shared) + 64;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  cudaLaunchAttribute cluster{};
  cluster.id = cudaLaunchAttributeClusterDimension;
  cluster.val.clusterDim.x = 2; cluster.val.clusterDim.y = 1; cluster.val.clusterDim.z = 1;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(2); cfg.blockDim = dim3(kWgThreads); cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cfg.attrs = &cluster; cfg.numAttrs = 1;
  int dev = 0;
  e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
  if (s_max_clusters[dev] <= 0) {
    e = cudaOccupancyMaxActiveClusters(&s_max_clusters[dev], kernel, &cfg);
    if (e != cudaSuccess) return e;
    if (s_max_clusters[dev] <= 0) return cudaErrorInvalidConfiguration;
  }
  const int max_ctas = min(num_sms, 2 * s_max_clusters[dev]) & ~1;

  // Every CTA streams at about the same bytes/clk (the kernel is HBM-bound), so the launch ends when the CTA with the
  // most bytes ends: start with one split per job and hand each further split (its halves' CTAs) to the job whose CTAs
  // currently carry the most (chunks per tile x tiles per CTA).
  int splits[16], halves[16], used = 0;
  for (int j = 0; j < n; ++j) {
    splits[j] = 1;
    halves[j] = job_halves(jobs[j]);
    used += halves[j];
  }
  const int tiles = p.n_tiles > 0 ? p.n_tiles : 1;
  for (;;) {
    int best = -1;
    long long best_load = -1;
    for (int j = 0; j < n; ++j) {
      const int sp = splits[j];
      if (sp >= tiles || used + halves[j] > max_ctas) continue;   // a CTA needs at least one tile
      const long long load = static_cast<long long>(kJobCost[jobs[j]]) * ((tiles + sp - 1) / sp);
      if (load > best_load) { best_load = load; best = j; }
    }
    if (best < 0) break;
    ++splits[best];
    used += halves[best];
  }
  // CTA order: the two-half jobs first, so that the halves of every split are the two CTAs of one cluster; then the
  // one-CTA jobs (head, bender; all jobs of the compact launch), two splits to a cluster without multicast, and one
  // idle CTA when their count is odd.  The scratch partials follow the same order (the reduce kernels look jobs up).
  p.n_jobs = 0;
  for (int h = 2; h >= 1; --h)
    for (int j = 0; j < n; ++j)
      if (halves[j] == h) { p.job_ids[p.n_jobs] = jobs[j]; p.splits[p.n_jobs] = splits[j]; p.halves[p.n_jobs] = h; ++p.n_jobs; }
  if (p.n_tiles > 0) {
    cfg.gridDim = dim3((used + 1) & ~1);
    e = cudaLaunchKernelEx(&cfg, kernel, p, args...);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}
}  // namespace

cudaError_t launch_wgrad(WgradParams p, bool has_bender, int num_sms, const WgradDst& dst, int out_ch, cudaStream_t st,
                         const float* tc_dw_lat) {
  int first = 0, last = has_bender ? 12 : 10;
  if (p.compact) { first = 10; last = 12; p.stash_tile_bytes = kTanTileBytes; p.gstash_tile_bytes = kAdjTileBytes; }
  else { p.stash_tile_bytes = kStashTileBytes; p.gstash_tile_bytes = kGradTileBytes; }

  int jobs[12], n_jobs = 0;
  for (int j = first; j < last; ++j) jobs[n_jobs++] = j;
  static int s_max_clusters[64];   // per device
  cudaError_t e = launch_jobs(wgrad_kernel, s_max_clusters, p, jobs, n_jobs, num_sms, st);
  if (e != cudaSuccess) return e;
  const int n = dst.nerf_n + dst.bend_n;
  if (n > 0 && tc_dw_lat) wgrad_reduce_tc_kernel<<<(n + 255) / 256, 256, 0, st>>>(p, dst, out_ch, tc_dw_lat);
  else if (n > 0) wgrad_reduce_kernel<<<(n + 255) / 256, 256, 0, st>>>(p, dst, out_ch);
  return cudaGetLastError();
}

cudaError_t launch_wgrad_views(WgradParams p, const WgradViewParams& v, int num_sms, const WgradDst& dst, cudaStream_t st) {
  // the trunk's jobs 0-9, then 12 feature, 13 views (feature columns), 14 rgb, 15 views (directions)
  int jobs[14];
  for (int j = 0; j < 14; ++j) jobs[j] = j < 10 ? j : kJobFeature + (j - 10);
  p.stash_tile_bytes = kStashTileBytes; p.gstash_tile_bytes = kGradTileBytes;
  static int s_max_clusters[64];   // per device
  cudaError_t e = launch_jobs(wgrad_views_kernel, s_max_clusters, p, jobs, 14, num_sms, st, v);
  if (e != cudaSuccess) return e;
  if (dst.nerf_n > 0) wgrad_views_reduce_kernel<<<(dst.nerf_n + 255) / 256, 256, 0, st>>>(p, dst);
  return cudaGetLastError();
}

}  // namespace nrn
