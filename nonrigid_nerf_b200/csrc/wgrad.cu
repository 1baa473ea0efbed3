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
// of dW and a NeRF layer's 256-row dW is split over two CTAs ("halves") that stream the same activation blocks at
// the same time (adjacent CTAs: the second read of a block is an L2 hit).  A pipeline stage holds ONE whole 128-point
// block, A and B alternating through a 3 x 64 KB ring, fetched with a handful of 16 KB bulk copies.  Every job is
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

constexpr long long kWaitLimitCycles = 1ll << 28;
constexpr int kWgStages = 3;
constexpr int kStageBytes = 32 * kChunkBytes;      // one block of up to 32 chunk images (128 points x 8 features each)
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
__device__ __forceinline__ Job job_desc(int j, int half, int g, int compact) {
  Job jb{};
  if (j <= 9) {
    int a_off, a_cols, b_off, b_cols, bias = 1;
    if (j == 0) { a_off = kGsRaw; a_cols = 16; b_off = kStH + 7 * kHBytes; b_cols = 256; }
    else if (j == 8) { a_off = kGsY + 5 * kHBytes; a_cols = 256; b_off = kStE; b_cols = 64; bias = 0; }
    else if (j == 9) { a_off = kGsY; a_cols = 256; b_off = kStE; b_cols = 64; }
    else { a_off = kGsY + j * kHBytes; a_cols = 256; b_off = kStH + (j - 1) * kHBytes; b_cols = 256; }
    jb.a_off = a_off + half * 16 * kChunkBytes; jb.a_chunks = min(a_cols / 8 - 16 * half, 16);
    jb.b_off = b_off; jb.b_chunks = b_cols / 8;
    jb.bias = bias; jb.bias_off = half * 128;
    const int m0 = half * 128 + g * 64;
    jb.u[0] = {8 * g, 0, m0 * 256, 256, max(min(a_cols - m0, 64), 0)};
    return jb;
  }
  // bender jobs: the images of a job are adjacent in both stashes (nrn_common.cuh); in compact mode the stashes hold
  // only the bender images
  const int ga = compact ? kGsYb4 : 0, sa = compact ? kStBin : 0;
  if (j == 10) {
    // A: Yb4 (2 chunks) Yb3 (8) Yb2 (10)      B: Hb2 (12) Hb3 (8) Hb4 (8)
    jb.a_off = kGsYb4 - ga; jb.a_chunks = 20;
    jb.b_off = kStHb2 - sa; jb.b_chunks = 28;
    if (g == 0) {
      jb.u[0] = {0, 20, 0, 128, 16};                  // dYb4 x Hb4      (N = 64)
      jb.u[1] = {2, 12, 16384, 128, 64};              // dYb3 x Hb3      (N = 64)
    } else {
      jb.u[0] = {10, 0, 2 * 16384, 128, 64};          // dYb2 x Hb2      (N = 96), rows 0-63
      jb.u[1] = {18, 0, 2 * 16384 + 64 * 128, 128, 16};  //               rows 64-79
    }
  } else {
    // A: Yb1 (12) Yb0 (12)                    B: bender input (6) Hb1 (12)
    jb.a_off = kGsYb1 - ga; jb.a_chunks = 24;
    jb.b_off = kStBin - sa; jb.b_chunks = 18;
    if (g == 0) {
      jb.u[0] = {0, 6, 0, 128, 64};                   // dYb1 x Hb1      (N = 96), rows 0-63
      jb.u[1] = {8, 6, 64 * 128, 128, 32};            //                 rows 64-95
    } else {
      jb.u[0] = {12, 0, 16384, 128, 64};              // dYb0 x input    (N = 48), rows 0-63
      jb.u[1] = {20, 0, 16384 + 64 * 128, 128, 32};   //                 rows 64-95
    }
  }
  jb.bias = compact ? 0 : 1;   // the tangent chain of the divergence term has no bias
  return jb;
}

struct Shared {
  uint64_t full[kWgStages];
  uint64_t empty[kWgStages];
  int abort_flag;
};

struct Waiter {
  int* s_abort;
  int* g_err;
  __device__ __forceinline__ bool wait(uint64_t* bar, uint32_t parity, int code) const {
    if (mbar_try_wait(bar, parity)) return true;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
      if (*reinterpret_cast<volatile int*>(s_abort)) return false;
      if (clock64() - t0 > kWaitLimitCycles) {
        atomicExch(s_abort, code);
        atomicCAS(g_err, 0, code);
        return false;
      }
    }
    return true;
  }
};

// One halving step of warp_transpose_reduce on the first N entries (a compile-time N keeps every index static, so v
// stays in registers).
template <int N>
__device__ __forceinline__ void transpose_reduce_step(float (&v)[32], int lane) {
  if constexpr (N > 1) {
    constexpr int off = N / 2;
    const bool upper = (lane & off) != 0;
#pragma unroll
    for (int i = 0; i < off; ++i) {
      const float lo = v[i], hi = v[i + off];
      v[i] = (upper ? hi : lo) + __shfl_xor_sync(0xffffffffu, upper ? lo : hi, off);
    }
    transpose_reduce_step<off>(v, lane);
  }
}

// Sum over the warp's 32 lanes of v[j] for each j; lane L returns the total of column L.
__device__ __forceinline__ float warp_transpose_reduce(float (&v)[32], int lane) {
  transpose_reduce_step<32>(v, lane);
  return v[0];
}

// which (job, split, half) does this CTA own, and which scratch partial is the split's?  job_ids[] / splits[] /
// halves[] come from the host (WgradParams); the halves of one split are adjacent CTAs.
__device__ __forceinline__ bool locate(const WgradParams& p, int cta, int& job, int& split, int& nsplit, int& half, int& part) {
  int base = 0, pbase = 0;
  for (int j = 0; j < p.n_jobs; ++j) {
    const int n = p.splits[j] * p.halves[j];
    if (cta < base + n) {
      job = p.job_ids[j]; split = (cta - base) / p.halves[j]; half = (cta - base) % p.halves[j]; nsplit = p.splits[j];
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
__device__ __forceinline__ void consume(const Job& jb, const Unit& u0, const Unit& u1, uint8_t* smem, Shared* sh, const Waiter& W,
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
    const uint32_t sa = stage;
    W.wait(&sh->full[sa], phase, 201);
    if (++stage == kWgStages) { stage = 0; phase ^= 1u; }
    const uint32_t sb = stage;
    W.wait(&sh->full[sb], phase, 202);
    if (++stage == kWgStages) { stage = 0; phase ^= 1u; }
    const uint32_t a0 = smem_u32(smem + sa * kStageBytes), b0 = smem_u32(smem + sb * kStageBytes);
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
        const uint8_t* src = smem + sa * kStageBytes + c * kChunkBytes + lane * 16;
        float t8[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (c < jb.a_chunks) {        // chunks beyond the block hold stale data
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            const uint4 w = *reinterpret_cast<const uint4*>(src + r * 512);
            const uint32_t wv[4] = {w.x, w.y, w.z, w.w};   // unpacked by value: no address of a local, no stack frame
#pragma unroll
            for (int qq = 0; qq < 4; ++qq) {
              t8[2 * qq] += __half2float(__ushort_as_half(static_cast<unsigned short>(wv[qq] & 0xffffu)));
              t8[2 * qq + 1] += __half2float(__ushort_as_half(static_cast<unsigned short>(wv[qq] >> 16)));
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
      mbar_arrive(&sh->empty[sa]);
      mbar_arrive(&sh->empty[sb]);
    }
  }
  if (!have || n_tiles_local == 0) return;
  if (jb.bias && (warp * 4 + (lane >> 3)) < jb.a_chunks) part[65536 + jb.bias_off + warp * 32 + lane] = bias_acc;
  if constexpr (N0 > 0) unit_drain(acc0, u0, part);
  if constexpr (N1 > 0) unit_drain(acc1, u1, part);
}

}  // namespace

__global__ void __launch_bounds__(kWgThreads, 1) wgrad_kernel(const WgradParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  Shared* sh = reinterpret_cast<Shared*>(smem + kWgStages * kStageBytes);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  int job_id = 0, split = 0, nsplit = 1, half = 0, part_idx = 0;
  const bool have = locate(p, blockIdx.x, job_id, split, nsplit, half, part_idx);
  const Job jb = job_desc(job_id, half, (warp >> 2) & 1, p.compact);
  // contiguous tile range of this split
  const int per = (p.n_tiles + nsplit - 1) / nsplit;
  const int t_begin = have ? min(split * per, p.n_tiles) : 0;
  const int t_end = have ? min(t_begin + per, p.n_tiles) : 0;
  const int n_local = t_end - t_begin;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kWgStages; ++i) {
      mbar_init(&sh->full[i], 1);
      mbar_init(&sh->empty[i], 8);   // one arrival per consumer warp
    }
    sh->abort_flag = 0;
    fence_mbar_init();
  }
  __syncthreads();
  const Waiter W{&sh->abort_flag, p.err};

  if (warp >= 8) {
    setmaxnreg_dec<kProducerRegs>();
    // ===================== producer: whole image blocks, 16 KB bulk copies =====================
    if (warp == 8 && lane == 0) {
      uint32_t stage = 0, phase = 0;
      for (int it = 0; it < 2 * n_local; ++it) {   // per tile: the A block, then the B block
        const long long tile = t_begin + (it >> 1);
        const bool is_b = (it & 1) != 0;
        const uint8_t* src = is_b ? p.stash + tile * p.stash_tile_bytes + jb.b_off : p.gstash + tile * p.gstash_tile_bytes + jb.a_off;
        const uint32_t bytes = static_cast<uint32_t>(is_b ? jb.b_chunks : jb.a_chunks) * kChunkBytes;
        W.wait(&sh->empty[stage], phase ^ 1u, 101);
        mbar_arrive_expect_tx(&sh->full[stage], bytes);
        uint8_t* dst = smem + stage * kStageBytes;
        for (uint32_t o = 0; o < bytes; o += 16384u) tma_bulk_g2s(dst + o, src + o, bytes - o < 16384u ? bytes - o : 16384u, &sh->full[stage]);
        if (++stage == kWgStages) { stage = 0; phase ^= 1u; }
      }
    }
    return;
  }

  setmaxnreg_inc<kConsumerRegs>();
  const int g = warp >> 2;
  float* part = p.scratch + static_cast<size_t>(part_idx) * kWgScratchFloats;
  const Unit& u0 = jb.u[0];
  const Unit& u1 = jb.u[1];
  if (job_id <= 9) {
    const bool mine = u0.rows > 0;
    if (job_id == 8 || job_id == 9) {
      if (mine) consume<64, 0>(jb, u0, u1, smem, sh, W, n_local, part, have);
      else consume<0, 0>(jb, u0, u1, smem, sh, W, n_local, part, have);
    } else {
      if (mine) consume<256, 0>(jb, u0, u1, smem, sh, W, n_local, part, have);
      else consume<0, 0>(jb, u0, u1, smem, sh, W, n_local, part, have);
    }
  } else if (job_id == 10) {
    if (g == 0) consume<64, 64>(jb, u0, u1, smem, sh, W, n_local, part, have);
    else consume<96, 96>(jb, u0, u1, smem, sh, W, n_local, part, have);
  } else {
    if (g == 0) consume<96, 96>(jb, u0, u1, smem, sh, W, n_local, part, have);
    else consume<48, 48>(jb, u0, u1, smem, sh, W, n_local, part, have);
  }
}

// ------------------------------------------------------------------------------------------------
// Deterministic reduction of the split partials into the reference's parameter layout.
// One thread per destination element of the flat gradient buffers:
//   NeRF   : W0[256x63] b0 W1 b1 ... W7 b7 Wout[out_ch x 256] bout
//   bender : net_w0[64x35] net_b0 net_w1 net_b1 net_w2 net_b2 net_w3 net_b3 net_w4[3x64]
//            rig_w0[32x3] rig_b0 rig_w1[32x32] rig_b1 rig_w2[1x32] rig_b2
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

__device__ __forceinline__ Src nerf_src(int idx, int out_ch, bool& ok) {
  ok = true;
  const int sz0 = 256 * 63 + 256, szl = 256 * 256 + 256, sz5 = 256 * 319 + 256;
  if (idx < sz0) {
    if (idx < 256 * 63) return nerf_w(9, idx / 63, idx % 63);
    return nerf_b(9, idx - 256 * 63);
  }
  idx -= sz0;
  for (int l = 1; l < 8; ++l) {
    const int sz = l == 5 ? sz5 : szl;
    if (idx < sz) {
      if (l == 5) {
        if (idx < 256 * 319) {
          const int m = idx / 319, k = idx % 319;
          return k < 63 ? nerf_w(8, m, k) : nerf_w(5, m, k - 63);
        }
        return nerf_b(5, idx - 256 * 319);
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

// A-chunk layout of the bender jobs (bias index = column inside the concatenated A images):
//   job 10: Yb4 cols 0-15 | Yb3 cols 16-79 | Yb2 cols 80-159      job 11: Yb1 cols 0-95 | Yb0 cols 96-191
__device__ __forceinline__ Src bender_src(int idx, bool& ok) {
  ok = true;
  if (idx < 64 * 35) {  // net_w0: xyz columns collect the hi and lo operand columns
    const int m = idx / 35, k = idx % 35;
    return k < 3 ? bend_w(11, 1, m, k, k + 3) : bend_w(11, 1, m, 6 + (k - 3));
  }
  idx -= 64 * 35;
  if (idx < 64) return {11, 96 + idx, -1, 1};                                    // net_b0
  idx -= 64;
  if (idx < 4096) return bend_w(11, 0, idx >> 6, idx & 63);                      // net_w1
  idx -= 4096;
  if (idx < 64) return {11, idx, -1, 1};                                         // net_b1
  idx -= 64;
  if (idx < 4096) return bend_w(10, 2, idx >> 6, idx & 63);                      // net_w2
  idx -= 4096;
  if (idx < 64) return {10, 80 + idx, -1, 1};                                    // net_b2
  idx -= 64;
  if (idx < 4096) return bend_w(10, 1, idx >> 6, idx & 63);                      // net_w3
  idx -= 4096;
  if (idx < 64) return {10, 16 + idx, -1, 1};                                    // net_b3
  idx -= 64;
  if (idx < 192) return bend_w(10, 0, idx >> 6, idx & 63);                       // net_w4
  idx -= 192;
  if (idx < 96) return bend_w(11, 1, 64 + idx / 3, idx % 3, idx % 3 + 3);        // rig_w0
  idx -= 96;
  if (idx < 32) return {11, 96 + 64 + idx, -1, 1};                               // rig_b0
  idx -= 32;
  if (idx < 1024) return bend_w(11, 0, 64 + (idx >> 5), 64 + (idx & 31));        // rig_w1
  idx -= 1024;
  if (idx < 32) return {11, 64 + idx, -1, 1};                                    // rig_b1
  idx -= 32;
  if (idx < 32) return bend_w(10, 2, 64, 64 + idx);                              // rig_w2
  idx -= 32;
  return {10, 80 + 64, -1, 1};                                                   // rig_b2
}

}  // namespace

__global__ void wgrad_reduce_kernel(const WgradParams p, const WgradDst dst, int out_ch) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int nerf_n = dst.nerf_n, bend_n = dst.bend_n;
  if (idx >= nerf_n + bend_n) return;
  bool ok;
  const Src s = idx < nerf_n ? nerf_src(idx, out_ch, ok) : bender_src(idx - nerf_n, ok);
  float scale = 1.0f;
  {
    const float amax = p.amax ? __ldg(p.amax) : 0.f;
    if (amax > 0.f && amax < 3.0e38f) {
      int e;
      frexpf(amax, &e);
      scale = ldexpf(1.0f, min(max(10 - e, -60), 60));
    }
  }
  float sum = 0.f;
  if (ok && !(s.bias && p.compact)) {
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
  }
  const float v = sum / scale;
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

// ------------------------------------------------------------------------------------------------
cudaError_t launch_wgrad(WgradParams p, bool has_bender, int num_sms, const WgradDst& dst, int out_ch, cudaStream_t st) {
  // relative cost of one tile of every job's CTAs = 2 KB chunks a CTA moves (a NeRF layer's half: 16 gradient chunks +
  // the activation block); the head job (a 4 KB gradient block alternating with a 64 KB activation block keeps fewer
  // bytes in flight) and the three-MMA bender job stream a little slower per byte, hence their surcharge
  static const int kJobChunks[12] = {46, 48, 48, 48, 48, 48, 48, 48, 16 + 8 + 8, 16 + 8 + 8, 54, 24 + 18};
  int first = 0, last = has_bender ? 12 : 10;
  if (p.compact) { first = 10; last = 12; p.stash_tile_bytes = kTanTileBytes; p.gstash_tile_bytes = kAdjTileBytes; }
  else { p.stash_tile_bytes = kStashTileBytes; p.gstash_tile_bytes = kGradTileBytes; }
  p.n_jobs = last - first;
  // Every CTA streams at about the same bytes/clk (the kernel is HBM-bound), so the launch ends when the CTA with the
  // most bytes ends: start with one split per job and hand each further split (its halves' CTAs) to the job whose CTAs
  // currently carry the most (chunks per tile x tiles per CTA).
  int used = 0;
  for (int j = first; j < last; ++j) {
    p.job_ids[j - first] = j; p.splits[j - first] = 1;
    p.halves[j - first] = (j >= 1 && j <= 9) ? 2 : 1;   // the head's 16-row dW and the bender jobs fit one CTA
    used += p.halves[j - first];
  }
  const int tiles = p.n_tiles > 0 ? p.n_tiles : 1;
  for (;;) {
    int best = -1;
    long long best_load = -1;
    for (int j = first; j < last; ++j) {
      const int sp = p.splits[j - first];
      if (sp >= tiles || used + p.halves[j - first] > num_sms) continue;   // a CTA needs at least one tile
      const long long load = static_cast<long long>(kJobChunks[j]) * ((tiles + sp - 1) / sp);
      if (load > best_load) { best_load = load; best = j; }
    }
    if (best < 0) break;
    ++p.splits[best - first];
    used += p.halves[best - first];
  }
  if (p.n_tiles > 0) {
    const size_t smem = kWgStages * kStageBytes + sizeof(Shared) + 64;
    cudaError_t e = cudaFuncSetAttribute(wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    wgrad_kernel<<<used, kWgThreads, smem, st>>>(p);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  const int n = dst.nerf_n + dst.bend_n;
  if (n > 0) wgrad_reduce_kernel<<<(n + 255) / 256, 256, 0, st>>>(p, dst, out_ch);
  return cudaGetLastError();
}

}  // namespace nrn
