// Bender steps on tensor cores at fp32 accuracy with the weight images resident in shared memory: the machinery of the
// divergence kernels (div.cu) and the inverse bender (deform.cu).
//
// Every operand x is carried as x_hi = fp16(x) plus a residual x_lo = fp16((x - x_hi) * kBendLoScale), weights included
// (ops.pack_bender writes the residual images), and a step is
//   acc = (A_lo . W_hi + A_hi . W_lo) / kBendLoScale + A_hi . W_hi       (fp32 accumulators; A_lo . W_lo is below fp32)
//
// CTA: four consumer warpgroups, persistent over tiles; warpgroups 2p and 2p + 1 work on one tile (rows 0-63 / 64-127), so
// two tiles are in flight per SM.  The weight images and their residuals are loaded once per CTA by bulk TMA and stay
// resident, so there is no producer warp and no ring.
#pragma once
#include "field_mma.cuh"

namespace nrn {

namespace {

constexpr int kResTilesPerCta = 2;                       // tiles in flight per CTA, two warpgroups each
constexpr int kResWgs = 2 * kResTilesPerCta;
constexpr int kResThreads = 128 * kResWgs;
constexpr int kResStageLd = 12;                          // floats per staged row: B4 columns 0-7, column 64 of B2 at 8
constexpr int kResImgBytes = kStHb1.chunks * kChunkBytes;  // widest image of the bender chains: 96 columns
constexpr float kLoInv = 1.0f / kBendLoScale;

struct ResShared {
  uint64_t w_full;
  int abort_flag;
};

// shared memory: [per tile in flight: A image hi | A image lo] [weights hi | weights lo] [per-row staging] [barrier]
constexpr size_t res_smem_bytes(int wbytes) {
  return 2 * kResTilesPerCta * kResImgBytes + 2 * wbytes + kResWgs * kWgRows * kResStageLd * sizeof(float) + sizeof(ResShared);
}

struct ResSmem {
  uint8_t* img_hi;   // this warpgroup's tile: fp16 parts
  uint8_t* img_lo;   //                        scaled residuals
  uint8_t* w_hi;
  uint8_t* w_lo;
  float* stage;      // this warpgroup's 64 rows
  ResShared* sh;
};
__device__ __forceinline__ ResSmem res_smem(uint8_t* smem, int wbytes, int wg) {
  ResSmem s;
  s.img_hi = smem + (wg >> 1) * 2 * kResImgBytes;
  s.img_lo = s.img_hi + kResImgBytes;
  s.w_hi = smem + 2 * kResTilesPerCta * kResImgBytes;
  s.w_lo = s.w_hi + wbytes;
  float* stage_all = reinterpret_cast<float*>(s.w_lo + wbytes);
  s.stage = stage_all + wg * kWgRows * kResStageLd;
  s.sh = reinterpret_cast<ResShared*>(stage_all + kResWgs * kWgRows * kResStageLd);
  return s;
}

// one thread starts the bulk copies of the weight images and their residuals; every consumer waits on sh->w_full
// (phase 0) before its first MMA
__device__ __forceinline__ void load_resident_weights(const ResSmem& s, const uint8_t* hi, const uint8_t* lo, uint32_t bytes) {
  if (threadIdx.x == 0) {
    mbar_init(&s.sh->w_full, 1);
    s.sh->abort_flag = 0;
    fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(&s.sh->w_full, 2 * bytes);
    for (uint32_t off = 0; off < bytes; off += 16384u) {
      tma_bulk_g2s(s.w_hi + off, hi + off, min(bytes - off, 16384u), &s.sh->w_full);
      tma_bulk_g2s(s.w_lo + off, lo + off, min(bytes - off, 16384u), &s.sh->w_full);
    }
  }
}

// acc[64 x N] = (A_lo . W_hi + A_hi . W_lo) / kBendLoScale + A_hi . W_hi over the k16 steps of 16 columns of bender step S
// (fwd:: or dgrad::), all operands in shared memory: A = this warpgroup's rows of chunk-major images of kTileM rows (fenced
// for the async proxy, warpgroup synced), W = the step's resident N-row weight images.  A_LO = false: the A residual is
// zero (the probe input, whose hi / lo split lives in its columns).  The small terms are summed first, scaled exactly,
// then the main products added.
template <auto S, bool A_LO>
__device__ __forceinline__ void wg_mma_split(Acc<S>& acc, uint32_t a_hi, uint32_t a_lo, const ResSmem& s) {
  constexpr int N = step(S).N;
  constexpr uint32_t w0 = w_off(S), k16 = step(S).k16;
  const uint64_t ahi = gmma_desc(a_hi, kChunkBytes, 128), alo = gmma_desc(a_lo, kChunkBytes, 128);
  const uint64_t whi = gmma_desc(smem_u32(s.w_hi) + w0, N * 16, 128), wlo = gmma_desc(smem_u32(s.w_lo) + w0, N * 16, 128);
#pragma unroll
  for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
  acc_fence(acc);
  wgmma_fence();
#pragma unroll 1
  for (uint32_t k = 0; k < k16; ++k) {
    if (A_LO) wgmma<N, 0, 0>(acc, gmma_desc_advance(alo, k * 2 * kChunkBytes), gmma_desc_advance(whi, k * 2 * N * 16), 1u);
    wgmma<N, 0, 0>(acc, gmma_desc_advance(ahi, k * 2 * kChunkBytes), gmma_desc_advance(wlo, k * 2 * N * 16), 1u);
  }
  wgmma_commit();
  wgmma_wait<0>();
  acc_fence(acc);
#pragma unroll
  for (int i = 0; i < N / 2; ++i) acc[i] *= kLoInv;
  acc_fence(acc);
  wgmma_fence();
#pragma unroll 1
  for (uint32_t k = 0; k < k16; ++k)
    wgmma<N, 0, 0>(acc, gmma_desc_advance(ahi, k * 2 * kChunkBytes), gmma_desc_advance(whi, k * 2 * N * 16), 1u);
  wgmma_commit();
  wgmma_wait<0>();
  acc_fence(acc);
}

// fp32 pair -> {fp16 part, scaled fp16 residual}, each packed as fp16x2 (saturating)
__device__ __forceinline__ uint2 split_h2(float a, float b) {
  const uint32_t hi = pack_h2_sat(a, b);
  const float2 h = __half22float2(*reinterpret_cast<const __half2*>(&hi));
  return make_uint2(hi, pack_h2_sat((a - h.x) * kBendLoScale, (b - h.y) * kBendLoScale));
}

// Accumulator columns [0, NCOLS) times the primal ReLU mask bits -> this warpgroup's rows (half `h` of the tile) of the
// next A operand, as fp16 parts (img_hi) and residuals (img_lo)
template <int NCOLS, int NR>
__device__ __forceinline__ void epi_mask_split(const float (&acc)[NR], const ReluMask<NCOLS>& m, const ResSmem& s, int h) {
  const int r0 = h * kWgRows + acc_r0(), q = acc_q();
#pragma unroll
  for (int j = 0; j < NCOLS / 8; ++j) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const uint2 v = split_h2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]);
      const int off = j * kChunkBytes + (r0 + 8 * i) * 16 + 4 * q;
      *reinterpret_cast<uint32_t*>(s.img_hi + off) = m.apply(i, j, v.x);
      *reinterpret_cast<uint32_t*>(s.img_lo + off) = m.apply(i, j, v.y);
    }
  }
}

}  // namespace

}  // namespace nrn
