// Pieces shared by the fused field kernels (field_fwd.cu, field_bwd.cu).
//
// CTA layout: warps 0-3 and 4-7 are two consumer warpgroups, one thread of warp 8 streams the weight slabs (warps 8-11
// form the producer warpgroup only so that the consumers can take over its registers).  A tile is
// 128 points; warpgroup g owns rows [64 g, 64 g + 64) of every activation image and issues its own
// wgmma (M = 64) over them, so the two warpgroups never wait for each other: they only share the weight
// ring, and the epilogue of one overlaps the tensor-core work of the other.
#pragma once
#include "nrn_common.cuh"
#include "sm90_ptx.cuh"

namespace nrn {

namespace {

constexpr long long kWaitLimitCycles = 1ll << 28;  // ~0.15 s: protocol bug => error flag, not a hang
constexpr int kWgRows = kTileM / 2;                 // rows of a tile owned by one consumer warpgroup

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

struct Ring {
  uint8_t* buf;      // kRingStages x kRingStageBytes
  uint64_t* full;    // TMA bytes landed (count 1 + tx)
  uint64_t* empty;   // slab consumed: one arrival per consumer warp (count 8)
  uint32_t stage = 0, phase = 0;
  __device__ __forceinline__ void next() {
    if (++stage == kRingStages) { stage = 0; phase ^= 1u; }
  }
};

// producer (one thread): one weight slab global -> ring
__device__ __forceinline__ void ring_put(Ring& r, const uint8_t* src, uint32_t bytes, const Waiter& W) {
  W.wait(&r.empty[r.stage], r.phase ^ 1u, 101);
  uint8_t* dst = r.buf + r.stage * kRingStageBytes;
  mbar_arrive_expect_tx(&r.full[r.stage], bytes);
  for (uint32_t off = 0; off < bytes; off += 16384u) tma_bulk_g2s(dst + off, src + off, min(bytes - off, 16384u), &r.full[r.stage]);
  r.next();
}

// consumer warpgroup: acc[64 x N] = A . W^T accumulated over `nslabs` weight slabs of the ring (slab j: N rows x 16 k16
// column chunks of W, K-major).  a_addr(j): shared address of this warpgroup's first row of slab j's A operand, a
// K-major image with kTileM rows.  The A operand must have been fenced for the async proxy and the warpgroup synced.
template <int N, typename AAddr>
__device__ __forceinline__ void wg_gemm(float (&acc)[N / 2], Ring& r, uint32_t nslabs, uint32_t k16, AAddr a_addr,
                                        const Waiter& W, int code) {
  const int lane = threadIdx.x & 31;
  uint32_t prev = 0;
  // the first MMA overwrites the accumulators; defined inputs keep ptxas from spilling and serialising the wgmma chain
#pragma unroll
  for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
#pragma unroll 1
  for (uint32_t j = 0; j < nslabs; ++j) {
    W.wait(&r.full[r.stage], r.phase, code);
    const uint64_t adesc = gmma_desc(a_addr(j), kChunkBytes, 128);
    const uint64_t bdesc = gmma_desc(smem_u32(r.buf + r.stage * kRingStageBytes), N * 16, 128);
    acc_fence(acc);
    wgmma_fence();
#pragma unroll 1
    for (uint32_t k = 0; k < k16; ++k)
      wgmma<N, 0, 0>(acc, gmma_desc_advance(adesc, k * 2 * kChunkBytes), gmma_desc_advance(bdesc, k * 2 * N * 16), (j | k) ? 1u : 0u);
    wgmma_commit();
    if (j > 0) {   // the previous slab's MMAs have retired: hand its stage back while this slab's run
      wgmma_wait<1>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&r.empty[prev]);
    }
    prev = r.stage;
    r.next();
  }
  wgmma_wait<0>();
  acc_fence(acc);
  __syncwarp();
  if (lane == 0) mbar_arrive(&r.empty[prev]);
}

// Coordinates of this thread's accumulator elements (sm90_ptx.cuh): rows r0 and r0 + 8 of the warpgroup's 64,
// columns 8 j + 2 q and 8 j + 2 q + 1 of every group j.
__device__ __forceinline__ int acc_r0() { return ((threadIdx.x >> 5) & 3) * 16 + ((threadIdx.x & 31) >> 2); }
__device__ __forceinline__ int acc_q() { return threadIdx.x & 3; }

// Column groups [J0, J0 + NJ) of the accumulator -> stage[row][8 (j - J0) + col % 8] (row = warpgroup-local, fp32),
// for the per-row work of one thread per row.
template <int J0, int NJ, int NR>
__device__ __forceinline__ void stage_cols(const float (&acc)[NR], float* stage, int ld) {
  const int r0 = acc_r0(), q = acc_q();
#pragma unroll
  for (int j = J0; j < J0 + NJ; ++j) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float* d = stage + (r0 + 8 * i) * ld + 8 * (j - J0) + 2 * q;
      d[0] = acc[4 * j + 2 * i];
      d[1] = acc[4 * j + 2 * i + 1];
    }
  }
}

// Bulk stores of this warpgroup's rows of a finished chunk-major image (one thread; 1 KB per chunk).
__device__ __forceinline__ void store_rows(uint8_t* gdst, const uint8_t* img, int g, uint32_t chunks) {
  for (uint32_t c = 0; c < chunks; ++c)
    tma_bulk_s2g(gdst + c * kChunkBytes + g * kWgRows * 16, img + c * kChunkBytes + g * kWgRows * 16, kWgRows * 16);
  tma_bulk_commit();
}

}  // namespace

}  // namespace nrn
