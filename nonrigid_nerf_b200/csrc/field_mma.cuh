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

constexpr int kWgRows = kTileM / 2;                 // rows of a tile owned by one consumer warpgroup

// Weight ring of S stages of kRingStageBytes (a per-kernel depth: what the kernel's activation images leave of shared
// memory).  Barriers; one thread initialises them before the CTA's first barrier.
template <int S>
struct RingShared {
  uint64_t w_full[S];
  uint64_t w_empty[S];
  int abort_flag;
  __device__ __forceinline__ void init() {
    for (int i = 0; i < S; ++i) {
      mbar_init(&w_full[i], 1);
      mbar_init(&w_empty[i], 8);
    }
    abort_flag = 0;
    fence_mbar_init();
  }
};

template <int S>
struct Ring {
  uint8_t* buf;      // S x kRingStageBytes
  uint64_t* full;    // TMA bytes landed (count 1 + tx)
  uint64_t* empty;   // slab consumed: one arrival per consumer warp (count 8)
  uint32_t stage = 0, phase = 0;
  __device__ __forceinline__ void next() {
    if (++stage == S) { stage = 0; phase ^= 1u; }
  }
};

// producer (one thread): one weight slab global -> ring
template <int S>
__device__ __forceinline__ void ring_put(Ring<S>& r, const uint8_t* src, uint32_t bytes, const Waiter& W) {
  W.wait(&r.empty[r.stage], r.phase ^ 1u, 101);
  uint8_t* dst = r.buf + r.stage * kRingStageBytes;
  mbar_arrive_expect_tx(&r.full[r.stage], bytes);
  for (uint32_t off = 0; off < bytes; off += 16384u) tma_bulk_g2s(dst + off, src + off, min(bytes - off, 16384u), &r.full[r.stage]);
  r.next();
}

// Producer thread: for every tile of this CTA, the weight images of steps [first, last) through the ring (shapes from
// step_at(step)), those of steps before `split` from `w_lo`, the others from `w_hi`.
template <typename StepAt, int S>
__device__ __forceinline__ void produce(const uint8_t* w_lo, const uint8_t* w_hi, int n_tiles, int first, int last, int split,
                                        StepAt step_at, Ring<S>& ring, const Waiter& W) {
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    uint32_t glo = 0, ghi = 0;
#pragma unroll 1
    for (int step = first; step < last; ++step) {
      const Step s = step_at(step);
      const uint8_t* src = step < split ? w_lo + glo : w_hi + ghi;
      for (uint32_t j = 0; j < s.nslabs; ++j) ring_put(ring, src + j * s.slab_bytes, s.slab_bytes, W);
      if (step < split) glo += s.nslabs * s.slab_bytes; else ghi += s.nslabs * s.slab_bytes;
    }
  }
}

// consumer warpgroup: acc[64 x N] = A . W^T accumulated over `nslabs` weight slabs of the ring (slab j: N rows x 16 k16
// column chunks of W, K-major).  a_addr(j): shared address of this warpgroup's first row of slab j's A operand, a
// K-major image with kTileM rows.  The A operand must have been fenced for the async proxy and the warpgroup synced.
template <int N, typename AAddr, int S>
__device__ __forceinline__ void wg_gemm(float (&acc)[N / 2], Ring<S>& r, uint32_t nslabs, uint32_t k16, AAddr a_addr,
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

// wg_gemm with the A operand in registers: slab j (K16 MMAs) takes the A fragments K16 j .. K16 j + K16 - 1 of `a`, the
// fragments of this warpgroup's 64 rows x 16 KF columns (sm90_ptx.cuh: wgmma_rs).  lead: one slab of K16 MMAs with A from
// shared memory at a_lead (as in wg_gemm) comes first (the embedding columns of the skip layer); it has LEAD_K16 MMAs.
// ACC: add to the accumulators instead of overwriting them (two weight images into one accumulator).
template <int N, int K16, int LEAD_K16 = K16, bool ACC = false, int KF, int S>
__device__ __forceinline__ void wg_gemm_rs(float (&acc)[N / 2], uint32_t (&a)[KF][4], Ring<S>& r, bool lead, uint32_t a_lead,
                                           const Waiter& W, int code) {
  static_assert(KF % K16 == 0, "whole slabs of A fragments");
  const int lane = threadIdx.x & 31;
  uint32_t prev = 0;
  if constexpr (!ACC) {
#pragma unroll
    for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
  }
  if (lead) {
    W.wait(&r.full[r.stage], r.phase, code);
    const uint64_t adesc = gmma_desc(a_lead, kChunkBytes, 128);
    const uint64_t bdesc = gmma_desc(smem_u32(r.buf + r.stage * kRingStageBytes), N * 16, 128);
    acc_fence(acc);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < LEAD_K16; ++k)
      wgmma<N, 0, 0>(acc, gmma_desc_advance(adesc, k * 2 * kChunkBytes), gmma_desc_advance(bdesc, k * 2 * N * 16), k ? 1u : 0u);
    wgmma_commit();
    prev = r.stage;
    r.next();
  }
#pragma unroll
  for (int j = 0; j < KF / K16; ++j) {
    W.wait(&r.full[r.stage], r.phase, code);
    const uint64_t bdesc = gmma_desc(smem_u32(r.buf + r.stage * kRingStageBytes), N * 16, 128);
    acc_fence(acc);
    frag_fence(a);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < K16; ++k)
      wgmma_rs<N, 0>(acc, a[j * K16 + k], gmma_desc_advance(bdesc, k * 2 * N * 16), (ACC || lead || j || k) ? 1u : 0u);
    wgmma_commit();
    if (lead || j > 0) {   // the previous slab's MMAs have retired: hand its stage back while this slab's run
      wgmma_wait<1>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&r.empty[prev]);
    }
    prev = r.stage;
    r.next();
  }
  wgmma_wait<0>();
  acc_fence(acc);
  frag_fence(a);
  __syncwarp();
  if (lane == 0) mbar_arrive(&r.empty[prev]);
}

// Accumulators and wg_gemm of a step known at compile time (fwd:: or dgrad:: id): N, slabs and k16 from its table entry
template <auto S>
using Acc = float[step(S).N / 2];
template <auto ID, typename AAddr, int S>
__device__ __forceinline__ void wg_gemm_step(Acc<ID>& acc, Ring<S>& r, AAddr a_addr, const Waiter& W, int code) {
  constexpr Step s = step(ID);
  wg_gemm<s.N>(acc, r, s.nslabs, s.k16, a_addr, W, code);
}

// A step's shape as immediates, for run-time step switches (a copied constexpr Step would be read from memory)
template <auto S>
__device__ __forceinline__ Step step_imm() {
  constexpr Step s = step(S);
  return {s.N, s.nslabs, s.slab_bytes, s.k16};
}

// Coordinates of this thread's accumulator elements (sm90_ptx.cuh): rows r0 and r0 + 8 of the warpgroup's 64,
// columns 8 j + 2 q and 8 j + 2 q + 1 of every group j.
__device__ __forceinline__ int acc_r0() { return ((threadIdx.x >> 5) & 3) * 16 + ((threadIdx.x & 31) >> 2); }
__device__ __forceinline__ int acc_q() { return threadIdx.x & 3; }

// ReLU masks (layout in nrn_common.cuh), stored in the order of the accumulator so that the forward epilogue writes and
// the DGRAD epilogue reads only its own words.  A row holds one 32-bit word per (q, h) with h < kH (h = 0 only for images
// of at most 128 columns): bit k is [h > 0] of column 8 (16 h + k) + 2 q and bit 16 + k that of column
// 8 (16 h + k) + 2 q + 1, k = 0..15.  A thread's kH words of row r0 + 8 i are contiguous, so a warp's words of one i
// are 128 kH contiguous bytes.
template <int NCOLS>
struct ReluMask {
  static constexpr int kH = NCOLS > 128 ? 2 : 1;
  uint32_t w[2][kH];
  // this thread's words of row r0 + 8 i in the mask image `img` of tile rows [64 g, 64 g + 64)
  static __device__ __forceinline__ size_t offset(int g, int i) {
    return static_cast<size_t>(g * kWgRows + acc_r0() + 8 * i) * (16 * kH) + acc_q() * (4 * kH);
  }
  __device__ __forceinline__ void clear() {
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int h = 0; h < kH; ++h) w[i][h] = 0u;
  }
  // forward: add column group j of row r0 + 8 i from the packed fp16 pair `h2` the epilogue stores (the same half > 0
  // test DGRAD applied to the stashed fp16 activation, so an fp32 value that rounds to fp16 zero stays masked)
  __device__ __forceinline__ void pack(int i, int j, uint32_t h2) {
    w[i][j >> 4] |= __hgt2_mask(*reinterpret_cast<const __half2*>(&h2), __float2half2_rn(0.f)) & (0x00010001u << (j & 15));
  }
  __device__ __forceinline__ void store(uint8_t* img, int g) const {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      if constexpr (kH == 2) *reinterpret_cast<uint2*>(img + offset(g, i)) = make_uint2(w[i][0], w[i][1]);
      else *reinterpret_cast<uint32_t*>(img + offset(g, i)) = w[i][0];
    }
  }
  __device__ __forceinline__ void load(const uint8_t* __restrict__ img, int g) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      if constexpr (kH == 2) {
        const uint2 v = __ldg(reinterpret_cast<const uint2*>(img + offset(g, i)));
        w[i][0] = v.x; w[i][1] = v.y;
      } else {
        w[i][0] = __ldg(reinterpret_cast<const unsigned int*>(img + offset(g, i)));
      }
    }
  }
  // DGRAD: fp16 pair g2 of column group j, row r0 + 8 i, times the 0/1 mask: the same __hmul2 as with the stashed
  // activation, so -0 for a masked negative gradient and NaN propagation are unchanged
  __device__ __forceinline__ uint32_t apply(int i, int j, uint32_t g2) const {
    const uint32_t one = ((w[i][j >> 4] >> (j & 15)) & 0x00010001u) * 0x3c00u;   // fp16 1.0 where the bit is set
    const __half2 r2 = __hmul2(*reinterpret_cast<const __half2*>(&g2), *reinterpret_cast<const __half2*>(&one));
    return *reinterpret_cast<const uint32_t*>(&r2);
  }
};

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

// A warpgroup's writer of finished images to a tile's stash block by bulk TMA stores of one thread (`leader`), so the
// epilogue threads spend no load/store slots on it (OPTIONAL: a null `tile` stores nothing).  begin(): the previous stores
// have finished READING shared memory, and every warp's wgmma reads of an operand are done, before any image is rewritten.
// ready(): the image `img` is complete and visible to the async proxy (wgmma operand, TMA store); it goes to `im`.
template <bool OPTIONAL>
struct StashWriter {
  uint8_t* tile;
  bool leader;
  int bar, g;
  __device__ __forceinline__ void begin() const {
    if ((!OPTIONAL || tile) && leader) tma_bulk_wait_read<0>();
    wg_bar(bar);
  }
  __device__ __forceinline__ void ready(Image im, const uint8_t* img) const {
    fence_proxy_async_smem();
    wg_bar(bar);
    if ((!OPTIONAL || tile) && leader && im.chunks) store_rows(tile + static_cast<uint32_t>(im.off), img, g, im.chunks);
  }
};

// Launch of a persistent field kernel: one CTA per SM at most, `smem` bytes of dynamic shared memory; `extra`: the kernel's
// arguments after p
template <typename Kernel, typename Params, typename... Extra>
cudaError_t launch_field(Kernel kernel, const Params& p, int num_sms, size_t smem, cudaStream_t stream, const Extra&... extra) {
  if (p.n_tiles <= 0) return cudaSuccess;
  const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  kernel<<<p.n_tiles < num_sms ? p.n_tiles : num_sms, kFwdThreads, smem, stream>>>(p, extra...);
  return cudaGetLastError();
}

}  // namespace

}  // namespace nrn
