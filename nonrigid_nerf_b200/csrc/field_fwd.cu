// Fused point-wise field evaluation, forward:  (ray, z) -> bent point -> PE -> 8x256 MLP -> raw.
//
// Replaces, for one coarse or fine pass, the reference call chain
//   run_network (train.py:57-105) -> batchify (train.py:27-54) -> NeRF.forward
//   (run_nerf_helpers.py:240-314) -> ray_bending.forward (run_nerf_helpers.py:507-584)
//   -> Embedder.embed (run_nerf_helpers.py:149-150)
// with ONE persistent sm_90a kernel.  No [P,95] / [P,256] tensor ever touches HBM.
//
// Work decomposition (field_mma.cuh)
//   tile   = 128 consecutive sample points; CTA = 1 per SM, persistent over tiles
//   warps  : 0-3 / 4-7 consumer warpgroups (rows 0-63 / 64-127 of the tile), 8 weight producer (bulk TMA ring)
//   a "step" = one dense layer:  D[64 x N] (registers, fp32) = A[64 x K] (smem, fp16) . W[N x K]^T (smem ring,
//            fp16) with wgmma; the same warpgroup then applies bias/ReLU/(bend + positional encoding) and writes
//            the next A operand in place.
//   steps  : B0..B4 (ray bender, offset + rigidity MLPs fused block-diagonally), L0..L7, head
//
// Shared memory (per CTA): H 64 KB + E 16 KB activations, 4 x 32 KB weight ring, per-row staging, barriers.
#include "field_mma.cuh"

namespace nrn {

namespace {

constexpr int kFwdStageLd = 12;   // floats per staged row (8 used)

struct Shared {
  uint64_t w_full[kRingStages];
  uint64_t w_empty[kRingStages];
  int abort_flag;
};

struct StepShape {
  uint32_t N, nslabs, slab_bytes, k16;
};

// step index: 0-4 bender B0..B4, 5-12 NeRF L0..L7, 13 head
__device__ __forceinline__ StepShape step_shape(int step) {
  switch (step) {
    case 0: return {96u, 1u, (uint32_t)kBendB0Bytes, 3u};
    case 1: return {96u, 1u, (uint32_t)kBendB1Bytes, 6u};
    case 2: return {80u, 1u, (uint32_t)kBendB2Bytes, 6u};
    case 3: return {64u, 1u, (uint32_t)kBendB3Bytes, 4u};
    case 4: return {16u, 1u, (uint32_t)kBendB4Bytes, 4u};
    case 5: return {256u, 1u, 32768u, 4u};
    case 10: return {256u, 5u, 32768u, 4u};
    case 13: return {16u, 1u, (uint32_t)kNerfHeadBytes, 16u};
    default: return {256u, 4u, 32768u, 4u};
  }
}
// byte offset (inside the activation region: H at 0, E at kHBytes) of the A operand of slab j
__device__ __forceinline__ uint32_t a_operand_offset(int step, uint32_t j) {
  if (step == 0 || step == 5) return kHBytes;                       // bender input / embedding live in E
  if (step == 10) return j == 0 ? kHBytes : (j - 1) * 8 * kChunkBytes;  // skip: [embedding | h]
  if (step < 5 || step == 13) return 0;
  return j * 8 * kChunkBytes;
}

// Accumulator columns [0, NCOLS) + bias, ReLU, fp16 -> this warpgroup's rows of the chunk-major image `img`.  MASK
// (training kernel): also the ReLU mask bits of those elements -> this thread's words of the tile's mask image at
// byte `mask_off` of `mask_tile`.
template <int NCOLS, bool MASK, int NR>
__device__ __forceinline__ void epi_bias_relu_store(const float (&acc)[NR], const float* __restrict__ bias, uint8_t* img, int g,
                                                    uint8_t* mask_tile, int mask_off) {
  const int r0 = g * kWgRows + acc_r0(), q = acc_q();
  ReluMask<NCOLS> m;
  if constexpr (MASK) m.clear();
#pragma unroll
  for (int j = 0; j < NCOLS / 8; ++j) {
    const float2 b = __ldg(reinterpret_cast<const float2*>(bias + 8 * j + 2 * q));
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      // one cvt.rn.relu.satfinite.f16x2 per two outputs: ReLU, clamp to fp16 range and pack in a single instruction
      const uint32_t h2 = pack_h2_relu_sat(acc[4 * j + 2 * i] + b.x, acc[4 * j + 2 * i + 1] + b.y);
      *reinterpret_cast<uint32_t*>(img + j * kChunkBytes + (r0 + 8 * i) * 16 + 4 * q) = h2;
      if constexpr (MASK) m.pack(i, j, h2);
    }
  }
  if constexpr (MASK) m.store(mask_tile + mask_off, g);
}

// Positional encoding of one point (Embedder.embed, run_nerf_helpers.py:149-150 with the settings of
// get_embedder :157-164: raw xyz first, then per octave sin(2^k xyz), cos(2^k xyz); k = 0..9).
// Written as fp16 chunks 0..7 of the row (63 features + one zero pad column).
// sin/cos: the argument 2^k * x is reduced EXACTLY to [-0.5, 0.5) turns (x / 2pi carried as a
// two-float value), then evaluated with MUFU (abs err ~4e-7), well below fp16 resolution.
__device__ __forceinline__ void write_pe(const float (&x)[3], uint8_t* dst_row) {
  float f[64];
  f[0] = x[0]; f[1] = x[1]; f[2] = x[2];
  const float kInv2PiHi = 0.15915494f;      // fl(1/2pi)
  const float kInv2PiLo = 6.4206199e-09f;   // 1/2pi - fl(1/2pi)
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const float thi = x[d] * kInv2PiHi;
    const float tlo = fmaf(x[d], kInv2PiLo, fmaf(x[d], kInv2PiHi, -thi));
#pragma unroll
    for (int k = 0; k < 10; ++k) {
      const float sc = static_cast<float>(1 << k);
      const float a = thi * sc;
      const float ph = (a - rintf(a)) + tlo * sc;
      const float ang = ph * 6.2831853071795865f;
      f[3 + 6 * k + d] = __sinf(ang);
      f[3 + 6 * k + 3 + d] = __cosf(ang);
    }
  }
  f[63] = 1.f;  // pad column: its weight column is zero (forward unaffected); WGRAD reads it as the bias input
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    uint4 pk;
    pk.x = pack_h2(f[c * 8 + 0], f[c * 8 + 1]);
    pk.y = pack_h2(f[c * 8 + 2], f[c * 8 + 3]);
    pk.z = pack_h2(f[c * 8 + 4], f[c * 8 + 5]);
    pk.w = pack_h2(f[c * 8 + 6], f[c * 8 + 7]);
    *reinterpret_cast<uint4*>(dst_row + c * kChunkBytes) = pk;
  }
}

}  // namespace

// TRAIN: p.stash and p.relu_mask are given (the inference kernel carries none of the mask code)
template <bool HAS_BENDER, bool TRAIN>
__global__ void __launch_bounds__(kFwdThreads, 1) field_fwd_kernel(const FieldFwdParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* act = smem;                                  // H | E, 128 rows
  uint8_t* ring_buf = smem + kSlotBytes;                // kRingStages x 32 KB
  float* stage_all = reinterpret_cast<float*>(ring_buf + kRingStages * kRingStageBytes);   // 2 x 64 rows x kFwdStageLd
  Shared* sh = reinterpret_cast<Shared*>(stage_all + 2 * kWgRows * kFwdStageLd);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  constexpr int kFirstStep = HAS_BENDER ? 0 : 5;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kRingStages; ++i) {
      mbar_init(&sh->w_full[i], 1);
      mbar_init(&sh->w_empty[i], 8);
    }
    sh->abort_flag = 0;
    fence_mbar_init();
  }
  __syncthreads();
  const Waiter W{&sh->abort_flag, p.err};
  Ring ring{ring_buf, sh->w_full, sh->w_empty};

  if (warp >= 8) {
    setmaxnreg_dec<kProducerRegs>();
    // ===================== weight producer: global -> smem ring (bulk TMA) =====================
    if (warp == 8 && lane == 0) {
      for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
        uint32_t gb = 0, gn = 0;
#pragma unroll 1
        for (int step = kFirstStep; step < 14; ++step) {
          const StepShape s = step_shape(step);
          const uint8_t* src = step < 5 ? p.bend_w + gb : p.nerf_w + gn;
          for (uint32_t j = 0; j < s.nslabs; ++j) ring_put(ring, src + j * s.slab_bytes, s.slab_bytes, W);
          if (step < 5) gb += s.nslabs * s.slab_bytes; else gn += s.nslabs * s.slab_bytes;
        }
      }
    }
    return;
  }

  // ===================== consumer warpgroups =====================
  setmaxnreg_inc<kConsumerRegs>();
  const int g = warp >> 2;
  const int tw = threadIdx.x & 127;
  const bool row_thread = tw < kWgRows;   // threads 0-63 of the warpgroup each own one row for the per-point work
  const int bar = 1 + g;
  const bool wg_leader = tw == 0;
  uint8_t* Hs = act;
  uint8_t* Es = act + kHBytes;
  uint8_t* e_row = Es + (g * kWgRows + tw) * 16;
  const uint32_t a_h = smem_u32(Hs) + g * kWgRows * 16;
  const uint32_t a_e = smem_u32(Es) + g * kWgRows * 16;
  float* stg = stage_all + g * kWgRows * kFwdStageLd;
  float* my_stg = stg + tw * kFwdStageLd;

  for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
    const long long pt = static_cast<long long>(tile) * kTileM + g * kWgRows + tw;
    const bool valid = row_thread && pt < p.P;
    // Training stash: every finished activation image is written to this tile's stash block with bulk TMA stores
    // issued by one thread of the warpgroup (its 64 rows of each chunk); the epilogue threads spend no load/store
    // slots on it.  stash_begin(): the previous stores must have finished READING shared memory before any image is
    // overwritten; it also orders every warp's wgmma reads of an operand before any warp rewrites it in place.
    // ready(): the image is complete and visible to the async proxy (wgmma operand, TMA store).
    uint8_t* st = p.stash ? p.stash + static_cast<long long>(tile) * kStashTileBytes : nullptr;
    // ReLU masks for DGRAD (training): every row of the tile is written, those past P of a ragged last tile included
    uint8_t* mk = TRAIN ? p.relu_mask + static_cast<long long>(tile) * kMaskTileBytes : nullptr;
    auto stash_begin = [&]() {
      if (st && wg_leader) tma_bulk_wait_read<0>();
      wg_bar(bar);
    };
    auto ready = [&](uint32_t stash_off, const uint8_t* img, uint32_t chunks) {
      fence_proxy_async_smem();
      wg_bar(bar);
      if (st && wg_leader && chunks) store_rows(st + stash_off, img, g, chunks);
    };
    float x[3] = {0.f, 0.f, 0.f};
    long long ray = 0;
    if (valid) {
      ray = pt / p.S;
      if (p.pts) {
        const float* q = p.pts + pt * p.pts_stride;  // point mode: NeRF.forward(x) reads x[:, :3]
        x[0] = __ldg(q + 0); x[1] = __ldg(q + 1); x[2] = __ldg(q + 2);
      } else {
        const float z = __ldg(p.z_vals + pt);
        const float* r = p.rays + ray * 8;
        // pts = rays_o + rays_d * z  (train.py:871-873), multiply then add like the reference
        x[0] = __fadd_rn(__ldg(r + 0), __fmul_rn(__ldg(r + 3), z));
        x[1] = __fadd_rn(__ldg(r + 1), __fmul_rn(__ldg(r + 4), z));
        x[2] = __fadd_rn(__ldg(r + 2), __fmul_rn(__ldg(r + 5), z));
      }
      if (p.d_init) {
        p.d_init[pt * 3 + 0] = x[0]; p.d_init[pt * 3 + 1] = x[1]; p.d_init[pt * 3 + 2] = x[2];
      }
    }
    float rigidity = 0.f;
    if (HAS_BENDER) {
      // ---- bender input row: [xyz_hi(3) xyz_lo(3) latent(32) 0(10)] fp16, chunks 0..5 of E ----
      stash_begin();
      if (row_thread) {
        float in[48];
#pragma unroll
        for (int d = 0; d < 3; ++d) {
          const float hi = __half2float(__float2half_rn(x[d]));
          in[d] = hi;
          in[3 + d] = x[d] - hi;
        }
        const float* lat = p.latents + ray * p.latent_stride;
#pragma unroll
        for (int i = 0; i < kLatent; ++i) in[6 + i] = valid ? __ldg(lat + i) : 0.f;
#pragma unroll
        for (int i = 38; i < 48; ++i) in[i] = 0.f;
#pragma unroll
        for (int c = 0; c < 6; ++c) {
          uint4 pk;
          pk.x = pack_h2(in[c * 8 + 0], in[c * 8 + 1]);
          pk.y = pack_h2(in[c * 8 + 2], in[c * 8 + 3]);
          pk.z = pack_h2(in[c * 8 + 4], in[c * 8 + 5]);
          pk.w = pack_h2(in[c * 8 + 6], in[c * 8 + 7]);
          *reinterpret_cast<uint4*>(e_row + c * kChunkBytes) = pk;
        }
      }
      ready(kStBin, Es, 6);
      // ---- B0, B1: 96 hidden units (64 offset | 32 rigidity) ----
      {
        float acc[48];
        wg_gemm<96>(acc, ring, 1, 3, [&](uint32_t) { return a_e; }, W, 301);
        stash_begin();
        epi_bias_relu_store<96, TRAIN>(acc, p.bend_bias, Hs, g, mk, kMkHb1);
        ready(kStHb1, Hs, 12);
        wg_gemm<96>(acc, ring, 1, 6, [&](uint32_t) { return a_h; }, W, 302);
        stash_begin();
        epi_bias_relu_store<96, TRAIN>(acc, p.bend_bias + 96, Hs, g, mk, kMkHb2);
        ready(kStHb2, Hs, 12);
      }
      // ---- B2: 64 offset hidden + rigidity output (column 64) ----
      {
        float acc[40];
        wg_gemm<80>(acc, ring, 1, 6, [&](uint32_t) { return a_h; }, W, 303);
        stash_begin();
        epi_bias_relu_store<64, TRAIN>(acc, p.bend_bias + 192, Hs, g, mk, kMkHb3);
        if (acc_q() == 0) {
          stg[acc_r0() * kFwdStageLd] = acc[32];
          stg[(acc_r0() + 8) * kFwdStageLd] = acc[34];
        }
        ready(kStHb3, Hs, 8);
        if (row_thread) {
          const float rr = my_stg[0] + __ldg(p.bend_bias + 192 + 64);
          rigidity = (tanhf(rr) + 1.0f) * 0.5f;   // run_nerf_helpers.py:559-561
          if (p.use_cutoff && rigidity <= p.cutoff) rigidity = 0.f;  // :563-564
        }
      }
      // ---- B3 ----
      {
        float acc[32];
        wg_gemm<64>(acc, ring, 1, 4, [&](uint32_t) { return a_h; }, W, 304);
        stash_begin();
        epi_bias_relu_store<64, TRAIN>(acc, p.bend_bias + 272, Hs, g, mk, kMkHb4);
        ready(kStHb4, Hs, 8);
      }
      // ---- B4: offsets; bend ----
      {
        float acc[8];
        wg_gemm<16>(acc, ring, 1, 4, [&](uint32_t) { return a_h; }, W, 305);
        stage_cols<0, 1>(acc, stg, kFwdStageLd);
        wg_bar(bar);
        if (row_thread) {
          float un[3], ma[3];
#pragma unroll
          for (int d = 0; d < 3; ++d) {
            un[d] = my_stg[d];
            ma[d] = __fmul_rn(rigidity, un[d]);              // :567
            if (p.use_scaling) ma[d] = __fmul_rn(ma[d], p.scaling);  // :568-569
          }
          if (valid) {
            if (p.d_unmasked) { p.d_unmasked[pt * 3 + 0] = un[0]; p.d_unmasked[pt * 3 + 1] = un[1]; p.d_unmasked[pt * 3 + 2] = un[2]; }
            if (p.d_masked) { p.d_masked[pt * 3 + 0] = ma[0]; p.d_masked[pt * 3 + 1] = ma[1]; p.d_masked[pt * 3 + 2] = ma[2]; }
            if (p.d_rigid) p.d_rigid[pt] = rigidity;
          }
#pragma unroll
          for (int d = 0; d < 3; ++d) x[d] = __fadd_rn(x[d], ma[d]);  // :570
        }
      }
    }
    if (valid && p.d_bent) {
      p.d_bent[pt * 3 + 0] = x[0]; p.d_bent[pt * 3 + 1] = x[1]; p.d_bent[pt * 3 + 2] = x[2];
    }
    // ---- positional encoding of the (bent) point -> E ----
    stash_begin();
    if (row_thread) write_pe(x, e_row);
    ready(kStE, Es, 8);
    // ---- L0 .. L7 ----
#pragma unroll 1
    for (int L = 0; L < 8; ++L) {
      const int step = 5 + L;
      const StepShape s = step_shape(step);
      float acc[128];
      wg_gemm<256>(acc, ring, s.nslabs, s.k16, [&](uint32_t j) { return a_h + a_operand_offset(step, j); }, W, 310 + L);
      stash_begin();
      epi_bias_relu_store<256, TRAIN>(acc, p.nerf_bias + L * 256, Hs, g, mk, kMkH + L * kMaskHBytes);
      ready(kStH + L * kHBytes, Hs, 32);
    }
    // ---- head: raw = output_linear(h) (run_nerf_helpers.py:306) ----
    {
      float acc[8];
      wg_gemm<16>(acc, ring, 1, 16, [&](uint32_t) { return a_h; }, W, 320);
      stage_cols<0, 1>(acc, stg, kFwdStageLd);
      wg_bar(bar);
      if (valid) {
        float o[5];
#pragma unroll
        for (int c = 0; c < 5; ++c) o[c] = my_stg[c] + __ldg(p.nerf_bias + 2048 + c);
        // test-time non-rigid object removal (run_nerf_helpers.py:309-310)
        if (HAS_BENDER && p.use_removal && rigidity >= p.removal) o[3] *= 0.f;
        float* dst = p.raw + pt * p.out_ch;
        for (int c = 0; c < p.out_ch; ++c) dst[c] = o[c];
      }
    }
    // the staging rows are rewritten only after further warpgroup barriers (next tile's B2 / head)
  }
  if (p.stash && wg_leader) tma_bulk_wait<0>();   // all stash stores complete before the CTA exits
}

// ------------------------------------------------------------------------------------------------
size_t field_fwd_smem_bytes() {
  return kSlotBytes + kRingStages * kRingStageBytes + 2 * kWgRows * kFwdStageLd * sizeof(float) + sizeof(Shared) + 64;
}

template <bool HAS_BENDER, bool TRAIN>
static cudaError_t launch_field_fwd_t(const FieldFwdParams& p, int grid, size_t smem, cudaStream_t stream) {
  const cudaError_t e = cudaFuncSetAttribute(field_fwd_kernel<HAS_BENDER, TRAIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  field_fwd_kernel<HAS_BENDER, TRAIN><<<grid, kFwdThreads, smem, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_field_fwd(const FieldFwdParams& p, bool has_bender, int num_sms, cudaStream_t stream) {
  const size_t smem = field_fwd_smem_bytes();
  if (p.n_tiles <= 0) return cudaSuccess;
  const int grid = p.n_tiles < num_sms ? p.n_tiles : num_sms;
  const bool train = p.relu_mask != nullptr;   // the C ABI passes the ReLU masks exactly when it passes the stash
  if (has_bender) return train ? launch_field_fwd_t<true, true>(p, grid, smem, stream) : launch_field_fwd_t<true, false>(p, grid, smem, stream);
  return train ? launch_field_fwd_t<false, true>(p, grid, smem, stream) : launch_field_fwd_t<false, false>(p, grid, smem, stream);
}

}  // namespace nrn
