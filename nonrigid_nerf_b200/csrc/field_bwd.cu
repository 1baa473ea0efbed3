// Fused point-wise field evaluation, backward data-gradient chain (DGRAD).
//
// What torch.autograd derives for NeRF.forward + ray_bending.forward + Embedder.embed
// (run_nerf_helpers.py:240-314, :507-584, :149-150) given dL/draw: the gradient w.r.t. every
// layer's pre-activation ("dY_l"), the per-ray latent gradient, and -- through the gradient stash --
// the inputs of the weight-gradient kernel (wgrad.cu).  SURVEY.md appendix C is the specification.
//
// Same machine as field_fwd.cu (field_mma.cuh): persistent CTA over 128-point tiles, two consumer
// warpgroups (wgmma + epilogue, 64 rows each), weights (here W^T images) streamed by bulk TMA.
//   step  0      head^T   dh8 = d_raw . Wout          -> dY7 = dh8 * [h8 > 0]
//   steps 1,2    L7^T,L6^T                            -> dY6, dY5
//   step  3      L5e^T    dE  = dY5 . W5[:, :63]      -> PE backward -> d(bent xyz)
//   steps 4..8   L5h^T, L4^T..L1^T                    -> dY4..dY0
//   step  9      L0^T     dE += ...                   -> PE backward; bend backward -> dYb4
//   steps 10..13 B4^T..B1^T (offset + rigidity MLPs, block diagonal) -> dYb3..dYb0
//   step  14     B0^T     d(bender input)             -> per-ray latent gradient (fp32 atomics)
// All gradients travel in fp16 scaled by a power-of-two loss scale derived on the device from
// max|d_raw| (no host sync); WGRAD and the latent reduction divide it out again in fp32.
#include "field_mma.cuh"

namespace nrn {

namespace {

constexpr int kBwdStageLd = 66;   // floats per staged row (64 used)

struct Shared {
  uint64_t w_full[kRingStages];
  uint64_t w_empty[kRingStages];
  int abort_flag;
};

struct StepShape {
  uint32_t N, nslabs, slab_bytes, k16;
};

__device__ __forceinline__ StepShape step_shape(int step) {
  switch (step) {
    case 0: return {256u, 1u, (uint32_t)kNerfTHeadBytes, 1u};
    case 3: return {64u, 1u, 32768u, 16u};
    case 9: return {64u, 1u, 32768u, 16u};
    case 10: return {64u, 1u, (uint32_t)kBendTB4Bytes, 1u};
    case 11: return {64u, 1u, (uint32_t)kBendTB3Bytes, 4u};
    case 12: return {96u, 1u, (uint32_t)kBendTB2Bytes, 5u};
    case 13: return {96u, 1u, (uint32_t)kBendTB1Bytes, 6u};
    case 14: return {48u, 1u, (uint32_t)kBendTB0Bytes, 6u};
    default: return {256u, 4u, 32768u, 4u};
  }
}

__device__ __forceinline__ float clamp_h(float v) { return fminf(fmaxf(v, -65504.f), 65504.f); }

// dY = dh * [h > 0]: accumulator columns [0, NCOLS), masked with the forward's ReLU mask bits `m` (loaded before the
// step's MMAs), written as fp16 to this warpgroup's rows of the next A operand `img`; the whole image then goes to the
// gradient stash with bulk TMA stores.
template <int NCOLS, int NR>
__device__ __forceinline__ void epi_mask_store(const float (&acc)[NR], const ReluMask<NCOLS>& m, uint8_t* img, int g) {
  const int r0 = g * kWgRows + acc_r0(), q = acc_q();
#pragma unroll
  for (int j = 0; j < NCOLS / 8; ++j) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      // saturating convert, then multiply by the 0/1 mask on packed halves
      const uint32_t g2 = pack_h2_sat(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]);
      *reinterpret_cast<uint32_t*>(img + j * kChunkBytes + (r0 + 8 * i) * 16 + 4 * q) = m.apply(i, j, g2);
    }
  }
}

__device__ __forceinline__ float h_lo(uint32_t w) { return __half2float(__ushort_as_half(static_cast<unsigned short>(w & 0xffffu))); }
__device__ __forceinline__ float h_hi(uint32_t w) { return __half2float(__ushort_as_half(static_cast<unsigned short>(w >> 16))); }

// Backward of the positional encoding: dx_d += dE[d] + sum_k 2^k (dE[sin_kd] cos_kd - dE[cos_kd] sin_kd)
// de: this row's 64 staged accumulator columns; sin/cos: the forward embedding stashed as fp16.
__device__ __forceinline__ void pe_backward(const float* de, const uint8_t* __restrict__ e_row, float (&dx)[3]) {
  float e[64];
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const uint4 w = __ldg(reinterpret_cast<const uint4*>(e_row + c * kChunkBytes));
    e[c * 8 + 0] = h_lo(w.x); e[c * 8 + 1] = h_hi(w.x); e[c * 8 + 2] = h_lo(w.y); e[c * 8 + 3] = h_hi(w.y);
    e[c * 8 + 4] = h_lo(w.z); e[c * 8 + 5] = h_hi(w.z); e[c * 8 + 6] = h_lo(w.w); e[c * 8 + 7] = h_hi(w.w);
  }
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    float acc = de[d];
#pragma unroll
    for (int k = 0; k < 10; ++k) {
      const float f = static_cast<float>(1 << k);
      const float s = e[3 + 6 * k + d], c = e[3 + 6 * k + 3 + d];
      acc += f * (de[3 + 6 * k + d] * c - de[3 + 6 * k + 3 + d] * s);
    }
    dx[d] += acc;
  }
}

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

}  // namespace

template <bool HAS_BENDER>
__global__ void __launch_bounds__(kFwdThreads, 1) field_bwd_kernel(const FieldBwdParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* act = smem;                               // 64 KB gradient operand, 128 rows
  uint8_t* ring_buf = smem + kHBytes;                // kRingStages x 32 KB
  float* stage_all = reinterpret_cast<float*>(ring_buf + kRingStages * kRingStageBytes);   // 2 x 64 rows x kBwdStageLd
  Shared* sh = reinterpret_cast<Shared*>(stage_all + 2 * kWgRows * kBwdStageLd);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  constexpr int kNumSteps = HAS_BENDER ? 15 : 10;

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
    // ===================== weight producer (W^T images) =====================
    if (warp == 8 && lane == 0) {
      for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
        uint32_t gn = 0, gb = 0;
#pragma unroll 1
        for (int step = 0; step < kNumSteps; ++step) {
          const StepShape s = step_shape(step);
          const uint8_t* src = step < 10 ? p.nerf_wT + gn : p.bend_wT + gb;
          for (uint32_t j = 0; j < s.nslabs; ++j) ring_put(ring, src + j * s.slab_bytes, s.slab_bytes, W);
          if (step < 10) gn += s.nslabs * s.slab_bytes; else gb += s.nslabs * s.slab_bytes;
        }
      }
    }
    return;
  }

  // ===================== consumer warpgroups =====================
  setmaxnreg_inc<kConsumerRegs>();
  const int g = warp >> 2;
  const int tw = threadIdx.x & 127;
  const bool row_thread = tw < kWgRows;   // threads 0-63 (warps 0, 1 of the warpgroup) each own one row
  const int bar = 1 + g;
  const bool wg_leader = tw == 0;
  const int row = g * kWgRows + tw;       // tile row of a row thread
  uint8_t* a_row = act + row * 16;
  const uint32_t a_base = smem_u32(act) + g * kWgRows * 16;
  auto a_slab = [&](uint32_t j) { return a_base + j * 8 * kChunkBytes; };
  float* stg = stage_all + g * kWgRows * kBwdStageLd;
  const float* my_stg = stg + tw * kBwdStageLd;

  // power-of-two loss scale from max|d_raw| (written by the compositing backward kernel)
  float scale = 1.0f;
  {
    const float amax = p.amax ? __ldg(p.amax) : 0.f;
    if (amax > 0.f && amax < 3.0e38f) {
      int e;
      frexpf(amax, &e);                       // amax = m * 2^e, m in [0.5, 1)
      scale = ldexpf(1.0f, min(max(10 - e, -60), 60));  // max|d_raw| * scale in [512, 1024)
    }
  }
  const float inv_scale = 1.0f / scale;

  for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
    const long long pt = static_cast<long long>(tile) * kTileM + row;
    const bool valid = row_thread && pt < p.P;
    const uint8_t* st_tile = p.stash + static_cast<long long>(tile) * kStashTileBytes;
    const uint8_t* st = st_tile + row * 16;
    uint8_t* gs = p.gstash + static_cast<long long>(tile) * kGradTileBytes;
    // gradient stash: bulk TMA stores of finished images from shared memory (see field_fwd.cu)
    auto stash_begin = [&]() {
      if (wg_leader) tma_bulk_wait_read<0>();
      wg_bar(bar);
    };
    auto ready = [&](uint32_t off, uint32_t chunks) {
      fence_proxy_async_smem();
      wg_bar(bar);
      if (wg_leader && chunks) store_rows(gs + off, act, g, chunks);
    };
    // The ReLU masks are bits the forward kernel wrote (ReluMask): each thread loads its few words of a step's mask
    // before that step's MMAs, which hide the latency.  The embedding pe_backward reads from the forward stash is pulled
    // into L2 by one thread while the epilogue of the step before runs.
    const uint8_t* mk = p.relu_mask + static_cast<long long>(tile) * kMaskTileBytes;
    auto prefetch_e = [&]() {
      if (wg_leader) tma_prefetch_l2(st_tile + kStE, kEBytes);
    };
    // ---- d_raw image: [g_r g_g g_b g_sigma 0 ...] (K = 16) ----
    stash_begin();
    if (row_thread) {
      float gr[4] = {0.f, 0.f, 0.f, 0.f};
      if (valid) {
        const float* q = p.d_raw + pt * p.out_ch;
#pragma unroll
        for (int c = 0; c < 4; ++c) gr[c] = clamp_h(__ldg(q + c) * scale);
      }
      *reinterpret_cast<uint4*>(a_row) = make_uint4(pack_h2(gr[0], gr[1]), pack_h2(gr[2], gr[3]), 0u, 0u);
      *reinterpret_cast<uint4*>(a_row + kChunkBytes) = make_uint4(0u, 0u, 0u, 0u);
    }
    ready(kGsRaw, 2);
    float dx[3] = {0.f, 0.f, 0.f};
    // ---- head^T, L7^T, L6^T : dY7, dY6, dY5 ----
#pragma unroll 1
    for (int s = 0; s < 3; ++s) {
      const StepShape sh_ = step_shape(s);
      float acc[128];
      ReluMask<256> m;
      m.load(mk + kMkH + (7 - s) * kMaskHBytes, g);
      wg_gemm<256>(acc, ring, sh_.nslabs, sh_.k16, a_slab, W, 300 + s);
      if (s == 2) prefetch_e();
      stash_begin();
      epi_mask_store<256>(acc, m, act, g);
      ready(kGsY + (7 - s) * kHBytes, 32);
    }
    // ---- L5e^T: gradient into the skip-connected embedding ----
    {
      float acc[32];
      wg_gemm<64>(acc, ring, 1, 16, a_slab, W, 303);
      stage_cols<0, 8>(acc, stg, kBwdStageLd);
      wg_bar(bar);
      if (row_thread) pe_backward(my_stg, st + kStE, dx);
      // A operand (dY5) untouched; the staging rows are rewritten only after the barriers of the next steps
    }
    // ---- L5h^T, L4^T .. L1^T : dY4 .. dY0 ----
#pragma unroll 1
    for (int s = 0; s < 5; ++s) {
      float acc[128];
      ReluMask<256> m;
      m.load(mk + kMkH + (4 - s) * kMaskHBytes, g);
      wg_gemm<256>(acc, ring, 4, 4, a_slab, W, 304 + s);
      if (s == 4) prefetch_e();
      stash_begin();
      epi_mask_store<256>(acc, m, act, g);
      ready(kGsY + (4 - s) * kHBytes, 32);
    }
    // ---- L0^T: gradient into the embedding; then through the bend ----
    {
      float acc[32];
      wg_gemm<64>(acc, ring, 1, 16, a_slab, W, 309);
      stage_cols<0, 8>(acc, stg, kBwdStageLd);
      wg_bar(bar);
      if (row_thread) pe_backward(my_stg, st + kStE, dx);
    }
    if (!HAS_BENDER) continue;   // xyz has no learnable upstream without a bender (appendix C)

    float drpre = 0.f;
    stash_begin();
    if (row_thread) {
      float rig = 0.f, un[3] = {0.f, 0.f, 0.f}, dun[3], dm[3];
      float up_r = 0.f, up_u[3] = {0.f, 0.f, 0.f};
      if (valid) {
        rig = __ldg(p.rigidity + pt);
#pragma unroll
        for (int d = 0; d < 3; ++d) un[d] = __ldg(p.unmasked + pt * 3 + d);
        if (p.d_rigid_up) up_r = __ldg(p.d_rigid_up + pt) * scale;
        if (p.d_unmasked_up) {
#pragma unroll
          for (int d = 0; d < 3; ++d) up_u[d] = __ldg(p.d_unmasked_up + pt * 3 + d) * scale;
        }
      }
      float dr = up_r;
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        dm[d] = p.use_scaling ? dx[d] * p.scaling : dx[d];   // masked = rig * un (* scaling); bent = xyz + masked
        dun[d] = rig * dm[d] + up_u[d];
        dr += un[d] * dm[d];
      }
      // rigidity = (tanh(pre) + 1) / 2  =>  d/dpre = (1 - tanh^2) / 2 = 2 r (1 - r); cut-off entries carry no gradient
      drpre = dr * 2.0f * rig * (1.0f - rig);
      if (p.use_cutoff && rig <= p.cutoff) drpre = 0.f;
      if (!valid) { dun[0] = dun[1] = dun[2] = 0.f; drpre = 0.f; }
      *reinterpret_cast<uint4*>(a_row) = make_uint4(pack_h2(clamp_h(dun[0]), clamp_h(dun[1])), pack_h2(clamp_h(dun[2]), 0.f), 0u, 0u);
      *reinterpret_cast<uint4*>(a_row + kChunkBytes) = make_uint4(0u, 0u, 0u, 0u);
    }
    ready(kGsYb4, 2);
    // ---- B4^T -> dYb3 ----
    {
      float acc[32];
      ReluMask<64> m;
      m.load(mk + kMkHb4, g);
      wg_gemm<64>(acc, ring, 1, 1, a_slab, W, 310);
      stash_begin();
      epi_mask_store<64>(acc, m, act, g);
      ready(kGsYb3, 8);
    }
    // ---- B3^T -> dYb2 = [dh * mask (64) | d rigidity pre-activation | 0 (15)] ----
    {
      float acc[32];
      ReluMask<64> m;
      m.load(mk + kMkHb3, g);
      wg_gemm<64>(acc, ring, 1, 4, a_slab, W, 311);
      stash_begin();
      epi_mask_store<64>(acc, m, act, g);
      if (row_thread) {
        *reinterpret_cast<uint4*>(a_row + 8 * kChunkBytes) = make_uint4(pack_h2(clamp_h(drpre), 0.f), 0u, 0u, 0u);
        *reinterpret_cast<uint4*>(a_row + 9 * kChunkBytes) = make_uint4(0u, 0u, 0u, 0u);
      }
      ready(kGsYb2, 10);
    }
    // ---- B2^T -> dYb1, B1^T -> dYb0 ----
    {
      float acc[48];
      ReluMask<96> m;
      m.load(mk + kMkHb2, g);
      wg_gemm<96>(acc, ring, 1, 5, a_slab, W, 312);
      stash_begin();
      epi_mask_store<96>(acc, m, act, g);
      ready(kGsYb1, 12);
      m.load(mk + kMkHb1, g);
      wg_gemm<96>(acc, ring, 1, 6, a_slab, W, 313);
      stash_begin();
      epi_mask_store<96>(acc, m, act, g);
      ready(kGsYb0, 12);
    }
    // ---- B0^T: d(bender input); columns 6..37 are the latent code -> per-ray reduction ----
    {
      float acc[24];
      wg_gemm<48>(acc, ring, 1, 6, a_slab, W, 314);
      stage_cols<0, 5>(acc, stg, kBwdStageLd);
      wg_bar(bar);
      if (row_thread) {   // warps 0 and 1 of the warpgroup: 32 consecutive rows each
        float dl[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) dl[i] = my_stg[6 + i] * inv_scale;
        const long long ray = valid ? pt / p.S : -1;
        const long long ray0 = __shfl_sync(0xffffffffu, ray, 0);
        if (__all_sync(0xffffffffu, ray == ray0 && valid)) {
          const float tot = warp_transpose_reduce(dl, lane);   // lane j holds latent dim j
          atomicAdd(p.d_latents + ray0 * kLatent + lane, tot);
        } else if (valid) {
#pragma unroll
          for (int i = 0; i < 32; ++i) atomicAdd(p.d_latents + ray * kLatent + i, dl[i]);
        }
      }
    }
    // next: the next tile's d_raw image (after stash_begin's barrier)
  }
  if (wg_leader) tma_bulk_wait<0>();   // all gradient-stash stores complete before the CTA exits
}

// ------------------------------------------------------------------------------------------------
cudaError_t launch_field_bwd(const FieldBwdParams& p, bool has_bender, int num_sms, cudaStream_t stream) {
  const size_t smem = kHBytes + kRingStages * kRingStageBytes + 2 * kWgRows * kBwdStageLd * sizeof(float) + sizeof(Shared) + 64;
  if (p.n_tiles <= 0) return cudaSuccess;
  const int grid = p.n_tiles < num_sms ? p.n_tiles : num_sms;
  cudaError_t e;
  if (has_bender) {
    e = cudaFuncSetAttribute(field_bwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    field_bwd_kernel<true><<<grid, kFwdThreads, smem, stream>>>(p);
  } else {
    e = cudaFuncSetAttribute(field_bwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    field_bwd_kernel<false><<<grid, kFwdThreads, smem, stream>>>(p);
  }
  return cudaGetLastError();
}

}  // namespace nrn
