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
//   step  14     B0^T     d(bender input)             -> per-ray latent gradient (fp32 atomics; field_bwd_det_kernel:
//                                                         per-point rows for det_reduce.cu's fixed-order sum)
// All gradients travel in fp16 scaled by a power-of-two loss scale derived on the device from
// max|d_raw| (no host sync); WGRAD and the latent reduction divide it out again in fp32.
// field_bwd_views_kernel (view-dependent head, no bender): Rgb^T, ViewsF^T and Feature^T + head^T in front of L7^T.
// field_bwd_held_kernel (bender, held-out rays): the same chain; the gradient-stash rows of held-out rays' points are zero.
#include "field_epilogue.cuh"

namespace nrn {

namespace {

// A = d_raw [4 channels, 0 ...] (K = 16) of this warpgroup's rows, times the loss scale and clamped to fp16: one register
// fragment built from global memory (lanes q < 2 hold columns 2q, 2q + 1 of rows r0, r0 + 8; every other word is zero,
// rows past P too), and the same words -> the tile's kGsRaw image, its zero columns and zero second chunk included (A of
// WGRAD's head and rgb_linear jobs)
__device__ __forceinline__ void d_raw_frag(const FieldBwdParams& p, int tile, float scale, uint8_t* gs, int g, uint32_t (&a)[1][4]) {
  const int r0 = g * kWgRows + acc_r0(), q = acc_q();
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const long long pti = static_cast<long long>(tile) * kTileM + r0 + 8 * i;
    float g0 = 0.f, g1 = 0.f;
    if (q < 2 && pti < p.P) {
      const float* src = p.d_raw + pti * p.out_ch + 2 * q;
      g0 = clamp_h(__ldg(src) * scale);
      g1 = clamp_h(__ldg(src + 1) * scale);
    }
    a[0][i] = q < 2 ? pack_h2(g0, g1) : 0u;
    a[0][2 + i] = 0u;
  }
#pragma unroll
  for (int j = 0; j < 2; ++j)
#pragma unroll
    for (int i = 0; i < 2; ++i)
      *reinterpret_cast<uint32_t*>(gs + kGsRaw.off + j * kChunkBytes + (r0 + 8 * i) * 16 + 4 * q) = frag_pair(a, j, i);
}

// Held-out rays (field_bwd_held_kernel): bit i is set when this thread's accumulator row r0 + 8 i is a point of a held-out
// ray.  The epilogues store the gradient-stash words of every row as usual and then overwrite those of held-out rows with
// zeros (clear_held_rows), so that the gradient itself travels on unchanged.
struct HeldRows {
  uint32_t bits = 0u;
};

// Held-out rays: which of this thread's accumulator rows of warpgroup g in `tile` are held out (rows past P are stored as
// they are, like the bulk stores of field_bwd_kernel do)
__device__ __forceinline__ HeldRows held_rows(const FieldBwdParams& p, const uint8_t* __restrict__ held, int tile, int g) {
  HeldRows k;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const long long pt = static_cast<long long>(tile) * kTileM + g * kWgRows + acc_r0() + 8 * i;
    if (pt < p.P && __ldg(held + pt / p.S)) k.bits |= 1u << i;
  }
  return k;
}

// Held-out rays: zeros over this thread's words of its held-out rows in columns [0, NCOLS) of the chunk-major image `img`
// of warpgroup g, after the epilogue's own stores of them (same thread, so they land last)
template <int NCOLS>
__device__ __forceinline__ void clear_held_rows(uint8_t* img, int g, const HeldRows& k) {
  if (!k.bits) return;
  const int r0 = g * kWgRows + acc_r0(), q = acc_q();
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    if ((k.bits >> i) & 1u) {
#pragma unroll
      for (int j = 0; j < NCOLS / 8; ++j) *reinterpret_cast<uint32_t*>(img + j * kChunkBytes + (r0 + 8 * i) * 16 + 4 * q) = 0u;
    }
  }
}

// Held-out rays: a finished bender gradient image `im` of `act` (written, fenced and warpgroup-synced as for
// StashWriter::ready) -> the tile's gradient stash by one row thread per row, as zeros for a held-out row.  act itself
// stays as it is: it is the next step's A operand, which carries the held-out rays' latent gradient.
__device__ __forceinline__ void store_row_held(uint8_t* gs, Image im, const uint8_t* act, int row, bool held_row) {
  for (uint32_t c = 0; c < im.chunks; ++c) {
    const uint4 v = held_row ? make_uint4(0u, 0u, 0u, 0u) : *reinterpret_cast<const uint4*>(act + c * kChunkBytes + row * 16);
    *reinterpret_cast<uint4*>(gs + im.off + c * kChunkBytes + row * 16) = v;
  }
}

// step -> shape in the view-head DGRAD's streaming order Rgb^T, ViewsF^T, Feature^T, head^T, L7^T, L6^T, L5h^T .. L1^T
static_assert(vdgrad::step(vdgrad::FeatureT) == dgrad::step(dgrad::L7T), "step_at_views: Feature^T has the trunk's shape");
__device__ __forceinline__ Step step_at_views(int step) {
  switch (step) {
    case dgrad::HeadT: return step_imm<dgrad::HeadT>();
    case vdgrad::RgbT: return step_imm<vdgrad::RgbT>();
    case vdgrad::ViewsFT: return step_imm<vdgrad::ViewsFT>();
    default: return step_imm<dgrad::L7T>();   // Feature^T, L7^T, L6^T, L5h^T, L4^T .. L1^T
  }
}


}  // namespace

// DET = false: B0^T adds each warp's latent rows into d_latents with fp32 atomics, in no fixed order.
// DET = true (deterministic mode): it writes them to latent_rows [P][32] instead (det_reduce.cu's rule: a warp whose 32 rows
// are all valid and of one ray stores their transpose-reduced sum in the row of its first point, 32k; any other warp stores
// each valid row), and latent_reduce_kernel sums them per ray in a fixed order.
// HELD (bender only): `held` [n_rays] bytes, nonzero for a held-out ray.  Every step runs as without it, so a held-out ray's
// latent gradient is formed as before, but every gradient-stash row of its points (kGsRaw, dY7 .. dY0, dYb4 .. dYb0) is
// stored as zeros, so that WGRAD's weight and bias sums leave it out.  The bender images then go to the stash by per-row
// stores instead of bulk stores of act.
template <bool HAS_BENDER, bool DET, bool HELD = false>
__device__ __forceinline__ void field_bwd_body(const FieldBwdParams& p, float* latent_rows, const uint8_t* held = nullptr) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* act = smem;                               // bender gradient operand (24 KB), 128 rows
  uint8_t* ring_buf = smem + kBwdActBytes;           // kBwdRingStages x 32 KB
  float* stage_all = reinterpret_cast<float*>(ring_buf + kBwdRingStages * kRingStageBytes);   // 2 x 64 rows x kBwdStageLd
  auto* sh = reinterpret_cast<RingShared<kBwdRingStages>*>(stage_all + 2 * kWgRows * kBwdStageLd);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) sh->init();
  __syncthreads();
  const Waiter W{&sh->abort_flag, p.err};
  Ring<kBwdRingStages> ring{ring_buf, sh->w_full, sh->w_empty};

  if (warp >= 8) {
    setmaxnreg_dec<kProducerRegs>();
    // ===================== weight producer (W^T images) =====================
    if (warp == 8 && lane == 0) produce(p.nerf_wT, p.bend_wT, p.n_tiles, 0, HAS_BENDER ? dgrad::kCount : dgrad::B4T, dgrad::B4T, dgrad_step_at, ring, W);
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
  auto a_slab = [&](uint32_t j) { return a_base + j * kSlabA; };
  float* stg = stage_all + g * kWgRows * kBwdStageLd;
  const float* my_stg = stg + tw * kBwdStageLd;

  const float scale = loss_scale(p.amax);   // max|d_raw| is written by the compositing backward kernel
  const float inv_scale = 1.0f / scale;

  for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
    const long long pt = static_cast<long long>(tile) * kTileM + row;
    const bool valid = row_thread && pt < p.P;
    const uint8_t* st_tile = p.stash + static_cast<long long>(tile) * kStashTileBytes;
    const uint8_t* st = st_tile + row * 16;
    uint8_t* gs = p.gstash + static_cast<long long>(tile) * kGradTileBytes;
    const StashWriter<false> sw{gs, wg_leader, bar, g};
    // The ReLU masks are bits the forward kernel wrote (ReluMask): each thread loads its few words of a step's mask
    // before that step's MMAs, which hide the latency.  The embedding pe_backward reads from the forward stash is pulled
    // into L2 by one thread while the epilogue of the step before runs.
    const uint8_t* mk = p.relu_mask + static_cast<long long>(tile) * kMaskTileBytes;
    auto prefetch_e = [&]() {
      if (wg_leader) tma_prefetch_l2(st_tile + kStE.off, kEBytes);
    };
    // The trunk's gradients dY7 .. dY0 stay in registers: each epilogue packs them into the A fragments h of the next step
    // (wg_gemm_rs) and stores them to the gradient stash from there.  Only the staging rows stg are shared, and each of
    // their rewrites is ordered after the reads before it by an explicit warpgroup barrier (L5e^T, L0^T).
    constexpr Step kTrunk = dgrad::step(dgrad::L7T), kEmb = dgrad::step(dgrad::L5eT);
    static_assert(dgrad::step(dgrad::L0T) == kEmb && kEmb.nslabs == 1 && kEmb.k16 == kMaskHCols / 16, "L5e^T, L0^T: one slab, K = 256");
    uint32_t h[kMaskHCols / 16][4];
    HeldRows hr;
    if constexpr (HELD) hr = held_rows(p, held, tile, g);
    // ---- head^T: A = d_raw [g_r g_g g_b g_sigma 0 ...] (K = 16), one fragment built from global memory ----
    {
      static_assert(dgrad::step(dgrad::HeadT).N == kTrunk.N && dgrad::step(dgrad::HeadT).nslabs == 1 &&
                    dgrad::step(dgrad::HeadT).k16 == 1 && kGsRaw.chunks == 2, "head^T: one K = 16 MMA");
      uint32_t a[1][4];
      d_raw_frag(p, tile, scale, gs, g, a);
      if constexpr (HELD) clear_held_rows<16>(gs + kGsRaw.off, g, hr);
      Acc<dgrad::HeadT> acc;
      ReluMask<kMaskHCols> m;
      m.load(mk + kMkH + 7 * kMaskHBytes, g);
      wg_gemm_rs<kTrunk.N, 1>(acc, a, ring, false, 0u, W, 300);
      epi_grad_frag<kMaskHCols, true>(acc, m, h, gs + kGsY + 7 * kHBytes, g);
      if constexpr (HELD) clear_held_rows<kMaskHCols>(gs + kGsY + 7 * kHBytes, g, hr);
    }
    float dx[3] = {0.f, 0.f, 0.f};
    // ---- L7^T, L6^T : dY6, dY5 ----
#pragma unroll 1
    for (int s = 0; s < 2; ++s) {
      Acc<dgrad::L7T> acc;
      ReluMask<kMaskHCols> m;
      m.load(mk + kMkH + (6 - s) * kMaskHBytes, g);
      wg_gemm_rs<kTrunk.N, kTrunk.k16>(acc, h, ring, false, 0u, W, 301 + s);
      if (s == 1) prefetch_e();
      epi_grad_frag<kMaskHCols, true>(acc, m, h, gs + kGsY + (6 - s) * kHBytes, g);
      if constexpr (HELD) clear_held_rows<kMaskHCols>(gs + kGsY + (6 - s) * kHBytes, g, hr);
    }
    // ---- L5e^T: gradient into the skip-connected embedding; h (dY5) stays as it is for L5h^T ----
    {
      Acc<dgrad::L5eT> acc;
      wg_gemm_rs<kEmb.N, kEmb.k16>(acc, h, ring, false, 0u, W, 303);
      wg_bar(bar);   // stg: every read of the previous tile (L0^T's pe_backward / B0^T's latent rows) is done
      stage_cols<0, 8>(acc, stg, kBwdStageLd);
      wg_bar(bar);
      if (row_thread) pe_backward(my_stg, st + kStE.off, dx);
    }
    // ---- L5h^T, L4^T .. L1^T : dY4 .. dY0 (one shape) ----
#pragma unroll 1
    for (int s = 0; s < 5; ++s) {
      Acc<dgrad::L4T> acc;
      ReluMask<kMaskHCols> m;
      m.load(mk + kMkH + (4 - s) * kMaskHBytes, g);
      wg_gemm_rs<kTrunk.N, kTrunk.k16>(acc, h, ring, false, 0u, W, 304 + s);
      if (s == 4) prefetch_e();
      epi_grad_frag<kMaskHCols, true>(acc, m, h, gs + kGsY + (4 - s) * kHBytes, g);
      if constexpr (HELD) clear_held_rows<kMaskHCols>(gs + kGsY + (4 - s) * kHBytes, g, hr);
    }
    // ---- L0^T: gradient into the embedding; then through the bend ----
    {
      Acc<dgrad::L0T> acc;
      wg_gemm_rs<kEmb.N, kEmb.k16>(acc, h, ring, false, 0u, W, 309);
      wg_bar(bar);   // stg: L5e^T's pe_backward reads are done
      stage_cols<0, 8>(acc, stg, kBwdStageLd);
      wg_bar(bar);
      if (row_thread) pe_backward(my_stg, st + kStE.off, dx);
    }
    if (!HAS_BENDER) continue;   // xyz has no learnable upstream without a bender (appendix C)
    // a finished bender image of act -> the stash: bulk stores, or (HELD) per-row stores that zero the held-out rows
    bool held_row = false;
    if constexpr (HELD) held_row = valid && __ldg(held + pt / p.S);
    auto ready = [&](Image im) {
      if constexpr (HELD) {
        fence_proxy_async_smem();
        wg_bar(bar);
        if (row_thread) store_row_held(gs, im, act, row, held_row);
      } else {
        sw.ready(im, act);
      }
    };

    float drpre = 0.f;
    sw.begin();
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
    ready(kGsYb4);
    // ---- B4^T -> dYb3 ----
    {
      Acc<dgrad::B4T> acc;
      ReluMask<kMkHb4.cols> m;
      m.load(mk + kMkHb4.off, g);
      wg_gemm_step<dgrad::B4T>(acc, ring, a_slab, W, 310);
      sw.begin();
      epi_mask_store<kMkHb4.cols>(acc, m, act, g);
      ready(kGsYb3);
    }
    // ---- B3^T -> dYb2 = [dh * mask (64) | d rigidity pre-activation | 0 (15)] ----
    {
      Acc<dgrad::B3T> acc;
      ReluMask<kMkHb3.cols> m;
      m.load(mk + kMkHb3.off, g);
      wg_gemm_step<dgrad::B3T>(acc, ring, a_slab, W, 311);
      sw.begin();
      epi_mask_store<kMkHb3.cols>(acc, m, act, g);
      if (row_thread) {
        *reinterpret_cast<uint4*>(a_row + 8 * kChunkBytes) = make_uint4(pack_h2(clamp_h(drpre), 0.f), 0u, 0u, 0u);
        *reinterpret_cast<uint4*>(a_row + 9 * kChunkBytes) = make_uint4(0u, 0u, 0u, 0u);
      }
      ready(kGsYb2);
    }
    // ---- B2^T -> dYb1, B1^T -> dYb0 ----
    {
      Acc<dgrad::B2T> acc;
      ReluMask<kMkHb2.cols> m;
      m.load(mk + kMkHb2.off, g);
      wg_gemm_step<dgrad::B2T>(acc, ring, a_slab, W, 312);
      sw.begin();
      epi_mask_store<kMkHb2.cols>(acc, m, act, g);
      ready(kGsYb1);
      m.load(mk + kMkHb1.off, g);
      wg_gemm_step<dgrad::B1T>(acc, ring, a_slab, W, 313);
      sw.begin();
      epi_mask_store<kMkHb1.cols>(acc, m, act, g);
      ready(kGsYb0);
    }
    // ---- B0^T: d(bender input); columns 6..37 are the latent code -> per-ray reduction ----
    {
      Acc<dgrad::B0T> acc;
      wg_gemm_step<dgrad::B0T>(acc, ring, a_slab, W, 314);
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
          if constexpr (DET) latent_rows[(pt - lane) * kLatent + lane] = tot;   // the row of the warp's first point, 32k
          else atomicAdd(p.d_latents + ray0 * kLatent + lane, tot);
        } else if (valid) {
          if constexpr (DET) {
            float4* dst = reinterpret_cast<float4*>(latent_rows + pt * kLatent);
#pragma unroll
            for (int i = 0; i < 8; ++i) dst[i] = make_float4(dl[4 * i], dl[4 * i + 1], dl[4 * i + 2], dl[4 * i + 3]);
          } else {
#pragma unroll
            for (int i = 0; i < 32; ++i) atomicAdd(p.d_latents + ray * kLatent + i, dl[i]);
          }
        }
      }
    }
    // next: the next tile's L5e^T rewrites stg only after its own barrier; act only after the bender's sw.begin()
  }
  if (wg_leader) tma_bulk_wait<0>();   // all gradient-stash stores complete before the CTA exits
}

template <bool HAS_BENDER>
__global__ void __launch_bounds__(kFwdThreads, 1) field_bwd_kernel(const FieldBwdParams p) { field_bwd_body<HAS_BENDER, false>(p, nullptr); }
// deterministic mode (bender only): the per-ray latent gradient goes through latent_rows and latent_reduce_kernel
__global__ void __launch_bounds__(kFwdThreads, 1) field_bwd_det_kernel(const FieldBwdParams p, float* latent_rows) {
  field_bwd_body<true, true>(p, latent_rows);
}
// held-out rays (bender only): the latent gradient as field_bwd_kernel (DET = false) or field_bwd_det_kernel (DET = true)
// forms it, the gradient-stash rows of held-out rays zero
template <bool DET>
__global__ void __launch_bounds__(kFwdThreads, 1) field_bwd_held_kernel(const FieldBwdParams p, float* latent_rows, const uint8_t* held) {
  field_bwd_body<true, DET, true>(p, latent_rows, held);
}


// View-dependent head without a bender (training): Rgb^T, ViewsF^T and Feature^T + head^T replace head^T; then L7^T, L6^T
// and L5h^T .. L1^T as in field_bwd_kernel.  L5e^T and L0^T only feed the embedding gradient, which has no consumer
// without a bender: they are neither streamed nor run.
__global__ void __launch_bounds__(kFwdThreads, 1) field_bwd_views_kernel(const FieldBwdParams p, const ViewBwdParams v) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* ring_buf = smem + kBwdActBytes;           // the same shared-memory layout as field_bwd_kernel
  float* stage_all = reinterpret_cast<float*>(ring_buf + kBwdRingStages * kRingStageBytes);
  auto* sh = reinterpret_cast<RingShared<kBwdRingStages>*>(stage_all + 2 * kWgRows * kBwdStageLd);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) sh->init();
  __syncthreads();
  const Waiter W{&sh->abort_flag, p.err};
  Ring<kBwdRingStages> ring{ring_buf, sh->w_full, sh->w_empty};

  if (warp >= 8) {
    setmaxnreg_dec<kProducerRegs>();
    // per tile: Rgb^T .. Feature^T (the view block), head^T, L7^T, L6^T, then L5h^T .. L1^T (skipping L5e^T and L0^T)
    if (warp == 8 && lane == 0) {
      auto put = [&](const uint8_t* src, int first, int last) {
#pragma unroll 1
        for (int step = first; step < last; ++step) {
          const Step s = step_at_views(step);
          for (uint32_t j = 0; j < s.nslabs; ++j) ring_put(ring, src + j * s.slab_bytes, s.slab_bytes, W);
          src += s.nslabs * s.slab_bytes;
        }
      };
      for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
        put(v.wT, vdgrad::RgbT, vdgrad::kEnd);
        put(p.nerf_wT, dgrad::HeadT, dgrad::L5eT);
        put(p.nerf_wT + dgrad::w_off(dgrad::L5hT), dgrad::L5hT, dgrad::L0T);
      }
    }
    return;
  }

  // ===================== consumer warpgroups =====================
  setmaxnreg_inc<kConsumerRegs>();
  const int g = warp >> 2;
  const float scale = loss_scale(p.amax);   // max|d_raw| over the four channels

  constexpr Step kTrunk = dgrad::step(dgrad::L7T), kRgbT = vdgrad::step(vdgrad::RgbT), kViewsFT = vdgrad::step(vdgrad::ViewsFT);
  static_assert(kRgbT.nslabs == 1 && kRgbT.k16 == 1 && kViewsFT.N == kTrunk.N && kVgYv.chunks == 2 * kViewsFT.nslabs * kViewsFT.k16 &&
                dgrad::step(dgrad::HeadT).N == kTrunk.N && dgrad::step(dgrad::HeadT).k16 == 1 && kGsRaw.chunks == 2,
                "Rgb^T and head^T: one K = 16 MMA on the d_raw fragment; ViewsF^T: K = the 128 columns of dYv");
  for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
    uint8_t* gs = p.gstash + static_cast<long long>(tile) * kGradTileBytes;
    uint8_t* vgs = v.vgstash + static_cast<long long>(tile) * kVGradTileBytes;
    const uint8_t* mk = p.relu_mask + static_cast<long long>(tile) * kMaskTileBytes;
    uint32_t h[kMaskHCols / 16][4];
    // ---- A = d_raw [g_r g_g g_b g_alpha 0 ...] (K = 16) ----
    uint32_t a[1][4];
    d_raw_frag(p, tile, scale, gs, g, a);
    uint32_t dyv[kVgYv.chunks / 2][4];
    {   // ---- Rgb^T: dhv = d_raw . rgb_linear (channel 3 meets a zero column) -> dYv = dhv * [hv > 0] ----
      Acc<vdgrad::RgbT> acc;
      ReluMask<kMkHv.cols> m;
      m.load(v.hv_mask + static_cast<long long>(tile) * kHvMaskTileBytes, g);
      wg_gemm_rs<kRgbT.N, 1>(acc, a, ring, false, 0u, W, 320);
      epi_grad_frag<kMkHv.cols, true>(acc, m, dyv, vgs + kVgYv.off, g);
    }
    {   // ---- ViewsF^T: dF = dYv . views_linears.0[:, :256] (feature_linear has no ReLU) ----
      Acc<vdgrad::ViewsFT> acc;
      wg_gemm_rs<kViewsFT.N, kViewsFT.k16>(acc, dyv, ring, false, 0u, W, 321);
      epi_grad_frag<kMaskHCols, false>(acc, ReluMask<kMaskHCols>{}, h, vgs + kVgF.off, g);
    }
    {   // ---- Feature^T + head^T into one accumulator: dh8 = dF . feature_linear + d_alpha alpha_linear -> dY7 ----
      Acc<vdgrad::FeatureT> acc;
      ReluMask<kMaskHCols> m;
      m.load(mk + kMkH + 7 * kMaskHBytes, g);
      wg_gemm_rs<kTrunk.N, kTrunk.k16>(acc, h, ring, false, 0u, W, 322);
      wg_gemm_rs<kTrunk.N, 1, 1, true>(acc, a, ring, false, 0u, W, 300);
      epi_grad_frag<kMaskHCols, true>(acc, m, h, gs + kGsY + 7 * kHBytes, g);
    }
    // ---- L7^T, L6^T : dY6, dY5; then L5h^T, L4^T .. L1^T : dY4 .. dY0 (one shape) ----
#pragma unroll 1
    for (int s = 0; s < 7; ++s) {
      const int l = 6 - s;   // dY_l = dh_{l+1} * [h_{l+1} > 0]: dY6, dY5 (L7^T, L6^T), dY4 .. dY0 (L5h^T, L4^T .. L1^T)
      Acc<dgrad::L7T> acc;
      ReluMask<kMaskHCols> m;
      m.load(mk + kMkH + l * kMaskHBytes, g);
      wg_gemm_rs<kTrunk.N, kTrunk.k16>(acc, h, ring, false, 0u, W, 301 + s);
      epi_grad_frag<kMaskHCols, true>(acc, m, h, gs + kGsY + l * kHBytes, g);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Time-conditioned baseline: the latent enters L0 and L5 as a per-ray bias (field_fwd.cu), so its gradients are per-ray
// sums of those layers' pre-activation gradients dY0, dY5 (gradient stash):
//   s_l[ray] = sum over the ray's samples of dY_l,   d z[ray] = W0[:, 63:95]^T s_0 + W5[:, 63:95]^T s_5,
//   dW_l[:, 63:95] = sum over rays of s_l[ray] (x) z[ray].
// Every sum runs in a fixed order (samples, output features, rays), so the results are bit-reproducible.
namespace {
constexpr int kTcSumRays = 4;   // rays per block of tc_ray_sums_kernel: 64 threads = 2 layers x 32 column chunks each
constexpr int kTcDzRays = 8;    // rays per block of tc_dz_kernel: 32 threads (latent dims) each

// thread = (ray, layer, 8-column chunk): one 16-byte row piece of the chunk-major dY image per sample
__global__ void __launch_bounds__(256) tc_ray_sums_kernel(const TcBwdParams p) {
  const int ray = blockIdx.x * kTcSumRays + threadIdx.x / 64;
  const int l = (threadIdx.x / 32) & 1, c = threadIdx.x & 31;
  if (ray >= p.n_rays) return;
  const float inv_scale = 1.0f / loss_scale(p.amax);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  const uint8_t* base = p.gstash + kGsY + (l ? 5 : 0) * kHBytes + c * kChunkBytes;
  for (int s = 0; s < p.S; ++s) {
    const long long pt = static_cast<long long>(ray) * p.S + s;
    const uint4 w = __ldg(reinterpret_cast<const uint4*>(base + (pt / kTileM) * kGradTileBytes + (pt % kTileM) * 16));
    const uint32_t wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      acc[2 * q] += h_lo(wv[q]);
      acc[2 * q + 1] += h_hi(wv[q]);
    }
  }
  float* dst = p.sums + static_cast<long long>(ray) * 512 + l * 256 + c * 8;
#pragma unroll
  for (int e = 0; e < 8; ++e) dst[e] = acc[e] * inv_scale;
}

// thread = (ray, latent dim k): d z[ray][k] over the 256 outputs of both layers
__global__ void __launch_bounds__(256) tc_dz_kernel(const TcBwdParams p) {
  const int ray = blockIdx.x * kTcDzRays + threadIdx.x / 32, k = threadIdx.x & 31;
  if (ray >= p.n_rays) return;
  const float* s = p.sums + static_cast<long long>(ray) * 512;
  float d = 0.f;
#pragma unroll 4
  for (int o = 0; o < 256; ++o) {
    d = fmaf(__ldg(p.w0 + o * (kPeCols + kLatent) + kPeCols + k), __ldg(s + o), d);
    d = fmaf(__ldg(p.w5 + o * (kPeCols + kLatent + 256) + kPeCols + k), __ldg(s + 256 + o), d);
  }
  p.d_latents[static_cast<long long>(ray) * kLatent + k] = d;
}

// thread = (layer, latent dim k, output o): dW_l[o][63 + k] over the rays (o fastest: coalesced reads of the sums)
__global__ void __launch_bounds__(256) tc_dw_lat_kernel(const TcBwdParams p) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= 2 * kLatent * 256) return;
  const int o = idx & 255, k = (idx >> 8) & (kLatent - 1), l = idx >> 13;
  const float* s = p.sums + l * 256 + o;
  const float* z = p.latents + k;
  float a = 0.f;
#pragma unroll 8
  for (int r = 0; r < p.n_rays; ++r) a = fmaf(__ldg(s + static_cast<long long>(r) * 512), __ldg(z + r * p.latent_stride), a);
  p.dw_lat[(l * 256 + o) * kLatent + k] = a;
}
}  // namespace

cudaError_t launch_field_bwd(const FieldBwdParams& p, bool has_bender, int num_sms, cudaStream_t stream) {
  return launch_field(has_bender ? field_bwd_kernel<true> : field_bwd_kernel<false>, p, num_sms, kBwdSmemBytes, stream);
}

cudaError_t launch_field_bwd_det(const FieldBwdParams& p, float* latent_rows, int num_sms, cudaStream_t stream) {
  return launch_field(field_bwd_det_kernel, p, num_sms, kBwdSmemBytes, stream, latent_rows);
}

cudaError_t launch_field_bwd_held(const FieldBwdParams& p, float* latent_rows, const uint8_t* held, int num_sms, cudaStream_t stream) {
  if (latent_rows) return launch_field(field_bwd_held_kernel<true>, p, num_sms, kBwdSmemBytes, stream, latent_rows, held);
  return launch_field(field_bwd_held_kernel<false>, p, num_sms, kBwdSmemBytes, stream, latent_rows, held);
}

cudaError_t launch_field_bwd_views(const FieldBwdParams& p, const ViewBwdParams& v, int num_sms, cudaStream_t stream) {
  return launch_field(field_bwd_views_kernel, p, num_sms, kBwdSmemBytes, stream, v);
}

cudaError_t launch_tc_latent_bwd(const TcBwdParams& p, cudaStream_t stream) {
  if (p.n_rays <= 0) return cudaSuccess;
  tc_ray_sums_kernel<<<(p.n_rays + kTcSumRays - 1) / kTcSumRays, 64 * kTcSumRays, 0, stream>>>(p);
  tc_dz_kernel<<<(p.n_rays + kTcDzRays - 1) / kTcDzRays, 32 * kTcDzRays, 0, stream>>>(p);
  tc_dw_lat_kernel<<<2 * kLatent * 256 / 256, 256, 0, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace nrn
