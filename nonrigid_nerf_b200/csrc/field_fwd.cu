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
//   a "step" = one dense layer:  D[64 x N] (registers, fp32) = A[64 x K] (fp16) . W[N x K]^T (smem ring,
//            fp16) with wgmma; the same warpgroup then applies bias/ReLU/(bend + positional encoding) and writes
//            the next A operand.  B0..B4, L0 and the embedding slab of L5 read A from shared memory; L1..L7 and the
//            head take it from registers: the fp16 fragments the previous trunk epilogue packed (wg_gemm_rs), which
//            the training kernel also stores to the stash from registers.
//   steps  : B0..B4 (ray bender, offset + rigidity MLPs fused block-diagonally), L0..L7, head
//
// Shared memory (per CTA): bender H 24 KB + E 16 KB activations, 5 x 32 KB weight ring, per-row staging, barriers.
//
// View-dependent head (NeRF(use_viewdirs=True)), three more instantiations of the same body:
//   bend pass (with a bender): B0..B4 only; every point's bent xyz and rigidity -> the bend workspace (16 B / point)
//   view-head kernel: points from the workspace (or, without a bender, from rays + z), L0..L7, Head (alpha in column 3),
//            Feature, ViewsE + ViewsF (one N = 128 accumulator), Rgb.  The direction of point r is the normalised
//            backward difference of the bent points r - 1 and r of its ray (r + 1 and r for sample 0), read from the
//            workspace in global memory, so it does not matter which tile or CTA owns the neighbour.  No bender H
//            buffer: 24 KB less shared memory than the other kernels.
//   view-head training kernel (no bender): the view-head kernel that also writes the trunk's stash and masks, the view
//            stash (direction encoding, feature, hv) and hv's mask bits for field_bwd_views_kernel.
//
// Baked radiance grid (render(..., baked=)): the bend pass that also looks every bent point up in the grid (baked.cuh)
// and writes raw of the points inside its box; the trunk runs afterwards on the others alone (c_abi.cu).  With a baked
// deformation grid as well, the bend pass runs only on the rays that fall back to the exact bender, gathered, with their
// count read on the device.
#include "baked.cuh"
#include "field_epilogue.cuh"

namespace nrn {

namespace {

// Direction encoding of the view-dependent head (embeddirs_fn, get_embedder(multires_views = 4): d, then sin(2^k d),
// cos(2^k d) for k = 0..3, the same turn reduction as write_pe) as fp16 chunks 0..3 of the row: 27 columns + 5 zero.
__device__ __forceinline__ void write_dir_enc(const float (&d)[3], uint8_t* dst_row) {
  float f[32];
  encode_octaves<4>(d, f);
#pragma unroll
  for (int i = views::kDirCols; i < 32; ++i) f[i] = 0.f;
  pack_row(f, dst_row);
}

static_assert(views::step(views::Feature) == fwd::step(fwd::L1), "step_at_views: Feature has the trunk's shape");
// step -> shape in the view-head kernel's streaming order L0..Head, Feature..Rgb
__device__ __forceinline__ Step step_at_views(int step) {
  switch (step) {
    case fwd::L0: return step_imm<fwd::L0>();
    case fwd::L5: return step_imm<fwd::L5>();
    case fwd::Head: return step_imm<fwd::Head>();
    case views::ViewsE: return step_imm<views::ViewsE>();
    case views::ViewsF: return step_imm<views::ViewsF>();
    case views::Rgb: return step_imm<views::Rgb>();
    default: return step_imm<fwd::L1>();   // L1-L4, L6, L7, Feature
  }
}

// Which part of the forward a kernel runs: all of it, the bend pass of the view-dependent head, its view-head kernel, or
// the bend pass with the baked grid's lookup
enum Part : int { kFull, kBend, kViews, kBaked };

}  // namespace

// TRAIN: p.stash and p.relu_mask are given (the inference kernel carries none of the mask code).
// LATENT_BIAS (time-conditioned baseline, no bender): the L0 and L5 epilogues add the ray-bias rows p.ray_bias of their
// rows' rays instead of the layers' bias vectors.
// PART (view-dependent head): kBend runs B0..B4 and writes v.ws; kViews (HAS_BENDER false) runs the trunk and the view
// head, reading its points and rigidities from v.ws when that is given.  kViews with TRAIN (no bender, v.ws null): the
// trunk's stash and masks as the full kernel writes them, and the view stash and Hv masks of t.
// kBaked (with a bender, inference): kBend, and each point inside the box of the grid bg gets raw from bg's lookup.
template <bool HAS_BENDER, bool TRAIN, bool LATENT_BIAS, int PART = kFull>
__device__ __forceinline__ void field_fwd_body(const FieldFwdParams& p, const ViewParams& v = ViewParams{},
                                               const ViewTrainParams& t = ViewTrainParams{}, const BakedGrid& bg = BakedGrid{}) {
  static_assert(!(HAS_BENDER && LATENT_BIAS), "the time-conditioned baseline has no bender");
  static_assert(PART == kFull || (!LATENT_BIAS && (PART == kBend || PART == kBaked) == HAS_BENDER && (!TRAIN || PART == kViews)),
                "bend and view-head parts: inference, or training of the view-head kernel without a bender");
  constexpr int kHBytes = PART == kViews ? 0 : kFwdHBytes;   // the view-head kernel has no bender images
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* act = smem;                                  // H (bender) | E, 128 rows
  uint8_t* ring_buf = smem + kHBytes + kEBytes;         // kFwdRingStages x 32 KB
  float* stage_all = reinterpret_cast<float*>(ring_buf + kFwdRingStages * kRingStageBytes);   // 2 x 64 rows x kFwdStageLd
  auto* sh = reinterpret_cast<RingShared<kFwdRingStages>*>(stage_all + 2 * kWgRows * kFwdStageLd);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) sh->init();
  __syncthreads();
  const Waiter W{&sh->abort_flag, p.err};
  Ring<kFwdRingStages> ring{ring_buf, sh->w_full, sh->w_empty};

  if (warp >= 8) {
    setmaxnreg_dec<kProducerRegs>();
    // ===================== weight producer: global -> smem ring (bulk TMA) =====================
    if (warp == 8 && lane == 0) {
      if constexpr (PART == kViews) produce(p.nerf_w, v.w, p.n_tiles, fwd::L0, views::kEnd, views::Feature, step_at_views, ring, W);
      else produce(p.bend_w, p.nerf_w, p.n_tiles, HAS_BENDER ? fwd::B0 : fwd::L0, PART == kBend || PART == kBaked ? fwd::L0 : fwd::kCount, fwd::L0,
                   fwd_step_at, ring, W);
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
    // Training stash: every finished activation image goes to this tile's stash block
    uint8_t* st = p.stash ? p.stash + static_cast<long long>(tile) * kStashTileBytes : nullptr;
    const StashWriter<true> sw{st, wg_leader, bar, g};
    // ReLU masks for DGRAD (training): every row of the tile is written, those past P of a ragged last tile included
    uint8_t* mk = TRAIN ? p.relu_mask + static_cast<long long>(tile) * kMaskTileBytes : nullptr;
    float x[3] = {0.f, 0.f, 0.f};
    long long ray = 0;
    if (valid) {
      ray = pt / p.S;
      if (PART == kViews && v.ws) {
        // bent point of the bend pass, and the view direction: the normalised backward difference along the ray
        // (run_nerf_helpers.py:316-356, difference_type "backward"; sample 0 takes sample 1's)
        const float4 q = __ldg(v.ws + pt);
        const bool first = pt % p.S == 0;
        const float4 o = __ldg(v.ws + (first ? pt + 1 : pt - 1));
        x[0] = q.x; x[1] = q.y; x[2] = q.z;
        const float dx = first ? o.x - q.x : q.x - o.x, dy = first ? o.y - q.y : q.y - o.y, dz = first ? o.z - q.z : q.z - o.z;
        const float nrm = __fadd_rn(__fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz))), 1e-6f);
        my_stg[8] = __fdiv_rn(dx, nrm); my_stg[9] = __fdiv_rn(dy, nrm); my_stg[10] = __fdiv_rn(dz, nrm);
        my_stg[11] = q.w;   // rigidity, for the object removal
      } else if (p.pts) {
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
      if (PART == kViews && !v.ws) {   // no bender: the given direction (ray mode: the ray's, point mode: the point's)
        const float* vd = v.viewdirs + (p.pts ? pt : ray) * v.viewdirs_stride;
        my_stg[8] = __ldg(vd + 0); my_stg[9] = __ldg(vd + 1); my_stg[10] = __ldg(vd + 2);
      }
      if (p.d_init) {
        p.d_init[pt * 3 + 0] = x[0]; p.d_init[pt * 3 + 1] = x[1]; p.d_init[pt * 3 + 2] = x[2];
      }
    }
    float rigidity = 0.f;
    if (HAS_BENDER) {
      // ---- bender input row: [xyz_hi(3) xyz_lo(3) latent(32) 0(10)] fp16, chunks 0..5 of E ----
      sw.begin();
      if (row_thread) write_bender_input(x, p.latents + ray * p.latent_stride, valid, e_row);
      sw.ready(kStBin, Es);
      // ---- B0, B1: 96 hidden units (64 offset | 32 rigidity) ----
      {
        Acc<fwd::B0> acc;
        wg_gemm_step<fwd::B0>(acc, ring, [&](uint32_t) { return a_e; }, W, 301);
        sw.begin();
        epi_bias_relu_store<kMkHb1.cols, TRAIN>(acc, p.bend_bias + fwd::b_off(fwd::B0), Hs, g, mk, kMkHb1.off);
        sw.ready(kStHb1, Hs);
        wg_gemm_step<fwd::B1>(acc, ring, [&](uint32_t) { return a_h; }, W, 302);
        sw.begin();
        epi_bias_relu_store<kMkHb2.cols, TRAIN>(acc, p.bend_bias + fwd::b_off(fwd::B1), Hs, g, mk, kMkHb2.off);
        sw.ready(kStHb2, Hs);
      }
      // ---- B2: 64 offset hidden + rigidity output (column 64) ----
      {
        Acc<fwd::B2> acc;
        wg_gemm_step<fwd::B2>(acc, ring, [&](uint32_t) { return a_h; }, W, 303);
        sw.begin();
        epi_bias_relu_store<kMkHb3.cols, TRAIN>(acc, p.bend_bias + fwd::b_off(fwd::B2), Hs, g, mk, kMkHb3.off);
        if (acc_q() == 0) {
          stg[acc_r0() * kFwdStageLd] = acc[32];
          stg[(acc_r0() + 8) * kFwdStageLd] = acc[34];
        }
        sw.ready(kStHb3, Hs);
        if (row_thread) {
          const float rr = my_stg[0] + __ldg(p.bend_bias + fwd::b_off(fwd::B2) + 64);
          rigidity = (tanhf(rr) + 1.0f) * 0.5f;   // run_nerf_helpers.py:559-561
          if (p.use_cutoff && rigidity <= p.cutoff) rigidity = 0.f;  // :563-564
        }
      }
      // ---- B3 ----
      {
        Acc<fwd::B3> acc;
        wg_gemm_step<fwd::B3>(acc, ring, [&](uint32_t) { return a_h; }, W, 304);
        sw.begin();
        epi_bias_relu_store<kMkHb4.cols, TRAIN>(acc, p.bend_bias + fwd::b_off(fwd::B3), Hs, g, mk, kMkHb4.off);
        sw.ready(kStHb4, Hs);
      }
      // ---- B4: offsets; bend ----
      {
        Acc<fwd::B4> acc;
        wg_gemm_step<fwd::B4>(acc, ring, [&](uint32_t) { return a_h; }, W, 305);
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
    if constexpr (PART == kBend || PART == kBaked) {   // the bend pass ends here: bent point and rigidity -> the workspace
      if (valid) v.ws[pt] = make_float4(x[0], x[1], x[2], rigidity);
      // the baked grid: raw of a point inside its box, the object removal applied as the head below applies it
      if constexpr (PART == kBaked)
        if (valid) baked_raw(bg, x, p.use_removal && rigidity >= p.removal, p.raw, pt, p.out_ch);
      continue;
    }
    // ---- positional encoding of the (bent) point -> E ----
    sw.begin();
    if (row_thread) write_pe(x, e_row);
    sw.ready(kStE, Es);
    // ---- L0 .. L7 (every one 256 wide): L0 reads E, every later step its A fragments h (L5: E first, then h) ----
    uint32_t h[kMaskHCols / 16][4];
    // LATENT_BIAS: the rays of this thread's accumulator rows r0 and r0 + 8 (rows past P take the last point's)
    int ray_r0 = 0, ray_r8 = 0;
    if constexpr (LATENT_BIAS) {
      const long long r0 = static_cast<long long>(tile) * kTileM + g * kWgRows + acc_r0();
      ray_r0 = static_cast<int>(min(r0, p.P - 1) / p.S);
      ray_r8 = static_cast<int>(min(r0 + 8, p.P - 1) / p.S);
    }
#pragma unroll 1
    for (int L = 0; L < 8; ++L) {
      Acc<fwd::L1> acc;
      if (L == 0) wg_gemm_step<fwd::L0>(acc, ring, [&](uint32_t) { return a_e; }, W, 310);
      else wg_gemm_rs<fwd::step(fwd::L1).N, fwd::step(fwd::L1).k16>(acc, h, ring, L == 5, a_e, W, 310 + L);
      if (LATENT_BIAS && (L == 0 || L == 5)) {
        const float* rb = p.ray_bias + (L == 5 ? fwd::b_off(fwd::L1) : 0);
        epi_bias_frag<kMaskHCols, true, TRAIN, true>(acc, rb + ray_r0 * p.ray_bias_stride, h, st + st_h(L + 1).off, g,
                                                     mk + kMkH + L * kMaskHBytes, rb + ray_r8 * p.ray_bias_stride);
      } else {
        epi_bias_frag<kMaskHCols, true, TRAIN>(acc, p.nerf_bias + L * fwd::b_off(fwd::L1), h, st + st_h(L + 1).off, g,
                                               mk + kMkH + L * kMaskHBytes);
      }
    }
    if constexpr (PART == kViews) {
      // training: the view stash of this tile (Dir by bulk store from E, F and Hv from registers) and its Hv masks
      uint8_t* vst = TRAIN ? t.vstash + static_cast<long long>(tile) * kVStashTileBytes : nullptr;
      const StashWriter<true> vsw{vst, wg_leader, bar, g};
      // ---- Head: alpha = alpha_linear(h) in column 3 (run_nerf_helpers.py:285) ----
      {
        Acc<fwd::Head> acc;
        wg_gemm_rs<fwd::step(fwd::Head).N, fwd::step(fwd::Head).k16>(acc, h, ring, false, 0u, W, 320);
        stage_cols<0, 1>(acc, stg, kFwdStageLd);
        // also: every warp of this warpgroup is past L5, the last reader of E; training: the bulk store of E to the stash
        // has finished reading it before the direction encoding overwrites it
        if constexpr (TRAIN) sw.begin();
        else wg_bar(bar);
        if (row_thread) {
          float alpha = my_stg[3] + __ldg(p.nerf_bias + fwd::b_off(fwd::Head) + 3);
          // test-time non-rigid object removal (run_nerf_helpers.py:309-310)
          if (v.ws && p.use_removal && my_stg[11] >= p.removal) alpha *= 0.f;
          // training: rows past P (ragged last tile) never staged a direction; they encode d = 0, so that their stashed
          // Dir and Hv rows are finite (WGRAD multiplies them by their zero gradients)
          const bool dir_ok = !TRAIN || valid;
          const float d[3] = {dir_ok ? my_stg[8] : 0.f, dir_ok ? my_stg[9] : 0.f, dir_ok ? my_stg[10] : 0.f};
          my_stg[11] = alpha;
          write_dir_enc(d, e_row);   // the direction encoding -> E, the A operand of ViewsE
        }
      }
      // ---- Feature: feature_linear(h), no ReLU (run_nerf_helpers.py:286); the result replaces h as the A fragments ----
      {
        Acc<views::Feature> acc;
        wg_gemm_rs<views::step(views::Feature).N, views::step(views::Feature).k16>(acc, h, ring, false, 0u, W, 330);
        epi_bias_frag<256, false, TRAIN>(acc, v.bias + views::b_off(views::Feature), h, TRAIN ? vst + kVsF.off : nullptr, g);
      }
      // the direction encoding is visible to the tensor cores (training: and goes to the view stash)
      if constexpr (TRAIN) {
        vsw.ready(kVsDir, Es);
      } else {
        fence_proxy_async_smem();
        wg_bar(bar);
      }
      // ---- views_linears.0 on cat[feature, dirs]: ViewsE (E) then ViewsF (feature fragments), bias + ReLU ----
      uint32_t hv[8][4];
      {
        Acc<views::ViewsF> acc;
        wg_gemm_rs<views::step(views::ViewsF).N, views::step(views::ViewsF).k16, views::step(views::ViewsE).k16>(acc, h, ring, true, a_e, W, 331);
        epi_bias_frag<128, true, TRAIN>(acc, v.bias + views::b_off(views::ViewsF), hv, TRAIN ? vst + kVsHv.off : nullptr, g,
                                        TRAIN ? t.hv_mask + static_cast<long long>(tile) * kHvMaskTileBytes : nullptr);
      }
      // ---- Rgb: rgb_linear(hv); raw = [rgb, alpha] (run_nerf_helpers.py:303-304) ----
      {
        Acc<views::Rgb> acc;
        wg_gemm_rs<views::step(views::Rgb).N, views::step(views::Rgb).k16>(acc, hv, ring, false, 0u, W, 332);
        stage_cols<0, 1>(acc, stg, kFwdStageLd);
        wg_bar(bar);
        if (valid) {
          float* dst = p.raw + pt * 4;
#pragma unroll
          for (int c = 0; c < 3; ++c) dst[c] = my_stg[c] + __ldg(v.bias + views::b_off(views::Rgb) + c);
          dst[3] = my_stg[11];
        }
      }
      continue;
    }
    // ---- head: raw = output_linear(h) (run_nerf_helpers.py:306) ----
    {
      Acc<fwd::Head> acc;
      wg_gemm_rs<fwd::step(fwd::Head).N, fwd::step(fwd::Head).k16>(acc, h, ring, false, 0u, W, 320);
      stage_cols<0, 1>(acc, stg, kFwdStageLd);
      wg_bar(bar);
      if (valid) {
        float o[5];
#pragma unroll
        for (int c = 0; c < 5; ++c) o[c] = my_stg[c] + __ldg(p.nerf_bias + fwd::b_off(fwd::Head) + c);
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

template <bool HAS_BENDER, bool TRAIN>
__global__ void __launch_bounds__(kFwdThreads, 1) field_fwd_kernel(const FieldFwdParams p) { field_fwd_body<HAS_BENDER, TRAIN, false>(p); }
template <bool TRAIN>
__global__ void __launch_bounds__(kFwdThreads, 1) field_fwd_tc_kernel(const FieldFwdParams p) { field_fwd_body<false, TRAIN, true>(p); }
__global__ void __launch_bounds__(kFwdThreads, 1) field_bend_kernel(const FieldFwdParams p, const ViewParams v) {
  field_fwd_body<true, false, false, kBend>(p, v);
}
__global__ void __launch_bounds__(kFwdThreads, 1) field_views_kernel(const FieldFwdParams p, const ViewParams v) {
  field_fwd_body<false, false, false, kViews>(p, v);
}
__global__ void __launch_bounds__(kFwdThreads, 1) field_baked_kernel(const FieldFwdParams p, const ViewParams v, const BakedGrid g) {
  field_fwd_body<true, false, false, kBaked>(p, v, ViewTrainParams{}, g);
}
// The point-mode trunk (no bender) over the points an occupancy lookup kept (occupancy.cu): their count is read from device
// memory, so a render pass that skips empty space needs no host synchronisation and can be captured in a CUDA graph
__global__ void __launch_bounds__(kFwdThreads, 1) field_fwd_kept_kernel(FieldFwdParams p, const int* __restrict__ kept) {
  p.P = *kept;
  p.n_rays = static_cast<int>(p.P);
  p.n_tiles = static_cast<int>((p.P + kTileM - 1) / kTileM);
  field_fwd_body<false, false, false>(p);
}
// The bend pass over rays whose count is read from device memory (the fallback rays of a pass with a baked deformation
// grid, baked.cu): no host synchronisation, so such a pass can be captured in a CUDA graph
__global__ void __launch_bounds__(kFwdThreads, 1) field_bend_rays_kernel(FieldFwdParams p, const ViewParams v, const int* __restrict__ n_rays) {
  p.n_rays = *n_rays;
  p.P = static_cast<long long>(p.n_rays) * p.S;
  p.n_tiles = static_cast<int>((p.P + kTileM - 1) / kTileM);
  field_fwd_body<true, false, false, kBend>(p, v);
}
__global__ void __launch_bounds__(kFwdThreads, 1) field_views_train_kernel(const FieldFwdParams p, const ViewParams v, const ViewTrainParams t) {
  field_fwd_body<false, true, false, kViews>(p, v, t);
}

// Ray bias of the time-conditioned baseline: rb[n][l][o] = b_l[o] + sum_k W_l[o][63 + k] z[n][k] for l = L0, L5, in fp32
// from the nn.Linear weights (W0 [256][95], W5 [256][351]).  Thread o of a block keeps both layers' 32 latent weights
// of row o in registers and walks kTcRaysPerBlock rays.
constexpr int kTcRaysPerBlock = 16;
__global__ void __launch_bounds__(256) tc_latent_bias_kernel(const float* __restrict__ lat, long long lat_stride, int n_rays,
                                                             const float* __restrict__ w0, const float* __restrict__ b0,
                                                             const float* __restrict__ w5, const float* __restrict__ b5,
                                                             float* __restrict__ rb) {
  __shared__ float zs[kTcRaysPerBlock][kLatent];
  const int o = threadIdx.x;
  const int n0 = blockIdx.x * kTcRaysPerBlock;
  for (int i = threadIdx.x; i < kTcRaysPerBlock * kLatent; i += blockDim.x) {
    const int r = n0 + i / kLatent;
    zs[i / kLatent][i % kLatent] = r < n_rays ? __ldg(lat + r * lat_stride + i % kLatent) : 0.f;
  }
  float wa[kLatent], wb[kLatent];
#pragma unroll
  for (int k = 0; k < kLatent; ++k) {
    wa[k] = __ldg(w0 + o * (kPeCols + kLatent) + kPeCols + k);
    wb[k] = __ldg(w5 + o * (kPeCols + kLatent + 256) + kPeCols + k);
  }
  const float ba = __ldg(b0 + o), bb = __ldg(b5 + o);
  __syncthreads();
  for (int i = 0; i < kTcRaysPerBlock && n0 + i < n_rays; ++i) {
    float sa = 0.f, sb = 0.f;
#pragma unroll
    for (int k = 0; k < kLatent; ++k) {
      sa = fmaf(wa[k], zs[i][k], sa);
      sb = fmaf(wb[k], zs[i][k], sb);
    }
    float* dst = rb + static_cast<long long>(n0 + i) * 512;
    dst[o] = ba + sa;
    dst[256 + o] = bb + sb;
  }
}

// ------------------------------------------------------------------------------------------------
size_t field_fwd_smem_bytes() { return kFwdSmemBytes; }

cudaError_t launch_field_fwd(const FieldFwdParams& p, bool has_bender, int num_sms, cudaStream_t stream) {
  const size_t smem = field_fwd_smem_bytes();
  const bool train = p.relu_mask != nullptr;   // the C ABI passes the ReLU masks exactly when it passes the stash
  if (has_bender) return launch_field(train ? field_fwd_kernel<true, true> : field_fwd_kernel<true, false>, p, num_sms, smem, stream);
  return launch_field(train ? field_fwd_kernel<false, true> : field_fwd_kernel<false, false>, p, num_sms, smem, stream);
}

// The view-dependent head: with a bender the bend pass (-> v.ws) runs first, then the view-head kernel (c_abi.cu)
size_t field_views_smem_bytes() { return kFwdSmemBytes - kFwdHBytes; }

cudaError_t launch_field_bend(const FieldFwdParams& p, const ViewParams& v, int num_sms, cudaStream_t stream) {
  return launch_field(field_bend_kernel, p, num_sms, field_fwd_smem_bytes(), stream, v);
}

// The bend pass with the baked grid's lookup: v.ws as launch_field_bend writes it, and p.raw of the points inside g's box
cudaError_t launch_field_baked(const FieldFwdParams& p, const ViewParams& v, const BakedGrid& g, int num_sms, cudaStream_t stream) {
  return launch_field(field_baked_kernel, p, num_sms, field_fwd_smem_bytes(), stream, v, g);
}

// p.n_rays (and p.P, p.n_tiles) bound the ray count: they size the grid; the kernel takes the count itself from `n_rays`
cudaError_t launch_field_bend_rays(const FieldFwdParams& p, const ViewParams& v, const int* n_rays, int num_sms, cudaStream_t stream) {
  return launch_field(field_bend_rays_kernel, p, num_sms, field_fwd_smem_bytes(), stream, v, n_rays);
}

cudaError_t launch_field_views(const FieldFwdParams& p, const ViewParams& v, int num_sms, cudaStream_t stream) {
  return launch_field(field_views_kernel, p, num_sms, field_views_smem_bytes(), stream, v);
}

// Training the view-dependent head without a bender: p.stash / p.relu_mask and t's buffers are written
cudaError_t launch_field_views_train(const FieldFwdParams& p, const ViewParams& v, const ViewTrainParams& t, int num_sms, cudaStream_t stream) {
  return launch_field(field_views_train_kernel, p, num_sms, field_views_smem_bytes(), stream, v, t);
}

// p.P (and p.n_tiles) bound the kept count: they size the grid; the kernel takes the count itself from `kept`
cudaError_t launch_field_fwd_kept(const FieldFwdParams& p, const int* kept, int num_sms, cudaStream_t stream) {
  return launch_field(field_fwd_kept_kernel, p, num_sms, field_fwd_smem_bytes(), stream, kept);
}

cudaError_t launch_field_fwd_tc(const FieldFwdParams& p, int num_sms, cudaStream_t stream) {
  const bool train = p.relu_mask != nullptr;
  return launch_field(train ? field_fwd_tc_kernel<true> : field_fwd_tc_kernel<false>, p, num_sms, field_fwd_smem_bytes(), stream);
}

cudaError_t launch_tc_latent_bias(const float* lat, long long lat_stride, int n_rays, const float* w0, const float* b0, const float* w5,
                                  const float* b5, float* rb, cudaStream_t stream) {
  tc_latent_bias_kernel<<<(n_rays + kTcRaysPerBlock - 1) / kTcRaysPerBlock, 256, 0, stream>>>(lat, lat_stride, n_rays, w0, b0, w5, b5, rb);
  return cudaGetLastError();
}

}  // namespace nrn
