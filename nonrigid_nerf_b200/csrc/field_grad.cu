// The density gradient at points: g = d raw[3] / d x of NeRF.forward in point mode (geometry.density_gradient).
//
// Two persistent kernels on the machine of the field kernels (field_mma.cuh), per chunk of points:
//   field_fwd_grad_kernel  the point-mode forward of field_fwd.cu (bender B0..B4, PE, L0..L7; time-conditioned L0 / L5
//                          take ray-bias rows) writing only what the DGRAD chain reads: every ReLU mask bit (kMaskTileBytes
//                          per tile), the positional encoding E (kEBytes per tile) and the bender's unmasked offsets and
//                          rigidity.  No other activation image is stored, and the head is not run.
//   field_bwd_grad_kernel  the DGRAD chain of field_bwd.cu for d raw = e_3 at every point: head^T .. L0^T with two
//                          positional-encoding backwards into dx = d raw[3] / d bent, then (bender) the bend backward and
//                          B4^T .. B0^T, whose xyz columns add (d bent / d x)^T dx.  No gradient stash, no WGRAD, no latent
//                          reduction.
// The kernels are their own bodies rather than flags of field_fwd_body / field_bwd_body, so that the training and
// inference kernels keep their machine code.  They share those bodies' layouts, step tables, encodings and epilogues
// (field_epilogue.cuh), so their mask bits and E are the training forward's.
#include "field_epilogue.cuh"

namespace nrn {

namespace {

// head^T's A operand: d raw = e_3 times the loss scale for every point of the tile, rows past P zero (lanes q = 1 hold
// columns 2, 3 of rows r0, r0 + 8)
__device__ __forceinline__ void sigma_frag(long long P, int tile, float scale, int g, uint32_t (&a)[1][4]) {
  const int r0 = g * kWgRows + acc_r0(), q = acc_q();
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const long long pti = static_cast<long long>(tile) * kTileM + r0 + 8 * i;
    a[0][i] = q == 1 && pti < P ? pack_h2(0.f, scale) : 0u;
    a[0][2 + i] = 0u;
  }
}

// The loss-scale source: |d raw| = 1, so every trunk gradient travels in fp16 at loss_scale(1) = 2^9
__device__ const float kUnitAmax = 1.0f;

// Power-of-two scale that puts a row's largest bender-chain input v in [512, 1024) (loss_scale's rule; 1 for 0 or a
// non-finite v).  The bender chain is linear and row-wise, so a per-row scale is exact and keeps d unmasked = r~ s dx
// clear of fp16 saturation and underflow whatever the size of dx.
__device__ __forceinline__ float row_scale(float v) {
  float scale = 1.0f;
  if (v > 0.f && v < 3.0e38f) {
    int e;
    frexpf(v, &e);
    scale = ldexpf(1.0f, min(max(10 - e, -60), 60));
  }
  return scale;
}

}  // namespace

// Point-mode forward: p.pts, p.latents (bender) / p.ray_bias (LATENT_BIAS), p.stash = E [n_tiles][kEBytes], p.relu_mask
// [n_tiles][kMaskTileBytes], with a bender p.d_unmasked [P][3] and p.d_rigid [P] (rigidity after the cutoff).
template <bool HAS_BENDER, bool LATENT_BIAS>
__global__ void __launch_bounds__(kFwdThreads, 1) field_fwd_grad_kernel(const FieldFwdParams p) {
  static_assert(!(HAS_BENDER && LATENT_BIAS), "the time-conditioned baseline has no bender");
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* act = smem;
  uint8_t* ring_buf = smem + kFwdHBytes + kEBytes;
  float* stage_all = reinterpret_cast<float*>(ring_buf + kFwdRingStages * kRingStageBytes);
  auto* sh = reinterpret_cast<RingShared<kFwdRingStages>*>(stage_all + 2 * kWgRows * kFwdStageLd);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) sh->init();
  __syncthreads();
  const Waiter W{&sh->abort_flag, p.err};
  Ring<kFwdRingStages> ring{ring_buf, sh->w_full, sh->w_empty};

  if (warp >= 8) {
    setmaxnreg_dec<kProducerRegs>();
    // B0..B4 (bender), L0..L7: the head's weights are not streamed
    if (warp == 8 && lane == 0) produce(p.bend_w, p.nerf_w, p.n_tiles, HAS_BENDER ? fwd::B0 : fwd::L0, fwd::Head, fwd::L0, fwd_step_at, ring, W);
    return;
  }

  setmaxnreg_inc<kConsumerRegs>();
  const int g = warp >> 2;
  const int tw = threadIdx.x & 127;
  const bool row_thread = tw < kWgRows;
  const int bar = 1 + g;
  const bool wg_leader = tw == 0;
  uint8_t* Hs = act;
  uint8_t* Es = act + kFwdHBytes;
  uint8_t* e_row = Es + (g * kWgRows + tw) * 16;
  const uint32_t a_h = smem_u32(Hs) + g * kWgRows * 16;
  const uint32_t a_e = smem_u32(Es) + g * kWgRows * 16;
  float* stg = stage_all + g * kWgRows * kFwdStageLd;
  float* my_stg = stg + tw * kFwdStageLd;
  constexpr Image kNone{0, 0};   // a finished image that is not stored

  for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
    const long long pt = static_cast<long long>(tile) * kTileM + g * kWgRows + tw;
    const bool valid = row_thread && pt < p.P;
    // E alone goes to global memory (at offset kStE.off = 0 of its kEBytes block); the writer also orders every rewrite of
    // Es after the previous tile's store of it has read it
    const StashWriter<false> sw{p.stash + static_cast<long long>(tile) * kEBytes, wg_leader, bar, g};
    uint8_t* mk = p.relu_mask + static_cast<long long>(tile) * kMaskTileBytes;   // every row, those past P included
    float x[3] = {0.f, 0.f, 0.f};
    if (valid) {
      const float* q = p.pts + pt * p.pts_stride;
      x[0] = __ldg(q + 0); x[1] = __ldg(q + 1); x[2] = __ldg(q + 2);
    }
    if constexpr (HAS_BENDER) {
      // ---- bender input row [xyz_hi(3) xyz_lo(3) latent(32) 0(10)] -> E ----
      sw.begin();
      if (row_thread) write_bender_input(x, p.latents + pt * p.latent_stride, valid, e_row);
      sw.ready(kNone, Es);
      float rigidity = 0.f;
      {
        Acc<fwd::B0> acc;
        wg_gemm_step<fwd::B0>(acc, ring, [&](uint32_t) { return a_e; }, W, 401);
        sw.begin();
        epi_bias_relu_store<kMkHb1.cols, true>(acc, p.bend_bias + fwd::b_off(fwd::B0), Hs, g, mk, kMkHb1.off);
        sw.ready(kNone, Hs);
        wg_gemm_step<fwd::B1>(acc, ring, [&](uint32_t) { return a_h; }, W, 402);
        sw.begin();
        epi_bias_relu_store<kMkHb2.cols, true>(acc, p.bend_bias + fwd::b_off(fwd::B1), Hs, g, mk, kMkHb2.off);
        sw.ready(kNone, Hs);
      }
      {
        Acc<fwd::B2> acc;
        wg_gemm_step<fwd::B2>(acc, ring, [&](uint32_t) { return a_h; }, W, 403);
        sw.begin();
        epi_bias_relu_store<kMkHb3.cols, true>(acc, p.bend_bias + fwd::b_off(fwd::B2), Hs, g, mk, kMkHb3.off);
        if (acc_q() == 0) {
          stg[acc_r0() * kFwdStageLd] = acc[32];
          stg[(acc_r0() + 8) * kFwdStageLd] = acc[34];
        }
        sw.ready(kNone, Hs);
        if (row_thread) {
          const float rr = my_stg[0] + __ldg(p.bend_bias + fwd::b_off(fwd::B2) + 64);
          rigidity = (tanhf(rr) + 1.0f) * 0.5f;
          if (p.use_cutoff && rigidity <= p.cutoff) rigidity = 0.f;
        }
      }
      {
        Acc<fwd::B3> acc;
        wg_gemm_step<fwd::B3>(acc, ring, [&](uint32_t) { return a_h; }, W, 404);
        sw.begin();
        epi_bias_relu_store<kMkHb4.cols, true>(acc, p.bend_bias + fwd::b_off(fwd::B3), Hs, g, mk, kMkHb4.off);
        sw.ready(kNone, Hs);
      }
      {   // ---- B4: offsets; bend = x + rigidity * unmasked (* scaling), rounded as field_fwd.cu does ----
        Acc<fwd::B4> acc;
        wg_gemm_step<fwd::B4>(acc, ring, [&](uint32_t) { return a_h; }, W, 405);
        stage_cols<0, 1>(acc, stg, kFwdStageLd);
        wg_bar(bar);
        if (row_thread) {
          float un[3], ma[3];
#pragma unroll
          for (int d = 0; d < 3; ++d) {
            un[d] = my_stg[d];
            ma[d] = __fmul_rn(rigidity, un[d]);
            if (p.use_scaling) ma[d] = __fmul_rn(ma[d], p.scaling);
          }
          if (valid) {
            p.d_unmasked[pt * 3 + 0] = un[0]; p.d_unmasked[pt * 3 + 1] = un[1]; p.d_unmasked[pt * 3 + 2] = un[2];
            p.d_rigid[pt] = rigidity;
          }
#pragma unroll
          for (int d = 0; d < 3; ++d) x[d] = __fadd_rn(x[d], ma[d]);
        }
      }
    }
    // ---- positional encoding of the (bent) point -> E, and to its block in global memory ----
    sw.begin();
    if (row_thread) write_pe(x, e_row);
    sw.ready(kStE, Es);
    // ---- L0 .. L7 with their mask bits (LATENT_BIAS: L0 and L5 take the ray-bias rows of their rows' points) ----
    uint32_t h[kMaskHCols / 16][4];
    int ray_r0 = 0, ray_r8 = 0;
    if constexpr (LATENT_BIAS) {
      const long long r0 = static_cast<long long>(tile) * kTileM + g * kWgRows + acc_r0();
      ray_r0 = static_cast<int>(min(r0, p.P - 1));
      ray_r8 = static_cast<int>(min(r0 + 8, p.P - 1));
    }
#pragma unroll 1
    for (int L = 0; L < 8; ++L) {
      Acc<fwd::L1> acc;
      if (L == 0) wg_gemm_step<fwd::L0>(acc, ring, [&](uint32_t) { return a_e; }, W, 410);
      else wg_gemm_rs<fwd::step(fwd::L1).N, fwd::step(fwd::L1).k16>(acc, h, ring, L == 5, a_e, W, 410 + L);
      const float* b = p.nerf_bias + L * fwd::b_off(fwd::L1);
      const float* b8 = b;
      if (LATENT_BIAS && (L == 0 || L == 5)) {
        const float* rb = p.ray_bias + (L == 5 ? fwd::b_off(fwd::L1) : 0);
        b = rb + ray_r0 * p.ray_bias_stride;
        b8 = rb + ray_r8 * p.ray_bias_stride;
      }
      // the mask bits and no stash; one epilogue for every layer, with b8 = b outside LATENT_BIAS's L0 / L5
      epi_bias_frag<kMaskHCols, /*RELU*/ true, /*TRAIN*/ true, /*ROW_BIAS*/ true, /*STASH*/ false>(acc, b, h, nullptr, g,
                                                                                                mk + kMkH + L * kMaskHBytes, b8);
    }
  }
  if (wg_leader) tma_bulk_wait<0>();   // the E stores complete before the CTA exits
}

// d raw[3] / d x -> pg.grad [P][3] from field_fwd_grad_kernel's E (p.stash, kEBytes per tile), masks and bender details.
// Without a bender dx after L0^T.  With one, dx plus B0^T's output columns 0..2: B0's input row carries x twice, as
// fp16 xyz_hi (columns 0..2) and its residual xyz_lo (3..5), both against W0[:, :3]; the B0^T image holds W0[:, :3]^T in
// the xyz_hi rows only and zeros in the xyz_lo rows (pack.cu), so columns 0..2 carry the whole xyz gradient and 3..5 are
// zero.  Points whose raw[3] the object removal zeroes (rigidity >= removal) get g = 0.
template <bool HAS_BENDER>
__global__ void __launch_bounds__(kFwdThreads, 1) field_bwd_grad_kernel(const FieldBwdParams p, const PointGradParams pg) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* act = smem;
  uint8_t* ring_buf = smem + kBwdActBytes;
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
    if (warp == 8 && lane == 0) produce(p.nerf_wT, p.bend_wT, p.n_tiles, 0, HAS_BENDER ? dgrad::kCount : dgrad::B4T, dgrad::B4T, dgrad_step_at, ring, W);
    return;
  }

  setmaxnreg_inc<kConsumerRegs>();
  const int g = warp >> 2;
  const int tw = threadIdx.x & 127;
  const bool row_thread = tw < kWgRows;
  const int bar = 1 + g;
  const int row = g * kWgRows + tw;
  uint8_t* a_row = act + row * 16;
  const uint32_t a_base = smem_u32(act) + g * kWgRows * 16;
  auto a_slab = [&](uint32_t j) { return a_base + j * kSlabA; };
  float* stg = stage_all + g * kWgRows * kBwdStageLd;
  const float* my_stg = stg + tw * kBwdStageLd;
  const StashWriter<true> sw{nullptr, false, bar, g};   // orders the bender images: no stores

  const float scale = loss_scale(&kUnitAmax);
  const float inv_scale = 1.0f / scale;

  for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
    const long long pt = static_cast<long long>(tile) * kTileM + row;
    const bool valid = row_thread && pt < p.P;
    const uint8_t* e_row = p.stash + static_cast<long long>(tile) * kEBytes + row * 16;
    const uint8_t* mk = p.relu_mask + static_cast<long long>(tile) * kMaskTileBytes;
    constexpr Step kTrunk = dgrad::step(dgrad::L7T), kEmb = dgrad::step(dgrad::L5eT);
    static_assert(dgrad::step(dgrad::L0T) == kEmb && kEmb.nslabs == 1 && kEmb.k16 == kMaskHCols / 16, "L5e^T, L0^T: one slab, K = 256");
    uint32_t h[kMaskHCols / 16][4];
    {   // ---- head^T: dh8 = e_3 . Wout (alpha_linear for a view-dependent trunk) -> dY7 ----
      uint32_t a[1][4];
      sigma_frag(p.P, tile, scale, g, a);
      Acc<dgrad::HeadT> acc;
      ReluMask<kMaskHCols> m;
      m.load(mk + kMkH + 7 * kMaskHBytes, g);
      wg_gemm_rs<kTrunk.N, 1>(acc, a, ring, false, 0u, W, 500);
      epi_grad_frag<kMaskHCols, true, /*STASH*/ false>(acc, m, h, nullptr, g);
    }
    float dx[3] = {0.f, 0.f, 0.f};
#pragma unroll 1
    for (int s = 0; s < 2; ++s) {   // ---- L7^T, L6^T : dY6, dY5 ----
      Acc<dgrad::L7T> acc;
      ReluMask<kMaskHCols> m;
      m.load(mk + kMkH + (6 - s) * kMaskHBytes, g);
      wg_gemm_rs<kTrunk.N, kTrunk.k16>(acc, h, ring, false, 0u, W, 501 + s);
      epi_grad_frag<kMaskHCols, true, /*STASH*/ false>(acc, m, h, nullptr, g);
    }
    {   // ---- L5e^T: gradient into the skip-connected embedding ----
      Acc<dgrad::L5eT> acc;
      wg_gemm_rs<kEmb.N, kEmb.k16>(acc, h, ring, false, 0u, W, 503);
      wg_bar(bar);   // stg: every read of the previous tile is done
      stage_cols<0, 8>(acc, stg, kBwdStageLd);
      wg_bar(bar);
      if (row_thread) pe_backward(my_stg, e_row, dx);
    }
#pragma unroll 1
    for (int s = 0; s < 5; ++s) {   // ---- L5h^T, L4^T .. L1^T : dY4 .. dY0 ----
      Acc<dgrad::L4T> acc;
      ReluMask<kMaskHCols> m;
      m.load(mk + kMkH + (4 - s) * kMaskHBytes, g);
      wg_gemm_rs<kTrunk.N, kTrunk.k16>(acc, h, ring, false, 0u, W, 504 + s);
      epi_grad_frag<kMaskHCols, true, /*STASH*/ false>(acc, m, h, nullptr, g);
    }
    {   // ---- L0^T: gradient into the embedding ----
      Acc<dgrad::L0T> acc;
      wg_gemm_rs<kEmb.N, kEmb.k16>(acc, h, ring, false, 0u, W, 509);
      wg_bar(bar);
      stage_cols<0, 8>(acc, stg, kBwdStageLd);
      wg_bar(bar);
      if (row_thread) pe_backward(my_stg, e_row, dx);
    }
    if constexpr (!HAS_BENDER) {
      if (valid) {
#pragma unroll
        for (int d = 0; d < 3; ++d) pg.grad[pt * 3 + d] = dx[d] * inv_scale;
      }
    } else {
      // ---- bend backward: bent = x + masked, masked = rig * un (* scaling) -> dYb4 = d unmasked, d rigidity pre-activation ----
      float drpre = 0.f, rig = 0.f, rs = 1.f;   // rs: this row's scale of the bender chain (row_scale)
      sw.begin();
      if (row_thread) {
        float un[3] = {0.f, 0.f, 0.f}, dun[3], dm[3];
        if (valid) {
          rig = __ldg(p.rigidity + pt);
#pragma unroll
          for (int d = 0; d < 3; ++d) un[d] = __ldg(p.unmasked + pt * 3 + d);
        }
        float dr = 0.f;
#pragma unroll
        for (int d = 0; d < 3; ++d) {
          dm[d] = p.use_scaling ? dx[d] * p.scaling : dx[d];
          dun[d] = rig * dm[d];
          dr += un[d] * dm[d];
        }
        drpre = dr * 2.0f * rig * (1.0f - rig);
        if (p.use_cutoff && rig <= p.cutoff) drpre = 0.f;
        if (!valid) { dun[0] = dun[1] = dun[2] = 0.f; drpre = 0.f; }
        rs = row_scale(fmaxf(fmaxf(fabsf(dun[0]), fabsf(dun[1])), fmaxf(fabsf(dun[2]), fabsf(drpre))));
        dun[0] *= rs; dun[1] *= rs; dun[2] *= rs; drpre *= rs;
        *reinterpret_cast<uint4*>(a_row) = make_uint4(pack_h2(clamp_h(dun[0]), clamp_h(dun[1])), pack_h2(clamp_h(dun[2]), 0.f), 0u, 0u);
        *reinterpret_cast<uint4*>(a_row + kChunkBytes) = make_uint4(0u, 0u, 0u, 0u);
      }
      sw.ready(kGsYb4, act);
      {   // ---- B4^T -> dYb3 ----
        Acc<dgrad::B4T> acc;
        ReluMask<kMkHb4.cols> m;
        m.load(mk + kMkHb4.off, g);
        wg_gemm_step<dgrad::B4T>(acc, ring, a_slab, W, 510);
        sw.begin();
        epi_mask_store<kMkHb4.cols>(acc, m, act, g);
        sw.ready(kGsYb3, act);
      }
      {   // ---- B3^T -> dYb2 = [dh * mask (64) | d rigidity pre-activation | 0 (15)] ----
        Acc<dgrad::B3T> acc;
        ReluMask<kMkHb3.cols> m;
        m.load(mk + kMkHb3.off, g);
        wg_gemm_step<dgrad::B3T>(acc, ring, a_slab, W, 511);
        sw.begin();
        epi_mask_store<kMkHb3.cols>(acc, m, act, g);
        if (row_thread) {
          *reinterpret_cast<uint4*>(a_row + 8 * kChunkBytes) = make_uint4(pack_h2(clamp_h(drpre), 0.f), 0u, 0u, 0u);
          *reinterpret_cast<uint4*>(a_row + 9 * kChunkBytes) = make_uint4(0u, 0u, 0u, 0u);
        }
        sw.ready(kGsYb2, act);
      }
      {   // ---- B2^T -> dYb1, B1^T -> dYb0 ----
        Acc<dgrad::B2T> acc;
        ReluMask<kMkHb2.cols> m;
        m.load(mk + kMkHb2.off, g);
        wg_gemm_step<dgrad::B2T>(acc, ring, a_slab, W, 512);
        sw.begin();
        epi_mask_store<kMkHb2.cols>(acc, m, act, g);
        sw.ready(kGsYb1, act);
        m.load(mk + kMkHb1.off, g);
        wg_gemm_step<dgrad::B1T>(acc, ring, a_slab, W, 513);
        sw.begin();
        epi_mask_store<kMkHb1.cols>(acc, m, act, g);
        sw.ready(kGsYb0, act);
      }
      {   // ---- B0^T: d(bender input); its xyz_hi columns 0..2 -> d x = dx + (d masked / d x)^T dx ----
        Acc<dgrad::B0T> acc;
        wg_gemm_step<dgrad::B0T>(acc, ring, a_slab, W, 514);
        stage_cols<0, 1>(acc, stg, kBwdStageLd);
        wg_bar(bar);
        if (valid) {
          const bool removed = pg.use_removal && rig >= pg.removal;
#pragma unroll
          for (int d = 0; d < 3; ++d) pg.grad[pt * 3 + d] = removed ? 0.f : dx[d] * inv_scale + my_stg[d] * (inv_scale / rs);
        }
      }
    }
    // next: the next tile's L5e^T rewrites stg only after its own barrier; act only after the bender's sw.begin()
  }
}

cudaError_t launch_field_fwd_grad(const FieldFwdParams& p, bool has_bender, int num_sms, cudaStream_t stream) {
  if (has_bender) return launch_field(field_fwd_grad_kernel<true, false>, p, num_sms, kFwdSmemBytes, stream);
  if (p.ray_bias) return launch_field(field_fwd_grad_kernel<false, true>, p, num_sms, kFwdSmemBytes, stream);
  return launch_field(field_fwd_grad_kernel<false, false>, p, num_sms, kFwdSmemBytes, stream);
}

cudaError_t launch_field_bwd_grad(const FieldBwdParams& p, const PointGradParams& pg, bool has_bender, int num_sms, cudaStream_t stream) {
  return launch_field(has_bender ? field_bwd_grad_kernel<true> : field_bwd_grad_kernel<false>, p, num_sms, kBwdSmemBytes, stream, pg);
}

}  // namespace nrn
