// Divergence regulariser of the ray-bending offset field, forward and backward, without autograd.
//
// Reference: training_wrapper_class.forward (train.py:245-286) -> compute_divergence_loss /
// divergence_approx (run_nerf_helpers.py:22-116): for every COARSE sample point the Hutchinson
// estimate  d = e^T J e,  J = d(masked offsets)/d(xyz),  e ~ N(0, I), is formed with
// autograd.grad(create_graph=True) and the loss  mean_s( w d^2 )  is differentiated again w.r.t. the
// bender weights (a double backward).  Here the same quantities are computed in closed form:
//
//   masked = r * off,   off = W4 relu(W3 relu(W2 relu(W1 relu(W0 [x, l] + b0) ..))),  r = (tanh(c3)+1)/2
//   J e    = r * (W4 D4 W3 D3 W2 D2 W1 D1 W0[:, :3] e)  +  off * r'(c3) * (R2 E2 R1 E1 R0 e)
//          = r * tau_off + off * tau_r                       (D_i, E_i: ReLU masks of the primal pass)
//   d      = r * alpha + beta * tau_r,   alpha = e . tau_off,  beta = e . off,  tau_r = 2 r (1 - r) tau_c
//
// Both chains run on tensor cores as the bender steps of the field kernels (field_mma.cuh), with the ReLU mask bits the
// primal pass wrote (ReluMask), at fp32 accuracy: every operand x is carried as x_hi = fp16(x) plus a residual
// x_lo = fp16((x - x_hi) * 2048), weights included (ops.pack_bender writes the residual images), and a step is
//   acc = (A_lo . W_hi + A_hi . W_lo) / 2048 + A_hi . W_hi       (fp32 accumulators; the A_lo . W_lo term is below fp32)
// so the tangent is the derivative of the fp32 network, as an fp32 SIMT evaluation would give it.  The images stored for
// WGRAD are the x_hi parts, i.e. the fp16 roundings of those fp32 values.
//   forward  = the field forward's B0..B4 on the input row [e_hi e_lo | 0] (no bias; the epilogue multiplies by the
//              primal mask instead of applying bias + ReLU).  tau_c is column 64 of B2, tau_off columns 0-2 of B4.
//              The tangent images [e | t1 s1 | t2 s2 | t3 | t4] go to the tangent stash (layout of the forward stash's
//              bender section).
//   backward = DGRAD's B4^T..B1^T on [taubar_off | 0], with taubar_c in column 64 of the B3^T output (where DGRAD puts
//              the rigidity pre-activation gradient), under the power-of-two loss scale of max|dL/dd|.  The adjoint
//              images go to the adjoint stash (layout of the gradient stash's bender section).
// The weight gradients  sum_p abar_i t_{i-1}^T  are then formed by the WGRAD kernel (compact mode) exactly like the
// primal bender layers.  ReLU masks are piecewise constant, so no gradient flows into them (autograd's double backward
// gives the same zeros).  The dependence on the PRIMAL quantities r and off is returned as gradients w.r.t. the coarse
// pass's `rigidity_mask` and `unmasked_offsets` outputs and continues through the ordinary field backward:
//   dL/d off = G tau_r e,     dL/d r = G (alpha + 2 beta tau_c (1 - 2 r))
//
// CTA: four consumer warpgroups, persistent over tiles; warpgroups 2p and 2p + 1 work on one tile (rows 0-63 / 64-127), so
// two tiles are in flight per SM.  The weight images and their residuals (104 KB forward, 86 KB backward) are loaded once
// per CTA by bulk TMA and stay resident, so there is no producer warp and no ring.
#include "resident_mma.cuh"
#include "div.cuh"

namespace nrn {

namespace {

// resident weights (each with its residual image): B0..B4 (forward); B4^T..B1^T (backward: the probe e is not
// differentiated)
constexpr int kDivFwdWBytes = kBendWBytes;
constexpr int kDivBwdWBytes = dgrad::w_off(dgrad::B0T);
static_assert(res_smem_bytes(kDivFwdWBytes) <= 227 * 1024, "div kernels: shared memory of one CTA per SM");

}  // namespace

// ------------------------------------------------------------------------------------------------
// DET = false: the per-ray loss is added into p.loss with fp32 atomics, in no fixed order.
// DET = true (deterministic mode): a warp whose 32 rows are all valid and of one ray stores its butterfly sum in
// loss_rows[32k], its first point; any other warp stores each valid row's share; div_loss_reduce_kernel sums them per ray.
template <bool DET>
__device__ __forceinline__ void div_fwd_body(const DivParams& p, float* loss_rows) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int wg = threadIdx.x >> 7;
  const int h = wg & 1;                   // half of the tile: rows [64 h, 64 h + 64)
  const ResSmem s = res_smem(smem, kDivFwdWBytes, wg);
  load_resident_weights(s, p.bender, p.bender + kBendLoOffset, kDivFwdWBytes);
  const Waiter W{&s.sh->abort_flag, p.err};

  const int tw = threadIdx.x & 127;
  const int lane = threadIdx.x & 31;
  const bool row_thread = tw < kWgRows;   // threads 0-63 (warps 0, 1) of the warpgroup each own one row
  const int bar = 1 + wg;
  const bool wg_leader = tw == 0;
  const int row_off = (h * kWgRows + tw) * 16;
  const uint32_t a_hi = smem_u32(s.img_hi) + h * kWgRows * 16, a_lo = smem_u32(s.img_lo) + h * kWgRows * 16;
  const float* my_stg = s.stage + tw * kResStageLd;
  const long long n_tiles = (p.P + kTileM - 1) / kTileM;

  for (long long tile = static_cast<long long>(blockIdx.x) * kResTilesPerCta + (wg >> 1); tile < n_tiles;
       tile += static_cast<long long>(gridDim.x) * kResTilesPerCta) {
    const long long pt = tile * kTileM + h * kWgRows + tw;
    const bool valid = row_thread && pt < p.P;
    uint8_t* tn = p.tan + tile * kTanTileBytes;
    const uint8_t* mk = p.relu_mask + tile * kMaskTileBytes;
    const StashWriter<false> sw{tn, wg_leader, bar, h};   // every finished fp16 image goes to the tangent stash

    float e[3] = {0.f, 0.f, 0.f}, off[3] = {0.f, 0.f, 0.f};
    float r = 0.f, w = 0.f;
    if (valid) {
#pragma unroll
      for (int d = 0; d < 3; ++d) { e[d] = __ldg(p.e + pt * 3 + d); off[d] = __ldg(p.unmasked + pt * 3 + d); }
      r = __ldg(p.rigidity + pt);
      w = __ldg(p.w + pt);
      if (p.w_is_alpha) w = 1.0f - expf(-fmaxf(w, 0.f));
    }
    // ---- tangent input row: [e_hi(3) e_lo(3) 0(42)], the bender-input layout (B0 applies W0[:, :3] to hi and lo) ----
    sw.begin();
    if (row_thread) {
      float hi[3], lo[3];
#pragma unroll
      for (int d = 0; d < 3; ++d) { hi[d] = __half2float(__float2half_rn(e[d])); lo[d] = e[d] - hi[d]; }
      uint8_t* a_row = s.img_hi + row_off;
      *reinterpret_cast<uint4*>(a_row) = make_uint4(pack_h2(hi[0], hi[1]), pack_h2(hi[2], lo[0]), pack_h2(lo[1], lo[2]), 0u);
#pragma unroll
      for (int c = 1; c < 6; ++c) *reinterpret_cast<uint4*>(a_row + c * kChunkBytes) = make_uint4(0u, 0u, 0u, 0u);
    }
    sw.ready(tan_image(kStBin), s.img_hi);
    // ---- B0, B1: [t1 | s1] = D1/E1 (B0 [e]), [t2 | s2] = D2/E2 (B1 [t1 | s1]) ----
    {
      Acc<fwd::B0> acc;
      ReluMask<kMkHb1.cols> m;
      m.load(mk + kMkHb1.off, h);
      W.wait(&s.sh->w_full, 0, 330);
      wg_mma_split<fwd::B0, false>(acc, a_hi, a_lo, s);
      sw.begin();
      epi_mask_split<kMkHb1.cols>(acc, m, s, h);
      sw.ready(tan_image(kStHb1), s.img_hi);
      m.load(mk + kMkHb2.off, h);
      wg_mma_split<fwd::B1, true>(acc, a_hi, a_lo, s);
      sw.begin();
      epi_mask_split<kMkHb2.cols>(acc, m, s, h);
      sw.ready(tan_image(kStHb2), s.img_hi);
    }
    // ---- B2: t3 = D3 (W2 t2); column 64 = tau_c = R2 s2 ----
    {
      Acc<fwd::B2> acc;
      ReluMask<kMkHb3.cols> m;
      m.load(mk + kMkHb3.off, h);
      wg_mma_split<fwd::B2, true>(acc, a_hi, a_lo, s);
      sw.begin();
      epi_mask_split<kMkHb3.cols>(acc, m, s, h);
      if (acc_q() == 0) {
        s.stage[acc_r0() * kResStageLd + 8] = acc[32];
        s.stage[(acc_r0() + 8) * kResStageLd + 8] = acc[34];
      }
      sw.ready(tan_image(kStHb3), s.img_hi);
    }
    // ---- B3: t4 = D4 (W3 t3) ----
    {
      Acc<fwd::B3> acc;
      ReluMask<kMkHb4.cols> m;
      m.load(mk + kMkHb4.off, h);
      wg_mma_split<fwd::B3, true>(acc, a_hi, a_lo, s);
      sw.begin();
      epi_mask_split<kMkHb4.cols>(acc, m, s, h);
      sw.ready(tan_image(kStHb4), s.img_hi);
    }
    // ---- B4: tau_off = W4 t4; per-point scalars and the per-ray loss ----
    {
      Acc<fwd::B4> acc;
      wg_mma_split<fwd::B4, true>(acc, a_hi, a_lo, s);
      stage_cols<0, 1>(acc, s.stage, kResStageLd);
      wg_bar(bar);
      if (row_thread) {   // warps 0 and 1 of the warpgroup: 32 consecutive rows each
        const float tau_c = my_stg[8];
        const float alpha = e[0] * my_stg[0] + e[1] * my_stg[1] + e[2] * my_stg[2];
        const float beta = e[0] * off[0] + e[1] * off[1] + e[2] * off[2];
        const float tau_r = 2.0f * r * (1.0f - r) * tau_c;
        const float d = r * alpha + beta * tau_r;
        float part = 0.f;   // this point's share of mean over the ray's samples of w |d|^2
        if (valid) {
          p.d[pt] = d; p.adot[pt] = alpha; p.beta[pt] = beta; p.tauc[pt] = tau_c;
          part = w * d * d / static_cast<float>(p.S);
        }
        const long long ray = valid ? pt / p.S : -1;
        const long long ray0 = __shfl_sync(0xffffffffu, ray, 0);
        if (__all_sync(0xffffffffu, valid && ray == ray0)) {
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
          if constexpr (DET) {
            if (lane == 0) loss_rows[pt] = part;   // lane 0's point is the warp's first, 32k
          } else {
            if (lane == 0) atomicAdd(p.loss + ray0, part);
          }
        } else if (valid) {
          if constexpr (DET) loss_rows[pt] = part;
          else atomicAdd(p.loss + ray, part);
        }
      }
    }
    // the staging rows are rewritten only after the next tile's warpgroup barriers
  }
  if (wg_leader) tma_bulk_wait<0>();   // all tangent-stash stores complete before the CTA exits
}

__global__ void __launch_bounds__(kResThreads, 1) div_fwd_kernel(const DivParams p) { div_fwd_body<false>(p, nullptr); }
__global__ void __launch_bounds__(kResThreads, 1) div_fwd_det_kernel(const DivParams p, float* loss_rows) {
  div_fwd_body<true>(p, loss_rows);
}

// ------------------------------------------------------------------------------------------------
// HELD: `held` [n_rays] bytes, nonzero for a held-out ray.  The adjoint chain of a held-out ray's points starts from zero,
// so its adjoint-stash rows are zero and the compact WGRAD (no bias term) leaves it out of the bender's weight gradient;
// d_unmasked / d_rigid, which carry its latent gradient into DGRAD, are written as without it.
template <bool HELD>
__device__ __forceinline__ void div_bwd_body(const DivParams& p, const uint8_t* held) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int wg = threadIdx.x >> 7;
  const int h = wg & 1;
  const ResSmem s = res_smem(smem, kDivBwdWBytes, wg);
  load_resident_weights(s, p.bender + kBendTOffset, p.bender + kBendTLoOffset, kDivBwdWBytes);
  const Waiter W{&s.sh->abort_flag, p.err};

  const int tw = threadIdx.x & 127;
  const bool row_thread = tw < kWgRows;
  const int bar = 1 + wg;
  const bool wg_leader = tw == 0;
  const int row_off = (h * kWgRows + tw) * 16;
  const uint32_t a_hi = smem_u32(s.img_hi) + h * kWgRows * 16, a_lo = smem_u32(s.img_lo) + h * kWgRows * 16;
  const long long n_tiles = (p.P + kTileM - 1) / kTileM;

  const float scale = loss_scale(p.amax);   // max|G| is written by div_G_kernel / absmax

  for (long long tile = static_cast<long long>(blockIdx.x) * kResTilesPerCta + (wg >> 1); tile < n_tiles;
       tile += static_cast<long long>(gridDim.x) * kResTilesPerCta) {
    const long long pt = tile * kTileM + h * kWgRows + tw;
    const bool valid = row_thread && pt < p.P;
    uint8_t* ad = p.adj + tile * kAdjTileBytes;
    const uint8_t* mk = p.relu_mask + tile * kMaskTileBytes;
    const StashWriter<false> sw{ad, wg_leader, bar, h};   // every finished fp16 image goes to the adjoint stash

    float e[3] = {0.f, 0.f, 0.f};
    float r = 0.f, G = 0.f, beta = 0.f;
    if (valid) {
#pragma unroll
      for (int d = 0; d < 3; ++d) e[d] = __ldg(p.e + pt * 3 + d);
      r = __ldg(p.rigidity + pt); G = __ldg(p.G + pt); beta = __ldg(p.beta + pt);
      const float alpha = __ldg(p.adot + pt), tau_c = __ldg(p.tauc + pt);
      const float tau_r = 2.0f * r * (1.0f - r) * tau_c;
#pragma unroll
      for (int d = 0; d < 3; ++d) p.d_unmasked[pt * 3 + d] = G * tau_r * e[d];
      p.d_rigid[pt] = G * (alpha + 2.0f * beta * tau_c * (1.0f - 2.0f * r));
    }
    float Gs = G * scale;
    if constexpr (HELD) {
      if (valid && __ldg(held + pt / p.S)) Gs = 0.f;
    }
    const float rp = 2.0f * r * (1.0f - r);
    const float tb_c = Gs * beta * rp;   // adjoint of tau_c
    // ---- [taubar_off (3) | 0], taubar_off = G r e ----
    sw.begin();
    if (row_thread) {
      const uint2 t01 = split_h2(Gs * r * e[0], Gs * r * e[1]), t2 = split_h2(Gs * r * e[2], 0.f);
      *reinterpret_cast<uint4*>(s.img_hi + row_off) = make_uint4(t01.x, t2.x, 0u, 0u);
      *reinterpret_cast<uint4*>(s.img_lo + row_off) = make_uint4(t01.y, t2.y, 0u, 0u);
      *reinterpret_cast<uint4*>(s.img_hi + row_off + kChunkBytes) = make_uint4(0u, 0u, 0u, 0u);
      *reinterpret_cast<uint4*>(s.img_lo + row_off + kChunkBytes) = make_uint4(0u, 0u, 0u, 0u);
    }
    sw.ready(adj_image(kGsYb4), s.img_hi);
    // ---- B4^T -> abar4 = D4 (W4^T taubar_off); B3^T -> [abar3 = D3 (W3^T abar4) | taubar_c | 0] ----
    {
      Acc<dgrad::B4T> acc;
      ReluMask<kMkHb4.cols> m;
      m.load(mk + kMkHb4.off, h);
      W.wait(&s.sh->w_full, 0, 340);
      wg_mma_split<dgrad::B4T, true>(acc, a_hi, a_lo, s);
      sw.begin();
      epi_mask_split<kMkHb4.cols>(acc, m, s, h);
      sw.ready(adj_image(kGsYb3), s.img_hi);
      m.load(mk + kMkHb3.off, h);
      wg_mma_split<dgrad::B3T, true>(acc, a_hi, a_lo, s);
      sw.begin();
      epi_mask_split<kMkHb3.cols>(acc, m, s, h);
      if (row_thread) {
        const uint2 t = split_h2(tb_c, 0.f);
        *reinterpret_cast<uint4*>(s.img_hi + row_off + 8 * kChunkBytes) = make_uint4(t.x, 0u, 0u, 0u);
        *reinterpret_cast<uint4*>(s.img_lo + row_off + 8 * kChunkBytes) = make_uint4(t.y, 0u, 0u, 0u);
        *reinterpret_cast<uint4*>(s.img_hi + row_off + 9 * kChunkBytes) = make_uint4(0u, 0u, 0u, 0u);
        *reinterpret_cast<uint4*>(s.img_lo + row_off + 9 * kChunkBytes) = make_uint4(0u, 0u, 0u, 0u);
      }
      sw.ready(adj_image(kGsYb2), s.img_hi);
    }
    // ---- B2^T -> [abar2 | qbar2] = D2/E2 [W2^T abar3 | R2^T taubar_c];  B1^T -> [abar1 | qbar1] ----
    {
      Acc<dgrad::B2T> acc;
      ReluMask<kMkHb2.cols> m;
      m.load(mk + kMkHb2.off, h);
      wg_mma_split<dgrad::B2T, true>(acc, a_hi, a_lo, s);
      sw.begin();
      epi_mask_split<kMkHb2.cols>(acc, m, s, h);
      sw.ready(adj_image(kGsYb1), s.img_hi);
      m.load(mk + kMkHb1.off, h);
      wg_mma_split<dgrad::B1T, true>(acc, a_hi, a_lo, s);
      sw.begin();
      epi_mask_split<kMkHb1.cols>(acc, m, s, h);
      sw.ready(adj_image(kGsYb0), s.img_hi);
    }
  }
  if (wg_leader) tma_bulk_wait<0>();   // all adjoint-stash stores complete before the CTA exits
}

__global__ void __launch_bounds__(kResThreads, 1) div_bwd_kernel(const DivParams p) { div_bwd_body<false>(p, nullptr); }
__global__ void __launch_bounds__(kResThreads, 1) div_bwd_held_kernel(const DivParams p, const uint8_t* held) {
  div_bwd_body<true>(p, held);
}

// ------------------------------------------------------------------------------------------------
namespace {
__global__ void div_G_kernel(const DivParams p, const float* __restrict__ g_ray, float* __restrict__ G, float* __restrict__ amax) {
  const long long pt = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  float v = 0.f;
  if (pt < p.P) {
    float w = p.w[pt];
    if (p.w_is_alpha) w = 1.0f - expf(-fmaxf(w, 0.f));
    v = g_ray[pt / p.S] * (2.0f / static_cast<float>(p.S)) * w * p.d[pt];
    G[pt] = v;
  }
  float m = fabsf(v);
  if (!(m < 3.0e38f)) m = 0.f;   // ignore inf / nan: the scale must stay finite
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(reinterpret_cast<int*>(amax), __float_as_int(m));   // non-negative floats order like ints
}

template <typename Kernel, typename... Extra>
cudaError_t launch_div(Kernel kernel, int wbytes, const DivParams& p, int num_sms, cudaStream_t st, const Extra&... extra) {
  const long long tiles = (p.P + kTileM - 1) / kTileM;
  if (tiles <= 0) return cudaSuccess;
  const int smem = static_cast<int>(res_smem_bytes(wbytes));
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return e;
  const long long pairs = (tiles + kResTilesPerCta - 1) / kResTilesPerCta;
  kernel<<<static_cast<unsigned>(pairs < num_sms ? pairs : num_sms), kResThreads, smem, st>>>(p, extra...);
  return cudaGetLastError();
}
}  // namespace

cudaError_t launch_div_G(const DivParams& p, const float* g_ray, float* G, float* amax, cudaStream_t st) {
  cudaError_t e = cudaMemsetAsync(amax, 0, sizeof(float), st);
  if (e != cudaSuccess || p.P <= 0) return e;
  div_G_kernel<<<static_cast<unsigned>((p.P + 255) / 256), 256, 0, st>>>(p, g_ray, G, amax);
  return cudaGetLastError();
}

cudaError_t launch_div_fwd(const DivParams& p, int num_sms, cudaStream_t st) {
  return launch_div(div_fwd_kernel, kDivFwdWBytes, p, num_sms, st);
}
cudaError_t launch_div_bwd(const DivParams& p, int num_sms, cudaStream_t st) {
  return launch_div(div_bwd_kernel, kDivBwdWBytes, p, num_sms, st);
}
cudaError_t launch_div_bwd_held(const DivParams& p, const uint8_t* held, int num_sms, cudaStream_t st) {
  return launch_div(div_bwd_held_kernel, kDivBwdWBytes, p, num_sms, st, held);
}
cudaError_t launch_div_fwd_det(const DivParams& p, float* loss_rows, int num_sms, cudaStream_t st) {
  return launch_div(div_fwd_det_kernel, kDivFwdWBytes, p, num_sms, st, loss_rows);
}

}  // namespace nrn
