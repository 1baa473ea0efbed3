// The inverse of the ray bender: for canonical points c and latent codes z, the observed points x with b(x; z) = c.
//
//   b(x; z) = x + s r~(x) o(x, z)      (ray_bending.forward, run_nerf_helpers.py:507-584, with the test-time knobs)
//   J(x)    = I + s (r~ do/dx + o (x) grad r~),   grad r~ = 2 r (1 - r) grad rho   (0 where the cutoff zeroes r)
//
// Per point: x_0 = c - s r~(c) o(c, z); then `iterations` Newton steps x <- x - J(x)^-1 (b(x) - c), each skipped once
// |b(x) - c|_2 <= tol (the point is frozen, so its result does not depend on how long the others iterate), with the
// fixed-point step x <- x - (b(x) - c) where J is singular (|det J| <= kDeformSingular times Hadamard's bound) or the
// Newton step is not finite; a last evaluation gives the residual, converged = residual <= tol, and r~(x).  A point or
// latent with a non-finite value gives NaN x, residual and rigidity and converged = 0.
//
// One evaluation is the field kernels' bender steps B0..B4 on tensor cores at fp32 accuracy (resident_mma.cuh: operands
// and weights as fp16 parts and residuals): the primal on the input row [x | 0 | z | 0] with bias and ReLU, recording the
// ReLU mask bits in registers; then per axis a the tangent J e_a.  The tangent of e_a after B0 is D1 W0[:, a], read from
// the resident weight image without an MMA; B1..B4 run on it under the primal masks as in the divergence kernels.  The
// 3 x 3 solve is per point on the CUDA cores (Cramer's rule on J's columns).
//
// Work: one persistent launch over (frame, 128-point tile) pairs, two tiles in flight per CTA (resident_mma.cuh).  A
// warpgroup stops iterating a tile once none of its points is still active; that changes no result.
#include "resident_mma.cuh"
#include "deform.cuh"

namespace nrn {

namespace {

constexpr int kDeformJLd = 6;   // floats per row: J's columns 0 and 1 while column 2 is formed
constexpr size_t kDeformSmemBytes = res_smem_bytes(kBendWBytes) + kResWgs * kWgRows * kDeformJLd * sizeof(float);
static_assert(kDeformSmemBytes <= 227 * 1024, "deform kernel: shared memory of one CTA per SM");

// Primal epilogue: accumulator columns [0, NCOLS) + bias, ReLU -> this warpgroup's rows of the next A operand as fp16 parts
// and residuals; the mask bits of the fp32 values (> 0) -> m, in ReluMask's order
template <int NCOLS, int NR>
__device__ __forceinline__ void epi_bias_relu_split(const float (&acc)[NR], const float* __restrict__ bias, ReluMask<NCOLS>& m,
                                                    const ResSmem& s, int h) {
  const int r0 = h * kWgRows + acc_r0(), q = acc_q();
  m.clear();
#pragma unroll
  for (int j = 0; j < NCOLS / 8; ++j) {
    const float2 b = __ldg(reinterpret_cast<const float2*>(bias + 8 * j + 2 * q));
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const float u = acc[4 * j + 2 * i] + b.x, v = acc[4 * j + 2 * i + 1] + b.y;
      m.w[i][j >> 4] |= (u > 0.f ? 1u << (j & 15) : 0u) | (v > 0.f ? 0x10000u << (j & 15) : 0u);
      const uint2 hl = split_h2(fmaxf(u, 0.f), fmaxf(v, 0.f));
      const int off = j * kChunkBytes + (r0 + 8 * i) * 16 + 4 * q;
      *reinterpret_cast<uint32_t*>(s.img_hi + off) = hl.x;
      *reinterpret_cast<uint32_t*>(s.img_lo + off) = hl.y;
    }
  }
}

// The bender input row [x(3) | 0(3) | z(32) | 0(10)] (the B0 image's K layout, xyz_lo columns unused: x's residual is in
// the lo image) as fp16 parts and residuals; z = null: zeros
__device__ __forceinline__ void write_input_row(const float (&x)[3], const float* __restrict__ z, const ResSmem& s, int row_off) {
  float in[48];
#pragma unroll
  for (int d = 0; d < 3; ++d) { in[d] = x[d]; in[3 + d] = 0.f; }
#pragma unroll
  for (int i = 0; i < kLatent; ++i) in[6 + i] = z ? __ldg(z + i) : 0.f;
#pragma unroll
  for (int i = 6 + kLatent; i < 48; ++i) in[i] = 0.f;
#pragma unroll
  for (int c = 0; c < 6; ++c) {
    const uint2 a = split_h2(in[8 * c], in[8 * c + 1]), b = split_h2(in[8 * c + 2], in[8 * c + 3]);
    const uint2 e = split_h2(in[8 * c + 4], in[8 * c + 5]), g = split_h2(in[8 * c + 6], in[8 * c + 7]);
    *reinterpret_cast<uint4*>(s.img_hi + row_off + c * kChunkBytes) = make_uint4(a.x, b.x, e.x, g.x);
    *reinterpret_cast<uint4*>(s.img_lo + row_off + c * kChunkBytes) = make_uint4(a.y, b.y, e.y, g.y);
  }
}

// bar.sync of the warpgroup that also returns whether `pred` holds for any of its threads
__device__ __forceinline__ bool wg_bar_any(int id, bool pred) {
  uint32_t r;
  asm volatile("{\n\t.reg .pred p, q;\n\tsetp.ne.u32 p, %1, 0;\n\tbar.red.or.pred q, %2, 128, p;\n\tselp.u32 %0, 1, 0, q;\n\t}"
               : "=r"(r) : "r"(static_cast<uint32_t>(pred)), "r"(id) : "memory");
  return r != 0;
}

// The image just written is complete and visible to the async proxy (wgmma operand) for the whole warpgroup
__device__ __forceinline__ void image_ready(int bar) {
  fence_proxy_async_smem();
  wg_bar(bar);
}

}  // namespace

__global__ void __launch_bounds__(kResThreads, 1) deform_kernel(const DeformParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int wg = threadIdx.x >> 7;
  const int h = wg & 1;   // half of the tile: rows [64 h, 64 h + 64)
  const ResSmem s = res_smem(smem, kBendWBytes, wg);
  load_resident_weights(s, p.bender, p.bender + kBendLoOffset, kBendWBytes);
  const Waiter W{&s.sh->abort_flag, p.err};
  W.wait(&s.sh->w_full, 0, 410);

  const int tw = threadIdx.x & 127;
  const bool row_thread = tw < kWgRows;   // threads 0-63 (warps 0, 1) of the warpgroup each own one point
  const int bar = 1 + wg;
  const int row_off = (h * kWgRows + tw) * 16;
  const uint32_t a_hi = smem_u32(s.img_hi) + h * kWgRows * 16, a_lo = smem_u32(s.img_lo) + h * kWgRows * 16;
  const float* my_stg = s.stage + tw * kResStageLd;
  float* my_j = reinterpret_cast<float*>(s.sh + 1) + (wg * kWgRows + tw) * kDeformJLd;   // row threads only
  const float* bias = reinterpret_cast<const float*>(p.bender + kBendWBytes);
  const __half* w0_hi = reinterpret_cast<const __half*>(s.w_hi);   // B0 image: element (n, k < 8) at n * 8 + k
  const __half* w0_lo = reinterpret_cast<const __half*>(s.w_lo);
  const float sc = p.use_scaling ? p.scaling : 1.f;
  const long long tiles = (p.P + kTileM - 1) / kTileM;
  const long long items = tiles * p.F;

  for (long long item = static_cast<long long>(blockIdx.x) * kResTilesPerCta + (wg >> 1); item < items;
       item += static_cast<long long>(gridDim.x) * kResTilesPerCta) {
    const long long f = item / tiles;
    const long long pt = (item - f * tiles) * kTileM + h * kWgRows + tw;
    const bool valid = row_thread && pt < p.P;
    const float* z = p.latents + f * p.latent_stride;
    float c[3] = {0.f, 0.f, 0.f};
    bool bad = !valid;
    if (valid) {
#pragma unroll
      for (int d = 0; d < 3; ++d) { c[d] = __ldg(p.points + pt * 3 + d); bad |= !isfinite(c[d]); }
#pragma unroll
      for (int i = 0; i < kLatent; ++i) bad |= !isfinite(__ldg(z + i));
      if (bad) c[0] = c[1] = c[2] = 0.f;
    }

    // per point (row threads): x, and at the last evaluation the offsets o, r, r~, s r~ o and b(x) - c
    float x[3] = {c[0], c[1], c[2]}, o[3], g[3];
    float r = 0.f, rt = 0.f, res = 0.f;
    ReluMask<kMkHb1.cols> m1;
    ReluMask<kMkHb2.cols> m2;
    ReluMask<kMkHb3.cols> m3;
    ReluMask<kMkHb4.cols> m4;

    // b at x: B0..B4 with bias and ReLU, the ReLU masks into m1..m4.  start: x = c (so b - c = s r~ o) becomes x_0 = c - s r~ o
    auto primal = [&](bool start) {
      wg_bar(bar);   // every warp's MMAs on the images are done
      if (row_thread) write_input_row(x, bad ? nullptr : z, s, row_off);
      image_ready(bar);
      {
        Acc<fwd::B0> acc;
        wg_mma_split<fwd::B0, true>(acc, a_hi, a_lo, s);
        wg_bar(bar);
        epi_bias_relu_split<kMkHb1.cols>(acc, bias + fwd::b_off(fwd::B0), m1, s, h);
        image_ready(bar);
        wg_mma_split<fwd::B1, true>(acc, a_hi, a_lo, s);
        wg_bar(bar);
        epi_bias_relu_split<kMkHb2.cols>(acc, bias + fwd::b_off(fwd::B1), m2, s, h);
        image_ready(bar);
      }
      {
        Acc<fwd::B2> acc;
        wg_mma_split<fwd::B2, true>(acc, a_hi, a_lo, s);
        wg_bar(bar);
        epi_bias_relu_split<kMkHb3.cols>(acc, bias + fwd::b_off(fwd::B2), m3, s, h);
        if (acc_q() == 0) {   // column 64: the rigidity pre-activation without its bias
          s.stage[acc_r0() * kResStageLd + 8] = acc[32];
          s.stage[(acc_r0() + 8) * kResStageLd + 8] = acc[34];
        }
        image_ready(bar);
      }
      {
        Acc<fwd::B3> acc;
        wg_mma_split<fwd::B3, true>(acc, a_hi, a_lo, s);
        wg_bar(bar);
        epi_bias_relu_split<kMkHb4.cols>(acc, bias + fwd::b_off(fwd::B3), m4, s, h);
        image_ready(bar);
      }
      {
        Acc<fwd::B4> acc;
        wg_mma_split<fwd::B4, true>(acc, a_hi, a_lo, s);
        stage_cols<0, 1>(acc, s.stage, kResStageLd);
        wg_bar(bar);
      }
      if (row_thread) {   // run_nerf_helpers.py:559-570, each operation rounded like the reference's
        r = (tanhf(my_stg[8] + __ldg(bias + fwd::b_off(fwd::B2) + 64)) + 1.0f) * 0.5f;
        rt = p.use_cutoff && r <= p.cutoff ? 0.f : r;
#pragma unroll
        for (int d = 0; d < 3; ++d) {
          o[d] = my_stg[d];
          float ma = __fmul_rn(rt, o[d]);
          if (p.use_scaling) ma = __fmul_rn(ma, p.scaling);
          if (start) x[d] = __fsub_rn(c[d], ma);
          g[d] = __fsub_rn(__fadd_rn(x[d], ma), c[d]);
        }
        res = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(g[0], g[0]), __fmul_rn(g[1], g[1])), __fmul_rn(g[2], g[2])));
      }
    };

    // column a of J at the last evaluated x (row threads)
    auto tangent = [&](int a, float* col) {
      {
        Acc<fwd::B0> acc;   // B0's tangent W0[:, a], the same for every row
        const int q = acc_q();
#pragma unroll
        for (int j = 0; j < kMkHb1.cols / 8; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int n = 8 * j + 2 * q + e;
            const float w = __half2float(w0_hi[n * 8 + a]) + __half2float(w0_lo[n * 8 + a]) * kLoInv;
            acc[4 * j + e] = w;
            acc[4 * j + 2 + e] = w;
          }
        }
        epi_mask_split<kMkHb1.cols>(acc, m1, s, h);
        image_ready(bar);
        wg_mma_split<fwd::B1, true>(acc, a_hi, a_lo, s);
        wg_bar(bar);
        epi_mask_split<kMkHb2.cols>(acc, m2, s, h);
        image_ready(bar);
      }
      {
        Acc<fwd::B2> acc;
        wg_mma_split<fwd::B2, true>(acc, a_hi, a_lo, s);
        wg_bar(bar);
        epi_mask_split<kMkHb3.cols>(acc, m3, s, h);
        if (acc_q() == 0) {   // column 64: d rho / d x_a
          s.stage[acc_r0() * kResStageLd + 8] = acc[32];
          s.stage[(acc_r0() + 8) * kResStageLd + 8] = acc[34];
        }
        image_ready(bar);
      }
      {
        Acc<fwd::B3> acc;
        wg_mma_split<fwd::B3, true>(acc, a_hi, a_lo, s);
        wg_bar(bar);
        epi_mask_split<kMkHb4.cols>(acc, m4, s, h);
        image_ready(bar);
      }
      {
        Acc<fwd::B4> acc;
        wg_mma_split<fwd::B4, true>(acc, a_hi, a_lo, s);
        stage_cols<0, 1>(acc, s.stage, kResStageLd);
        wg_bar(bar);
      }
      if (row_thread) {
        const float gr = rt == 0.f ? 0.f : 2.0f * r * (1.0f - r) * my_stg[8];
#pragma unroll
        for (int d = 0; d < 3; ++d) col[d] = (d == a ? 1.f : 0.f) + sc * (rt * my_stg[d] + o[d] * gr);
      }
    };

    primal(true);
    bool frozen = false;
    for (int it = 0;; ++it) {
      primal(false);
      frozen |= res <= p.tol;
      if (it == p.iterations) break;
      const bool active = valid && !bad && !frozen;
      if (!wg_bar_any(bar, active)) break;   // nothing of this warpgroup's rows moves any more
      float j2[3];
      tangent(0, my_j);
      tangent(1, my_j + 3);
      tangent(2, j2);
      if (active) {
        const float j0[3] = {my_j[0], my_j[1], my_j[2]}, j1[3] = {my_j[3], my_j[4], my_j[5]};
        // J^-1 g by Cramer's rule: the rows of J^-1 are (j1 x j2, j2 x j0, j0 x j1) / det
        const float k0[3] = {j1[1] * j2[2] - j1[2] * j2[1], j1[2] * j2[0] - j1[0] * j2[2], j1[0] * j2[1] - j1[1] * j2[0]};
        const float k1[3] = {j2[1] * j0[2] - j2[2] * j0[1], j2[2] * j0[0] - j2[0] * j0[2], j2[0] * j0[1] - j2[1] * j0[0]};
        const float k2[3] = {j0[1] * j1[2] - j0[2] * j1[1], j0[2] * j1[0] - j0[0] * j1[2], j0[0] * j1[1] - j0[1] * j1[0]};
        const float det = j0[0] * k0[0] + j0[1] * k0[1] + j0[2] * k0[2];
        const float had = sqrtf(j0[0] * j0[0] + j0[1] * j0[1] + j0[2] * j0[2]) * sqrtf(j1[0] * j1[0] + j1[1] * j1[1] + j1[2] * j1[2]) *
                          sqrtf(j2[0] * j2[0] + j2[1] * j2[1] + j2[2] * j2[2]);
        float st[3] = {(k0[0] * g[0] + k0[1] * g[1] + k0[2] * g[2]) / det, (k1[0] * g[0] + k1[1] * g[1] + k1[2] * g[2]) / det,
                       (k2[0] * g[0] + k2[1] * g[1] + k2[2] * g[2]) / det};
        if (!(fabsf(det) > kDeformSingular * had) || !isfinite(st[0]) || !isfinite(st[1]) || !isfinite(st[2])) {
          st[0] = g[0]; st[1] = g[1]; st[2] = g[2];   // the fixed-point step
        }
#pragma unroll
        for (int d = 0; d < 3; ++d) x[d] -= st[d];
      }
    }

    if (valid) {
      const long long q = f * p.P + pt;
      const float nan = __int_as_float(0x7fc00000);
      p.out[q * 3 + 0] = bad ? nan : x[0];
      p.out[q * 3 + 1] = bad ? nan : x[1];
      p.out[q * 3 + 2] = bad ? nan : x[2];
      if (p.residual) p.residual[q] = bad ? nan : res;
      if (p.converged) p.converged[q] = !bad && res <= p.tol ? 1 : 0;
      if (p.rigidity) p.rigidity[q] = bad ? nan : rt;
    }
  }
}

cudaError_t launch_deform(const DeformParams& p, int num_sms, cudaStream_t st) {
  const long long items = (p.P + kTileM - 1) / kTileM * p.F;
  if (items <= 0) return cudaSuccess;
  cudaError_t e = cudaFuncSetAttribute(deform_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kDeformSmemBytes));
  if (e != cudaSuccess) return e;
  const long long pairs = (items + kResTilesPerCta - 1) / kResTilesPerCta;
  deform_kernel<<<static_cast<unsigned>(pairs < num_sms ? pairs : num_sms), kResThreads, kDeformSmemBytes, st>>>(p);
  return cudaGetLastError();
}

}  // namespace nrn
