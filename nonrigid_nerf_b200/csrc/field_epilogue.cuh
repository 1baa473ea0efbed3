// Device helpers of the fused field kernels: the shared-memory layouts, step tables, epilogues and encodings that the
// forward (field_fwd.cu), DGRAD (field_bwd.cu) and point-gradient (field_grad.cu) kernels share.  The point-gradient
// kernels' mask bits and E must be those of the training forward bit for bit, so they use these same helpers.
#pragma once
#include "field_mma.cuh"

namespace nrn {

namespace {

// ---- forward: shared-memory layout and step table ----
constexpr int kFwdStageLd = 12;   // floats per staged row (8 used)
// Activations in shared memory: the bender's hidden images (A operands of B1..B4, at most 96 columns) and E.  The trunk's
// 256-wide activations stay in registers (epi_bias_frag), so the rest of shared memory goes to the weight ring.
constexpr int kFwdHBytes = kStHb1.chunks * kChunkBytes;   // 24 KB
static_assert(kStHb2.chunks <= kStHb1.chunks && kStHb3.chunks <= kStHb1.chunks && kStHb4.chunks <= kStHb1.chunks, "bender images fit H");
constexpr int kFwdRingStages = 5;
constexpr size_t kFwdSmemBytes = kFwdHBytes + kEBytes + kFwdRingStages * kRingStageBytes + 2 * kWgRows * kFwdStageLd * sizeof(float) +
                                 sizeof(RingShared<kFwdRingStages>) + 64;
static_assert(kFwdSmemBytes <= 227 * 1024, "forward kernel: dynamic shared memory per block");

static_assert(fwd::step(fwd::L2) == fwd::step(fwd::L1) && fwd::step(fwd::L3) == fwd::step(fwd::L1) &&
              fwd::step(fwd::L4) == fwd::step(fwd::L1) && fwd::step(fwd::L6) == fwd::step(fwd::L1) &&
              fwd::step(fwd::L7) == fwd::step(fwd::L1), "fwd_step_at: one default shape");
// step -> shape for a run-time step index: a switch over immediate table entries (no table in memory)
__device__ __forceinline__ Step fwd_step_at(int step) {
  switch (step) {
    case fwd::B0: return step_imm<fwd::B0>();
    case fwd::B1: return step_imm<fwd::B1>();
    case fwd::B2: return step_imm<fwd::B2>();
    case fwd::B3: return step_imm<fwd::B3>();
    case fwd::B4: return step_imm<fwd::B4>();
    case fwd::L0: return step_imm<fwd::L0>();
    case fwd::L5: return step_imm<fwd::L5>();
    case fwd::Head: return step_imm<fwd::Head>();
    default: return step_imm<fwd::L1>();   // L1-L4, L6, L7: one shape
  }
}

// ---- DGRAD: shared-memory layout and step table ----
constexpr int kBwdStageLd = 66;   // floats per staged row (64 used)
// Gradient images in shared memory: only the bender chain's (A operands of B4^T..B0^T, at most 96 columns).  The trunk's
// 256-wide gradients stay in registers (epi_grad_frag), so the rest of shared memory goes to the weight ring.
constexpr int kBwdActBytes = kGsYb1.chunks * kChunkBytes;   // 24 KB
static_assert(kGsYb4.chunks <= kGsYb1.chunks && kGsYb3.chunks <= kGsYb1.chunks && kGsYb2.chunks <= kGsYb1.chunks &&
              kGsYb0.chunks <= kGsYb1.chunks, "bender gradient images fit act");
constexpr int kBwdRingStages = 5;
constexpr size_t kBwdSmemBytes = kBwdActBytes + kBwdRingStages * kRingStageBytes + 2 * kWgRows * kBwdStageLd * sizeof(float) +
                                 sizeof(RingShared<kBwdRingStages>) + 64;
static_assert(kBwdSmemBytes <= 227 * 1024, "DGRAD kernel: dynamic shared memory per block");

static_assert(dgrad::step(dgrad::L6T) == dgrad::step(dgrad::L7T) && dgrad::step(dgrad::L5hT) == dgrad::step(dgrad::L7T) &&
              dgrad::step(dgrad::L4T) == dgrad::step(dgrad::L7T) && dgrad::step(dgrad::L3T) == dgrad::step(dgrad::L7T) &&
              dgrad::step(dgrad::L2T) == dgrad::step(dgrad::L7T) && dgrad::step(dgrad::L1T) == dgrad::step(dgrad::L7T),
              "dgrad_step_at: one default shape; the consumers run L5h^T .. L1^T as one loop");
constexpr uint32_t kSlabA = 2 * dgrad::step(dgrad::L4T).k16 * kChunkBytes;   // A operand bytes of one weight slab

// step -> shape for a run-time step index: a switch over immediate table entries (no table in memory)
__device__ __forceinline__ Step dgrad_step_at(int step) {
  switch (step) {
    case dgrad::HeadT: return step_imm<dgrad::HeadT>();
    case dgrad::L5eT: return step_imm<dgrad::L5eT>();
    case dgrad::L0T: return step_imm<dgrad::L0T>();
    case dgrad::B4T: return step_imm<dgrad::B4T>();
    case dgrad::B3T: return step_imm<dgrad::B3T>();
    case dgrad::B2T: return step_imm<dgrad::B2T>();
    case dgrad::B1T: return step_imm<dgrad::B1T>();
    case dgrad::B0T: return step_imm<dgrad::B0T>();
    default: return step_imm<dgrad::L7T>();   // L7^T, L6^T, L5h^T, L4^T .. L1^T
  }
}

// ---- forward epilogues and encodings ----

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

// The same for a layer whose output stays in registers: accumulator columns [0, NCOLS) + bias (RELU: then ReLU), fp16
// with saturation -> the next step's A fragments `a`.  TRAIN with RELU: also the mask bits of those elements -> this
// thread's words of the tile's mask image `mask_img`.  STASH (TRAIN unless given): also the fp16 pairs straight to this
// warpgroup's rows of the tile's stash image `st_img` (a warp's 32 words of one column group and row half are one
// contiguous 128-byte line of the chunk-major image).  ROW_BIAS (time-conditioned L0 / L5): accumulator rows r0 and r0 + 8
// take their biases from their own rows `bias` and `bias8` (their rays' ray-bias rows) instead of one vector.
template <int NCOLS, bool RELU, bool TRAIN, bool ROW_BIAS = false, bool STASH = TRAIN>
__device__ __forceinline__ void epi_bias_frag(const float (&acc)[NCOLS / 2], const float* __restrict__ bias, uint32_t (&a)[NCOLS / 16][4],
                                              uint8_t* st_img, int g, uint8_t* mask_img = nullptr,
                                              const float* __restrict__ bias8 = nullptr) {
  const int r0 = g * kWgRows + acc_r0(), q = acc_q();
  ReluMask<NCOLS> m;
  if constexpr (TRAIN && RELU) m.clear();
#pragma unroll
  for (int j = 0; j < NCOLS / 8; ++j) {
    const float2 b = __ldg(reinterpret_cast<const float2*>(bias + 8 * j + 2 * q));
    float2 b8 = b;
    if constexpr (ROW_BIAS) b8 = __ldg(reinterpret_cast<const float2*>(bias8 + 8 * j + 2 * q));
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const float2 bi = i ? b8 : b;
      const float u = acc[4 * j + 2 * i] + bi.x, v = acc[4 * j + 2 * i + 1] + bi.y;
      const uint32_t h2 = RELU ? pack_h2_relu_sat(u, v) : pack_h2_sat(u, v);
      frag_pair(a, j, i) = h2;
      if constexpr (TRAIN && RELU) m.pack(i, j, h2);
      if constexpr (STASH) *reinterpret_cast<uint32_t*>(st_img + j * kChunkBytes + (r0 + 8 * i) * 16 + 4 * q) = h2;
    }
  }
  if constexpr (TRAIN && RELU) m.store(mask_img, g);
}

// The floats f as fp16 -> chunks 0 .. NF / 8 - 1 of a chunk-major image row
template <int NF>
__device__ __forceinline__ void pack_row(const float (&f)[NF], uint8_t* dst_row) {
  static_assert(NF % 8 == 0, "whole 8-column chunks");
#pragma unroll
  for (int c = 0; c < NF / 8; ++c) {
    uint4 pk;
    pk.x = pack_h2(f[c * 8 + 0], f[c * 8 + 1]);
    pk.y = pack_h2(f[c * 8 + 2], f[c * 8 + 3]);
    pk.z = pack_h2(f[c * 8 + 4], f[c * 8 + 5]);
    pk.w = pack_h2(f[c * 8 + 6], f[c * 8 + 7]);
    *reinterpret_cast<uint4*>(dst_row + c * kChunkBytes) = pk;
  }
}

// The bender's input row of point x: [xyz_hi(3) xyz_lo(3) latent(32) 0(10)] as fp16, chunks 0..5 of the row.  xyz_hi is
// fp16(x) and xyz_lo its residual, both against W0[:, :3]; the latent is read from `lat`, or zero for an invalid row.
__device__ __forceinline__ void write_bender_input(const float (&x)[3], const float* __restrict__ lat, bool valid, uint8_t* dst_row) {
  float in[48];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const float hi = __half2float(__float2half_rn(x[d]));
    in[d] = hi;
    in[3 + d] = x[d] - hi;
  }
#pragma unroll
  for (int i = 0; i < kLatent; ++i) in[6 + i] = valid ? __ldg(lat + i) : 0.f;
#pragma unroll
  for (int i = 38; i < 48; ++i) in[i] = 0.f;
  pack_row(in, dst_row);
}

// Positional encoding of one point (Embedder.embed, run_nerf_helpers.py:149-150 with the settings of
// get_embedder :157-164: raw xyz first, then per octave sin(2^k xyz), cos(2^k xyz); k = 0..9).
// Written as fp16 chunks 0..7 of the row (63 features + one zero pad column).
// sin/cos: the argument 2^k * x is reduced EXACTLY to [-0.5, 0.5) turns (x / 2pi carried as a
// two-float value), then evaluated with MUFU (abs err ~4e-7), well below fp16 resolution.
// The encoding of NF octaves, [x, sin(2^k x), cos(2^k x)] for k < NF, as floats f[0, 3 + 6 NF).
template <int NF, int NR>
__device__ __forceinline__ void encode_octaves(const float (&x)[3], float (&f)[NR]) {
  f[0] = x[0]; f[1] = x[1]; f[2] = x[2];
  const float kInv2PiHi = 0.15915494f;      // fl(1/2pi)
  const float kInv2PiLo = 6.4206199e-09f;   // 1/2pi - fl(1/2pi)
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const float thi = x[d] * kInv2PiHi;
    const float tlo = fmaf(x[d], kInv2PiLo, fmaf(x[d], kInv2PiHi, -thi));
#pragma unroll
    for (int k = 0; k < NF; ++k) {
      const float sc = static_cast<float>(1 << k);
      const float a = thi * sc;
      const float ph = (a - rintf(a)) + tlo * sc;
      const float ang = ph * 6.2831853071795865f;
      f[3 + 6 * k + d] = __sinf(ang);
      f[3 + 6 * k + 3 + d] = __cosf(ang);
    }
  }
}

__device__ __forceinline__ void write_pe(const float (&x)[3], uint8_t* dst_row) {
  float f[64];
  encode_octaves<10>(x, f);
  f[63] = 1.f;  // pad column: its weight column is zero (forward unaffected); WGRAD reads it as the bias input
  pack_row(f, dst_row);
}

// ---- DGRAD epilogues ----

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

// The same for a gradient that stays in registers: NCOLS accumulator columns as fp16 (MASK: dY = dh * [h > 0] with the
// forward's ReLU mask bits `m`) -> the next step's A fragments `a` (wg_gemm_rs).  STASH: also the same fp16 pairs straight
// to this warpgroup's rows of the tile's gradient-stash image `gs_img` (a warp's 32 words of one column group and row half
// are one contiguous 128-byte line of the chunk-major image).
template <int NCOLS, bool MASK, bool STASH = true, int NR>
__device__ __forceinline__ void epi_grad_frag(const float (&acc)[NR], const ReluMask<NCOLS>& m, uint32_t (&a)[NCOLS / 16][4],
                                              uint8_t* gs_img, int g) {
  const int r0 = g * kWgRows + acc_r0(), q = acc_q();
#pragma unroll
  for (int j = 0; j < NCOLS / 8; ++j) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      uint32_t g2 = pack_h2_sat(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]);
      if constexpr (MASK) g2 = m.apply(i, j, g2);
      frag_pair(a, j, i) = g2;
      if constexpr (STASH) *reinterpret_cast<uint32_t*>(gs_img + j * kChunkBytes + (r0 + 8 * i) * 16 + 4 * q) = g2;
    }
  }
}

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

}  // namespace

}  // namespace nrn
