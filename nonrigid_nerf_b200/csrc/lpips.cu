// LPIPS v0.1, AlexNet backbone (free_viewpoint_rendering.py:788-849): input scaling, the five convolutions as implicit
// GEMMs on wgmma, the two max-pools, and the per-tap distances with fixed-order per-frame sums.
//
// Convolution kernel (one template over the five layers): a work item is 128 output pixels of one image times one N
// half (conv3's 384 channels go as two halves of 192).  Warps 0-3 and 4-7 are two consumer warpgroups owning 64 pixels
// each; one thread of warp 8 streams the weight slabs (N x 64 K columns, fp16, K-major chunk-major) through the bulk-TMA
// ring of the field kernels (field_mma.cuh).  Each consumer thread gathers, per slab, four 16-byte chunks of its pixel's
// receptive field (8 input channels of one tap; zeros outside the image and past K) with cp.async into a 4-stage A ring of
// its warpgroup, two slabs ahead of the MMAs.  The epilogue adds the bias, applies ReLU and stores fp16 NHWC with a
// saturating convert; a value above 65504 (the largest fp16) sets bit L of its image's saturation word, and the reduce
// kernel scores such a frame NaN from that tap on.  Nothing is split across images or along K, so an image's features do
// not depend on its batch.
#include "field_mma.cuh"
#include "lpips.cuh"
#include "eval.cuh"
#include "jet.cuh"

namespace nrn {
namespace {

constexpr int kLpRingStages = 4;
constexpr int kLpAStages = 4;                                   // A ring per warpgroup; gathers run 2 slabs ahead
constexpr int kLpABytes = kLpipsSlabChunks * kWgRows * 16;      // one warpgroup's A of one slab: 8 chunks x 64 rows
constexpr int kLpRingOff = 1024;
constexpr int kLpAOff = kLpRingOff + kLpRingStages * kRingStageBytes;
constexpr int kLpConvSmem = kLpAOff + 2 * kLpAStages * kLpABytes;
static_assert(sizeof(RingShared<kLpRingStages>) <= kLpRingOff && kLpConvSmem <= 227 * 1024, "LPIPS conv shared memory");

__device__ __forceinline__ void wgmma_m64n192(float (&d)[96], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %98, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n192k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95}, "
      "%96, %97, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <int N>
__device__ __forceinline__ void lp_wgmma(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  if constexpr (N == 192) wgmma_m64n192(d, adesc, bdesc, accumulate);
  else wgmma<N, 0, 0>(d, adesc, bdesc, accumulate);
}

// 16-byte global -> shared copy; src_bytes = 0 writes zeros (padding taps, K past the layer's)
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

struct ConvParams {
  const __half* in;        // [images][hin][win][cin]
  __half* out;             // [images][hout][wout][cout]
  const uint8_t* w;        // the layer's packed B image
  const float* bias;       // [cout]
  int hin, win, hout, wout;
  int tiles_per_image, n_items;
  int* err;
  unsigned* sat;           // [images] saturation words: bit L set when layer L clamped an output of the image
};

template <int L>
__global__ void __launch_bounds__(kFwdThreads, 1) lpips_conv_kernel(ConvParams p) {
  constexpr LpipsConv S = kLpipsConv[L];
  constexpr int N = S.n(), CIN = S.cin, KS = S.ks, SLABS = S.slabs(), KCH = S.k_chunks(), CPT = CIN / 8;
  extern __shared__ __align__(1024) uint8_t smem[];
  auto* sh = reinterpret_cast<RingShared<kLpRingStages>*>(smem);
  if (threadIdx.x == 0) sh->init();
  __syncthreads();
  const Waiter W{&sh->abort_flag, p.err};
  Ring<kLpRingStages> ring{smem + kLpRingOff, sh->w_full, sh->w_empty};
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (warp >= 8) {
    setmaxnreg_dec<kProducerRegs>();
    if (warp == 8 && lane == 0)
      for (int item = blockIdx.x; item < p.n_items; item += gridDim.x) {
        const uint8_t* w = p.w + static_cast<size_t>(item % S.split) * SLABS * S.slab_bytes();
#pragma unroll 1
        for (int j = 0; j < SLABS; ++j) ring_put(ring, w + static_cast<size_t>(j) * S.slab_bytes(), S.slab_bytes(), W);
      }
    return;
  }

  setmaxnreg_inc<kConsumerRegs>();
  const int g = warp >> 2;
  const int t = threadIdx.x & 127;
  const int row = t & (kWgRows - 1), c0 = t >> 6;   // this thread gathers chunks c0, c0 + 2, c0 + 4, c0 + 6 of its row
  uint8_t* abuf = smem + kLpAOff + g * kLpAStages * kLpABytes;
  const uint32_t a_dst = smem_u32(abuf) + row * 16;
  const int hw = p.hout * p.wout;
  float acc[N / 2];

  for (int item = blockIdx.x; item < p.n_items; item += gridDim.x) {
    const int half = item % S.split, tile = item / S.split;
    const int img = tile / p.tiles_per_image;
    const int pix0 = (tile - img * p.tiles_per_image) * kTileM + g * kWgRows;
    const int pix = pix0 + row;
    const bool valid = pix < hw;
    const int oy = valid ? pix / p.wout : 0, ox = valid ? pix - oy * p.wout : 0;
    const int iy0 = oy * S.stride - S.pad, ix0 = ox * S.stride - S.pad;
    const __half* src_img = p.in + static_cast<size_t>(img) * p.hin * p.win * CIN;
    // A of slab j into stage j % kLpAStages (one cp.async group per slab, empty past the last)
    auto gather = [&](int j) {
      if (j < SLABS) {
        const uint32_t dst = a_dst + (j % kLpAStages) * kLpABytes;
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int c = c0 + 2 * u, kc = j * kLpipsSlabChunks + c;
          const int tap = kc / CPT, cg = kc - tap * CPT;
          const int ky = tap / KS, kx = tap - ky * KS;
          const int iy = iy0 + ky, ix = ix0 + kx;
          const bool in = valid && kc < KCH && iy >= 0 && iy < p.hin && ix >= 0 && ix < p.win;
          const __half* src = in ? src_img + (static_cast<size_t>(iy) * p.win + ix) * CIN + cg * 8 : p.in;
          cp_async16(dst + c * kWgRows * 16, src, in ? 16u : 0u);
        }
      }
      cp_async_commit();
    };
    wg_bar(1 + g);   // every warp's MMAs of the previous item have retired before its A stages are rewritten
    gather(0);
    gather(1);
    uint32_t prev = 0;
#pragma unroll 1
    for (int j = 0; j < SLABS; ++j) {
      cp_async_wait<1>();          // slab j's chunks of this thread have landed
      fence_proxy_async_smem();
      wg_bar(1 + g);               // ... of every thread; and every warp has retired slab j - 2
      gather(j + 2);
      W.wait(&ring.full[ring.stage], ring.phase, 201);
      const uint64_t adesc = gmma_desc(smem_u32(abuf + (j % kLpAStages) * kLpABytes), kWgRows * 16, 128);
      const uint64_t bdesc = gmma_desc(smem_u32(ring.buf + ring.stage * kRingStageBytes), N * 16, 128);
      acc_fence(acc);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kLpipsSlabChunks / 2; ++k)
        lp_wgmma<N>(acc, gmma_desc_advance(adesc, k * 2 * kWgRows * 16), gmma_desc_advance(bdesc, k * 2 * N * 16), (j | k) ? 1u : 0u);
      wgmma_commit();
      if (j > 0) {   // slab j - 1 has retired: hand its weight stage back
        wgmma_wait<1>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&ring.empty[prev]);
      }
      prev = ring.stage;
      ring.next();
    }
    wgmma_wait<0>();
    acc_fence(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&ring.empty[prev]);
    cp_async_wait<0>();

    // epilogue: bias, ReLU, fp16 (saturating) NHWC; the largest value before the convert flags a clamped output
    const int r0 = acc_r0(), q = acc_q();
    const float* bias = p.bias + half * N;
    __half* out = p.out + static_cast<size_t>(img) * hw * S.cout + half * N;
    float vmax = 0.f;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int px = pix0 + r0 + 8 * i;
      if (px >= hw) continue;
      uint32_t* o = reinterpret_cast<uint32_t*>(out + static_cast<size_t>(px) * S.cout);
#pragma unroll
      for (int j = 0; j < N / 8; ++j) {
        const int col = 8 * j + 2 * q;
        const float a = acc[4 * j + 2 * i] + __ldg(bias + col), b = acc[4 * j + 2 * i + 1] + __ldg(bias + col + 1);
        vmax = fmaxf(vmax, fmaxf(a, b));
        o[col / 2] = pack_h2_relu_sat(a, b);
      }
    }
    if (__any_sync(0xffffffffu, vmax > kLpipsHalfMax) && lane == 0) atomicOr(p.sat + img, 1u << L);
  }
}

// ---- weight packing: OIHW fp32 -> [split][slabs * 8][n][8] fp16, K = [ky][kx][cin] ----
__global__ void lpips_pack_kernel(const float* __restrict__ w, LpipsConv s, __half* __restrict__ out) {
  const long long n_out = static_cast<long long>(s.w_bytes()) / 2;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= n_out) return;
  const int e = static_cast<int>(idx % 8);
  const int n = static_cast<int>((idx / 8) % s.n());
  const int kc = static_cast<int>((idx / (8 * s.n())) % (s.slabs() * kLpipsSlabChunks));
  const int half = static_cast<int>(idx / (8LL * s.n() * s.slabs() * kLpipsSlabChunks));
  const int k = kc * 8 + e, tap = k / s.cin, ci = k - tap * s.cin;
  const int ky = tap / s.ks, kx = tap - ky * s.ks, co = half * s.n() + n;
  const float v = (kc < s.k_chunks() && ci < s.cin_real) ? w[((static_cast<size_t>(co) * s.cin_real + ci) * s.ks + ky) * s.ks + kx] : 0.f;
  out[idx] = __float2half_rn(v);
}

// ---- input: mask, 2x - 1, (t - shift) / scale in fp32 (the reference's order), fp16 NHWC with channels 3..7 zero ----
__global__ void lpips_input_kernel(const float* __restrict__ gt, const float* __restrict__ gen, const uint8_t* __restrict__ mask,
                                   const float* __restrict__ shift, const float* __restrict__ scale, int fc, long long hw,
                                   __half* __restrict__ out) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= 2 * fc * hw) return;
  const long long b = idx / hw, px = idx - b * hw;
  const float* src = b < fc ? gt + (b * hw + px) * 3 : gen + ((b - fc) * hw + px) * 3;
  const bool m = mask[px] != 0;
  __half h[8];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float x = m ? 0.f : src[c];
    const float tv = __fsub_rn(__fmul_rn(2.f, x), 1.f);
    h[c] = __float2half_rn(__fdiv_rn(__fsub_rn(tv, __ldg(shift + c)), __ldg(scale + c)));
  }
#pragma unroll
  for (int c = 3; c < 8; ++c) h[c] = __float2half_rn(0.f);
  *reinterpret_cast<uint4*>(out + idx * 8) = *reinterpret_cast<const uint4*>(h);
}

// ---- 3 x 3 / 2 max-pool (floor), 8 channels per thread ----
__global__ void lpips_pool_kernel(const __half* __restrict__ in, __half* __restrict__ out, long long n, int hin, int win, int hout,
                                  int wout, int cchunks) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  const int c = static_cast<int>(idx % cchunks);
  const long long pix = idx / cchunks;
  const int ox = static_cast<int>(pix % wout), oy = static_cast<int>((pix / wout) % hout);
  const long long img = pix / (static_cast<long long>(wout) * hout);
  const __half* base = in + ((img * hin + 2 * oy) * win + 2 * ox) * (cchunks * 8) + c * 8;
  uint4 m = *reinterpret_cast<const uint4*>(base);
  __half2* mh = reinterpret_cast<__half2*>(&m);
#pragma unroll
  for (int dy = 0; dy < 3; ++dy)
#pragma unroll
    for (int dx = 0; dx < 3; ++dx) {
      const uint4 v = *reinterpret_cast<const uint4*>(base + (static_cast<long long>(dy) * win + dx) * (cchunks * 8));
      const __half2* vh = reinterpret_cast<const __half2*>(&v);
#pragma unroll
      for (int k = 0; k < 4; ++k) mh[k] = __hmax2(mh[k], vh[k]);
    }
  *reinterpret_cast<uint4*>(out + idx * 8) = m;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

// ---- per-tap distance: per pixel sum_c w[c] (g_c / (|g| + 1e-10) - r_c / (|r| + 1e-10))^2, in fp32; one warp per
// pixel, lanes over 8-channel chunks.  Block b of frame f sums pixels [256 b, 256 b + 256): warp w takes w, w + 8, ..
// in order, then the 8 warp sums in warp order (fp64), into partials[f][b].  The layout depends only on the frame size.
// kMap: lane 0 also stores the pixel's distance, the value added to the sum, into map[f][px] (spatial maps).
template <int C, bool kMap>
__device__ __forceinline__ void lpips_distance(const __half* __restrict__ feat, int fc, long long hw, const float* __restrict__ w,
                                               double* __restrict__ partials, int stride, float* __restrict__ map) {
  constexpr int kCh = C / 8, kPer = (kCh + 31) / 32;
  __shared__ double warp_sums[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, f = blockIdx.y;
  const __half* g = feat + static_cast<size_t>(f) * hw * C;
  const __half* r = feat + static_cast<size_t>(fc + f) * hw * C;
  float wl[kPer][8];
#pragma unroll
  for (int u = 0; u < kPer; ++u)
#pragma unroll
    for (int e = 0; e < 8; ++e) wl[u][e] = (lane + 32 * u < kCh) ? __ldg(w + (lane + 32 * u) * 8 + e) : 0.f;
  double sum = 0.0;
  for (int i = 0; i < kLpipsDistPixels / 8; ++i) {
    const long long px = static_cast<long long>(blockIdx.x) * kLpipsDistPixels + warp + 8 * i;
    if (px >= hw) break;
    float gv[kPer][8], rv[kPer][8];
    float sg = 0.f, sr = 0.f;
#pragma unroll
    for (int u = 0; u < kPer; ++u) {
      const int ch = lane + 32 * u;
      uint4 a = make_uint4(0, 0, 0, 0), b = make_uint4(0, 0, 0, 0);
      if (ch < kCh) {
        a = __ldg(reinterpret_cast<const uint4*>(g + px * C + ch * 8));
        b = __ldg(reinterpret_cast<const uint4*>(r + px * C + ch * 8));
      }
      const __half* ah = reinterpret_cast<const __half*>(&a);
      const __half* bh = reinterpret_cast<const __half*>(&b);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        gv[u][e] = __half2float(ah[e]);
        rv[u][e] = __half2float(bh[e]);
        sg = __fmaf_rn(gv[u][e], gv[u][e], sg);
        sr = __fmaf_rn(rv[u][e], rv[u][e], sr);
      }
    }
    const float ng = __fadd_rn(__fsqrt_rn(warp_sum(sg)), 1e-10f), nr = __fadd_rn(__fsqrt_rn(warp_sum(sr)), 1e-10f);
    float v = 0.f;
#pragma unroll
    for (int u = 0; u < kPer; ++u)
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float d = __fsub_rn(__fdiv_rn(gv[u][e], ng), __fdiv_rn(rv[u][e], nr));
        v = __fmaf_rn(wl[u][e], __fmul_rn(d, d), v);
      }
    v = warp_sum(v);
    if (kMap && lane == 0) map[static_cast<size_t>(f) * hw + px] = v;
    sum += static_cast<double>(v);
  }
  if (lane == 0) warp_sums[warp] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int k = 0; k < 8; ++k) s += warp_sums[k];
    partials[static_cast<size_t>(f) * stride + blockIdx.x] = s;
  }
}

template <int C>
__global__ void __launch_bounds__(256) lpips_distance_kernel(const __half* __restrict__ feat, int fc, long long hw,
                                                             const float* __restrict__ w, double* __restrict__ partials, int stride) {
  lpips_distance<C, false>(feat, fc, hw, w, partials, stride, nullptr);
}
template <int C>
__global__ void __launch_bounds__(256) lpips_distance_map_kernel(const __half* __restrict__ feat, int fc, long long hw,
                                                                 const float* __restrict__ w, double* __restrict__ partials,
                                                                 int stride, float* __restrict__ map) {
  lpips_distance<C, true>(feat, fc, hw, w, partials, stride, map);
}

// ---- spatial maps: one thread per output pixel of a chunk.  Per tap PyTorch's bilinear rule (align_corners=False, an
// explicit output size) in fp32 with every operation rounded on its own: src = max(scale (y + 0.5) - 0.5, 0), i0 = (int)
// src, i1 = i0 + (i0 < h_l - 1), l1 = src - i0, l0 = 1 - l1, v = hl0 (wl0 x00 + wl1 x01) + hl1 (wl0 x10 + wl1 x11); NaN
// from the frame's first clamped tap on; map = (((up_0 + up_1) + up_2) + up_3) + up_4.  The 4 neighbours of every tap
// map come from L2 (a 1008 x 756 frame's five maps are about 270 KB).
struct UpsampleAxis {
  int i0, i1;
  float l0, l1;
};
__device__ __forceinline__ UpsampleAxis upsample_axis(int dst, float scale, int n) {
  float src = __fsub_rn(__fmul_rn(scale, __fadd_rn(static_cast<float>(dst), 0.5f)), 0.5f);
  src = src < 0.f ? 0.f : src;
  UpsampleAxis a;
  a.i0 = static_cast<int>(src);
  a.i1 = a.i0 + (a.i0 < n - 1 ? 1 : 0);
  a.l1 = __fsub_rn(src, static_cast<float>(a.i0));
  a.l0 = __fsub_rn(1.f, a.l1);
  return a;
}

__global__ void __launch_bounds__(256) lpips_upsample_kernel(LpipsUpsampleParams p) {
  const long long hw = static_cast<long long>(p.H) * p.W;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= p.fc * hw) return;
  const int f = static_cast<int>(idx / hw);
  const long long px = idx - f * hw;
  const int y = static_cast<int>(px / p.W), x = static_cast<int>(px - static_cast<long long>(y) * p.W);
  const unsigned clamped = p.sat[f] | p.sat[p.fc + f];
  const int first = clamped ? __ffs(static_cast<int>(clamped)) - 1 : kLpipsTaps;
  float total = 0.f;
#pragma unroll
  for (int l = 0; l < kLpipsTaps; ++l) {
    const UpsampleAxis ay = upsample_axis(y, p.scale_y[l], p.h[l]), ax = upsample_axis(x, p.scale_x[l], p.w[l]);
    const float* t = p.tap[l] + static_cast<size_t>(f) * p.h[l] * p.w[l];
    const float* r0 = t + static_cast<size_t>(ay.i0) * p.w[l];
    const float* r1 = t + static_cast<size_t>(ay.i1) * p.w[l];
    const float top = __fadd_rn(__fmul_rn(ax.l0, __ldg(r0 + ax.i0)), __fmul_rn(ax.l1, __ldg(r0 + ax.i1)));
    const float bot = __fadd_rn(__fmul_rn(ax.l0, __ldg(r1 + ax.i0)), __fmul_rn(ax.l1, __ldg(r1 + ax.i1)));
    float v = __fadd_rn(__fmul_rn(ay.l0, top), __fmul_rn(ay.l1, bot));
    if (l >= first) v = __int_as_float(0x7fc00000);
    total = l == 0 ? v : __fadd_rn(total, v);
    if (p.layer_maps) p.layer_maps[(static_cast<size_t>(f) * kLpipsTaps + l) * hw + px] = v;
  }
  p.map[idx] = total;
  if (p.error_image) {
    const int k = lut_index(total);
    uint8_t* o = p.error_image + static_cast<size_t>(idx) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = c_jet.rgb8[k * 3 + c];
  }
}

struct TapCounts {
  int blocks[kLpipsTaps];
  double px[kLpipsTaps];
};

// per frame: the tap means (block partials in block order, fp64) and their sum in tap order; NaN from the first tap
// whose convolution clamped an output of either image of the frame on
__global__ void lpips_reduce_kernel(const double* __restrict__ partials, const unsigned* __restrict__ sat, int fc, int stride,
                                    TapCounts tc, float* __restrict__ lpips, float* __restrict__ per_layer) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= fc) return;
  const unsigned clamped = sat[f] | sat[fc + f];
  const int first = clamped ? __ffs(static_cast<int>(clamped)) - 1 : kLpipsTaps;
  double total = 0.0;
  for (int k = 0; k < kLpipsTaps; ++k) {
    const double* p = partials + (static_cast<size_t>(k) * fc + f) * stride;
    double s = 0.0;
    for (int b = 0; b < tc.blocks[k]; ++b) s += p[b];
    const double mean = k < first ? s / tc.px[k] : __longlong_as_double(0x7ff8000000000000LL);
    if (per_layer) per_layer[f * kLpipsTaps + k] = static_cast<float>(mean);
    total += mean;
  }
  lpips[f] = static_cast<float>(total);
}

template <int L>
cudaError_t launch_conv_layer(const LpipsDims& d, const __half* in, __half* out, const uint8_t* packed, int n_images, int num_sms,
                              int* err, unsigned* sat, cudaStream_t st) {
  constexpr LpipsConv S = kLpipsConv[L];
  constexpr int kInStage[kLpipsTaps] = {0, 2, 4, 5, 6};
  const int so = kInStage[L], si = kLpipsTapStage[L];
  ConvParams p;
  p.in = in;
  p.out = out;
  p.w = packed + lpips_w_off(L);
  p.bias = reinterpret_cast<const float*>(packed + kLpipsBiasOff) + lpips_c_off(L);
  p.hin = d.h[so]; p.win = d.w[so]; p.hout = d.h[si]; p.wout = d.w[si];
  p.tiles_per_image = static_cast<int>((d.px(si) + kTileM - 1) / kTileM);
  const long long items = static_cast<long long>(n_images) * p.tiles_per_image * S.split;
  p.n_items = static_cast<int>(items);
  p.err = err;
  p.sat = sat;
  if (items <= 0) return cudaSuccess;
  const cudaError_t e = cudaFuncSetAttribute(lpips_conv_kernel<L>, cudaFuncAttributeMaxDynamicSharedMemorySize, kLpConvSmem);
  if (e != cudaSuccess) return e;
  lpips_conv_kernel<L><<<items < num_sms ? static_cast<int>(items) : num_sms, kFwdThreads, kLpConvSmem, st>>>(p);
  return cudaGetLastError();
}

int blocks_of(long long n, int per) { return static_cast<int>((n + per - 1) / per); }
size_t align256(size_t v) { return (v + 255) / 256 * 256; }

}  // namespace

LpipsDims lpips_dims(int H, int W) {
  LpipsDims d{};
  d.h[0] = H; d.w[0] = W;
  auto conv = [](int n, const LpipsConv& s) { return (n + 2 * s.pad - s.ks) / s.stride + 1; };
  auto pool = [](int n) { return n >= 3 ? (n - 3) / 2 + 1 : 0; };
  d.h[1] = conv(H, kLpipsConv[0]); d.w[1] = conv(W, kLpipsConv[0]);
  d.h[2] = pool(d.h[1]); d.w[2] = pool(d.w[1]);
  d.h[3] = conv(d.h[2], kLpipsConv[1]); d.w[3] = conv(d.w[2], kLpipsConv[1]);
  d.h[4] = pool(d.h[3]); d.w[4] = pool(d.w[3]);
  for (int s = 5; s < kLpipsStages; ++s) { d.h[s] = d.h[4]; d.w[s] = d.w[4]; }
  return d;
}

size_t lpips_mask_bytes(int H, int W) { return align256(static_cast<size_t>(H) * W); }

static int max_dist_blocks(const LpipsDims& d) {
  int m = 0;
  for (int k = 0; k < kLpipsTaps; ++k) m = d.dist_blocks(k) > m ? d.dist_blocks(k) : m;
  return m;
}

size_t lpips_frame_bytes(int H, int W) {
  const LpipsDims d = lpips_dims(H, W);
  size_t b = 0;
  for (int s = 0; s < kLpipsStages; ++s) b += align256(2 * static_cast<size_t>(d.image_bytes(s)));
  return b + align256(static_cast<size_t>(kLpipsTaps) * max_dist_blocks(d) * sizeof(double) + 2 * sizeof(unsigned));
}

LpipsChunk lpips_chunk(void* ws, int fc, int H, int W) {
  const LpipsDims d = lpips_dims(H, W);
  LpipsChunk c{};
  c.fc = fc;
  c.max_blocks = max_dist_blocks(d);
  uint8_t* p = static_cast<uint8_t*>(ws) + lpips_mask_bytes(H, W);
  for (int s = 0; s < kLpipsStages; ++s) {
    c.act[s] = reinterpret_cast<__half*>(p);
    p += align256(2 * static_cast<size_t>(fc) * d.image_bytes(s));
  }
  c.partials = reinterpret_cast<double*>(p);
  c.sat = reinterpret_cast<unsigned*>(c.partials + static_cast<size_t>(kLpipsTaps) * fc * c.max_blocks);
  return c;
}

// align256(fc * b) <= fc * align256(b) for fc >= 1, so fc map frames hold a chunk's buffers and its tap maps
size_t lpips_map_frame_bytes(int H, int W) {
  const LpipsDims d = lpips_dims(H, W);
  size_t b = lpips_frame_bytes(H, W);
  for (int k = 0; k < kLpipsTaps; ++k) b += align256(static_cast<size_t>(d.px(kLpipsTapStage[k])) * sizeof(float));
  return b;
}

float* lpips_tap_map(void* ws, int fc, int H, int W, int tap) {
  const LpipsDims d = lpips_dims(H, W);
  uint8_t* p = static_cast<uint8_t*>(ws) + lpips_mask_bytes(H, W) + static_cast<size_t>(fc) * lpips_frame_bytes(H, W);
  for (int k = 0; k < tap; ++k) p += align256(static_cast<size_t>(fc) * d.px(kLpipsTapStage[k]) * sizeof(float));
  return reinterpret_cast<float*>(p);
}

cudaError_t launch_lpips_pack(const LpipsPackSources& s, uint8_t* packed, cudaStream_t st) {
  for (int l = 0; l < kLpipsTaps; ++l) {
    const long long n = kLpipsConv[l].w_bytes() / 2;
    lpips_pack_kernel<<<blocks_of(n, 256), 256, 0, st>>>(s.conv_w[l], kLpipsConv[l], reinterpret_cast<__half*>(packed + lpips_w_off(l)));
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    const size_t bytes = kLpipsConv[l].cout * sizeof(float);
    e = cudaMemcpyAsync(packed + kLpipsBiasOff + lpips_c_off(l) * 4, s.conv_b[l], bytes, cudaMemcpyDeviceToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(packed + kLpipsLinOff + lpips_c_off(l) * 4, s.lin[l], bytes, cudaMemcpyDeviceToDevice, st);
    if (e != cudaSuccess) return e;
  }
  cudaError_t e = cudaMemcpyAsync(packed + kLpipsShiftOff, s.shift, 12, cudaMemcpyDeviceToDevice, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(packed + kLpipsScaleOff, s.scale, 12, cudaMemcpyDeviceToDevice, st);
  return e;
}

cudaError_t launch_lpips_input(const float* gt, const float* gen, const uint8_t* mask, const uint8_t* packed, int fc, int H, int W,
                               __half* out, cudaStream_t st) {
  const long long hw = static_cast<long long>(H) * W;
  lpips_input_kernel<<<blocks_of(2 * fc * hw, 256), 256, 0, st>>>(gt, gen, mask, reinterpret_cast<const float*>(packed + kLpipsShiftOff),
                                                                   reinterpret_cast<const float*>(packed + kLpipsScaleOff), fc, hw, out);
  return cudaGetLastError();
}

cudaError_t launch_lpips_conv(int layer, const LpipsDims& d, const __half* in, __half* out, const uint8_t* packed, int n_images,
                              int num_sms, int* err, unsigned* sat, cudaStream_t st) {
  switch (layer) {
    case 0: return launch_conv_layer<0>(d, in, out, packed, n_images, num_sms, err, sat, st);
    case 1: return launch_conv_layer<1>(d, in, out, packed, n_images, num_sms, err, sat, st);
    case 2: return launch_conv_layer<2>(d, in, out, packed, n_images, num_sms, err, sat, st);
    case 3: return launch_conv_layer<3>(d, in, out, packed, n_images, num_sms, err, sat, st);
    default: return launch_conv_layer<4>(d, in, out, packed, n_images, num_sms, err, sat, st);
  }
}

cudaError_t launch_lpips_pool(const __half* in, __half* out, int n_images, int hin, int win, int hout, int wout, int channels,
                              cudaStream_t st) {
  const long long n = static_cast<long long>(n_images) * hout * wout * (channels / 8);
  if (n == 0) return cudaSuccess;
  lpips_pool_kernel<<<blocks_of(n, 256), 256, 0, st>>>(in, out, n, hin, win, hout, wout, channels / 8);
  return cudaGetLastError();
}

cudaError_t launch_lpips_distance(int tap, const LpipsDims& d, const LpipsChunk& c, const uint8_t* packed, cudaStream_t st) {
  const int s = kLpipsTapStage[tap];
  const dim3 grid(d.dist_blocks(tap), c.fc);
  const float* w = reinterpret_cast<const float*>(packed + kLpipsLinOff) + lpips_c_off(tap);
  double* part = c.partials + static_cast<size_t>(tap) * c.fc * c.max_blocks;
  const long long hw = d.px(s);
  switch (tap) {
    case 0: lpips_distance_kernel<64><<<grid, 256, 0, st>>>(c.act[s], c.fc, hw, w, part, c.max_blocks); break;
    case 1: lpips_distance_kernel<192><<<grid, 256, 0, st>>>(c.act[s], c.fc, hw, w, part, c.max_blocks); break;
    case 2: lpips_distance_kernel<384><<<grid, 256, 0, st>>>(c.act[s], c.fc, hw, w, part, c.max_blocks); break;
    default: lpips_distance_kernel<256><<<grid, 256, 0, st>>>(c.act[s], c.fc, hw, w, part, c.max_blocks); break;
  }
  return cudaGetLastError();
}

cudaError_t launch_lpips_reduce(const LpipsDims& d, const LpipsChunk& c, float* lpips, float* per_layer, cudaStream_t st) {
  TapCounts tc;
  for (int k = 0; k < kLpipsTaps; ++k) {
    tc.blocks[k] = d.dist_blocks(k);
    tc.px[k] = static_cast<double>(d.px(kLpipsTapStage[k]));
  }
  lpips_reduce_kernel<<<blocks_of(c.fc, 128), 128, 0, st>>>(c.partials, c.sat, c.fc, c.max_blocks, tc, lpips, per_layer);
  return cudaGetLastError();
}

cudaError_t launch_lpips_distance_map(int tap, const LpipsDims& d, const LpipsChunk& c, const uint8_t* packed, float* tap_map,
                                      cudaStream_t st) {
  const int s = kLpipsTapStage[tap];
  const dim3 grid(d.dist_blocks(tap), c.fc);
  const float* w = reinterpret_cast<const float*>(packed + kLpipsLinOff) + lpips_c_off(tap);
  double* part = c.partials + static_cast<size_t>(tap) * c.fc * c.max_blocks;
  const long long hw = d.px(s);
  switch (tap) {
    case 0: lpips_distance_map_kernel<64><<<grid, 256, 0, st>>>(c.act[s], c.fc, hw, w, part, c.max_blocks, tap_map); break;
    case 1: lpips_distance_map_kernel<192><<<grid, 256, 0, st>>>(c.act[s], c.fc, hw, w, part, c.max_blocks, tap_map); break;
    case 2: lpips_distance_map_kernel<384><<<grid, 256, 0, st>>>(c.act[s], c.fc, hw, w, part, c.max_blocks, tap_map); break;
    default: lpips_distance_map_kernel<256><<<grid, 256, 0, st>>>(c.act[s], c.fc, hw, w, part, c.max_blocks, tap_map); break;
  }
  return cudaGetLastError();
}

cudaError_t launch_lpips_upsample(const LpipsUpsampleParams& p, cudaStream_t st) {
  const long long n = static_cast<long long>(p.fc) * p.H * p.W;
  if (n == 0) return cudaSuccess;
  lpips_upsample_kernel<<<blocks_of(n, 256), 256, 0, st>>>(p);
  return cudaGetLastError();
}

}  // namespace nrn
