// Per-ray operations of the volumetric renderer: one warp per ray, scans by warp shuffle.
//   sample_coarse_kernel      <- render_rays sampling part            (train.py:847-869)
//   composite_kernel          <- raw2outputs                          (train.py:724-789)
//                                + sample_pdf                         (run_nerf_helpers.py:651-698)
//                                + sort(cat[z, z_samples]) and z_std  (train.py:920, 959)
//   sample_pdf_kernel         <- sample_pdf stand-alone (op-level parity)
//   composite_bwd_kernel      <- autograd of raw2outputs w.r.t. raw (SURVEY.md appendix C)
// These are HBM/latency-bound streaming kernels (a few KB per ray); everything a ray needs lives in
// registers / a few hundred bytes of shared memory.
#include "nrn_common.cuh"
#include "ray_ops.cuh"

namespace nrn {

namespace {

constexpr int kWarpsPerBlock = 4;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// inclusive product scan over the warp
__device__ __forceinline__ float warp_scan_mul(float v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v *= t;
  }
  return v;
}
__device__ __forceinline__ float warp_scan_add(float v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  return v;
}
// torch.linspace(0, 1, S)[i] for float32 as the CUDA backend evaluates it (aten RangeFactories.cu:
// start + step*i below the midpoint, end - step*(S-1-i) above, each contracted to one FMA)
__device__ __forceinline__ float linspace01(int i, int S) {
  if (S == 1) return 0.f;
  const float step = 1.0f / static_cast<float>(S - 1);
  return i < S / 2 ? __fmul_rn(step, static_cast<float>(i)) : fmaf(-step, static_cast<float>(S - 1 - i), 1.0f);
}
__device__ __forceinline__ float z_at(float near, float far, int i, int S, int lindisp) {
  const float t = linspace01(i, S);
  if (!lindisp) return __fadd_rn(__fmul_rn(near, __fsub_rn(1.0f, t)), __fmul_rn(far, t));
  return __fdiv_rn(1.0f, __fadd_rn(__fmul_rn(__fdiv_rn(1.0f, near), __fsub_rn(1.0f, t)), __fmul_rn(__fdiv_rn(1.0f, far), t)));
}

}  // namespace

// z_vals[n][i]; stratified jitter when t_rand != null (train.py:855-869)
__global__ void sample_coarse_kernel(const float* __restrict__ rays, const float* __restrict__ t_rand, int n, int S,
                                     int lindisp, float* __restrict__ z_out) {
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= static_cast<long long>(n) * S) return;
  const int ray = static_cast<int>(idx / S), i = static_cast<int>(idx - static_cast<long long>(ray) * S);
  const float near = rays[ray * 8 + 6], far = rays[ray * 8 + 7];
  const float z = z_at(near, far, i, S, lindisp);
  if (!t_rand) { z_out[idx] = z; return; }
  const float zp = i > 0 ? z_at(near, far, i - 1, S, lindisp) : z;
  const float zn = i < S - 1 ? z_at(near, far, i + 1, S, lindisp) : z;
  const float lower = i > 0 ? __fmul_rn(0.5f, __fadd_rn(z, zp)) : z;
  const float upper = i < S - 1 ? __fmul_rn(0.5f, __fadd_rn(zn, z)) : z;
  z_out[idx] = __fadd_rn(lower, __fmul_rn(__fsub_rn(upper, lower), t_rand[idx]));
}

// ------------------------------------------------------------------------------------------------
// Inverse-CDF sampling of one ray by one warp.  bins[nb], w[nb-1] -> out[n_samp].
// cdf is built in shared memory (cdf_s, nb entries).  Semantics follow run_nerf_helpers.py:651-698:
// +1e-5 on the weights, searchsorted(right=False), index clamps, denom < 1e-5 -> 1.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void warp_sample_pdf(const float* bins_s, const float* w_s, int nb, float* cdf_s,
                                                const float* __restrict__ u, int n_samp, float* out, int lane) {
  const int nw = nb - 1;
  float part = 0.f;
  for (int j = lane; j < nw; j += 32) part += w_s[j] + 1e-5f;
  const float total = warp_sum(part);
  float carry = 0.f;
  if (lane == 0) cdf_s[0] = 0.f;
  for (int j0 = 0; j0 < nw; j0 += 32) {
    const int j = j0 + lane;
    const float pdf = j < nw ? (w_s[j] + 1e-5f) / total : 0.f;
    const float inc = warp_scan_add(pdf, lane) + carry;
    if (j < nw) cdf_s[j + 1] = inc;
    carry = __shfl_sync(0xffffffffu, inc, 31);
  }
  __syncwarp();
  for (int i = lane; i < n_samp; i += 32) {
    const float uu = u ? u[i] : (n_samp == 1 ? 0.f : linspace01(i, n_samp));
    int lo = 0, hi = nb;  // first index with cdf[idx] >= uu
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (cdf_s[mid] < uu) lo = mid + 1; else hi = mid;
    }
    const int below = max(0, lo - 1), above = min(nb - 1, lo);
    const float cb = cdf_s[below], ca = cdf_s[above];
    float denom = ca - cb;
    if (denom < 1e-5f) denom = 1.0f;
    const float t = (uu - cb) / denom;
    out[i] = bins_s[below] + t * (bins_s[above] - bins_s[below]);
  }
  __syncwarp();
}

// ------------------------------------------------------------------------------------------------
// raw2outputs for one pass, optionally followed (coarse pass) by importance resampling:
//   z_out[n][S + n_imp] = sort(cat[z, sample_pdf(z_mid, w[1:-1])]),  z_std[n]
// Shared memory per warp: z[S] w[S] cdf[S] all[S + n_imp]
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
composite_kernel(const CompositeParams p) {
  extern __shared__ float sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ray = blockIdx.x * kWarpsPerBlock + warp;
  if (ray >= p.n) return;
  const int S = p.S, T = S + p.n_imp;
  float* z_s = sm + static_cast<size_t>(warp) * (3 * S + T);
  float* w_s = z_s + S;
  float* cdf_s = w_s + S;
  float* all_s = cdf_s + S;

  const float* d = p.rays_d + static_cast<long long>(ray) * p.rays_d_stride;
  const float dx = d[0], dy = d[1], dz = d[2];
  const float dnorm = ray_dnorm(dx, dy, dz);
  const float* zr = p.z + static_cast<long long>(ray) * S;
  const float* rawr = p.raw + static_cast<long long>(ray) * S * p.C;
  for (int i = lane; i < S; i += 32) z_s[i] = zr[i];
  __syncwarp();

  float carry = 1.0f, acc_r = 0.f, acc_g = 0.f, acc_b = 0.f, acc_d = 0.f, acc_w = 0.f;
  for (int i0 = 0; i0 < S; i0 += 32) {
    const int i = i0 + lane;
    float alpha = 0.f, r = 0.f, g = 0.f, b = 0.f, zi = 0.f;
    if (i < S) {
      zi = z_s[i];
      const float gap = i + 1 < S ? z_s[i + 1] - zi : 1e10f;            // train.py:743-748
      const float* q = rawr + static_cast<long long>(i) * p.C;
      float sigma = q[3];
      if (p.noise) sigma += p.noise[static_cast<long long>(ray) * S + i];  // noise already scaled by raw_noise_std
      alpha = composite_alpha(sigma, gap, dnorm);                      // :740-741, 761
      r = 1.0f / (1.0f + expf(-q[0]));
      g = 1.0f / (1.0f + expf(-q[1]));
      b = 1.0f / (1.0f + expf(-q[2]));
    }
    const float om = i < S ? 1.0f - alpha + 1e-10f : 1.0f;             // :769
    const float incl = warp_scan_mul(om, lane);
    float excl = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) excl = 1.0f;
    const float T_i = carry * excl;
    const float w = alpha * T_i;
    carry *= __shfl_sync(0xffffffffu, incl, 31);
    if (i < S) {
      w_s[i] = w;
      if (p.weights) p.weights[static_cast<long long>(ray) * S + i] = w;
      if (p.alpha) p.alpha[static_cast<long long>(ray) * S + i] = alpha;
    }
    acc_r += w * r; acc_g += w * g; acc_b += w * b; acc_d += w * zi; acc_w += w;
  }
  acc_r = warp_sum(acc_r); acc_g = warp_sum(acc_g); acc_b = warp_sum(acc_b);
  acc_d = warp_sum(acc_d); acc_w = warp_sum(acc_w);
  if (lane == 0) {
    const float bg = p.white_bkgd ? 1.0f - acc_w : 0.f;                // :786-787
    p.rgb[ray * 3 + 0] = acc_r + bg; p.rgb[ray * 3 + 1] = acc_g + bg; p.rgb[ray * 3 + 2] = acc_b + bg;
    p.acc[ray] = acc_w;
    if (p.depth) p.depth[ray] = acc_d;
    const float q = acc_d / acc_w;                                     // :781-784; 0/0 = NaN when acc == 0 and
    p.disp[ray] = 1.0f / (q != q ? q : fmaxf(1e-10f, q));              // torch.max propagates it (fmaxf would not)
  }
  if (p.n_imp <= 0) return;
  __syncwarp();

  // ---- hierarchical resampling: bins = z_mid (S-1), weights = w[1:-1] (S-2)  (train.py:910-918) ----
  float* bins_s = all_s;  // temporarily: S-1 midpoints
  for (int j = lane; j < S - 1; j += 32) bins_s[j] = 0.5f * (z_s[j + 1] + z_s[j]);
  __syncwarp();
  // the new samples are staged in the tail of this ray's output row (each lane re-reads only the
  // entries it wrote itself), so they alias neither bins, cdf nor w
  float* zout = p.z_out + static_cast<long long>(ray) * T;
  warp_sample_pdf(bins_s, w_s + 1, S - 1, cdf_s, p.u ? p.u + static_cast<long long>(ray) * p.n_imp : nullptr,
                  p.n_imp, zout + S, lane);
  // z_std (population std over the new samples, train.py:959)
  float s1 = 0.f;
  for (int i = lane; i < p.n_imp; i += 32) s1 += zout[S + i];
  const float mean = warp_sum(s1) / static_cast<float>(p.n_imp);
  float s2 = 0.f;
  for (int i = lane; i < p.n_imp; i += 32) { const float t = zout[S + i] - mean; s2 += t * t; }
  s2 = warp_sum(s2);
  if (lane == 0 && p.z_std) p.z_std[ray] = sqrtf(s2 / static_cast<float>(p.n_imp));
  // ---- merge: sort(cat[z, samples]) by stable rank counting (train.py:920) ----
  for (int i = lane; i < S; i += 32) all_s[i] = z_s[i];
  for (int i = lane; i < p.n_imp; i += 32) all_s[S + i] = zout[S + i];
  __syncwarp();
  for (int e = lane; e < T; e += 32) {
    const float v = all_s[e];
    int rank = 0;
    for (int j = 0; j < T; ++j) {
      const float x = all_s[j];
      rank += (x < v) || (x == v && j < e);
    }
    zout[rank] = v;
  }
}

// stand-alone sample_pdf (op-level parity with run_nerf_helpers.py:651-698)
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
sample_pdf_kernel(const float* __restrict__ bins, const float* __restrict__ weights, const float* __restrict__ u,
                  int n, int nb, int n_samp, float* __restrict__ out) {
  extern __shared__ float sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ray = blockIdx.x * kWarpsPerBlock + warp;
  if (ray >= n) return;
  float* bins_s = sm + static_cast<size_t>(warp) * (3 * nb);
  float* w_s = bins_s + nb;
  float* cdf_s = w_s + nb;
  for (int j = lane; j < nb; j += 32) bins_s[j] = bins[static_cast<long long>(ray) * nb + j];
  for (int j = lane; j < nb - 1; j += 32) w_s[j] = weights[static_cast<long long>(ray) * (nb - 1) + j];
  __syncwarp();
  warp_sample_pdf(bins_s, w_s, nb, cdf_s, u ? u + static_cast<long long>(ray) * n_samp : nullptr, n_samp,
                  out + static_cast<long long>(ray) * n_samp, lane);
}

// ------------------------------------------------------------------------------------------------
// Backward of raw2outputs w.r.t. raw, for upstream gradients on rgb_map (and optionally acc / depth
// are not used by the training loss: SURVEY.md appendix C).  Closed forms:
//   g_i   = sum_c dL/drgb_c * rgb_ic (+ dL/dacc + dL/ddepth * z_i)      = dL/dw_i
//   dL/dalpha_i = g_i T_i - (sum_{k>i} g_k w_k) / (1 - alpha_i + 1e-10)
//   dalpha/dsigma = dist (1 - alpha) [sigma + noise > 0]
//   dL/draw_ic = w_i dL/drgb_c s (1 - s)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
composite_bwd_kernel(const CompositeBwdParams p) {
  extern __shared__ float sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ray = blockIdx.x * kWarpsPerBlock + warp;
  if (ray >= p.n) return;
  const int S = p.S;
  float* gw_s = sm + static_cast<size_t>(warp) * S;  // g_i * w_i
  const float* d = p.rays_d + static_cast<long long>(ray) * p.rays_d_stride;
  const float dnorm = ray_dnorm(d[0], d[1], d[2]);
  const float* zr = p.z + static_cast<long long>(ray) * S;
  const float* rawr = p.raw + static_cast<long long>(ray) * S * p.C;
  float* outr = p.d_raw + static_cast<long long>(ray) * S * p.C;
  const float gr = p.d_rgb[ray * 3 + 0], gg = p.d_rgb[ray * 3 + 1], gb = p.d_rgb[ray * 3 + 2];
  const float ga = p.d_acc ? p.d_acc[ray] : 0.f;
  float g_white = 0.f;
  if (p.white_bkgd) g_white = -(gr + gg + gb);  // rgb_map += 1 - acc
  // pass 1 (forward order): weights, transmittance; stash per-sample quantities in registers is not
  // possible for arbitrary S, so recompute in pass 2; here we need suffix sums of g_k w_k.
  float carry = 1.0f;
  for (int i0 = 0; i0 < S; i0 += 32) {
    const int i = i0 + lane;
    float alpha = 0.f, gi = 0.f;
    if (i < S) {
      const float zi = zr[i];
      const float gap = i + 1 < S ? zr[i + 1] - zi : 1e10f;
      const float* q = rawr + static_cast<long long>(i) * p.C;
      float sigma = q[3];
      if (p.noise) sigma += p.noise[static_cast<long long>(ray) * S + i];
      alpha = composite_alpha(sigma, gap, dnorm);
      const float r = 1.0f / (1.0f + expf(-q[0])), g = 1.0f / (1.0f + expf(-q[1])), b = 1.0f / (1.0f + expf(-q[2]));
      gi = gr * r + gg * g + gb * b + ga + g_white;
    }
    const float om = i < S ? 1.0f - alpha + 1e-10f : 1.0f;
    const float incl = warp_scan_mul(om, lane);
    float excl = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) excl = 1.0f;
    const float T_i = carry * excl;
    carry *= __shfl_sync(0xffffffffu, incl, 31);
    if (i < S) gw_s[i] = gi * alpha * T_i;
  }
  __syncwarp();
  // suffix sums: suffix[i] = sum_{k>i} gw[k], computed chunk-wise from the back
  float tail = 0.f;  // sum over all later chunks
  const int nchunks = (S + 31) / 32;
  // second forward recomputation fused with the suffix scan, chunk by chunk from the end
  for (int c = nchunks - 1; c >= 0; --c) {
    const int i = c * 32 + lane;
    const float v = i < S ? gw_s[i] : 0.f;
    // inclusive suffix within the chunk: reverse scan
    float s = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float t = __shfl_down_sync(0xffffffffu, s, o);
      if (lane + o < 32) s += t;
    }
    const float suffix_excl = s - v + tail;  // sum_{k>i}
    tail += __shfl_sync(0xffffffffu, s, 0);
    if (i < S) gw_s[i] = suffix_excl;        // overwrite with the exclusive suffix sum
  }
  __syncwarp();
  carry = 1.0f;
  for (int i0 = 0; i0 < S; i0 += 32) {
    const int i = i0 + lane;
    float alpha = 0.f;
    float dist = 0.f, sig = 0.f, r = 0.f, g = 0.f, b = 0.f;
    if (i < S) {
      const float zi = zr[i];
      dist = (i + 1 < S ? zr[i + 1] - zi : 1e10f) * dnorm;
      const float* q = rawr + static_cast<long long>(i) * p.C;
      sig = q[3];
      if (p.noise) sig += p.noise[static_cast<long long>(ray) * S + i];
      alpha = 1.0f - expf(-fmaxf(sig, 0.f) * dist);
      r = 1.0f / (1.0f + expf(-q[0])); g = 1.0f / (1.0f + expf(-q[1])); b = 1.0f / (1.0f + expf(-q[2]));
    }
    const float om = i < S ? 1.0f - alpha + 1e-10f : 1.0f;
    const float incl = warp_scan_mul(om, lane);
    float excl = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) excl = 1.0f;
    const float T_i = carry * excl;
    carry *= __shfl_sync(0xffffffffu, incl, 31);
    if (i < S) {
      const float w = alpha * T_i;
      const float gi = gr * r + gg * g + gb * b + ga + g_white;
      const float dalpha = gi * T_i - gw_s[i] / om;
      // d alpha / d sigma = dist * exp(-relu(sigma) dist) for sigma > 0 (autograd of train.py:741)
      const float dsig = sig > 0.f ? dalpha * dist * expf(-sig * dist) : 0.f;
      float* o = outr + static_cast<long long>(i) * p.C;
      o[0] = w * gr * r * (1.0f - r);
      o[1] = w * gg * g * (1.0f - g);
      o[2] = w * gb * b * (1.0f - b);
      o[3] = dsig;
      for (int c = 4; c < p.C; ++c) o[c] = 0.f;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Ray generation (get_rays / get_rays_np, run_nerf_helpers.py:588-622) for whole frames or for a random batch of
// (image, x, y) pixels (train.py:1498-1517 builds a host table of every ray of every image and train.py:1546-1564
// gathers N_rand rows of it per step; here the rows are computed on demand from the 3x4 poses and the intrinsics).
//   dirs = [(x - cx) / fx, -(y - cy) / fy, -1];  rays_d[r] = dirs . c2w[r, :3]  (sum over the three products in index
//   order, no FMA contraction: bit-identical to numpy's / torch's float32 evaluation);  rays_o = c2w[:, 3]
__device__ __forceinline__ void ray_from_pixel(const float* __restrict__ c2w, const float* __restrict__ K, float x, float y,
                                               float* __restrict__ o, float* __restrict__ d) {
  const float dx = __fdiv_rn(__fsub_rn(x, K[2]), K[0]);
  const float dy = -__fdiv_rn(__fsub_rn(y, K[3]), K[1]);
  const float dz = -1.0f;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    d[r] = __fadd_rn(__fadd_rn(__fmul_rn(dx, c2w[r * 4 + 0]), __fmul_rn(dy, c2w[r * 4 + 1])), __fmul_rn(dz, c2w[r * 4 + 2]));
    o[r] = c2w[r * 4 + 3];
  }
}

// one frame: pixel (row j, column i) -> ray j * W + i  (the [H, W, 3] layout of get_rays)
__global__ void get_rays_kernel(const float* __restrict__ c2w, const float* __restrict__ K, int H, int W, float* __restrict__ rays_o,
                                float* __restrict__ rays_d) {
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= static_cast<long long>(H) * W) return;
  const int j = static_cast<int>(idx / W), i = static_cast<int>(idx - static_cast<long long>(j) * W);
  float o[3], d[3];
  ray_from_pixel(c2w, K, static_cast<float>(i), static_cast<float>(j), o, d);
#pragma unroll
  for (int r = 0; r < 3; ++r) { rays_o[idx * 3 + r] = o[r]; rays_d[idx * 3 + r] = d[r]; }
}

// a training batch: pix [n][3] = (image, x, y) int64 (the reference's batch_pixel_indices); poses [n_img][3][4];
// intrinsics [n_views][4] = (fx, fy, cx, cy), view of an image through image_to_view (or view 0 when null);
// images [n_img][H][W][3] fp32 -> target [n][3]
__global__ void ray_batch_kernel(const long long* __restrict__ pix, int n, const float* __restrict__ poses, const float* __restrict__ K,
                                 const int* __restrict__ image_to_view, const float* __restrict__ images, int H, int W,
                                 float* __restrict__ rays_o, float* __restrict__ rays_d, float* __restrict__ target) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  const long long img = pix[idx * 3 + 0], x = pix[idx * 3 + 1], y = pix[idx * 3 + 2];
  const int view = image_to_view ? image_to_view[img] : 0;
  float o[3], d[3];
  ray_from_pixel(poses + img * 12, K + view * 4, static_cast<float>(x), static_cast<float>(y), o, d);
#pragma unroll
  for (int r = 0; r < 3; ++r) { rays_o[idx * 3 + r] = o[r]; rays_d[idx * 3 + r] = d[r]; }
  if (images && target) {
    const float* px = images + ((img * H + y) * W + x) * 3;
#pragma unroll
    for (int r = 0; r < 3; ++r) target[idx * 3 + r] = px[r];
  }
}

// ------------------------------------------------------------------------------------------------
// Free-viewpoint post-processing (free_viewpoint_rendering.py:623-629): per pixel the sample whose accumulated
// visibility is closest to 0.5 -- "most likely on the visible surface".  cumsum in index order (one thread per ray, the
// order of a sequential cumsum), first minimum wins like torch.min.
__global__ void median_index_kernel(const float* __restrict__ w, int n, int S, long long* __restrict__ idx_out) {
  const int ray = blockIdx.x * blockDim.x + threadIdx.x;
  if (ray >= n) return;
  const float* row = w + static_cast<long long>(ray) * S;
  float acc = 0.f, best = 3.0e38f;
  int arg = 0;
  for (int i = 0; i < S; ++i) {
    acc = __fadd_rn(acc, row[i]);
    const float dist = fabsf(__fsub_rn(acc, 0.5f));
    if (dist < best) { best = dist; arg = i; }
  }
  idx_out[ray] = arg;
}

// rays [n][8] = (o, d, near, far) from rays_o / rays_d [n][3] and scalar near / far (render, train.py:393-398: four small
// PyTorch kernels and a concatenation there)
__global__ void pack_rays_kernel(const float* __restrict__ o, const float* __restrict__ d, float near, float far, int n, float* __restrict__ rays) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float* r = rays + static_cast<long long>(i) * 8;
  r[0] = o[i * 3]; r[1] = o[i * 3 + 1]; r[2] = o[i * 3 + 2];
  r[3] = d[i * 3]; r[4] = d[i * 3 + 1]; r[5] = d[i * 3 + 2];
  r[6] = near; r[7] = far;
}
cudaError_t launch_pack_rays(const float* o, const float* d, float near, float far, int n, float* rays, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  pack_rays_kernel<<<(n + 255) / 256, 256, 0, st>>>(o, d, near, far, n, rays);
  return cudaGetLastError();
}

cudaError_t launch_get_rays(const float* c2w, const float* K, int H, int W, float* rays_o, float* rays_d, cudaStream_t st) {
  const long long total = static_cast<long long>(H) * W;
  if (total == 0) return cudaSuccess;
  get_rays_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(c2w, K, H, W, rays_o, rays_d);
  return cudaGetLastError();
}
cudaError_t launch_ray_batch(const long long* pix, int n, const float* poses, const float* K, const int* image_to_view,
                             const float* images, int H, int W, float* rays_o, float* rays_d, float* target, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  ray_batch_kernel<<<(n + 255) / 256, 256, 0, st>>>(pix, n, poses, K, image_to_view, images, H, W, rays_o, rays_d, target);
  return cudaGetLastError();
}
cudaError_t launch_median_index(const float* w, int n, int S, long long* idx, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  median_index_kernel<<<(n + 127) / 128, 128, 0, st>>>(w, n, S, idx);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
cudaError_t launch_sample_coarse(const float* rays, const float* t_rand, int n, int S, int lindisp, float* z_out,
                                 cudaStream_t st) {
  const long long total = static_cast<long long>(n) * S;
  if (total == 0) return cudaSuccess;
  sample_coarse_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(rays, t_rand, n, S, lindisp, z_out);
  return cudaGetLastError();
}
cudaError_t launch_composite(const CompositeParams& p, cudaStream_t st) {
  if (p.n == 0) return cudaSuccess;
  const size_t smem = sizeof(float) * kWarpsPerBlock * (3 * p.S + p.S + p.n_imp);
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(composite_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  composite_kernel<<<(p.n + kWarpsPerBlock - 1) / kWarpsPerBlock, kWarpsPerBlock * 32, smem, st>>>(p);
  return cudaGetLastError();
}
cudaError_t launch_sample_pdf(const float* bins, const float* weights, const float* u, int n, int nb, int n_samp,
                              float* out, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  const size_t smem = sizeof(float) * kWarpsPerBlock * 3 * nb;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(sample_pdf_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  sample_pdf_kernel<<<(n + kWarpsPerBlock - 1) / kWarpsPerBlock, kWarpsPerBlock * 32, smem, st>>>(bins, weights, u, n, nb,
                                                                                                n_samp, out);
  return cudaGetLastError();
}
cudaError_t launch_composite_bwd(const CompositeBwdParams& p, cudaStream_t st) {
  if (p.n == 0) return cudaSuccess;
  const size_t smem = sizeof(float) * kWarpsPerBlock * p.S;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(composite_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  composite_bwd_kernel<<<(p.n + kWarpsPerBlock - 1) / kWarpsPerBlock, kWarpsPerBlock * 32, smem, st>>>(p);
  return cudaGetLastError();
}

}  // namespace nrn
