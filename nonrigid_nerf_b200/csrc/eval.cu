// Evaluation and visualisation of rendered frames (free_viewpoint_rendering.py:725-876, run_nerf_helpers.py:701-793):
// PSNR and Gaussian SSIM with the SSIM map and the two error images, jet and Blinn-Phong disparity images, and the
// background-stability map.  Frames are fp32 [F][H][W][3] ([F][H][W] for disparity), any F, H, W.  Every score is a
// fixed-order sum (per-tile partials in fp64, then one block per frame), so scores are bit-reproducible.
//
// Where the reference rounds in fp32 (numpy on float32 arrays: masks, norms, np.gradient, np.std, the LUT indices) the
// kernels do the same operations in the same order with explicit _rn intrinsics, so that no multiply-add is contracted.
#include <math.h>
#include "eval.cuh"
#include "jet.cuh"

namespace nrn {
namespace {

// numpy's sum over a contiguous axis of three: ((a + b) + c)
__device__ __forceinline__ float sum3(float a, float b, float c) { return __fadd_rn(__fadd_rn(a, b), c); }
__device__ __forceinline__ float sumsq3(float a, float b, float c) {
  return sum3(__fmul_rn(a, a), __fmul_rn(b, b), __fmul_rn(c, c));
}

// ---- PSNR / SSIM -------------------------------------------------------------------------------------------------------
// skimage.metrics.structural_similarity(data_range=1, gaussian_weights=True, sigma=1.5, use_sample_covariance=False,
// multichannel=True, full=True): per channel the five moments through scipy.ndimage.gaussian_filter(sigma=1.5,
// truncate=3.5, mode="reflect"), i.e. 11 taps, C1 = 0.01^2, C2 = 0.03^2, cov_norm = 1; the score is the mean of S over
// the image cropped by 5 pixels on every side, over the channels.
constexpr int kRadius = 5;
constexpr int kTaps = 2 * kRadius + 1;
constexpr int kHaloW = kEvalTileW + 2 * kRadius;
constexpr int kHaloH = kEvalTileH + 2 * kRadius;
constexpr int kScoreThreads = 256;
constexpr int kRowsPerThread = kEvalTileH * kEvalTileW / kScoreThreads;
static_assert(kEvalTileW == 32 && kEvalTileH % kRowsPerThread == 0, "one warp per tile row");

struct GaussTaps {
  double w[kTaps];
};

// scipy.ndimage mode="reflect" (d c b a | a b c d | d c b a), repeated for windows wider than the image
__device__ __forceinline__ int reflect_index(int i, int n) {
  const int period = 2 * n;
  int m = i % period;
  if (m < 0) m += period;
  return m < n ? m : period - 1 - m;
}

__device__ __forceinline__ double block_sum(double v, double* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x / 32;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[warp] = v;
  __syncthreads();
  double s = 0.0;
  for (int i = 0; i < static_cast<int>(blockDim.x / 32); ++i) s += red[i];
  return s;
}

// mask[p] = (sum over the channels of gt frame 0 == 0), free_viewpoint_rendering.py:820-821
__global__ void frame_mask_kernel(const float* __restrict__ gt, long long n_pix, uint8_t* __restrict__ mask) {
  const long long p = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= n_pix) return;
  mask[p] = sum3(gt[p * 3], gt[p * 3 + 1], gt[p * 3 + 2]) == 0.f;
}

// One CTA per 32 x 8 output tile of one frame: the tile and its 5-pixel halo of both images (masked pixels zeroed) into
// shared memory, per channel a horizontal then a vertical pass of the five moments, S, the error images and the tile's
// squared-error and cropped-SSIM sums.  The moments are filtered in fp64: in fp32, E[x^2] - E[x]^2 of a flat region
// keeps ~1e-7 of noise that only C2 = 9e-4 divides, 5e-4 of error in S (measured on an H100)
__global__ void __launch_bounds__(kScoreThreads) ssim_tile_kernel(ImageScoreParams p, GaussTaps taps, int tiles_x, int tiles_per_frame) {
  __shared__ float sx[kHaloH][kHaloW * 3];
  __shared__ float sy[kHaloH][kHaloW * 3];
  __shared__ double sh[5][kHaloH][kEvalTileW];
  __shared__ double red[kScoreThreads / 32];
  const int f = blockIdx.x / tiles_per_frame;
  const int t = blockIdx.x - f * tiles_per_frame;
  const int x0 = (t % tiles_x) * kEvalTileW, y0 = (t / tiles_x) * kEvalTileH;
  const int H = p.H, W = p.W;
  const size_t frame = static_cast<size_t>(f) * H * W * 3;
  const float* gt = p.gt + frame;
  const float* gen = p.gen + frame;
  for (int i = threadIdx.x; i < kHaloH * kHaloW * 3; i += kScoreThreads) {
    const int r = i / (kHaloW * 3), q = i - r * (kHaloW * 3), px = q / 3, c = q - px * 3;
    const size_t pix = static_cast<size_t>(reflect_index(y0 - kRadius + r, H)) * W + reflect_index(x0 - kRadius + px, W);
    const bool masked = p.mask[pix] != 0;
    sx[r][q] = masked ? 0.f : __ldg(gt + pix * 3 + c);
    sy[r][q] = masked ? 0.f : __ldg(gen + pix * 3 + c);
  }
  const int tx = threadIdx.x % 32, ty = threadIdx.x / 32;
  double S[kRowsPerThread][3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    __syncthreads();   // halo loaded / the previous channel's vertical pass done with sh
    for (int i = threadIdx.x; i < kHaloH * kEvalTileW; i += kScoreThreads) {
      const int r = i / kEvalTileW, j = i - r * kEvalTileW;
      double mx = 0.0, my = 0.0, mxx = 0.0, myy = 0.0, mxy = 0.0;
#pragma unroll
      for (int k = 0; k < kTaps; ++k) {
        const double a = sx[r][(j + k) * 3 + c], b = sy[r][(j + k) * 3 + c], w = taps.w[k];
        mx += w * a; my += w * b; mxx += w * (a * a); myy += w * (b * b); mxy += w * (a * b);
      }
      sh[0][r][j] = mx; sh[1][r][j] = my; sh[2][r][j] = mxx; sh[3][r][j] = myy; sh[4][r][j] = mxy;
    }
    __syncthreads();
#pragma unroll
    for (int h = 0; h < kRowsPerThread; ++h) {
      const int oy = ty + h * (kScoreThreads / 32);
      double ux = 0.0, uy = 0.0, uxx = 0.0, uyy = 0.0, uxy = 0.0;
#pragma unroll
      for (int k = 0; k < kTaps; ++k) {
        const double w = taps.w[k];
        ux += w * sh[0][oy + k][tx]; uy += w * sh[1][oy + k][tx]; uxx += w * sh[2][oy + k][tx];
        uyy += w * sh[3][oy + k][tx]; uxy += w * sh[4][oy + k][tx];
      }
      const double vx = uxx - ux * ux, vy = uyy - uy * uy, vxy = uxy - ux * uy;
      const double C1 = 0.01 * 0.01, C2 = 0.03 * 0.03;
      const double A1 = 2.0 * ux * uy + C1, A2 = 2.0 * vxy + C2;
      const double B1 = ux * ux + uy * uy + C1, B2 = vx + vy + C2;
      S[h][c] = (A1 * A2) / (B1 * B2);
    }
  }
  double sse = 0.0, ssum = 0.0;
#pragma unroll
  for (int h = 0; h < kRowsPerThread; ++h) {
    const int oy = ty + h * (kScoreThreads / 32);
    const int gy = y0 + oy, gx = x0 + tx;
    if (gy >= H || gx >= W) continue;
    const size_t pix = static_cast<size_t>(gy) * W + gx;
    const bool masked = p.mask[pix] != 0;
    float d[3];
    for (int c = 0; c < 3; ++c) {
      d[c] = masked ? 0.f : __fsub_rn(__ldg(gt + pix * 3 + c), __ldg(gen + pix * 3 + c));
      sse += static_cast<double>(d[c]) * d[c];
    }
    if (gy >= kRadius && gy < H - kRadius && gx >= kRadius && gx < W - kRadius) ssum += (S[h][0] + S[h][1]) + S[h][2];
    const float Sf[3] = {static_cast<float>(S[h][0]), static_cast<float>(S[h][1]), static_cast<float>(S[h][2])};
    const size_t o = frame + pix * 3;
    if (p.ssim_map)
      for (int c = 0; c < 3; ++c) p.ssim_map[o + c] = Sf[c];
    if (p.error_rgb) {   // jet(clip(10 |gt - gen| / sqrt(3), 0, 1)), free_viewpoint_rendering.py:847-850 (float64 after the norm)
      const int k = lut_index(static_cast<double>(__fsqrt_rn(sumsq3(d[0], d[1], d[2]))) / sqrt(3.0) * 10.0);
      for (int c = 0; c < 3; ++c) p.error_rgb[o + c] = c_jet.rgb8[k * 3 + c];
    }
    if (p.error_ssim) {  // jet(1 - mean_c S), :855 (S is float64 there)
      const int k = lut_index(1.0 - ((static_cast<double>(Sf[0]) + Sf[1]) + Sf[2]) / 3.0);   // of the map as written
      for (int c = 0; c < 3; ++c) p.error_ssim[o + c] = c_jet.rgb8[k * 3 + c];
    }
  }
  sse = block_sum(sse, red);
  ssum = block_sum(ssum, red);
  if (threadIdx.x == 0) {
    p.partials[static_cast<size_t>(blockIdx.x) * 2] = sse;
    p.partials[static_cast<size_t>(blockIdx.x) * 2 + 1] = ssum;
  }
}

// One block per frame: the tiles' partial sums in tile order -> psnr = -10 log10(mse), ssim = cropped mean of S
__global__ void score_reduce_kernel(ImageScoreParams p, int tiles_per_frame) {
  __shared__ double red[kScoreThreads / 32];
  const double* part = p.partials + static_cast<size_t>(blockIdx.x) * tiles_per_frame * 2;
  double sse = 0.0, ssum = 0.0;
  for (int i = threadIdx.x; i < tiles_per_frame; i += kScoreThreads) { sse += part[i * 2]; ssum += part[i * 2 + 1]; }
  sse = block_sum(sse, red);
  ssum = block_sum(ssum, red);
  if (threadIdx.x == 0) {
    const double n = 3.0 * p.H * p.W;
    const double n_crop = (p.H > 2 * kRadius && p.W > 2 * kRadius) ? 3.0 * (p.H - 2 * kRadius) * (p.W - 2 * kRadius) : 0.0;
    p.psnr[blockIdx.x] = static_cast<float>(-10.0 * log10(sse / n));   // identical frames: log10(0), psnr = +inf
    p.ssim[blockIdx.x] = static_cast<float>(ssum / n_crop);            // empty crop: the mean of nothing, NaN
  }
}

// ---- disparity images, run_nerf_helpers.py:701-793 ----------------------------------------------------------------------
// Blinn-Phong colour of pixel (y, x) of an H x W disparity map read through at(yy, xx), d = at(y, x): normals from
// np.gradient(d, 2 / (H - 1)) (central differences inside, one-sided at the edges, fp32 as numpy computes them for a
// float32 map), then the reference's light / view / half vectors and constants, in fp32
template <typename At>
__device__ __forceinline__ void blinn_phong(At at, float d, int y, int x, int H, int W, float inv_c, float inv_e, float rgb[3]) {
  const float zy = y == 0 ? __fdiv_rn(__fsub_rn(at(1, x), at(0, x)), inv_e)
                 : y == H - 1 ? __fdiv_rn(__fsub_rn(at(H - 1, x), at(H - 2, x)), inv_e)
                              : __fdiv_rn(__fsub_rn(at(y + 1, x), at(y - 1, x)), inv_c);
  const float zx = x == 0 ? __fdiv_rn(__fsub_rn(at(y, 1), at(y, 0)), inv_e)
                 : x == W - 1 ? __fdiv_rn(__fsub_rn(at(y, W - 1), at(y, W - 2)), inv_e)
                              : __fdiv_rn(__fsub_rn(at(y, x + 1), at(y, x - 1)), inv_c);
  const float nl = __fsqrt_rn(sumsq3(-zx, zy, 1.f));
  const float nx = __fdiv_rn(-zx, nl), ny = __fdiv_rn(zy, nl), nz = __fdiv_rn(1.f, nl);
  // vertPos = (x / W, y / W, d): both image axes divided by the width, as the reference does
  const float px = __fdiv_rn(static_cast<float>(x), static_cast<float>(W)), py = __fdiv_rn(static_cast<float>(y), static_cast<float>(W));
  float lx = 1.f - px, ly = 1.f - py, lz = 1.f - d;   // lightPos (1, 1, 1) - vertPos
  const float dist = sqrtf(lx * lx + ly * ly + lz * lz);
  lx /= dist; ly /= dist; lz /= dist;
  const float att = (dist + 1.f) * (dist + 1.f);
  const float ldotn = lx * nx + ly * ny + lz * nz;
  const float lambertian = ldotn < 0.f ? 0.f : ldotn;   // np.clip(a_min=0) keeps NaN
  const float vl = sqrtf(px * px + py * py + d * d);
  const float vx = -px / vl, vy = -py / vl, vz = -d / vl;
  float hx = lx + vx, hy = ly + vy, hz = lz + vz;
  const float hl = sqrtf(hx * hx + hy * hy + hz * hz);
  hx /= hl; hy /= hl; hz /= hl;
  const float sdot = -(hx * nx + hy * ny + hz * nz);
  const float spec_angle = sdot < 0.f ? 0.f : sdot;
  const float specular = lambertian <= 0.f ? 0.f : spec_angle * spec_angle;   // invalid_mask
  const float light_power = 2.f;
  const float diffuse[3] = {0.5f, 0.f, 0.f}, ambient[3] = {0.1f, 0.f, 0.f};
  for (int c = 0; c < 3; ++c) rgb[c] = lambertian * diffuse[c] * light_power / att + specular * light_power / att + ambient[c];
}

// jet: the LUT colour of clip(d, 0, 1); Blinn-Phong as above
__global__ void disparity_kernel(const float* __restrict__ disp, int F, int H, int W, float* __restrict__ jet,
                                 float* __restrict__ phong, float inv_c, float inv_e) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long n_pix = static_cast<long long>(H) * W;
  if (i >= n_pix * F) return;
  const long long f = i / n_pix;
  const int y = static_cast<int>((i - f * n_pix) / W), x = static_cast<int>(i - f * n_pix - static_cast<long long>(y) * W);
  const float* dm = disp + f * n_pix;
  const float d = dm[static_cast<long long>(y) * W + x];
  if (jet) {
    const int k = lut_index(d);
    for (int c = 0; c < 3; ++c) jet[i * 3 + c] = c_jet.rgbf[k * 3 + c];
  }
  if (!phong) return;
  float rgb[3];
  blinn_phong([&](int yy, int xx) { return dm[static_cast<long long>(yy) * W + xx]; }, d, y, x, H, W, inv_c, inv_e, rgb);
  for (int c = 0; c < 3; ++c) phong[i * 3 + c] = rgb[c];
}

// ---- the saved 8-bit images of free_viewpoint_rendering.py:615-766 ------------------------------------------------------
// to8b(v) = uint8(255 * clip(v, 0, 1)) is lut_index(v): the fp32 form for the float32 arrays (rgb, disparity, rigidity,
// the Phong value), the fp64 form for the float64 correspondence image.
constexpr int kMaxThreads = 1024;
// The canonical space is cut into 100 voxels per axis, each spanning the whole colour cube (free_viewpoint_rendering.py:641)
constexpr int kCorrespondenceVoxels = 100;
constexpr int kImageThreads = 256;
constexpr unsigned kImageMaxBlocks = 16384;   // grid-stride beyond this: the stack maximum is reduced once per block

// np.max semantics: a NaN anywhere makes the maximum NaN
__device__ __forceinline__ float max_nan(float a, float b) { return (a != a || a > b) ? a : b; }
__device__ __forceinline__ float warp_max_nan(float v) {
  for (int o = 16; o > 0; o >>= 1) v = max_nan(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// One block per frame: disp_max[f] = np.max(disp[f]).  A maximum does not depend on the order it is taken in.
__global__ void __launch_bounds__(kMaxThreads) disp_max_kernel(const float* __restrict__ disp, long long n_pix,
                                                               float* __restrict__ disp_max) {
  __shared__ float red[kMaxThreads / 32];
  const float* d = disp + static_cast<long long>(blockIdx.x) * n_pix;
  float m = -INFINITY;
#pragma unroll 8
  for (long long i = threadIdx.x; i < n_pix; i += kMaxThreads) m = max_nan(m, __ldg(d + i));
  m = warp_max_nan(m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x / 32] = m;
  __syncthreads();
  if (threadIdx.x < 32) {
    m = warp_max_nan(red[threadIdx.x]);
    if (threadIdx.x == 0) disp_max[blockIdx.x] = m;
  }
}

// Every requested uint8 image of every pixel of the stack.  The correspondence image (:640-644) is float64 in the
// reference (float32 points minus the float64 extent of the checkpoint): c = (p - min) / (max - min) * 100 with _rn
// intrinsics so that nothing is contracted into an FMA, then c - c.astype(int).  astype(int) truncates toward zero, so a
// point below min gives a negative fraction that to8b clips to 0 (c - floor(c) would not); out of int64's range (and
// for NaN) it gives INT64_MIN on x86 hosts, which the fraction reproduces.  disp / max is a float32 division (numpy
// divides the float32 map by its float32 maximum), the video's by the maximum over the whole stack (:727).
__global__ void __launch_bounds__(kImageThreads) frame_images_kernel(FrameImageParams p, float inv_c, float inv_e) {
  __shared__ float s_stack_max;
  const long long n_pix = static_cast<long long>(p.H) * p.W, n = n_pix * p.F;
  const int W = p.W;
  if (p.out_disp_video) {
    if (threadIdx.x < 32) {
      float m = -INFINITY;
      for (int f = threadIdx.x; f < p.F; f += 32) m = max_nan(m, p.disp_max[f]);
      m = warp_max_nan(m);
      if (threadIdx.x == 0) s_stack_max = m;
    }
    __syncthreads();
  }
  for (long long i = static_cast<long long>(blockIdx.x) * kImageThreads + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * kImageThreads) {
    const long long f = i / n_pix, pix = i - f * n_pix;
    if (p.out_rgb)
      for (int c = 0; c < 3; ++c) p.out_rgb[i * 3 + c] = static_cast<uint8_t>(lut_index(__ldg(p.rgb + i * 3 + c)));
    if (p.disp) {
      const float* dm = p.disp + f * n_pix;
      const float m = __ldg(p.disp_max + f);
      const float raw = __ldg(dm + pix);
      const float d = __fdiv_rn(raw, m);
      const int k = lut_index(d);
      if (p.out_disp) p.out_disp[i] = static_cast<uint8_t>(k);
      if (p.out_disp_video) p.out_disp_video[i] = static_cast<uint8_t>(lut_index(__fdiv_rn(raw, s_stack_max)));
      if (p.out_disp_jet)
        for (int c = 0; c < 3; ++c) p.out_disp_jet[i * 3 + c] = c_jet.rgb8[k * 3 + c];
      if (p.out_disp_phong) {
        const int y = static_cast<int>(pix / W), x = static_cast<int>(pix - static_cast<long long>(y) * W);
        float rgb[3];
        blinn_phong([&](int yy, int xx) { return __fdiv_rn(__ldg(dm + static_cast<long long>(yy) * W + xx), m); }, d, y, x,
                    p.H, W, inv_c, inv_e, rgb);
        for (int c = 0; c < 3; ++c) p.out_disp_phong[i * 3 + c] = static_cast<uint8_t>(lut_index(rgb[c]));
      }
    }
    if (p.out_correspondences)
      for (int c = 0; c < 3; ++c) {
        const double v = __dmul_rn(__ddiv_rn(__dsub_rn(static_cast<double>(__ldg(p.surface_pts + i * 3 + c)), p.min_point[c]),
                                             __dsub_rn(p.max_point[c], p.min_point[c])),
                                   static_cast<double>(kCorrespondenceVoxels));
        const double t = fabs(v) < 0x1p63 ? trunc(v) : -0x1p63;
        p.out_correspondences[i * 3 + c] = static_cast<uint8_t>(lut_index(__dsub_rn(v, t)));
      }
    if (p.surface_rigidity) {
      const int k = lut_index(__ldg(p.surface_rigidity + i));
      if (p.out_rigidity) p.out_rigidity[i] = static_cast<uint8_t>(k);
      if (p.out_rigidity_jet)
        for (int c = 0; c < 3; ++c) p.out_rigidity_jet[i * 3 + c] = c_jet.rgb8[k * 3 + c];
    }
  }
}

// ---- background stability, free_viewpoint_rendering.py:770-785 ---------------------------------------------------------
// per pixel and channel np.std over the frames (ddof 0) the way numpy computes it for float32: the mean from a
// frame-ordered sum, then the frame-ordered sum of squared deviations; the image is jet(10 * mean_c std)
__global__ void frame_std_kernel(const float* __restrict__ rgbs, int F, long long n_pix, float* __restrict__ std_out,
                                 float* __restrict__ image) {
  const long long p = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= n_pix) return;
  const long long stride = n_pix * 3;
  const float nf = static_cast<float>(F);
  float sd[3];
  for (int c = 0; c < 3; ++c) {
    const float* v = rgbs + p * 3 + c;
    float s = v[0];
    for (int f = 1; f < F; ++f) s = __fadd_rn(s, v[f * stride]);
    const float mean = __fdiv_rn(s, nf);
    float q = 0.f;
    for (int f = 0; f < F; ++f) {
      const float dv = __fsub_rn(v[f * stride], mean);
      q = f == 0 ? __fmul_rn(dv, dv) : __fadd_rn(q, __fmul_rn(dv, dv));
    }
    sd[c] = __fsqrt_rn(__fdiv_rn(q, nf));
    if (std_out) std_out[p * 3 + c] = sd[c];
  }
  if (image) {
    const int k = lut_index(__fmul_rn(10.f, __fdiv_rn(sum3(sd[0], sd[1], sd[2]), 3.f)));
    for (int c = 0; c < 3; ++c) image[p * 3 + c] = c_jet.rgbf[k * 3 + c];
  }
}

unsigned blocks_for(long long n, int threads) { return static_cast<unsigned>((n + threads - 1) / threads); }

// np.gradient(d, spacing) divides by 2 * spacing inside and by spacing at the edges, both Python floats that numpy
// rounds to float32 for a float32 map
void gradient_divisors(int H, float* inv_c, float* inv_e) {
  const double spacing = H > 1 ? 2.0 / (H - 1) : 1.0;
  *inv_c = static_cast<float>(2.0 * spacing);
  *inv_e = static_cast<float>(spacing);
}

}  // namespace

long long eval_tiles_per_frame(int H, int W) {
  return static_cast<long long>((W + kEvalTileW - 1) / kEvalTileW) * ((H + kEvalTileH - 1) / kEvalTileH);
}
size_t eval_partials_bytes(int F, int H, int W) {
  return static_cast<size_t>(F) * static_cast<size_t>(eval_tiles_per_frame(H, W)) * 2 * sizeof(double);
}

void jet_table(double* rgb, uint8_t* rgb8) {
  for (int i = 0; i < 256 * 3; ++i) {
    if (rgb) rgb[i] = kJet.rgb[i];
    if (rgb8) rgb8[i] = kJet.rgb8[i];
  }
}

cudaError_t launch_frame_mask(const float* gt, int H, int W, uint8_t* mask, cudaStream_t st) {
  const long long n = static_cast<long long>(H) * W;
  frame_mask_kernel<<<blocks_for(n, 256), 256, 0, st>>>(gt, n, mask);
  return cudaGetLastError();
}

cudaError_t launch_image_scores(const ImageScoreParams& p, cudaStream_t st) {
  // scipy.ndimage._gaussian_kernel1d(sigma=1.5, order=0, radius=int(3.5 * 1.5 + 0.5)) in float64
  GaussTaps taps;
  double phi[kTaps], sum = 0.0;
  for (int k = 0; k < kTaps; ++k) {
    const double x = k - kRadius;
    phi[k] = exp(-0.5 / (1.5 * 1.5) * (x * x));
    sum += phi[k];
  }
  for (int k = 0; k < kTaps; ++k) taps.w[k] = phi[k] / sum;
  const int tiles_x = (p.W + kEvalTileW - 1) / kEvalTileW;
  const int tiles = static_cast<int>(eval_tiles_per_frame(p.H, p.W));
  ssim_tile_kernel<<<static_cast<unsigned>(static_cast<long long>(tiles) * p.F), kScoreThreads, 0, st>>>(p, taps, tiles_x, tiles);
  return cudaGetLastError();
}

cudaError_t launch_score_reduce(const ImageScoreParams& p, cudaStream_t st) {
  score_reduce_kernel<<<p.F, kScoreThreads, 0, st>>>(p, static_cast<int>(eval_tiles_per_frame(p.H, p.W)));
  return cudaGetLastError();
}

cudaError_t launch_disparity_images(const float* disp, int F, int H, int W, float* jet, float* phong, cudaStream_t st) {
  float inv_c, inv_e;
  gradient_divisors(H, &inv_c, &inv_e);
  const long long n = static_cast<long long>(F) * H * W;
  disparity_kernel<<<blocks_for(n, 256), 256, 0, st>>>(disp, F, H, W, jet, phong, inv_c, inv_e);
  return cudaGetLastError();
}

cudaError_t launch_disp_max(const float* disp, int F, int H, int W, float* disp_max, cudaStream_t st) {
  disp_max_kernel<<<F, kMaxThreads, 0, st>>>(disp, static_cast<long long>(H) * W, disp_max);
  return cudaGetLastError();
}

cudaError_t launch_frame_images(const FrameImageParams& p, cudaStream_t st) {
  float inv_c, inv_e;
  gradient_divisors(p.H, &inv_c, &inv_e);
  const long long blocks = (static_cast<long long>(p.F) * p.H * p.W + kImageThreads - 1) / kImageThreads;
  frame_images_kernel<<<blocks < kImageMaxBlocks ? static_cast<unsigned>(blocks) : kImageMaxBlocks, kImageThreads, 0, st>>>(p, inv_c, inv_e);
  return cudaGetLastError();
}

cudaError_t launch_frame_std(const float* rgbs, int F, int H, int W, float* std_out, float* image, cudaStream_t st) {
  const long long n = static_cast<long long>(H) * W;
  frame_std_kernel<<<blocks_for(n, 128), 128, 0, st>>>(rgbs, F, n, std_out, image);
  return cudaGetLastError();
}

}  // namespace nrn
