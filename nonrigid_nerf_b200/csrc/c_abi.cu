// extern "C" boundary of libnrnerf_b200.so (declarations: include/nrnerf_b200.h).
// Argument validation, launch, error reporting.  No exceptions cross this file.
#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include "../../include/nrnerf_b200.h"
#include "nrn_common.cuh"
#include "pack.cuh"
#include "ray_ops.cuh"
#include "wgrad.cuh"
#include "div.cuh"
#include "loss.cuh"
#include "adam.cuh"
#include "peer.cuh"
#include "det_reduce.cuh"
#include "eval.cuh"
#include "mesh.cuh"
#include "lpips.cuh"
#include "match.cuh"
#include "occupancy.cuh"
#include "deform.cuh"

namespace nrn {
cudaError_t launch_field_fwd(const FieldFwdParams& p, bool has_bender, int num_sms, cudaStream_t stream);
cudaError_t launch_field_bwd(const FieldBwdParams& p, bool has_bender, int num_sms, cudaStream_t stream);
cudaError_t launch_field_bwd_det(const FieldBwdParams& p, float* latent_rows, int num_sms, cudaStream_t stream);
cudaError_t launch_field_bwd_held(const FieldBwdParams& p, float* latent_rows, const uint8_t* held, int num_sms, cudaStream_t stream);
cudaError_t launch_field_fwd_tc(const FieldFwdParams& p, int num_sms, cudaStream_t stream);
cudaError_t launch_tc_latent_bias(const float* lat, long long lat_stride, int n_rays, const float* w0, const float* b0, const float* w5,
                                  const float* b5, float* rb, cudaStream_t stream);
cudaError_t launch_tc_latent_bwd(const TcBwdParams& p, cudaStream_t stream);
cudaError_t launch_field_bend(const FieldFwdParams& p, const ViewParams& v, int num_sms, cudaStream_t stream);
cudaError_t launch_field_views(const FieldFwdParams& p, const ViewParams& v, int num_sms, cudaStream_t stream);
cudaError_t launch_field_views_train(const FieldFwdParams& p, const ViewParams& v, const ViewTrainParams& t, int num_sms, cudaStream_t stream);
cudaError_t launch_field_bwd_views(const FieldBwdParams& p, const ViewBwdParams& v, int num_sms, cudaStream_t stream);
cudaError_t launch_field_fwd_kept(const FieldFwdParams& p, const int* kept, int num_sms, cudaStream_t stream);
cudaError_t launch_field_fwd_grad(const FieldFwdParams& p, bool has_bender, int num_sms, cudaStream_t stream);
cudaError_t launch_field_bwd_grad(const FieldBwdParams& p, const PointGradParams& pg, bool has_bender, int num_sms, cudaStream_t stream);
}

namespace {

thread_local char g_err[512] = "";

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
int cuda_fail(cudaError_t e, const char* what) {
  return fail(NRN_E_CUDA, "%s: %s", what, cudaGetErrorString(e));
}

constexpr int kMaxDevices = 64;
struct DeviceState {
  int* err_word = nullptr;   // [0] error word, [1] loss-scale source (float) of the running backward
  int num_sms = 0;
};
DeviceState g_dev[kMaxDevices];

int device_state(DeviceState** out) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return cuda_fail(e, "cudaGetDevice");
  if (dev < 0 || dev >= kMaxDevices) return fail(NRN_E_INVALID, "device index %d out of range", dev);
  DeviceState& s = g_dev[dev];
  if (!s.err_word) {
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, dev);
    if (e != cudaSuccess) return cuda_fail(e, "cudaGetDeviceProperties");
    if (prop.major != 9 || prop.minor != 0)
      return fail(NRN_E_INVALID, "nrnerf_b200 is built for sm_90a (H100) only, found sm_%d%d", prop.major, prop.minor);
    s.num_sms = prop.multiProcessorCount;
    if (const char* g = getenv("NRN_GRID")) { const int v = atoi(g); if (v > 0 && v < s.num_sms) s.num_sms = v; }   // developer experiments
    e = cudaMalloc(&s.err_word, 4 * sizeof(int));
    if (e != cudaSuccess) return cuda_fail(e, "cudaMalloc(err word)");
    e = cudaMemset(s.err_word, 0, 4 * sizeof(int));
    if (e != cudaSuccess) return cuda_fail(e, "cudaMemset(err word)");
  }
  *out = &s;
  return NRN_OK;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// ---- optional per-kernel timing: CUDA events recorded on the launch stream around each kernel ----
struct TimedLaunch {
  cudaEvent_t a, b;
  int kind;
};
bool g_timing = false;
TimedLaunch g_timed[4096];
int g_timed_n = 0;
struct ScopedTimer {
  int idx = -1;
  cudaStream_t st;
  ScopedTimer(int kind, cudaStream_t s) : st(s) {
    if (!g_timing || g_timed_n >= 4096) return;
    TimedLaunch& t = g_timed[g_timed_n];
    if (cudaEventCreate(&t.a) != cudaSuccess || cudaEventCreate(&t.b) != cudaSuccess) return;
    t.kind = kind;
    idx = g_timed_n++;
    record(t.a);
  }
  ~ScopedTimer() {
    if (idx >= 0) record(g_timed[idx].b);
  }
  // inside a CUDA-graph capture the records become external event-record nodes: every replay of the graph
  // re-stamps them, and the elapsed time of the last replay can be read afterwards
  void record(cudaEvent_t ev) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    cudaStreamIsCapturing(st, &cs);
    cudaEventRecordWithFlags(ev, st, cs == cudaStreamCaptureStatusActive ? cudaEventRecordExternal : cudaEventRecordDefault);
  }
};

// One kernel launch `launch()`, timed as `kind`; a launch error is reported under the kernel's name
template <typename Launch>
int timed(int kind, cudaStream_t st, const char* kernel, Launch launch) {
  cudaError_t e;
  {
    ScopedTimer tm(kind, st);
    e = launch();
  }
  return e == cudaSuccess ? NRN_OK : cuda_fail(e, kernel);
}

// Tiles of kTileM points that P points fill
long long tile_count(long long P) { return (P + nrn::kTileM - 1) / nrn::kTileM; }
long long even_tiles(int n_rays, int n_samples) {
  return (tile_count(static_cast<long long>(n_rays) * n_samples) + 1) & ~1LL;   // rounded up to an even count: the stash layout of ABI version 2
}
int checked_tiles(long long P, const char* who, int* tiles) {
  const long long t = tile_count(P);
  if (t > 0x7fffffffLL) return fail(NRN_E_INVALID, "%s: too many points", who);
  *tiles = static_cast<int>(t);
  return NRN_OK;
}

// The checks every field forward entry point applies to its NrnFieldArgs.  *P = n_rays * n_samples; for an empty batch
// (P = 0) only the sizes and out_ch are checked, and nothing is to be launched.
int check_field_args(const NrnFieldArgs* a, const char* who, long long* P, int* tiles) {
  if (!a) return fail(NRN_E_INVALID, "%s: null args", who);
  if (a->n_rays < 0 || a->n_samples < 1) return fail(NRN_E_INVALID, "%s: bad sizes n=%d S=%d", who, a->n_rays, a->n_samples);
  if (a->out_ch < 4 || a->out_ch > 5) return fail(NRN_E_INVALID, "%s: out_ch=%d unsupported (4 or 5)", who, a->out_ch);
  if ((a->stash != nullptr) != (a->relu_mask != nullptr))
    return fail(NRN_E_INVALID, "%s: training needs both the stash and the ReLU mask buffer (relu_mask)", who);
  *P = static_cast<long long>(a->n_rays) * a->n_samples;
  *tiles = 0;
  if (*P == 0) return NRN_OK;
  if (!a->nerf_packed) return fail(NRN_E_INVALID, "%s: null nerf_packed", who);
  if (a->points) {
    if (a->points_stride < 3) return fail(NRN_E_INVALID, "%s: point mode needs points_stride >= 3", who);
  } else if (!a->rays || !a->z_vals) {
    return fail(NRN_E_INVALID, "%s: null rays / z_vals", who);
  }
  if (a->bender_packed && !a->latents) return fail(NRN_E_INVALID, "%s: bender given without latents", who);
  if (a->stash && a->points) return fail(NRN_E_INVALID, "%s: the training stash needs ray mode", who);
  if (!aligned16(a->nerf_packed) || (a->bender_packed && !aligned16(a->bender_packed)))
    return fail(NRN_E_INVALID, "%s: packed weights must be 16-byte aligned", who);
  // the forward kernels store the stash with bulk copies, which need 16-byte aligned destinations
  if (a->stash && (!aligned16(a->stash) || !aligned16(a->relu_mask)))
    return fail(NRN_E_INVALID, "%s: stash and relu_mask must be 16-byte aligned", who);
  return checked_tiles(*P, who, tiles);
}

nrn::FieldFwdParams field_fwd_params(const NrnFieldArgs* a, long long P, int tiles, int* err) {
  nrn::FieldFwdParams p{};
  p.rays = a->rays; p.z_vals = a->z_vals; p.pts = a->points; p.pts_stride = a->points_stride; p.latents = a->latents; p.latent_stride = a->latent_stride;
  p.n_rays = a->n_rays; p.S = a->n_samples; p.P = P; p.n_tiles = tiles;
  const uint8_t* np = static_cast<const uint8_t*>(a->nerf_packed);
  p.nerf_w = np; p.nerf_bias = reinterpret_cast<const float*>(np + nrn::kNerfWBytes);
  if (a->bender_packed) {
    const uint8_t* bp = static_cast<const uint8_t*>(a->bender_packed);
    p.bend_w = bp; p.bend_bias = reinterpret_cast<const float*>(bp + nrn::kBendWBytes);
  }
  p.cutoff = a->rigidity_cutoff; p.use_cutoff = a->use_cutoff;
  p.scaling = a->scaling; p.use_scaling = a->use_scaling;
  p.removal = a->removal_threshold; p.use_removal = a->use_removal;
  p.out_ch = a->out_ch;
  p.raw = a->raw; p.d_init = a->initial_input_pts; p.d_bent = a->input_pts; p.d_unmasked = a->unmasked_offsets;
  p.d_masked = a->masked_offsets; p.d_rigid = a->rigidity_mask;
  p.stash = static_cast<uint8_t*>(a->stash);
  p.relu_mask = static_cast<uint8_t*>(a->relu_mask);
  p.err = err;
  return p;
}

// The checks every field backward entry point applies to its NrnFieldBwdArgs.  *P = n_rays * n_samples; an empty shard
// (P = 0) needs only its gradient destinations.
int check_field_bwd_args(const NrnFieldBwdArgs* a, const char* who, long long* P, int* tiles) {
  if (!a) return fail(NRN_E_INVALID, "%s: null args", who);
  if (a->n_rays < 0 || a->n_samples < 1) return fail(NRN_E_INVALID, "%s: bad sizes", who);
  if (a->out_ch < 4 || a->out_ch > 5) return fail(NRN_E_INVALID, "%s: out_ch=%d unsupported", who, a->out_ch);
  if (!a->nerf_grad) return fail(NRN_E_INVALID, "%s: null nerf_grad", who);
  if (a->bender_packed && (!a->unmasked_offsets || !a->rigidity_mask || !a->bender_grad || !a->d_latents))
    return fail(NRN_E_INVALID, "%s: null argument: a bender needs unmasked_offsets, rigidity_mask, bender_grad, d_latents", who);
  *P = static_cast<long long>(a->n_rays) * a->n_samples;
  *tiles = 0;
  if (*P == 0) return NRN_OK;
  if (!a->nerf_packed || !a->d_raw || !a->stash || !a->grad_stash || !a->wgrad_scratch || !a->relu_mask)
    return fail(NRN_E_INVALID, "%s: null argument: nerf_packed, d_raw, stash, grad_stash, wgrad_scratch or relu_mask (the ReLU masks of the forward call)", who);
  if (!aligned16(a->nerf_packed) || !aligned16(a->stash) || !aligned16(a->grad_stash) || !aligned16(a->relu_mask))
    return fail(NRN_E_INVALID, "%s: packed weights and stashes must be 16-byte aligned", who);
  return checked_tiles(*P, who, tiles);
}

nrn::FieldBwdParams field_bwd_params(const NrnFieldBwdArgs* a, long long P, int tiles, float* amax, int* err) {
  nrn::FieldBwdParams p{};
  p.P = P; p.n_tiles = tiles;
  p.S = a->n_samples; p.n_rays = a->n_rays; p.out_ch = a->out_ch;
  p.d_raw = a->d_raw; p.amax = amax;
  p.stash = static_cast<const uint8_t*>(a->stash); p.gstash = static_cast<uint8_t*>(a->grad_stash);
  p.nerf_wT = static_cast<const uint8_t*>(a->nerf_packed) + nrn::kNerfTOffset;
  if (a->bender_packed) p.bend_wT = static_cast<const uint8_t*>(a->bender_packed) + nrn::kBendTOffset;
  p.unmasked = a->unmasked_offsets; p.rigidity = a->rigidity_mask;
  p.d_unmasked_up = a->d_unmasked_offsets; p.d_rigid_up = a->d_rigidity_mask;
  p.cutoff = a->rigidity_cutoff; p.use_cutoff = a->use_cutoff; p.scaling = a->scaling; p.use_scaling = a->use_scaling;
  p.d_latents = a->d_latents; p.err = err;
  p.relu_mask = static_cast<const uint8_t*>(a->relu_mask);
  return p;
}

// An empty shard contributes zero gradients: the destinations that are overwritten rather than accumulated are cleared.
// nerf_n floats of NeRF gradient, the last head_n of them at nerf_grad_head when that is given; bend_n of the bender's.
int zero_grads(const NrnFieldBwdArgs* a, int nerf_n, int head_n, int bend_n, cudaStream_t st) {
  cudaError_t e = cudaSuccess;
  if (!a->accumulate_nerf) {
    if (!a->nerf_grad_head) head_n = 0;
    e = cudaMemsetAsync(a->nerf_grad, 0, sizeof(float) * (nerf_n - head_n), st);
    if (e == cudaSuccess && head_n) e = cudaMemsetAsync(a->nerf_grad_head, 0, sizeof(float) * head_n, st);
  }
  if (e == cudaSuccess && bend_n && !a->accumulate_bender) e = cudaMemsetAsync(a->bender_grad, 0, sizeof(float) * bend_n, st);
  return e == cudaSuccess ? NRN_OK : cuda_fail(e, "memset grads");
}

nrn::WgradParams wgrad_params(const uint8_t* stash, uint8_t* gstash, float* scratch, float* amax, int n_tiles, int* err) {
  nrn::WgradParams w{};
  w.stash = stash; w.gstash = gstash; w.scratch = scratch; w.amax = amax; w.n_tiles = n_tiles; w.err = err;
  return w;
}

}  // namespace

extern "C" {

int nrn_abi_version(void) { return NRN_ABI_VERSION; }
const char* nrn_last_error(void) { return g_err; }

int nrn_device_error(int* code_out) {
  DeviceState* ds;
  int rc = device_state(&ds);
  if (rc) return rc;
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return cuda_fail(e, "cudaDeviceSynchronize");
  int code = 0;
  e = cudaMemcpy(&code, ds->err_word, sizeof(int), cudaMemcpyDeviceToHost);
  if (e != cudaSuccess) return cuda_fail(e, "cudaMemcpy(err word)");
  if (code) cudaMemset(ds->err_word, 0, sizeof(int));
  if (code_out) *code_out = code;
  if (code) return fail(NRN_E_DEVICE, "device-side protocol error: wait id %d timed out", code);
  return NRN_OK;
}

size_t nrn_packed_nerf_bytes(void) { return nrn::kNerfPackedBytes; }
size_t nrn_packed_bender_bytes(void) { return nrn::kBendPackedBytes; }

int nrn_pack_nerf(const float* const* w, const float* const* b, int input_ch, int out_ch, void* packed, void* stream) {
  if (!w || !b || !packed) return fail(NRN_E_INVALID, "nrn_pack_nerf: null argument");
  if ((input_ch < 1 || input_ch > 63) && input_ch != nrn::kPeCols + nrn::kLatent)
    return fail(NRN_E_INVALID, "nrn_pack_nerf: input_ch=%d unsupported (1..63; multires=10 gives 63; 95 = 63 + 32: time-conditioned baseline)", input_ch);
  if (out_ch < 4 || out_ch > 16) return fail(NRN_E_INVALID, "nrn_pack_nerf: out_ch=%d unsupported", out_ch);
  if (!aligned16(packed)) return fail(NRN_E_INVALID, "nrn_pack_nerf: packed buffer must be 16-byte aligned");
  nrn::NerfSrc src;
  for (int i = 0; i < 9; ++i) {
    if (!w[i] || !b[i]) return fail(NRN_E_INVALID, "nrn_pack_nerf: null layer %d", i);
    src.w[i] = w[i];
    src.b[i] = b[i];
  }
  cudaError_t e = nrn::launch_pack_nerf(src, input_ch, out_ch, packed, static_cast<cudaStream_t>(stream));
  return e == cudaSuccess ? NRN_OK : cuda_fail(e, "pack_nerf_kernel");
}

int nrn_pack_bender(const float* const* net_w, const float* const* net_b, const float* const* rig_w,
                    const float* const* rig_b, int latent_size, void* packed, void* stream) {
  if (!net_w || !net_b || !rig_w || !rig_b || !packed) return fail(NRN_E_INVALID, "nrn_pack_bender: null argument");
  if (latent_size != nrn::kLatent) return fail(NRN_E_INVALID, "nrn_pack_bender: ray_bending_latent_size=%d unsupported (32)", latent_size);
  if (!aligned16(packed)) return fail(NRN_E_INVALID, "nrn_pack_bender: packed buffer must be 16-byte aligned");
  nrn::BenderSrc src;
  for (int i = 0; i < 5; ++i) src.net_w[i] = net_w[i];
  for (int i = 0; i < 4; ++i) src.net_b[i] = net_b[i];
  for (int i = 0; i < 3; ++i) { src.rig_w[i] = rig_w[i]; src.rig_b[i] = rig_b[i]; }
  cudaError_t e = nrn::launch_pack_bender(src, packed, static_cast<cudaStream_t>(stream));
  return e == cudaSuccess ? NRN_OK : cuda_fail(e, "pack_bender_kernel");
}

int nrn_sample_coarse(const float* rays, const float* t_rand, int n_rays, int n_samples, int lindisp, float* z_vals,
                      void* stream) {
  if (n_rays < 0 || n_samples < 1) return fail(NRN_E_INVALID, "nrn_sample_coarse: bad sizes n=%d S=%d", n_rays, n_samples);
  if (n_rays == 0) return NRN_OK;
  if (!rays || !z_vals) return fail(NRN_E_INVALID, "nrn_sample_coarse: null argument");
  cudaError_t e = nrn::launch_sample_coarse(rays, t_rand, n_rays, n_samples, lindisp, z_vals, static_cast<cudaStream_t>(stream));
  return e == cudaSuccess ? NRN_OK : cuda_fail(e, "sample_coarse_kernel");
}

int nrn_get_rays(const float* c2w, const float* K, int H, int W, float* rays_o, float* rays_d, void* stream) {
  if (H < 0 || W < 0) return fail(NRN_E_INVALID, "nrn_get_rays: bad sizes");
  if (H == 0 || W == 0) return NRN_OK;
  if (!c2w || !K || !rays_o || !rays_d) return fail(NRN_E_INVALID, "nrn_get_rays: null argument");
  const cudaError_t e = nrn::launch_get_rays(c2w, K, H, W, rays_o, rays_d, static_cast<cudaStream_t>(stream));
  return e == cudaSuccess ? NRN_OK : cuda_fail(e, "get_rays_kernel");
}

int nrn_pack_rays(const float* rays_o, const float* rays_d, float near, float far, int n_rays, float* rays, void* stream) {
  if (n_rays < 0) return fail(NRN_E_INVALID, "nrn_pack_rays: bad size");
  if (n_rays == 0) return NRN_OK;
  if (!rays_o || !rays_d || !rays) return fail(NRN_E_INVALID, "nrn_pack_rays: null argument");
  const cudaError_t e = nrn::launch_pack_rays(rays_o, rays_d, near, far, n_rays, rays, static_cast<cudaStream_t>(stream));
  return e == cudaSuccess ? NRN_OK : cuda_fail(e, "pack_rays_kernel");
}

int nrn_ray_batch(const int64_t* pix, int n, const float* poses, const float* K, const int32_t* image_to_view, const float* images,
                  int H, int W, float* rays_o, float* rays_d, float* target, void* stream) {
  if (n < 0 || H < 1 || W < 1) return fail(NRN_E_INVALID, "nrn_ray_batch: bad sizes");
  if (n == 0) return NRN_OK;
  if (!pix || !poses || !K || !rays_o || !rays_d || (images && !target)) return fail(NRN_E_INVALID, "nrn_ray_batch: null argument");
  static_assert(sizeof(long long) == sizeof(int64_t), "int64");
  const cudaError_t e = nrn::launch_ray_batch(reinterpret_cast<const long long*>(pix), n, poses, K, image_to_view, images, H, W, rays_o, rays_d,
                                              target, static_cast<cudaStream_t>(stream));
  return e == cudaSuccess ? NRN_OK : cuda_fail(e, "ray_batch_kernel");
}

int nrn_median_visibility_index(const float* weights, int n_rays, int n_samples, int64_t* index, void* stream) {
  if (n_rays < 0 || n_samples < 1) return fail(NRN_E_INVALID, "nrn_median_visibility_index: bad sizes");
  if (n_rays == 0) return NRN_OK;
  if (!weights || !index) return fail(NRN_E_INVALID, "nrn_median_visibility_index: null argument");
  const cudaError_t e = nrn::launch_median_index(weights, n_rays, n_samples, reinterpret_cast<long long*>(index), static_cast<cudaStream_t>(stream));
  return e == cudaSuccess ? NRN_OK : cuda_fail(e, "median_index_kernel");
}

// nrn_field_forward, or with ray_bias (time-conditioned baseline, no bender) nrn_field_forward_tc
static int field_forward(const NrnFieldArgs* a, const float* ray_bias, const char* who) {
  long long P;
  int tiles;
  int rc = check_field_args(a, who, &P, &tiles);
  if (rc || P == 0) return rc;
  if (!a->raw) return fail(NRN_E_INVALID, "%s: null argument", who);
  if (a->points && a->n_samples != 1) return fail(NRN_E_INVALID, "%s: point mode needs n_samples=1, stride>=3", who);
  DeviceState* ds;
  rc = device_state(&ds);
  if (rc) return rc;
  nrn::FieldFwdParams p = field_fwd_params(a, P, tiles, ds->err_word);
  p.ray_bias = ray_bias; p.ray_bias_stride = a->latent_stride == 0 ? 0 : 2 * 256;
  cudaStream_t st = static_cast<cudaStream_t>(a->stream);
  if (ray_bias) return timed(0, st, "field_fwd_tc_kernel", [&] { return nrn::launch_field_fwd_tc(p, ds->num_sms, st); });
  return timed(0, st, "field_fwd_kernel", [&] { return nrn::launch_field_fwd(p, a->bender_packed != nullptr, ds->num_sms, st); });
}

int nrn_field_forward(const NrnFieldArgs* a) { return field_forward(a, nullptr, "nrn_field_forward"); }

int nrn_field_forward_tc(const NrnFieldArgs* a, const float* ray_bias) {
  if (!a) return fail(NRN_E_INVALID, "nrn_field_forward_tc: null args");
  if (a->bender_packed) return fail(NRN_E_INVALID, "nrn_field_forward_tc: the time-conditioned baseline has no bender (bender_packed must be NULL)");
  if (a->latent_stride < 0) return fail(NRN_E_INVALID, "nrn_field_forward_tc: latent_stride < 0");
  if (a->n_rays > 0 && !ray_bias) return fail(NRN_E_INVALID, "nrn_field_forward_tc: null ray_bias (nrn_tc_latent_bias output)");
  return field_forward(a, ray_bias, "nrn_field_forward_tc");
}

size_t nrn_packed_views_bytes(void) { return nrn::kViewsPackedBytes; }

int nrn_pack_views(const float* const* w, const float* const* b, void* packed, void* stream) {
  if (!w || !b || !packed) return fail(NRN_E_INVALID, "nrn_pack_views: null argument");
  if (!aligned16(packed)) return fail(NRN_E_INVALID, "nrn_pack_views: packed buffer must be 16-byte aligned");
  nrn::ViewsSrc src;
  for (int i = 0; i < 3; ++i) {
    if (!w[i] || !b[i]) return fail(NRN_E_INVALID, "nrn_pack_views: null layer %d", i);
    src.w[i] = w[i];
    src.b[i] = b[i];
  }
  const cudaError_t e = nrn::launch_pack_views(src, packed, static_cast<cudaStream_t>(stream));
  return e == cudaSuccess ? NRN_OK : cuda_fail(e, "pack_views_kernel");
}

size_t nrn_views_workspace_bytes(int n_rays, int n_samples) {
  if (n_rays < 0 || n_samples < 1) return 0;
  return static_cast<size_t>(n_rays) * n_samples * sizeof(float4);
}

// The view-dependent head: with a bender the bend pass (bent points and rigidities -> workspace, and the details), then,
// unless raw is NULL, the view-head kernel; without a bender the view-head kernel alone, on the given view directions.
int nrn_field_forward_views(const NrnFieldArgs* a, const NrnViewArgs* v) {
  const char* who = "nrn_field_forward_views";
  if (!a || !v) return fail(NRN_E_INVALID, "%s: null args", who);
  if (a->stash || a->relu_mask)
    return fail(NRN_E_INVALID, "%s: use_viewdirs=True is inference only (stash / relu_mask must be NULL; training is not implemented)", who);
  long long P;
  int tiles;
  int rc = check_field_args(a, who, &P, &tiles);
  if (rc) return rc;
  if (a->out_ch != 4) return fail(NRN_E_INVALID, "%s: out_ch=%d unsupported (use_viewdirs=True: 4 = rgb + alpha)", who, a->out_ch);
  const bool bend = a->bender_packed != nullptr;
  if (bend && a->raw && a->n_samples < 2)
    return fail(NRN_E_INVALID, "%s: use_viewdirs=True with a bender needs n_samples >= 2 (finite-difference view directions)", who);
  if (!bend && !a->raw) return fail(NRN_E_INVALID, "%s: raw is NULL without a bender (the bend pass alone needs one)", who);
  if (!bend && !v->viewdirs) return fail(NRN_E_INVALID, "%s: use_viewdirs=True without a bender needs viewdirs", who);
  if (!bend && v->viewdirs_stride < 3) return fail(NRN_E_INVALID, "%s: viewdirs_stride=%lld < 3", who, (long long)v->viewdirs_stride);
  if (P == 0) return NRN_OK;
  if (a->raw && !v->views_packed) return fail(NRN_E_INVALID, "%s: null nerf_packed / views_packed", who);
  if (bend && (!v->workspace || !aligned16(v->workspace)))
    return fail(NRN_E_INVALID, "%s: a bender needs the workspace (nrn_views_workspace_bytes, 16-byte aligned)", who);
  if (v->views_packed && !aligned16(v->views_packed)) return fail(NRN_E_INVALID, "%s: packed weights must be 16-byte aligned", who);
  DeviceState* ds;
  rc = device_state(&ds);
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(a->stream);
  nrn::FieldFwdParams p = field_fwd_params(a, P, tiles, ds->err_word);
  nrn::ViewParams vp{};
  const uint8_t* vw = static_cast<const uint8_t*>(v->views_packed);
  vp.w = vw; vp.bias = vw ? reinterpret_cast<const float*>(vw + nrn::kViewsWBytes) : nullptr;
  vp.viewdirs = v->viewdirs; vp.viewdirs_stride = v->viewdirs_stride;
  if (bend) {
    nrn::FieldFwdParams b = p;   // point mode: every point its own latent row
    if (a->points) { b.n_rays = static_cast<int>(P); b.S = 1; }
    vp.ws = static_cast<float4*>(v->workspace);
    rc = timed(8, st, "field_bend_kernel", [&] { return nrn::launch_field_bend(b, vp, ds->num_sms, st); });
    if (rc || !a->raw) return rc;
    p.d_init = p.d_bent = nullptr;   // the bend pass wrote them; the view-head kernel reads the bent points from the workspace
  }
  return timed(9, st, "field_views_kernel", [&] { return nrn::launch_field_views(p, vp, ds->num_sms, st); });
}

// ---- training the view-dependent head without a bender ----
size_t nrn_packed_views_t_bytes(void) { return nrn::kViewsTWBytes; }

int nrn_pack_views_t(const float* const* w, void* packed, void* stream) {
  if (!w || !packed) return fail(NRN_E_INVALID, "nrn_pack_views_t: null argument");
  if (!aligned16(packed)) return fail(NRN_E_INVALID, "nrn_pack_views_t: packed buffer must be 16-byte aligned");
  nrn::ViewsSrc src{};
  for (int i = 0; i < 3; ++i) {
    if (!w[i]) return fail(NRN_E_INVALID, "nrn_pack_views_t: null layer %d", i);
    src.w[i] = w[i];
  }
  const cudaError_t e = nrn::launch_pack_views_t(src, packed, static_cast<cudaStream_t>(stream));
  return e == cudaSuccess ? NRN_OK : cuda_fail(e, "pack_views_t_kernel");
}

size_t nrn_views_stash_bytes(int n_rays, int n_samples) {
  return n_rays < 0 || n_samples < 1 ? 0 : static_cast<size_t>(even_tiles(n_rays, n_samples)) * nrn::kVStashTileBytes;
}
size_t nrn_views_grad_stash_bytes(int n_rays, int n_samples) {
  return n_rays < 0 || n_samples < 1 ? 0 : static_cast<size_t>(even_tiles(n_rays, n_samples)) * nrn::kVGradTileBytes;
}
size_t nrn_hv_mask_bytes(int n_rays, int n_samples) {
  return n_rays < 0 || n_samples < 1 ? 0 : static_cast<size_t>(even_tiles(n_rays, n_samples)) * nrn::kHvMaskTileBytes;
}
int nrn_nerf_views_grad_floats(void) { return nrn::nerf_views_grad_floats(); }

int nrn_field_forward_views_train(const NrnFieldArgs* a, const NrnViewArgs* v, const NrnViewTrainArgs* t) {
  const char* who = "nrn_field_forward_views_train";
  if (!a || !v || !t) return fail(NRN_E_INVALID, "%s: null args", who);
  long long P;
  int tiles;
  int rc = check_field_args(a, who, &P, &tiles);
  if (rc) return rc;
  if (a->bender_packed)
    return fail(NRN_E_INVALID, "%s: training with the view-dependent head is not implemented with a ray bender (bender_packed must be NULL)", who);
  if (a->points) return fail(NRN_E_INVALID, "%s: training needs ray mode (points must be NULL)", who);
  if (a->out_ch != 4) return fail(NRN_E_INVALID, "%s: out_ch=%d unsupported (use_viewdirs=True: 4 = rgb + alpha)", who, a->out_ch);
  if (a->use_removal) return fail(NRN_E_INVALID, "%s: the object removal is a test-time knob; it is not differentiable", who);
  if (!v->viewdirs || v->viewdirs_stride < 3) return fail(NRN_E_INVALID, "%s: needs viewdirs with viewdirs_stride >= 3", who);
  if (P == 0) return NRN_OK;
  if (!a->raw || !v->views_packed) return fail(NRN_E_INVALID, "%s: null argument", who);
  if (!a->stash || !a->relu_mask || !t->views_stash || !t->hv_mask)
    return fail(NRN_E_INVALID, "%s: null stash, relu_mask, views_stash or hv_mask", who);
  if (!aligned16(v->views_packed) || !aligned16(t->views_stash) || !aligned16(t->hv_mask))
    return fail(NRN_E_INVALID, "%s: packed weights and stashes must be 16-byte aligned", who);
  DeviceState* ds;
  rc = device_state(&ds);
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(a->stream);
  const nrn::FieldFwdParams p = field_fwd_params(a, P, tiles, ds->err_word);
  nrn::ViewParams vp{};
  const uint8_t* vw = static_cast<const uint8_t*>(v->views_packed);
  vp.w = vw; vp.bias = reinterpret_cast<const float*>(vw + nrn::kViewsWBytes);
  vp.viewdirs = v->viewdirs; vp.viewdirs_stride = v->viewdirs_stride;
  const nrn::ViewTrainParams tp{static_cast<uint8_t*>(t->views_stash), static_cast<uint8_t*>(t->hv_mask)};
  return timed(10, st, "field_views_train_kernel", [&] { return nrn::launch_field_views_train(p, vp, tp, ds->num_sms, st); });
}

int nrn_field_backward_views(const NrnFieldBwdArgs* a, const NrnViewBwdArgs* v) {
  const char* who = "nrn_field_backward_views";
  if (!a || !v) return fail(NRN_E_INVALID, "%s: null args", who);
  if (a->bender_packed)
    return fail(NRN_E_INVALID, "%s: training with the view-dependent head is not implemented with a ray bender (bender_packed must be NULL)", who);
  long long P;
  int tiles;
  int rc = check_field_bwd_args(a, who, &P, &tiles);
  if (rc) return rc;
  if (a->out_ch != 4) return fail(NRN_E_INVALID, "%s: out_ch=%d unsupported (use_viewdirs=True: 4 = rgb + alpha)", who, a->out_ch);
  const int n_all = nrn::nerf_views_grad_floats();
  cudaStream_t st = static_cast<cudaStream_t>(a->stream);
  if (P == 0) return zero_grads(a, n_all, n_all - nrn::kViewsTrunkFloats, 0, st);
  if (!v->views_t_packed || !v->views_stash || !v->views_grad_stash || !v->hv_mask)
    return fail(NRN_E_INVALID, "%s: null views_t_packed, views_stash, views_grad_stash or hv_mask", who);
  if (!aligned16(v->views_t_packed) || !aligned16(v->views_stash) || !aligned16(v->views_grad_stash) || !aligned16(v->hv_mask))
    return fail(NRN_E_INVALID, "%s: packed weights and stashes must be 16-byte aligned", who);
  DeviceState* ds;
  rc = device_state(&ds);
  if (rc) return rc;
  if (ds->num_sms + 16 > nrn::kWgMaxCtas) return fail(NRN_E_INVALID, "%s: %d SMs exceed the scratch layout", who, ds->num_sms);
  float* amax = reinterpret_cast<float*>(ds->err_word + 1);
  const nrn::FieldBwdParams p = field_bwd_params(a, P, tiles, amax, ds->err_word);
  const nrn::ViewBwdParams vp{static_cast<const uint8_t*>(v->views_t_packed), static_cast<const uint8_t*>(v->hv_mask),
                              static_cast<uint8_t*>(v->views_grad_stash)};
  // the loss scale: max |d_raw| over the four channels (rgb and alpha)
  const cudaError_t e = nrn::launch_absmax(a->d_raw, P * 4, amax, st, false, 4, 4);
  if (e != cudaSuccess) return cuda_fail(e, "absmax_kernel");
  rc = timed(11, st, "field_bwd_views_kernel", [&] { return nrn::launch_field_bwd_views(p, vp, ds->num_sms, st); });
  if (rc) return rc;
  const nrn::WgradParams w = wgrad_params(p.stash, p.gstash, a->wgrad_scratch, amax, tiles, ds->err_word);
  const nrn::WgradViewParams wv{static_cast<const uint8_t*>(v->views_stash), vp.vgstash};
  const nrn::WgradDst dst{a->nerf_grad, a->nerf_grad_head, nullptr, n_all, 0, a->accumulate_nerf, 0};
  return timed(12, st, "wgrad_views_kernel", [&] { return nrn::launch_wgrad_views(w, wv, ds->num_sms, dst, st); });
}

int nrn_tc_latent_bias(const float* latents, int64_t latent_stride, int n_rays, const float* w0, const float* b0, const float* w5,
                       const float* b5, float* ray_bias, void* stream) {
  if (n_rays < 0 || latent_stride < 0) return fail(NRN_E_INVALID, "nrn_tc_latent_bias: bad sizes n=%d stride=%lld", n_rays, (long long)latent_stride);
  if (n_rays == 0) return NRN_OK;
  if (!latents || !w0 || !b0 || !w5 || !b5 || !ray_bias) return fail(NRN_E_INVALID, "nrn_tc_latent_bias: null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  return timed(6, st, "tc_latent_bias_kernel",
               [&] { return nrn::launch_tc_latent_bias(latents, latent_stride, n_rays, w0, b0, w5, b5, ray_bias, st); });
}

int nrn_composite(const NrnCompositeArgs* a) {
  if (!a) return fail(NRN_E_INVALID, "nrn_composite: null args");
  if (a->n_rays < 0 || a->n_samples < 1 || a->channels < 4) return fail(NRN_E_INVALID, "nrn_composite: bad sizes");
  if (a->n_rays == 0) return NRN_OK;
  if (!a->raw || !a->z_vals || !a->rays_d || !a->rgb_map || !a->disp_map || !a->acc_map) return fail(NRN_E_INVALID, "nrn_composite: null argument");
  if (a->n_importance < 0) return fail(NRN_E_INVALID, "nrn_composite: n_importance < 0");
  if (a->n_importance > 0 && (!a->z_vals_out || a->n_samples < 3)) return fail(NRN_E_INVALID, "nrn_composite: resampling needs z_vals_out and >= 3 samples");
  if (4 * a->n_samples + a->n_importance > 12000) return fail(NRN_E_INVALID, "nrn_composite: too many samples per ray");
  nrn::CompositeParams p{};
  p.raw = a->raw; p.z = a->z_vals; p.rays_d = a->rays_d; p.rays_d_stride = a->rays_d_stride; p.noise = a->noise;
  p.n = a->n_rays; p.S = a->n_samples; p.C = a->channels; p.white_bkgd = a->white_bkgd;
  p.rgb = a->rgb_map; p.disp = a->disp_map; p.acc = a->acc_map; p.depth = a->depth_map; p.weights = a->weights; p.alpha = a->alpha;
  p.n_imp = a->n_importance; p.u = a->u; p.z_out = a->z_vals_out; p.z_std = a->z_std;
  cudaStream_t st = static_cast<cudaStream_t>(a->stream);
  return timed(3, st, "composite_kernel", [&] { return nrn::launch_composite(p, st); });
}

int nrn_sample_pdf(const float* bins, const float* weights, const float* u, int n, int nbins, int n_samples, float* samples,
                   void* stream) {
  if (n < 0 || nbins < 2 || n_samples < 1 || nbins > 4000) return fail(NRN_E_INVALID, "nrn_sample_pdf: bad sizes");
  if (n == 0) return NRN_OK;
  if (!bins || !weights || !samples) return fail(NRN_E_INVALID, "nrn_sample_pdf: null argument");
  cudaError_t e = nrn::launch_sample_pdf(bins, weights, u, n, nbins, n_samples, samples, static_cast<cudaStream_t>(stream));
  return e == cudaSuccess ? NRN_OK : cuda_fail(e, "sample_pdf_kernel");
}

int nrn_composite_backward(const NrnCompositeBwdArgs* a) {
  if (!a) return fail(NRN_E_INVALID, "nrn_composite_backward: null args");
  if (a->n_rays < 0 || a->n_samples < 1 || a->channels < 4 || a->n_samples > 12000) return fail(NRN_E_INVALID, "nrn_composite_backward: bad sizes");
  if (a->n_rays == 0) return NRN_OK;
  if (!a->raw || !a->z_vals || !a->rays_d || !a->d_rgb_map || !a->d_raw) return fail(NRN_E_INVALID, "nrn_composite_backward: null argument");
  nrn::CompositeBwdParams p{};
  p.raw = a->raw; p.z = a->z_vals; p.rays_d = a->rays_d; p.rays_d_stride = a->rays_d_stride; p.noise = a->noise;
  p.n = a->n_rays; p.S = a->n_samples; p.C = a->channels; p.white_bkgd = a->white_bkgd;
  p.d_rgb = a->d_rgb_map; p.d_acc = a->d_acc_map; p.d_raw = a->d_raw;
  cudaStream_t st = static_cast<cudaStream_t>(a->stream);
  return timed(4, st, "composite_bwd_kernel", [&] { return nrn::launch_composite_bwd(p, st); });
}

size_t nrn_stash_bytes(int n_rays, int n_samples) { return static_cast<size_t>(even_tiles(n_rays, n_samples)) * nrn::kStashTileBytes; }
size_t nrn_grad_stash_bytes(int n_rays, int n_samples) { return static_cast<size_t>(even_tiles(n_rays, n_samples)) * nrn::kGradTileBytes; }
size_t nrn_relu_mask_bytes(int n_rays, int n_samples) { return static_cast<size_t>(even_tiles(n_rays, n_samples)) * nrn::kMaskTileBytes; }
size_t nrn_wgrad_scratch_bytes(void) { return static_cast<size_t>(nrn::kWgMaxCtas) * nrn::kWgScratchFloats * sizeof(float); }
int nrn_nerf_grad_floats(int out_ch) { return nrn::nerf_grad_floats(out_ch); }
int nrn_bender_grad_floats(void) { return nrn::bparam::total(); }
int nrn_nerf_tc_grad_floats(int out_ch) { return nrn::nerf_tc_grad_floats(out_ch); }
size_t nrn_tc_workspace_bytes(int n_rays) { return n_rays < 0 ? 0 : (static_cast<size_t>(n_rays) * 2 * 256 + 2 * 256 * nrn::kLatent) * sizeof(float); }

// nrn_field_backward, or with t (time-conditioned baseline, no bender) nrn_field_backward_tc, or with latent_rows
// (deterministic mode, bender) nrn_field_backward_det; with held (bender) the held-out variants of the last two
static int field_backward(const NrnFieldBwdArgs* a, const NrnTcBwdArgs* t, const char* who, float* latent_rows = nullptr,
                          const uint8_t* held = nullptr) {
  long long P;
  int tiles;
  int rc = check_field_bwd_args(a, who, &P, &tiles);
  if (rc) return rc;
  DeviceState* ds;
  rc = device_state(&ds);
  if (rc) return rc;
  if (ds->num_sms + 16 > nrn::kWgMaxCtas) return fail(NRN_E_INVALID, "%s: %d SMs exceed the scratch layout", who, ds->num_sms);
  cudaStream_t st = static_cast<cudaStream_t>(a->stream);
  const bool bend = a->bender_packed != nullptr;
  const int nerf_n = t ? nrn_nerf_tc_grad_floats(a->out_ch) : nrn_nerf_grad_floats(a->out_ch);
  const int bend_n = bend ? nrn_bender_grad_floats() : 0;
  cudaError_t e;
  if (bend && !latent_rows) {   // deterministic mode overwrites d_latents with the fixed-order sums
    e = cudaMemsetAsync(a->d_latents, 0, sizeof(float) * static_cast<size_t>(a->n_rays) * nrn::kLatent, st);
    if (e != cudaSuccess) return cuda_fail(e, "memset d_latents");
  }
  if (P == 0) return zero_grads(a, nerf_n, a->out_ch * 257, bend_n, st);
  float* amax = reinterpret_cast<float*>(ds->err_word + 1);
  const nrn::FieldBwdParams p = field_bwd_params(a, P, tiles, amax, ds->err_word);
  // DGRAD reads channels 0-3 of d_raw; channel 4 never reaches the loss and must not set the scale
  e = nrn::launch_absmax(a->d_raw, P * a->out_ch, amax, st, false, a->out_ch, 4);
  // the regularisers' upstream gradients share the fp16 loss scale: they take part in the maximum, otherwise a large
  // offsets_loss_weight saturates them (or, with a vanishing data term, lets them underflow)
  if (e == cudaSuccess && bend && p.d_unmasked_up) e = nrn::launch_absmax(p.d_unmasked_up, P * 3, amax, st, true);
  if (e == cudaSuccess && bend && p.d_rigid_up) e = nrn::launch_absmax(p.d_rigid_up, P, amax, st, true);
  if (e != cudaSuccess) return cuda_fail(e, "absmax_kernel");
  if (held) {
    rc = timed(15, st, "field_bwd_held_kernel", [&] { return nrn::launch_field_bwd_held(p, latent_rows, held, ds->num_sms, st); });
  } else if (latent_rows) {
    rc = timed(1, st, "field_bwd_det_kernel", [&] { return nrn::launch_field_bwd_det(p, latent_rows, ds->num_sms, st); });
  } else {
    rc = timed(1, st, "field_bwd_kernel", [&] { return nrn::launch_field_bwd(p, bend, ds->num_sms, st); });
  }
  if (rc) return rc;
  if (latent_rows) {
    rc = timed(13, st, "latent_reduce_kernel", [&] { return nrn::launch_latent_reduce(latent_rows, a->d_latents, a->n_rays, a->n_samples, st); });
    if (rc) return rc;
  }
  float* dw_lat = nullptr;
  if (t) {   // per-ray sums of dY0 / dY5 -> d z and the latent columns of dW0 / dW5 (before WGRAD's reduction reads them)
    nrn::TcBwdParams q{};
    q.gstash = p.gstash; q.amax = amax; q.P = P; q.S = p.S; q.n_rays = a->n_rays;
    q.latents = t->latents; q.latent_stride = t->latent_stride; q.w0 = t->w0; q.w5 = t->w5;
    q.sums = t->workspace; q.dw_lat = dw_lat = t->workspace + static_cast<size_t>(a->n_rays) * 2 * 256; q.d_latents = t->d_latents;
    rc = timed(7, st, "tc_ray_sums_kernel", [&] { return nrn::launch_tc_latent_bwd(q, st); });
    if (rc) return rc;
  }
  const nrn::WgradParams w = wgrad_params(p.stash, p.gstash, a->wgrad_scratch, amax, tiles, ds->err_word);
  const nrn::WgradDst dst{a->nerf_grad, a->nerf_grad_head, a->bender_grad, nerf_n, bend_n, a->accumulate_nerf, a->accumulate_bender};
  return timed(2, st, "wgrad_kernel", [&] { return nrn::launch_wgrad(w, bend, ds->num_sms, dst, a->out_ch, st, dw_lat); });
}

int nrn_field_backward(const NrnFieldBwdArgs* a) { return field_backward(a, nullptr, "nrn_field_backward"); }

size_t nrn_latent_rows_bytes(int n_rays, int n_samples) {
  return n_rays < 0 || n_samples < 1 ? 0 : static_cast<size_t>(n_rays) * n_samples * nrn::kLatent * sizeof(float);
}
size_t nrn_div_loss_rows_bytes(int n_rays, int n_samples) {
  return n_rays < 0 || n_samples < 1 ? 0 : static_cast<size_t>(n_rays) * n_samples * sizeof(float);
}

int nrn_field_backward_det(const NrnFieldBwdArgs* a, float* latent_rows) {
  const char* who = "nrn_field_backward_det";
  if (!a) return fail(NRN_E_INVALID, "%s: null args", who);
  if (!a->bender_packed || !a->d_latents)
    return fail(NRN_E_INVALID, "%s: needs a bender (bender_packed) and d_latents: only the bender's latent gradient has a fixed-order variant", who);
  if (a->n_rays == 0) return field_backward(a, nullptr, who);   // an empty shard: zero gradients, no kernel
  if (!latent_rows || !aligned16(latent_rows)) return fail(NRN_E_INVALID, "%s: null or unaligned latent_rows (nrn_latent_rows_bytes, 16-byte aligned)", who);
  return field_backward(a, nullptr, who, latent_rows);
}

// the checks both held-out entry points add to those of field_backward
static int check_held_out(const NrnFieldBwdArgs* a, const uint8_t* held, const char* who) {
  if (!a) return fail(NRN_E_INVALID, "%s: null args", who);
  if (!a->bender_packed || !a->d_latents)
    return fail(NRN_E_INVALID, "%s: needs a bender (bender_packed) and d_latents; without a bender a held-out ray contributes "
                "nothing: zero its rows of d_raw and call nrn_field_backward", who);
  if (a->n_rays > 0 && !held) return fail(NRN_E_INVALID, "%s: null held_out_rays", who);
  return NRN_OK;
}

int nrn_field_backward_held_out(const NrnFieldBwdArgs* a, const uint8_t* held_out_rays) {
  const char* who = "nrn_field_backward_held_out";
  const int rc = check_held_out(a, held_out_rays, who);
  if (rc) return rc;
  return field_backward(a, nullptr, who, nullptr, a->n_rays > 0 ? held_out_rays : nullptr);
}

int nrn_field_backward_det_held_out(const NrnFieldBwdArgs* a, float* latent_rows, const uint8_t* held_out_rays) {
  const char* who = "nrn_field_backward_det_held_out";
  const int rc = check_held_out(a, held_out_rays, who);
  if (rc) return rc;
  if (a->n_rays == 0) return field_backward(a, nullptr, who);   // an empty shard: zero gradients, no kernel
  if (!latent_rows || !aligned16(latent_rows)) return fail(NRN_E_INVALID, "%s: null or unaligned latent_rows (nrn_latent_rows_bytes, 16-byte aligned)", who);
  return field_backward(a, nullptr, who, latent_rows, held_out_rays);
}

int nrn_field_backward_tc(const NrnFieldBwdArgs* a, const NrnTcBwdArgs* t) {
  if (!a || !t) return fail(NRN_E_INVALID, "nrn_field_backward_tc: null args");
  if (a->bender_packed) return fail(NRN_E_INVALID, "nrn_field_backward_tc: the time-conditioned baseline has no bender (bender_packed must be NULL)");
  if (t->latent_stride < 0) return fail(NRN_E_INVALID, "nrn_field_backward_tc: latent_stride < 0");
  if (a->n_rays > 0 && (!t->latents || !t->w0 || !t->w5 || !t->d_latents || !t->workspace))
    return fail(NRN_E_INVALID, "nrn_field_backward_tc: null latents, w0, w5, d_latents or workspace");
  return field_backward(a, t, "nrn_field_backward_tc");
}

size_t nrn_div_stash_bytes(int n_rays, int n_samples) {
  return static_cast<size_t>(tile_count(static_cast<long long>(n_rays) * n_samples)) * nrn::kTanTileBytes;
}
size_t nrn_div_grad_stash_bytes(int n_rays, int n_samples) {
  return static_cast<size_t>(tile_count(static_cast<long long>(n_rays) * n_samples)) * nrn::kAdjTileBytes;
}

static int fill_div(const NrnDivArgs* a, nrn::DivParams& p, const char* who) {
  if (!a) return fail(NRN_E_INVALID, "%s: null args", who);
  if (a->n_rays < 0 || a->n_samples < 1) return fail(NRN_E_INVALID, "%s: bad sizes", who);
  if (!a->relu_mask) return fail(NRN_E_INVALID, "%s: null relu_mask (the ReLU masks of the coarse nrn_field_forward call)", who);
  if (!a->bender_packed) return fail(NRN_E_INVALID, "%s: null bender_packed (the nrn_pack_bender output the coarse pass ran with)", who);
  if (!aligned16(a->bender_packed)) return fail(NRN_E_INVALID, "%s: bender_packed must be 16-byte aligned", who);
  if (!a->e || !a->unmasked_offsets || !a->rigidity_mask || !a->weights || !a->tangent_stash || !a->d || !a->alpha || !a->beta ||
      !a->tau_c)
    return fail(NRN_E_INVALID, "%s: null argument", who);
  p.P = static_cast<long long>(a->n_rays) * a->n_samples;
  p.S = a->n_samples; p.n_rays = a->n_rays;
  p.relu_mask = static_cast<const uint8_t*>(a->relu_mask);
  p.bender = static_cast<const uint8_t*>(a->bender_packed);
  p.e = a->e; p.unmasked = a->unmasked_offsets; p.rigidity = a->rigidity_mask; p.w = a->weights; p.w_is_alpha = a->weights_are_opacity_alpha != 0;
  p.tan = static_cast<uint8_t*>(a->tangent_stash);
  p.d = a->d; p.adot = a->alpha; p.beta = a->beta; p.tauc = a->tau_c;
  return NRN_OK;
}

int nrn_divergence_forward(const NrnDivArgs* a) {
  nrn::DivParams p{};
  int rc = fill_div(a, p, "nrn_divergence_forward");
  if (rc) return rc;
  if (!a->loss) return fail(NRN_E_INVALID, "nrn_divergence_forward: null loss");
  DeviceState* ds;
  rc = device_state(&ds);
  if (rc) return rc;
  p.err = ds->err_word;
  cudaStream_t st = static_cast<cudaStream_t>(a->stream);
  cudaError_t e = cudaMemsetAsync(a->loss, 0, sizeof(float) * static_cast<size_t>(a->n_rays), st);
  if (e != cudaSuccess) return cuda_fail(e, "memset loss");
  p.loss = a->loss;
  return timed(5, st, "div_fwd_kernel", [&] { return nrn::launch_div_fwd(p, ds->num_sms, st); });
}

int nrn_divergence_forward_det(const NrnDivArgs* a, float* loss_rows) {
  const char* who = "nrn_divergence_forward_det";
  nrn::DivParams p{};
  int rc = fill_div(a, p, who);
  if (rc) return rc;
  if (!a->loss) return fail(NRN_E_INVALID, "%s: null loss", who);
  if (a->n_rays == 0) return NRN_OK;
  if (!loss_rows) return fail(NRN_E_INVALID, "%s: null loss_rows (nrn_div_loss_rows_bytes)", who);
  DeviceState* ds;
  rc = device_state(&ds);
  if (rc) return rc;
  p.err = ds->err_word;
  cudaStream_t st = static_cast<cudaStream_t>(a->stream);
  rc = timed(5, st, "div_fwd_det_kernel", [&] { return nrn::launch_div_fwd_det(p, loss_rows, ds->num_sms, st); });
  if (rc) return rc;
  return timed(14, st, "div_loss_reduce_kernel", [&] { return nrn::launch_div_loss_reduce(loss_rows, a->loss, a->n_rays, a->n_samples, st); });
}

// nrn_divergence_backward, or with held its held-out variant
static int divergence_backward(const NrnDivArgs* a, const uint8_t* held, const char* who) {
  nrn::DivParams p{};
  int rc = fill_div(a, p, who);
  if (rc) return rc;
  if ((!a->G && !(a->g_ray && a->G_workspace)) || !a->adjoint_stash || !a->wgrad_scratch || !a->d_unmasked_offsets || !a->d_rigidity_mask ||
      !a->bender_grad)
    return fail(NRN_E_INVALID, "%s: null argument", who);
  DeviceState* ds;
  rc = device_state(&ds);
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(a->stream);
  float* amax = reinterpret_cast<float*>(ds->err_word + 2);
  p.G = a->G ? a->G : a->G_workspace; p.amax = amax; p.adj = static_cast<uint8_t*>(a->adjoint_stash);
  p.d_unmasked = a->d_unmasked_offsets; p.d_rigid = a->d_rigidity_mask; p.err = ds->err_word;
  cudaError_t e = a->G ? nrn::launch_absmax(a->G, p.P, amax, st) : nrn::launch_div_G(p, a->g_ray, a->G_workspace, amax, st);
  if (e != cudaSuccess) return cuda_fail(e, "absmax_kernel");
  if (held) rc = timed(16, st, "div_bwd_held_kernel", [&] { return nrn::launch_div_bwd_held(p, held, ds->num_sms, st); });
  else rc = timed(5, st, "div_bwd_kernel", [&] { return nrn::launch_div_bwd(p, ds->num_sms, st); });
  if (rc) return rc;
  nrn::WgradParams w = wgrad_params(p.tan, p.adj, a->wgrad_scratch, amax, static_cast<int>(tile_count(p.P)), ds->err_word);
  w.compact = 1;
  const nrn::WgradDst dst{nullptr, nullptr, a->bender_grad, 0, nrn_bender_grad_floats(), 0, a->accumulate_bender};
  return timed(2, st, "wgrad_kernel (divergence)", [&] { return nrn::launch_wgrad(w, true, ds->num_sms, dst, 5, st); });
}

int nrn_divergence_backward(const NrnDivArgs* a) { return divergence_backward(a, nullptr, "nrn_divergence_backward"); }

int nrn_divergence_backward_held_out(const NrnDivArgs* a, const uint8_t* held_out_rays) {
  const char* who = "nrn_divergence_backward_held_out";
  if (a && a->n_rays > 0 && !held_out_rays) return fail(NRN_E_INVALID, "%s: null held_out_rays", who);
  return divergence_backward(a, held_out_rays, who);
}

int nrn_ray_loss(const NrnRayLossArgs* a) {
  if (!a) return fail(NRN_E_INVALID, "nrn_ray_loss: null args");
  if (a->n_rays < 0 || a->n_samples < 1) return fail(NRN_E_INVALID, "nrn_ray_loss: bad sizes");
  if (a->n_rays == 0) return NRN_OK;
  if (!a->rgb || !a->target || !a->loss || !a->u_rgb || (a->rgb0 && !a->u_rgb0)) return fail(NRN_E_INVALID, "nrn_ray_loss: null argument");
  if (a->unmasked_offsets && (!a->weights || !a->rigidity_mask || !a->u_unmasked_offsets || !a->u_rigidity_mask))
    return fail(NRN_E_INVALID, "nrn_ray_loss: the offsets term needs weights, rigidity_mask and both gradient outputs");
  if (a->divergence && !a->u_divergence) return fail(NRN_E_INVALID, "nrn_ray_loss: the divergence term needs u_divergence");
  if (a->sched_step && !(a->sched_n_iters > 0.f)) return fail(NRN_E_INVALID, "nrn_ray_loss: sched_n_iters must be positive");
  nrn::RayLossParams p{};
  p.n = a->n_rays; p.S = a->n_samples;
  p.rgb = a->rgb; p.rgb0 = a->rgb0; p.target = a->target; p.w = a->weights; p.off = a->unmasked_offsets; p.rig = a->rigidity_mask;
  p.lam_o = a->lam_offsets; p.lam_r = a->lam_rigidity;
  p.sched_step = a->sched_step; p.sched_n_iters = a->sched_n_iters; p.div = a->divergence; p.lam_div = a->lam_divergence; p.u_div = a->u_divergence;
  p.loss = a->loss; p.u_rgb = a->u_rgb; p.u_rgb0 = a->u_rgb0; p.u_off = a->u_unmasked_offsets; p.u_rig = a->u_rigidity_mask;
  cudaError_t e = nrn::launch_ray_loss(p, static_cast<cudaStream_t>(a->stream));
  return e == cudaSuccess ? NRN_OK : cuda_fail(e, "ray_loss_kernel");
}

int nrn_ray_loss_backward(const NrnRayLossBwdArgs* a) {
  if (!a) return fail(NRN_E_INVALID, "nrn_ray_loss_backward: null args");
  if (a->n_rays < 0 || a->n_samples < 1) return fail(NRN_E_INVALID, "nrn_ray_loss_backward: bad sizes");
  if (a->n_rays == 0) return NRN_OK;
  if (!a->g) return fail(NRN_E_INVALID, "nrn_ray_loss_backward: null upstream gradient");
  nrn::RayLossBwdParams p{};
  p.n = a->n_rays; p.S = a->n_samples; p.g = a->g;
  const float* u[5] = {a->u_rgb, a->u_rgb0, a->u_unmasked_offsets, a->u_rigidity_mask, a->u_divergence};
  float* d[5] = {a->d_rgb, a->d_rgb0, a->d_unmasked_offsets, a->d_rigidity_mask, a->d_divergence};
  for (int k = 0; k < 5; ++k) {
    if ((u[k] == nullptr) != (d[k] == nullptr)) return fail(NRN_E_INVALID, "nrn_ray_loss_backward: unit / output pair %d half given", k);
    p.u[k] = u[k]; p.d[k] = d[k];
  }
  const cudaError_t e = nrn::launch_ray_loss_bwd(p, static_cast<cudaStream_t>(a->stream));
  return e == cudaSuccess ? NRN_OK : cuda_fail(e, "ray_loss_bwd_kernel");
}

int nrn_scale_rows(const float* g, const float* unit, float* out, int64_t n, int per_row, void* stream) {
  if (n < 0 || per_row < 1) return fail(NRN_E_INVALID, "nrn_scale_rows: bad sizes");
  if (n == 0) return NRN_OK;
  if (!g || !unit || !out) return fail(NRN_E_INVALID, "nrn_scale_rows: null argument");
  cudaError_t e = nrn::launch_ray_loss_scale(g, unit, out, n, per_row, static_cast<cudaStream_t>(stream));
  return e == cudaSuccess ? NRN_OK : cuda_fail(e, "ray_loss_scale_kernel");
}

static int fill_adam(const NrnAdamArgs* a, nrn::AdamParams& p, const char* who, bool need_grads);
int nrn_adam_step(const NrnAdamArgs* a) {
  nrn::AdamParams p{};
  const int rc = fill_adam(a, p, "nrn_adam_step", true);
  if (rc) return rc;
  const cudaError_t e = nrn::launch_adam(p, a->n_tensors, a->n_blocks, static_cast<cudaStream_t>(a->stream));
  return e == cudaSuccess ? NRN_OK : cuda_fail(e, "adam_kernel");
}

static int fill_adam(const NrnAdamArgs* a, nrn::AdamParams& p, const char* who, bool need_grads) {
  if (!a) return fail(NRN_E_INVALID, "%s: null args", who);
  if (a->n_blocks < 0 || a->n_tensors < 0) return fail(NRN_E_INVALID, "%s: n_tensors = %d, n_blocks = %d", who, a->n_tensors, a->n_blocks);
  if (!a->params || !a->exp_avg || !a->exp_avg_sq || (need_grads && !a->grad_ptrs) || !a->blocks || !a->lr || !a->step)
    return fail(NRN_E_INVALID, "%s: null buffer", who);
  if (!(a->beta1 >= 0.f && a->beta1 < 1.f && a->beta2 >= 0.f && a->beta2 < 1.f && a->eps >= 0.f))
    return fail(NRN_E_INVALID, "%s: betas / eps out of range", who);
  p.params = static_cast<float*>(a->params); p.exp_avg = static_cast<float*>(a->exp_avg); p.exp_avg_sq = static_cast<float*>(a->exp_avg_sq);
  p.grads = static_cast<const float* const*>(a->grad_ptrs); p.blocks = static_cast<const nrn::AdamBlock*>(a->blocks);
  p.lr = static_cast<const float*>(a->lr); p.step = static_cast<long long*>(a->step);
  p.beta1 = a->beta1; p.beta2 = a->beta2; p.eps = a->eps;
  return NRN_OK;
}

size_t nrn_peer_window_bytes(int64_t arena_floats, int64_t slot_floats) {
  if (arena_floats < 0 || slot_floats < 0) return 0;
  const size_t slot_bytes = (static_cast<size_t>(slot_floats) * 4 + 255) / 256 * 256;
  return nrn::kPeerFlagBytes + 2 * slot_bytes + (static_cast<size_t>(arena_floats) * 4 + 255) / 256 * 256;
}

int nrn_peer_alloc(size_t bytes, void** dev_ptr, void* ipc_handle) {
  if (!dev_ptr || !ipc_handle || bytes < nrn::kPeerFlagBytes) return fail(NRN_E_INVALID, "nrn_peer_alloc: bad arguments");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handle size");
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, bytes);
  if (e != cudaSuccess) return cuda_fail(e, "cudaMalloc(peer window)");
  e = cudaMemset(p, 0, bytes);
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  cudaIpcMemHandle_t h;
  if (e == cudaSuccess) e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) { cudaFree(p); return cuda_fail(e, "cudaIpcGetMemHandle"); }
  memcpy(ipc_handle, &h, sizeof(h));
  *dev_ptr = p;
  return NRN_OK;
}

int nrn_peer_open(const void* ipc_handle, void** dev_ptr) {
  if (!ipc_handle || !dev_ptr) return fail(NRN_E_INVALID, "nrn_peer_open: null argument");
  cudaIpcMemHandle_t h;
  memcpy(&h, ipc_handle, sizeof(h));
  void* p = nullptr;
  const cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) return cuda_fail(e, "cudaIpcOpenMemHandle (peer-to-peer access between the GPUs of this node is required)");
  *dev_ptr = p;
  return NRN_OK;
}

int nrn_peer_close(void* dev_ptr) {
  if (!dev_ptr) return NRN_OK;
  const cudaError_t e = cudaIpcCloseMemHandle(dev_ptr);
  return e == cudaSuccess ? NRN_OK : cuda_fail(e, "cudaIpcCloseMemHandle");
}

int nrn_peer_free(void* dev_ptr) {
  if (!dev_ptr) return NRN_OK;
  const cudaError_t e = cudaFree(dev_ptr);
  return e == cudaSuccess ? NRN_OK : cuda_fail(e, "cudaFree(peer window)");
}

static int fill_peer(const NrnPeerCtx* c, nrn::PeerCtx& p, const char* who) {
  if (!c) return fail(NRN_E_INVALID, "%s: null context", who);
  if (c->world < 1 || c->world > nrn::kPeerMaxRanks || c->rank < 0 || c->rank >= c->world)
    return fail(NRN_E_INVALID, "%s: world = %d, rank = %d (at most %d ranks of one node)", who, c->world, c->rank, nrn::kPeerMaxRanks);
  if (!c->state || c->arena_floats < 0 || c->slot_floats < 0) return fail(NRN_E_INVALID, "%s: bad context", who);
  for (int r = 0; r < c->world; ++r) {
    if (!c->window[r]) return fail(NRN_E_INVALID, "%s: window of rank %d not mapped", who, r);
    p.window[r] = static_cast<uint8_t*>(c->window[r]);
  }
  p.world = c->world; p.rank = c->rank;
  p.slot_off = nrn::kPeerFlagBytes;
  p.slot_bytes = (static_cast<size_t>(c->slot_floats) * 4 + 255) / 256 * 256;
  p.arena_off = p.slot_off + 2 * p.slot_bytes;
  return NRN_OK;
}

int nrn_peer_reduce_adam(const NrnPeerCtx* c, const NrnAdamArgs* a) {
  nrn::PeerCtx pc{};
  int rc = fill_peer(c, pc, "nrn_peer_reduce_adam");
  if (rc) return rc;
  nrn::AdamParams p{};
  rc = fill_adam(a, p, "nrn_peer_reduce_adam", false);
  if (rc) return rc;
  if (!c->reduced) return fail(NRN_E_INVALID, "nrn_peer_reduce_adam: null workspace");
  DeviceState* ds;
  rc = device_state(&ds);
  if (rc) return rc;
  uint32_t* state = static_cast<uint32_t*>(c->state);
  const cudaError_t e = nrn::launch_peer_reduce_adam(pc, p, a->n_tensors, a->n_blocks, c->arena_floats, state, c->reduced, state + 3,
                                                     ds->err_word, static_cast<cudaStream_t>(a->stream));
  return e == cudaSuccess ? NRN_OK : cuda_fail(e, "peer_adam_kernel");
}

int nrn_peer_gather_rows(const NrnPeerCtx* c, const float* local, int n_per_rank, float* out, void* stream) {
  nrn::PeerCtx pc{};
  int rc = fill_peer(c, pc, "nrn_peer_gather_rows");
  if (rc) return rc;
  if (n_per_rank < 0 || n_per_rank > c->slot_floats) return fail(NRN_E_INVALID, "nrn_peer_gather_rows: %d floats per rank exceed the slot (%lld)", n_per_rank, (long long)c->slot_floats);
  if (n_per_rank == 0) return NRN_OK;
  if (!local || !out) return fail(NRN_E_INVALID, "nrn_peer_gather_rows: null argument");
  DeviceState* ds;
  rc = device_state(&ds);
  if (rc) return rc;
  const cudaError_t e = nrn::launch_peer_gather(pc, static_cast<uint32_t*>(c->state), local, n_per_rank, out, ds->err_word, static_cast<cudaStream_t>(stream));
  return e == cudaSuccess ? NRN_OK : cuda_fail(e, "peer_collect_kernel");
}

// ---- evaluation and visualisation of rendered frames (eval.cu) ----
int nrn_jet_colormap(double* rgb, uint8_t* rgb8) {
  if (!rgb && !rgb8) return fail(NRN_E_INVALID, "nrn_jet_colormap: null argument");
  nrn::jet_table(rgb, rgb8);
  return NRN_OK;
}

static bool aligned4(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3u) == 0; }   // NULL passes
static size_t eval_mask_offset(int F, int H, int W) { return (nrn::eval_partials_bytes(F, H, W) + 15) / 16 * 16; }

size_t nrn_image_scores_bytes(int n_frames, int height, int width) {
  if (n_frames < 0 || height < 1 || width < 1) return 0;
  return eval_mask_offset(n_frames, height, width) + (static_cast<size_t>(height) * width + 15) / 16 * 16;
}

// The sizes every evaluation entry point accepts: n_frames >= 0, height and width >= 1, and a grid of at most 2^31 - 1
// blocks of `per_block` elements (n_frames * height * width pixels or SSIM tiles)
static int check_frames(int F, int H, int W, long long per_frame, long long per_block, const char* who) {
  if (F < 0 || H < 1 || W < 1) return fail(NRN_E_INVALID, "%s: bad sizes F=%d H=%d W=%d", who, F, H, W);
  if ((static_cast<long long>(F) * per_frame + per_block - 1) / per_block > 0x7fffffffLL) return fail(NRN_E_INVALID, "%s: too many frames", who);
  return NRN_OK;
}

int nrn_image_scores(const NrnImageScoreArgs* a) {
  const char* who = "nrn_image_scores";
  if (!a) return fail(NRN_E_INVALID, "%s: null args", who);
  int rc = check_frames(a->n_frames, a->height, a->width, nrn::eval_tiles_per_frame(a->height, a->width), 1, who);
  if (rc) return rc;
  if (a->n_frames == 0) return NRN_OK;
  if (!a->gt || !a->generated || !a->psnr || !a->ssim || !a->workspace) return fail(NRN_E_INVALID, "%s: null argument", who);
  if (!aligned16(a->workspace)) return fail(NRN_E_INVALID, "%s: workspace must be 16-byte aligned", who);
  if (!aligned4(a->gt) || !aligned4(a->generated) || !aligned4(a->psnr) || !aligned4(a->ssim) || !aligned4(a->ssim_map))
    return fail(NRN_E_INVALID, "%s: float arrays must be 4-byte aligned", who);
  const int F = a->n_frames, H = a->height, W = a->width;
  uint8_t* derived = static_cast<uint8_t*>(a->workspace) + eval_mask_offset(F, H, W);
  nrn::ImageScoreParams p{a->gt, a->generated, a->mask ? a->mask : derived, F, H, W, a->psnr, a->ssim, a->ssim_map,
                          a->error_rgb, a->error_ssim, static_cast<double*>(a->workspace)};
  const cudaStream_t st = static_cast<cudaStream_t>(a->stream);
  if (!a->mask) {
    rc = timed(17, st, "frame_mask_kernel", [&] { return nrn::launch_frame_mask(a->gt, H, W, derived, st); });
    if (rc) return rc;
  }
  rc = timed(17, st, "ssim_tile_kernel", [&] { return nrn::launch_image_scores(p, st); });
  if (rc) return rc;
  return timed(17, st, "score_reduce_kernel", [&] { return nrn::launch_score_reduce(p, st); });
}

int nrn_disparity_images(const float* disp, int F, int H, int W, float* jet, float* phong, void* stream) {
  const char* who = "nrn_disparity_images";
  int rc = check_frames(F, H, W, static_cast<long long>(H) * W, 256, who);
  if (rc) return rc;
  if (phong && (H < 2 || W < 2)) return fail(NRN_E_INVALID, "%s: the Phong image needs height and width >= 2 (np.gradient)", who);
  if (F == 0) return NRN_OK;
  if (!disp || (!jet && !phong)) return fail(NRN_E_INVALID, "%s: null argument", who);
  if (!aligned4(disp) || !aligned4(jet) || !aligned4(phong)) return fail(NRN_E_INVALID, "%s: float arrays must be 4-byte aligned", who);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  return timed(18, st, "disparity_kernel", [&] { return nrn::launch_disparity_images(disp, F, H, W, jet, phong, st); });
}

int nrn_frame_std_image(const float* rgbs, int F, int H, int W, float* std_out, float* image, void* stream) {
  const char* who = "nrn_frame_std_image";
  int rc = check_frames(1, H, W, static_cast<long long>(H) * W, 128, who);
  if (rc) return rc;
  if (F < 0) return fail(NRN_E_INVALID, "%s: bad sizes F=%d", who, F);
  if (F == 0) return NRN_OK;
  if (!rgbs || (!std_out && !image)) return fail(NRN_E_INVALID, "%s: null argument", who);
  if (!aligned4(rgbs) || !aligned4(std_out) || !aligned4(image)) return fail(NRN_E_INVALID, "%s: float arrays must be 4-byte aligned", who);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  return timed(19, st, "frame_std_kernel", [&] { return nrn::launch_frame_std(rgbs, F, H, W, std_out, image, st); });
}

int nrn_frame_images(const NrnFrameImageArgs* a) {
  const char* who = "nrn_frame_images";
  if (!a) return fail(NRN_E_INVALID, "%s: null args", who);
  const int F = a->n_frames, H = a->height, W = a->width;
  if (F < 0 || H < 0 || W < 0) return fail(NRN_E_INVALID, "%s: bad sizes F=%d H=%d W=%d", who, F, H, W);
  if (static_cast<double>(F) * H * W * 3 > 9.0e18) return fail(NRN_E_INVALID, "%s: too many pixels", who);
  if (static_cast<long long>(F) * H * W == 0) return NRN_OK;
  const bool disp_out = a->out_disp || a->out_disp_video || a->out_disp_jet || a->out_disp_phong;
  if (!a->out_rgb && !disp_out && !a->out_correspondences && !a->out_rigidity && !a->out_rigidity_jet)
    return fail(NRN_E_INVALID, "%s: no output", who);
  if ((a->out_rgb && !a->rgb) || (disp_out && (!a->disp || !a->disp_max)) ||
      (a->out_correspondences && (!a->surface_pts || !a->min_point || !a->max_point)) ||
      ((a->out_rigidity || a->out_rigidity_jet) && !a->surface_rigidity))
    return fail(NRN_E_INVALID, "%s: an output without its input (null argument)", who);
  if (a->out_disp_phong && (H < 2 || W < 2))
    return fail(NRN_E_INVALID, "%s: the Phong image needs height and width >= 2 (np.gradient)", who);
  if (!aligned4(a->rgb) || !aligned4(a->disp) || !aligned4(a->surface_pts) || !aligned4(a->surface_rigidity) || !aligned4(a->disp_max))
    return fail(NRN_E_INVALID, "%s: float arrays must be 4-byte aligned", who);
  nrn::FrameImageParams p{};
  if (a->out_correspondences)
    for (int c = 0; c < 3; ++c) {
      if (!(a->max_point[c] > a->min_point[c])) return fail(NRN_E_INVALID, "%s: max_point must exceed min_point on every axis", who);
      p.min_point[c] = a->min_point[c];
      p.max_point[c] = a->max_point[c];
    }
  // inputs whose outputs are not asked for stay unread
  p.rgb = a->out_rgb ? a->rgb : nullptr;
  p.disp = disp_out ? a->disp : nullptr;
  p.surface_pts = a->out_correspondences ? a->surface_pts : nullptr;
  p.surface_rigidity = (a->out_rigidity || a->out_rigidity_jet) ? a->surface_rigidity : nullptr;
  p.F = F; p.H = H; p.W = W;
  p.disp_max = a->disp_max;
  p.out_rgb = a->out_rgb; p.out_disp = a->out_disp; p.out_disp_video = a->out_disp_video; p.out_disp_jet = a->out_disp_jet;
  p.out_disp_phong = a->out_disp_phong; p.out_correspondences = a->out_correspondences; p.out_rigidity = a->out_rigidity;
  p.out_rigidity_jet = a->out_rigidity_jet;
  const cudaStream_t st = static_cast<cudaStream_t>(a->stream);
  if (disp_out) {
    const int rc = timed(20, st, "disp_max_kernel", [&] { return nrn::launch_disp_max(a->disp, F, H, W, a->disp_max, st); });
    if (rc) return rc;
  }
  return timed(20, st, "frame_images_kernel", [&] { return nrn::launch_frame_images(p, st); });
}

// ---- triangle meshes --------------------------------------------------------------------------------------------------
static bool mesh_plane_ok(int nx, int ny) {
  return nx >= 2 && ny >= 2 && nx <= nrn::kMeshMaxAxis && ny <= nrn::kMeshMaxAxis && static_cast<long long>(nx) * ny <= nrn::kMeshMaxPlane;
}

// The grid of a slab call: sizes in range, 0 <= k < nz, and (when the extent is needed) finite min < max on every axis
static int mesh_grid(const float* lo, const float* hi, int nx, int ny, int nz, int k, bool need_extent, const char* who, nrn::MeshGrid* g) {
  if (!mesh_plane_ok(nx, ny) || nz < 2 || nz > nrn::kMeshMaxAxis || k < 0 || k >= nz)
    return fail(NRN_E_INVALID, "%s: bad sizes nx=%d ny=%d nz=%d k=%d (2 <= n <= 2^24 per axis, nx * ny <= 2^28, 0 <= k < nz)", who, nx, ny, nz, k);
  *g = nrn::MeshGrid{};
  g->n[0] = nx; g->n[1] = ny; g->n[2] = nz;
  if (!need_extent) return NRN_OK;
  if (!lo || !hi) return fail(NRN_E_INVALID, "%s: null min_point / max_point", who);
  for (int a = 0; a < 3; ++a) {
    if (!(hi[a] > lo[a]) || !isfinite(lo[a]) || !isfinite(hi[a]))
      return fail(NRN_E_INVALID, "%s: max_point must exceed min_point on every axis (finite values)", who);
    g->lo[a] = lo[a]; g->hi[a] = hi[a];
  }
  return NRN_OK;
}

int nrn_mesh_grid_points(const float* min_point, const float* max_point, int nx, int ny, int nz, int k, float* points, void* stream) {
  const char* who = "nrn_mesh_grid_points";
  nrn::MeshGrid g;
  const int rc = mesh_grid(min_point, max_point, nx, ny, nz, k, true, who, &g);
  if (rc) return rc;
  if (!points) return fail(NRN_E_INVALID, "%s: null points", who);
  if (!aligned4(points)) return fail(NRN_E_INVALID, "%s: points must be 4-byte aligned", who);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  return timed(21, st, "mesh_grid_points_kernel", [&] { return nrn::launch_mesh_grid_points(g, k, points, st); });
}

int nrn_mesh_sigma(const float* raw, long long n, int out_ch, float* sigma, void* stream) {
  const char* who = "nrn_mesh_sigma";
  if (n < 0 || out_ch < 4 || out_ch > 5 || n > (1LL << 40)) return fail(NRN_E_INVALID, "%s: bad sizes n=%lld out_ch=%d", who, n, out_ch);
  if (n == 0) return NRN_OK;
  if (!raw || !sigma) return fail(NRN_E_INVALID, "%s: null argument", who);
  if (!aligned4(raw) || !aligned4(sigma)) return fail(NRN_E_INVALID, "%s: float arrays must be 4-byte aligned", who);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  return timed(21, st, "mesh_sigma_kernel", [&] { return nrn::launch_mesh_sigma(raw, n, out_ch, sigma, st); });
}

size_t nrn_mesh_workspace_bytes(int nx, int ny) { return mesh_plane_ok(nx, ny) ? nrn::mesh_workspace_bytes(nx, ny) : 0; }

// The checks both slab entry points share: sizes, the planes (sigma1 exactly when k < nz - 1) and the workspace
static int mesh_slab(const NrnMeshSlabArgs* a, bool emit, const char* who, nrn::MeshGrid* g) {
  if (!a) return fail(NRN_E_INVALID, "%s: null args", who);
  const int rc = mesh_grid(a->min_point, a->max_point, a->nx, a->ny, a->nz, a->k, emit, who, g);
  if (rc) return rc;
  if (!a->sigma0 || !a->workspace) return fail(NRN_E_INVALID, "%s: null sigma0 / workspace", who);
  if ((a->sigma1 != nullptr) != (a->k + 1 < a->nz))
    return fail(NRN_E_INVALID, "%s: sigma1 (plane k + 1) must be given exactly when k < nz - 1", who);
  if (!(a->threshold == a->threshold)) return fail(NRN_E_INVALID, "%s: threshold is NaN", who);
  if (!aligned4(a->sigma0) || !aligned4(a->sigma1) || (reinterpret_cast<uintptr_t>(a->workspace) & 255u))
    return fail(NRN_E_INVALID, "%s: sigma must be 4-byte and the workspace 256-byte aligned", who);
  return NRN_OK;
}

int nrn_mesh_count(const NrnMeshSlabArgs* a) {
  const char* who = "nrn_mesh_count";
  nrn::MeshGrid g;
  int rc = mesh_slab(a, false, who, &g);
  if (rc) return rc;
  if (!a->totals || !aligned4(a->totals)) return fail(NRN_E_INVALID, "%s: null or misaligned totals", who);
  const int nx = a->nx, ny = a->ny;
  const long long n = static_cast<long long>(nx) * ny, nc = static_cast<long long>(nx - 1) * (ny - 1);
  const nrn::MeshPlaneState s = nrn::mesh_plane_state(a->workspace, nx, ny, a->k % nrn::kMeshSlots);
  int32_t* partials = nrn::mesh_scan_partials(a->workspace, nx, ny);
  const cudaStream_t st = static_cast<cudaStream_t>(a->stream);
  return timed(22, st, "mesh_count_kernel", [&] {
    cudaError_t e = nrn::launch_mesh_count(g, a->sigma0, a->sigma1, a->threshold, s, st);
    if (e == cudaSuccess) e = nrn::launch_mesh_scan(s.voff, n + 1, partials, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(a->totals, s.voff + n, sizeof(int32_t), cudaMemcpyDeviceToDevice, st);
    if (e == cudaSuccess && a->sigma1) e = nrn::launch_mesh_scan(s.toff, nc + 1, partials, st);
    if (e == cudaSuccess) e = a->sigma1 ? cudaMemcpyAsync(a->totals + 1, s.toff + nc, sizeof(int32_t), cudaMemcpyDeviceToDevice, st)
                                        : cudaMemsetAsync(a->totals + 1, 0, sizeof(int32_t), st);
    return e;
  });
}

int nrn_mesh_emit(const NrnMeshSlabArgs* a) {
  const char* who = "nrn_mesh_emit";
  nrn::MeshGrid g;
  int rc = mesh_slab(a, true, who, &g);
  if (rc) return rc;
  if (!a->vertices || (a->k > 0 && !a->faces)) return fail(NRN_E_INVALID, "%s: null vertices / faces", who);
  if (!aligned4(a->vertices) || !aligned4(a->faces)) return fail(NRN_E_INVALID, "%s: vertices and faces must be 4-byte aligned", who);
  const long long lim = 0x7fffffffLL;
  if (a->vertex_base < 0 || a->vertex_base_prev < 0 || a->face_base < 0 || a->vertex_base > lim || a->face_base > lim ||
      (a->k > 0 && a->vertex_base_prev > a->vertex_base))
    return fail(NRN_E_INVALID, "%s: bases out of range (0 <= vertex_base_prev <= vertex_base < 2^31, 0 <= face_base < 2^31)", who);
  const int slot = a->k % nrn::kMeshSlots;
  const nrn::MeshPlaneState s = nrn::mesh_plane_state(a->workspace, a->nx, a->ny, slot);
  const cudaStream_t st = static_cast<cudaStream_t>(a->stream);
  return timed(23, st, "mesh_emit_kernels", [&] {
    cudaError_t e = nrn::launch_mesh_vertices(g, a->k, a->sigma0, a->sigma1, a->threshold, s, a->vertex_base, a->vertices, st);
    if (e == cudaSuccess && a->k > 0) {
      const nrn::MeshPlaneState lower = nrn::mesh_plane_state(a->workspace, a->nx, a->ny, (a->k - 1) % nrn::kMeshSlots);
      e = nrn::launch_mesh_faces(g, lower, s, a->vertex_base_prev, a->vertex_base, a->face_base, a->faces, st);
    }
    return e;
  });
}

int nrn_mesh_colors(const float* raw, long long n, int out_ch, uint8_t* colors, void* stream) {
  const char* who = "nrn_mesh_colors";
  if (n < 0 || out_ch < 4 || out_ch > 5 || n > (1LL << 40)) return fail(NRN_E_INVALID, "%s: bad sizes n=%lld out_ch=%d", who, n, out_ch);
  if (n == 0) return NRN_OK;
  if (!raw || !colors) return fail(NRN_E_INVALID, "%s: null argument", who);
  if (!aligned4(raw)) return fail(NRN_E_INVALID, "%s: raw must be 4-byte aligned", who);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  return timed(24, st, "mesh_colors_kernel", [&] { return nrn::launch_mesh_colors(raw, n, out_ch, colors, st); });
}

int nrn_mesh_cube_table(int32_t* counts, int8_t* edges) {
  nrn::mesh_cube_table(counts, edges);
  return NRN_OK;
}

// ---- LPIPS (lpips.cu) -------------------------------------------------------------------------------------------------
size_t nrn_lpips_packed_bytes(void) { return nrn::kLpipsPackedBytes; }

int nrn_lpips_pack(const float* const* tensors, void* packed, void* stream) {
  const char* who = "nrn_lpips_pack";
  if (!tensors || !packed) return fail(NRN_E_INVALID, "%s: null argument", who);
  for (int i = 0; i < 17; ++i)
    if (!tensors[i]) return fail(NRN_E_INVALID, "%s: null tensor %d", who, i);
    else if (!aligned4(tensors[i])) return fail(NRN_E_INVALID, "%s: tensor %d must be 4-byte aligned", who, i);
  if (!aligned16(packed)) return fail(NRN_E_INVALID, "%s: packed buffer must be 16-byte aligned", who);
  nrn::LpipsPackSources s;
  for (int l = 0; l < nrn::kLpipsTaps; ++l) {
    s.conv_w[l] = tensors[2 * l];
    s.conv_b[l] = tensors[2 * l + 1];
    s.lin[l] = tensors[10 + l];
  }
  s.shift = tensors[15];
  s.scale = tensors[16];
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const cudaError_t e = nrn::launch_lpips_pack(s, static_cast<uint8_t*>(packed), st);
  return e == cudaSuccess ? NRN_OK : cuda_fail(e, "lpips_pack_kernel");
}

static bool lpips_size_ok(int H, int W) {
  return H >= nrn::kLpipsMinSide && W >= nrn::kLpipsMinSide && H <= nrn::kLpipsMaxSide && W <= nrn::kLpipsMaxSide;
}

// The default workspace of F frames whose per-frame bytes are frame_bytes(H, W)
static size_t lpips_default_workspace(int n_frames, int height, int width, size_t (*frame_bytes)(int, int)) {
  if (n_frames < 0 || !lpips_size_ok(height, width)) return 0;
  const size_t frame = frame_bytes(height, width);
  size_t fc = nrn::kLpipsChunkBudget / frame;
  fc = fc < 1 ? 1 : (fc > static_cast<size_t>(nrn::kLpipsMaxChunk) ? nrn::kLpipsMaxChunk : fc);
  if (fc > static_cast<size_t>(n_frames)) fc = n_frames;
  return nrn::lpips_mask_bytes(height, width) + fc * frame;
}

size_t nrn_lpips_workspace_bytes(int n_frames, int height, int width) {
  return lpips_default_workspace(n_frames, height, width, nrn::lpips_frame_bytes);
}

size_t nrn_lpips_maps_workspace_bytes(int n_frames, int height, int width) {
  return lpips_default_workspace(n_frames, height, width, nrn::lpips_map_frame_bytes);
}

// nrn_lpips (m == NULL) and nrn_lpips_maps: the same checks, chunks and kernels; with maps the distance kernels also
// store their tap maps and the upsample kernel turns them into the chunk's maps after the reduce
static int lpips_run(const NrnLpipsArgs* a, const NrnLpipsMapArgs* m, const char* who) {
  if (!a) return fail(NRN_E_INVALID, "%s: null args", who);
  const int F = a->n_frames, H = a->height, W = a->width;
  if (F < 0 || H < 0 || W < 0) return fail(NRN_E_INVALID, "%s: bad sizes F=%d H=%d W=%d", who, F, H, W);
  if (!lpips_size_ok(H, W))
    return fail(NRN_E_INVALID, "%s: frames of %d x %d pixels: height and width must be at least %d (every AlexNet tap needs a pixel) "
                "and at most %d", who, H, W, nrn::kLpipsMinSide, nrn::kLpipsMaxSide);
  if (F == 0) return NRN_OK;
  if (!a->gt || !a->generated || !a->packed || !a->lpips || !a->workspace || (m && !m->map))
    return fail(NRN_E_INVALID, "%s: null argument", who);
  if (!aligned4(a->gt) || !aligned4(a->generated) || !aligned4(a->lpips) || !aligned4(a->per_layer) ||
      (m && (!aligned4(m->map) || !aligned4(m->layer_maps))))
    return fail(NRN_E_INVALID, "%s: float arrays must be 4-byte aligned", who);
  if (!aligned16(a->packed) || (reinterpret_cast<uintptr_t>(a->workspace) & 255u))
    return fail(NRN_E_INVALID, "%s: packed weights must be 16-byte and the workspace 256-byte aligned", who);
  const size_t mask_bytes = nrn::lpips_mask_bytes(H, W), frame = m ? nrn::lpips_map_frame_bytes(H, W) : nrn::lpips_frame_bytes(H, W);
  if (a->workspace_bytes < mask_bytes + frame)
    return fail(NRN_E_INVALID, "%s: workspace of %zu bytes holds no frame (%zu needed for one)", who, a->workspace_bytes, mask_bytes + frame);
  size_t fc_max = (a->workspace_bytes - mask_bytes) / frame;
  if (fc_max > static_cast<size_t>(nrn::kLpipsMaxChunk)) fc_max = nrn::kLpipsMaxChunk;
  DeviceState* ds = nullptr;
  int rc = device_state(&ds);
  if (rc) return rc;
  const cudaStream_t st = static_cast<cudaStream_t>(a->stream);
  const uint8_t* packed = static_cast<const uint8_t*>(a->packed);
  uint8_t* mask = static_cast<uint8_t*>(a->workspace);
  if (a->mask) mask = const_cast<uint8_t*>(a->mask);
  else if ((rc = timed(25, st, "frame_mask_kernel", [&] { return nrn::launch_frame_mask(a->gt, H, W, mask, st); }))) return rc;
  const nrn::LpipsDims d = nrn::lpips_dims(H, W);
  const size_t frame_floats = static_cast<size_t>(H) * W * 3;
  for (int f0 = 0; f0 < F; f0 += static_cast<int>(fc_max)) {
    const int fc = F - f0 < static_cast<int>(fc_max) ? F - f0 : static_cast<int>(fc_max);
    const nrn::LpipsChunk c = nrn::lpips_chunk(a->workspace, fc, H, W);
    const cudaError_t ze = cudaMemsetAsync(c.sat, 0, 2 * static_cast<size_t>(fc) * sizeof(unsigned), st);
    if (ze != cudaSuccess) return cuda_fail(ze, "lpips saturation words");
    rc = timed(25, st, "lpips_input_kernel", [&] {
      return nrn::launch_lpips_input(a->gt + f0 * frame_floats, a->generated + f0 * frame_floats, mask, packed, fc, H, W, c.act[0], st);
    });
    for (int l = 0; l < nrn::kLpipsTaps && !rc; ++l) {
      const int si = nrn::kLpipsTapStage[l];
      if (l == 1 || l == 2)   // conv2 and conv3 read the max-pool of the stage before theirs
        rc = timed(27, st, "lpips_pool_kernel", [&] {
          return nrn::launch_lpips_pool(c.act[si - 2], c.act[si - 1], 2 * fc, d.h[si - 2], d.w[si - 2], d.h[si - 1], d.w[si - 1],
                                        nrn::kLpipsStageChannels[si - 2], st);
        });
      if (!rc)
        rc = timed(26, st, "lpips_conv_kernel", [&] {
          return nrn::launch_lpips_conv(l, d, c.act[l == 0 ? 0 : si - 1], c.act[si], packed, 2 * fc, ds->num_sms, ds->err_word, c.sat, st);
        });
      if (!rc)
        rc = timed(28, st, "lpips_distance_kernel", [&] {
          return m ? nrn::launch_lpips_distance_map(l, d, c, packed, nrn::lpips_tap_map(a->workspace, fc, H, W, l), st)
                   : nrn::launch_lpips_distance(l, d, c, packed, st);
        });
    }
    if (!rc)
      rc = timed(28, st, "lpips_reduce_kernel", [&] {
        return nrn::launch_lpips_reduce(d, c, a->lpips + f0, a->per_layer ? a->per_layer + static_cast<size_t>(f0) * nrn::kLpipsTaps : nullptr, st);
      });
    if (!rc && m)
      rc = timed(44, st, "lpips_upsample_kernel", [&] {
        nrn::LpipsUpsampleParams p;
        for (int l = 0; l < nrn::kLpipsTaps; ++l) {
          const int s = nrn::kLpipsTapStage[l];
          p.tap[l] = nrn::lpips_tap_map(a->workspace, fc, H, W, l);
          p.h[l] = d.h[s];
          p.w[l] = d.w[s];
          p.scale_y[l] = static_cast<float>(d.h[s]) / static_cast<float>(H);
          p.scale_x[l] = static_cast<float>(d.w[s]) / static_cast<float>(W);
        }
        p.sat = c.sat;
        p.fc = fc;
        p.H = H;
        p.W = W;
        const size_t px0 = static_cast<size_t>(f0) * H * W;
        p.map = m->map + px0;
        p.layer_maps = m->layer_maps ? m->layer_maps + px0 * nrn::kLpipsTaps : nullptr;
        p.error_image = m->error_image ? m->error_image + px0 * 3 : nullptr;
        return nrn::launch_lpips_upsample(p, st);
      });
    if (rc) return rc;
  }
  return NRN_OK;
}

int nrn_lpips(const NrnLpipsArgs* a) { return lpips_run(a, nullptr, "nrn_lpips"); }

int nrn_lpips_maps(const NrnLpipsArgs* a, const NrnLpipsMapArgs* maps) {
  if (!maps) return fail(NRN_E_INVALID, "nrn_lpips_maps: null args");
  return lpips_run(a, maps, "nrn_lpips_maps");
}

// ---- correspondences (match.cu) ---------------------------------------------------------------------------------------
static bool match_frame_ok(int H, int W) {
  return H >= 1 && W >= 1 && H <= nrn::kMatchMaxSide && W <= nrn::kMatchMaxSide &&
         static_cast<long long>(H) * W <= nrn::kMatchMaxPoints;
}

// The output frame count of Fq query frames against Ft target frames, or -1 when they do not pair
static int match_pairs(int Fq, int Ft) {
  if (Fq < 0 || Ft < 0 || Fq > nrn::kMatchMaxFrames || Ft > nrn::kMatchMaxFrames) return -1;
  if (Fq == Ft || Ft == 1) return Fq;
  if (Fq == 1) return Ft;
  return -1;
}

size_t nrn_match_workspace_bytes(int n_query_frames, int query_height, int query_width, int n_target_frames, int target_height,
                                 int target_width, int round_trip) {
  if (match_pairs(n_query_frames, n_target_frames) < 0 || !match_frame_ok(query_height, query_width) ||
      !match_frame_ok(target_height, target_width))
    return 0;
  size_t b = nrn::match_cloud_bytes(n_target_frames, static_cast<long long>(target_height) * target_width);
  if (round_trip) b += nrn::match_cloud_bytes(n_query_frames, static_cast<long long>(query_height) * query_width);
  return b;
}

int nrn_match(const NrnMatchArgs* a) {
  const char* who = "nrn_match";
  if (!a) return fail(NRN_E_INVALID, "%s: null args", who);
  const int Fq = a->n_query_frames, Ft = a->n_target_frames;
  if (!match_frame_ok(a->query_height, a->query_width) || !match_frame_ok(a->target_height, a->target_width))
    return fail(NRN_E_INVALID, "%s: frames of %d x %d (query) and %d x %d (target) pixels: height and width must be 1 to %d and "
                "a frame at most %lld points", who, a->query_height, a->query_width, a->target_height, a->target_width,
                nrn::kMatchMaxSide, nrn::kMatchMaxPoints);
  const int F = match_pairs(Fq, Ft);
  if (F < 0)
    return fail(NRN_E_INVALID, "%s: %d query frames do not pair with %d target frames (equal counts, or one frame on either "
                "side, at most %d)", who, Fq, Ft, nrn::kMatchMaxFrames);
  if (!(a->max_distance >= 0.f)) return fail(NRN_E_INVALID, "%s: max_distance %g must be >= 0 (not NaN)", who, a->max_distance);
  if (a->round_trip && !(a->round_trip_pixels >= 0.f))
    return fail(NRN_E_INVALID, "%s: round_trip_pixels %g must be >= 0 (not NaN)", who, a->round_trip_pixels);
  if (F == 0) return NRN_OK;
  if (!a->query || !a->target || !a->index || !a->distance || !a->flow || !a->workspace || (a->round_trip && !a->consistent))
    return fail(NRN_E_INVALID, "%s: null argument", who);
  if (!aligned4(a->query) || !aligned4(a->target) || !aligned4(a->index) || !aligned4(a->distance) || !aligned4(a->flow))
    return fail(NRN_E_INVALID, "%s: float and index arrays must be 4-byte aligned", who);
  if (reinterpret_cast<uintptr_t>(a->workspace) & 255u) return fail(NRN_E_INVALID, "%s: the workspace must be 256-byte aligned", who);
  const size_t need = nrn_match_workspace_bytes(Fq, a->query_height, a->query_width, Ft, a->target_height, a->target_width, a->round_trip);
  if (a->workspace_bytes < need) return fail(NRN_E_INVALID, "%s: workspace of %zu bytes, %zu needed", who, a->workspace_bytes, need);
  DeviceState* ds = nullptr;
  int rc = device_state(&ds);
  if (rc) return rc;
  const cudaStream_t st = static_cast<cudaStream_t>(a->stream);
  const long long Nq = static_cast<long long>(a->query_height) * a->query_width;
  const long long Nt = static_cast<long long>(a->target_height) * a->target_width;
  nrn::MatchQueryParams p{};
  p.t = nrn::match_cloud(a->workspace, a->target, a->target_mask, Ft, Nt);
  if (a->round_trip) {
    p.q = nrn::match_cloud(static_cast<uint8_t*>(a->workspace) + nrn::match_cloud_bytes(Ft, Nt), a->query, a->query_mask, Fq, Nq);
  } else {
    p.q = nrn::MatchCloud{};
    p.q.pts = a->query; p.q.mask = a->query_mask; p.q.F = Fq; p.q.N = Nq;
  }
  p.F = F; p.Wq = a->query_width; p.Wt = a->target_width;
  p.max_d2 = a->max_distance * a->max_distance;
  p.round_trip = a->round_trip ? 1 : 0;
  p.rt_tol2 = a->round_trip_pixels * a->round_trip_pixels;
  p.index = a->index; p.distance = a->distance; p.flow = a->flow;
  p.consistent = a->round_trip ? a->consistent : nullptr;
  rc = timed(29, st, "match_build_kernels", [&] { return nrn::launch_match_build(p.t, ds->num_sms, st); });
  if (!rc && a->round_trip) rc = timed(29, st, "match_build_kernels", [&] { return nrn::launch_match_build(p.q, ds->num_sms, st); });
  if (!rc) rc = timed(30, st, "match_query_kernel", [&] { return nrn::launch_match_query(p, st); });
  return rc;
}

// ---- occupancy grid: build, lookup + compaction, and the render pass that skips empty cells ----
static size_t align256(size_t n) { return (n + 255) & ~static_cast<size_t>(255); }
static bool occ_sides_ok(int nx, int ny, int nz) {
  return nx >= 1 && ny >= 1 && nz >= 1 && nx <= nrn::kOccMaxSide && ny <= nrn::kOccMaxSide && nz <= nrn::kOccMaxSide;
}
static size_t occ_block_count_bytes(long long P) { return align256(sizeof(int32_t) * ((P + nrn::kOccTile - 1) / nrn::kOccTile + 1)); }

// The grid as the kernels read it; NRN_E_INVALID for a malformed one
static int occ_grid(const NrnOccupancyGrid* g, const char* who, nrn::OccGrid* out) {
  if (!g) return fail(NRN_E_INVALID, "%s: null grid", who);
  if (!occ_sides_ok(g->nx, g->ny, g->nz))
    return fail(NRN_E_INVALID, "%s: grid resolution %d x %d x %d out of range (1..%d cells per axis)", who, g->nx, g->ny, g->nz, nrn::kOccMaxSide);
  if (!g->bits || (reinterpret_cast<uintptr_t>(g->bits) & 3u)) return fail(NRN_E_INVALID, "%s: grid bits null or not 4-byte aligned", who);
  nrn::OccGrid o{};
  o.bits = g->bits; o.nx = g->nx; o.ny = g->ny; o.nz = g->nz;
  const int n[3] = {g->nx, g->ny, g->nz};
  for (int d = 0; d < 3; ++d) {
    const float lo = g->min_point[d], hi = g->max_point[d];
    if (!(std::isfinite(lo) && std::isfinite(hi) && hi > lo)) return fail(NRN_E_INVALID, "%s: grid box must be finite with max > min on every axis", who);
    const float ext = hi - lo;
    const float sc = static_cast<float>(n[d]) / ext;
    if (!(std::isfinite(ext) && std::isfinite(sc) && sc > 0.f)) return fail(NRN_E_INVALID, "%s: grid box extent out of fp32 range", who);
    o.lo[d] = lo; o.hi[d] = hi; o.scale[d] = sc;
  }
  *out = o;
  return NRN_OK;
}

size_t nrn_occupancy_words(int nx, int ny, int nz) {
  if (!occ_sides_ok(nx, ny, nz)) return 0;
  return static_cast<size_t>((static_cast<long long>(nx) * ny * nz + 31) / 32);
}

size_t nrn_occupancy_build_workspace_bytes(int nx, int ny, int nz) {
  if (!occ_sides_ok(nx, ny, nz)) return 0;
  return 2 * static_cast<size_t>(nx) * ny * nz;
}

int nrn_occupancy_build(const float* sigma, int nx, int ny, int nz, float threshold, int dilation, void* workspace, uint32_t* bits,
                        void* stream) {
  const char* who = "nrn_occupancy_build";
  if (!occ_sides_ok(nx, ny, nz)) return fail(NRN_E_INVALID, "%s: resolution %d x %d x %d out of range (1..%d cells per axis)", who, nx, ny, nz, nrn::kOccMaxSide);
  if (dilation < 0 || dilation > nrn::kOccMaxDilation) return fail(NRN_E_INVALID, "%s: dilation=%d out of range (0..%d)", who, dilation, nrn::kOccMaxDilation);
  if (threshold != threshold) return fail(NRN_E_INVALID, "%s: threshold is NaN", who);
  if (!sigma || !workspace || !bits) return fail(NRN_E_INVALID, "%s: null argument", who);
  if (reinterpret_cast<uintptr_t>(bits) & 3u) return fail(NRN_E_INVALID, "%s: bits must be 4-byte aligned", who);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  return timed(31, st, "occupancy_build", [&] {
    return nrn::launch_occupancy_build(sigma, nx, ny, nz, threshold, dilation, static_cast<uint8_t*>(workspace), bits, st);
  });
}

size_t nrn_occupancy_compact_workspace_bytes(int64_t n_points) {
  if (n_points < 0 || n_points > nrn::kOccMaxPoints) return 0;
  return occ_block_count_bytes(n_points);
}

int nrn_occupancy_compact(const NrnOccupancyGrid* grid, const float* points, int64_t n_points, int64_t points_stride, float* kept_xyz,
                          int32_t* kept_index, int32_t* count, void* workspace, void* stream) {
  const char* who = "nrn_occupancy_compact";
  nrn::OccGrid g;
  int rc = occ_grid(grid, who, &g);
  if (rc) return rc;
  if (n_points < 0 || n_points > nrn::kOccMaxPoints) return fail(NRN_E_INVALID, "%s: n_points=%lld out of range (0..2^31 - 1)", who, (long long)n_points);
  if (points_stride < 3) return fail(NRN_E_INVALID, "%s: points_stride < 3", who);
  if (!count || !workspace || (n_points > 0 && (!points || !kept_xyz || !kept_index))) return fail(NRN_E_INVALID, "%s: null argument", who);
  if (reinterpret_cast<uintptr_t>(workspace) & 255u) return fail(NRN_E_INVALID, "%s: workspace must be 256-byte aligned", who);
  nrn::OccPoints s{};
  s.pts = points; s.pts_stride = points_stride; s.P = n_points; s.S = 1;
  nrn::OccCompact c{};
  c.kept_xyz = kept_xyz; c.kept_idx = kept_index; c.count = count; c.block_counts = static_cast<int32_t*>(workspace);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  return timed(33, st, "occupancy_compact", [&] { return nrn::launch_occupancy_compact(g, s, c, st); });
}

size_t nrn_occupancy_workspace_bytes(int n_rays, int n_samples, int out_ch, int has_bender) {
  if (n_rays < 0 || n_samples < 1 || out_ch < 4 || out_ch > 5) return 0;
  const long long P = static_cast<long long>(n_rays) * n_samples;
  if (P > nrn::kOccMaxPoints) return 0;
  const size_t p = static_cast<size_t>(P);
  return (has_bender ? align256(p * sizeof(float4)) : 0) + align256(p * 3 * sizeof(float)) + align256(p * sizeof(int32_t)) +
         align256(p * out_ch * sizeof(float)) + align256(sizeof(int32_t)) + occ_block_count_bytes(P);
}

int nrn_field_forward_occupancy(const NrnFieldArgs* a, const NrnOccupancyGrid* grid, void* workspace, size_t workspace_bytes) {
  const char* who = "nrn_field_forward_occupancy";
  long long P;
  int tiles;
  int rc = check_field_args(a, who, &P, &tiles);
  if (rc) return rc;
  if (a->stash || a->relu_mask) return fail(NRN_E_INVALID, "%s: inference only (stash / relu_mask must be NULL)", who);
  if (a->points) return fail(NRN_E_INVALID, "%s: needs ray mode (rays and z_vals; points must be NULL)", who);
  nrn::OccGrid g;
  rc = occ_grid(grid, who, &g);
  if (rc) return rc;
  if (P > nrn::kOccMaxPoints) return fail(NRN_E_INVALID, "%s: %lld points in one pass (at most 2^31 - 1)", who, P);
  if (P == 0) return NRN_OK;
  const bool bend = a->bender_packed != nullptr;
  if (!a->raw) return fail(NRN_E_INVALID, "%s: null raw", who);
  const size_t need = nrn_occupancy_workspace_bytes(a->n_rays, a->n_samples, a->out_ch, bend);
  if (!workspace || (reinterpret_cast<uintptr_t>(workspace) & 255u) || workspace_bytes < need)
    return fail(NRN_E_INVALID, "%s: workspace null, not 256-byte aligned or smaller than nrn_occupancy_workspace_bytes (%zu)", who, need);
  DeviceState* ds;
  rc = device_state(&ds);
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(a->stream);
  const size_t p = static_cast<size_t>(P);
  uint8_t* w = static_cast<uint8_t*>(workspace);
  float4* ws = nullptr;
  if (bend) { ws = reinterpret_cast<float4*>(w); w += align256(p * sizeof(float4)); }
  float* kept_xyz = reinterpret_cast<float*>(w); w += align256(p * 3 * sizeof(float));
  int32_t* kept_idx = reinterpret_cast<int32_t*>(w); w += align256(p * sizeof(int32_t));
  float* craw = reinterpret_cast<float*>(w); w += align256(p * a->out_ch * sizeof(float));
  int32_t* count = reinterpret_cast<int32_t*>(w); w += align256(sizeof(int32_t));
  int32_t* block_counts = reinterpret_cast<int32_t*>(w);

  nrn::FieldFwdParams p0 = field_fwd_params(a, P, tiles, ds->err_word);
  // a. the bend pass: bent points and rigidities -> ws, and the details
  if (bend) {
    nrn::ViewParams vp{};
    vp.ws = ws;
    rc = timed(32, st, "field_bend_kernel", [&] { return nrn::launch_field_bend(p0, vp, ds->num_sms, st); });
    if (rc) return rc;
  }
  // b. lookup and compaction (without a bender the points come from the rays and depths, with their details)
  nrn::OccPoints s{};
  s.ws = ws; s.rays = a->rays; s.z_vals = a->z_vals; s.S = a->n_samples; s.P = P;
  nrn::OccCompact c{};
  c.kept_xyz = kept_xyz; c.kept_idx = kept_idx; c.count = count; c.block_counts = block_counts;
  if (!bend) { c.d_init = a->initial_input_pts; c.d_bent = a->input_pts; }
  rc = timed(33, st, "occupancy_compact", [&] { return nrn::launch_occupancy_compact(g, s, c, st); });
  if (rc) return rc;
  // c. the point-mode trunk on the kept points, their count read on the device
  nrn::FieldFwdParams q{};
  q.pts = kept_xyz; q.pts_stride = 3; q.n_rays = static_cast<int>(P); q.S = 1; q.P = P; q.n_tiles = tiles;
  q.nerf_w = p0.nerf_w; q.nerf_bias = p0.nerf_bias; q.out_ch = a->out_ch; q.raw = craw; q.err = ds->err_word;
  rc = timed(34, st, "field_fwd_kept_kernel", [&] { return nrn::launch_field_fwd_kept(q, count, ds->num_sms, st); });
  if (rc) return rc;
  // d. raw of every sample: the trunk's where kept (with the object removal), zero elsewhere
  return timed(35, st, "occupancy_scatter", [&] {
    return nrn::launch_occupancy_scatter(craw, kept_idx, count, P, a->out_ch, ws, a->use_removal, a->removal_threshold, a->raw, ds->num_sms, st);
  });
}

// ---- early ray termination: a render pass in depth-ordered rounds over segments of nrn_termination_segment() samples ----
int nrn_termination_segment(void) { return nrn::kTermSegment; }

size_t nrn_termination_workspace_bytes(int n_rays, int n_samples, int out_ch, int has_bender) {
  if (n_rays < 0 || n_samples < 1 || out_ch < 4 || out_ch > 5) return 0;
  const long long P = static_cast<long long>(n_rays) * n_samples;
  if (P > nrn::kOccMaxPoints) return 0;
  const size_t p = static_cast<size_t>(P);
  const long long Pk = static_cast<long long>(n_rays) * std::min(nrn::kTermSegment, n_samples);   // the slots of one round
  const size_t pk = static_cast<size_t>(Pk);
  return (has_bender ? align256(p * sizeof(float4)) : 0) + align256(pk * 3 * sizeof(float)) + align256(pk * sizeof(int32_t)) +
         align256(pk * out_ch * sizeof(float)) + align256(sizeof(int32_t)) + occ_block_count_bytes(Pk) +
         align256(static_cast<size_t>(n_rays) * sizeof(float));
}

int nrn_field_forward_terminate(const NrnFieldArgs* a, const NrnOccupancyGrid* grid, const NrnTerminationArgs* term, void* workspace,
                                size_t workspace_bytes) {
  const char* who = "nrn_field_forward_terminate";
  long long P;
  int tiles;
  int rc = check_field_args(a, who, &P, &tiles);
  if (rc) return rc;
  if (a->stash || a->relu_mask) return fail(NRN_E_INVALID, "%s: inference only (stash / relu_mask must be NULL)", who);
  if (a->points) return fail(NRN_E_INVALID, "%s: needs ray mode (rays and z_vals; points must be NULL)", who);
  if (!term) return fail(NRN_E_INVALID, "%s: null termination args", who);
  if (!(term->threshold >= 0.f && term->threshold <= 1.f))
    return fail(NRN_E_INVALID, "%s: early-termination threshold %g outside [0, 1]", who, static_cast<double>(term->threshold));
  nrn::OccGrid g{};
  if (grid) {
    rc = occ_grid(grid, who, &g);
    if (rc) return rc;
  }
  if (P > nrn::kOccMaxPoints) return fail(NRN_E_INVALID, "%s: %lld points in one pass (at most 2^31 - 1)", who, P);
  if (P == 0) return NRN_OK;
  const bool bend = a->bender_packed != nullptr;
  if (!a->raw) return fail(NRN_E_INVALID, "%s: null raw", who);
  if (!term->termination_index) return fail(NRN_E_INVALID, "%s: null termination_index", who);
  const size_t need = nrn_termination_workspace_bytes(a->n_rays, a->n_samples, a->out_ch, bend);
  if (!workspace || (reinterpret_cast<uintptr_t>(workspace) & 255u) || workspace_bytes < need)
    return fail(NRN_E_INVALID, "%s: workspace null, not 256-byte aligned or smaller than nrn_termination_workspace_bytes (%zu)", who, need);
  DeviceState* ds;
  rc = device_state(&ds);
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(a->stream);
  const int S = a->n_samples, K = std::min(nrn::kTermSegment, S);
  const size_t p = static_cast<size_t>(P);
  const long long Pk = static_cast<long long>(a->n_rays) * K;
  const size_t pk = static_cast<size_t>(Pk);
  uint8_t* w = static_cast<uint8_t*>(workspace);
  float4* ws = nullptr;
  if (bend) { ws = reinterpret_cast<float4*>(w); w += align256(p * sizeof(float4)); }
  float* kept_xyz = reinterpret_cast<float*>(w); w += align256(pk * 3 * sizeof(float));
  int32_t* kept_idx = reinterpret_cast<int32_t*>(w); w += align256(pk * sizeof(int32_t));
  float* craw = reinterpret_cast<float*>(w); w += align256(pk * a->out_ch * sizeof(float));
  int32_t* count = reinterpret_cast<int32_t*>(w); w += align256(sizeof(int32_t));
  int32_t* block_counts = reinterpret_cast<int32_t*>(w); w += occ_block_count_bytes(Pk);
  float* T = reinterpret_cast<float*>(w);

  nrn::FieldFwdParams p0 = field_fwd_params(a, P, tiles, ds->err_word);
  // the bend pass over every sample: bent points and rigidities -> ws, and the details
  if (bend) {
    nrn::ViewParams vp{};
    vp.ws = ws;
    rc = timed(36, st, "field_bend_kernel", [&] { return nrn::launch_field_bend(p0, vp, ds->num_sms, st); });
    if (rc) return rc;
  }
  nrn::TermPass t{};
  t.raw = a->raw; t.z = a->z_vals; t.rays = a->rays; t.noise = term->noise;
  t.n = a->n_rays; t.S = S; t.out_ch = a->out_ch; t.threshold = term->threshold;
  t.T = T; t.term = term->termination_index;
  // raw is zeroed once: a sample no round evaluates keeps 0
  rc = timed(39, st, "termination_zero_raw", [&] { return cudaMemsetAsync(a->raw, 0, p * a->out_ch * sizeof(float), st); });
  if (rc) return rc;
  rc = timed(40, st, "term_init_kernel", [&] { return nrn::launch_termination_init(t, st); });
  if (rc) return rc;
  nrn::OccPoints s{};
  s.ws = ws; s.rays = a->rays; s.z_vals = a->z_vals; s.S = S; s.P = P;
  nrn::OccCompact c{};
  c.kept_xyz = kept_xyz; c.kept_idx = kept_idx; c.count = count; c.block_counts = block_counts;
  if (!bend) { c.d_init = a->initial_input_pts; c.d_bent = a->input_pts; }
  nrn::FieldFwdParams q{};
  q.pts = kept_xyz; q.pts_stride = 3; q.n_rays = static_cast<int>(Pk); q.S = 1; q.P = Pk; q.n_tiles = static_cast<int>(tile_count(Pk));
  q.nerf_w = p0.nerf_w; q.nerf_bias = p0.nerf_bias; q.out_ch = a->out_ch; q.raw = craw; q.err = ds->err_word;
  for (int s0 = 0; s0 < S; s0 += K) {
    const int len = std::min(K, S - s0);
    nrn::OccSegment seg{};
    seg.s0 = s0; seg.len = len; seg.P = static_cast<long long>(a->n_rays) * len; seg.term = term->termination_index;
    seg.use_grid = grid != nullptr;
    // 1. the lookup of this segment's samples: the ray alive (and the grid keeping the point), compacted in order
    rc = timed(37, st, "termination_compact", [&] { return nrn::launch_termination_compact(g, s, seg, c, st); });
    if (rc) return rc;
    // 2. the point-mode trunk on the kept points, their count read on the device
    rc = timed(38, st, "field_fwd_kept_kernel", [&] { return nrn::launch_field_fwd_kept(q, count, ds->num_sms, st); });
    if (rc) return rc;
    // 3. their raw into the pass's output (with the object removal)
    rc = timed(39, st, "occ_scatter_kernel", [&] {
      return nrn::launch_termination_scatter(craw, kept_idx, count, seg.P, a->out_ch, ws, a->use_removal, a->removal_threshold, a->raw,
                                             ds->num_sms, st);
    });
    if (rc) return rc;
    // 4. the transmittance over the segment; rays below the threshold die
    rc = timed(40, st, "term_transmittance_kernel", [&] { return nrn::launch_termination_transmittance(t, s0, len, st); });
    if (rc) return rc;
  }
  return NRN_OK;
}

// ---- the inverse of the ray bender ----
int nrn_deform_points(const NrnDeformArgs* a) {
  const char* who = "nrn_deform_points";
  if (!a) return fail(NRN_E_INVALID, "%s: null args", who);
  if (!a->points || !a->latents || !a->bender_packed || !a->out) return fail(NRN_E_INVALID, "%s: null argument", who);
  if (a->n_points < 0 || a->n_latents < 0)
    return fail(NRN_E_INVALID, "%s: negative sizes (n_points %lld, n_latents %d)", who, static_cast<long long>(a->n_points), a->n_latents);
  if (a->latent_stride < nrn::kLatent) return fail(NRN_E_INVALID, "%s: latent_stride %lld below %d", who, static_cast<long long>(a->latent_stride), nrn::kLatent);
  if (a->iterations < 1 || a->iterations > nrn::kDeformMaxIterations)
    return fail(NRN_E_INVALID, "%s: iterations %d outside 1..%d", who, a->iterations, nrn::kDeformMaxIterations);
  if (!(std::isfinite(a->tol) && a->tol >= 0.f)) return fail(NRN_E_INVALID, "%s: tol %g must be finite and >= 0", who, a->tol);
  if (a->use_scaling && !std::isfinite(a->scaling)) return fail(NRN_E_INVALID, "%s: scaling %g is not finite", who, a->scaling);
  if (a->use_cutoff && !std::isfinite(a->rigidity_cutoff))
    return fail(NRN_E_INVALID, "%s: rigidity_cutoff %g is not finite", who, a->rigidity_cutoff);
  if (!aligned4(a->points) || !aligned4(a->latents) || !aligned4(a->out) || !aligned4(a->residual) || !aligned4(a->rigidity))
    return fail(NRN_E_INVALID, "%s: float arrays must be 4-byte aligned", who);
  if (!aligned16(a->bender_packed)) return fail(NRN_E_INVALID, "%s: bender_packed must be 16-byte aligned", who);
  if (a->n_points == 0 || a->n_latents == 0) return NRN_OK;
  DeviceState* ds = nullptr;
  const int rc = device_state(&ds);
  if (rc) return rc;
  const cudaStream_t st = static_cast<cudaStream_t>(a->stream);
  nrn::DeformParams p{};
  p.points = a->points; p.P = a->n_points;
  p.latents = a->latents; p.latent_stride = a->latent_stride; p.F = a->n_latents;
  p.bender = static_cast<const uint8_t*>(a->bender_packed);
  p.use_cutoff = a->use_cutoff ? 1 : 0; p.cutoff = a->rigidity_cutoff;
  p.use_scaling = a->use_scaling ? 1 : 0; p.scaling = a->scaling;
  p.iterations = a->iterations; p.tol = a->tol;
  p.out = a->out; p.residual = a->residual; p.converged = a->converged; p.rigidity = a->rigidity;
  p.err = ds->err_word;
  return timed(41, st, "deform_kernel", [&] { return nrn::launch_deform(p, ds->num_sms, st); });
}

// ---- the density gradient ----
namespace {
// Points per launch pair: 512 tiles, about four waves of persistent CTAs on 132 SMs
constexpr long long kGradChunk = 1LL << 16;
// Workspace of one chunk of n points (256-byte aligned pieces): ReLU masks, E, unmasked offsets [n][3], rigidity [n], and
// the time-conditioned ray biases ([n][2][256] with latents per point, else one row)
struct GradWorkspace {
  size_t mask, e, unmasked, rigidity, ray_bias, total;
};
GradWorkspace grad_workspace(long long n_points, bool per_point_ray_bias) {
  const long long n = std::min(std::max(n_points, 0LL), kGradChunk);
  const long long tiles = (tile_count(n) + 1) & ~1LL;
  auto up = [](size_t b) { return (b + 255) / 256 * 256; };
  GradWorkspace w;
  w.mask = 0;
  w.e = w.mask + up(static_cast<size_t>(tiles) * nrn::kMaskTileBytes);
  w.unmasked = w.e + up(static_cast<size_t>(tiles) * nrn::kEBytes);
  w.rigidity = w.unmasked + up(static_cast<size_t>(n) * 3 * sizeof(float));
  w.ray_bias = w.rigidity + up(static_cast<size_t>(n) * sizeof(float));
  w.total = w.ray_bias + up(static_cast<size_t>(per_point_ray_bias ? n : 1) * 2 * 256 * sizeof(float));
  return w;
}
bool knob_ok(int use, float v) { return !use || std::isfinite(v); }
}  // namespace

int64_t nrn_density_gradient_chunk(void) { return kGradChunk; }

size_t nrn_density_gradient_workspace_bytes(int64_t n_points, int per_point_ray_bias) {
  return n_points < 0 ? 0 : grad_workspace(n_points, per_point_ray_bias != 0).total;
}

int nrn_field_density_gradient(const NrnDensityGradArgs* a) {
  const char* who = "nrn_field_density_gradient";
  if (!a) return fail(NRN_E_INVALID, "%s: null args", who);
  if (!a->points || !a->grad || !a->nerf_packed) return fail(NRN_E_INVALID, "%s: null argument (points, grad or nerf_packed)", who);
  if (a->n_points < 0) return fail(NRN_E_INVALID, "%s: n_points %lld < 0", who, static_cast<long long>(a->n_points));
  if (a->points_stride < 3) return fail(NRN_E_INVALID, "%s: points_stride %lld below 3", who, static_cast<long long>(a->points_stride));
  const int n_tc = (a->tc_w0 != nullptr) + (a->tc_b0 != nullptr) + (a->tc_w5 != nullptr) + (a->tc_b5 != nullptr);
  if (n_tc != 0 && n_tc != 4) return fail(NRN_E_INVALID, "%s: the time-conditioned baseline needs all of tc_w0, tc_b0, tc_w5, tc_b5", who);
  const bool tc = n_tc == 4, bender = a->bender_packed != nullptr;
  if (tc && bender) return fail(NRN_E_INVALID, "%s: the time-conditioned baseline has no bender (bender_packed must be NULL)", who);
  if ((tc || bender) != (a->latents != nullptr))
    return fail(NRN_E_INVALID, "%s: latents are needed exactly with a bender or the time-conditioned weights", who);
  if (a->latents && a->latent_stride != 0 && a->latent_stride < nrn::kLatent)
    return fail(NRN_E_INVALID, "%s: latent_stride %lld must be 0 or at least %d", who, static_cast<long long>(a->latent_stride), nrn::kLatent);
  if (!knob_ok(a->use_cutoff, a->rigidity_cutoff) || !knob_ok(a->use_scaling, a->scaling) || !knob_ok(a->use_removal, a->removal_threshold))
    return fail(NRN_E_INVALID, "%s: a test-time knob in use (rigidity_cutoff, scaling, removal_threshold) is not finite", who);
  if (!aligned4(a->points) || !aligned4(a->latents) || !aligned4(a->grad) || !aligned4(a->tc_w0) || !aligned4(a->tc_b0) ||
      !aligned4(a->tc_w5) || !aligned4(a->tc_b5))
    return fail(NRN_E_INVALID, "%s: float arrays must be 4-byte aligned", who);
  if (!aligned16(a->nerf_packed) || (bender && !aligned16(a->bender_packed)) || !aligned16(a->workspace))
    return fail(NRN_E_INVALID, "%s: packed weights and the workspace must be 16-byte aligned", who);
  const bool per_point_bias = tc && a->latent_stride != 0;
  const GradWorkspace w = grad_workspace(a->n_points, per_point_bias);
  if (a->n_points == 0) return NRN_OK;
  if (!a->workspace || a->workspace_bytes < w.total)
    return fail(NRN_E_INVALID, "%s: workspace of %zu bytes, %zu needed (nrn_density_gradient_workspace_bytes)", who, a->workspace_bytes, w.total);
  DeviceState* ds = nullptr;
  int rc = device_state(&ds);
  if (rc) return rc;
  const cudaStream_t st = static_cast<cudaStream_t>(a->stream);
  uint8_t* ws = static_cast<uint8_t*>(a->workspace);
  float* unmasked = reinterpret_cast<float*>(ws + w.unmasked);
  float* rigidity = reinterpret_cast<float*>(ws + w.rigidity);
  float* ray_bias = reinterpret_cast<float*>(ws + w.ray_bias);
  const uint8_t* np = static_cast<const uint8_t*>(a->nerf_packed);
  const uint8_t* bp = static_cast<const uint8_t*>(a->bender_packed);
  for (long long c0 = 0; c0 < a->n_points; c0 += kGradChunk) {
    const long long n = std::min(kGradChunk, static_cast<long long>(a->n_points) - c0);
    const int tiles = static_cast<int>(tile_count(n));
    nrn::FieldFwdParams p{};
    p.pts = a->points + c0 * a->points_stride; p.pts_stride = a->points_stride;
    if (a->latents) { p.latents = a->latents + c0 * a->latent_stride; p.latent_stride = a->latent_stride; }
    p.n_rays = static_cast<int>(n); p.S = 1; p.P = n; p.n_tiles = tiles;
    p.nerf_w = np; p.nerf_bias = reinterpret_cast<const float*>(np + nrn::kNerfWBytes);
    if (bender) { p.bend_w = bp; p.bend_bias = reinterpret_cast<const float*>(bp + nrn::kBendWBytes); }
    p.cutoff = a->rigidity_cutoff; p.use_cutoff = a->use_cutoff;
    p.scaling = a->scaling; p.use_scaling = a->use_scaling;
    p.out_ch = 4;
    if (bender) { p.d_unmasked = unmasked; p.d_rigid = rigidity; }
    p.stash = ws + w.e; p.relu_mask = ws + w.mask;
    p.err = ds->err_word;
    if (tc) { p.ray_bias = ray_bias; p.ray_bias_stride = per_point_bias ? 2 * 256 : 0; }
    rc = timed(42, st, "field_fwd_grad_kernel", [&] {
      if (tc) {
        const cudaError_t e = nrn::launch_tc_latent_bias(p.latents, a->latent_stride, per_point_bias ? p.n_rays : 1, a->tc_w0, a->tc_b0,
                                                         a->tc_w5, a->tc_b5, ray_bias, st);
        if (e != cudaSuccess) return e;
      }
      return nrn::launch_field_fwd_grad(p, bender, ds->num_sms, st);
    });
    if (rc) return rc;
    nrn::FieldBwdParams q{};
    q.P = n; q.n_tiles = tiles; q.S = 1; q.n_rays = static_cast<int>(n); q.out_ch = 4;
    q.stash = ws + w.e; q.relu_mask = ws + w.mask;
    q.nerf_wT = np + nrn::kNerfTOffset;
    if (bender) { q.bend_wT = bp + nrn::kBendTOffset; q.unmasked = unmasked; q.rigidity = rigidity; }
    q.cutoff = a->rigidity_cutoff; q.use_cutoff = a->use_cutoff; q.scaling = a->scaling; q.use_scaling = a->use_scaling;
    q.err = ds->err_word;
    nrn::PointGradParams pg{};
    pg.grad = a->grad + c0 * 3; pg.removal = a->removal_threshold; pg.use_removal = bender && a->use_removal;
    rc = timed(43, st, "field_bwd_grad_kernel", [&] { return nrn::launch_field_bwd_grad(q, pg, bender, ds->num_sms, st); });
    if (rc) return rc;
  }
  return NRN_OK;
}

// Turning timing off only stops recording: a CUDA graph captured while it was on keeps event-record nodes that refer to
// these events and may still be replayed.  They are released when a new timing session starts.
int nrn_timing_enable(int on) {
  if (on) {
    for (int i = 0; i < g_timed_n; ++i) { cudaEventDestroy(g_timed[i].a); cudaEventDestroy(g_timed[i].b); }
    g_timed_n = 0;
  }
  g_timing = on != 0;
  return NRN_OK;
}

int nrn_timing_read(double* ms_sum, int* counts, int n_kinds) {
  if (!ms_sum || !counts || n_kinds < 1) return fail(NRN_E_INVALID, "nrn_timing_read: bad arguments");
  for (int k = 0; k < n_kinds; ++k) { ms_sum[k] = 0.0; counts[k] = 0; }
  for (int i = 0; i < g_timed_n; ++i) {
    cudaError_t e = cudaEventSynchronize(g_timed[i].b);
    if (e != cudaSuccess) return cuda_fail(e, "cudaEventSynchronize");
    float ms = 0.f;
    e = cudaEventElapsedTime(&ms, g_timed[i].a, g_timed[i].b);
    if (e != cudaSuccess) return cuda_fail(e, "cudaEventElapsedTime");
    if (g_timed[i].kind < n_kinds) { ms_sum[g_timed[i].kind] += ms; counts[g_timed[i].kind] += 1; }
  }
  return NRN_OK;
}

}  // extern "C"
