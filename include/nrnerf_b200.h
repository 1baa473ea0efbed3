/* nrnerf_b200 -- C ABI of the H100-native (sm_90a) NR-NeRF render hot path (libnrnerf_b200.so).
 *
 * Plain C: raw device pointers, sizes, a cudaStream_t passed as void*.  No torch types, no C++
 * types, no exceptions.  Every function returns 0 on success or a negative NRN_E_* code; the
 * message is available from nrn_last_error() (thread-local).  All work is enqueued on the given
 * stream; nothing synchronises except nrn_device_error().
 *
 * The reference (facebookresearch/nonrigid_nerf) has no FFI layer: its boundary for this path is a
 * set of Python callables.  Each entry point below names the reference function(s) it replaces
 * (paths relative to the reference checkout); INTEGRATION.md shows the ctypes binding.
 */
#ifndef NRNERF_B200_H
#define NRNERF_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NRN_ABI_VERSION 4

#define NRN_OK 0
#define NRN_E_INVALID (-1)   /* bad argument / unsupported configuration */
#define NRN_E_CUDA (-2)      /* CUDA runtime error (see nrn_last_error) */
#define NRN_E_DEVICE (-3)    /* device-side protocol error recorded by a kernel */

int nrn_abi_version(void);
const char* nrn_last_error(void);

/* Synchronises the current device, reads and clears the device-side error word written by the
 * fused kernels (0 = ok; non-zero = id of the mbarrier wait that timed out). */
int nrn_device_error(int* code_out);

/* ---- weight packing -------------------------------------------------------------------------
 * fp32 nn.Linear tensors in the reference's checkpoint layout ([out][in] row-major) -> fp16 wgmma
 * operand images.  Replaces nothing in the reference (derived data); sources are
 * NeRF.pts_linears / output_linear (run_nerf_helpers.py:218-238) and ray_bending.network /
 * rigidity_network (run_nerf_helpers.py:411-482). */
size_t nrn_packed_nerf_bytes(void);
size_t nrn_packed_bender_bytes(void);
/* w[0..7] = pts_linears.i.weight, w[8] = output_linear.weight; b likewise. input_ch = 63 (95: time-conditioned baseline). */
int nrn_pack_nerf(const float* const* w, const float* const* b, int input_ch, int out_ch, void* packed,
                  void* stream);
int nrn_pack_bender(const float* const* net_w /*5*/, const float* const* net_b /*4*/,
                    const float* const* rig_w /*3*/, const float* const* rig_b /*3*/, int latent_size,
                    void* packed, void* stream);

/* ---- ray generation: get_rays / get_rays_np (run_nerf_helpers.py:588-622) on the device -----------------------------
 * c2w [3][4] row-major, intrinsics = (focal_x, focal_y, center_x, center_y); rays_o / rays_d [H*W][3] in the [H, W, 3]
 * order of the reference.  Bit-identical to the reference's float32 arithmetic. */
int nrn_get_rays(const float* c2w, const float* intrinsics, int height, int width, float* rays_o, float* rays_d, void* stream);
/* rays [n][8] = (o, d, near, far) as render() assembles them before batchify_rays (train.py:388-398), scalar near / far. */
int nrn_pack_rays(const float* rays_o, const float* rays_d, float near, float far, int n_rays, float* rays, void* stream);
/* A training batch computed on demand instead of gathered from the host table of every ray of every image
 * (train.py:1498-1517, :1546-1564): pix [n][3] int64 = (image, x, y) as in batch_pixel_indices; poses [n_images][3][4];
 * intrinsics [n_views][4]; image_to_view [n_images] int32 or NULL (single view); images [n_images][H][W][3] fp32 or NULL
 * (then target may be NULL). */
int nrn_ray_batch(const int64_t* pix, int n, const float* poses, const float* intrinsics, const int32_t* image_to_view,
                  const float* images, int height, int width, float* rays_o, float* rays_d, float* target, void* stream);
/* ---- free-viewpoint post-processing, free_viewpoint_rendering.py:623-629: per ray the index of the sample whose
 * accumulated visibility weight is closest to 0.5 (first minimum).  weights [n][n_samples] -> index [n] int64. */
int nrn_median_visibility_index(const float* weights, int n_rays, int n_samples, int64_t* index, void* stream);

/* ---- coarse depth sampling: render_rays, train.py:847-869 ------------------------------------
 * rays [n][8] = (o, d, near, far); t_rand [n][S] uniform randoms or NULL (perturb == 0). */
int nrn_sample_coarse(const float* rays, const float* t_rand, int n_rays, int n_samples, int lindisp,
                      float* z_vals, void* stream);

/* ---- fused field evaluation: run_network (train.py:57-105) + NeRF.forward
 * (run_nerf_helpers.py:240-314) + ray_bending.forward (:507-584) + Embedder.embed (:149-150) --- */
typedef struct NrnFieldArgs {
  const float* rays;          /* [n_rays][8] (o, d, near, far) */
  const float* z_vals;        /* [n_rays][n_samples] */
  const float* points;        /* point mode (NeRF.forward(x), run_nerf_helpers.py:240): rays = z_vals = NULL,
                                 n_samples = 1, n_rays = number of points; xyz = points[i*points_stride + 0..2] */
  int64_t points_stride;
  const float* latents;       /* [n_rays][32], NULL when bender_packed is NULL */
  int64_t latent_stride;      /* floats between consecutive rays' latents (0 = broadcast one row) */
  int32_t n_rays;
  int32_t n_samples;
  const void* nerf_packed;    /* nrn_pack_nerf output */
  const void* bender_packed;  /* nrn_pack_bender output or NULL (canonical rendering, ray_bender=(None,)) */
  int32_t out_ch;             /* 4 or 5 (output_linear rows) */
  int32_t use_cutoff;  float rigidity_cutoff;   /* ray_bending.rigidity_test_time_cutoff */
  int32_t use_scaling; float scaling;           /* ray_bending.test_time_scaling */
  int32_t use_removal; float removal_threshold; /* NeRF.test_time_nonrigid_object_removal_threshold */
  float* raw;                 /* out [n_rays][n_samples][out_ch] */
  float* initial_input_pts;   /* out [P][3] or NULL  (details of detailed_output=True) */
  float* input_pts;           /* out [P][3] or NULL */
  float* unmasked_offsets;    /* out [P][3] or NULL */
  float* masked_offsets;      /* out [P][3] or NULL */
  float* rigidity_mask;       /* out [P]    or NULL */
  void* stash;                /* training only: activation stash of nrn_stash_bytes() bytes, else NULL */
  void* stream;
  void* relu_mask;            /* training only (given with stash, else NULL): ReLU masks for the backward pass,
                                 nrn_relu_mask_bytes() bytes */
} NrnFieldArgs;
int nrn_field_forward(const NrnFieldArgs* args);

/* ---- compositing: raw2outputs (train.py:724-789), optionally fused with sample_pdf
 * (run_nerf_helpers.py:651-698), the sort of train.py:920 and z_std of train.py:959 ------------ */
typedef struct NrnCompositeArgs {
  const float* raw;           /* [n][S][C] */
  const float* z_vals;        /* [n][S] */
  const float* rays_d;        /* ray directions, row stride rays_d_stride floats */
  int32_t rays_d_stride;
  const float* noise;         /* [n][S] sigma noise already multiplied by raw_noise_std, or NULL */
  int32_t n_rays, n_samples, channels, white_bkgd;
  float* rgb_map;             /* out [n][3] */
  float* disp_map;            /* out [n] */
  float* acc_map;             /* out [n] */
  float* depth_map;           /* out [n] or NULL */
  float* weights;             /* out [n][S] or NULL */
  float* alpha;               /* out [n][S] or NULL */
  int32_t n_importance;       /* 0 = composite only */
  const float* u;             /* [n][n_importance] or NULL (deterministic linspace, perturb == 0) */
  float* z_vals_out;          /* out [n][S + n_importance] sorted union */
  float* z_std;               /* out [n] or NULL */
  void* stream;
} NrnCompositeArgs;
int nrn_composite(const NrnCompositeArgs* args);

/* stand-alone sample_pdf (run_nerf_helpers.py:651-698): bins [n][nbins], weights [n][nbins-1] */
int nrn_sample_pdf(const float* bins, const float* weights, const float* u, int n, int nbins, int n_samples,
                   float* samples, void* stream);

/* ---- backward of raw2outputs w.r.t. raw (what torch.autograd derives for train.py:724-789) ---- */
typedef struct NrnCompositeBwdArgs {
  const float* raw; const float* z_vals; const float* rays_d; int32_t rays_d_stride; const float* noise;
  int32_t n_rays, n_samples, channels, white_bkgd;
  const float* d_rgb_map;     /* [n][3] */
  const float* d_acc_map;     /* [n] or NULL */
  float* d_raw;               /* out [n][S][C] */
  void* stream;
} NrnCompositeBwdArgs;
int nrn_composite_backward(const NrnCompositeBwdArgs* args);

/* ---- backward of the fused field (what torch.autograd derives for NeRF.forward +
 * ray_bending.forward, run_nerf_helpers.py:240-314 / :507-584; SURVEY.md appendix C):
 * DGRAD chain + WGRAD + deterministic split reduction.  Needs the stash written by
 * nrn_field_forward (ray mode) and, with a bender, that call's unmasked_offsets / rigidity_mask. */
size_t nrn_stash_bytes(int n_rays, int n_samples);
size_t nrn_grad_stash_bytes(int n_rays, int n_samples);
size_t nrn_relu_mask_bytes(int n_rays, int n_samples);   /* 1 bit per hidden activation: 40 KB per 128-point tile */
size_t nrn_wgrad_scratch_bytes(void);
int nrn_nerf_grad_floats(int out_ch);   /* flat order: W0 b0 W1 b1 ... W7 b7 Wout bout (reference shapes) */
int nrn_bender_grad_floats(void);       /* flat order: network.0.w .0.b .1.w .1.b .2.w .2.b .3.w .3.b .4.w,
                                           rigidity_network.0.w .0.b .1.w .1.b .2.w .2.b */
typedef struct NrnFieldBwdArgs {
  int32_t n_rays, n_samples, out_ch;
  const float* d_raw;             /* [n_rays][n_samples][out_ch] upstream gradient */
  const void* stash;              /* from the forward call */
  void* grad_stash;               /* workspace, nrn_grad_stash_bytes() */
  float* wgrad_scratch;           /* workspace, nrn_wgrad_scratch_bytes() */
  const void* nerf_packed;
  const void* bender_packed;      /* or NULL */
  const float* unmasked_offsets;  /* [P][3] forward output (bender only) */
  const float* rigidity_mask;     /* [P]    forward output (bender only) */
  const float* d_unmasked_offsets;/* [P][3] upstream gradient (offsets regulariser) or NULL */
  const float* d_rigidity_mask;   /* [P]    upstream gradient (rigidity regulariser) or NULL */
  int32_t use_cutoff;  float rigidity_cutoff;
  int32_t use_scaling; float scaling;
  float* nerf_grad;               /* out, nrn_nerf_grad_floats(out_ch) floats, overwritten */
  float* bender_grad;             /* out, nrn_bender_grad_floats() floats, overwritten (or NULL) */
  float* d_latents;               /* out [n_rays][32], overwritten (or NULL without bender) */
  void* stream;
  /* Gradients written where PyTorch keeps them (SURVEY.md 8b "gradient buffers that alias param.grad"):
   * nerf_grad_head, if not NULL, receives the output_linear part (Wout bout) instead of the tail of nerf_grad -- in
   * module.parameters() order the dead views_linears sit between pts_linears and output_linear; accumulate_* != 0
   * adds to the destination instead of overwriting it (what autograd's AccumulateGrad would do). */
  float* nerf_grad_head;
  int32_t accumulate_nerf, accumulate_bender;
  const void* relu_mask;          /* from the forward call (nrn_relu_mask_bytes()) */
} NrnFieldBwdArgs;
int nrn_field_backward(const NrnFieldBwdArgs* args);

/* ---- time-conditioned baseline (NeRF(time_conditioned_baseline=True), run_nerf_helpers.py:206-209, 273-282; no bender,
 * train.py:574-578): the per-ray latent z is concatenated to the embedding at L0 ([PE(63) | z(32)], W0 [256][95]) and at
 * the skip layer L5 ([PE | z | h], W5 [256][351]).  z is the same for every sample of a ray, so W_l[:, 63:95] . z + b_l is
 * one fp32 bias row per ray and layer ("ray bias" [n][2][256], L0 then L5) and the fused kernels run the geometry of
 * the 63-input NeRF.  nrn_pack_nerf with input_ch = 95 packs such weights (the latent columns are skipped). */
/* ray_bias[n][l][o] = b_l[o] + sum_k W_l[o][63 + k] latents[n * latent_stride + k]  (fp32; w0 [256][95], w5 [256][351]) */
int nrn_tc_latent_bias(const float* latents, int64_t latent_stride, int n_rays, const float* w0, const float* b0, const float* w5,
                       const float* b5, float* ray_bias, void* stream);
/* nrn_field_forward with the L0 / L5 biases taken from ray_bias: one row per ray (row stride 512 floats), or, when
 * args->latent_stride == 0, one row for every ray.  args->bender_packed must be NULL; args->latents is not read. */
int nrn_field_forward_tc(const NrnFieldArgs* args, const float* ray_bias);
int nrn_nerf_tc_grad_floats(int out_ch);   /* flat order as nrn_nerf_grad_floats, with W0 [256][95] and W5 [256][351] */

/* ---- view-dependent head, inference only: NeRF(use_viewdirs=True, approx_nonrigid_viewdirs=True)
 * (run_nerf_helpers.py:233-236, 284-304, 316-356; train.py:364-399).  raw = [rgb_linear(relu(views_linears.0(
 * cat[feature_linear(h8), dir_enc]))), alpha_linear(h8)], dir_enc = [d, sin(2^k d), cos(2^k d)], k = 0..3 (27 columns).
 * With a bender d is the normalised backward difference of the BENT points of the ray, (p_i - p_{i-1}) / (|.| + 1e-6),
 * and d_0 = d_1; without one it is the given viewdirs row.  The trunk is packed by nrn_pack_nerf with out_ch = 4 and a
 * head of zeros in rows 0-2 and alpha_linear in row 3; feature_linear, views_linears.0 and rgb_linear by nrn_pack_views. */
size_t nrn_packed_views_bytes(void);
/* w / b [0] = feature_linear [256][256], [1] = views_linears.0 [128][256 + 27], [2] = rgb_linear [3][128] */
int nrn_pack_views(const float* const* w, const float* const* b, void* packed, void* stream);
size_t nrn_views_workspace_bytes(int n_rays, int n_samples);   /* bend workspace: 16 bytes per point */
typedef struct NrnViewArgs {
  const void* views_packed;   /* nrn_pack_views output (16-byte aligned); may be NULL when args->raw is NULL */
  const float* viewdirs;      /* no bender: normalised view directions, one row per ray (ray mode) or per point (point
                                 mode); not read with a bender */
  int64_t viewdirs_stride;    /* floats between rows, >= 3 */
  void* workspace;            /* with a bender: nrn_views_workspace_bytes(n_rays, n_samples), 16-byte aligned */
} NrnViewArgs;
/* args as for nrn_field_forward, with out_ch = 4 and no stash / relu_mask (training: nrn_field_forward_views_train).  With a bender
 * n_samples >= 2: the finite differences run over each ray's n_samples consecutive points.  Point mode takes
 * n_rays * n_samples points, n_samples consecutive ones forming a ray; latents (and viewdirs) are read per point.  With a
 * bender, raw = NULL runs the bend pass alone (the details: bent points, offsets, rigidity). */
int nrn_field_forward_views(const NrnFieldArgs* args, const NrnViewArgs* views);
/* ---- training the view-dependent head without a ray bender (rigid scenes; NeRF(use_viewdirs=True), ray_bender None):
 * the view direction is the ray's own normalised direction, so the gradient stops at views_linears.0's direction
 * columns.  The forward keeps, next to the trunk's stash and ReLU masks, a view stash (direction encoding, feature,
 * post-ReLU views_linears.0 output) and the ReLU mask bits of that output; the backward runs the head's transposed
 * steps in front of the trunk's DGRAD and the head's weight gradients in the same WGRAD launch.  Buffers are per
 * 128-point tile, rounded up to an even tile count like nrn_stash_bytes. */
size_t nrn_packed_views_t_bytes(void);   /* transposed head images: rgb_linear^T | views_linears.0[:, :256]^T | feature_linear^T */
/* w[0] = feature_linear.weight [256][256], w[1] = views_linears.0.weight [128][256 + 27], w[2] = rgb_linear.weight [3][128] */
int nrn_pack_views_t(const float* const* w, void* packed, void* stream);
size_t nrn_views_stash_bytes(int n_rays, int n_samples);        /* 104 KB per tile */
size_t nrn_views_grad_stash_bytes(int n_rays, int n_samples);   /* 96 KB per tile */
size_t nrn_hv_mask_bytes(int n_rays, int n_samples);            /* 2 KB per tile */
/* flat order of the view model's parameters: W0 b0 ... W7 b7 (as nrn_nerf_grad_floats), then views_linears.0.w [128][283]
 * .b, feature_linear.w [256][256] .b, alpha_linear.w [1][256] .b, rgb_linear.w [3][128] .b: 595,844 floats */
int nrn_nerf_views_grad_floats(void);
typedef struct NrnViewTrainArgs {
  void* views_stash;          /* nrn_views_stash_bytes(), 16-byte aligned */
  void* hv_mask;              /* nrn_hv_mask_bytes(), 16-byte aligned */
} NrnViewTrainArgs;
/* The forward of nrn_field_forward_views without a bender, keeping what the backward needs: args in ray mode with
 * out_ch = 4, bender_packed NULL, use_removal 0, stash and relu_mask given (nrn_stash_bytes / nrn_relu_mask_bytes);
 * views->views_packed and views->viewdirs given.  raw equals nrn_field_forward_views' bit for bit. */
int nrn_field_forward_views_train(const NrnFieldArgs* args, const NrnViewArgs* views, const NrnViewTrainArgs* train);
typedef struct NrnViewBwdArgs {
  const void* views_t_packed;   /* nrn_pack_views_t output */
  const void* views_stash;      /* from the forward call */
  void* views_grad_stash;       /* workspace, nrn_views_grad_stash_bytes() */
  const void* hv_mask;          /* from the forward call */
} NrnViewBwdArgs;
/* Backward of nrn_field_forward_views_train: args as for nrn_field_backward with out_ch = 4, bender_packed NULL and
 * nerf_packed the nrn_pack_nerf image the forward ran with (its head^T holds alpha_linear in column 3).  nerf_grad receives
 * the flat layout of nrn_nerf_views_grad_floats(); nerf_grad_head, if not NULL, receives the head block (views_linears.0
 * .. rgb_linear.b) instead of the tail of nerf_grad.  Deterministic: every sum runs in a fixed order. */
int nrn_field_backward_views(const NrnFieldBwdArgs* args, const NrnViewBwdArgs* views);
size_t nrn_tc_workspace_bytes(int n_rays);   /* per-ray sums [n][2][256] + latent columns of dW0 / dW5 [2][256][32] */
typedef struct NrnTcBwdArgs {
  const float* latents;           /* [n_rays][32] the forward call's latents ... */
  int64_t latent_stride;          /* ... row stride in floats (0 = one row for every ray) */
  const float* w0;                /* fp32 pts_linears.0.weight [256][95] */
  const float* w5;                /* fp32 pts_linears.5.weight [256][351] */
  float* d_latents;               /* out [n_rays][32], overwritten */
  float* workspace;               /* nrn_tc_workspace_bytes(n_rays) */
} NrnTcBwdArgs;
/* nrn_field_backward of a nrn_field_forward_tc call (args->bender_packed NULL): nerf_grad (and nerf_grad_head) in the
 * time-conditioned flat layout of nrn_nerf_tc_grad_floats, the latent columns of W0 / W5 included, and d_latents.
 * Deterministic: every sum runs in a fixed order. */
int nrn_field_backward_tc(const NrnFieldBwdArgs* args, const NrnTcBwdArgs* tc);

/* ---- divergence regulariser of the offset field on the coarse samples: compute_divergence_loss /
 * divergence_approx (run_nerf_helpers.py:22-116) as driven by train.py:245-286, forward and backward
 * in closed form (no double backward), on tensor cores with the fp16 bender weights the coarse pass ran with.
 * Needs that pass's ReLU masks (relu_mask of the training nrn_field_forward call) and its packed bender. ------ */
size_t nrn_div_stash_bytes(int n_rays, int n_samples);
size_t nrn_div_grad_stash_bytes(int n_rays, int n_samples);
typedef struct NrnDivArgs {
  int32_t n_rays, n_samples;
  const void* relu_mask;           /* ReLU masks written by the coarse nrn_field_forward call (nrn_relu_mask_bytes()) */
  const float* e;                  /* [P][3] probe vectors ~ N(0, I) (torch.randn_like, run_nerf_helpers.py:110) */
  const float* unmasked_offsets;   /* [P][3] coarse pass output */
  const float* rigidity_mask;      /* [P]    coarse pass output */
  const float* weights;            /* [P]    1 - exp(-relu(opacity_alpha)), detached (train.py:267) ... */
  int32_t weights_are_opacity_alpha; /* ... or, if 1, opacity_alpha itself: the kernels apply 1 - exp(-relu(.)) */
  const void* bender_packed;       /* nrn_pack_bender output the coarse pass ran with (16-byte aligned) */
  void* tangent_stash;             /* nrn_div_stash_bytes(): written by forward, read by backward */
  float* d; float* alpha; float* beta; float* tau_c;   /* [P] each: written by forward, read by backward */
  float* loss;                     /* forward out [n_rays]: mean over the ray's samples of weights * d^2 */
  /* backward only */
  const float* G;                  /* [P] dL/dd = g_ray * 2 * weights * d / n_samples, or NULL with g_ray / G_workspace: */
  const float* g_ray;              /* [n_rays] upstream gradient of `loss`; G is then computed into G_workspace [P] */
  float* G_workspace;
  void* adjoint_stash;             /* workspace, nrn_div_grad_stash_bytes() */
  float* wgrad_scratch;            /* workspace, nrn_wgrad_scratch_bytes() */
  float* d_unmasked_offsets;       /* out [P][3] gradient w.r.t. the coarse unmasked offsets */
  float* d_rigidity_mask;          /* out [P]    gradient w.r.t. the coarse rigidity mask */
  float* bender_grad;              /* out, nrn_bender_grad_floats(): weight gradients of the tangent chain */
  void* stream;
  int32_t accumulate_bender;       /* != 0: add to bender_grad instead of overwriting it */
} NrnDivArgs;
int nrn_divergence_forward(const NrnDivArgs* args);
int nrn_divergence_backward(const NrnDivArgs* args);

/* ---- deterministic mode (what torch.use_deterministic_algorithms(True) selects): the per-ray sums that the entry points
 * above form with fp32 atomics -- the latent gradient of nrn_field_backward with a bender, the loss of
 * nrn_divergence_forward -- run in a fixed order instead, so that a training step is bit-reproducible on one GPU model.
 * The kernels write per-point rows to a caller-owned workspace, then one small kernel sums each ray's rows in increasing
 * point order: points form 32-aligned blocks [32k, 32k + 32); a block whose points all exist (32k + 31 < P) and lie in one
 * ray holds its in-warp sum in the row of point 32k and is skipped as a whole, every other point holds its own row.
 * Only the rows that order reaches are written, so the workspace needs no initialisation. ------------------------------ */
size_t nrn_latent_rows_bytes(int n_rays, int n_samples);     /* [n_rays * n_samples][32] fp32 */
size_t nrn_div_loss_rows_bytes(int n_rays, int n_samples);   /* [n_rays * n_samples] fp32 */
/* nrn_field_backward with a bender (bender_packed and d_latents given); latent_rows: nrn_latent_rows_bytes(), 16-byte
 * aligned.  d_latents is overwritten with the fixed-order sums; every other output is as nrn_field_backward's.  An
 * empty batch (n_rays = 0) launches no kernel and, like nrn_field_backward, zeroes the gradients it does not accumulate. */
int nrn_field_backward_det(const NrnFieldBwdArgs* args, float* latent_rows);
/* nrn_divergence_forward with loss written in a fixed order; loss_rows: nrn_div_loss_rows_bytes() */
int nrn_divergence_forward_det(const NrnDivArgs* args, float* loss_rows);

/* ---- held-out rays: the reference trains the latent codes of held-out frames (test_block_size, train.py:1376-1395) with a
 * second backward pass whose network gradients it discards (train.py:1595-1608).  These entry points give one backward
 * both: held_out_rays [n_rays] (device, one byte per ray, nonzero = held out) marks rays whose gradient reaches their
 * latent code only.  Every kernel step runs as without it; the gradient-stash rows (adjoint-stash rows for the divergence
 * regulariser) of a held-out ray's points are written as zeros, so the weight gradients leave them out.  With
 * held_out_rays all zero the results equal those of the entry points without the suffix bit for bit.  Without a bender a
 * held-out ray contributes nothing at all: zero its rows of d_raw and call nrn_field_backward (or _tc / _views). ------- */
/* nrn_field_backward with a bender (bender_packed and d_latents given): d_latents as nrn_field_backward forms it for
 * every ray; nerf_grad and bender_grad without the held-out rays' share (the data terms and the offsets / rigidity
 * upstream gradients alike) */
int nrn_field_backward_held_out(const NrnFieldBwdArgs* args, const uint8_t* held_out_rays);
/* the same in deterministic mode: d_latents as nrn_field_backward_det forms it */
int nrn_field_backward_det_held_out(const NrnFieldBwdArgs* args, float* latent_rows, const uint8_t* held_out_rays);
/* nrn_divergence_backward with bender_grad without the held-out rays' share; d_unmasked_offsets and d_rigidity_mask, which
 * carry their latent gradient into nrn_field_backward_held_out, as nrn_divergence_backward writes them */
int nrn_divergence_backward_held_out(const NrnDivArgs* args, const uint8_t* held_out_rays);

/* ---- per-ray training loss of training_wrapper_class.forward (train.py:208-242): image terms (fine +
 * coarse) and the offsets / rigidity regulariser on the coarse samples, with the gradients per unit
 * upstream gradient written in the same pass (the loss is linear in dL/dloss[ray]). ----------------- */
typedef struct NrnRayLossArgs {
  int32_t n_rays, n_samples;
  const float* rgb;                /* [n][3] rgb_map */
  const float* rgb0;               /* [n][3] coarse rgb_map or NULL */
  const float* target;             /* [n][3] */
  const float* weights;            /* [n][S] coarse visibility weights (detached) or NULL */
  const float* unmasked_offsets;   /* [n][S][3] or NULL: no offsets term */
  const float* rigidity_mask;      /* [n][S] */
  float lam_offsets;               /* offsets_loss_weight (times the schedule, unless sched_step is given) */
  float lam_rigidity;              /* rigidity_loss_weight */
  float* loss;                     /* out [n] */
  float* u_rgb; float* u_rgb0;     /* out [n][3]: d loss / d rgb, d loss / d rgb0 */
  float* u_unmasked_offsets;       /* out [n][S][3] */
  float* u_rigidity_mask;          /* out [n][S] */
  void* stream;
  /* Regulariser schedule (1/100)^(1 - global_step / N_iters) of train.py:229 / :281 evaluated on the device: sched_step is a
   * device scalar holding global_step (NULL: the caller folded the schedule into the weights), so that a captured CUDA graph
   * follows the schedule.  divergence [n] (or NULL) is the per-ray divergence regulariser (nrn_divergence_forward), added as
   * lam_divergence * schedule * divergence; u_divergence [n] receives d loss / d divergence. */
  const float* sched_step;
  float sched_n_iters;
  const float* divergence;
  float lam_divergence;
  float* u_divergence;
} NrnRayLossArgs;
int nrn_ray_loss(const NrnRayLossArgs* args);
/* out[i] = g[i / per_row] * unit[i] */
int nrn_scale_rows(const float* g, const float* unit, float* out, int64_t n, int per_row, void* stream);
/* Backward of nrn_ray_loss in ONE launch: every out_k[i] = g[ray of i] * unit_k[i] for the (up to five) unit-gradient arrays
 * nrn_ray_loss wrote (NULL pairs are skipped): rgb [n][3], rgb0 [n][3], unmasked_offsets [n][S][3], rigidity_mask [n][S],
 * divergence [n]. */
typedef struct NrnRayLossBwdArgs {
  int32_t n_rays, n_samples;
  const float* g;                  /* [n] upstream gradient of the per-ray loss */
  const float* u_rgb; const float* u_rgb0; const float* u_unmasked_offsets; const float* u_rigidity_mask; const float* u_divergence;
  float* d_rgb; float* d_rgb0; float* d_unmasked_offsets; float* d_rigidity_mask; float* d_divergence;
  void* stream;
} NrnRayLossBwdArgs;
int nrn_ray_loss_backward(const NrnRayLossBwdArgs* args);

/* ---- optimizer step: replaces torch.optim.Adam(params=grad_vars, lr, betas=(0.9, 0.999)) of train.py:656-658 and its
 * optimizer.step() at train.py:1608.  All trainable tensors live in one flat fp32 buffer (the host side makes the
 * nn.Parameters views into it); `blocks` (device, int32 x 4 per entry: tensor index, first element inside the tensor,
 * element count <= 2048, offset inside the flat buffers) maps CUDA blocks to tensors; `grad_ptrs` (device, one
 * const float* per tensor, NULL = parameter without gradient, skipped like torch does) is where autograd left each
 * gradient.  lr (scalar) and step (one int64 per tensor, as torch counts steps per parameter) live on the device
 * (CUDA-graph replay); the call increments the step of every tensor that has a gradient, then applies
 * m += (g-m)(1-b1); v = b2 v + (1-b2) g^2; p -= lr/(1-b1^t) m / (sqrt(v)/sqrt(1-b2^t) + eps). */
typedef struct NrnAdamArgs {
  void* params;            /* float [total] */
  void* exp_avg;           /* float [total] */
  void* exp_avg_sq;        /* float [total] */
  const void* grad_ptrs;   /* device array of n_tensors pointers */
  const void* blocks;      /* device array of n_blocks x 4 int32 */
  int n_tensors, n_blocks;
  const void* lr;          /* device float */
  void* step;              /* device int64 [n_tensors] */
  float beta1, beta2, eps;
  void* stream;
} NrnAdamArgs;
int nrn_adam_step(const NrnAdamArgs* args);

/* ---- multi-GPU: gradient all-reduce fused into the optimizer step over NVLink peer memory.  Replaces the gradient
 * reduction torch.nn.DataParallel performs on GPU 0 (train.py:290-297; backward of the scatter at :1566-1577) plus the
 * optimizer.step() at :1608, for one process per GPU on one node.  Every rank allocates a window
 *   [ 1024 B flags | 2 x slot_floats floats (double-buffered row slots) | arena_floats floats (gradient arena) ]
 * with nrn_peer_alloc, publishes its 64-byte CUDA IPC handle to the other ranks (any side channel: the host side uses
 * torch.distributed.all_gather_object), maps theirs with nrn_peer_open, and points every parameter's .grad into its own
 * window's arena.  nrn_peer_reduce_adam then sums the ranks' arenas in rank order while reading them over NVLink and applies
 * Adam (same arithmetic as nrn_adam_step; grad_ptrs is ignored, gradients come from the arenas at the blocks' flat
 * offsets); afterwards the arena holds the reduced gradient.  nrn_peer_gather_rows all-gathers n_per_rank floats per rank
 * (the per-ray losses the caller logs) through the slots.  All launches are plain kernels on `stream` (CUDA-graph
 * capturable); a peer that never arrives becomes device error 901/902/903 (nrn_device_error), not a hang. */
size_t nrn_peer_window_bytes(int64_t arena_floats, int64_t slot_floats);
int nrn_peer_alloc(size_t bytes, void** dev_ptr, void* ipc_handle_64bytes);
int nrn_peer_open(const void* ipc_handle_64bytes, void** dev_ptr);
int nrn_peer_close(void* dev_ptr);
int nrn_peer_free(void* dev_ptr);
typedef struct NrnPeerCtx {
  void* window[8];          /* all ranks' windows as mapped into this process; window[rank] = own allocation */
  int32_t world, rank;
  int64_t arena_floats, slot_floats;
  void* state;              /* device, 16 bytes, zero-initialised once: 3 epoch counters + block counter */
  float* reduced;           /* device workspace, arena_floats floats */
} NrnPeerCtx;
int nrn_peer_reduce_adam(const NrnPeerCtx* ctx, const NrnAdamArgs* adam);
int nrn_peer_gather_rows(const NrnPeerCtx* ctx, const float* local, int n_per_rank, float* out, void* stream);

/* ---- evaluation and visualisation of rendered frames: what free_viewpoint_rendering.py does on the host with numpy,
 * scikit-image and matplotlib once the frames are rendered.  Frames are fp32 [n_frames][height][width][3] (disparity
 * [n_frames][height][width]), any sizes >= 1; n_frames = 0 returns NRN_OK and launches nothing.  Every score is a sum in
 * a fixed order (no atomics): bit-reproducible.  Colour images index matplotlib's 256-entry cm.jet table with
 * uint8(255 * clip(v, 0, 1)) (truncation, as .astype("uint8")); a NaN value takes entry 0. ---------------------------- */
/* The cm.jet table the kernels use, built from matplotlib's published segment data (_jet_data) the way matplotlib's
 * LinearSegmentedColormap builds it: rgb [256][3] = cm.jet(i)[:3] (float64), rgb8 [256][3] = to8b(rgb); either may be
 * NULL.  Host only: no CUDA call. */
int nrn_jet_colormap(double* rgb, uint8_t* rgb8);
/* Scores of free_viewpoint_rendering.py:818-862.  The mask (:820-823): pixels whose ground-truth channels sum to 0 in the
 * FIRST frame scored are zeroed in both images of every frame.  psnr = -10 log10(mean((gt - gen)^2)) over all
 * height * width * 3 values (+inf for identical frames, as the reference's log10(0)).  ssim = skimage
 * structural_similarity(data_range=1, gaussian_weights=True, sigma=1.5, use_sample_covariance=False, multichannel=True,
 * full=True): per channel, 11-tap Gaussian window (truncate 3.5) with mode "reflect", C1 = 0.01^2, C2 = 0.03^2; the
 * score is the mean of the map S over the frame cropped by 5 pixels on every side and over the channels (NaN when
 * height or width <= 10, as the mean of an empty crop).  The error images (:845-856) are to8b(jet(clip(10 |gt - gen|_2 /
 * sqrt(3)))) and to8b(jet(1 - mean_c S)).  The Gaussian moments and S in fp64 (S written as fp32), sums in fp64. */
size_t nrn_image_scores_bytes(int n_frames, int height, int width);   /* workspace: per-tile partial sums + a derived mask */
typedef struct NrnImageScoreArgs {
  const float* gt;            /* [F][H][W][3] ground truth */
  const float* generated;     /* [F][H][W][3] rendered */
  const uint8_t* mask;        /* [H][W] nonzero = masked, or NULL: derived from gt frame 0 into the workspace */
  int32_t n_frames, height, width;
  float* psnr;                /* out [F] */
  float* ssim;                /* out [F] */
  float* ssim_map;            /* out [F][H][W][3] the map S, or NULL */
  uint8_t* error_rgb;         /* out [F][H][W][3] scaled RGB error on jet, or NULL */
  uint8_t* error_ssim;        /* out [F][H][W][3] 1 - SSIM on jet, or NULL */
  void* workspace;            /* nrn_image_scores_bytes(), 16-byte aligned */
  void* stream;
} NrnImageScoreArgs;
int nrn_image_scores(const NrnImageScoreArgs* args);
/* visualize_disparity_with_jet_color_scheme and visualize_disparity_with_blinn_phong (run_nerf_helpers.py:701-793) for
 * every frame of disp [F][H][W]: jet [F][H][W][3] = the cm.jet colour of clip(d, 0, 1); phong [F][H][W][3] = the
 * reference's Blinn-Phong shading of the normals of np.gradient(d, 2 / (H - 1)) (needs H, W >= 2, as np.gradient does),
 * in fp32 (the reference mixes float32 and float64).  Either output may be NULL, not both. */
int nrn_disparity_images(const float* disp, int n_frames, int height, int width, float* jet, float* phong, void* stream);
/* Background stability of a fixed-camera sequence (free_viewpoint_rendering.py:770-785) over rgbs [F][H][W][3]:
 * std [H][W][3] = np.std(rgbs, axis=0) (ddof 0, two passes in fp32, frame-ordered sums as numpy's), image [H][W][3] =
 * the cm.jet colour of 10 * mean_c std.  Either output may be NULL, not both. */
int nrn_frame_std_image(const float* rgbs, int n_frames, int height, int width, float* std, float* image, void* stream);
/* The 8-bit images free_viewpoint_rendering.py saves per frame and as videos (:615-766), for a stack of F frames of
 * H x W pixels, in at most two launches (the per-frame maxima of disp, then every image).  Each output is written only
 * when its pointer is not NULL, and needs its input:
 *   out_rgb [F][H][W][3]             to8b(rgb)                                   (convert_rgb_to_saveable)
 *   out_disp [F][H][W]               to8b(disp / max of that frame), fp32        (convert_disparity_to_saveable)
 *   out_disp_video [F][H][W]         to8b(disp / max over all F frames)          (the disparity video, :725-730)
 *   out_disp_jet [F][H][W][3]        to8b(jet(disp / frame max))                 (convert_disparity_to_jet)
 *   out_disp_phong [F][H][W][3]      to8b of nrn_disparity_images' fp32 Phong value of disp / frame max (needs H, W >= 2)
 *   out_correspondences [F][H][W][3] c = (p - min) / (max - min) * 100 in fp64, to8b(c - trunc(c))    (:640-644)
 *   out_rigidity [F][H][W]           to8b(rigidity)                              (normalize=False)
 *   out_rigidity_jet [F][H][W][3]    to8b(jet(rigidity))                         (normalize=False)
 * to8b(v) = uint8(255 * clip(v, 0, 1)), truncated, NaN -> 0.  The disparity maxima follow np.max (a NaN makes the frame's
 * maximum NaN) and are written to disp_max, which every disparity output needs.  NULL args, negative sizes, an output
 * without its input, max_point <= min_point on an axis and float arrays not 4-byte aligned return NRN_E_INVALID before
 * any CUDA call; F = 0 or H * W = 0 returns NRN_OK and launches nothing. */
typedef struct NrnFrameImageArgs {
  const float* rgb;                /* [F][H][W][3] rendered colours, or NULL */
  const float* disp;               /* [F][H][W] disparity, or NULL */
  const float* surface_pts;        /* [F][H*W][3] canonical point of each pixel's median-visibility sample, or NULL */
  const float* surface_rigidity;   /* [F][H*W] its rigidity, or NULL (no bender) */
  const double* min_point;         /* host [3]: the checkpoint's min_nerf_volume_point (needed by out_correspondences) */
  const double* max_point;         /* host [3]: max_nerf_volume_point */
  int32_t n_frames, height, width;
  float* disp_max;                 /* out [F]: the maximum of each disparity frame (needed by every disparity output) */
  uint8_t* out_rgb;
  uint8_t* out_disp;
  uint8_t* out_disp_video;
  uint8_t* out_disp_jet;
  uint8_t* out_disp_phong;
  uint8_t* out_correspondences;
  uint8_t* out_rigidity;
  uint8_t* out_rigidity_jet;
  void* stream;
} NrnFrameImageArgs;
int nrn_frame_images(const NrnFrameImageArgs* args);

/* ---- triangle meshes: density grids and marching cubes (geometry.py) -------------------------
 * No reference counterpart (the reference exports no geometry).  The grid has nx x ny x nz points; point (i, j, k) is
 * (x_i, y_j, z_k) with x_i = lo + (hi - lo) * (i / (n - 1)) per axis, each operation rounded in fp32 (lo, hi are fp32),
 * and x_{n-1} = hi exactly.  Sizes: 2 <= n <= 2^24 per axis and nx * ny <= 2^28.  A grid point is occupied when
 * sigma > threshold (NaN is not, and counts as 0 when a vertex is placed).
 *
 * nrn_mesh_grid_points: points [ny][nx][3] of z-plane k, the input of a point-mode nrn_field_forward.
 * nrn_mesh_sigma: sigma[i] = relu(raw[i][3]) (NaN stays NaN) of n rows of out_ch floats. */
int nrn_mesh_grid_points(const float* min_point, const float* max_point, int nx, int ny, int nz, int k, float* points, void* stream);
int nrn_mesh_sigma(const float* raw, long long n, int out_ch, float* sigma, void* stream);
/* The volume is meshed one z-slab at a time, in this order for k = 0 .. nz - 1 (nrn_mesh_count(k + 1) may be enqueued
 * before nrn_mesh_emit(k): the workspace keeps three planes' states):
 *   nrn_mesh_count(k): per point of plane k its crossed edges to +x, +y and (sigma1 = plane k + 1 given, k < nz - 1) +z,
 *     per cell between planes k and k + 1 its case index and triangle count; both scanned in place.  totals (device
 *     int32 [2]) receives the number of vertices of plane k and of faces of cell layer k.
 *   nrn_mesh_emit(k): the vertices of plane k at rows vertex_base.. of vertices [V][3] (ordered by edge key (j, i, axis)),
 *     each at p_a + ((t - s_a) / (s_b - s_a)) * (p_b - p_a) from its lower end a; and for k >= 1 the faces of cell layer
 *     k - 1 at rows face_base.. of faces [T][3] (ordered by cell (j, i), then by table order), whose vertex ids count from
 *     vertex_base_prev (plane k - 1) and vertex_base (plane k).
 * The caller carries the running bases (sums of totals) and keeps V and T below 2^31.  NULL args, bad sizes, a missing
 * pointer, a negative base and misaligned arrays return NRN_E_INVALID before any CUDA call. */
typedef struct NrnMeshSlabArgs {
  const float* sigma0;        /* [ny][nx] density of plane k */
  const float* sigma1;        /* [ny][nx] density of plane k + 1, NULL for k = nz - 1 */
  const float* min_point;     /* host [3], needed by nrn_mesh_emit */
  const float* max_point;     /* host [3] */
  float threshold;
  int32_t nx, ny, nz, k;
  void* workspace;            /* nrn_mesh_workspace_bytes(nx, ny), 256-byte aligned, the same for every k of one volume */
  int32_t* totals;            /* count: out device [2] */
  int64_t vertex_base_prev;   /* emit: global id of plane k - 1's first vertex */
  int64_t vertex_base;        /* emit: global id of plane k's first vertex */
  int64_t face_base;          /* emit: index of cell layer k - 1's first face */
  float* vertices;            /* emit: out [V][3] */
  int32_t* faces;             /* emit: out [T][3] */
  void* stream;
} NrnMeshSlabArgs;
size_t nrn_mesh_workspace_bytes(int nx, int ny);   /* 0 for sizes out of range */
int nrn_mesh_count(const NrnMeshSlabArgs* args);
int nrn_mesh_emit(const NrnMeshSlabArgs* args);
/* colors [n][3] = to8b(sigmoid(raw[i][0:3])) of n rows of out_ch floats (to8b as in nrn_frame_images). */
int nrn_mesh_colors(const float* raw, long long n, int out_ch, uint8_t* colors, void* stream);
/* Host copy of the cube table: counts [256] triangles per case, edges [256][5][3] their edges (-1 padded).  Corner c is
 * at offset (c & 1, c >> 1 & 1, c >> 2 & 1); edge e = 4 * axis + r runs along axis from the corner whose other two
 * offsets are (r & 1, r >> 1).  DESIGN.md describes the construction.  Either pointer may be NULL. */
int nrn_mesh_cube_table(int32_t* counts, int8_t* edges);

/* ---- LPIPS: the perceptual score of rendered frames (evaluation.py) ---------------------------
 * lpips.LPIPS(net='alex') (v0.1, eval mode) as free_viewpoint_rendering.py:788-849 scores every frame and :868 averages
 * the scores.  Per frame pair: zero the masked pixels of both images, t = 2x - 1, s = (t - shift) / scale (fp32), the
 * AlexNet features (conv1 11x11/4 pad 2 -> 64, max-pool 3/2, conv2 5x5 pad 2 -> 192, max-pool 3/2, conv3 3x3 -> 384,
 * conv4 -> 256, conv5 -> 256, each conv + bias + ReLU; the five ReLU outputs are the taps), and per tap k the mean over
 * its pixels of sum_c w_k[c] (f_gt[c] / (|f_gt| + 1e-10) - f_gen[c] / (|f_gen| + 1e-10))^2; LPIPS is the sum of the five.
 * The convolutions run on fp16 operands with fp32 accumulation, activations are stored in fp16, the distances are fp32
 * per pixel and fp64 per frame, summed in a fixed order: a frame's score does not depend on the batch or chunk it is in.
 * A convolution output above 65504 (the largest fp16) cannot be stored: a frame either of whose images has one scores
 * NaN, and so do its tap scores from that convolution's tap on (no synchronisation; the call stays graph-capturable).
 *
 * nrn_lpips_pack: the packed weight block (nrn_lpips_packed_bytes(), 16-byte aligned, device) from 17 device fp32 arrays:
 *   tensors[2 l], tensors[2 l + 1]  conv weight (OIHW) and bias of layer l = 0..4 (net.slice1.0, net.slice2.3,
 *                                   net.slice3.6, net.slice4.8, net.slice5.10)
 *   tensors[10 + k]                 tap weights w_k [C_k] (lin{k}.model.1.weight)
 *   tensors[15], tensors[16]        shift [3] and scale [3] (scaling_layer)
 * Once per weight set; the sources may be freed after the stream has run the pack.
 * nrn_lpips_workspace_bytes(F, H, W): the workspace nrn_lpips uses for F frames of H x W by default: the derived mask,
 *   ceil(H * W / 256) * 256 bytes, plus min(F, max(1, 256 MiB / B), 4096) frames of B bytes each, B the activations of
 *   both images of a frame at every stage (fp16 NHWC), its distance partials and saturation words.
 *   nrn_lpips_workspace_bytes(1, H, W) - nrn_lpips_workspace_bytes(0, H, W) is B.  0 for sizes out of range.
 * nrn_lpips: lpips [F] and, when per_layer is not NULL, the tap scores per_layer [F][5].  Frames go in chunks of
 *   (workspace_bytes - mask bytes) / B frames (at most 4096).  NULL args or pointers, negative sizes, H or W below 31 (the
 *   smallest frame every tap has a pixel of) or above 16384, float arrays not 4-byte aligned, packed weights not 16-byte
 *   aligned, a workspace not 256-byte aligned or too small for one frame return NRN_E_INVALID before any CUDA call;
 *   n_frames = 0 returns NRN_OK and launches nothing. */
typedef struct NrnLpipsArgs {
  const float* gt;            /* [F][H][W][3] ground truth in [0, 1] */
  const float* generated;     /* [F][H][W][3] renders */
  const uint8_t* mask;        /* [H][W] nonzero = masked, or NULL: the pixels of gt frame 0 whose channels sum to 0 */
  int32_t n_frames, height, width;
  const void* packed;         /* nrn_lpips_pack output */
  float* lpips;               /* out [F] */
  float* per_layer;           /* out [F][5] tap scores, or NULL */
  void* workspace;            /* 256-byte aligned */
  size_t workspace_bytes;
  void* stream;
} NrnLpipsArgs;
size_t nrn_lpips_packed_bytes(void);
int nrn_lpips_pack(const float* const* tensors, void* packed, void* stream);
size_t nrn_lpips_workspace_bytes(int n_frames, int height, int width);
int nrn_lpips(const NrnLpipsArgs* args);

/* Spatial LPIPS maps: what lpips.LPIPS(net='alex', spatial=True) returns (retPerLayer=True for the per-tap maps), which
 * free_viewpoint_rendering.py does not compute.  Per frame of H x W and tap l with per-pixel distances d_l [h_l][w_l]
 * (the values nrn_lpips averages): up_l = F.interpolate(d_l, size=(H, W), mode="bilinear", align_corners=False), in
 * fp32 with each operation rounded on its own (scale = (float)h_l / H, src = max(scale (y + 0.5) - 0.5, 0), i0 = (int)src,
 * i1 = i0 + (i0 < h_l - 1), l1 = src - i0, l0 = 1 - l1, the same along x, v = hl0 (wl0 x00 + wl1 x01) + hl1 (wl0 x10 +
 * wl1 x11)), and map = (((up_0 + up_1) + up_2) + up_3) + up_4.  The mask zeroes pixels before the network as in nrn_lpips;
 * the map covers every pixel.  A frame whose convolution l clamped an output gets NaN in up_l, in every later tap's map
 * and in map; its earlier taps' maps stay finite.  lpips and per_layer are those of nrn_lpips, bit for bit, and a frame's
 * maps do not depend on its chunk.
 * nrn_lpips_maps_workspace_bytes(F, H, W): nrn_lpips's layout with frames of B' bytes, B' = B plus the five fp32 tap
 *   maps of the frame (each rounded up to 256 bytes); chunks of min(F, max(1, 256 MiB / B'), 4096) frames by default.
 * nrn_lpips_maps: everything nrn_lpips checks, with chunks of (workspace_bytes - mask bytes) / B' frames, plus a NULL
 *   maps (always) or maps->map (n_frames > 0) and float outputs not 4-byte aligned: NRN_E_INVALID before any CUDA call. */
typedef struct NrnLpipsMapArgs {
  float* map;                 /* out [F][H][W], required */
  float* layer_maps;          /* out [F][5][H][W] per-tap maps, or NULL */
  uint8_t* error_image;       /* out [F][H][W][3] to8b(jet(clip(map, 0, 1))) (NaN: jet index 0), or NULL */
} NrnLpipsMapArgs;
size_t nrn_lpips_maps_workspace_bytes(int n_frames, int height, int width);
int nrn_lpips_maps(const NrnLpipsArgs* args, const NrnLpipsMapArgs* maps);

/* ---- correspondences between rendered frames (correspondence.py) ------------------------------
 * render(..., surface_output=True) gives every pixel its canonical surface point (train.py:159-176: the median-visibility
 * sample mapped back through the ray bender); free_viewpoint_rendering.py:615-645 only paints those points as a
 * checkerboard.  nrn_match turns them into pixel correspondences: for every valid query pixel, the target pixel of the paired
 * frame whose canonical point is nearest.
 *
 * Pairs: F = max(Fq, Ft) frame pairs, query frame (Fq == 1 ? 0 : f) against target frame (Ft == 1 ? 0 : f); Fq == Ft, Fq
 * == 1 or Ft == 1.  A point is valid when its mask byte is nonzero (or the mask is NULL) and its coordinates are finite.
 * The distance is d2 = (dx*dx + dy*dy) + dz*dz in fp32, each operation rounded on its own; the match is the valid target
 * point of smallest (d2, index), kept when d2 <= fl(max_distance^2): the brute-force answer, whatever the search order.
 *   index [F][Hq][Wq]       y * Wt + x of the match, or -1 (query pixel invalid, no valid target, or beyond max_distance)
 *   distance [F][Hq][Wq]    sqrt(d2) of the match, +inf where index is -1
 *   flow [F][Hq][Wq][2]     (x_t - x_q, y_t - y_q) in pixels, NaN where index is -1
 *   consistent [F][Hq][Wq]  (round_trip) 1 when the match's own match in the query frame, by the same rule, lies within
 *                           round_trip_pixels of the query pixel (fl(dx*dx + dy*dy) <= fl(tol^2)); 0 where index is -1
 * Each target frame's valid points go into an n^3 uniform grid over their bounding box (n^3 <= max(1, Ht*Wt / 2), n as
 * large as that allows), and each query searches rings of cells until no unsearched cell can hold a closer point.
 *
 * nrn_match_workspace_bytes: the workspace for these sizes (the target frames' grids, and with round_trip the query
 *   frames' grids), a sum of 256-byte aligned sections: per frame set of F frames of N = H * W points with C = n^3 cells,
 *   32 F, 4 F C, 4 F (C + 1) and 16 F N bytes.  0 for sizes out of range or frame counts that do not pair.
 * nrn_match: NULL args or pointers (consistent is needed with round_trip), H or W outside 1..2^24, H * W above 2^31 - 1,
 *   frame counts above 65535 or that do not pair, a NaN or negative max_distance or round_trip_pixels, float and index
 *   arrays not 4-byte aligned, a workspace not 256-byte aligned or smaller than nrn_match_workspace_bytes return
 *   NRN_E_INVALID before any CUDA call; F = 0 returns NRN_OK and launches nothing. */
typedef struct NrnMatchArgs {
  const float* query;           /* [Fq][Hq][Wq][3] canonical surface points */
  const float* target;          /* [Ft][Ht][Wt][3] */
  const uint8_t* query_mask;    /* [Fq][Hq][Wq] nonzero = a surface point, or NULL */
  const uint8_t* target_mask;   /* [Ft][Ht][Wt], or NULL */
  int32_t n_query_frames, query_height, query_width;
  int32_t n_target_frames, target_height, target_width;
  float max_distance;           /* canonical-space radius; +inf for none */
  int32_t round_trip;
  float round_trip_pixels;
  int32_t* index;               /* out [F][Hq][Wq] */
  float* distance;              /* out [F][Hq][Wq] */
  float* flow;                  /* out [F][Hq][Wq][2] */
  uint8_t* consistent;          /* out [F][Hq][Wq] (round_trip), else ignored */
  void* workspace;              /* 256-byte aligned */
  size_t workspace_bytes;
  void* stream;
} NrnMatchArgs;
size_t nrn_match_workspace_bytes(int n_query_frames, int query_height, int query_width, int n_target_frames, int target_height,
                                 int target_width, int round_trip);
int nrn_match(const NrnMatchArgs* args);

/* ---- occupancy grid: render passes that skip the NeRF trunk for samples in empty canonical space --------------------
 * A grid of nx * ny * nz cells over [min_point, max_point]; cell (i, j, k) is bit c % 32 of bits[c / 32], c = (k * ny + j)
 * * nx + i.  A point is KEPT when a coordinate is non-finite or outside the box (x < min or x > max), or when its cell is
 * occupied; its cell is min(floor(fl(fl(x - min) * scale)), n - 1) per axis with scale = fl(n / fl(max - min)), every
 * operation an fp32 one rounded on its own.
 *
 * nrn_occupancy_build: sigma [nz + 1][ny + 1][nx + 1] densities at the cells' corners.  A cell is occupied when any of its
 *   8 corners has sigma > threshold or NaN; the occupied set is then dilated by `dilation` cells (Chebyshev distance).
 *   bits: nrn_occupancy_words(nx, ny, nz) words; workspace: nrn_occupancy_build_workspace_bytes.  Sides outside
 *   1..4096, dilation outside 0..4096, a NaN threshold or null pointers return NRN_E_INVALID before any CUDA call.
 * nrn_occupancy_compact: the lookup of points [n_points][points_stride] (xyz first): kept points' xyz -> kept_xyz [K][3]
 *   and their indices -> kept_index [K] in ascending order, K -> *count (device memory); the order comes from a fixed
 *   block scan, so reruns are identical.  workspace: nrn_occupancy_compact_workspace_bytes(n_points), 256-byte aligned.
 * nrn_field_forward_occupancy: one inference pass of nrn_field_forward in ray mode (args as there, no stash / relu_mask,
 *   points NULL) that evaluates the NeRF trunk only on kept samples: with a bender the bend pass (bent points, rigidities
 *   and the details), then the lookup of the bent points (without one, of rays_o + rays_d * z), the point-mode trunk on
 *   the K kept points (K read on the device: no host synchronisation, CUDA-graph capturable), and the scatter.  raw of a
 *   kept sample equals nrn_field_forward's bit for bit (object removal included); raw of a skipped sample is 0.  The
 *   details are those of nrn_field_forward for every sample.  workspace: nrn_occupancy_workspace_bytes(n_rays, n_samples,
 *   out_ch, bender_packed != NULL), 256-byte aligned.  A malformed grid, more than 2^31 - 1 points or a short workspace
 *   return NRN_E_INVALID before any CUDA call. */
typedef struct NrnOccupancyGrid {
  const uint32_t* bits;
  int32_t nx, ny, nz;         /* cells per axis, 1..4096 */
  float min_point[3];
  float max_point[3];
} NrnOccupancyGrid;
size_t nrn_occupancy_words(int nx, int ny, int nz);
size_t nrn_occupancy_build_workspace_bytes(int nx, int ny, int nz);
int nrn_occupancy_build(const float* sigma, int nx, int ny, int nz, float threshold, int dilation, void* workspace, uint32_t* bits,
                        void* stream);
size_t nrn_occupancy_compact_workspace_bytes(int64_t n_points);
int nrn_occupancy_compact(const NrnOccupancyGrid* grid, const float* points, int64_t n_points, int64_t points_stride, float* kept_xyz,
                          int32_t* kept_index, int32_t* count, void* workspace, void* stream);
size_t nrn_occupancy_workspace_bytes(int n_rays, int n_samples, int out_ch, int has_bender);
int nrn_field_forward_occupancy(const NrnFieldArgs* args, const NrnOccupancyGrid* grid, void* workspace, size_t workspace_bytes);

/* ---- early ray termination: render passes that stop evaluating a ray's samples once its transmittance is small ------
 * The reference evaluates every sample of every ray (train.py:876-886, :927-937); this pass is an inference-only option
 * it does not have.  Samples 0..S-1 of a ray are split into segments of K = nrn_termination_segment() samples; round r
 * evaluates segment r, samples [r K, min((r + 1) K, S)), of every ray still alive (all rays are alive at round 0), and
 * ceil(S / K) rounds make a pass.  After round r every alive ray updates T <- T * (1 - alpha_i + 1e-10) over the
 * segment's samples in order, in fp32 with one rounded multiply per step, from T = 1, where alpha_i is compositing's own
 * (nrn_composite; train.py:740-761: relu(sigma + noise), the distance to the next depth, 1e10 past the last, times |d|)
 * on the raw that round wrote, object removal included.  The ray dies when T < threshold; a NaN T never does, nor does
 * any T for threshold 0.  A sample not evaluated gets raw = 0 (so alpha = 0 and a factor of exactly 1).
 *
 * nrn_field_forward_terminate: one inference pass of nrn_field_forward in ray mode (args as there, no stash / relu_mask,
 *   points NULL).  With a bender the bend pass runs first over every sample (bent points, rigidities and the details);
 *   then per round the lookup and compaction of that segment's samples only (kept: the ray is alive and, when grid is
 *   not NULL, the grid keeps the point, as in nrn_field_forward_occupancy; without a bender this step also writes every
 *   sample's initial_input_pts / input_pts), the point-mode trunk on the kept points, the scatter into raw (zeroed once
 *   before round 0) and the transmittance update.  raw of an evaluated sample equals nrn_field_forward's bit for bit.
 *   The rounds come from the shapes, so nothing waits on the host and the pass can be captured in a CUDA graph.
 *   termination_index [n_rays] (int32): the first sample skipped because of termination, i.e. the end of the segment in
 *   which T fell below the threshold, or S if the ray never died.  noise [n_rays][n_samples]: the additive sigma noise
 *   (already scaled by raw_noise_std) that compositing will use, or NULL.  workspace:
 *   nrn_termination_workspace_bytes(n_rays, n_samples, out_ch, bender_packed != NULL), 256-byte aligned.  A threshold
 *   outside [0, 1] or NaN, a null termination_index, a malformed grid, more than 2^31 - 1 points or a short workspace
 *   return NRN_E_INVALID before any CUDA call; n_rays = 0 launches nothing. */
typedef struct NrnTerminationArgs {
  float threshold;              /* in [0, 1]: a ray dies when its transmittance T < threshold */
  const float* noise;           /* [n_rays][n_samples] additive sigma noise, or NULL */
  int32_t* termination_index;   /* [n_rays] out */
} NrnTerminationArgs;
int nrn_termination_segment(void);
size_t nrn_termination_workspace_bytes(int n_rays, int n_samples, int out_ch, int has_bender);
int nrn_field_forward_terminate(const NrnFieldArgs* args, const NrnOccupancyGrid* grid /* NULL: none */, const NrnTerminationArgs* term,
                                void* workspace, size_t workspace_bytes);

/* ---- the inverse of the ray bender: canonical points into every frame (geometry.deform_points) -------------------------
 * The ray bender maps an observed point x of a frame with latent z to the canonical point c = b(x; z) = x + s r~(x) o(x, z)
 * (run_nerf_helpers.py:507-584: o the offset MLP on [x, z], r = (tanh(rho(x)) + 1) / 2 the rigidity, r~ = 0 where
 * r <= rigidity_cutoff (use_cutoff), s = scaling (use_scaling) or 1).  nrn_deform_points solves b(x; z_f) = c for every
 * canonical point c and every latent z_f: x_0 = c - s r~(c) o(c, z_f), then `iterations` Newton steps
 * x <- x - J(x)^-1 (b(x) - c), J = I + s (r~ do/dx + o grad(r~)^T).  A point whose |b(x) - c|_2 <= tol is frozen (its
 * later steps are skipped).  Where J is singular (|det J| <= 1e-6 |J e_0| |J e_1| |J e_2|) or the Newton step is not
 * finite, the step is the fixed-point one, x <- x - (b(x) - c).  Then residual = |b(x) - c|_2 at the result, converged =
 * residual <= tol, rigidity = r~(x).  A point or latent with a non-finite value gives NaN out, residual and rigidity and
 * converged = 0.  b and J are evaluated at fp32 accuracy.  The launch count does not depend on the data, so the call can
 * be captured in a CUDA graph, and a frame's results do not depend on the other frames of the call.
 *
 * NULL args, points, latents, bender_packed or out, negative sizes, latent_stride below 32, iterations outside 1..64,
 * a NaN, infinite or negative tol, a non-finite scaling or rigidity_cutoff (when used), float arrays not 4-byte aligned
 * or bender_packed not 16-byte aligned return NRN_E_INVALID before any CUDA call; n_points = 0 or n_latents = 0 returns
 * NRN_OK and launches nothing. */
typedef struct NrnDeformArgs {
  const float* points;  int64_t n_points;                          /* canonical c [P][3] */
  const float* latents; int32_t n_latents; int64_t latent_stride;  /* [F][32] */
  const void* bender_packed;                                       /* nrn_pack_bender output, 16-byte aligned */
  int32_t use_cutoff; float rigidity_cutoff; int32_t use_scaling; float scaling;
  int32_t iterations; float tol;
  float* out;            /* [F][P][3] */
  float* residual;       /* [F][P] or NULL */
  uint8_t* converged;    /* [F][P] or NULL */
  float* rigidity;       /* [F][P] r~ at the result, or NULL */
  void* stream;
} NrnDeformArgs;
int nrn_deform_points(const NrnDeformArgs* args);

/* ---- surface normals: the density gradient at points (geometry.density_gradient) -------------------------------------
 * grad[i] = d raw[i][3] / d x_i of NeRF.forward in point mode: the density before its ReLU, through the ray bender when
 * bender_packed is given (bent = x + r~ o (* s), with the test-time knobs use_cutoff / use_scaling, and raw[3] -- so its
 * gradient -- zeroed where r~ >= removal_threshold when use_removal), through the trunk alone otherwise.  The
 * time-conditioned baseline passes its fp32 nn.Linear weights tc_w0 [256][95], tc_b0, tc_w5 [256][351], tc_b5 (all four
 * or none; no bender), which fold each point's latent into L0 / L5 biases.  A view-dependent model passes its trunk
 * image (alpha in head row 3): the density needs only the trunk and the bender.
 * Points run in chunks of nrn_density_gradient_chunk() points; per chunk one forward kernel writes the ReLU mask bits, the
 * positional encoding and the bender's offsets and rigidity into the workspace, and one DGRAD kernel with d raw = e_3
 * (loss scale 2^9) writes grad.  The workspace holds one chunk, so its size is bounded independently of n_points.
 * Workspace layout for n = min(n_points, chunk) points in T = ceil(n / 128) rounded up to even tiles, each piece on a
 * 256-byte boundary: ReLU mask bits [T][40960] (the training layout), the positional encoding E [T][16384] (the training
 * stash's first image), unmasked offsets [n][3] fp32, rigidity [n] fp32, time-conditioned ray biases.  After the call it
 * holds the last chunk's.  No
 * host synchronisation: the call can be captured in a CUDA graph.  A non-finite point gives a non-finite gradient.
 *
 * NULL args, points, grad or nerf_packed, n_points < 0, points_stride < 3, latent_stride neither 0 nor >= 32, a bender
 * or time-conditioned weights without latents, latents with neither, a bender with time-conditioned weights, only some of
 * the four time-conditioned weights, a non-finite knob in use, float arrays not 4-byte aligned, packed weights or the
 * workspace not 16-byte aligned, or workspace_bytes below nrn_density_gradient_workspace_bytes(n_points, latents per
 * point of a time-conditioned call) return NRN_E_INVALID before any CUDA call; n_points = 0 launches nothing. */
typedef struct NrnDensityGradArgs {
  const float* points; int64_t n_points; int64_t points_stride;   /* [P][points_stride], xyz first */
  const float* latents; int64_t latent_stride;                    /* [P][latent_stride] (0: one row for every point) or NULL */
  const void* nerf_packed;                                        /* nrn_pack_nerf output */
  const void* bender_packed;                                      /* nrn_pack_bender output, or NULL */
  const float* tc_w0; const float* tc_b0; const float* tc_w5; const float* tc_b5;   /* time-conditioned baseline, or NULL */
  int32_t use_cutoff; float rigidity_cutoff; int32_t use_scaling; float scaling; int32_t use_removal; float removal_threshold;
  float* grad;                                                    /* [P][3] out */
  void* workspace; size_t workspace_bytes;
  void* stream;
} NrnDensityGradArgs;
int64_t nrn_density_gradient_chunk(void);
size_t nrn_density_gradient_workspace_bytes(int64_t n_points, int per_point_ray_bias);
int nrn_field_density_gradient(const NrnDensityGradArgs* args);

/* ---- optional per-kernel timing (measurement aid for bench.py) ---------------------------------
 * While enabled, every launch of the kernel kinds below is bracketed by CUDA events recorded on the
 * launch stream.  kinds: 0 field forward, 1 field DGRAD, 2 WGRAD (+reduce), 3 composite(+resample),
 * 4 composite backward, 5 divergence regulariser, 6 time-conditioned ray bias (nrn_tc_latent_bias), 7 time-conditioned
 * latent gradients (per-ray sums, d z, latent columns of dW0 / dW5), 8 bend pass of the view-dependent head, 9 its
 * view-head field kernel (nrn_field_forward_views), 10 its training forward (nrn_field_forward_views_train), 11 its DGRAD
 * and 12 its WGRAD (+reduce) (nrn_field_backward_views), 13 the fixed-order latent reduction (nrn_field_backward_det) and
 * 14 the fixed-order divergence loss reduction (nrn_divergence_forward_det), 15 the held-out DGRAD
 * (nrn_field_backward_held_out, nrn_field_backward_det_held_out) and 16 the held-out divergence backward
 * (nrn_divergence_backward_held_out; its WGRAD is kind 2), 17 nrn_image_scores (mask, SSIM tiles, per-frame reduction),
 * 18 nrn_disparity_images, 19 nrn_frame_std_image and 20 nrn_frame_images, 21 nrn_mesh_grid_points and nrn_mesh_sigma, 22
 * nrn_mesh_count (counts and scans), 23 nrn_mesh_emit (vertices and faces) and 24 nrn_mesh_colors, and of nrn_lpips 25 the
 * mask and input scaling, 26 the convolutions, 27 the max-pools and 28 the distances and per-frame sums, and of nrn_match 29
 * the grid builds (boxes, counts, scans, scatters) and 30 the queries with their round trips, 31 nrn_occupancy_build, and of
 * nrn_field_forward_occupancy 32 the bend pass, 33 the lookup and compaction (also nrn_occupancy_compact), 34 the trunk on
 * the kept points and 35 the scatter, and of nrn_field_forward_terminate 36 the bend pass, 37 the lookups and compactions,
 * 38 the trunk on the kept points, 39 the scatters (and the zeroing of raw) and 40 the transmittance updates (and their
 * initialisation), 41 nrn_deform_points, and of nrn_field_density_gradient 42 the forward (with the time-conditioned
 * biases) and 43 the DGRAD, 44 the upsampling of nrn_lpips_maps (its other kernels are kinds 25 to 28, the distances
 * with their tap maps kind 28).  nrn_timing_read synchronises the recorded events and returns per-kind sums.
 * nrn_timing_enable(0) stops recording and keeps the events; nrn_timing_enable(1) releases the previous session's events,
 * so a CUDA graph captured during that session must be released before timing is enabled again. */
int nrn_timing_enable(int on);
int nrn_timing_read(double* ms_sum, int* counts, int n_kinds);

#ifdef __cplusplus
}
#endif
#endif /* NRNERF_B200_H */
