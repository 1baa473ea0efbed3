// Fixed-order per-ray reductions of deterministic mode (torch.use_deterministic_algorithms(True)).
//
// The field DGRAD kernel (B0^T epilogue, per-ray latent gradient) and the divergence forward (B4 epilogue, per-ray loss)
// normally add each warp's rows into the per-ray result with fp32 atomics, whose order depends on scheduling.  Their
// deterministic variants write per-point rows instead, by one rule: warps cover 32-aligned blocks [32k, 32k + 32) of global
// point indices (tiles are 128 rows, row warps 32), and a block is "uniform" when all its points exist (32k + 31 < P) and
// lie in one ray.  A uniform warp stores its in-warp sum (fixed order) in the row of its first point 32k; any other warp
// stores each valid point's row.  The kernels here walk each ray's points in increasing order: at the first point of a
// uniform block they add that row and skip 32 points, otherwise they add the row and step by one.  Whether a block is
// uniform depends only on (k, S, P), so the order of every addition is fixed by construction.
#include "nrn_common.cuh"
#include "det_reduce.cuh"

namespace nrn {

namespace {

__device__ __forceinline__ long long det_step(long long pt, int S, long long P) {
  return (pt & 31) == 0 && pt + 31 < P && pt / S == (pt + 31) / S ? 32 : 1;
}

// one warp per ray, lane = latent dim: d_latents[ray] = sum of the ray's latent rows (overwritten)
__global__ void __launch_bounds__(256) latent_reduce_kernel(const float* __restrict__ rows, float* __restrict__ d_latents, int n_rays,
                                                            int S) {
  const long long ray = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (ray >= n_rays) return;
  const long long P = static_cast<long long>(n_rays) * S, end = (ray + 1) * S;
  float acc = 0.f;
  for (long long pt = ray * S; pt < end; pt += det_step(pt, S, P)) acc += __ldg(rows + pt * kLatent + lane);
  d_latents[ray * kLatent + lane] = acc;
}

// one thread per ray: loss[ray] = sum of the ray's loss rows (overwritten)
__global__ void __launch_bounds__(256) div_loss_reduce_kernel(const float* __restrict__ rows, float* __restrict__ loss, int n_rays, int S) {
  const long long ray = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (ray >= n_rays) return;
  const long long P = static_cast<long long>(n_rays) * S, end = (ray + 1) * S;
  float acc = 0.f;
  for (long long pt = ray * S; pt < end; pt += det_step(pt, S, P)) acc += __ldg(rows + pt);
  loss[ray] = acc;
}

}  // namespace

cudaError_t launch_latent_reduce(const float* rows, float* d_latents, int n_rays, int S, cudaStream_t st) {
  if (n_rays <= 0) return cudaSuccess;
  latent_reduce_kernel<<<static_cast<unsigned>((n_rays + 7) / 8), 256, 0, st>>>(rows, d_latents, n_rays, S);
  return cudaGetLastError();
}

cudaError_t launch_div_loss_reduce(const float* rows, float* loss, int n_rays, int S, cudaStream_t st) {
  if (n_rays <= 0) return cudaSuccess;
  div_loss_reduce_kernel<<<static_cast<unsigned>((n_rays + 255) / 256), 256, 0, st>>>(rows, loss, n_rays, S);
  return cudaGetLastError();
}

}  // namespace nrn
