// NeuS SDF -> alpha (NeuSModel.get_alpha, models/neus.py:117-139) fused with the normalisation of the analytic normal
// (F.normalize(sdf_grad), models/neus.py:225): one elementwise kernel per direction instead of ~15 (forward) + ~25 (backward)
// torch kernels over [K]-sized tensors.
//   n         = g / max(|g|, 1e-12)
//   true_cos  = d . n
//   iter_cos  = -(relu(-true_cos/2 + 1/2) (1 - a) + relu(-true_cos) a)          a = cos_anneal_ratio
//   prev/next = sdf -/+ iter_cos * dist / 2
//   alpha     = clip((sigmoid(s prev) - sigmoid(s next) + 1e-5) / (sigmoid(s prev) + 1e-5), 0, 1)      s = inv_s (device scalar)
#include "neus_shade.cuh"

namespace {

__global__ void __launch_bounds__(256) neus_alpha_fwd_kernel(const float* __restrict__ sdf, const float* __restrict__ sdf_grad,
                                                             const float* __restrict__ dirs, const float* __restrict__ dists,
                                                             const float* __restrict__ inv_s, float cos_anneal, const float* __restrict__ cos_dev,
                                                             float* __restrict__ alpha, float* __restrict__ normal, int64_t n_cap,
                                                             const int64_t* __restrict__ n_dev) {
  const int64_t n = n_dev ? min(*n_dev, n_cap) : n_cap;
  if (cos_dev) cos_anneal = __ldg(cos_dev);  // schedule value kept on the device: a captured graph follows update_step()
  const int64_t i = blockIdx.x * 256ll + threadIdx.x;
  if (i >= n) return;
  const AlphaTerms t = alpha_terms(sdf[i], sdf_grad[i * 3], sdf_grad[i * 3 + 1], sdf_grad[i * 3 + 2], dirs[i * 3], dirs[i * 3 + 1], dirs[i * 3 + 2],
                                   dists[i], __ldg(inv_s), cos_anneal);
  alpha[i] = fminf(fmaxf(t.q, 0.f), 1.f);
  normal[i * 3] = t.nx;
  normal[i * 3 + 1] = t.ny;
  normal[i * 3 + 2] = t.nz;
}

// inputs: d alpha [K], d normal [K,3] (sum of every consumer of the normal: colour network input, composited normal);
// outputs: d sdf [K], d sdf_grad [K,3], d inv_s (one atomicAdd per block).
__global__ void __launch_bounds__(256) neus_alpha_bwd_kernel(const float* __restrict__ sdf, const float* __restrict__ sdf_grad,
                                                             const float* __restrict__ dirs, const float* __restrict__ dists,
                                                             const float* __restrict__ inv_s, float cos_anneal, const float* __restrict__ cos_dev,
                                                             const float* __restrict__ d_alpha, const float* __restrict__ d_normal,
                                                             float* __restrict__ d_sdf, float* __restrict__ d_sdf_grad,
                                                             float* __restrict__ d_inv_s, int64_t n_cap, const int64_t* __restrict__ n_dev) {
  const int64_t n = n_dev ? min(*n_dev, n_cap) : n_cap;
  if (cos_dev) cos_anneal = __ldg(cos_dev);
  const int64_t i = blockIdx.x * 256ll + threadIdx.x;
  float ds_part = 0.f;
  if (i < n) {
    const float dx = dirs[i * 3], dy = dirs[i * 3 + 1], dz = dirs[i * 3 + 2], s = __ldg(inv_s);
    const AlphaTerms t = alpha_terms(sdf[i], sdf_grad[i * 3], sdf_grad[i * 3 + 1], sdf_grad[i * 3 + 2], dx, dy, dz, dists[i], s, cos_anneal);
    const float dq = (t.q >= 0.f && t.q <= 1.f) ? d_alpha[i] : 0.f;  // clip passes the gradient on the closed interval
    const float inv_c = 1.f / (t.pc + 1e-5f);
    const float dp = dq * inv_c, dc = -dq * t.q * inv_c;
    const float d_ps = (dp + dc) * t.pc * (1.f - t.pc);  // w.r.t. (prev * s)
    const float d_ns = -dp * t.nc * (1.f - t.nc);         // w.r.t. (next * s)
    ds_part = d_ps * t.prev + d_ns * t.next;
    const float d_prev = d_ps * s, d_next = d_ns * s;
    d_sdf[i] = d_prev + d_next;
    const float d_iter = (d_next - d_prev) * t.dist * 0.5f;
    const float u = -t.true_cos * 0.5f + 0.5f, v = -t.true_cos;
    const float d_tc = d_iter * ((u > 0.f ? 0.5f * (1.f - cos_anneal) : 0.f) + (v > 0.f ? cos_anneal : 0.f));
    float gnx = d_tc * dx, gny = d_tc * dy, gnz = d_tc * dz;
    if (d_normal) {
      gnx += d_normal[i * 3];
      gny += d_normal[i * 3 + 1];
      gnz += d_normal[i * 3 + 2];
    }
    // n = g / max(|g|, eps): d g = (d n - n (n . d n)) / |g| away from the clamp, d n / eps inside it
    const bool clamped = t.inv_norm >= 1e12f;
    const float dot = clamped ? 0.f : (t.nx * gnx + t.ny * gny + t.nz * gnz);
    d_sdf_grad[i * 3] = (gnx - t.nx * dot) * t.inv_norm;
    d_sdf_grad[i * 3 + 1] = (gny - t.ny * dot) * t.inv_norm;
    d_sdf_grad[i * 3 + 2] = (gnz - t.nz * dot) * t.inv_norm;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ds_part += __shfl_xor_sync(0xffffffffu, ds_part, o);
  __shared__ float ws[8];
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = ds_part;
  __syncthreads();
  if (threadIdx.x == 0) {
    float tot = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) tot += ws[w];
    if (tot != 0.f) atomicAdd(d_inv_s, tot);
  }
}

}  // namespace

extern "C" int nsr_neus_alpha_fwd(const float* sdf, const float* sdf_grad, const float* dirs, const float* dists,
                                  const float* inv_s, float cos_anneal_ratio, const float* cos_anneal_dev, float* alpha,
                                  float* normal, int64_t n, const int64_t* n_dev, void* stream) {
  NSR_REQUIRE(inv_s != nullptr, "nsr_neus_alpha_fwd: inv_s (device scalar) is NULL");
  if (n == 0) return 0;
  neus_alpha_fwd_kernel<<<nsr_blocks(n, 256), 256, 0, (cudaStream_t)stream>>>(sdf, sdf_grad, dirs, dists, inv_s,
                                                                               cos_anneal_ratio, cos_anneal_dev, alpha, normal, n, n_dev);
  NSR_CHECK_LAUNCH("nsr_neus_alpha_fwd");
  return 0;
}

extern "C" int nsr_neus_alpha_bwd(const float* sdf, const float* sdf_grad, const float* dirs, const float* dists,
                                  const float* inv_s, float cos_anneal_ratio, const float* cos_anneal_dev,
                                  const float* d_alpha, const float* d_normal, float* d_sdf, float* d_sdf_grad, float* d_inv_s, int64_t n,
                                  const int64_t* n_dev, void* stream) {
  NSR_REQUIRE(inv_s != nullptr && d_inv_s != nullptr, "nsr_neus_alpha_bwd: inv_s / d_inv_s is NULL");
  if (n == 0) return 0;
  neus_alpha_bwd_kernel<<<nsr_blocks(n, 256), 256, 0, (cudaStream_t)stream>>>(sdf, sdf_grad, dirs, dists, inv_s,
                                                                               cos_anneal_ratio, cos_anneal_dev, d_alpha, d_normal, d_sdf, d_sdf_grad, d_inv_s, n, n_dev);
  NSR_CHECK_LAUNCH("nsr_neus_alpha_bwd");
  return 0;
}
