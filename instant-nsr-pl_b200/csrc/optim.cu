// Fused AdamW over a flat fp32 parameter vector (SURVEY 8f-2; the reference builds `torch.optim.AdamW(lr 1e-2, betas (0.9, 0.99),
// eps 1e-15)` in systems/utils.py:314-325 from configs/nerf-blender.yaml:74-79 and wraps it in AMP's GradScaler).
// One pass over the 12.6 M-entry hash table does what the reference spreads over ~8 table-sized passes: gradient un-scaling,
// the non-finite check's skip, decoupled weight decay, both moment updates, the parameter update AND the fp16 copy the
// kernels read (tcnn re-casts the whole vector in every forward).  HBM-bound: 16 B read + 12 B (+2 B fp16) written per
// parameter.  Arithmetic follows torch's single-tensor AdamW step by step (lerp for exp_avg, sqrt(v)/sqrt(bc2) + eps).
#include "common.cuh"
#include <math.h>

namespace {

struct AdamConsts {
  float decay;      // 1 - lr * weight_decay
  float beta1, beta2, eps;
  float step_size;  // lr / (1 - beta1^t)
  float bc2_sqrt;   // sqrt(1 - beta2^t)
  float inv_scale;  // gradients are multiplied by this first (1 / GradScaler scale)
  float lr, weight_decay;
};

__device__ __forceinline__ void adam_one(float& p, float g, float& m, float& v, const AdamConsts& c) {
  g *= c.inv_scale;
  p *= c.decay;
  m = m + (g - m) * (1.f - c.beta1);
  v = v * c.beta2 + (1.f - c.beta2) * g * g;
  const float denom = sqrtf(v) / c.bc2_sqrt + c.eps;
  p -= c.step_size * (m / denom);
}

// U float4 groups per thread per iteration (all loads issued before the first use), grid-stride over U * blockDim chunks.  nsr_adamw_step
// launches U = 1 with one CTA per chunk: U = 2 / 4 and grids capped at 8 or 16 CTAs per SM were not faster on the H100.
template <int U>
__global__ void __launch_bounds__(256) adamw_kernel(AdamConsts c, float* __restrict__ params, const float* __restrict__ grads,
                                                    float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq,
                                                    __half* __restrict__ params_half, const float* __restrict__ dev_lr_step,
                                                    const float* __restrict__ found_inf, int64_t n) {
  if (found_inf != nullptr && *found_inf != 0.f) return;  // GradScaler semantics: skip the whole step
  if (dev_lr_step != nullptr) {  // capturable mode: learning rate and step number live on the device
    const float lr = dev_lr_step[0], t = dev_lr_step[1];
    c.decay = 1.f - lr * c.weight_decay;
    c.step_size = lr / (1.f - powf(c.beta1, t));
    c.bc2_sqrt = sqrtf(1.f - powf(c.beta2, t));
  }
  const int64_t n4 = n >> 2;
  const int64_t chunk = (int64_t)blockDim.x * U;
  for (int64_t base = blockIdx.x * chunk; base < n4; base += (int64_t)gridDim.x * chunk) {
    float4 p[U], g[U], m[U], v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = base + u * blockDim.x + threadIdx.x;
      if (i < n4) {
        p[u] = reinterpret_cast<float4*>(params)[i];
        g[u] = __ldcs(reinterpret_cast<const float4*>(grads) + i);
        m[u] = __ldcs(reinterpret_cast<float4*>(exp_avg) + i);
        v[u] = __ldcs(reinterpret_cast<float4*>(exp_avg_sq) + i);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = base + u * blockDim.x + threadIdx.x;
      if (i < n4) {
        adam_one(p[u].x, g[u].x, m[u].x, v[u].x, c);
        adam_one(p[u].y, g[u].y, m[u].y, v[u].y, c);
        adam_one(p[u].z, g[u].z, m[u].z, v[u].z, c);
        adam_one(p[u].w, g[u].w, m[u].w, v[u].w, c);
        reinterpret_cast<float4*>(params)[i] = p[u];
        __stcs(reinterpret_cast<float4*>(exp_avg) + i, m[u]);
        __stcs(reinterpret_cast<float4*>(exp_avg_sq) + i, v[u]);
        if (params_half != nullptr) {
          uint2 h;
          h.x = nsr_pack_h2(p[u].x, p[u].y);
          h.y = nsr_pack_h2(p[u].z, p[u].w);
          reinterpret_cast<uint2*>(params_half)[i] = h;
        }
      }
    }
  }
  // tail (n not a multiple of 4)
  const int64_t t = (n4 << 2) + blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t < n) {
    float p = params[t], m = exp_avg[t], v = exp_avg_sq[t];
    adam_one(p, grads[t], m, v, c);
    params[t] = p;
    exp_avg[t] = m;
    exp_avg_sq[t] = v;
    if (params_half != nullptr) params_half[t] = __float2half_rn(p);
  }
}

// found_inf[0] = 1 if any gradient entry is inf / nan (torch._amp_foreach_non_finite_check_and_unscale_, check only)
__global__ void __launch_bounds__(256) nonfinite_kernel(const float* __restrict__ grads, float* __restrict__ found_inf, int64_t n) {
  bool bad = false;
  const int64_t n4 = n >> 2;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 g = reinterpret_cast<const float4*>(grads)[i];
    bad |= !(isfinite(g.x) && isfinite(g.y) && isfinite(g.z) && isfinite(g.w));
  }
  const int64_t t = (n4 << 2) + blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t < n) bad |= !isfinite(grads[t]);
  if (__syncthreads_or(bad) && threadIdx.x == 0) *found_inf = 1.f;
}

int stream_grid(int64_t n4) {
  const int64_t want = (n4 + 255) / 256;
  const int64_t cap = (int64_t)nsr_sm_count() * 8;  // 8 x 256 threads = full occupancy; grid-stride beyond that
  return (int)max((int64_t)1, min(want, cap));
}

}  // namespace

extern "C" int nsr_adamw_step(const nsr_adamw_t* h, float* params, const float* grads, float* exp_avg, float* exp_avg_sq,
                              void* params_half, const float* dev_lr_step, const float* found_inf, int64_t n, void* stream) {
  NSR_REQUIRE(h != nullptr, "nsr_adamw_step: hyper-parameter struct is NULL");
  NSR_REQUIRE(h->step >= 1 || dev_lr_step != nullptr, "nsr_adamw_step: step must be >= 1 (1-based number of this update)");
  NSR_REQUIRE(h->beta1 >= 0.f && h->beta1 < 1.f && h->beta2 >= 0.f && h->beta2 < 1.f, "nsr_adamw_step: betas must be in [0, 1)");
  NSR_REQUIRE(((uintptr_t)params | (uintptr_t)grads | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq) % 16 == 0 &&
                  (uintptr_t)params_half % 8 == 0,
              "nsr_adamw_step: buffers must be 16-byte aligned (fp16 copy: 8-byte)");
  if (n == 0) return 0;
  AdamConsts c;
  const double t = h->step >= 1 ? (double)h->step : 1.0;
  // torch computes the bias corrections and step size in Python doubles, then applies them as fp32 scalars
  c.decay = (float)(1.0 - (double)h->lr * (double)h->weight_decay);
  c.beta1 = h->beta1;
  c.beta2 = h->beta2;
  c.eps = h->eps;
  c.step_size = (float)((double)h->lr / (1.0 - pow((double)h->beta1, t)));
  c.bc2_sqrt = (float)sqrt(1.0 - pow((double)h->beta2, t));
  c.inv_scale = h->inv_grad_scale;
  c.lr = h->lr;
  c.weight_decay = h->weight_decay;
  const int grid = (int)max((int64_t)1, ((n >> 2) + 255) / 256);   // one CTA per 1024-float chunk
  adamw_kernel<1><<<grid, 256, 0, (cudaStream_t)stream>>>(c, params, grads, exp_avg, exp_avg_sq, (__half*)params_half, dev_lr_step, found_inf, n);
  NSR_CHECK_LAUNCH("nsr_adamw_step");
  return 0;
}

extern "C" int nsr_grad_nonfinite(const float* grads, float* found_inf, int64_t n, void* stream) {
  NSR_REQUIRE(found_inf != nullptr, "nsr_grad_nonfinite: found_inf is NULL");
  NSR_REQUIRE((uintptr_t)grads % 16 == 0, "nsr_grad_nonfinite: gradient buffer must be 16-byte aligned");
  if (n == 0) return 0;
  nonfinite_kernel<<<stream_grid(n >> 2), 256, 0, (cudaStream_t)stream>>>(grads, found_inf, n);
  NSR_CHECK_LAUNCH("nsr_grad_nonfinite");
  return 0;
}
