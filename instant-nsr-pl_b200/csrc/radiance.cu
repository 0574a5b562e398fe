// VolumeRadiance as one kernel per direction (models/texture.py:23-30): cat[feature | SH4(dir) | extra (NeuS: normal)] -> FullyFused
// 64-wide MLP with two hidden layers -> 3 colours (+ colour activation).  Replaces: (d+1)/2, SH kernel, cat, fp16 cast, MLP kernel,
// float cast, sigmoid -- and their ~15 autograd kernels -- of the composed path.  Tensor-core math as in mlp_warp.cuh; the
// backward recomputes the activations, chains the dgrads in registers and keeps the three weight-gradient GEMMs in register
// accumulators for the whole kernel (one atomicAdd per weight per CTA).
// VANILLA = true: the same kernels for the reference's VanillaMLP colour networks (configs/neus-dtu.yaml:58-70,93-105;
// models/network_utils.py:95-139: ReLU, 64 wide, two hidden layers, BIASES, fp32 output): accumulators start from the fp32 bias,
// the output is not rounded to fp16, the input may be narrower than 32 (zero padded: background texture 8 + 16 = 24) and the
// backward also emits the three bias gradients (column sums of the pre-activation gradient tiles).
#include "radiance.cuh"

namespace {

// one warp fills its 16 rows of the [rows][40] input tile: 2 lanes per row
__device__ __forceinline__ void stage_inputs(__half* X, int r0, int64_t row0, int64_t n, const nsr_radiance_t& P, const float* __restrict__ feat,
                                             const float* __restrict__ dirs,
                                             const float* __restrict__ extra) {
  const int lane = threadIdx.x & 31, r = lane >> 1, part = lane & 1;
  const int64_t i = row0 + r0 + r;
  __half* x = X + (size_t)(r0 + r) * LD32;
  if (i >= n) {
    for (int c = part * 16; c < part * 16 + 16; ++c) x[c] = __float2half_rn(0.f);
    return;
  }
  if (part == 0) {
    for (int c = 0; c < P.n_feat; ++c) x[c] = __float2half_rn(feat[i * P.n_feat + c]);
    for (int c = 0; c < P.n_extra; ++c) x[P.n_feat + 16 + c] = __float2half_rn(extra[i * P.n_extra + c]);
    for (int c = P.n_feat + 16 + P.n_extra; c < 32; ++c) x[c] = __float2half_rn(0.f);  // narrower than 32: zero padding
  } else {
    float s[16];
    nsr_sh4(dirs[i * 3], dirs[i * 3 + 1], dirs[i * 3 + 2], s);
#pragma unroll
    for (int c = 0; c < 16; ++c) x[P.n_feat + c] = __float2half_rn(s[c]);
  }
}

constexpr int kFwdWarps = 4;
constexpr int kFwdRows = kFwdWarps * 16;
constexpr size_t kFwdSmemHalves = (size_t)(W_TOTAL + kFwdRows * LD32);
template <bool VANILLA>
constexpr size_t fwd_smem() { return kFwdSmemHalves * sizeof(__half) + (VANILLA ? N_BIAS * sizeof(float) : 0); }

template <bool VANILLA>
__global__ void __launch_bounds__(kFwdWarps * 32) radiance_fwd_kernel(const __grid_constant__ nsr_radiance_t P, const float* __restrict__ feat,
                                                                      const float* __restrict__ dirs,
                                                                      const float* __restrict__ extra, const __half* __restrict__ params,
                                                                      const float* __restrict__ bias,
                                                                      float* __restrict__ rgb, int64_t n_cap, const int64_t* __restrict__ n_dev) {
  const int64_t n = n_dev ? min(*n_dev, n_cap) : n_cap;
  extern __shared__ __align__(16) __half smem[];
  __half* X = smem + W_TOTAL;
  float* bias_sm = reinterpret_cast<float*>(smem + kFwdSmemHalves);  // VANILLA only
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, c = lane & 3, r0 = warp * 16;
  stage_weights(smem, params);
  if (VANILLA) stage_bias(bias_sm, bias);
  __syncthreads();
  const int64_t n_tiles = (n + kFwdRows - 1) / kFwdRows;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t row0 = tile * kFwdRows;
    __syncwarp();
    stage_inputs(X, r0, row0, n, P, feat, dirs, extra);
    __syncwarp();
    float acc16[1][2][4];
    radiance_rows16<VANILLA>(acc16, X, r0, smem, bias_sm);
    if (c < 2) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int64_t i = row0 + r0 + g + hh * 8;
        if (i < n) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = c * 2 + e;
            if (col < 3) rgb[i * 3 + col] = out_value<VANILLA>(acc16[0][0][hh * 2 + e], P.act_mode);
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------- backward
constexpr int kWarps = 4;
constexpr int kRows = kWarps * 16;
constexpr int T_X = 0;                          // [64][40] input
constexpr int T_G1 = T_X + kRows * LD32;        // [64][72] hidden 1 (post ReLU)
constexpr int T_G2 = T_G1 + kRows * NSR_LD64;   // [64][72] hidden 2
constexpr int T_D3 = T_G2 + kRows * NSR_LD64;   // [64][24] d(raw)
constexpr int T_DG2 = T_D3 + kRows * 24;        // [64][72]
constexpr int T_DG1 = T_DG2 + kRows * NSR_LD64; // [64][72]
constexpr int T_TOTAL = T_DG1 + kRows * NSR_LD64;
constexpr size_t kBwdSmemHalves = (size_t)(W_TOTAL + T_TOTAL);
template <bool VANILLA>
constexpr size_t bwd_smem() { return kBwdSmemHalves * sizeof(__half) + (VANILLA ? N_BIAS * sizeof(float) : 0); }
constexpr int kSlots = 28 / kWarps;  // 8 + 16 + 4 pair-tiles

struct WgradTile {
  int dy_off, ldy, x_off, ldx, m0, n0, base, in_dim;
};
__device__ __forceinline__ WgradTile wgrad_tile(int t) {
  WgradTile w;
  if (t < 8) {
    w = {T_DG1, NSR_LD64, T_X, LD32, (t / 2) * 16, (t % 2) * 16, 0, 32};
  } else if (t < 24) {
    const int u = t - 8;
    w = {T_DG2, NSR_LD64, T_G1, NSR_LD64, (u / 4) * 16, (u % 4) * 16, 64 * 32, 64};
  } else {
    w = {T_D3, 24, T_G2, NSR_LD64, 0, (t - 24) * 16, 64 * 32 + 64 * 64, 64};
  }
  return w;
}

__device__ __forceinline__ void relu_mask_pack(const float (&acc)[1][8][4], const uint32_t (&post)[1][4][4], uint32_t (&out)[1][4][4]) {
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const __half2 hv = *reinterpret_cast<const __half2*>(&post[0][k][j]);
      const int nt = 2 * k + (j >> 1), i0 = (j & 1) * 2;
      out[0][k][j] = nsr_pack_h2(__low2float(hv) > 0.f ? acc[0][nt][i0] : 0.f, __high2float(hv) > 0.f ? acc[0][nt][i0 + 1] : 0.f);
    }
}

template <bool VANILLA>
__global__ void __launch_bounds__(kWarps * 32, 2) radiance_bwd_kernel(const __grid_constant__ nsr_radiance_t P, const float* __restrict__ feat,
                                                                      const float* __restrict__ dirs,
                                                                      const float* __restrict__ extra, const __half* __restrict__ params,
                                                                      const float* __restrict__ bias,
                                                                      const float* __restrict__ d_rgb, float loss_scale,
                                                                      const float* __restrict__ amax_ptr, float* __restrict__ d_feat,
                                                                      float* __restrict__ d_extra, float* __restrict__ grad_params,
                                                                      float* __restrict__ grad_bias, int64_t n_cap,
                                                                      const int64_t* __restrict__ n_dev) {
  const int64_t n = n_dev ? min(*n_dev, n_cap) : n_cap;
  extern __shared__ __align__(16) __half smem[];
  __half* T = smem + W_TOTAL;
  float* bias_sm = reinterpret_cast<float*>(smem + kBwdSmemHalves);  // VANILLA only
  float bsum = 0.f, bsum3 = 0.f;  // VANILLA: this thread's column of d(pre-activation 1 | 2) and of d(raw), summed over all tiles
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, c = lane & 3, r0 = warp * 16;
  if (loss_scale <= 0.f) {  // automatic: bring the largest incoming gradient to ~2^8
    const float amax = fmaxf(__ldg(amax_ptr), 1e-30f);
    loss_scale = exp2f(fminf(fmaxf(floorf(log2f(256.f / amax)), -24.f), 60.f));
  }
  const float inv_scale = 1.f / loss_scale;
  stage_weights(smem, params);
  if (VANILLA) stage_bias(bias_sm, bias);
  float wacc[kSlots][2][4];
#pragma unroll
  for (int s = 0; s < kSlots; ++s)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int i = 0; i < 4; ++i) wacc[s][j][i] = 0.f;

  const int64_t n_tiles = (n + kRows - 1) / kRows;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t row0 = tile * kRows;
    __syncthreads();  // previous tile's wgrad has consumed the smem tiles (first iteration: weights are staged)
    stage_inputs(T + T_X, r0, row0, n, P, feat, dirs, extra);
    __syncwarp();
    uint32_t a_in[1][2][4], a_g1[1][4][4], a_g2[1][4][4];
    float acc[1][8][4], acc16[1][2][4];
    nsr_load_afrag<1, 2>(a_in, T + T_X, LD32, r0);
    init_acc<VANILLA>(acc, bias_sm);
    nsr_gemm_w<1, 2, 8>(acc, a_in, smem + W_OFF1, LD32);
    nsr_acc_to_afrag<1, 8>(acc, a_g1, NSR_ACT_RELU);
    nsr_store_afrag<1, 4>(a_g1, T + T_G1, NSR_LD64, r0);
    init_acc<VANILLA>(acc, bias_sm + 64);
    nsr_gemm_w<1, 4, 8>(acc, a_g1, smem + W_OFF2, NSR_LD64);
    nsr_acc_to_afrag<1, 8>(acc, a_g2, NSR_ACT_RELU);
    nsr_store_afrag<1, 4>(a_g2, T + T_G2, NSR_LD64, r0);
    init_acc<VANILLA>(acc16, bias_sm + 128);
    nsr_gemm_w<1, 4, 2>(acc16, a_g2, smem + W_OFF3, NSR_LD64);
    // d(raw) = d_rgb * act'(raw); columns 0..2 only
    const int64_t ia = row0 + r0 + g, ib = ia + 8;
    uint32_t a_d3[1][1][4];
    {
      float dp[4] = {0.f, 0.f, 0.f, 0.f};
      if (c < 2) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int64_t i = hh ? ib : ia;
          if (i < n) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int col = c * 2 + e;
              if (col < 3) {
                float d = d_rgb[i * 3 + col] * loss_scale;
                if (P.act_mode != 0) {
                  const float raw = VANILLA ? acc16[0][0][hh * 2 + e] : __half2float(__float2half_rn(acc16[0][0][hh * 2 + e]));
                  const float s = 1.f / (1.f + expf(-raw));
                  d *= s * (1.f - s);
                }
                dp[hh * 2 + e] = d;
              }
            }
          }
        }
      }
      a_d3[0][0][0] = nsr_pack_h2(dp[0], dp[1]);
      a_d3[0][0][1] = nsr_pack_h2(dp[2], dp[3]);
      a_d3[0][0][2] = 0u;
      a_d3[0][0][3] = 0u;
      nsr_store_afrag<1, 1>(a_d3, T + T_D3, 24, r0);
    }
    uint32_t a_d[1][4][4];
    nsr_zero_acc(acc);
    nsr_gemm_wt<1, 1, 8>(acc, a_d3, smem + W_OFF3, NSR_LD64);
    relu_mask_pack(acc, a_g2, a_d);
    nsr_store_afrag<1, 4>(a_d, T + T_DG2, NSR_LD64, r0);
    nsr_zero_acc(acc);
    nsr_gemm_wt<1, 4, 8>(acc, a_d, smem + W_OFF2, NSR_LD64);
    relu_mask_pack(acc, a_g1, a_d);
    nsr_store_afrag<1, 4>(a_d, T + T_DG1, NSR_LD64, r0);
    float accI[1][4][4];
    nsr_zero_acc(accI);
    nsr_gemm_wt<1, 4, 4>(accI, a_d, smem + W_OFF1, LD32);
    // input gradients straight from the accumulator layout: rows (g, g+8), columns nt*8 + c*2 + {0,1}
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int64_t i = hh ? ib : ia;
      if (i < n) {
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = nt * 8 + c * 2 + e;
            const float v = accI[0][nt][hh * 2 + e] * inv_scale;
            if (col < P.n_feat) {
              if (d_feat) d_feat[i * P.n_feat + col] = v;
            } else if (col >= P.n_feat + 16 && col < P.n_feat + 16 + P.n_extra) {
              if (d_extra) d_extra[i * P.n_extra + (col - P.n_feat - 16)] = v;
            }
          }
      }
    }
    __syncthreads();
#pragma unroll
    for (int s = 0; s < kSlots; ++s) {
      const WgradTile w = wgrad_tile(warp + s * kWarps);
      nsr_wgrad_tile(wacc[s][0], wacc[s][1], T + w.dy_off, w.ldy, w.m0, T + w.x_off, w.ldx, w.n0, kRows);
    }
    if (VANILLA) {  // bias gradients: column sums of the three pre-activation gradient tiles (rows beyond n hold zeros)
      const __half* Dt = T + (threadIdx.x < 64 ? T_DG1 : T_DG2) + (threadIdx.x & 63);
      float s12 = 0.f;
#pragma unroll 8
      for (int r = 0; r < kRows; ++r) s12 += __half2float(Dt[(size_t)r * NSR_LD64]);
      bsum += s12;
      if (threadIdx.x < 16) {
        float s3 = 0.f;
#pragma unroll 8
        for (int r = 0; r < kRows; ++r) s3 += __half2float(T[T_D3 + r * 24 + threadIdx.x]);
        bsum3 += s3;
      }
    }
  }
  if (VANILLA) {
    if (bsum != 0.f) atomicAdd(grad_bias + threadIdx.x, bsum * inv_scale);  // threads 0..63: b1, 64..127: b2
    if (threadIdx.x < 16 && bsum3 != 0.f) atomicAdd(grad_bias + 128 + threadIdx.x, bsum3 * inv_scale);
  }
#pragma unroll
  for (int s = 0; s < kSlots; ++s) {
    const WgradTile w = wgrad_tile(warp + s * kWarps);
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int o = w.m0 + g + ((i >> 1) << 3), ii = w.n0 + j * 8 + c * 2 + (i & 1);
        const float v = wacc[s][j][i] * inv_scale;
        if (v != 0.f) atomicAdd(grad_params + w.base + (size_t)o * w.in_dim + ii, v);
      }
  }
}

int check_desc(const nsr_radiance_t* p, const char* who, bool vanilla) {
  if (p == nullptr) {
    nsr_set_error("%s: descriptor is NULL", who);
    return 1;
  }
  const int width = p->n_feat + 16 + p->n_extra;
  if (p->n_feat < 1 || p->n_extra < 0 || (vanilla ? width > 32 : width != 32)) {
    nsr_set_error("%s: fused radiance needs n_feat + 16 (SH degree 4) + n_extra %s 32, got %d + 16 + %d", who, vanilla ? "<=" : "==",
                  p->n_feat, p->n_extra);
    return 1;
  }
  if (p->act_mode < 0 || p->act_mode > 2) {
    nsr_set_error("%s: act_mode must be 0 (none), 1 (network Sigmoid) or 2 (fp32 sigmoid after the network)", who);
    return 1;
  }
  return 0;
}

template <bool VANILLA>
int launch_fwd(const char* who, const nsr_radiance_t* p, const float* feat, const float* dirs, const float* extra, const void* params_h,
               const float* bias, float* rgb, int64_t n, const int64_t* n_dev, void* stream) {
  if (check_desc(p, who, VANILLA)) return 1;
  if (n == 0) return 0;
  NSR_REQUIRE(p->n_extra == 0 || extra != nullptr, "%s: extra input is NULL", who);
  NSR_REQUIRE(!VANILLA || bias != nullptr, "%s: bias is NULL", who);
  static thread_local bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(radiance_fwd_kernel<VANILLA>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fwd_smem<VANILLA>());
    attr_set = true;
  }
  const int64_t tiles = (n + kFwdRows - 1) / kFwdRows;
  const int grid = (int)min((int64_t)nsr_sm_count() * 6, tiles);
  radiance_fwd_kernel<VANILLA><<<grid, kFwdWarps * 32, fwd_smem<VANILLA>(), (cudaStream_t)stream>>>(
      *p, feat, dirs, extra, (const __half*)params_h, bias, rgb, n, n_dev);
  NSR_CHECK_LAUNCH(who);
  return 0;
}

template <bool VANILLA>
int launch_bwd(const char* who, const nsr_radiance_t* p, const float* feat, const float* dirs, const float* extra, const void* params_h,
               const float* bias, const float* d_rgb, float loss_scale, const float* amax, float* d_feat, float* d_extra,
               float* grad_params, float* grad_bias, int64_t n, const int64_t* n_dev, void* stream) {
  if (check_desc(p, who, VANILLA)) return 1;
  if (n == 0) return 0;
  NSR_REQUIRE(p->n_extra == 0 || extra != nullptr, "%s: extra input is NULL", who);
  NSR_REQUIRE(loss_scale > 0.f || amax != nullptr, "%s: loss_scale <= 0 (automatic) needs the amax pointer", who);
  NSR_REQUIRE(grad_params != nullptr, "%s: grad_params is NULL", who);
  NSR_REQUIRE(!VANILLA || (bias != nullptr && grad_bias != nullptr), "%s: bias / grad_bias is NULL", who);
  static thread_local bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(radiance_bwd_kernel<VANILLA>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bwd_smem<VANILLA>());
    if (e != cudaSuccess) {
      nsr_set_error("%s: cannot reserve %zu B shared memory: %s", who, bwd_smem<VANILLA>(), cudaGetErrorString(e));
      return 2;
    }
    attr_set = true;
  }
  const int64_t tiles = (n + kRows - 1) / kRows;
  const int grid = (int)min((int64_t)nsr_sm_count() * 2, tiles);
  radiance_bwd_kernel<VANILLA><<<grid, kWarps * 32, bwd_smem<VANILLA>(), (cudaStream_t)stream>>>(
      *p, feat, dirs, extra, (const __half*)params_h, bias, d_rgb, loss_scale, amax, d_feat, d_extra, grad_params, grad_bias, n, n_dev);
  NSR_CHECK_LAUNCH(who);
  return 0;
}

}  // namespace

extern "C" int nsr_radiance_fwd(const nsr_radiance_t* p, const float* feat, const float* dirs,
                                const float* extra, const void* params_h, float* rgb, int64_t n, const int64_t* n_dev, void* stream) {
  return launch_fwd<false>("nsr_radiance_fwd", p, feat, dirs, extra, params_h, nullptr, rgb, n, n_dev, stream);
}

extern "C" int nsr_radiance_bwd(const nsr_radiance_t* p, const float* feat, const float* dirs,
                                const float* extra, const void* params_h, const float* d_rgb, float loss_scale, const float* amax,
                                float* d_feat, float* d_extra, float* grad_params, int64_t n, const int64_t* n_dev, void* stream) {
  return launch_bwd<false>("nsr_radiance_bwd", p, feat, dirs, extra, params_h, nullptr, d_rgb, loss_scale, amax, d_feat, d_extra, grad_params,
                           nullptr, n, n_dev, stream);
}

extern "C" int nsr_radiance_vanilla_fwd(const nsr_radiance_t* p, const float* feat, const float* dirs, const float* extra,
                                        const void* weights_h, const float* bias, float* rgb, int64_t n, const int64_t* n_dev,
                                        void* stream) {
  return launch_fwd<true>("nsr_radiance_vanilla_fwd", p, feat, dirs, extra, weights_h, bias, rgb, n, n_dev, stream);
}

extern "C" int nsr_radiance_vanilla_bwd(const nsr_radiance_t* p, const float* feat, const float* dirs, const float* extra,
                                        const void* weights_h, const float* bias, const float* d_rgb, float loss_scale, const float* amax,
                                        float* d_feat, float* d_extra, float* grad_weights, float* grad_bias, int64_t n,
                                        const int64_t* n_dev, void* stream) {
  return launch_bwd<true>("nsr_radiance_vanilla_bwd", p, feat, dirs, extra, weights_h, bias, d_rgb, loss_scale, amax, d_feat, d_extra,
                          grad_weights, grad_bias, n, n_dev, stream);
}
