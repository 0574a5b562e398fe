// Device pieces of the fused VolumeRadiance forward shared by radiance.cu (the per-sample kernels) and neus_render.cu (the per-ray
// NeuS eval renderer): the shared-memory weight layout, its staging, the output modes and the 16-row network pass.
#pragma once
#include "mlp_warp.cuh"

namespace {

constexpr int LD32 = 32 + NSR_LDW_PAD;  // 40
constexpr int W_OFF1 = 0;                     // [64][40]
constexpr int W_OFF2 = W_OFF1 + 64 * LD32;    // [64][72]
constexpr int W_OFF3 = W_OFF2 + 64 * NSR_LD64;  // [16][72]
constexpr int W_TOTAL = W_OFF3 + 16 * NSR_LD64;
constexpr int N_PARAMS = 64 * 32 + 64 * 64 + 16 * 64;
constexpr int N_BIAS = 64 + 64 + 16;  // VANILLA: b1 | b2 | b3 (padded to 16)

__device__ __forceinline__ void stage_weights(__half* smem, const __half* __restrict__ params) {
  nsr_stage_matrix(smem + W_OFF1, params, 64, 32, threadIdx.x, blockDim.x);
  nsr_stage_matrix(smem + W_OFF2, params + 64 * 32, 64, 64, threadIdx.x, blockDim.x);
  nsr_stage_matrix(smem + W_OFF3, params + 64 * 32 + 64 * 64, 16, 64, threadIdx.x, blockDim.x);
}

template <bool VANILLA>
__device__ __forceinline__ float out_value(float acc, int mode) {
  if (VANILLA) return mode == 0 ? acc : 1.f / (1.f + expf(-acc));  // fp32 network output; sigmoid as output / colour activation
  const float raw = __half2float(__float2half_rn(acc));  // the network emits fp16
  if (mode == 0) return raw;
  const float s = 1.f / (1.f + expf(-raw));
  return mode == 1 ? __half2float(__float2half_rn(s)) : s;  // 1: Sigmoid is the network's output activation (fp16), 2: applied in fp32 after
}

// accumulators of one 16-row tile start from zero (FullyFused: bias-free) or from the fp32 bias of their column
template <bool VANILLA, int NT>
__device__ __forceinline__ void init_acc(float (&acc)[1][NT][4], const float* bias_sm) {
  if (VANILLA) {
    const int c2 = (threadIdx.x & 3) * 2;
#pragma unroll
    for (int n = 0; n < NT; ++n) {
      const float b0 = bias_sm[n * 8 + c2], b1 = bias_sm[n * 8 + c2 + 1];
      acc[0][n][0] = b0, acc[0][n][1] = b1, acc[0][n][2] = b0, acc[0][n][3] = b1;
    }
  } else {
    nsr_zero_acc(acc);
  }
}

__device__ __forceinline__ void stage_bias(float* bias_sm, const float* __restrict__ bias) {
  for (int i = threadIdx.x; i < N_BIAS; i += blockDim.x) bias_sm[i] = bias[i];
}

// one warp's 16 input rows (X, rows r0 .. r0 + 15, [rows][LD32] fp16) -> the fp32 accumulators of the 3 (padded 16) outputs:
// lane (g, c) holds rows r0 + g (acc16[0][0][0..1]) and r0 + g + 8 (acc16[0][0][2..3]), columns 2c, 2c + 1
template <bool VANILLA>
__device__ __forceinline__ void radiance_rows16(float (&acc16)[1][2][4], const __half* X, int r0, const __half* smem, const float* bias_sm) {
  uint32_t a_in[1][2][4], a_h[1][4][4];
  float acc[1][8][4];
  nsr_load_afrag<1, 2>(a_in, X, LD32, r0);
  init_acc<VANILLA>(acc, bias_sm);
  nsr_gemm_w<1, 2, 8>(acc, a_in, smem + W_OFF1, LD32);
  nsr_acc_to_afrag<1, 8>(acc, a_h, NSR_ACT_RELU);
  init_acc<VANILLA>(acc, bias_sm + 64);
  nsr_gemm_w<1, 4, 8>(acc, a_h, smem + W_OFF2, NSR_LD64);
  nsr_acc_to_afrag<1, 8>(acc, a_h, NSR_ACT_RELU);
  init_acc<VANILLA>(acc16, bias_sm + 128);
  nsr_gemm_w<1, 4, 2>(acc16, a_h, smem + W_OFF3, NSR_LD64);
}

}  // namespace
