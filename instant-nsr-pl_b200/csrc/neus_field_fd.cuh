// Device pieces of the finite-difference NeuS SDF field shared by neus_field_fd.cu (the per-sample forward and backward kernels) and
// neus_render.cu (the per-ray eval renderer's finite-difference form): the fp32 weight staging, the unit-cube stencil queries in the
// torch path's operation order, the masked hash encoding and the 36 -> 64 -> n_out network evaluation on the CUDA cores.
// The math is described at the top of neus_field_fd.cu.  Namespace fd: neus_field.cuh and radiance.cuh define their own NOUTP and
// stage_weights.
#pragma once
#include "common.cuh"

namespace {
namespace fd {

constexpr int NIN = 35;     // 3 + 16 * 2
constexpr int NINP = 36;    // padded row length (float4 loads)
constexpr int NH = 64;
constexpr int NOUTP = 16;   // padded output width

struct FdW {  // shared-memory weights (floats)
  float W1[NH][NINP];       // [k][j]
  float W2T[NH][NOUTP];     // [k][o] = W2[o][k]
  float b1[NH];
  float b2[NOUTP];
};

__device__ __forceinline__ void stage_weights(FdW& w, const float* __restrict__ W1, const float* __restrict__ b1, const float* __restrict__ W2,
                                              const float* __restrict__ b2, int n_out) {
  for (int i = threadIdx.x; i < NH * NINP; i += blockDim.x) {
    const int k = i / NINP, j = i % NINP;
    w.W1[k][j] = j < NIN ? W1[k * NIN + j] : 0.f;
  }
  for (int i = threadIdx.x; i < NH * NOUTP; i += blockDim.x) {
    const int k = i / NOUTP, o = i % NOUTP;
    w.W2T[k][o] = o < n_out ? W2[o * NH + k] : 0.f;
  }
  for (int i = threadIdx.x; i < NH; i += blockDim.x) w.b1[i] = b1[i];
  for (int i = threadIdx.x; i < NOUTP; i += blockDim.x) w.b2[i] = i < n_out ? b2[i] : 0.f;
}

__device__ __forceinline__ float softplus100(float z, float& s) {
  const float bz = 100.f * z;
  s = 1.f / (1.f + __expf(-bz));
  return bz > 20.f ? z : log1pf(__expf(bz)) * 0.01f;  // torch.nn.Softplus(beta=100, threshold=20)
}

// unit-cube query of stencil point k (0 = centre, 1..6 = +x, -x, +y, -y, +z, -z, anything else = centre) in the torch path's fp32
// operation order: (p + offs).clamp(-r, r), then (q - (-r)) / (r - (-r)) with a true division
__device__ __forceinline__ void stencil_query(float px, float py, float pz, int k, float eps, float r, float& x, float& y, float& z) {
  const float two_r = 2.f * r;
  if (k >= 1 && k <= 6) {
    const int a = (k - 1) >> 1;
    const float d = ((k - 1) & 1) ? -eps : eps;
    px = fminf(fmaxf(__fadd_rn(px, a == 0 ? d : 0.f), -r), r);
    py = fminf(fmaxf(__fadd_rn(py, a == 1 ? d : 0.f), -r), r);
    pz = fminf(fmaxf(__fadd_rn(pz, a == 2 ? d : 0.f), -r), r);
  }
  x = __fdiv_rn(__fadd_rn(px, r), two_r);
  y = __fdiv_rn(__fadd_rn(py, r), two_r);
  z = __fdiv_rn(__fadd_rn(pz, r), two_r);
}

// e = [2 x - 1 | features of levels < n_active | 0 ...] (35 live entries, e[35] = 0)
__device__ __forceinline__ void encode(const nsr_grid_t& g, const __half2* __restrict__ table, float x, float y, float z, int n_active,
                                       float (&e)[NINP]) {
  e[0] = 2.f * x - 1.f;
  e[1] = 2.f * y - 1.f;
  e[2] = 2.f * z - 1.f;
#pragma unroll
  for (int j = 3; j < NINP; ++j) e[j] = 0.f;
#pragma unroll
  for (int l = 0; l < 16; ++l) {
    if (l >= n_active) break;
    const LevelInfo li = nsr_level(g, l);
    uint32_t cx, cy, cz, idx[8];
    float fx, fy, fz;
    nsr_pos_fract(x, li.scale, cx, fx);
    nsr_pos_fract(y, li.scale, cy, fy);
    nsr_pos_fract(z, li.scale, cz, fz);
    nsr_corner_indices(li, cx, cy, cz, idx);
    float a0 = 0.f, a1 = 0.f;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const float2 v = nsr_ld_table(table, idx[c]);
      const float w = nsr_corner_weight(c, fx, fy, fz);
      a0 = fmaf(w, v.x, a0);
      a1 = fmaf(w, v.y, a1);
    }
    e[3 + 2 * l] = a0;
    e[4 + 2 * l] = a1;
  }
}

// out[o] = (W2 softplus100(W1 e + b1) + b2)[o] for o < NO: NO = NOUTP gives every (padded) output, NO = 1 the SDF alone.  Each
// output's sums run in the same order for either NO, so out[0] is the same value.
template <int NO>
__device__ __forceinline__ void mlp_eval(const FdW& w, const float (&e)[NINP], float (&out)[NO]) {
  static_assert(NO == NOUTP || NO == 1, "all outputs or the SDF alone");
#pragma unroll
  for (int o = 0; o < NO; ++o) out[o] = w.b2[o];
#pragma unroll 2
  for (int h = 0; h < NH; ++h) {
    float row[NINP];
#pragma unroll
    for (int v = 0; v < NINP / 4; ++v) *reinterpret_cast<float4*>(&row[4 * v]) = *reinterpret_cast<const float4*>(&w.W1[h][4 * v]);
    float zk = w.b1[h];
#pragma unroll
    for (int j = 0; j < NINP; ++j) zk = fmaf(row[j], e[j], zk);
    float s;
    const float hk = softplus100(zk, s);
    if (NO == NOUTP) {
      float w2[NOUTP];
#pragma unroll
      for (int v = 0; v < NOUTP / 4; ++v) *reinterpret_cast<float4*>(&w2[4 * v]) = *reinterpret_cast<const float4*>(&w.W2T[h][4 * v]);
#pragma unroll
      for (int o = 0; o < NO; ++o) out[o] = fmaf(w2[o], hk, out[o]);
    } else {
      out[0] = fmaf(w.W2T[h][0], hk, out[0]);
    }
  }
}

}  // namespace fd
}  // namespace
