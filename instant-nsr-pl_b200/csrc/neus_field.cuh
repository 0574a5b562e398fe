// Device pieces of the fused NeuS SDF field forward shared by neus_field.cu (the per-sample field kernels) and neus_render.cu (the
// per-ray eval renderer): the hash gathers, the split-fp16 tensor-core network over 32 samples of a warp and the analytic normal.
// The math is described at the top of neus_field.cu.
#pragma once
#include "mlp_warp.cuh"

namespace {

constexpr int NIN = 35;     // 3 + 16 * 2
constexpr int NINP = 36;    // padded row length (float4 loads)
constexpr int NH = 64;
constexpr int NOUTP = 16;   // padded output width
constexpr int kNeusTcWarps = 4;   // warps of a tensor-core forward CTA (per-warp encoding tiles in NeusTcSmem)

__device__ __forceinline__ float softplus100(float z, float& s) {
  const float bz = 100.f * z;
  s = 1.f / (1.f + __expf(-bz));
  return bz > 20.f ? z : log1pf(__expf(bz)) * 0.01f;  // torch.nn.Softplus(beta=100, threshold=20)
}

// MASK: hash levels >= n_active contribute 0 (ProgressiveBandHashGrid: the level mask multiplies the features, so a masked level's
// features, Jacobian and table gradient are all zero).  The kernels read n_active on the device (uniform per CTA), so a captured graph
// follows the schedule; masked levels are neither gathered nor scattered.
__device__ __forceinline__ int load_n_active(const float* __restrict__ n_active) {
  return (int)fminf(fmaxf(__ldg(n_active), 0.f), 16.f);   // NaN -> 0
}

// gather: e[3..34] (features) and optionally qb[3..34] = J gx (directional derivative of every feature along gx); with MASK the
// columns of levels >= n_active are written as 0 (the tensor-core forward aliases q onto the encoding rows: no stale values)
template <bool WITH_QB, bool MASK = false>
__device__ __forceinline__ void gather_enc(const nsr_grid_t& g, const __half2* __restrict__ table, float x, float y, float z, float gx0,
                                           float gx1, float gx2, float (&e)[NINP], float (&qb)[NINP], int n_active = 16) {
#pragma unroll
  for (int l = 0; l < 16; ++l) {
    if (MASK && l >= n_active) {
      e[3 + 2 * l] = e[4 + 2 * l] = 0.f;
      if (WITH_QB) qb[3 + 2 * l] = qb[4 + 2 * l] = 0.f;
      continue;
    }
    const LevelInfo li = nsr_level(g, l);
    uint32_t cx, cy, cz, idx[8];
    float fx, fy, fz;
    nsr_pos_fract(x, li.scale, cx, fx);
    nsr_pos_fract(y, li.scale, cy, fy);
    nsr_pos_fract(z, li.scale, cz, fz);
    nsr_corner_indices(li, cx, cy, cz, idx);
    float a0 = 0.f, a1 = 0.f, d0 = 0.f, d1 = 0.f;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const float2 v = nsr_ld_table(table, idx[c]);
      const float w = nsr_corner_weight(c, fx, fy, fz);
      a0 = fmaf(w, v.x, a0);
      a1 = fmaf(w, v.y, a1);
      if (WITH_QB) {
        const float dw = gx0 * nsr_corner_dweight(c, 0, fx, fy, fz) + gx1 * nsr_corner_dweight(c, 1, fx, fy, fz) +
                         gx2 * nsr_corner_dweight(c, 2, fx, fy, fz);
        d0 = fmaf(dw, v.x, d0);
        d1 = fmaf(dw, v.y, d1);
      }
    }
    e[3 + 2 * l] = a0;
    e[4 + 2 * l] = a1;
    if (WITH_QB) {
      qb[3 + 2 * l] = d0 * li.scale;
      qb[4 + 2 * l] = d1 * li.scale;
    }
  }
}

// ---- forward with the three GEMMs of the SDF network on tensor cores ---------------------------------------------------------
// As scalar FMAs, the 64 x (36 + 16 + 36) products  z = W1 e,  out = W2 h,  q = W1^T u  and their weight loads from shared memory
// would be more than half of the forward's instructions.
// Here a warp owns 32 samples; the gathers stay thread-per-sample, the three products run as m16n8k16 MMAs with fp32 accumulation on
// operands SPLIT into fp16 hi + lo parts (x = hi + lo, hi = fp16(x), lo = fp16(x - hi)):  x w ~= hi_x hi_w + lo_x hi_w + hi_x lo_w, i.e.
// ~21 bits of every product survive (the dropped lo_x lo_w term is 2^-22 relative): fp32-level accuracy for the inv_s-amplified SDF,
// which a single fp16 product (11 bits) would not give.  Same outputs as fp32 FMAs to ~1e-6 relative.
constexpr int TC_K1 = 48;              // 35 inputs padded to three k16 steps
constexpr int TC_LD1 = TC_K1 + 8;      // 56 halves per row of the E / W1 tiles (ldmatrix conflict-free)

struct NeusTcSmem {
  __half W1hi[NH][TC_LD1], W1lo[NH][TC_LD1];        // [k][j]
  __half W2hi[NOUTP][NSR_LD64], W2lo[NOUTP][NSR_LD64];  // [o][k]
  float b1[NH], b2[NOUTP], w2row0[NH];              // w2row0[k] = W2[0][k] (u = s * W2[0])
  // per warp: the 32 encoding rows as fp16 hi / lo tiles; once a 16-row tile's A fragments are loaded its rows are dead and hold the
  // q vector of the same samples (36 floats: 28 in the row's hi storage, 8 in its lo storage) => 48 KB per CTA, four CTAs per SM
  __half Ehi[kNeusTcWarps][32][TC_LD1], Elo[kNeusTcWarps][32][TC_LD1];
};
static_assert(TC_LD1 * 2 == 28 * 4, "a 56-half row holds 28 floats");
__device__ __forceinline__ float& neus_q_slot(NeusTcSmem& S, int warp, int row, int j) {
  return j < 28 ? reinterpret_cast<float*>(S.Ehi[warp][row])[j] : reinterpret_cast<float*>(S.Elo[warp][row])[j - 28];
}

__device__ __forceinline__ void split_h(float x, __half& hi, __half& lo) {
  hi = __float2half_rn(x);
  lo = __float2half_rn(x - __half2float(hi));
}
// accumulator tile values f(acc) -> hi / lo A fragments of the next GEMM (MT = 1, 64 columns)
template <typename F>
__device__ __forceinline__ void acc_to_split_afrag(const float (&acc)[1][8][4], uint32_t (&ahi)[1][4][4], uint32_t (&alo)[1][4][4], F f) {
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int nt = 2 * k + (j >> 1), i0 = (j & 1) * 2;
      const float v0 = f(acc[0][nt][i0], nt, i0), v1 = f(acc[0][nt][i0 + 1], nt, i0 + 1);
      __half h0, l0, h1, l1;
      split_h(v0, h0, l0);
      split_h(v1, h1, l1);
      const __half2 hh = __halves2half2(h0, h1), ll = __halves2half2(l0, l1);
      ahi[0][k][j] = *reinterpret_cast<const uint32_t*>(&hh);
      alo[0][k][j] = *reinterpret_cast<const uint32_t*>(&ll);
    }
}

// W1 [64,35], b1, W2 [n_out,64], b2 -> split fp16 tiles and fp32 biases in shared memory (CTA of kNeusTcWarps warps)
__device__ __forceinline__ void stage_neus_tc_weights(NeusTcSmem& S, const float* __restrict__ W1, const float* __restrict__ b1,
                                                      const float* __restrict__ W2, const float* __restrict__ b2, int n_out) {
  const int tid = threadIdx.x;
  for (int i = tid; i < NH * TC_LD1; i += kNeusTcWarps * 32) {
    const int k = i / TC_LD1, j = i % TC_LD1;
    split_h(j < NIN ? W1[k * NIN + j] : 0.f, S.W1hi[k][j], S.W1lo[k][j]);
  }
  for (int i = tid; i < NOUTP * NSR_LD64; i += kNeusTcWarps * 32) {
    const int o = i / NSR_LD64, k = i % NSR_LD64;
    split_h((o < n_out && k < NH) ? W2[o * NH + k] : 0.f, S.W2hi[o][k], S.W2lo[o][k]);
  }
  for (int i = tid; i < NH; i += kNeusTcWarps * 32) {
    S.b1[i] = b1[i];
    S.w2row0[i] = W2[i];
  }
  for (int i = tid; i < NOUTP; i += kNeusTcWarps * 32) S.b2[i] = i < n_out ? b2[i] : 0.f;
}

// One warp's 32 samples through the field: lane `lane` holds the unit-cube position (x, y, z) of sample `lane` (ok: the sample is live;
// dead lanes pass any in-range position).  store_out(r0, gq, dr, col, v) receives out[r][col] = (W2 h + b2)[col] of sample
// r = r0 + gq + dr for every col < 16 (the accumulator layout spreads them over the warp; the row arrives in three parts so that the
// field kernel's row arithmetic stays what it was); store_grad(gx, gy, gz) runs on live lanes with d sdf / d x01 of the lane's sample
// (times 1 / (2 radius): the world-space gradient).  Uses the warp's encoding tiles of S; all lanes must call it.
template <bool MASK, typename StoreOut, typename StoreGrad>
__device__ __forceinline__ void neus_field_rows32(NeusTcSmem& S, int warp, int lane, const nsr_grid_t& g, const __half2* __restrict__ table,
                                                  float x, float y, float z, bool ok, int n_active, StoreOut store_out, StoreGrad store_grad) {
  const int gq = lane >> 2, cq = lane & 3;
  {  // ---- encoding row of this thread's sample -> hi / lo fp16 tiles
    float e[NINP], dummy[NINP];
    e[0] = 2.f * x - 1.f;
    e[1] = 2.f * y - 1.f;
    e[2] = 2.f * z - 1.f;
    e[NIN] = 0.f;
    gather_enc<false, MASK>(g, table, x, y, z, 0.f, 0.f, 0.f, e, dummy, n_active);   // masked columns written as 0
    __half* rh = S.Ehi[warp][lane];
    __half* rl = S.Elo[warp][lane];
#pragma unroll
    for (int j = 0; j < NINP; j += 2) {
      __half h0, l0, h1, l1;
      split_h(e[j], h0, l0);
      split_h(e[j + 1], h1, l1);
      *reinterpret_cast<__half2*>(rh + j) = __halves2half2(h0, h1);
      *reinterpret_cast<__half2*>(rl + j) = __halves2half2(l0, l1);
    }
#pragma unroll
    for (int j = NINP; j < TC_K1; j += 2) {
      *reinterpret_cast<__half2*>(rh + j) = __float2half2_rn(0.f);
      *reinterpret_cast<__half2*>(rl + j) = __float2half2_rn(0.f);
    }
  }
  __syncwarp();
#pragma unroll 1
  for (int m = 0; m < 2; ++m) {  // 16 rows at a time: keeps accumulators + two split fragment sets inside the register budget
    const int r0 = m * 16;
    float acc[1][8][4];
    {
      uint32_t ahi[1][3][4], alo[1][3][4];
      nsr_load_afrag<1, 3>(ahi, &S.Ehi[warp][0][0], TC_LD1, r0);
      nsr_load_afrag<1, 3>(alo, &S.Elo[warp][0][0], TC_LD1, r0);
      __syncwarp();   // rows r0 .. r0 + 15 of both tiles are dead from here on: they receive q below
#pragma unroll
      for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[0][nt][q] = S.b1[nt * 8 + cq * 2 + (q & 1)];
      nsr_gemm_w<1, 3, 8>(acc, ahi, &S.W1hi[0][0], TC_LD1);
      nsr_gemm_w<1, 3, 8>(acc, alo, &S.W1hi[0][0], TC_LD1);
      nsr_gemm_w<1, 3, 8>(acc, ahi, &S.W1lo[0][0], TC_LD1);
    }
    // z -> (h, s); out = W2 h + b2
    float sg[8][4];
    uint32_t fhi[1][4][4], flo[1][4][4];
    acc_to_split_afrag(acc, fhi, flo, [&](float zk, int nt, int q) {
      float s_;
      const float h = softplus100(zk, s_);
      sg[nt][q] = s_;
      return h;
    });
    {
      float acco[1][2][4];
#pragma unroll
      for (int nt = 0; nt < 2; ++nt)
#pragma unroll
        for (int q = 0; q < 4; ++q) acco[0][nt][q] = S.b2[nt * 8 + cq * 2 + (q & 1)];
      nsr_gemm_w<1, 4, 2>(acco, fhi, &S.W2hi[0][0], NSR_LD64);
      nsr_gemm_w<1, 4, 2>(acco, flo, &S.W2hi[0][0], NSR_LD64);
      nsr_gemm_w<1, 4, 2>(acco, fhi, &S.W2lo[0][0], NSR_LD64);
#pragma unroll
      for (int nt = 0; nt < 2; ++nt)
#pragma unroll
        for (int q = 0; q < 4; ++q) store_out(r0, gq, (q >> 1) << 3, nt * 8 + cq * 2 + (q & 1), acco[0][nt][q]);
    }
    // u = s * W2[0];  q = W1^T u
    acc_to_split_afrag(acc, fhi, flo, [&](float, int nt, int q) { return sg[nt][q] * S.w2row0[nt * 8 + cq * 2 + (q & 1)]; });
    {
      float accq[1][6][4];
      nsr_zero_acc(accq);
      nsr_gemm_wt<1, 4, 6>(accq, fhi, &S.W1hi[0][0], TC_LD1);
      nsr_gemm_wt<1, 4, 6>(accq, flo, &S.W1hi[0][0], TC_LD1);
      nsr_gemm_wt<1, 4, 6>(accq, fhi, &S.W1lo[0][0], TC_LD1);
#pragma unroll
      for (int nt = 0; nt < 5; ++nt)  // columns 0..35 (q has 35 live entries)
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int col = nt * 8 + cq * 2 + (q & 1);
          if (col < NINP) neus_q_slot(S, warp, r0 + gq + ((q >> 1) << 3), col) = accq[0][nt][q];
        }
    }
  }
  __syncwarp();
  // ---- analytic normal: second gather, features weighted by this sample's q
  if (ok) {
    float qr[NINP];
#pragma unroll
    for (int j = 0; j < NINP; ++j) qr[j] = neus_q_slot(S, warp, lane, j);
    float gx = 2.f * qr[0], gy = 2.f * qr[1], gz = 2.f * qr[2];
#pragma unroll
    for (int l = 0; l < 16; ++l) {
      if (MASK && l >= n_active) break;   // q of a masked level is a column of W1^T u, not 0
      const LevelInfo li = nsr_level(g, l);
      uint32_t cx, cy, cz, idx[8];
      float fx, fy, fz;
      nsr_pos_fract(x, li.scale, cx, fx);
      nsr_pos_fract(y, li.scale, cy, fy);
      nsr_pos_fract(z, li.scale, cz, fz);
      nsr_corner_indices(li, cx, cy, cz, idx);
      const float q0 = qr[3 + 2 * l], q1 = qr[4 + 2 * l];
      float lx = 0.f, ly = 0.f, lz = 0.f;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const float2 v = nsr_ld_table(table, idx[c]);
        const float sv = v.x * q0 + v.y * q1;
        lx = fmaf(nsr_corner_dweight(c, 0, fx, fy, fz), sv, lx);
        ly = fmaf(nsr_corner_dweight(c, 1, fx, fy, fz), sv, ly);
        lz = fmaf(nsr_corner_dweight(c, 2, fx, fy, fz), sv, lz);
      }
      gx = fmaf(li.scale, lx, gx);
      gy = fmaf(li.scale, ly, gy);
      gz = fmaf(li.scale, lz, gz);
    }
    store_grad(gx, gy, gz);
  }
  __syncwarp();  // the tiles are rewritten by the next chunk
}

}  // namespace
