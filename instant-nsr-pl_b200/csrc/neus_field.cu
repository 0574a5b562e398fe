// Fused NeuS SDF field: VolumeSDF.forward with grad_type='analytic' (models/geometry.py:158-180) -- hash-grid encoding with
// include_xyz (network_utils.py:68-79), fp32 VanillaMLP 35 -> 64 (Softplus beta=100) -> n_out (network_utils.py:95-139), and
// the analytic normal d sdf / d x -- as ONE forward kernel, and its first- AND second-order backward (what torch reaches through
// autograd.grad(create_graph=True) + the eikonal loss, systems/neus.py:106) as ONE backward kernel.  The math is the hand
// derivation checked against autograd in oracle/neus_field.py:
//   e = [2 x01 - 1 | hash(x01)];  z = W1 e + b1;  h = softplus(z);  s = sigmoid(beta z);  out = W2 h + b2;  u = s * W2[0]
//   q = W1^T u;  grad_world = (2 q_xyz + J^T q_hash) / (2 r)
//   backward(g_out, g_grad): gx = g_grad / (2r);  qb = [2 gx | J gx];  ub = W1 qb;  zb = (W2^T g_out) s + ub W2[0] beta s (1 - s)
//     eb = W1^T zb;  dW1 = u qb^T + zb e^T;  db1 = zb;  dW2 = g_out h^T (+ row 0: ub s);  db2 = g_out
//     dtable[c] += w_c eb_l + q_l scale_l (dw_c/dx . gx)        (ONE 8-byte RED per corner carries both orders)
// The SDF branch keeps fp32 accuracy (the reference runs it under autocast(False): the NeuS alpha multiplies sdf by inv_s up to 1e3+):
// the forward's products run on tensor cores with operands split into fp16 hi + lo parts (below); the backward stays on the CUDA cores,
// weights broadcast from shared memory, and only its weight-gradient outer products go through tensor cores.
#include "mlp_warp.cuh"

namespace {

constexpr int kThreads = 128;
constexpr int NIN = 35;     // 3 + 16 * 2
constexpr int NINP = 36;    // padded row length (float4 loads)
constexpr int NH = 64;
constexpr int NOUTP = 16;   // padded output width

struct NeusW {  // shared-memory weights (floats)
  float W1[NH][NINP];       // [k][j]
  float W2T[NH][NOUTP];     // [k][i] = W2[i][k]
  float b1[NH];
  float b2[NOUTP];
};

__device__ __forceinline__ void stage_neus_weights(NeusW& w, const float* __restrict__ W1, const float* __restrict__ b1,
                                                   const float* __restrict__ W2, const float* __restrict__ b2, int n_out) {
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
  __half Ehi[kThreads / 32][32][TC_LD1], Elo[kThreads / 32][32][TC_LD1];
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

template <bool MASK>
__global__ void __launch_bounds__(kThreads, 4) neus_field_fwd_tc_kernel(const __grid_constant__ nsr_grid_t g, const float* __restrict__ points,
                                                                        const __half2* __restrict__ table, const float* __restrict__ W1,
                                                                        const float* __restrict__ b1, const float* __restrict__ W2,
                                                                        const float* __restrict__ b2, float radius, int n_out,
                                                                        float* __restrict__ sdf, float* __restrict__ grad,
                                                                        float* __restrict__ feat, int64_t n_cap,
                                                                        const int64_t* __restrict__ n_dev, const float* __restrict__ n_active_p) {
  const int64_t n = n_dev ? min(*n_dev, n_cap) : n_cap;
  const int n_active = MASK ? load_n_active(n_active_p) : 16;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  NeusTcSmem& S = *reinterpret_cast<NeusTcSmem*>(smem_raw);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, gq = lane >> 2, cq = lane & 3;
  for (int i = tid; i < NH * TC_LD1; i += kThreads) {
    const int k = i / TC_LD1, j = i % TC_LD1;
    split_h(j < NIN ? W1[k * NIN + j] : 0.f, S.W1hi[k][j], S.W1lo[k][j]);
  }
  for (int i = tid; i < NOUTP * NSR_LD64; i += kThreads) {
    const int o = i / NSR_LD64, k = i % NSR_LD64;
    split_h((o < n_out && k < NH) ? W2[o * NH + k] : 0.f, S.W2hi[o][k], S.W2lo[o][k]);
  }
  for (int i = tid; i < NH; i += kThreads) {
    S.b1[i] = b1[i];
    S.w2row0[i] = W2[i];
  }
  for (int i = tid; i < NOUTP; i += kThreads) S.b2[i] = i < n_out ? b2[i] : 0.f;
  __syncthreads();
  const float inv2r = 1.f / (2.f * radius);
  const int64_t n32 = (n + 31) & ~31ll;
  for (int64_t base = (blockIdx.x * (int64_t)(kThreads / 32) + warp) * 32; base < n32; base += (int64_t)gridDim.x * kThreads) {
    const int64_t i = base + lane;
    const bool ok = i < n;
    float x = 0.5f, y = 0.5f, z = 0.5f;
    if (ok) {
      x = (points[i * 3 + 0] + radius) * inv2r;
      y = (points[i * 3 + 1] + radius) * inv2r;
      z = (points[i * 3 + 2] + radius) * inv2r;
    }
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
          for (int q = 0; q < 4; ++q) {
            const int64_t row = base + r0 + gq + ((q >> 1) << 3);
            const int col = nt * 8 + cq * 2 + (q & 1);
            if (row < n) {
              if (col == 0) sdf[row] = acco[0][nt][q];
              if (col < n_out) feat[row * n_out + col] = acco[0][nt][q];
            }
          }
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
      grad[i * 3 + 0] = gx * inv2r;
      grad[i * 3 + 1] = gy * inv2r;
      grad[i * 3 + 2] = gz * inv2r;
    }
    __syncwarp();  // the tiles are rewritten by the next chunk
  }
}

// ---- backward ------------------------------------------------------------------------------------------------------
// transposed fp16 tiles [feature][sample] (ld = 128 + 8): thread `row` writes consecutive halves => conflict-free
constexpr int LDT = kThreads + 8;  // 136
constexpr int TT_U = 0;                       // [64] u          (unscaled)
constexpr int TT_ZB = TT_U + NH * LDT;        // [64] zb         (scaled)
constexpr int TT_H = TT_ZB + NH * LDT;        // [64] h          (unscaled)
constexpr int TT_US = TT_H + NH * LDT;        // [64] ub * s     (scaled)
constexpr int TT_QB = TT_US + NH * LDT;       // [48] qb         (scaled)
constexpr int TT_E = TT_QB + 48 * LDT;        // [48] e          (unscaled)
constexpr int TT_GO = TT_E + 48 * LDT;        // [16] g_out      (scaled)
constexpr int TT_TOTAL = TT_GO + 16 * LDT;    // 368 rows x 272 B + weights = 113.7 KB => two CTAs per SM
constexpr size_t kBwdSmem = sizeof(NeusW) + (size_t)TT_TOTAL * sizeof(__half);

// acc[1][2] (16 x 16 output block) += A^T-tile rows m0..m0+15 (x 128 samples) * B-tile rows n0..n0+15
__device__ __forceinline__ void wgrad_block(float (&acc)[1][2][4], const __half* At, int m0, const __half* Bt, int n0) {
  uint32_t a[1][8][4];
  nsr_load_afrag<1, 8>(a, At, LDT, m0);
  nsr_gemm_w<1, 8, 2>(acc, a, Bt + (size_t)n0 * LDT, LDT);
}

template <bool MASK>
__global__ void __launch_bounds__(kThreads, 2) neus_field_bwd_kernel(const __grid_constant__ nsr_grid_t g, const float* __restrict__ points,
                                                                     const __half2* __restrict__ table, const float* __restrict__ W1,
                                                                     const float* __restrict__ b1, const float* __restrict__ W2,
                                                                     const float* __restrict__ b2, float radius, int n_out,
                                                                     const float* __restrict__ g_out, const float* __restrict__ g_sdf,
                                                                     const float* __restrict__ g_grad,
                                                                     const float* __restrict__ amax_ptr, float* __restrict__ grad_table,
                                                                     float* __restrict__ dW1, float* __restrict__ db1, float* __restrict__ dW2,
                                                                     float* __restrict__ db2, int64_t n_cap,
                                                                     const int64_t* __restrict__ n_dev, const float* __restrict__ n_active_p) {
  const int64_t n = n_dev ? min(*n_dev, n_cap) : n_cap;
  const int n_active = MASK ? load_n_active(n_active_p) : 16;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  NeusW& w = *reinterpret_cast<NeusW*>(smem_raw);
  __half* T = reinterpret_cast<__half*>(smem_raw + sizeof(NeusW));
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, gq = lane >> 2, cq = lane & 3;
  stage_neus_weights(w, W1, b1, W2, b2, n_out);
  const float amax = fmaxf(amax_ptr ? __ldg(amax_ptr) : 1.f, 1e-30f);
  const float scale = exp2f(fminf(fmaxf(floorf(log2f(4.f / amax)), -24.f), 40.f));
  const float inv_scale = 1.f / scale, inv2r = 1.f / (2.f * radius);
  __syncthreads();

  // weight-gradient accumulators: dW1 [64 x 48] = 12 blocks + dW2 [16 x 64] = 4 blocks => 4 per warp, on tensor cores;
  // the three "times a vector of ones" products (db1 = sum_s zb, db2 = sum_s g_out, dW2[0] += sum_s ub s) are row sums of the
  // transposed tiles: thread t owns row t of [ZB (64) | US (64)], threads 0..15 additionally row t of GO.
  constexpr int kBlocks = 16, kSlots = 4;
  float wacc[kSlots][1][2][4];
#pragma unroll
  for (int s = 0; s < kSlots; ++s)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int i = 0; i < 4; ++i) wacc[s][0][j][i] = 0.f;
  float rsum = 0.f, rsum_go = 0.f;

  const int64_t n_tiles = (n + kThreads - 1) / kThreads;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t i = tile * kThreads + tid;
    const bool ok = i < n;
    __syncthreads();  // previous tile's wgrad is done with the tiles
    float e[NINP], qb[NINP], eb[NINP], q[NINP], go[NOUTP];
    float x = 0.f, y = 0.f, z = 0.f, gx0 = 0.f, gx1 = 0.f, gx2 = 0.f;
#pragma unroll
    for (int j = 0; j < NINP; ++j) e[j] = qb[j] = eb[j] = q[j] = 0.f;
#pragma unroll
    for (int o = 0; o < NOUTP; ++o) go[o] = 0.f;
    if (ok) {
      x = (points[i * 3 + 0] + radius) * inv2r;
      y = (points[i * 3 + 1] + radius) * inv2r;
      z = (points[i * 3 + 2] + radius) * inv2r;
      gx0 = g_grad ? g_grad[i * 3 + 0] * inv2r : 0.f;
      gx1 = g_grad ? g_grad[i * 3 + 1] * inv2r : 0.f;
      gx2 = g_grad ? g_grad[i * 3 + 2] * inv2r : 0.f;
      if (g_out) {
#pragma unroll
        for (int o = 0; o < NOUTP; ++o)
          if (o < n_out) go[o] = g_out[i * n_out + o];
      }
      if (g_sdf) go[0] += g_sdf[i];
      e[0] = 2.f * x - 1.f;
      e[1] = 2.f * y - 1.f;
      e[2] = 2.f * z - 1.f;
      qb[0] = 2.f * gx0;
      qb[1] = 2.f * gx1;
      qb[2] = 2.f * gx2;
      gather_enc<true, MASK>(g, table, x, y, z, gx0, gx1, gx2, e, qb, n_active);   // e = qb = 0 on masked levels: their dW1 columns get 0
    }
#pragma unroll 2
    for (int k = 0; k < NH; ++k) {
      float row[NINP];
#pragma unroll
      for (int v = 0; v < NINP / 4; ++v) *reinterpret_cast<float4*>(&row[4 * v]) = *reinterpret_cast<const float4*>(&w.W1[k][4 * v]);
      float zk = w.b1[k], ubk = 0.f;
#pragma unroll
      for (int j = 0; j < NINP; ++j) {
        zk = fmaf(row[j], e[j], zk);
        ubk = fmaf(row[j], qb[j], ubk);
      }
      float s;
      const float h = softplus100(zk, s);
      float w2[NOUTP];
#pragma unroll
      for (int v = 0; v < NOUTP / 4; ++v) *reinterpret_cast<float4*>(&w2[4 * v]) = *reinterpret_cast<const float4*>(&w.W2T[k][4 * v]);
      float tk = 0.f;
#pragma unroll
      for (int o = 0; o < NOUTP; ++o) tk = fmaf(w2[o], go[o], tk);
      const float u = s * w2[0];
      const float zbk = tk * s + ubk * w2[0] * (100.f * s * (1.f - s));
#pragma unroll
      for (int j = 0; j < NINP; ++j) {
        eb[j] = fmaf(row[j], zbk, eb[j]);
        q[j] = fmaf(row[j], u, q[j]);
      }
      T[TT_U + k * LDT + tid] = __float2half(ok ? u : 0.f);
      T[TT_ZB + k * LDT + tid] = __float2half(ok ? zbk * scale : 0.f);
      T[TT_H + k * LDT + tid] = __float2half(ok ? h : 0.f);
      T[TT_US + k * LDT + tid] = __float2half(ok ? ubk * s * scale : 0.f);
    }
#pragma unroll
    for (int j = 0; j < 48; ++j) {
      T[TT_QB + j * LDT + tid] = __float2half(j < NIN ? qb[j < NINP ? j : 0] * scale : 0.f);
      T[TT_E + j * LDT + tid] = __float2half(j < NIN ? e[j < NINP ? j : 0] : 0.f);
    }
#pragma unroll
    for (int o = 0; o < NOUTP; ++o) T[TT_GO + o * LDT + tid] = __float2half(go[o] * scale);
    // ---- table gradient: first- and second-order terms in one RED per corner.
    // Levels 0..kMergeLevels-1 can merge runs of equal cells across neighbouring lanes (consecutive samples of a ray) with a segmented
    // warp scan so that only the last lane of a run issues the 8 REDs (as in nerf_fused_bwd.cu).  Merging was measured
    // slower than plain REDs here -- with one sample per thread the 85 shuffles per level cost more than the REDs
    // they save (this kernel is not RED-bound), so merging is compiled out.
    constexpr int kMergeLevels = 0;
#pragma unroll
    for (int l = 0; l < 16; ++l) {
      if (MASK && l >= n_active) break;   // eb and q of a masked level are not 0: its table slice is left untouched
      const float eb0 = eb[3 + 2 * l], eb1 = eb[4 + 2 * l], q0 = q[3 + 2 * l], q1 = q[4 + 2 * l];
      const LevelInfo li = nsr_level(g, l);
      uint32_t cx, cy, cz, idx[8];
      float fx, fy, fz;
      nsr_pos_fract(x, li.scale, cx, fx);
      nsr_pos_fract(y, li.scale, cy, fy);
      nsr_pos_fract(z, li.scale, cz, fz);
      if (l < kMergeLevels) {
        float v[16];
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const float wc = nsr_corner_weight(c, fx, fy, fz);
          const float coef = li.scale * (gx0 * nsr_corner_dweight(c, 0, fx, fy, fz) + gx1 * nsr_corner_dweight(c, 1, fx, fy, fz) +
                                         gx2 * nsr_corner_dweight(c, 2, fx, fy, fz));
          v[2 * c] = ok ? wc * eb0 + coef * q0 : 0.f;
          v[2 * c + 1] = ok ? wc * eb1 + coef * q1 : 0.f;
        }
        const uint32_t key = ok ? (cx + li.res * (cy + li.res * cz)) : (0xFFFFFFC0u + lane);
        const uint32_t key_prev = __shfl_up_sync(0xffffffffu, key, 1);
        const bool head = (lane == 0) || (key_prev != key);
        const int next_head = __shfl_down_sync(0xffffffffu, (int)head, 1);
        const bool tail = (lane == 31) || next_head;
        bool flag = head;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int f_up = __shfl_up_sync(0xffffffffu, (int)flag, o);
          const bool take = (lane >= o) && !flag;
#pragma unroll
          for (int e2 = 0; e2 < 16; ++e2) {
            const float up = __shfl_up_sync(0xffffffffu, v[e2], o);
            if (take) v[e2] += up;
          }
          if (take) flag = f_up;
        }
        if (ok && tail) {
          nsr_corner_indices(li, cx, cy, cz, idx);
#pragma unroll
          for (int c = 0; c < 8; ++c)
            if (v[2 * c] != 0.f || v[2 * c + 1] != 0.f) nsr_red_add_f32x2(grad_table + 2 * (size_t)idx[c], v[2 * c], v[2 * c + 1]);
        }
      } else if (ok) {
        nsr_corner_indices(li, cx, cy, cz, idx);
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const float wc = nsr_corner_weight(c, fx, fy, fz);
          const float coef = li.scale * (gx0 * nsr_corner_dweight(c, 0, fx, fy, fz) + gx1 * nsr_corner_dweight(c, 1, fx, fy, fz) +
                                         gx2 * nsr_corner_dweight(c, 2, fx, fy, fz));
          const float v0 = wc * eb0 + coef * q0, v1 = wc * eb1 + coef * q1;
          if (v0 != 0.f || v1 != 0.f) nsr_red_add_f32x2(grad_table + 2 * (size_t)idx[c], v0, v1);
        }
      }
    }
    __syncthreads();
    // ---- weight gradients on tensor cores over the 128 samples of the tile
#pragma unroll
    for (int s = 0; s < kSlots; ++s) {
      const int t = warp + s * 4;
      if (t < 12) {            // dW1 block (m, n): u qb^T + zb e^T
        const int m0 = (t / 3) * 16, n0 = (t % 3) * 16;
        wgrad_block(wacc[s], T + TT_U, m0, T + TT_QB, n0);
        wgrad_block(wacc[s], T + TT_ZB, m0, T + TT_E, n0);
      } else if (t < kBlocks) {  // dW2 block: g_out h^T
        wgrad_block(wacc[s], T + TT_GO, 0, T + TT_H, (t - 12) * 16);
      }
    }
    // ---- row sums over the tile's 128 samples (fp16 tiles, fp32 accumulation)
    {
      const __half* row = T + (tid < NH ? TT_ZB + tid * LDT : TT_US + (tid - NH) * LDT);
      float a = 0.f;
#pragma unroll
      for (int v = 0; v < kThreads / 8; ++v) {
        const uint4 q4 = *reinterpret_cast<const uint4*>(row + v * 8);
        const __half2* h2 = reinterpret_cast<const __half2*>(&q4);
#pragma unroll
        for (int e2 = 0; e2 < 4; ++e2) {
          const float2 f = __half22float2(h2[e2]);
          a += f.x + f.y;
        }
      }
      rsum += a;
      if (tid < NOUTP) {
        const __half* rg = T + TT_GO + tid * LDT;
        float b = 0.f;
#pragma unroll
        for (int v = 0; v < kThreads / 8; ++v) {
          const uint4 q4 = *reinterpret_cast<const uint4*>(rg + v * 8);
          const __half2* h2 = reinterpret_cast<const __half2*>(&q4);
#pragma unroll
          for (int e2 = 0; e2 < 4; ++e2) {
            const float2 f = __half22float2(h2[e2]);
            b += f.x + f.y;
          }
        }
        rsum_go += b;
      }
    }
  }
  // ---- flush
#pragma unroll
  for (int s = 0; s < kSlots; ++s) {
    const int t = warp + s * 4;
    if (t >= kBlocks) continue;
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = gq + ((i >> 1) << 3), cidx = j * 8 + cq * 2 + (i & 1);
        const float val = wacc[s][0][j][i] * inv_scale;
        if (val == 0.f) continue;
        if (t < 12) {
          const int m = (t / 3) * 16 + r, nn = (t % 3) * 16 + cidx;
          if (nn < NIN) atomicAdd(dW1 + m * NIN + nn, val);
        } else {
          const int nn = (t - 12) * 16 + cidx;
          if (r < n_out) atomicAdd(dW2 + r * NH + nn, val);
        }
      }
  }
  if (rsum != 0.f) {
    if (tid < NH)
      atomicAdd(db1 + tid, rsum * inv_scale);
    else
      atomicAdd(dW2 + (tid - NH), rsum * inv_scale);  // row 0 of dW2: + sum_s ub s
  }
  if (tid < n_out && rsum_go != 0.f) atomicAdd(db2 + tid, rsum_go * inv_scale);
}

int check(const nsr_grid_t* g, int n_out, const char* name) {
  NSR_REQUIRE(g != nullptr && g->n_levels == 16 && g->n_features == 2, "%s: needs a 16-level F=2 hash grid", name);
  NSR_REQUIRE(n_out >= 1 && n_out <= 16, "%s: n_out must be in [1,16]", name);
  return 0;
}

// MASK selects the level-masked instantiations (n_active: device float); the unmasked ones never read it
template <bool MASK>
int field_fwd(const char* name, const nsr_grid_t* g, const float* points, const void* table_h, const float* W1, const float* b1, const float* W2,
              const float* b2, float radius, int32_t n_out, const float* n_active, float* sdf, float* grad, float* feature, int64_t n,
              const int64_t* n_dev, void* stream) {
  if (int e = check(g, n_out, name)) return e;
  NSR_REQUIRE(!MASK || n_active != nullptr, "%s: n_active (device float) is NULL", name);
  if (n == 0) return 0;
  // neus_field_fwd_tc_kernel: the SDF network on tensor cores, hi / lo split operands.
  // The kernel is bound by the latency of its two gathers: fewer instructions only pay once the freed registers / shared memory buy a
  // fourth CTA per SM (q aliased onto the encoding rows).  Issuing the corner loads of four levels together, as the NeRF forward does,
  // was not faster and is not kept.
  static thread_local bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(neus_field_fwd_tc_kernel<MASK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(NeusTcSmem));
    if (e != cudaSuccess) {
      nsr_set_error("%s: cannot reserve %zu B shared memory: %s", name, sizeof(NeusTcSmem), cudaGetErrorString(e));
      return 2;
    }
    attr_set = true;
  }
  const int grid = (int)min((int64_t)nsr_sm_count() * 4, (n + kThreads - 1) / kThreads);
  neus_field_fwd_tc_kernel<MASK><<<grid, kThreads, sizeof(NeusTcSmem), (cudaStream_t)stream>>>(*g, points, (const __half2*)table_h, W1, b1, W2, b2,
                                                                                                radius, n_out, sdf, grad, feature, n, n_dev, n_active);
  NSR_CHECK_LAUNCH(name);
  return 0;
}

template <bool MASK>
int field_bwd(const char* name, const nsr_grid_t* g, const float* points, const void* table_h, const float* W1, const float* b1, const float* W2,
              const float* b2, float radius, int32_t n_out, const float* n_active, const float* g_out, const float* g_sdf, const float* g_grad,
              const float* amax, float* grad_table, float* dW1, float* db1, float* dW2, float* db2, int64_t n, const int64_t* n_dev, void* stream) {
  if (int e = check(g, n_out, name)) return e;
  NSR_REQUIRE(!MASK || n_active != nullptr, "%s: n_active (device float) is NULL", name);
  if (n == 0) return 0;
  static thread_local bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(neus_field_bwd_kernel<MASK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBwdSmem);
    if (e != cudaSuccess) {
      nsr_set_error("%s: cannot reserve %zu B shared memory: %s", name, kBwdSmem, cudaGetErrorString(e));
      return 2;
    }
    attr_set = true;
  }
  const int grid = (int)min((int64_t)nsr_sm_count() * 2, (n + kThreads - 1) / kThreads);  // two CTAs per SM: their gather / MLP / scatter phases overlap
  neus_field_bwd_kernel<MASK><<<grid, kThreads, kBwdSmem, (cudaStream_t)stream>>>(*g, points, (const __half2*)table_h, W1, b1, W2, b2, radius, n_out,
                                                                                  g_out, g_sdf, g_grad, amax, grad_table, dW1, db1, dW2, db2, n, n_dev,
                                                                                  n_active);
  NSR_CHECK_LAUNCH(name);
  return 0;
}

}  // namespace

extern "C" int nsr_neus_field_fwd(const nsr_grid_t* g, const float* points, const void* table_h, const float* W1, const float* b1,
                                  const float* W2, const float* b2, float radius, int32_t n_out, float* sdf, float* grad, float* feature,
                                  int64_t n, const int64_t* n_dev, void* stream) {
  return field_fwd<false>("nsr_neus_field_fwd", g, points, table_h, W1, b1, W2, b2, radius, n_out, nullptr, sdf, grad, feature, n, n_dev, stream);
}

extern "C" int nsr_neus_field_bwd(const nsr_grid_t* g, const float* points, const void* table_h, const float* W1, const float* b1,
                                  const float* W2, const float* b2, float radius, int32_t n_out, const float* g_out, const float* g_sdf,
                                  const float* g_grad, const float* amax, float* grad_table, float* dW1, float* db1, float* dW2, float* db2, int64_t n,
                                  const int64_t* n_dev, void* stream) {
  return field_bwd<false>("nsr_neus_field_bwd", g, points, table_h, W1, b1, W2, b2, radius, n_out, nullptr, g_out, g_sdf, g_grad, amax, grad_table,
                          dW1, db1, dW2, db2, n, n_dev, stream);
}

extern "C" int nsr_neus_field_fwd_levels(const nsr_grid_t* g, const float* points, const void* table_h, const float* W1, const float* b1,
                                         const float* W2, const float* b2, float radius, int32_t n_out, const float* n_active, float* sdf,
                                         float* grad, float* feature, int64_t n, const int64_t* n_dev, void* stream) {
  return field_fwd<true>("nsr_neus_field_fwd_levels", g, points, table_h, W1, b1, W2, b2, radius, n_out, n_active, sdf, grad, feature, n, n_dev,
                         stream);
}

extern "C" int nsr_neus_field_bwd_levels(const nsr_grid_t* g, const float* points, const void* table_h, const float* W1, const float* b1,
                                         const float* W2, const float* b2, float radius, int32_t n_out, const float* n_active, const float* g_out,
                                         const float* g_sdf, const float* g_grad, const float* amax, float* grad_table, float* dW1, float* db1,
                                         float* dW2, float* db2, int64_t n, const int64_t* n_dev, void* stream) {
  return field_bwd<true>("nsr_neus_field_bwd_levels", g, points, table_h, W1, b1, W2, b2, radius, n_out, n_active, g_out, g_sdf, g_grad, amax,
                         grad_table, dW1, db1, dW2, db2, n, n_dev, stream);
}

namespace {
__global__ void __launch_bounds__(256) absmax_kernel(const float* __restrict__ a, int64_t na, const float* __restrict__ b, int64_t nb,
                                                     const float* __restrict__ c, int64_t nc, float* __restrict__ out, int64_t rows_cap,
                                                     const int64_t* __restrict__ rows_dev) {
  if (rows_dev != nullptr) {  // arrays are [rows_cap, width]: only the first *rows_dev rows are live
    const int64_t rows = min(*rows_dev, rows_cap);
    na = na / rows_cap * rows;
    nb = nb / rows_cap * rows;
    nc = nc / rows_cap * rows;
  }
  float m = 0.f;
  const int64_t stride = (int64_t)gridDim.x * 256, t0 = blockIdx.x * 256ll + threadIdx.x;
  for (int64_t i = t0; i < na; i += stride) m = fmaxf(m, fabsf(a[i]));
  for (int64_t i = t0; i < nb; i += stride) m = fmaxf(m, fabsf(b[i]));
  for (int64_t i = t0; i < nc; i += stride) m = fmaxf(m, fabsf(c[i]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(reinterpret_cast<int*>(out), __float_as_int(m));  // non-negative floats order like ints
}
}  // namespace

extern "C" int nsr_absmax3(const float* a, int64_t na, const float* b, int64_t nb, const float* c, int64_t nc, float* out, int64_t rows_cap,
                           const int64_t* rows_dev, void* stream) {
  NSR_REQUIRE(out != nullptr, "nsr_absmax3: out is NULL");
  NSR_REQUIRE(rows_dev == nullptr || rows_cap > 0, "nsr_absmax3: rows_dev needs rows_cap > 0");
  if (a == nullptr) na = 0;
  if (b == nullptr) nb = 0;
  if (c == nullptr) nc = 0;
  cudaMemsetAsync(out, 0, sizeof(float), (cudaStream_t)stream);
  const int64_t nmax = max(na, max(nb, nc));
  if (nmax == 0) return 0;
  const int grid = (int)min((int64_t)nsr_sm_count() * 4, (nmax + 255) / 256);
  absmax_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(a, na, b, nb, c, nc, out, rows_cap, rows_dev);
  NSR_CHECK_LAUNCH("nsr_absmax3");
  return 0;
}
