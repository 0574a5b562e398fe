// Hopper tensor-core form of the fused NeRF backward (autograd of VolumeRadiance + VolumeDensity + HashGrid, models/texture.py:23-30,
// models/geometry.py:122-130; tcnn: FullyFusedMLP backward + grid backward): warpgroup MMAs (wgmma.mma_async, sm_90a) with both
// operands in shared memory, tile inputs staged by the TMA engine (cp.async.bulk + mbarrier), warp-specialised roles.
//
// One CTA = 16 warps, one CTA per SM, persistent over 128-row tiles of kept samples (packed, ray-major order):
//   warps 0-7   two chain warpgroups; warpgroup c owns rows [64 c, 64 c + 64) of every tile and walks the ten dependent GEMMs of its
//               half -- five forward-recompute layers, five dgrad layers -- plus, next to each dgrad, the weight-gradient GEMM of that
//               layer (M = 64, K = the 64 samples).  Accumulators are registers; the epilogue (activation / ReLU mask from the fp16
//               activations the tile holds / incoming-gradient injection) re-packs to fp16 and stores into the next GEMM's A operand in
//               the canonical K-major layout, which read through an MN-major descriptor is also the weight-gradient GEMM's operand: no
//               transposes anywhere.  Weight-gradient partials are added into a shared fp32 accumulator, flushed once at the end.
//               The last GEMM's d(encoding) goes to a two-slot shared buffer for the scatter warps.
//   warps 8-15  scatter, two groups that alternate tiles and own one stage of the two-stage input ring each: thread = row; read
//               d(encoding) (16 fp16 pairs), then per level corner weights, warp-wide merging of runs that share a cell, paired 16-byte
//               REDs into the fp32 gradient table.  Once every reader is done with the group's stage, one lane refills it with the
//               tile after next: four cp.async.bulk copies (encodings in the canonical tile layout written by nsr_pack_kept, position +
//               direction, d sigma_raw, d rgb = 13 KB).  (A separate producer warp would cost the chain 32 registers per thread.)
// The GEMM chain of tile t+1 runs while the scatter warps are still issuing the REDs of tiles t and t-1.
//
// Shared memory (170 KB): weights of both networks, canonical [out][in] (one copy serves the forward GEMMs as K-major B and the dgrad
// GEMMs as MN-major B); activation tiles H1, CI, G1, G2 which the dgrad epilogues overwrite in place with dH1, dG1, dG2; dC3, dO;
// two stages of tile inputs; two d(encoding) slots; the weight-gradient accumulator.
#include "nerf_fused.cuh"
#include "wgmma.cuh"

namespace {

constexpr int kThreads = 512;
constexpr int kRows = 128;

// ---- shared-memory map (bytes) ----------------------------------------------------------------------------------------------
constexpr int W_DW1 = 0;                    // [64][32]
constexpr int W_DW2 = W_DW1 + 64 * 32 * 2;  // [16][64]
constexpr int W_CW1 = W_DW2 + 16 * 64 * 2;  // [64][32]
constexpr int W_CW2 = W_CW1 + 64 * 32 * 2;  // [64][64]
constexpr int W_CW3 = W_CW2 + 64 * 64 * 2;  // [16][64]
constexpr int W_END = W_CW3 + 16 * 64 * 2;  // 20480
constexpr int A_H1 = W_END;                 // [128][64]  H1, later dH1
constexpr int A_CI = A_H1 + kRows * 64 * 2; // [128][32]  out16 | SH16
constexpr int A_G1 = A_CI + kRows * 32 * 2; // [128][64]  G1, later dG1
constexpr int A_G2 = A_G1 + kRows * 64 * 2; // [128][64]  G2, later dG2
constexpr int A_DC3 = A_G2 + kRows * 64 * 2;  // [128][16]
constexpr int A_DO = A_DC3 + kRows * 16 * 2;  // [128][16]
constexpr int A_END = A_DO + kRows * 16 * 2;
// one stage of tile inputs: encodings (canonical [128][32] halves), xyz+dir [128][6] f32, d_sraw [128] f32, d_rgb [128][3] f32
constexpr int S_X0 = 0, S_XYZ = S_X0 + kRows * 32 * 2, S_DS = S_XYZ + kRows * 6 * 4, S_DRGB = S_DS + kRows * 4, S_STAGE = S_DRGB + kRows * 3 * 4;
constexpr int kStageBytes = S_STAGE;  // 13312
constexpr int STAGES = A_END;
// d(encoding) slots: [128 rows][16 levels] fp16 pairs, rows padded to 20 words (conflict-free 16-byte reads by the scatter warps)
constexpr int DE_STRIDE = 20;
constexpr int DE = STAGES + 2 * kStageBytes;
constexpr int kDeBytes = kRows * DE_STRIDE * 4;
// weight-gradient accumulator: one fp32 slot per (accumulator register, chain thread): both warpgroups add into the same slots
constexpr int G_DW1 = 0, G_DW2 = G_DW1 + 16, G_CW1 = G_DW2 + 8, G_CW2 = G_CW1 + 16, G_CW3 = G_CW2 + 32, G_SLOTS = G_CW3 + 8;  // 80
constexpr int WACC = DE + 2 * kDeBytes;
constexpr int BARS = WACC + G_SLOTS * 128 * 4;
constexpr int kSmemBytes = BARS + 128;
static_assert(kStageBytes % 16 == 0 && STAGES % 128 == 0 && DE % 16 == 0 && WACC % 16 == 0, "alignment");
static_assert(kSmemBytes <= 227 * 1024, "shared memory");

// barrier slots (8 bytes each)
enum { B_FULL0 = 0, B_FULL1, B_EMPTY0, B_EMPTY1, B_DEFULL0, B_DEFULL1, B_DEEMPTY0, B_DEEMPTY1, B_COUNT };

__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_bulk(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
// barrier of the 128 threads of chain warpgroup c (ids 1, 2); id 3 joins both chain warpgroups
__device__ __forceinline__ void wg_bar(int c) { asm volatile("bar.sync %0, 128;" ::"r"(1 + c) : "memory"); }
__device__ __forceinline__ void chain_bar() { asm volatile("bar.sync 3, 256;" ::: "memory"); }

// row-major [rows][K] fp16 matrix (global) -> canonical smem tile
__device__ __forceinline__ void stage_canonical(uint8_t* dst, const __half* __restrict__ src, int rows, int K) {
  const int vec_per_row = K / 8;
  for (int i = threadIdx.x; i < rows * vec_per_row; i += blockDim.x) {
    const int r = i / vec_per_row, kc = i % vec_per_row;
    *reinterpret_cast<uint4*>(dst + nsr_canon_off(r, kc * 8, K)) = __ldg(reinterpret_cast<const uint4*>(src + (size_t)r * K) + kc);
  }
}

// descriptors of a canonical tile at byte address `addr`, k16 step kk:
//   K-major  [rows][K]: LBO = 128 B (the two 8-wide K chunks), SBO = (K/8)*128 B (8-row groups); step kk starts 256 B further
//   MN-major [k rows][C] read with M / N along C: SBO = 128 B (8-column chunks), LBO = (C/8)*128 B (8-row k groups); step kk = 2 LBO
__device__ __forceinline__ uint64_t dk(uint32_t addr, int K, int kk) { return nsr_wg_desc(addr + 256u * (uint32_t)kk, 128u, (uint32_t)(K / 8) * 128u); }
__device__ __forceinline__ uint64_t dm(uint32_t addr, int C, int kk) { return nsr_wg_desc_mn(addr, C, kk); }

struct TcArgs {
  const uint8_t* enc_tiles;  // canonical [tile][128][32] fp16
  const float* xyzdir;       // [rows][6]
  const float* d_sraw;       // [rows]
  const float* d_rgb;        // [rows][3]
  const __half* dparams;
  const __half* cparams;
  float* grad_dparams;
  float* grad_cparams;
  const float* amax;
  const int64_t* n_dev;
  int64_t n_cap;
  float loss_scale;
  int* status;
};

// epilogue of a 64-wide hidden layer from the accumulator fragment into a canonical K = 64 tile (rows rr[0], rr[1])
//   MODE 0: ReLU on the packed pair (round, then max with +0: same value as rounding max(x, 0))
//   MODE 1: dgrad through ReLU, IN PLACE: the tile still holds this layer's fp16 activations (written by this same thread in the
//           forward epilogue); a gradient survives where its activation is > 0 (__hgt2_mask: ordered compare, a NaN activation masks)
// Rows past the end of the batch (keep = 0) are written as zeros.
template <int MODE>
__device__ __forceinline__ void epi64(const float (&d)[32], uint8_t* tile, const int (&rr)[2], const uint32_t (&keep)[2], int c0) {
  const __half2 zero = __float2half2_rn(0.f);
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      uint32_t* p = reinterpret_cast<uint32_t*>(tile + nsr_canon_off(rr[h], 8 * j + c0, 64));
      const __half2 v = __floats2half2_rn(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]);
      if (MODE == 0) {
        const __half2 r = __hmax2(v, zero);
        *p = *reinterpret_cast<const uint32_t*>(&r) & keep[h];
      } else {
        const uint32_t act = *p;
        *p = *reinterpret_cast<const uint32_t*>(&v) & __hgt2_mask(*reinterpret_cast<const __half2*>(&act), zero) & keep[h];
      }
    }
}

template <int R>
__device__ __forceinline__ void wacc_add(float* wacc, int slot0, int t, const float (&w)[R]) {
#pragma unroll
  for (int r = 0; r < R; ++r) atomicAdd(wacc + (slot0 + r) * 128 + t, w[r]);
}

__global__ void __launch_bounds__(kThreads, 1) nerf_bwd_tc_kernel(const __grid_constant__ nsr_nerf_t P, const TcArgs a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int64_t n = a.n_dev ? min(*a.n_dev, a.n_cap) : a.n_cap;
  const int64_t n_tiles = (n + kRows - 1) / kRows;
  float loss_scale = a.loss_scale;
  if (loss_scale <= 0.f) {  // automatic: bring the largest incoming gradient to ~2^8 (same rule as nerf_bwd_kernel)
    const float amax = fmaxf(__ldg(a.amax), 1e-30f);
    loss_scale = exp2f(fminf(fmaxf(floorf(log2f(256.f / amax)), -24.f), 60.f));
  }
  const float inv_scale = 1.f / loss_scale;
  const uint32_t sbase = nsr_smem_u32(smem);
  const uint32_t bars = sbase + BARS;
  auto bar = [&](int i) { return bars + 8u * (uint32_t)i; };
  float* wacc = reinterpret_cast<float*>(smem + WACC);

  if (tid == 0) {
    mbar_init(bar(B_FULL0), 1);
    mbar_init(bar(B_FULL1), 1);
    mbar_init(bar(B_EMPTY0), 12);  // 8 chain warps + 4 scatter warps
    mbar_init(bar(B_EMPTY1), 12);
    mbar_init(bar(B_DEFULL0), 8);
    mbar_init(bar(B_DEFULL1), 8);
    mbar_init(bar(B_DEEMPTY0), 4);
    mbar_init(bar(B_DEEMPTY1), 4);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  stage_canonical(smem + W_DW1, a.dparams, 64, 32);
  stage_canonical(smem + W_DW2, a.dparams + 64 * 32, 16, 64);
  stage_canonical(smem + W_CW1, a.cparams, 64, 32);
  stage_canonical(smem + W_CW2, a.cparams + 64 * 32, 64, 64);
  stage_canonical(smem + W_CW3, a.cparams + 64 * 32 + 64 * 64, 16, 64);
  for (int i = tid; i < G_SLOTS * 128; i += kThreads) wacc[i] = 0.f;
  nsr_proxy_fence();
  __syncthreads();
  const int64_t my_tiles = n_tiles > (int64_t)blockIdx.x ? (n_tiles - 1 - blockIdx.x) / gridDim.x + 1 : 0;

  if (warp < 8) {
    // ================================ chain warpgroups ================================
    const int c = warp >> 2, t = tid & 127;
    const int R0 = 64 * c;
    // accumulator fragment of this thread: rows rr[0], rr[1] of the tile, columns 8 j + c0 (+1)
    const int c0 = 2 * (lane & 3);
    const int rr[2] = {R0 + 16 * (warp & 3) + (lane >> 2), R0 + 16 * (warp & 3) + (lane >> 2) + 8};
    // operand addresses of this warpgroup's 64-row half (64 rows of a [128][K] canonical tile = K * 128 bytes)
    const uint32_t h1 = sbase + A_H1 + c * 64 * 128, ci = sbase + A_CI + c * 32 * 128, g1 = sbase + A_G1 + c * 64 * 128;
    const uint32_t g2 = sbase + A_G2 + c * 64 * 128, dc3 = sbase + A_DC3 + c * 16 * 128, dO = sbase + A_DO + c * 16 * 128;
    const uint32_t w_dw1 = sbase + W_DW1, w_dw2 = sbase + W_DW2, w_cw1 = sbase + W_CW1, w_cw2 = sbase + W_CW2, w_cw3 = sbase + W_CW3;
    // every GEMM step: make this warpgroup's epilogue stores visible to the tensor core, issue, wait; then a barrier so that no thread
    // overwrites an operand tile in place before the whole warpgroup's MMAs have read it
    auto begin = [&]() {
      nsr_proxy_fence();
      wg_bar(c);
      nsr_wg_fence();
    };
    auto end = [&]() {
      nsr_wg_commit();
      nsr_wg_wait0();
      wg_bar(c);
    };
    for (int64_t it = 0; it < my_tiles; ++it) {
      const int s = (int)(it & 1);
      const int64_t tile = blockIdx.x + it * gridDim.x;
      uint8_t* st = smem + STAGES + s * kStageBytes;
      const uint32_t x0 = sbase + STAGES + (uint32_t)s * kStageBytes + S_X0 + c * 32 * 128;
      const bool live[2] = {tile * kRows + rr[0] < n, tile * kRows + rr[1] < n};
      const uint32_t keep[2] = {live[0] ? 0xFFFFFFFFu : 0u, live[1] ? 0xFFFFFFFFu : 0u};
      mbar_wait(bar(B_FULL0 + s), (uint32_t)((it >> 1) & 1), a.status, 3);
      float drgb[2][3], dsraw[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float* rg = reinterpret_cast<const float*>(st + S_DRGB) + rr[h] * 3;
#pragma unroll
        for (int e = 0; e < 3; ++e) drgb[h][e] = live[h] ? rg[e] : 0.f;
        dsraw[h] = live[h] ? reinterpret_cast<const float*>(st + S_DS)[rr[h]] : 0.f;
      }
      {  // thread pair per row: SH of the view direction -> columns 16..31 of the colour network's input; rows past the end: zero
         // encodings (the buffers hold whatever they contained: keep 0 * NaN out of the weight-gradient sums)
        const int row = R0 + (t >> 1), part = t & 1;
        const bool row_live = tile * kRows + row < n;
        const float* rf = reinterpret_cast<const float*>(st + S_XYZ) + row * 6;
        uint4 sv = make_uint4(0, 0, 0, 0);
        if (row_live) {
          float sh[16];
          nsr_sh4(rf[3], rf[4], rf[5], sh);
          const float* q = sh + 8 * part;
          sv = make_uint4(nsr_pack_h2(q[0], q[1]), nsr_pack_h2(q[2], q[3]), nsr_pack_h2(q[4], q[5]), nsr_pack_h2(q[6], q[7]));
        } else {
          *reinterpret_cast<uint4*>(st + S_X0 + nsr_canon_off(row, 16 * part, 32)) = make_uint4(0, 0, 0, 0);
          *reinterpret_cast<uint4*>(st + S_X0 + nsr_canon_off(row, 16 * part + 8, 32)) = make_uint4(0, 0, 0, 0);
        }
        *reinterpret_cast<uint4*>(smem + A_CI + nsr_canon_off(row, 16 + 8 * part, 32)) = sv;
      }
      // 1: H1 = relu(X0 . DW1^T)
      {
        float d[32];
        begin();
#pragma unroll
        for (int kk = 0; kk < 2; ++kk) nsr_wgmma_n64<0, 0>(d, dk(x0, 32, kk), dk(w_dw1, 32, kk), kk > 0);
        end();
        nsr_wg_fence_regs(d);
        epi64<0>(d, smem + A_H1, rr, keep, c0);
      }
      // 2: out16 = H1 . DW2^T (fp16) -> columns 0..15 of the colour input
      {
        float d[8];
        begin();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) nsr_wgmma_n16<0, 0>(d, dk(h1, 64, kk), dk(w_dw2, 64, kk), kk > 0);
        end();
        nsr_wg_fence_regs(d);
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h)
            *reinterpret_cast<uint32_t*>(smem + A_CI + nsr_canon_off(rr[h], 8 * j + c0, 32)) = nsr_pack_h2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]) & keep[h];
      }
      // 3, 4: colour hidden layers G1 = relu([O | SH] . CW1^T), G2 = relu(G1 . CW2^T)
      {
        float d[32];
        begin();
#pragma unroll
        for (int kk = 0; kk < 2; ++kk) nsr_wgmma_n64<0, 0>(d, dk(ci, 32, kk), dk(w_cw1, 32, kk), kk > 0);
        end();
        nsr_wg_fence_regs(d);
        epi64<0>(d, smem + A_G1, rr, keep, c0);
      }
      {
        float d[32];
        begin();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) nsr_wgmma_n64<0, 0>(d, dk(g1, 64, kk), dk(w_cw2, 64, kk), kk > 0);
        end();
        nsr_wg_fence_regs(d);
        epi64<0>(d, smem + A_G2, rr, keep, c0);
      }
      // 5: rgb_pre = G2 . CW3^T; d(rgb pre-activation) = d_rgb * s (1 - s), s = sigmoid(fp16(raw)) on columns 0..2, zero elsewhere
      {
        float d[8];
        begin();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) nsr_wgmma_n16<0, 0>(d, dk(g2, 64, kk), dk(w_cw3, 64, kk), kk > 0);
        end();
        nsr_wg_fence_regs(d);
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float dp[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int col = 8 * j + c0 + e;
              dp[e] = 0.f;
              if (col < 3) {
                const float raw = __half2float(__float2half_rn(d[4 * j + 2 * h + e]));
                const float sg = 1.f / (1.f + expf(-raw));
                const float dr = col == 0 ? drgb[h][0] : (col == 1 ? drgb[h][1] : drgb[h][2]);
                dp[e] = live[h] ? dr * sg * (1.f - sg) * loss_scale : 0.f;
              }
            }
            *reinterpret_cast<uint32_t*>(smem + A_DC3 + nsr_canon_off(rr[h], 8 * j + c0, 16)) = nsr_pack_h2(dp[0], dp[1]);
          }
      }
      // 6: dG2pre = dC3 . CW3 ; dCW3^T += G2^T . dC3 ; dG2 in place over G2
      {
        {
          float w[8];
          begin();
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) nsr_wgmma_n16<1, 1>(w, dm(g2, 64, kk), dm(dc3, 16, kk), kk > 0);
          end();
          nsr_wg_fence_regs(w);
          wacc_add(wacc, G_CW3, t, w);
        }
        float d[32];
        nsr_wg_fence();
        nsr_wgmma_n64<0, 1>(d, dk(dc3, 16, 0), dm(w_cw3, 64, 0), 0u);
        end();
        nsr_wg_fence_regs(d);
        epi64<1>(d, smem + A_G2, rr, keep, c0);
      }
      // 7: dG1pre = dG2 . CW2 ; dCW2 += dG2^T . G1 ; dG1 in place over G1
      {
        {
          float w[32];
          begin();
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) nsr_wgmma_n64<1, 1>(w, dm(g2, 64, kk), dm(g1, 64, kk), kk > 0);
          end();
          nsr_wg_fence_regs(w);
          wacc_add(wacc, G_CW2, t, w);
        }
        float d[32];
        nsr_wg_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) nsr_wgmma_n64<0, 1>(d, dk(g2, 64, kk), dm(w_cw2, 64, kk), kk > 0);
        end();
        nsr_wg_fence_regs(d);
        epi64<1>(d, smem + A_G1, rr, keep, c0);
      }
      // 8: dOpre = dG1 . CW1[:, 0:16] ; dCW1 += dG1^T . CI ; d(out16) = colour path + d sigma_raw on column 0
      {
        {
          float w[16];
          begin();
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) nsr_wgmma_n32<1, 1>(w, dm(g1, 64, kk), dm(ci, 32, kk), kk > 0);
          end();
          nsr_wg_fence_regs(w);
          wacc_add(wacc, G_CW1, t, w);
        }
        float d[8];
        nsr_wg_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) nsr_wgmma_n16<0, 1>(d, dk(g1, 64, kk), dm(w_cw1, 32, kk), kk > 0);
        end();
        nsr_wg_fence_regs(d);
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const float f0 = d[4 * j + 2 * h] + (j == 0 && c0 == 0 ? dsraw[h] * loss_scale : 0.f);
            *reinterpret_cast<uint32_t*>(smem + A_DO + nsr_canon_off(rr[h], 8 * j + c0, 16)) = nsr_pack_h2(f0, d[4 * j + 2 * h + 1]) & keep[h];
          }
      }
      // 9: dH1pre = dO . DW2 ; dDW2^T += H1^T . dO ; dH1 in place over H1
      {
        {
          float w[8];
          begin();
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) nsr_wgmma_n16<1, 1>(w, dm(h1, 64, kk), dm(dO, 16, kk), kk > 0);
          end();
          nsr_wg_fence_regs(w);
          wacc_add(wacc, G_DW2, t, w);
        }
        float d[32];
        nsr_wg_fence();
        nsr_wgmma_n64<0, 1>(d, dk(dO, 16, 0), dm(w_dw2, 64, 0), 0u);
        end();
        nsr_wg_fence_regs(d);
        epi64<1>(d, smem + A_H1, rr, keep, c0);
      }
      // 10: dE = dH1 . DW1 ; dDW1 += dH1^T . X0 -> d(encoding) slot s (the scatter group of tile it - 2 must have drained it)
      {
        {
          float w[16];
          begin();
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) nsr_wgmma_n32<1, 1>(w, dm(h1, 64, kk), dm(x0, 32, kk), kk > 0);
          end();
          nsr_wg_fence_regs(w);
          __syncwarp();
          if (lane == 0) mbar_arrive(bar(B_EMPTY0 + s));  // the stage's inputs are not read any more
          wacc_add(wacc, G_DW1, t, w);
        }
        float d[16];
        nsr_wg_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) nsr_wgmma_n32<0, 1>(d, dk(h1, 64, kk), dm(w_dw1, 32, kk), kk > 0);
        end();
        nsr_wg_fence_regs(d);
        if (it >= 2) mbar_wait(bar(B_DEEMPTY0 + s), (uint32_t)(((it - 2) >> 1) & 1), a.status, 4);
        uint32_t* de = reinterpret_cast<uint32_t*>(smem + DE + s * kDeBytes);
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h) de[rr[h] * DE_STRIDE + 4 * j + (lane & 3)] = nsr_pack_h2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]);
        __syncwarp();
        if (lane == 0) mbar_arrive(bar(B_DEFULL0 + s));
      }
    }
    // ---- weight gradients: shared accumulator -> global, slots split between the two warpgroups
    chain_bar();
    if (my_tiles > 0) {
      auto flush = [&](int slot0, int N, float* dst, int stride_m, int stride_n) {
        for (int r = c; r < N / 2; r += 2) {
          const int j = r >> 2, h = (r >> 1) & 1, e = r & 1;
          const int m = 16 * (warp & 3) + (lane >> 2) + 8 * h, col = 8 * j + c0 + e;
          atomicAdd(dst + (size_t)m * stride_m + (size_t)col * stride_n, wacc[(slot0 + r) * 128 + t] * inv_scale);
        }
      };
      flush(G_DW1, 32, a.grad_dparams, 32, 1);                     // dDW1 [out m][in n]
      flush(G_DW2, 16, a.grad_dparams + 64 * 32, 1, 64);           // dDW2^T [in m][out n] -> DW2 [out][in]
      flush(G_CW1, 32, a.grad_cparams, 32, 1);                     // dCW1 [out m][in n]
      flush(G_CW2, 64, a.grad_cparams + 64 * 32, 64, 1);           // dCW2 [out m][in n]
      flush(G_CW3, 16, a.grad_cparams + 64 * 32 + 64 * 64, 1, 64); // dCW3^T [in m][out n] -> CW3 [out][in]
    }
  } else {
    // ================================ scatter ================================
    const int grp = (warp - 8) >> 2;  // tiles alternate between the two groups
    const int row = (warp & 3) * 32 + lane;
    const bool loader = (warp & 3) == 0 && lane == 0;
    float* grad_table = a.grad_dparams + NF_DENSITY_PARAMS;
    auto load = [&](int64_t it) {  // tile inputs of the CTA's tile `it` -> stage it & 1
      const int64_t tile = blockIdx.x + it * gridDim.x, row0 = tile * kRows;
      const uint32_t dst = sbase + STAGES + (uint32_t)(it & 1) * kStageBytes, fb = bar(B_FULL0 + (int)(it & 1));
      mbar_expect_tx(fb, kStageBytes);
      tma_bulk(dst + S_X0, a.enc_tiles + tile * (kRows * 32 * 2), kRows * 32 * 2, fb);
      tma_bulk(dst + S_XYZ, a.xyzdir + row0 * 6, kRows * 6 * 4, fb);
      tma_bulk(dst + S_DS, a.d_sraw + row0, kRows * 4, fb);
      tma_bulk(dst + S_DRGB, a.d_rgb + row0 * 3, kRows * 3 * 4, fb);
    };
    if (loader && grp < my_tiles) load(grp);
    for (int64_t it = grp; it < my_tiles; it += 2) {
      const int s = (int)(it & 1);  // == grp
      const int64_t tile = blockIdx.x + it * gridDim.x, grow = tile * kRows + row;
      const bool ok = grow < n;
      const uint8_t* st = smem + STAGES + s * kStageBytes;
      mbar_wait(bar(B_FULL0 + s), (uint32_t)((it >> 1) & 1), a.status, 8);
      const float* rf = reinterpret_cast<const float*>(st + S_XYZ) + row * 6;
      const float x = rf[0], y = rf[1], z = rf[2];
      __syncwarp();
      if (lane == 0) mbar_arrive(bar(B_EMPTY0 + s));
      mbar_wait(bar(B_DEFULL0 + s), (uint32_t)((it >> 1) & 1), a.status, 9);
      uint32_t de[16];  // (feature 0, feature 1) of level l as fp16 pair, still multiplied by the loss scale
      {
        const uint4* src = reinterpret_cast<const uint4*>(smem + DE + s * kDeBytes + row * DE_STRIDE * 4);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const uint4 v = src[q];
          de[4 * q] = v.x;
          de[4 * q + 1] = v.y;
          de[4 * q + 2] = v.z;
          de[4 * q + 3] = v.w;
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bar(B_DEEMPTY0 + s));
      if (loader && it + 2 < my_tiles) {  // every reader of this tile's stage has arrived: refill it with the group's next tile
        mbar_wait(bar(B_EMPTY0 + s), (uint32_t)((it >> 1) & 1), a.status, 1);
        load(it + 2);
      }
#pragma unroll
      for (int l = 0; l < 16; ++l) {
        float2 d = __half22float2(*reinterpret_cast<const __half2*>(&de[l]));
        d.x = ok ? d.x * inv_scale : 0.f;
        d.y = ok ? d.y * inv_scale : 0.f;
        const LevelInfo li = nsr_level(P.grid, l);
        uint32_t cx, cy, cz, idx[8];
        float fx, fy, fz;
        nsr_pos_fract(x, li.scale, cx, fx);
        nsr_pos_fract(y, li.scale, cy, fy);
        nsr_pos_fract(z, li.scale, cz, fz);
        float v[16];
#pragma unroll
        for (int cc = 0; cc < 8; ++cc) {
          const float w = nsr_corner_weight(cc, fx, fy, fz);
          v[2 * cc] = w * d.x;
          v[2 * cc + 1] = w * d.y;
        }
        bool issue = ok && (d.x != 0.f || d.y != 0.f);
        if (l < 8) {  // runs of consecutive samples in one cell: sum across the warp, the last lane of a run issues
          const uint32_t key = ok ? (cx + li.res * (cy + li.res * cz)) : (0xFFFFFF00u + lane);
          const uint32_t prev = __shfl_up_sync(0xffffffffu, key, 1);
          const bool head = lane == 0 || prev != key;
          const uint32_t heads = __ballot_sync(0xffffffffu, head);
          const int my_head = 31 - __clz(heads & (0xffffffffu >> (31 - lane)));
          const bool tail = lane == 31 || ((heads >> (lane + 1)) & 1u);
          int maxrun = lane - my_head + 1;
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) maxrun = max(maxrun, __shfl_xor_sync(0xffffffffu, maxrun, o));
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            if (o < maxrun) {
              const bool take = lane - o >= my_head;
#pragma unroll
              for (int e = 0; e < 16; ++e) {
                const float u = __shfl_up_sync(0xffffffffu, v[e], o);
                if (take) v[e] += u;
              }
            }
          }
          issue = ok && tail;
        }
        if (issue) {
          nsr_corner_indices(li, cx, cy, cz, idx);
#pragma unroll
          for (int cc = 0; cc < 8; cc += 2) nsr_red_corner_pair(grad_table, idx[cc], idx[cc + 1], v[2 * cc], v[2 * cc + 1], v[2 * cc + 2], v[2 * cc + 3]);
        }
      }
    }
  }
}

}  // namespace

// wgmma / TMA form of nsr_nerf_field_bwd over the packed inputs.  enc_tiles_h: the kept samples' encodings in the canonical tile layout
// (nsr_pack_kept with enc_tiled = 1: tile t = rows [128 t, 128 t + 128), 8 KB each); xyzdir / d_sraw / d_rgb in packed row order.  All four
// buffers must be readable up to the end of the last 128-row tile (the kernel masks rows >= k itself).  status (device int, may be NULL)
// receives a non-zero code if an mbarrier wait timed out (the kernel then traps instead of hanging).
extern "C" int nsr_nerf_field_bwd_tc(const nsr_nerf_t* f, const void* enc_tiles_h, const void* dparams_h, const void* cparams_h,
                                     const float* d_sraw, const float* d_rgb, float* grad_dparams, float* grad_cparams, float loss_scale,
                                     const float* amax, int64_t k, const int64_t* k_dev, const float* xyzdir, int* status, void* stream) {
  NSR_REQUIRE(f != nullptr, "nsr_nerf_field_bwd_tc: field descriptor is NULL");
  NSR_REQUIRE(f->grid.n_levels == 16 && f->grid.n_features == 2 && f->feature_dim == 16 && f->density_hidden == 1 && f->color_hidden == 2 && f->contraction == 0,
              "nsr_nerf_field_bwd_tc: fused path needs L=16, F=2, feature_dim=16, hidden layers 1/2, AABB contraction");
  NSR_REQUIRE(loss_scale > 0.f || amax != nullptr, "nsr_nerf_field_bwd_tc: loss_scale <= 0 (automatic) needs the amax pointer");
  NSR_REQUIRE(enc_tiles_h != nullptr && xyzdir != nullptr && d_sraw != nullptr && d_rgb != nullptr, "nsr_nerf_field_bwd_tc: NULL input");
  if (k == 0) return 0;
  static thread_local bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(nerf_bwd_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
    if (e != cudaSuccess) {
      nsr_set_error("nsr_nerf_field_bwd_tc: cannot reserve %d B shared memory: %s", kSmemBytes, cudaGetErrorString(e));
      return 2;
    }
    attr_set = true;
  }
  TcArgs a;
  a.enc_tiles = (const uint8_t*)enc_tiles_h;
  a.xyzdir = xyzdir;
  a.d_sraw = d_sraw;
  a.d_rgb = d_rgb;
  a.dparams = (const __half*)dparams_h;
  a.cparams = (const __half*)cparams_h;
  a.grad_dparams = grad_dparams;
  a.grad_cparams = grad_cparams;
  a.amax = amax;
  a.n_dev = k_dev;
  a.n_cap = k;
  a.loss_scale = loss_scale;
  a.status = status;
  const int64_t tiles = (k + kRows - 1) / kRows;
  int grid = (int)min((int64_t)nsr_sm_count(), tiles);
  if (k_dev != nullptr) grid = nsr_sm_count();
  nerf_bwd_tc_kernel<<<grid, kThreads, kSmemBytes, (cudaStream_t)stream>>>(*f, a);
  NSR_CHECK_LAUNCH("nsr_nerf_field_bwd_tc");
  return 0;
}
