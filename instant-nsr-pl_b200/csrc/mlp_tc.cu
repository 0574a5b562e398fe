// Warpgroup-MMA (wgmma, sm_90a) version of the stand-alone fully-fused MLP forward (tiny-cuda-nn `Network(FullyFusedMLP)`,
// models/network_utils.py:181): asynchronous tensor-core GEMMs with both operands in shared memory instead of the warp-level
// mma.sync path of mlp.cu.
//
// One CTA = 128 threads = one warpgroup = one 128-row tile, issued as two m64 halves.  Every thread writes its input row into
// shared memory in the canonical K-major no-swizzle operand layout (8x16-byte core matrices; LBO = 128 B between core matrices along
// K, SBO = (K/8)*128 B between 8-row groups); the warpgroup issues wgmma.mma_async per 16-wide K step with fp32 accumulators in
// registers, waits for the group, applies the activation to its accumulator fragment and stores it as the next layer's A operand.
// Weights are staged once per CTA in the same canonical layout.
#include "common.cuh"
#include "mlp_warp.cuh"
#include "wgmma.cuh"

namespace {

constexpr int kThreads = 128;
constexpr int kRows = 128;

// stage a row-major [rows][K] fp16 matrix from global memory into the canonical layout
__device__ __forceinline__ void stage_canonical(uint8_t* dst, const __half* __restrict__ src, int rows, int K) {
  const int vec_per_row = K / 8;
  for (int i = threadIdx.x; i < rows * vec_per_row; i += blockDim.x) {
    const int r = i / vec_per_row, kc = i % vec_per_row;
    *reinterpret_cast<uint4*>(dst + nsr_canon_off(r, kc * 8, K)) = __ldg(reinterpret_cast<const uint4*>(src + (size_t)r * K) + kc);
  }
}

// one layer on the tensor core: D[128 x N] = A[128 x K] (smem) * W[N x K]^T (smem); d0 = rows 0..63, d1 = rows 64..127
template <int N>
__device__ __forceinline__ void layer(float (&d0)[N / 2], float (&d1)[N / 2], uint32_t a_saddr, uint32_t w_saddr, int K, bool swap) {
  const uint32_t lbo = 128, sbo = (uint32_t)(K / 8) * 128;
  const uint32_t a_half = (uint32_t)K * 128;  // 64 rows further down the A tile
  nsr_wg_fence();
  for (int kk = 0; kk < K / 16; ++kk) {
    const uint32_t adv = (uint32_t)kk * 256;  // two core matrices along K per k16 step
    const uint64_t db = swap ? nsr_wg_desc(w_saddr + adv, sbo, lbo) : nsr_wg_desc(w_saddr + adv, lbo, sbo);
    const uint64_t da0 = swap ? nsr_wg_desc(a_saddr + adv, sbo, lbo) : nsr_wg_desc(a_saddr + adv, lbo, sbo);
    const uint64_t da1 = swap ? nsr_wg_desc(a_saddr + a_half + adv, sbo, lbo) : nsr_wg_desc(a_saddr + a_half + adv, lbo, sbo);
    nsr_wgmma<N, 0, 0>(d0, da0, db, kk > 0 ? 1u : 0u);
    nsr_wgmma<N, 0, 0>(d1, da1, db, kk > 0 ? 1u : 0u);
  }
  nsr_wg_commit();
  nsr_wg_wait0();
  nsr_wg_fence_regs(d0);
  nsr_wg_fence_regs(d1);
}

template <int KT_IN>
__global__ void __launch_bounds__(kThreads) mlp_fwd_tc_kernel(nsr_mlp_t m, const __half* __restrict__ x, const __half* __restrict__ params,
                                                              __half* __restrict__ out, int64_t n, int swap) {
  constexpr int IN_PAD = KT_IN * 16;
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* sX = smem;                                   // [128][IN_PAD]
  uint8_t* sH = sX + kRows * IN_PAD * 2;                // [128][64]
  uint8_t* sW1 = sH + kRows * 64 * 2;                   // [64][IN_PAD]
  uint8_t* sWh = sW1 + 64 * IN_PAD * 2;                 // (n_hidden-1) x [64][64]
  uint8_t* sWl = sWh + (m.n_hidden - 1) * 64 * 64 * 2;  // [16][64]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // accumulator fragment: rows r0, r0 + 8 (+ 64 for the second half), columns 8 j + c0, 8 j + c0 + 1
  const int r0 = 16 * warp + (lane >> 2), c0 = 2 * (lane & 3);

  stage_canonical(sW1, params, 64, IN_PAD);
  {
    size_t off = (size_t)64 * IN_PAD;
    for (int h = 0; h < m.n_hidden - 1; ++h) {
      stage_canonical(sWh + h * 64 * 64 * 2, params + off, 64, 64);
      off += 64 * 64;
    }
    stage_canonical(sWl, params + off, 16, 64);
  }

  const int64_t n_tiles = (n + kRows - 1) / kRows;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t row = tile * kRows + tid;
    // ---- my input row -> canonical A operand
#pragma unroll
    for (int kc = 0; kc < IN_PAD / 8; ++kc) {
      uint4 v = make_uint4(0, 0, 0, 0);
      if (row < n) v = __ldg(reinterpret_cast<const uint4*>(x + row * IN_PAD) + kc);
      *reinterpret_cast<uint4*>(sX + nsr_canon_off(tid, kc * 8, IN_PAD)) = v;
    }
    nsr_proxy_fence();
    __syncthreads();
    // ---- hidden layers: D = A * W^T, activation, re-pack as the next A operand (in place over sH once every read of it has completed)
    for (int layer_i = 0; layer_i < m.n_hidden; ++layer_i) {
      float d[2][32];
      if (layer_i == 0)
        layer<64>(d[0], d[1], nsr_smem_u32(sX), nsr_smem_u32(sW1), IN_PAD, swap != 0);
      else
        layer<64>(d[0], d[1], nsr_smem_u32(sH), nsr_smem_u32(sWh + (layer_i - 1) * 64 * 64 * 2), 64, swap != 0);
      __syncthreads();
#pragma unroll
      for (int mh = 0; mh < 2; ++mh)
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h)
            *reinterpret_cast<uint32_t*>(sH + nsr_canon_off(64 * mh + r0 + 8 * h, 8 * j + c0, 64)) =
                nsr_pack_h2(nsr_apply_act(d[mh][4 * j + 2 * h], m.activation), nsr_apply_act(d[mh][4 * j + 2 * h + 1], m.activation));
      nsr_proxy_fence();
      __syncthreads();
    }
    // ---- output layer: D[128 x 16] = H * Wl^T
    {
      float d[2][8];
      layer<16>(d[0], d[1], nsr_smem_u32(sH), nsr_smem_u32(sWl), 64, swap != 0);
#pragma unroll
      for (int mh = 0; mh < 2; ++mh)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int64_t orow = tile * kRows + 64 * mh + r0 + 8 * h;
          if (orow < n) {
#pragma unroll
            for (int j = 0; j < 2; ++j)
              *reinterpret_cast<uint32_t*>(out + orow * 16 + 8 * j + c0) =
                  nsr_pack_h2(nsr_apply_act(d[mh][4 * j + 2 * h], m.out_activation), nsr_apply_act(d[mh][4 * j + 2 * h + 1], m.out_activation));
          }
        }
    }
    __syncthreads();  // the smem operands are free for the next tile
  }
}

}  // namespace

// wgmma variant of nsr_mlp_fwd (same arguments).  variant bit 0: swap the LBO / SBO fields of the smem descriptors (a descriptor
// layout check: the results are wrong with it set).  status is accepted for ABI compatibility and never written: the kernel has no
// barrier wait that could time out.
extern "C" int nsr_mlp_fwd_tc(const nsr_mlp_t* m, const void* x_h, const void* params_h, void* out_h, int64_t n, int variant, int* status,
                              void* stream) {
  (void)status;
  NSR_REQUIRE(m != nullptr && m->n_hidden >= 1 && m->n_hidden <= 3 && m->n_out >= 1 && m->n_out <= 16 && m->n_in >= 1 && m->n_in <= 64,
              "nsr_mlp_fwd_tc: unsupported network shape");
  if (n == 0) return 0;
  const int in_pad = (m->n_in + 15) / 16 * 16, kt = in_pad / 16;
  const size_t smem = (size_t)kRows * in_pad * 2 + kRows * 64 * 2 + 64 * in_pad * 2 + (size_t)(m->n_hidden - 1) * 64 * 64 * 2 + 16 * 64 * 2;
  const int64_t tiles = (n + kRows - 1) / kRows;
  // <= 64 KB smem per CTA: 3-4 CTAs per SM overlap each other's load / MMA / epilogue phases
  const int grid = (int)min((int64_t)nsr_sm_count() * 4, tiles);
#define NSR_LAUNCH_TC(KT)                                                                                                  \
  case KT: {                                                                                                               \
    cudaError_t e = cudaFuncSetAttribute(mlp_fwd_tc_kernel<KT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);   \
    if (e != cudaSuccess) {                                                                                                \
      nsr_set_error("nsr_mlp_fwd_tc: cannot reserve %zu B shared memory: %s", smem, cudaGetErrorString(e));                \
      return 2;                                                                                                            \
    }                                                                                                                      \
    mlp_fwd_tc_kernel<KT><<<grid, kThreads, smem, (cudaStream_t)stream>>>(*m, (const __half*)x_h, (const __half*)params_h, \
                                                                          (__half*)out_h, n, variant & 1);               \
  } break;
  switch (kt) {
    NSR_LAUNCH_TC(1) NSR_LAUNCH_TC(2) NSR_LAUNCH_TC(3) NSR_LAUNCH_TC(4)
    default: NSR_REQUIRE(false, "nsr_mlp_fwd_tc: unsupported padded input width %d", in_pad);
  }
#undef NSR_LAUNCH_TC
  NSR_CHECK_LAUNCH("nsr_mlp_fwd_tc");
  return 0;
}
