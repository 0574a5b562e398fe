// Development micro-benchmark (not part of the product path): gather-only variants of the 16-level hash
// encode, to pick the load strategy used by nf_gather.  positions [n,3] in [0,1] -> enc fp16 [n,32].
#include "../../instant-nsr-pl_b200/csrc/nerf_fused.cuh"

namespace {

template <int VARIANT>
__device__ __forceinline__ void gather_variant(const nsr_grid_t& g, const __half2* __restrict__ table, float x, float y, float z,
                                               uint32_t (&f)[16]) {
  if (VARIANT == 0) {  // level by level, 8 x 4-byte loads
#pragma unroll
    for (int l = 0; l < 16; ++l) {
      const LevelInfo li = nsr_level(g, l);
      uint32_t cx, cy, cz, idx[8];
      float fx, fy, fz;
      nsr_pos_fract(x, li.scale, cx, fx);
      nsr_pos_fract(y, li.scale, cy, fy);
      nsr_pos_fract(z, li.scale, cz, fz);
      nsr_corner_indices(li, cx, cy, cz, idx);
      float2 v[8];
#pragma unroll
      for (int c = 0; c < 8; ++c) v[c] = nsr_ld_table(table, idx[c]);
      float a0 = 0.f, a1 = 0.f;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const float w = nsr_corner_weight(c, fx, fy, fz);
        a0 = fmaf(w, v[c].x, a0);
        a1 = fmaf(w, v[c].y, a1);
      }
      f[l] = nsr_pack_h2(a0, a1);
    }
  } else if (VARIANT == 1 || VARIANT == 2 || VARIANT == 5) {  // batches of NB levels, 8 x 4-byte loads
    constexpr int NB = VARIANT == 1 ? 4 : (VARIANT == 2 ? 2 : 8);
#pragma unroll
    for (int l0 = 0; l0 < 16; l0 += NB) {
      uint32_t raw[NB][8];
      float fr[NB][3];
#pragma unroll
      for (int j = 0; j < NB; ++j) {
        const LevelInfo li = nsr_level(g, l0 + j);
        uint32_t cx, cy, cz, idx[8];
        nsr_pos_fract(x, li.scale, cx, fr[j][0]);
        nsr_pos_fract(y, li.scale, cy, fr[j][1]);
        nsr_pos_fract(z, li.scale, cz, fr[j][2]);
        nsr_corner_indices(li, cx, cy, cz, idx);
#pragma unroll
        for (int c = 0; c < 8; ++c) raw[j][c] = __ldg(reinterpret_cast<const uint32_t*>(table) + idx[c]);
      }
#pragma unroll
      for (int j = 0; j < NB; ++j) {
        float a0 = 0.f, a1 = 0.f;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const float w = nsr_corner_weight(c, fr[j][0], fr[j][1], fr[j][2]);
          const float2 v = __half22float2(*reinterpret_cast<const __half2*>(&raw[j][c]));
          a0 = fmaf(w, v.x, a0);
          a1 = fmaf(w, v.y, a1);
        }
        f[l0 + j] = nsr_pack_h2(a0, a1);
      }
    }
  } else if (VARIANT == 3) {
    nf_gather_paired<16, 1>(g, table, x, y, z, f);  // paired 8-byte loads, level by level
  } else {
    nf_gather_paired<16, 4>(g, table, x, y, z, f);  // paired + batches of 4
  }
}

template <int VARIANT>
__global__ void __launch_bounds__(256) dbg_gather_kernel(const __grid_constant__ nsr_grid_t g, const float* __restrict__ pos,
                                                         const __half2* __restrict__ table, __half* __restrict__ out, int64_t n) {
  extern __shared__ __half pad[];
  for (int64_t i = blockIdx.x * 256ll + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) {
    uint32_t f[16];
    gather_variant<VARIANT>(g, table, pos[i * 3], pos[i * 3 + 1], pos[i * 3 + 2], f);
    uint4* e = reinterpret_cast<uint4*>(out + i * 32);
    e[0] = make_uint4(f[0], f[1], f[2], f[3]);
    e[1] = make_uint4(f[4], f[5], f[6], f[7]);
    e[2] = make_uint4(f[8], f[9], f[10], f[11]);
    e[3] = make_uint4(f[12], f[13], f[14], f[15]);
  }
}

template <int V>
int launch(const nsr_grid_t* g, const float* pos, const void* table, void* out, int64_t n, int ctas_per_sm, cudaStream_t st) {
  // dynamic smem padding pins the occupancy: 227 KB / ctas_per_sm per CTA
  const int smem = ctas_per_sm >= 8 ? 0 : (220 * 1024 / ctas_per_sm) & ~15;
  cudaFuncSetAttribute(dbg_gather_kernel<V>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  const int grid = nsr_sm_count() * ctas_per_sm;
  dbg_gather_kernel<V><<<grid, 256, smem, st>>>(*g, pos, (const __half2*)table, (__half*)out, n);
  NSR_CHECK_LAUNCH("nsr_dbg_gather");
  return 0;
}

}  // namespace

extern "C" int nsr_dbg_gather(const nsr_grid_t* g, const float* pos, const void* table_h, void* out_h, int64_t n, int variant,
                              int ctas_per_sm, void* stream) {
  NSR_REQUIRE(g && g->n_levels == 16, "nsr_dbg_gather: 16 levels");
  cudaStream_t st = (cudaStream_t)stream;
  switch (variant) {
    case 0: return launch<0>(g, pos, table_h, out_h, n, ctas_per_sm, st);
    case 1: return launch<1>(g, pos, table_h, out_h, n, ctas_per_sm, st);
    case 2: return launch<2>(g, pos, table_h, out_h, n, ctas_per_sm, st);
    case 3: return launch<3>(g, pos, table_h, out_h, n, ctas_per_sm, st);
    case 4: return launch<4>(g, pos, table_h, out_h, n, ctas_per_sm, st);
    case 5: return launch<5>(g, pos, table_h, out_h, n, ctas_per_sm, st);
  }
  NSR_REQUIRE(false, "nsr_dbg_gather: unknown variant %d", variant);
}

// ---- scatter-only variants: dEnc fp16 [n,32] -> gradient table ---------------------------------------
namespace {

__device__ __forceinline__ void red_f16x2(__half2* addr, float a, float b) {
  const uint32_t v = nsr_pack_h2(a, b);
  asm volatile("red.global.add.noftz.f16x2 [%0], %1;" ::"l"(addr), "r"(v) : "memory");
}

template <int VARIANT>
__global__ void __launch_bounds__(256) dbg_scatter_kernel(const __grid_constant__ nsr_grid_t g, const float* __restrict__ pos,
                                                          const __half2* __restrict__ denc, float* __restrict__ grad, int64_t n) {
  // VARIANT 0: thread per sample, red.v2.f32 | 1: thread per sample, 2 x red.f32 | 2: thread per sample, red.f16x2 (grad viewed as half2)
  // VARIANT 3: thread per (sample, level), red.v2.f32 | 4: thread per (sample, level), red.f16x2
  // VARIANT 5: thread per sample, x-adjacent corner pairs as one red.v4.f32 when they are neighbours in memory
  const bool per_level = VARIANT >= 3;
  const int64_t total = per_level ? n * 16 : n;
  for (int64_t t = blockIdx.x * 256ll + threadIdx.x; t < total; t += (int64_t)gridDim.x * 256) {
    const int64_t i = per_level ? (t >> 4) : t;
    const float x = pos[i * 3], y = pos[i * 3 + 1], z = pos[i * 3 + 2];
    const int lbeg = per_level ? (int)(t & 15) : 0, lend = per_level ? lbeg + 1 : 16;
#pragma unroll 1
    for (int l = lbeg; l < lend; ++l) {
      const float2 d = __half22float2(denc[i * 16 + l]);
      const LevelInfo li = nsr_level(g, l);
      uint32_t cx, cy, cz, idx[8];
      float fx, fy, fz;
      nsr_pos_fract(x, li.scale, cx, fx);
      nsr_pos_fract(y, li.scale, cy, fy);
      nsr_pos_fract(z, li.scale, cz, fz);
      nsr_corner_indices(li, cx, cy, cz, idx);
      if (VARIANT == 5) {
#pragma unroll
        for (int c = 0; c < 8; c += 2) {
          const float w0 = nsr_corner_weight(c, fx, fy, fz), w1 = nsr_corner_weight(c + 1, fx, fy, fz);
          nsr_red_corner_pair(grad, idx[c], idx[c + 1], w0 * d.x, w0 * d.y, w1 * d.x, w1 * d.y);
        }
        continue;
      }
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const float w = nsr_corner_weight(c, fx, fy, fz);
        if (VARIANT == 0 || VARIANT == 3) {
          nsr_red_add_f32x2(grad + 2 * (size_t)idx[c], w * d.x, w * d.y);
        } else if (VARIANT == 1) {
          atomicAdd(grad + 2 * (size_t)idx[c], w * d.x);
          atomicAdd(grad + 2 * (size_t)idx[c] + 1, w * d.y);
        } else {
          red_f16x2(reinterpret_cast<__half2*>(grad) + idx[c], w * d.x, w * d.y);
        }
      }
    }
  }
}


// ---- warp-wide run merging + paired 16-byte REDs, thread per sample (what the scatter warps of the tensor-core backward do) -------
// lanes = 32 consecutive samples (ray-major order); on levels < MERGE_LEVELS runs of equal cells are summed with a segmented shuffle
// scan over the WHOLE warp and only the run's last lane issues REDs; x-adjacent corners that are
// neighbours in memory go out as one red.v4.f32.  PAIR = 0: 8-byte REDs only.
template <int MERGE_LEVELS, int PAIR>
__global__ void __launch_bounds__(256) dbg_scatter_merged_kernel(const __grid_constant__ nsr_grid_t g, const float* __restrict__ pos,
                                                                 const __half2* __restrict__ denc, float* __restrict__ grad, int64_t n) {
  const int lane = threadIdx.x & 31;
  const int64_t n32 = (n + 31) & ~31ll;
  for (int64_t i = blockIdx.x * 256ll + threadIdx.x; i < n32; i += (int64_t)gridDim.x * 256) {
    const bool ok = i < n;
    float x = 0.f, y = 0.f, z = 0.f;
    if (ok) {
      x = pos[i * 3];
      y = pos[i * 3 + 1];
      z = pos[i * 3 + 2];
    }
#pragma unroll 1
    for (int l = 0; l < 16; ++l) {
      float2 d = make_float2(0.f, 0.f);
      if (ok) d = __half22float2(denc[i * 16 + l]);
      const LevelInfo li = nsr_level(g, l);
      uint32_t cx, cy, cz, idx[8];
      float fx, fy, fz;
      nsr_pos_fract(x, li.scale, cx, fx);
      nsr_pos_fract(y, li.scale, cy, fy);
      nsr_pos_fract(z, li.scale, cz, fz);
      float v[16];
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const float w = nsr_corner_weight(c, fx, fy, fz);
        v[2 * c] = w * d.x;
        v[2 * c + 1] = w * d.y;
      }
      bool issue = ok;
      if (l < MERGE_LEVELS) {
        const uint32_t key = ok ? (cx + li.res * (cy + li.res * cz)) : (0xFFFFFF00u + lane);
        const uint32_t prev = __shfl_up_sync(0xffffffffu, key, 1);
        const bool head = lane == 0 || prev != key;
        const uint32_t heads = __ballot_sync(0xffffffffu, head);
        const int my_head = 31 - __clz(heads & (0xffffffffu >> (31 - lane)));   // start lane of my run
        const bool tail = lane == 31 || ((heads >> (lane + 1)) & 1u);
        // longest run in the warp bounds the number of scan steps (warp-uniform)
        const int run_len = lane - my_head + 1;
        int maxrun = run_len;
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
        for (int c = 0; c < 8; c += 2) {
          if (PAIR)
            nsr_red_corner_pair(grad, idx[c], idx[c + 1], v[2 * c], v[2 * c + 1], v[2 * c + 2], v[2 * c + 3]);
          else {
            nsr_red_add_f32x2(grad + 2 * (size_t)idx[c], v[2 * c], v[2 * c + 1]);
            nsr_red_add_f32x2(grad + 2 * (size_t)idx[c + 1], v[2 * c + 2], v[2 * c + 3]);
          }
        }
      }
    }
  }
}

template <int ML, int PAIR>
int launch_scatter_merged(const nsr_grid_t* g, const float* pos, const void* denc, float* grad, int64_t n, int ctas_per_sm, cudaStream_t st) {
  const int grid = (int)min((int64_t)nsr_sm_count() * ctas_per_sm, (n + 255) / 256);
  dbg_scatter_merged_kernel<ML, PAIR><<<grid, 256, 0, st>>>(*g, pos, (const __half2*)denc, grad, n);
  NSR_CHECK_LAUNCH("nsr_dbg_scatter_merged");
  return 0;
}

template <int V>
int launch_scatter(const nsr_grid_t* g, const float* pos, const void* denc, float* grad, int64_t n, cudaStream_t st) {
  const int64_t total = V >= 3 ? n * 16 : n;
  const int grid = (int)min((int64_t)nsr_sm_count() * 8, (total + 255) / 256);
  dbg_scatter_kernel<V><<<grid, 256, 0, st>>>(*g, pos, (const __half2*)denc, grad, n);
  NSR_CHECK_LAUNCH("nsr_dbg_scatter");
  return 0;
}

}  // namespace

extern "C" int nsr_dbg_scatter(const nsr_grid_t* g, const float* pos, const void* denc_h, float* grad, int64_t n, int variant,
                               void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  switch (variant) {
    case 0: return launch_scatter<0>(g, pos, denc_h, grad, n, st);
    case 1: return launch_scatter<1>(g, pos, denc_h, grad, n, st);
    case 2: return launch_scatter<2>(g, pos, denc_h, grad, n, st);
    case 3: return launch_scatter<3>(g, pos, denc_h, grad, n, st);
    case 4: return launch_scatter<4>(g, pos, denc_h, grad, n, st);
    case 5: return launch_scatter<5>(g, pos, denc_h, grad, n, st);
  }
  NSR_REQUIRE(false, "nsr_dbg_scatter: unknown variant %d", variant);
}

// variant = merge_levels * 2 + pair; ctas_per_sm x 256 threads resident per SM (occupancy sweep: how many scatter warps saturate the RED path)
extern "C" int nsr_dbg_scatter_merged(const nsr_grid_t* g, const float* pos, const void* denc_h, float* grad, int64_t n, int merge_levels,
                                      int pair, int ctas_per_sm, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
#define NSR_SM(ML)                                                                                   \
  case ML:                                                                                           \
    return pair ? launch_scatter_merged<ML, 1>(g, pos, denc_h, grad, n, ctas_per_sm, st)             \
                : launch_scatter_merged<ML, 0>(g, pos, denc_h, grad, n, ctas_per_sm, st);
  switch (merge_levels) {
    NSR_SM(0) NSR_SM(6) NSR_SM(8) NSR_SM(10)
  }
#undef NSR_SM
  NSR_REQUIRE(false, "nsr_dbg_scatter_merged: merge_levels must be 0, 6, 8 or 10 (got %d)", merge_levels);
}
