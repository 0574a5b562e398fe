// Shared device/host helpers for the nsr_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/nsr_b200.h"

#define NSR_PRIME_Y 2654435761u
#define NSR_PRIME_Z 805459861u

void nsr_set_error(const char* fmt, ...);

#define NSR_CHECK_LAUNCH(name)                                              \
  do {                                                                      \
    cudaError_t e__ = cudaGetLastError();                                   \
    if (e__ != cudaSuccess) {                                               \
      nsr_set_error("%s: launch failed: %s", name, cudaGetErrorString(e__)); \
      return 2;                                                             \
    }                                                                       \
  } while (0)

#define NSR_REQUIRE(cond, ...)      \
  do {                              \
    if (!(cond)) {                  \
      nsr_set_error(__VA_ARGS__);   \
      return 1;                     \
    }                               \
  } while (0)

int nsr_sm_count();

static inline int nsr_blocks(int64_t n, int threads) { return (int)((n + threads - 1) / threads); }

// ------------------------------------------------------------------------------------------------
// Hash-grid corner addressing (tiny-cuda-nn Grid/Hash/Linear semantics; oracle/hashgrid.py).
// ------------------------------------------------------------------------------------------------
struct LevelInfo {
  float scale;
  uint32_t res, size, offset;
  bool dense;
};

__device__ __forceinline__ LevelInfo nsr_level(const nsr_grid_t& g, int l) {
  LevelInfo li;
  li.scale = g.scale[l];
  li.res = g.res[l];
  li.size = g.size[l];
  li.offset = g.offset[l];
  li.dense = (g.dense_mask >> l) & 1u;
  return li;
}

// pos = fma(scale, x, 0.5); cell = floor(pos); frac = pos - cell
__device__ __forceinline__ void nsr_pos_fract(float x, float scale, uint32_t& cell, float& frac) {
  float p = __fmaf_rn(scale, x, 0.5f);
  float fl = floorf(p);
  cell = (uint32_t)(int)fl;
  frac = p - fl;
}

// entry indices (absolute, in entries) of the 8 corners; corner c = bx | by<<1 | bz<<2
__device__ __forceinline__ void nsr_corner_indices(const LevelInfo& li, uint32_t cx, uint32_t cy, uint32_t cz,
                                                   uint32_t (&idx)[8]) {
  if (li.dense) {
    const uint32_t r = li.res, r2 = li.res * li.res;
    const uint32_t b = cx + cy * r + cz * r2;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      uint32_t i = b + (c & 1) + ((c >> 1) & 1) * r + ((c >> 2) & 1) * r2;
      // i % size without the integer division: a dense level has res^3 <= size, so an in-range cell gives i < 2 size (res >= 2) and
      // i % size == i - (i >= size) * size; anything else (a NaN / out-of-box position) is clamped first and stays in bounds.  The
      // integer division was a visible share of the per-ray forward kernel's instructions.
      i = min(i, 2u * li.size - 1u);          // (branch-free: clamp, then one conditional subtract)
      i -= i >= li.size ? li.size : 0u;
      idx[c] = i + li.offset;
    }
  } else {
    const uint32_t m = li.size - 1u;  // hashed levels always have size == 2^log2_hashmap_size
    const uint32_t hx0 = cx, hx1 = cx + 1u;
    const uint32_t hy0 = cy * NSR_PRIME_Y, hy1 = (cy + 1u) * NSR_PRIME_Y;
    const uint32_t hz0 = cz * NSR_PRIME_Z, hz1 = (cz + 1u) * NSR_PRIME_Z;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      uint32_t h = ((c & 1) ? hx1 : hx0) ^ (((c >> 1) & 1) ? hy1 : hy0) ^ (((c >> 2) & 1) ? hz1 : hz0);
      idx[c] = (h & m) + li.offset;
    }
  }
}

__device__ __forceinline__ float nsr_corner_weight(int c, float fx, float fy, float fz) {
  return ((c & 1) ? fx : 1.f - fx) * (((c >> 1) & 1) ? fy : 1.f - fy) * (((c >> 2) & 1) ? fz : 1.f - fz);
}

// d(weight)/d(frac_d) for axis d
__device__ __forceinline__ float nsr_corner_dweight(int c, int d, float fx, float fy, float fz) {
  float wx = (c & 1) ? fx : 1.f - fx, wy = ((c >> 1) & 1) ? fy : 1.f - fy, wz = ((c >> 2) & 1) ? fz : 1.f - fz;
  float sx = (c & 1) ? 1.f : -1.f, sy = ((c >> 1) & 1) ? 1.f : -1.f, sz = ((c >> 2) & 1) ? 1.f : -1.f;
  return d == 0 ? sx * wy * wz : (d == 1 ? wx * sy * wz : wx * wy * sz);
}

// vectorised fp32 reduction into global memory: one 8-byte RED per corner (sm_90+)
__device__ __forceinline__ void nsr_red_add_f32x2(float* addr, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

// 16-byte RED: two adjacent table entries (F = 2 features each) in one request; addr must be 16-byte aligned (sm_90+)
__device__ __forceinline__ void nsr_red_add_f32x4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// the two x-adjacent corners (i0 = x bit 0, i1 = x bit 1) of one (y, z) combination: when i1 == i0 ^ 1 (hashed levels: cx even;
// dense levels: i0 even) the entries are neighbours in memory and one 16-byte RED carries both, otherwise two 8-byte REDs.
__device__ __forceinline__ void nsr_red_corner_pair(float* grad_table, uint32_t i0, uint32_t i1, float a0, float a1, float b0, float b1) {
  if (i1 == (i0 ^ 1u)) {
    if (i0 & 1u)
      nsr_red_add_f32x4(grad_table + 2 * (size_t)i1, b0, b1, a0, a1);
    else
      nsr_red_add_f32x4(grad_table + 2 * (size_t)i0, a0, a1, b0, b1);
  } else {
    nsr_red_add_f32x2(grad_table + 2 * (size_t)i0, a0, a1);
    nsr_red_add_f32x2(grad_table + 2 * (size_t)i1, b0, b1);
  }
}

__device__ __forceinline__ float2 nsr_ld_table(const __half2* table, uint32_t idx) {
  return __half22float2(__ldg(table + idx));
}

// ------------------------------------------------------------------------------------------------
// Warp-level tensor-core primitives (legacy HMMA path; fp16 in, fp32 accumulate)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void nsr_mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void nsr_ldmatrix_x4(uint32_t (&r)[4], const void* smem_ptr) {
  uint32_t addr = (uint32_t)__cvta_generic_to_shared(smem_ptr);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}

__device__ __forceinline__ void nsr_ldmatrix_x4_trans(uint32_t (&r)[4], const void* smem_ptr) {
  uint32_t addr = (uint32_t)__cvta_generic_to_shared(smem_ptr);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}

__device__ __forceinline__ void nsr_ldmatrix_x2(uint32_t& r0, uint32_t& r1, const void* smem_ptr) {
  uint32_t addr = (uint32_t)__cvta_generic_to_shared(smem_ptr);
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0,%1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(addr));
}

__device__ __forceinline__ void nsr_ldmatrix_x2_trans(uint32_t& r0, uint32_t& r1, const void* smem_ptr) {
  uint32_t addr = (uint32_t)__cvta_generic_to_shared(smem_ptr);
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(addr));
}

__device__ __forceinline__ uint32_t nsr_pack_h2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// real spherical harmonics, degree 4 (16 coefficients) of the unit vector (x,y,z)
__device__ __forceinline__ void nsr_sh4(float x, float y, float z, float (&s)[16]) {
  const float xy = x * y, xz = x * z, yz = y * z, x2 = x * x, y2 = y * y, z2 = z * z;
  s[0] = 0.28209479177387814f;
  s[1] = -0.48860251190291987f * y;
  s[2] = 0.48860251190291987f * z;
  s[3] = -0.48860251190291987f * x;
  s[4] = 1.0925484305920792f * xy;
  s[5] = -1.0925484305920792f * yz;
  s[6] = 0.94617469575755997f * z2 - 0.31539156525251999f;
  s[7] = -1.0925484305920792f * xz;
  s[8] = 0.54627421529603959f * x2 - 0.54627421529603959f * y2;
  s[9] = 0.59004358992664352f * y * (-3.0f * x2 + y2);
  s[10] = 2.8906114426405538f * xy * z;
  s[11] = 0.45704579946446572f * y * (1.0f - 5.0f * z2);
  s[12] = 0.3731763325901154f * z * (5.0f * z2 - 3.0f);
  s[13] = 0.45704579946446572f * x * (1.0f - 5.0f * z2);
  s[14] = 1.4453057213202769f * z * (x2 - y2);
  s[15] = 0.59004358992664352f * x * (-x2 + 3.0f * y2);
}

// exclusive scan of int32 counts into int64 offsets[n+1] by ONE CTA (the "last CTA to finish" epilogues), optionally with
// `order`: the element indices bucketed by their number of 32-sample chunks, longest first (a longest-processing-time-first
// schedule for the per-ray kernel; order inside a bucket = index order, so the result is deterministic).
// Fast path (n <= 32 * blockDim.x): every thread holds 32 strided elements in registers, the scan is shuffles + two
// barriers, the bucketing is ballots + one barrier -- no shared-memory atomics, no per-row barriers.
constexpr int NSR_ORDER_BINS = 8;
__device__ __forceinline__ int nsr_chunk_bin(int cnt) {
  const int ch = (cnt + 31) >> 5;  // 32-sample chunks the per-ray kernel would walk
  return ch >= 17 ? 0 : (ch >= 13 ? 1 : (ch >= 9 ? 2 : (ch >= 5 ? 3 : (ch >= 3 ? 4 : (ch == 2 ? 5 : (ch == 1 ? 6 : 7))))));
}

template <int ROWS>
__device__ __forceinline__ void nsr_block_scan_counts(const int32_t* counts, int64_t* offsets, int64_t n, int64_t* warp_sums /* smem [32] */,
                                                      int32_t* order = nullptr) {
  static_assert(ROWS <= 32, "at most 32 rows");
  __shared__ int s_rw[32][33];                       // [row][warp] inclusive warp totals
  __shared__ int64_t s_rowbase[33];
  __shared__ int s_wb[32][NSR_ORDER_BINS];           // [warp][bin] counts, then bases
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, T = blockDim.x, W = T >> 5;
  if (n <= (int64_t)ROWS * T) {
    int v[ROWS], incl[ROWS];
#pragma unroll
    for (int j = 0; j < ROWS; ++j) {
      const int64_t i = (int64_t)j * T + tid;
      v[j] = i < n ? __ldcg(counts + i) : 0;
    }
#pragma unroll
    for (int j = 0; j < ROWS; ++j) {
      int x = v[j];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += u;
      }
      incl[j] = x;
      if (lane == 31) s_rw[j][warp] = x;
    }
    __syncthreads();
    if (warp == 0) {  // lane j: total of row j, then exclusive scan over the rows
      int64_t tot = 0;
      if (lane < ROWS)
        for (int w = 0; w < W; ++w) tot += s_rw[lane][w];
      int64_t x = tot;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int64_t u = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += u;
      }
      s_rowbase[lane] = x - tot;
      if (lane == 31) s_rowbase[32] = x;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < ROWS; ++j) {
      const int64_t i = (int64_t)j * T + tid;
      if (i < n) {
        int64_t wbase = 0;
        for (int w = 0; w < warp; ++w) wbase += s_rw[j][w];
        offsets[i] = s_rowbase[j] + wbase + incl[j] - v[j];
      }
    }
    if (tid == 0) offsets[n] = s_rowbase[32];
    if (order != nullptr) {
      int run[NSR_ORDER_BINS];
#pragma unroll
      for (int b = 0; b < NSR_ORDER_BINS; ++b) run[b] = 0;
#pragma unroll
      for (int j = 0; j < ROWS; ++j) {
        const bool ok = (int64_t)j * T + tid < n;
        const int bin = nsr_chunk_bin(v[j]);
#pragma unroll
        for (int b = 0; b < NSR_ORDER_BINS; ++b) run[b] += __popc(__ballot_sync(0xffffffffu, ok && bin == b));
      }
      if (lane < NSR_ORDER_BINS) {
        int mine = 0;
#pragma unroll
        for (int b = 0; b < NSR_ORDER_BINS; ++b)
          if (lane == b) mine = run[b];
        s_wb[warp][lane] = mine;
      }
      __syncthreads();
      if (tid == 0) {  // bases, bin-major: all of bin 0 (warp 0, 1, ...), then bin 1, ...; rows inside a warp keep their order
        int acc = 0;
        for (int b = 0; b < NSR_ORDER_BINS; ++b)
          for (int w = 0; w < W; ++w) {
            const int c = s_wb[w][b];
            s_wb[w][b] = acc;
            acc += c;
          }
      }
      __syncthreads();
#pragma unroll
      for (int b = 0; b < NSR_ORDER_BINS; ++b) run[b] = s_wb[warp][b];
#pragma unroll
      for (int j = 0; j < ROWS; ++j) {
        const int64_t i = (int64_t)j * T + tid;
        const bool ok = i < n;
        const int bin = nsr_chunk_bin(v[j]);
        int pos = 0;
#pragma unroll
        for (int b = 0; b < NSR_ORDER_BINS; ++b) {
          const uint32_t m = __ballot_sync(0xffffffffu, ok && bin == b);
          if (bin == b) pos = run[b] + __popc(m & ((1u << lane) - 1u));
          run[b] += __popc(m);
        }
        if (ok) order[pos] = (int32_t)i;
      }
    }
    return;
  }
  // ---- generic path (large n): contiguous chunk per thread; order = identity
  const int64_t per = (n + T - 1) / T;
  const int64_t b0 = (int64_t)tid * per, e0 = min(n, b0 + per);
  int64_t s0 = 0;
  for (int64_t i = b0; i < e0; ++i) s0 += __ldcg(counts + i);
  int64_t inc = s0;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t u = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += u;
  }
  if (lane == 31) warp_sums[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    int64_t w = lane < W ? warp_sums[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t u = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += u;
    }
    warp_sums[lane] = w;
  }
  __syncthreads();
  int64_t run = inc - s0 + (warp > 0 ? warp_sums[warp - 1] : 0);
  for (int64_t i = b0; i < e0; ++i) {
    offsets[i] = run;
    run += __ldcg(counts + i);
    if (order != nullptr) order[i] = (int32_t)i;
  }
  if (tid == T - 1) offsets[n] = warp_sums[W - 1];
}
