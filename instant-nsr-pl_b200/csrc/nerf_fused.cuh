// Shared pieces of the fused NeRF kernels (nerf_fused_fwd.cu / nerf_fused_bwd.cu): field description,
// shared-memory weight layout, sample -> position, the 16-level gather.
#pragma once
#include "mlp_warp.cuh"

// Weights of the two nerf-blender networks in shared memory (halves), padded rows:
//   density  W1 [64][32+8], W2 [16][64+8]            (geometry.mlp_network_config: 1 hidden layer)
//   colour   W1 [64][32+8], W2 [64][64+8], W3 [16][64+8]   (texture.mlp_network_config: 2 hidden layers)
constexpr int NF_LD32 = 32 + NSR_LDW_PAD;  // 40
constexpr int NF_OFF_DW1 = 0;
constexpr int NF_OFF_DW2 = NF_OFF_DW1 + 64 * NF_LD32;
constexpr int NF_OFF_CW1 = NF_OFF_DW2 + 16 * NSR_LD64;
constexpr int NF_OFF_CW2 = NF_OFF_CW1 + 64 * NF_LD32;
constexpr int NF_OFF_CW3 = NF_OFF_CW2 + 64 * NSR_LD64;
constexpr int NF_W_TOTAL = NF_OFF_CW3 + 16 * NSR_LD64;  // 12032 halves = 24064 B
constexpr int NF_DENSITY_PARAMS = 64 * 32 + 16 * 64;     // 3072
constexpr int NF_COLOR_PARAMS = 64 * 32 + 64 * 64 + 16 * 64;  // 7168

__device__ __forceinline__ void nf_stage_weights(__half* smem, const __half* __restrict__ dparams, const __half* __restrict__ cparams,
                                                 bool with_color) {
  const int tid = threadIdx.x, nt = blockDim.x;
  nsr_stage_matrix(smem + NF_OFF_DW1, dparams, 64, 32, tid, nt);
  nsr_stage_matrix(smem + NF_OFF_DW2, dparams + 64 * 32, 16, 64, tid, nt);
  if (with_color) {
    nsr_stage_matrix(smem + NF_OFF_CW1, cparams, 64, 32, tid, nt);
    nsr_stage_matrix(smem + NF_OFF_CW2, cparams + 64 * 32, 64, 64, tid, nt);
    nsr_stage_matrix(smem + NF_OFF_CW3, cparams + 64 * 32 + 64 * 64, 16, 64, tid, nt);
  }
}

// network variants of the two-pass field kernels (template parameter NET): both use the smem weight layout above
constexpr int NF_NET_FULLY_FUSED = 0;  // tcnn FullyFusedMLP (nerf-blender / nerf-colmap): bias-free, fp16 network outputs
constexpr int NF_NET_VANILLA = 1;      // the reference's VanillaMLP (NeuS learned background): fp32 biases, fp32 network outputs

// fp32 biases of the VanillaMLP variant in smem (floats): density b1 [64] | b2 [16] | colour b1 [64] | b2 [64] | b3 [16]
// (the density and colour vectors are the nsr_bg_field_* dbias [80] and cbias [144]; outputs padded to 16 with zero biases)
constexpr int NF_B_D1 = 0, NF_B_D2 = 64, NF_B_C1 = 80, NF_B_C2 = 144, NF_B_C3 = 208, NF_B_TOTAL = 224;

__device__ __forceinline__ void nf_stage_bias(float* bias_sm, const float* __restrict__ dbias, const float* __restrict__ cbias, bool with_color) {
  for (int i = threadIdx.x; i < (with_color ? NF_B_TOTAL : NF_B_C1); i += blockDim.x) bias_sm[i] = i < NF_B_C1 ? dbias[i] : cbias[i - NF_B_C1];
}

// accumulators of MT 16-row tiles start from zero (FullyFused) or from the fp32 bias of their column (VanillaMLP)
template <int NET, int MT, int NT>
__device__ __forceinline__ void nf_init_acc(float (&acc)[MT][NT][4], const float* bias_sm) {
  if (NET == NF_NET_VANILLA) {
    const int c2 = (threadIdx.x & 3) * 2;
#pragma unroll
    for (int n = 0; n < NT; ++n) {
      const float b0 = bias_sm[n * 8 + c2], b1 = bias_sm[n * 8 + c2 + 1];
#pragma unroll
      for (int m = 0; m < MT; ++m) acc[m][n][0] = b0, acc[m][n][1] = b1, acc[m][n][2] = b0, acc[m][n][3] = b1;
    }
  } else {
    nsr_zero_acc(acc);
  }
}

// contraction codes of nsr_nerf_t::contraction (nerfacc.ContractionType)
constexpr int NF_AABB = 0;
constexpr int NF_UNBOUNDED_SPHERE = 2;

// world position -> [0,1]^3 under UN_BOUNDED_SPHERE, in the op order of contract_to_unisphere (models/fields.py): scale to [0,1]
// (add, true division), v = 2u - 1, |v| > 1 -> (2 - 1/|v|) * (v / |v|), v/4 + 1/2
__device__ __forceinline__ void nf_contract_sphere(float radius, float& x, float& y, float& z) {
  const float span = 2.f * radius;
  float vx = __fsub_rn(__fmul_rn(__fdiv_rn(__fadd_rn(x, radius), span), 2.f), 1.f);
  float vy = __fsub_rn(__fmul_rn(__fdiv_rn(__fadd_rn(y, radius), span), 2.f), 1.f);
  float vz = __fsub_rn(__fmul_rn(__fdiv_rn(__fadd_rn(z, radius), span), 2.f), 1.f);
  const float mag = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(vx, vx), __fmul_rn(vy, vy)), __fmul_rn(vz, vz)));
  if (mag > 1.f) {
    const float s = __fsub_rn(2.f, __fdiv_rn(1.f, mag));
    vx = __fmul_rn(s, __fdiv_rn(vx, mag));
    vy = __fmul_rn(s, __fdiv_rn(vy, mag));
    vz = __fmul_rn(s, __fdiv_rn(vz, mag));
  }
  x = __fadd_rn(__fmul_rn(vx, 0.25f), 0.5f);
  y = __fadd_rn(__fmul_rn(vy, 0.25f), 0.5f);
  z = __fadd_rn(__fmul_rn(vz, 0.25f), 0.5f);
}

// world position -> unit-cube position of the field (contract_to_unisphere: models/geometry.py:17-19)
template <int CT>
__device__ __forceinline__ void nf_contract(const nsr_nerf_t& P, float& x, float& y, float& z) {
  if (CT == NF_UNBOUNDED_SPHERE) {
    nf_contract_sphere(P.radius, x, y, z);
  } else {
    const float inv = 1.f / (2.f * P.radius);
    x = (x + P.radius) * inv;
    y = (y + P.radius) * inv;
    z = (z + P.radius) * inv;
  }
}

// sample (ray, t0, t1) -> unit-cube position (contract_to_unisphere, AABB: models/geometry.py:17-19)
template <int CT = NF_AABB>
__device__ __forceinline__ void nf_sample_position(const nsr_nerf_t& P, const float* __restrict__ rays, int ray, float t0, float t1,
                                                   float& x, float& y, float& z, float& dx, float& dy, float& dz) {
  const float* r = rays + (size_t)ray * 6;
  const float ox = __ldg(r + 0), oy = __ldg(r + 1), oz = __ldg(r + 2);
  dx = __ldg(r + 3); dy = __ldg(r + 4); dz = __ldg(r + 5);
  const float mid = (t0 + t1) * 0.5f;
  x = fmaf(dx, mid, ox);
  y = fmaf(dy, mid, oy);
  z = fmaf(dz, mid, oz);
  nf_contract<CT>(P, x, y, z);
}

// x-adjacent corner pair (i0 = x bit 0, i1 = x bit 1) of one (y,z) combination.
// One aligned 8-byte load fetches entry i0 and its neighbour i0^1; when x is even that neighbour IS i1
// (hashed: (cx+1)^A == (cx^A)^1; dense: i0+1), so half of all pairs need a single request instead of two.
struct NfPair {
  uint2 pr;       // entries (i0 & ~1, i0 | 1)
  uint32_t extra; // entry i1 when not paired
  uint32_t i0;
  bool paired;
};

__device__ __forceinline__ uint32_t nf_dense_mod(uint32_t i, uint32_t size) {
  if (i >= size) i -= size;   // in-range inputs overshoot by less than one table length (SURVEY 8a wrap corner)
  if (i >= size) i %= size;   // out-of-range inputs: rare slow path
  return i;
}

__device__ __forceinline__ void nf_issue_pair(const uint32_t* __restrict__ table_u32, uint32_t i0, uint32_t i1, NfPair& p) {
  p.i0 = i0;
  p.paired = (i1 == (i0 ^ 1u));
  p.pr = __ldg(reinterpret_cast<const uint2*>(table_u32 + (i0 & ~1u)));
  p.extra = 0u;
  if (!p.paired) p.extra = __ldg(table_u32 + i1);
}

__device__ __forceinline__ void nf_pair_values(const NfPair& p, float2& v0, float2& v1) {
  const uint32_t a = (p.i0 & 1u) ? p.pr.y : p.pr.x;
  const uint32_t b = p.paired ? ((p.i0 & 1u) ? p.pr.x : p.pr.y) : p.extra;
  v0 = __half22float2(*reinterpret_cast<const __half2*>(&a));
  v1 = __half22float2(*reinterpret_cast<const __half2*>(&b));
}

// paired + batched variant kept for tools/gather_bench.py (measured: no faster than the plain loop below -- every
// variant converges to the same ~82 us / 446 k samples once occupancy is not the limit, see DESIGN.md "Gather").
template <int L, int NB>
__device__ __forceinline__ void nf_gather_paired(const nsr_grid_t& g, const __half2* __restrict__ table, float x, float y, float z,
                                                 uint32_t (&f)[L]) {
  static_assert(L % NB == 0, "level count must be a multiple of the batch");
  const uint32_t* tu = reinterpret_cast<const uint32_t*>(table);
#pragma unroll
  for (int l0 = 0; l0 < L; l0 += NB) {
    NfPair pairs[NB][4];
    float fr[NB][3];
#pragma unroll
    for (int j = 0; j < NB; ++j) {
      const LevelInfo li = nsr_level(g, l0 + j);
      uint32_t cx, cy, cz;
      nsr_pos_fract(x, li.scale, cx, fr[j][0]);
      nsr_pos_fract(y, li.scale, cy, fr[j][1]);
      nsr_pos_fract(z, li.scale, cz, fr[j][2]);
      if (li.dense) {
        const uint32_t r = li.res, r2 = li.res * li.res;
        const uint32_t b = cx + cy * r + cz * r2;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const uint32_t i = b + (q & 1) * r + (q >> 1) * r2;
          nf_issue_pair(tu, nf_dense_mod(i, li.size) + li.offset, nf_dense_mod(i + 1u, li.size) + li.offset, pairs[j][q]);
        }
      } else {
        const uint32_t m = li.size - 1u;
        const uint32_t hy0 = cy * NSR_PRIME_Y, hy1 = (cy + 1u) * NSR_PRIME_Y;
        const uint32_t hz0 = cz * NSR_PRIME_Z, hz1 = (cz + 1u) * NSR_PRIME_Z;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const uint32_t A = ((q & 1) ? hy1 : hy0) ^ ((q >> 1) ? hz1 : hz0);
          nf_issue_pair(tu, ((cx ^ A) & m) + li.offset, (((cx + 1u) ^ A) & m) + li.offset, pairs[j][q]);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < NB; ++j) {
      const float fx = fr[j][0], fy = fr[j][1], fz = fr[j][2];
      float a0 = 0.f, a1 = 0.f;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float2 v0, v1;
        nf_pair_values(pairs[j][q], v0, v1);
        const float wyz = ((q & 1) ? fy : 1.f - fy) * ((q >> 1) ? fz : 1.f - fz);
        const float w0 = (1.f - fx) * wyz, w1 = fx * wyz;
        a0 = fmaf(w0, v0.x, a0);
        a1 = fmaf(w0, v0.y, a1);
        a0 = fmaf(w1, v1.x, a0);
        a1 = fmaf(w1, v1.y, a1);
      }
      f[l0 + j] = nsr_pack_h2(a0, a1);
    }
  }
}

// all levels of one sample; features packed as half2 per level (fp16 = what tcnn's encoding emits)
template <int L>
__device__ __forceinline__ void nf_gather(const nsr_grid_t& g, const __half2* __restrict__ table, float x, float y, float z,
                                          uint32_t (&f)[L]) {
#pragma unroll
  for (int l = 0; l < L; ++l) {
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
}

// latency-oriented variant: all loads of NB levels are issued before any is consumed (8*NB requests in flight per thread).
// Used by the per-ray forward kernel, whose run time is set by the serial chunk chain of the longest rays; the
// throughput-bound sample-tile kernels keep the plain loop (tools/gather_bench.py: no difference at full occupancy).
template <int L, int NB>
__device__ __forceinline__ void nf_gather_batched(const nsr_grid_t& g, const __half2* __restrict__ table, float x, float y, float z,
                                                  uint32_t (&f)[L]) {
  static_assert(L % NB == 0, "level count must be a multiple of the batch");
  const uint32_t* tu = reinterpret_cast<const uint32_t*>(table);
#pragma unroll
  for (int l0 = 0; l0 < L; l0 += NB) {
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
      for (int c = 0; c < 8; ++c) raw[j][c] = __ldg(tu + idx[c]);
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
}

// write one 32-feature row (16 packed half2) of a [rows][NF_LD32] smem tile
__device__ __forceinline__ void nf_store_row32(__half* tile, int row, const uint32_t (&f)[16]) {
  uint4* p = reinterpret_cast<uint4*>(tile + row * NF_LD32);
  p[0] = make_uint4(f[0], f[1], f[2], f[3]);
  p[1] = make_uint4(f[4], f[5], f[6], f[7]);
  p[2] = make_uint4(f[8], f[9], f[10], f[11]);
  p[3] = make_uint4(f[12], f[13], f[14], f[15]);
}

__device__ __forceinline__ float nf_half_lo(uint32_t v) { return __low2float(*reinterpret_cast<const __half2*>(&v)); }
__device__ __forceinline__ float nf_half_hi(uint32_t v) { return __high2float(*reinterpret_cast<const __half2*>(&v)); }
