// Occupancy-grid ray marching: nerfacc 0.3.3 `ray_aabb_intersect` + `ray_marching` kernels
// (models/nerf.py:82-93, models/neus.py:153-169,209-220).
//
// THIS FILE IS COMPILED WITH -fmad=false: every float op below is a separate IEEE fp32 op (or an
// explicit __fmaf_rn) in exactly the order oracle/march.py performs it, so that the emitted sample
// SET is bit-identical to the oracle's.
//
// Design: instead of nerfacc's one-thread-per-ray serial march (<= ~1024 dependent iterations,
// long-tail divergence), the cone_angle == 0 case tests the step lattice in parallel -- one warp per
// ray, 32 lattice points per iteration, ballot + popc compaction -- against a packed BITfield
// (128^3 bits = 256 KB, L1/L2 resident; nerfacc reads 2 MB of bools).  Two passes (count, write)
// around a device-side exclusive scan keep nerfacc's exact-size, ray-ordered output contract.
#include "march.cuh"

namespace {

__device__ __forceinline__ bool occupied(const nsr_march_t& p, const uint32_t* __restrict__ bits, float px, float py, float pz) {
  const float lx = p.roi[0], ly = p.roi[1], lz = p.roi[2], hx = p.roi[3], hy = p.roi[4], hz = p.roi[5];
  // unit-cube coordinate = (p - lo) * (1 / (hi - lo)) with the reciprocal rounded to fp32 once (oracle/march.py does the same)
  float ux = (px - lx) * (1.f / (hx - lx)), uy = (py - ly) * (1.f / (hy - ly)), uz = (pz - lz) * (1.f / (hz - lz));
  if (p.contraction == 0) {
    if (!(px >= lx && px <= hx && py >= ly && py <= hy && pz >= lz && pz <= hz)) return false;
  } else {
    float vx = ux * 2.f - 1.f, vy = uy * 2.f - 1.f, vz = uz * 2.f - 1.f;
    const float n = sqrtf((vx * vx + vy * vy) + vz * vz);
    if (n > 1.f) {
      const float s = 2.f - 1.f / n;
      vx = s * (vx / n);
      vy = s * (vy / n);
      vz = s * (vz / n);
    }
    ux = vx * 0.25f + 0.5f;
    uy = vy * 0.25f + 0.5f;
    uz = vz * 0.25f + 0.5f;
  }
  const int R = p.res;
  const float fR = (float)R;
  int cx = (int)(ux * fR), cy = (int)(uy * fR), cz = (int)(uz * fR);
  cx = min(max(cx, 0), R - 1);
  cy = min(max(cy, 0), R - 1);
  cz = min(max(cz, 0), R - 1);
  const uint32_t idx = (uint32_t)cx * R * R + (uint32_t)cy * R + (uint32_t)cz;
  return (__ldg(bits + (idx >> 5)) >> (idx & 31u)) & 1u;
}

__global__ void ray_aabb_kernel(const float* __restrict__ o, const float* __restrict__ d, const float* __restrict__ aabb,
                                float* __restrict__ t_min, float* __restrict__ t_max, int64_t n) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  float near = -INFINITY, far = INFINITY;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float oa = o[i * 3 + a], da = d[i * 3 + a];
    const float t1 = (aabb[a] - oa) / da, t2 = (aabb[3 + a] - oa) / da;
    near = fmaxf(near, fminf(t1, t2));
    far = fminf(far, fmaxf(t1, t2));
  }
  const float near0 = fmaxf(near, 0.f);
  const bool hit = far > near0;
  t_min[i] = hit ? near0 : 1e10f;
  t_max[i] = hit ? far : 1e10f;
}

constexpr int kMarchWarps = 8;
constexpr uint32_t kMaxLattice = 1u << 24;

// cone_angle == 0: warp-per-ray lattice test.  WRITE=false: counts; WRITE=true: samples at offsets.
template <bool WRITE>
__global__ void __launch_bounds__(kMarchWarps * 32) march_lattice_kernel(nsr_march_t p, const float* __restrict__ rays_o,
                                                                         const float* __restrict__ rays_d,
                                                                         const float* __restrict__ t_min,
                                                                         const float* __restrict__ t_max,
                                                                         const uint32_t* __restrict__ bits, int32_t* __restrict__ counts,
                                                                         const int64_t* __restrict__ offsets,
                                                                         int32_t* __restrict__ ray_indices, float* __restrict__ t_starts,
                                                                         float* __restrict__ t_ends, int64_t n_rays) {
  const int lane = threadIdx.x & 31;
  const int64_t ray = blockIdx.x * (int64_t)kMarchWarps + (threadIdx.x >> 5);
  if (ray >= n_rays) return;
  const float ox = rays_o[ray * 3 + 0], oy = rays_o[ray * 3 + 1], oz = rays_o[ray * 3 + 2];
  const float dx = rays_d[ray * 3 + 0], dy = rays_d[ray * 3 + 1], dz = rays_d[ray * 3 + 2];
  const float tmin = t_min[ray], tmax = t_max[ray], step = p.step;
  int64_t out = WRITE ? offsets[ray] : 0;
  int cnt = 0;
  for (uint32_t base = 0; base < kMaxLattice; base += 32) {
    const float k = (float)(base + lane);
    const float t0 = __fmaf_rn(k, step, tmin);
    const float t1 = __fmaf_rn(k + 1.f, step, tmin);
    const float tm = (t0 + t1) * 0.5f;
    const bool valid = tm < tmax;
    bool occ = false;
    if (valid) occ = occupied(p, bits, __fmaf_rn(tm, dx, ox), __fmaf_rn(tm, dy, oy), __fmaf_rn(tm, dz, oz));
    const uint32_t m = __ballot_sync(0xffffffffu, occ);
    if (WRITE) {
      if (occ) {
        const int64_t pos = out + __popc(m & ((1u << lane) - 1u));
        ray_indices[pos] = (int32_t)ray;
        t_starts[pos] = t0;
        t_ends[pos] = t1;
      }
      out += __popc(m);
    } else {
      cnt += __popc(m);
    }
    if (!__shfl_sync(0xffffffffu, (int)valid, 31)) break;  // tm is monotone in k
  }
  if (!WRITE && lane == 0) counts[ray] = cnt;
}

// cone_angle > 0 (contracted background pass): blind sequential stepping, one thread per ray
template <bool WRITE>
__global__ void march_seq_kernel(nsr_march_t p, const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                 const float* __restrict__ t_min, const float* __restrict__ t_max, const uint32_t* __restrict__ bits,
                                 int32_t* __restrict__ counts, const int64_t* __restrict__ offsets, int32_t* __restrict__ ray_indices,
                                 float* __restrict__ t_starts, float* __restrict__ t_ends, int64_t n_rays) {
  const int64_t ray = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (ray >= n_rays) return;
  const float ox = rays_o[ray * 3 + 0], oy = rays_o[ray * 3 + 1], oz = rays_o[ray * 3 + 2];
  const float dx = rays_d[ray * 3 + 0], dy = rays_d[ray * 3 + 1], dz = rays_d[ray * 3 + 2];
  const float tmax = t_max[ray], step = p.step, cone = p.cone_angle;
  int64_t out = WRITE ? offsets[ray] : 0;
  int cnt = 0;
  float t0 = t_min[ray];
  float t1 = t0 + fminf(fmaxf(t0 * cone, step), 1e10f);
  float tm = (t0 + t1) * 0.5f;
  for (int it = 0; it < (1 << 16) && tm < tmax; ++it) {
    if (occupied(p, bits, __fmaf_rn(tm, dx, ox), __fmaf_rn(tm, dy, oy), __fmaf_rn(tm, dz, oz))) {
      if (WRITE) {
        ray_indices[out] = (int32_t)ray;
        t_starts[out] = t0;
        t_ends[out] = t1;
        ++out;
      } else {
        ++cnt;
      }
    }
    t0 = t1;
    t1 = t0 + fminf(fmaxf(t0 * cone, step), 1e10f);
    tm = (t0 + t1) * 0.5f;
  }
  if (!WRITE) counts[ray] = cnt;
}

// exclusive scan of int32 counts into int64 offsets[n+1]; one CTA (n is a ray count: small)
template <int ROWS>
__global__ void __launch_bounds__(1024) scan_counts_kernel(const int32_t* __restrict__ counts, int64_t* __restrict__ offsets,
                                                           int32_t* __restrict__ order, int64_t n) {
  __shared__ int64_t warp_sums[32];
  nsr_block_scan_counts<ROWS>(counts, offsets, n, warp_sums, order);
}

// ------------------------------------------------------------------------------------------------
// Fused-path marcher (AABB, cone_angle == 0): ray -> (t_min, t_max) -> lattice occupancy masks in ONE kernel,
// with a coarse "any bit set in this 4^3 block" bitfield staged in shared memory so that empty space costs no
// global load, and the exclusive scan of the per-ray counts done by the last CTA to finish.  The write pass only
// expands the stored masks (no second round of occupancy tests).  Same arithmetic as ray_aabb_kernel +
// march_lattice_kernel above => identical sample sets.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kMarchWarps * 32) march_rays_mask_kernel(nsr_march_t p, const float* __restrict__ rays,
                                                                           const float* __restrict__ jitter,
                                                                           const uint32_t* __restrict__ bits,
                                                                           const uint32_t* __restrict__ coarse, uint32_t* __restrict__ masks,
                                                                           int words, float* __restrict__ t_min_out,
                                                                           int32_t* __restrict__ counts, int64_t n_rays,
                                                                           int64_t* __restrict__ offsets, unsigned long long* __restrict__ alloc_total,
                                                                           int32_t* __restrict__ bin_counts, int32_t* __restrict__ order_bins) {
  __shared__ uint32_t s_coarse[1024];  // (R/4)^3 bits, R <= 128
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int Rc = p.res >> 2;
  const bool use_coarse = coarse != nullptr;
  if (use_coarse) {
    const int nw = (Rc * Rc * Rc + 31) >> 5;
    for (int i = threadIdx.x; i < nw; i += blockDim.x) s_coarse[i] = __ldg(coarse + i);
    __syncthreads();
  }
  const int64_t ray = blockIdx.x * (int64_t)kMarchWarps + warp;
  if (ray < n_rays) {
    const float* rr = rays + ray * 6;
    const float ox = rr[0], oy = rr[1], oz = rr[2], dx = rr[3], dy = rr[4], dz = rr[5];
    // ray_aabb_kernel, verbatim
    float near = -INFINITY, far = INFINITY;
    {
      const float o3[3] = {ox, oy, oz}, d3[3] = {dx, dy, dz};
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        const float t1 = (p.roi[a] - o3[a]) / d3[a], t2 = (p.roi[3 + a] - o3[a]) / d3[a];
        near = fmaxf(near, fminf(t1, t2));
        far = fminf(far, fmaxf(t1, t2));
      }
    }
    const float near0 = fmaxf(near, 0.f);
    const bool hit = far > near0;
    float tmin = hit ? near0 : 1e10f;
    const float tmax = hit ? far : 1e10f;
    const float step = p.step;
    if (jitter != nullptr) tmin = tmin + jitter[ray] * step;  // stratified: one draw per ray (unfused mul, add)
    const float lx = p.roi[0], ly = p.roi[1], lz = p.roi[2], hx = p.roi[3], hy = p.roi[4], hz = p.roi[5];
    const int R = p.res;
    const float fR = (float)R;
    const float ix = 1.f / (hx - lx), iy = 1.f / (hy - ly), iz = 1.f / (hz - lz);
    int cnt = 0;
    uint32_t* mrow = masks + ray * words;
    int w = 0;
    for (; w < words; ++w) {
      const float k = (float)(w * 32 + lane);
      const float t0 = __fmaf_rn(k, step, tmin);
      const float t1 = __fmaf_rn(k + 1.f, step, tmin);
      const float tm = (t0 + t1) * 0.5f;
      const bool valid = tm < tmax;
      bool occ = false;
      if (valid) {
        const float px = __fmaf_rn(tm, dx, ox), py = __fmaf_rn(tm, dy, oy), pz = __fmaf_rn(tm, dz, oz);
        if (px >= lx && px <= hx && py >= ly && py <= hy && pz >= lz && pz <= hz) {
          const float ux = (px - lx) * ix, uy = (py - ly) * iy, uz = (pz - lz) * iz;
          int cx = (int)(ux * fR), cy = (int)(uy * fR), cz = (int)(uz * fR);
          cx = min(max(cx, 0), R - 1);
          cy = min(max(cy, 0), R - 1);
          cz = min(max(cz, 0), R - 1);
          bool maybe = true;
          if (use_coarse) {
            const uint32_t ci = (uint32_t)(cx >> 2) * Rc * Rc + (uint32_t)(cy >> 2) * Rc + (uint32_t)(cz >> 2);
            maybe = (s_coarse[ci >> 5] >> (ci & 31u)) & 1u;
          }
          if (maybe) {
            const uint32_t idx = (uint32_t)cx * R * R + (uint32_t)cy * R + (uint32_t)cz;
            occ = (__ldg(bits + (idx >> 5)) >> (idx & 31u)) & 1u;
          }
        }
      }
      const uint32_t m = __ballot_sync(0xffffffffu, occ);
      if (lane == 0) mrow[w] = m;
      cnt += __popc(m);
      if (!__shfl_sync(0xffffffffu, (int)valid, 31)) {
        ++w;
        break;
      }
    }
    for (int z = w + lane; z < words; z += 32) mrow[z] = 0u;
    if (lane == 0) {
      counts[ray] = cnt;
      t_min_out[ray] = tmin;
      if (alloc_total != nullptr) {
        // nsr_march_rays_alloc: the ray reserves its slice of the sample buffers and its place in the longest-rays-first queue HERE (two
        // atomics per ray) instead of in a one-CTA scan kernel behind the marcher.  The slices are then in completion order, not ray order:
        // every consumer addresses samples as offsets[ray] + j, the ray-ordered view is the PACKED one (nsr_pack_kept).
        offsets[ray] = (int64_t)atomicAdd(alloc_total, (unsigned long long)cnt);
        const int b = nsr_chunk_bin(cnt);
        order_bins[(int64_t)b * n_rays + atomicAdd(bin_counts + b, 1)] = (int32_t)ray;
      }
    }
  }
}

__global__ void __launch_bounds__(kMarchWarps * 32) march_rays_expand_kernel(nsr_march_t p, const uint32_t* __restrict__ masks, int words,
                                                                             const float* __restrict__ t_min,
                                                                             const int64_t* __restrict__ offsets,
                                                                             int32_t* __restrict__ ray_indices, float* __restrict__ t_starts,
                                                                             float* __restrict__ t_ends, int64_t n_rays) {
  const int lane = threadIdx.x & 31;
  const int64_t ray = blockIdx.x * (int64_t)kMarchWarps + (threadIdx.x >> 5);
  if (ray >= n_rays) return;
  const int64_t beg = offsets[ray], end = offsets[ray + 1];  // offsets clamped to a buffer capacity truncate the tail rays
  if (end <= beg) return;
  const float tmin = t_min[ray], step = p.step;
  int64_t base = beg;
  for (int w0 = 0; w0 < words; w0 += 32) {
    const int w = w0 + lane;
    uint32_t m = w < words ? masks[ray * words + w] : 0u;
    const int c = __popc(m);
    int incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    int64_t pos = base + incl - c;
    while (m) {
      const int b = __ffs(m) - 1;
      m &= m - 1u;
      const float k = (float)(w * 32 + b);
      if (pos < end) {
        ray_indices[pos] = (int32_t)ray;
        t_starts[pos] = nsr_lattice_t(k, step, tmin);
        t_ends[pos] = nsr_lattice_t(k + 1.f, step, tmin);
      }
      ++pos;
    }
    base += __shfl_sync(0xffffffffu, incl, 31);
  }
}

// ------------------------------------------------------------------------------------------------
// Fused-path marcher for cone_angle > 0 (unbounded scenes): march_seq_kernel's serial recurrence, one warp per ray.  The step
// t1 = t0 + min(max(t0 * cone, step), 1e10) depends on the previous one, so it is not reassociated: every lane runs the SAME fp32
// chain over a 32-step chunk (arithmetic only, no loads) and lane k keeps step k (nsr_cone_chunk, march.cuh); the 32 occupancy tests of
// a chunk -- the loads -- then run in parallel.  The expand pass recomputes the chain instead of storing t per chunk.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kMarchWarps * 32) march_cone_mask_kernel(nsr_march_t p, const float* __restrict__ rays,
                                                                           const float* __restrict__ jitter, const float* __restrict__ t_min_in,
                                                                           const float* __restrict__ t_max_in, float near, float far,
                                                                           const uint32_t* __restrict__ bits, uint32_t* __restrict__ masks,
                                                                           int words, float* __restrict__ t_start, int32_t* __restrict__ counts,
                                                                           int64_t n_rays) {
  const int lane = threadIdx.x & 31;
  const int64_t ray = blockIdx.x * (int64_t)kMarchWarps + (threadIdx.x >> 5);
  if (ray >= n_rays) return;
  const float* rr = rays + ray * 6;
  const float ox = rr[0], oy = rr[1], oz = rr[2], dx = rr[3], dy = rr[4], dz = rr[5];
  const float step = p.step, cone = p.cone_angle;
  // nerfacc.ray_marching's order: interval (or [0, 1e10)), clamp to the near / far planes, then the stratified offset (unfused mul, add)
  float tmin = fmaxf(t_min_in ? t_min_in[ray] : 0.f, near);
  const float tmax = fminf(t_max_in ? t_max_in[ray] : 1e10f, far);
  if (jitter != nullptr) tmin = tmin + jitter[ray] * step;
  uint32_t* mrow = masks + ray * words;
  float t = tmin;
  int cnt = 0;
  for (int w = 0; w < words; ++w) {
    float t0 = 0.f, t1 = 0.f;
    t = nsr_cone_chunk(t, cone, step, lane, t0, t1);
    const float tm = (t0 + t1) * 0.5f;
    const bool valid = tm < tmax;
    const bool occ = valid && occupied(p, bits, __fmaf_rn(tm, dx, ox), __fmaf_rn(tm, dy, oy), __fmaf_rn(tm, dz, oz));
    const uint32_t m = __ballot_sync(0xffffffffu, occ);
    if (lane == 0) mrow[w] = m;
    cnt += __popc(m);
    if (!__shfl_sync(0xffffffffu, (int)valid, 31)) break;  // tm is monotone along the ray; words past here are never read
  }
  if (lane == 0) {
    counts[ray] = cnt;
    t_start[ray] = tmin;
  }
}

__global__ void __launch_bounds__(kMarchWarps * 32) march_cone_expand_kernel(nsr_march_t p, const uint32_t* __restrict__ masks, int words,
                                                                             const float* __restrict__ t_start,
                                                                             const int64_t* __restrict__ offsets, int32_t* __restrict__ ray_indices,
                                                                             float* __restrict__ t_starts, float* __restrict__ t_ends, int64_t cap,
                                                                             int32_t* __restrict__ overflow, int64_t n_rays) {
  const int lane = threadIdx.x & 31;
  const int64_t ray = blockIdx.x * (int64_t)kMarchWarps + (threadIdx.x >> 5);
  if (ray >= n_rays) return;
  const int64_t beg = offsets[ray], end = offsets[ray + 1];
  if (end <= beg) return;
  if (end > cap && overflow != nullptr && lane == 0) *overflow = 1;
  const float step = p.step, cone = p.cone_angle;
  const uint32_t* mrow = masks + ray * words;
  float t = t_start[ray];
  int64_t base = beg;
  for (int w = 0; w < words && base < end && base < cap; ++w) {
    float t0 = 0.f, t1 = 0.f;
    t = nsr_cone_chunk(t, cone, step, lane, t0, t1);
    const uint32_t m = mrow[w];
    if ((m >> lane) & 1u) {
      const int64_t pos = base + __popc(m & ((1u << lane) - 1u));
      if (pos < cap) {
        ray_indices[pos] = (int32_t)ray;
        t_starts[pos] = t0;
        t_ends[pos] = t1;
      }
    }
    base += __popc(m);
  }
}

template <bool WRITE>
int launch_march(const nsr_march_t* p, const float* rays_o, const float* rays_d, const float* t_min, const float* t_max,
                 const uint32_t* bits, int32_t* counts, const int64_t* offsets, int32_t* ray_indices, float* t_starts, float* t_ends,
                 int64_t n_rays, cudaStream_t st, const char* name) {
  NSR_REQUIRE(p != nullptr, "%s: march descriptor is NULL", name);
  NSR_REQUIRE(p->res >= 1 && p->res <= 1024, "%s: grid resolution %d out of range", name, p->res);
  NSR_REQUIRE(p->contraction == 0 || p->contraction == 2, "%s: contraction type %d not implemented (AABB=0, UN_BOUNDED_SPHERE=2)", name,
              p->contraction);
  NSR_REQUIRE(p->step > 0.f, "%s: render_step_size must be > 0", name);
  if (n_rays == 0) return 0;
  if (p->cone_angle == 0.f) {
    march_lattice_kernel<WRITE><<<nsr_blocks(n_rays, kMarchWarps), kMarchWarps * 32, 0, st>>>(
        *p, rays_o, rays_d, t_min, t_max, bits, counts, offsets, ray_indices, t_starts, t_ends, n_rays);
  } else {
    march_seq_kernel<WRITE><<<nsr_blocks(n_rays, 128), 128, 0, st>>>(*p, rays_o, rays_d, t_min, t_max, bits, counts, offsets,
                                                                      ray_indices, t_starts, t_ends, n_rays);
  }
  NSR_CHECK_LAUNCH(name);
  return 0;
}

}  // namespace

extern "C" int nsr_ray_aabb(const float* rays_o, const float* rays_d, const float* aabb6, float* t_min, float* t_max, int64_t n,
                            void* stream) {
  if (n == 0) return 0;
  ray_aabb_kernel<<<nsr_blocks(n, 256), 256, 0, (cudaStream_t)stream>>>(rays_o, rays_d, aabb6, t_min, t_max, n);
  NSR_CHECK_LAUNCH("nsr_ray_aabb");
  return 0;
}

extern "C" int nsr_march_count(const nsr_march_t* p, const float* rays_o, const float* rays_d, const float* t_min, const float* t_max,
                               const uint32_t* bits, int32_t* counts, int64_t n_rays, void* stream) {
  return launch_march<false>(p, rays_o, rays_d, t_min, t_max, bits, counts, nullptr, nullptr, nullptr, nullptr, n_rays,
                             (cudaStream_t)stream, "nsr_march_count");
}

extern "C" int nsr_march_write(const nsr_march_t* p, const float* rays_o, const float* rays_d, const float* t_min, const float* t_max,
                               const uint32_t* bits, const int64_t* offsets, int32_t* ray_indices, float* t_starts, float* t_ends,
                               int64_t n_rays, void* stream) {
  return launch_march<true>(p, rays_o, rays_d, t_min, t_max, bits, nullptr, offsets, ray_indices, t_starts, t_ends, n_rays,
                            (cudaStream_t)stream, "nsr_march_write");
}

static int launch_scan(const int32_t* counts, int64_t* offsets, int32_t* order, int64_t n, cudaStream_t st, const char* name) {
  if (n <= 8 * 1024)
    scan_counts_kernel<8><<<1, 1024, 0, st>>>(counts, offsets, order, n);
  else
    scan_counts_kernel<32><<<1, 1024, 0, st>>>(counts, offsets, order, n);
  NSR_CHECK_LAUNCH(name);
  return 0;
}

extern "C" int nsr_scan_counts(const int32_t* counts, int64_t* offsets, int64_t n, void* stream) {
  return launch_scan(counts, offsets, nullptr, n, (cudaStream_t)stream, "nsr_scan_counts");
}

extern "C" int nsr_scan_counts_order(const int32_t* counts, int64_t* offsets, int32_t* order, int64_t n, void* stream) {
  NSR_REQUIRE(order != nullptr, "nsr_scan_counts_order: order is NULL");
  return launch_scan(counts, offsets, order, n, (cudaStream_t)stream, "nsr_scan_counts_order");
}

// march + slice allocation + queue binning in one launch (see march_rays_mask_kernel).  alloc_total (uint64, zero on entry) ends as the number
// of marched samples; bin_counts int32[8] (zero on entry) / order_bins int32[8 * n]: rays grouped by 32-sample chunk count, longest group first.
extern "C" int nsr_march_rays_alloc(const nsr_march_t* p, const float* rays, const float* jitter, const uint32_t* bits, const uint32_t* coarse_bits,
                                    uint32_t* masks, int32_t words, float* t_min, int32_t* counts, int64_t* offsets, void* alloc_total,
                                    int32_t* bin_counts, int32_t* order_bins, int64_t n, void* stream) {
  NSR_REQUIRE(p != nullptr && p->contraction == 0 && p->cone_angle == 0.f, "nsr_march_rays_alloc: AABB roi and cone_angle == 0 only");
  NSR_REQUIRE(p->step > 0.f && p->res >= 1 && p->res <= 1024, "nsr_march_rays_alloc: bad step / resolution");
  NSR_REQUIRE(coarse_bits == nullptr || (p->res % 4 == 0 && p->res <= 128), "nsr_march_rays_alloc: coarse bits need res %% 4 == 0, res <= 128");
  NSR_REQUIRE(offsets != nullptr && alloc_total != nullptr && bin_counts != nullptr && order_bins != nullptr, "nsr_march_rays_alloc: NULL output");
  NSR_REQUIRE(words >= 1, "nsr_march_rays_alloc: words must be >= 1");
  if (n == 0) return 0;
  march_rays_mask_kernel<<<nsr_blocks(n, kMarchWarps), kMarchWarps * 32, 0, (cudaStream_t)stream>>>(*p, rays, jitter, bits, coarse_bits, masks, words, t_min,
                                                                                                  counts, n, offsets, (unsigned long long*)alloc_total,
                                                                                                  bin_counts, order_bins);
  NSR_CHECK_LAUNCH("nsr_march_rays_alloc");
  return 0;
}

extern "C" int nsr_march_rays_mask(const nsr_march_t* p, const float* rays, const float* jitter, const uint32_t* bits,
                                   const uint32_t* coarse_bits, uint32_t* masks, int32_t words, float* t_min_out, int32_t* counts,
                                   int64_t n_rays, void* stream) {
  NSR_REQUIRE(p != nullptr && p->contraction == 0 && p->cone_angle == 0.f, "nsr_march_rays_mask: AABB / cone_angle 0 only");
  NSR_REQUIRE(p->step > 0.f && p->res >= 1 && p->res <= 1024, "nsr_march_rays_mask: bad step / resolution");
  NSR_REQUIRE(coarse_bits == nullptr || (p->res % 4 == 0 && p->res <= 128), "nsr_march_rays_mask: coarse bits need res %% 4 == 0, res <= 128");
  NSR_REQUIRE(words >= 1, "nsr_march_rays_mask: words >= 1 is required");
  if (n_rays == 0) return 0;
  const int64_t blocks = (n_rays + kMarchWarps - 1) / kMarchWarps;
  march_rays_mask_kernel<<<(int)blocks, kMarchWarps * 32, 0, (cudaStream_t)stream>>>(*p, rays, jitter, bits, coarse_bits, masks, words,
                                                                                     t_min_out, counts, n_rays, nullptr, nullptr, nullptr, nullptr);
  NSR_CHECK_LAUNCH("nsr_march_rays_mask");
  return 0;
}

extern "C" int nsr_march_rays_expand(const nsr_march_t* p, const uint32_t* masks, int32_t words, const float* t_min, const int64_t* offsets,
                                     int32_t* ray_indices, float* t_starts, float* t_ends, int64_t n_rays, void* stream) {
  NSR_REQUIRE(p != nullptr, "nsr_march_rays_expand: descriptor is NULL");
  if (n_rays == 0) return 0;
  march_rays_expand_kernel<<<nsr_blocks(n_rays, kMarchWarps), kMarchWarps * 32, 0, (cudaStream_t)stream>>>(*p, masks, words, t_min, offsets,
                                                                                                           ray_indices, t_starts, t_ends,
                                                                                                           n_rays);
  NSR_CHECK_LAUNCH("nsr_march_rays_expand");
  return 0;
}

extern "C" int nsr_march_cone_mask(const nsr_march_t* p, const float* rays, const float* jitter, const float* t_min_in, const float* t_max_in,
                                   float near, float far, const uint32_t* bits, uint32_t* masks, int32_t words, float* t_start, int32_t* counts,
                                   int64_t n_rays, void* stream) {
  NSR_REQUIRE(p != nullptr, "nsr_march_cone_mask: march descriptor is NULL");
  NSR_REQUIRE(p->res >= 1 && p->res <= 1024, "nsr_march_cone_mask: grid resolution %d out of range", p->res);
  NSR_REQUIRE(p->contraction == 0 || p->contraction == 2, "nsr_march_cone_mask: contraction type %d not implemented (AABB=0, UN_BOUNDED_SPHERE=2)",
              p->contraction);
  NSR_REQUIRE(p->step > 0.f && p->cone_angle >= 0.f, "nsr_march_cone_mask: needs step > 0 and cone_angle >= 0");
  NSR_REQUIRE(words >= 1, "nsr_march_cone_mask: words must be >= 1");
  NSR_REQUIRE(rays != nullptr && bits != nullptr && masks != nullptr && t_start != nullptr && counts != nullptr, "nsr_march_cone_mask: NULL argument");
  if (n_rays == 0) return 0;
  march_cone_mask_kernel<<<nsr_blocks(n_rays, kMarchWarps), kMarchWarps * 32, 0, (cudaStream_t)stream>>>(
      *p, rays, jitter, t_min_in, t_max_in, near, far, bits, masks, words, t_start, counts, n_rays);
  NSR_CHECK_LAUNCH("nsr_march_cone_mask");
  return 0;
}

extern "C" int nsr_march_cone_expand(const nsr_march_t* p, const uint32_t* masks, int32_t words, const float* t_start, const int64_t* offsets,
                                     int32_t* ray_indices, float* t_starts, float* t_ends, int64_t cap, int32_t* overflow, int64_t n_rays,
                                     void* stream) {
  NSR_REQUIRE(p != nullptr && p->step > 0.f, "nsr_march_cone_expand: descriptor is NULL or step <= 0");
  NSR_REQUIRE(words >= 1 && cap >= 0, "nsr_march_cone_expand: needs words >= 1 and cap >= 0");
  if (n_rays == 0) return 0;
  march_cone_expand_kernel<<<nsr_blocks(n_rays, kMarchWarps), kMarchWarps * 32, 0, (cudaStream_t)stream>>>(
      *p, masks, words, t_start, offsets, ray_indices, t_starts, t_ends, cap, overflow, n_rays);
  NSR_CHECK_LAUNCH("nsr_march_cone_expand");
  return 0;
}

namespace {
// midpoints -> world positions, per-sample view directions and interval lengths (models/nerf.py:96-99, models/neus.py:222-225:
// positions = rays_o[ri] + rays_d[ri] * (t_starts + t_ends) / 2, dists = t_ends - t_starts) in one pass; this file is compiled
// without fma contraction, so the positions equal torch's mul-then-add bit for bit.
__global__ void __launch_bounds__(256) sample_points_kernel(const float* __restrict__ rays, const int32_t* __restrict__ ray_indices,
                                                            const float* __restrict__ t_starts, const float* __restrict__ t_ends,
                                                            float* __restrict__ positions, float* __restrict__ dirs,
                                                            float* __restrict__ dists, int64_t n_cap, const int64_t* __restrict__ n_dev) {
  const int64_t n = n_dev ? min(*n_dev, n_cap) : n_cap;
  const int64_t i = blockIdx.x * 256ll + threadIdx.x;
  if (i >= n) return;
  const float* r = rays + (size_t)ray_indices[i] * 6;
  const float t0 = t_starts[i], t1 = t_ends[i];
  const float mid = nsr_sample_mid(t0, t1);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float d = __ldg(r + 3 + c);
    positions[i * 3 + c] = nsr_sample_coord(__ldg(r + c), d, mid);
    if (dirs) dirs[i * 3 + c] = d;
  }
  if (dists) dists[i] = t1 - t0;
}
}  // namespace

extern "C" int nsr_sample_points(const float* rays, const int32_t* ray_indices, const float* t_starts, const float* t_ends,
                                 float* positions, float* dirs, float* dists, int64_t n, const int64_t* n_dev, void* stream) {
  NSR_REQUIRE(positions != nullptr, "nsr_sample_points: positions is NULL");
  if (n == 0) return 0;
  sample_points_kernel<<<nsr_blocks(n, 256), 256, 0, (cudaStream_t)stream>>>(rays, ray_indices, t_starts, t_ends, positions, dirs, dists, n, n_dev);
  NSR_CHECK_LAUNCH("nsr_sample_points");
  return 0;
}
