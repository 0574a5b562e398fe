// Distortion loss of mip-NeRF 360 (eq. 15) over packed samples sorted by ray -- what systems/nerf.py:103-106 and systems/neus.py:131-139
// compute with torch_efficient_distloss.flatten_eff_distloss.  Per ray, samples i in marching order (midpoints m non-decreasing):
//   L_ray = sum_i sum_j w_i w_j |m_i - m_j| + 1/3 sum_i w_i^2 d_i = sum_i [2 w_i S_i + 1/3 w_i^2 d_i]
//   S_i = sum_{j<i} w_j (m_i - m_j) = S_{i-1} + W_{<i} (m_i - m_{i-1})          (W_{<i}: exclusive prefix sum of w)
//   R_i = sum_{j>i} w_j (m_j - m_i) = R_{i+1} + W_{>i} (m_{i+1} - m_i)
//   loss = sum_rays L_ray / n_div,  n_div = ray_id[last live row] + 1 (= max(ray_id) + 1 for sorted ids)
//   dloss/dw_i = (2 (S_i + R_i) + 2/3 w_i d_i) / n_div
// The recurrences add non-negative terms only: no cancellation when the midpoints are large (unbounded scenes march to t = 1e4), unlike
// m_i * sum w_j - sum w_j m_j.  Segments come from the sorted ids alone: warp g owns every ray whose first row lies in [32 g, 32 g + 32);
// the rays that also end there take one pass of segmented warp scans, the one that runs on is walked 32 rows at a time.  No host synchronisation and nothing sized by the capacity is touched: rows at or past the live count
// (*n_dev, when given) are never read or written, so both entry points can sit inside a captured CUDA graph.
#include "common.cuh"

namespace {

constexpr int kThreads = 256;

struct DistIn {
  const float* w;          // weights (read at w_pos[i] when w_pos != NULL)
  const int64_t* w_pos;    // optional gather index of the weights (the fused NeRF path's loose layout)
  const float* a;          // midpoints (t_mode 0) or t_starts (t_mode 1)
  const float* b;          // intervals (t_mode 0) or t_ends (t_mode 1)
  const int32_t* rid;      // ray ids, non-decreasing over the live rows
  int32_t t_mode;
};

__device__ __forceinline__ int64_t live_rows(int64_t n, const int64_t* n_dev) { return n_dev ? min(max(*n_dev, (int64_t)0), n) : n; }

// One row of a ray's chunk: weight, midpoint, interval, where its weight lives, and whether it belongs to ray `id`.  The loads do not wait
// for the id test (rows < n_live are all live), so a batch of chunks has all its loads in flight at once.  The midpoint / interval of the
// (t_start, t_end) form round exactly like the exact-size dicts' (ts + te) / 2 and te - ts.
struct Row {
  float w, m, d;
  int64_t p;
  bool ok;
};

__device__ __forceinline__ Row load_row(const DistIn& in, int64_t j, int32_t id, int64_t n_live) {
  Row r{0.f, 0.f, 0.f, j, false};
  if (j < n_live) {
    r.p = in.w_pos ? in.w_pos[j] : j;
    const float x = in.a[j], y = in.b[j];
    r.ok = in.rid[j] == id;   // sorted ids: the rows of the ray are a prefix of the chunk
    const float w = in.w[r.p];
    if (r.ok) {
      r.w = w;
      r.m = in.t_mode ? (x + y) * 0.5f : x;
      r.d = in.t_mode ? y - x : y;
    }
  }
  return r;
}

__device__ __forceinline__ float warp_incl_scan(float v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  return v;
}

__device__ __forceinline__ float warp_incl_suffix_scan(float v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_down_sync(0xffffffffu, v, o);
    if (lane + o < 32) v += t;
  }
  return v;
}

// Chunks of 32 rows are loaded kBatch at a time: the walk of a long ray (> 1000 samples on unbounded scenes) is one warp's loop, and its
// time is load latency unless several chunks' loads are in flight together.
constexpr int kBatch = 4;

// Forward walk over one ray starting at row h: S_i for the lane's row of every chunk.  Calls f(row, S) per chunk; returns the number of
// chunks walked (the last one holds the ray's end).
template <class F>
__device__ __forceinline__ int64_t walk_forward(const DistIn& in, int64_t h, int32_t id, int64_t n_live, int lane, F&& f) {
  float carry_w = 0.f, carry_s = 0.f, m_prev_chunk = 0.f;
  for (int64_t c0 = 0;; c0 += kBatch) {
    Row rows[kBatch];
#pragma unroll
    for (int u = 0; u < kBatch; ++u) rows[u] = load_row(in, h + (c0 + u) * 32 + lane, id, n_live);
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {
      const Row& r = rows[u];
      const float w_incl = warp_incl_scan(r.w, lane);
      const float w_excl = carry_w + w_incl - r.w;     // W_{<i}
      float m_prev = __shfl_up_sync(0xffffffffu, r.m, 1);
      if (lane == 0) m_prev = m_prev_chunk;
      const bool has_prev = lane > 0 || c0 + u > 0;
      const float term = (r.ok && has_prev) ? w_excl * (r.m - m_prev) : 0.f;
      const float s = carry_s + warp_incl_scan(term, lane);
      f(r, s);
      if (__ballot_sync(0xffffffffu, r.ok) != 0xffffffffu) return c0 + u + 1;
      carry_w += __shfl_sync(0xffffffffu, w_incl, 31);
      carry_s = __shfl_sync(0xffffffffu, s, 31);
      m_prev_chunk = __shfl_sync(0xffffffffu, r.m, 31);
    }
  }
}

// The rays that start in group g (rows [32 g, 32 g + 32)) and also end in it -- most of them: short rays are common -- in one pass of
// segmented warp scans over the group's rows.  Returns the lane of the group's last head when that ray runs past the group (its id in
// *walk_id): the caller walks it chunk by chunk.  kGrad: write the gradient of the rows handled here; else add their loss terms to acc.
template <bool kGrad>
__device__ __forceinline__ int group_pass(const DistIn& in, int64_t g, int64_t n_live, int lane, float scale, float* __restrict__ g_w,
                                          float& acc, int32_t& walk_id) {
  const int64_t i = g * 32 + lane;
  int32_t id = 0;
  bool head = false, cont = false;
  Row r{0.f, 0.f, 0.f, i, false};
  if (i < n_live) {
    id = in.rid[i];
    head = i == 0 || in.rid[i - 1] != id;
    cont = lane == 31 && i + 1 < n_live && in.rid[i + 1] == id;
    r = load_row(in, i, id, n_live);
  }
  const unsigned heads = __ballot_sync(0xffffffffu, head);
  if (heads == 0) return -1;                            // the group continues a ray owned by an earlier group
  const int last = 31 - __clz(heads);
  cont = __shfl_sync(0xffffffffu, (int)cont, 31) != 0;  // the last ray runs past the group
  walk_id = __shfl_sync(0xffffffffu, id, last);
  const unsigned at_or_below = lane == 31 ? 0xffffffffu : (2u << lane) - 1u;
  const unsigned lo = heads & at_or_below, hi = heads & ~at_or_below;
  const int seg0 = lo ? 31 - __clz(lo) : -1;           // first lane of this lane's ray (-1: a ray from an earlier group)
  const int seg1 = hi ? __ffs(hi) - 2 : 31;            // last lane of this lane's ray
  const bool mine = r.ok && seg0 >= 0 && !(cont && seg0 == last);
  const float w = mine ? r.w : 0.f;
  float w_incl = w, s = 0.f;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, w_incl, o);
    if (lane - o >= seg0) w_incl += t;
  }
  const float m_prev = __shfl_up_sync(0xffffffffu, r.m, 1);
  s = (mine && lane > seg0) ? (w_incl - w) * (r.m - m_prev) : 0.f;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, s, o);
    if (lane - o >= seg0) s += t;
  }
  if (!kGrad) {
    if (mine) acc += 2.f * w * s + (1.f / 3.f) * w * w * r.d;
  } else {
    float w_suf = w, rr = 0.f;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float t = __shfl_down_sync(0xffffffffu, w_suf, o);
      if (lane + o <= seg1) w_suf += t;
    }
    const float m_next = __shfl_down_sync(0xffffffffu, r.m, 1);
    const bool ok_next = __shfl_down_sync(0xffffffffu, (int)mine, 1) != 0;
    rr = (mine && lane < seg1 && ok_next) ? (w_suf - w) * (m_next - r.m) : 0.f;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float t = __shfl_down_sync(0xffffffffu, rr, o);
      if (lane + o <= seg1) rr += t;
    }
    if (mine) g_w[r.p] = scale * (2.f * (s + rr) + (2.f / 3.f) * w * r.d);
  }
  return cont ? last : -1;
}

// accum[0] += sum over the live rows of 2 w_i S_i + 1/3 w_i^2 d_i  (zeroed by the entry point)
__global__ void __launch_bounds__(kThreads) distortion_fwd_kernel(const DistIn in, float* __restrict__ accum, int64_t n,
                                                                  const int64_t* __restrict__ n_dev) {
  const int64_t n_live = live_rows(n, n_dev);
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (kThreads / 32);
  float acc = 0.f;
  for (int64_t g = blockIdx.x * (int64_t)(kThreads / 32) + (threadIdx.x >> 5); g * 32 < n_live; g += warps) {
    int32_t hid = 0;
    const int l = group_pass<false>(in, g, n_live, lane, 0.f, nullptr, acc, hid);
    if (l >= 0)
      walk_forward(in, g * 32 + l, hid, n_live, lane, [&](const Row& r, float s) {
        if (r.ok) acc += 2.f * r.w * s + (1.f / 3.f) * r.w * r.w * r.d;
      });
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  __shared__ float ws[kThreads / 32];
  if (lane == 0) ws[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int k = 0; k < kThreads / 32; ++k) t += ws[k];
    if (t != 0.f) atomicAdd(accum, t);
  }
}

// accum[1] = accum[0] / n_div (0 for an empty batch)
__global__ void distortion_finalize_kernel(const int32_t* __restrict__ rid, float* __restrict__ accum, int64_t n, const int64_t* __restrict__ n_dev) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const int64_t n_live = live_rows(n, n_dev);
  accum[1] = n_live > 0 ? accum[0] / (float)((int64_t)rid[n_live - 1] + 1) : 0.f;
}

// g_w[pos(i)] = g * (2 (S_i + R_i) + 2/3 w_i d_i) / n_div on every live row.  A ray that runs past its group: a forward walk parks S_i in
// g_w, the reverse walk over the same chunks (each row stays on the same lane, so the lane reads back its own store) adds R_i.  Plain
// stores: bitwise reproducible.
__global__ void __launch_bounds__(kThreads) distortion_bwd_kernel(const DistIn in, const float* __restrict__ g_loss, float* __restrict__ g_w,
                                                                  int64_t n, const int64_t* __restrict__ n_dev) {
  const int64_t n_live = live_rows(n, n_dev);
  if (n_live == 0) return;
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (kThreads / 32);
  const float scale = (g_loss ? __ldg(g_loss) : 1.f) / (float)((int64_t)in.rid[n_live - 1] + 1);
  for (int64_t g = blockIdx.x * (int64_t)(kThreads / 32) + (threadIdx.x >> 5); g * 32 < n_live; g += warps) {
    int32_t hid = 0;
    float unused = 0.f;
    const int l = group_pass<true>(in, g, n_live, lane, scale, g_w, unused, hid);
    if (l < 0) continue;
    const int64_t h = g * 32 + l;
    const int64_t chunks = walk_forward(in, h, hid, n_live, lane, [&](const Row& r, float s) {
      if (r.ok) g_w[r.p] = s;
    });
    float carry_w = 0.f, carry_r = 0.f, m_next_chunk = 0.f;
    bool ok_next_chunk = false;
    for (int64_t c0 = chunks - 1; c0 >= 0; c0 -= kBatch) {
      Row rows[kBatch];
#pragma unroll
      for (int u = 0; u < kBatch; ++u) rows[u] = load_row(in, c0 - u >= 0 ? h + (c0 - u) * 32 + lane : n_live, hid, n_live);
#pragma unroll
      for (int u = 0; u < kBatch; ++u) {
        if (c0 - u < 0) break;
        const Row& r = rows[u];
        const float w_suf = warp_incl_suffix_scan(r.w, lane);
        const float w_after = carry_w + w_suf - r.w;    // W_{>i}
        float m_next = __shfl_down_sync(0xffffffffu, r.m, 1);
        bool has_next = __shfl_down_sync(0xffffffffu, (int)r.ok, 1) != 0;
        if (lane == 31) {
          m_next = m_next_chunk;
          has_next = ok_next_chunk;
        }
        const float term = (r.ok && has_next) ? w_after * (m_next - r.m) : 0.f;
        const float rr = carry_r + warp_incl_suffix_scan(term, lane);
        if (r.ok) g_w[r.p] = scale * (2.f * (g_w[r.p] + rr) + (2.f / 3.f) * r.w * r.d);
        carry_w += __shfl_sync(0xffffffffu, w_suf, 0);
        carry_r = __shfl_sync(0xffffffffu, rr, 0);
        m_next_chunk = __shfl_sync(0xffffffffu, r.m, 0);
        ok_next_chunk = __shfl_sync(0xffffffffu, (int)r.ok, 0) != 0;
      }
    }
  }
}

// persistent: 4 CTAs of 256 threads per SM are resident at <= 64 registers per thread
int grid_for(int64_t n) { return (int)max((int64_t)1, min((int64_t)nsr_sm_count() * 4, (n + kThreads - 1) / kThreads)); }

}  // namespace

extern "C" int nsr_distortion_fwd(const float* w, const int64_t* w_pos, const float* a, const float* b, int32_t t_mode, const int32_t* ray_ids,
                                  float* accum2, int64_t n, const int64_t* n_dev, void* stream) {
  NSR_REQUIRE(accum2 != nullptr, "nsr_distortion_fwd: accum is NULL");
  NSR_REQUIRE(n == 0 || (w != nullptr && a != nullptr && b != nullptr && ray_ids != nullptr), "nsr_distortion_fwd: an input is NULL");
  NSR_REQUIRE(t_mode == 0 || t_mode == 1, "nsr_distortion_fwd: t_mode must be 0 (midpoint, interval) or 1 (t_start, t_end)");
  cudaStream_t st = (cudaStream_t)stream;
  cudaMemsetAsync(accum2, 0, 2 * sizeof(float), st);
  if (n > 0) {
    const DistIn in{w, w_pos, a, b, ray_ids, t_mode};
    distortion_fwd_kernel<<<grid_for(n), kThreads, 0, st>>>(in, accum2, n, n_dev);
    distortion_finalize_kernel<<<1, 32, 0, st>>>(ray_ids, accum2, n, n_dev);
  }
  NSR_CHECK_LAUNCH("nsr_distortion_fwd");
  return 0;
}

extern "C" int nsr_distortion_bwd(const float* w, const int64_t* w_pos, const float* a, const float* b, int32_t t_mode, const int32_t* ray_ids,
                                  const float* g_loss, float* g_w, int64_t n, const int64_t* n_dev, void* stream) {
  NSR_REQUIRE(n == 0 || (w != nullptr && a != nullptr && b != nullptr && ray_ids != nullptr && g_w != nullptr),
              "nsr_distortion_bwd: an input / g_w is NULL");
  NSR_REQUIRE(t_mode == 0 || t_mode == 1, "nsr_distortion_bwd: t_mode must be 0 (midpoint, interval) or 1 (t_start, t_end)");
  if (n == 0) return 0;
  const DistIn in{w, w_pos, a, b, ray_ids, t_mode};
  distortion_bwd_kernel<<<grid_for(n), kThreads, 0, (cudaStream_t)stream>>>(in, g_loss, g_w, n, n_dev);
  NSR_CHECK_LAUNCH("nsr_distortion_bwd");
  return 0;
}
