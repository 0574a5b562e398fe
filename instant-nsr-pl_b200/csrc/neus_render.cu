// NeuS eval render (NeuSModel.forward_ in eval mode, models/neus.py:205-243 with randomized = False) as ONE kernel per pass of rays:
// a warp owns a ray (atomic ticket over the marcher's longest-first queue), walks its marched samples 32 at a time and runs, per group,
//   sample points -> SDF field + analytic normal (neus_field.cuh) -> alpha + unit normal (neus_shade.cuh) -> colour network
//   [feature | SH4(dir) | normal] (radiance.cuh) -> transmittance scan with the carry in a register and per-lane sums (warp_scan.cuh)
// and writes only per-ray results.  Nothing per sample reaches global memory.
// The finite-difference form (FD, Neuralangelo's geometry) replaces only the field stage: each lane runs its own sample's centre
// evaluation with every output and then the six stencil points for the SDF alone (neus_field_fd.cuh, fp32 on the CUDA cores, the
// operation order of neus_fd_fwd_kernel), so sdf, feature and normal are the per-sample path's values; the normal is the world-space
// central difference 0.5 (s+ - s-) / eps.
// The groups are 32 CONSECUTIVE samples of the ray counted from its first, the groups neus_composite_fwd_kernel scans, so the
// transmittance products and sums run in the same order as the per-sample path; samples and t come from march.cuh, so they are the
// marcher's bit for bit.  Every marched sample is composited (the reference's NeuS has no transmittance cut-off).
#include "march.cuh"
#include "neus_field.cuh"
#include "neus_field_fd.cuh"
#include "neus_shade.cuh"
#include "radiance.cuh"
#include "warp_scan.cuh"

namespace {

constexpr int kThreads = kNeusTcWarps * 32;   // 128: the field's per-warp encoding tiles are sized for this CTA
constexpr int kMaxWords = 64;                 // mask words a lane pair holds: 2048 lattice points per ray
constexpr int kFeat = 13;                     // colour input [feature 13 | SH4 16 | normal 3] (every NeuS config of the reference)

struct RenderWarpSmem {
  __half X[32][LD32];      // colour network input rows
  float out[32][NOUTP];    // field output rows (sdf, feature)
  float rgb[32][4];
  float sh[16];            // SH4 of the ray's view direction: the same for every sample of the ray
};
// shared memory: the field's weights (NeusTcSmem, or fd::FdW for the finite-difference form), the colour network, its bias, the warps' rows
template <bool FD>
constexpr size_t kFieldSmem = FD ? sizeof(fd::FdW) : sizeof(NeusTcSmem);
template <bool FD>
constexpr size_t kRenderSmem = kFieldSmem<FD> + W_TOTAL * sizeof(__half) + N_BIAS * sizeof(float) + kNeusTcWarps * sizeof(RenderWarpSmem);
static_assert(sizeof(NeusTcSmem) % 16 == 0 && sizeof(fd::FdW) % 16 == 0 && (W_TOTAL * sizeof(__half)) % 16 == 0 &&
                  (N_BIAS * sizeof(float)) % 16 == 0, "16-byte aligned");
// CTAs per SM: the analytic form's 168 registers allow two; the finite-difference form's fit in 128 (four CTAs, 16 warps per SM)
template <bool FD>
constexpr int kCtasPerSm = FD ? 4 : 2;

struct RenderArgs {
  const float* rays;            // [n, 6]
  const uint32_t* masks;        // [n, words]
  const float* t_min;           // [n]
  const int32_t* counts;        // [n]
  const int32_t* bin_counts;    // [8]
  const int32_t* order_bins;    // [8 * n]
  const __half2* table;
  const float *W1, *b1, *W2, *b2;
  const float* n_active;
  const __half* rgb_params;
  const float* rgb_bias;
  const float* inv_s;
  const float* cos_anneal;
  float *opacity, *depth, *comp_rgb, *comp_normal;
  uint32_t* ticket;
  float step, radius;
  int32_t words, n_out, act_mode;
  int64_t n_rays;
  const float* fd_state;        // finite-difference form: {eps, eps^2, n_active} (n_active above is unused)
};

// the next (up to) 32 set bits of the ray's mask: lane j gets lattice index k of the j-th, or -1.  (cur_w, cur_m) is the warp-uniform
// cursor; lane w holds mask words w (mw0) and w + 32 (mw1).
__device__ __forceinline__ int next_group(int lane, int words, uint32_t mw0, uint32_t mw1, int& cur_w, uint32_t& cur_m) {
  int k = -1, filled = 0;
  while (filled < 32) {
    if (cur_m == 0u) {
      if (++cur_w >= words) break;
      cur_m = cur_w < 32 ? __shfl_sync(0xffffffffu, mw0, cur_w) : __shfl_sync(0xffffffffu, mw1, cur_w - 32);
      continue;
    }
    const int cnt = __popc(cur_m), take = min(cnt, 32 - filled);
    if (lane >= filled && lane < filled + take) k = cur_w * 32 + (int)__fns(cur_m, 0, lane - filled + 1);
    if (take == cnt) {
      cur_m = 0u;
    } else {
      cur_m &= ~((2u << __fns(cur_m, 0, take)) - 1u);   // drop the bits taken
    }
    filled += take;
  }
  return k;
}

// The hash levels >= n_active (device float: the ProgressiveBandHashGrid schedule, 16 for a plain HashGrid) contribute 0, as in
// neus_field_fwd_tc_kernel<true>; with n_active = 16 that is the unmasked field's arithmetic.  One masked form only: the unmasked
// instantiation let the compiler hoist all sixteen levels' corner loads and spill.
// FD: the finite-difference field; eps and n_active come from fd_state, as in neus_fd_fwd_kernel.
template <bool VANILLA, bool FD>
__global__ void __launch_bounds__(kThreads, kCtasPerSm<FD>) neus_render_rays_kernel(const __grid_constant__ nsr_grid_t g,
                                                                                    const __grid_constant__ RenderArgs a) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  NeusTcSmem& S = *reinterpret_cast<NeusTcSmem*>(smem_raw);
  fd::FdW& Wf = *reinterpret_cast<fd::FdW*>(smem_raw);
  __half* RW = reinterpret_cast<__half*>(smem_raw + kFieldSmem<FD>);
  float* rbias = reinterpret_cast<float*>(RW + W_TOTAL);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  RenderWarpSmem& Wp = reinterpret_cast<RenderWarpSmem*>(rbias + N_BIAS)[warp];
  __shared__ int bins[NSR_ORDER_BINS];
  if constexpr (FD)
    fd::stage_weights(Wf, a.W1, a.b1, a.W2, a.b2, a.n_out);
  else
    stage_neus_tc_weights(S, a.W1, a.b1, a.W2, a.b2, a.n_out);
  stage_weights(RW, a.rgb_params);
  if (VANILLA) stage_bias(rbias, a.rgb_bias);
  if (tid < NSR_ORDER_BINS) bins[tid] = __ldg(a.bin_counts + tid);
  __syncthreads();
  const int n_active = FD ? (int)__ldg(a.fd_state + 2) : load_n_active(a.n_active);
  const float eps = FD ? __ldg(a.fd_state) : 0.f;
  const float inv_s = __ldg(a.inv_s), cos_anneal = __ldg(a.cos_anneal);
  const float inv2r = 1.f / (2.f * a.radius);

  for (;;) {
    int64_t ray = 0;
    if (lane == 0) ray = atomicAdd(a.ticket, 1u);
    ray = __shfl_sync(0xffffffffu, ray, 0);
    if (ray >= a.n_rays) break;
    {  // ticket t -> t-th ray of the binned longest-first queue (nsr_march_rays_alloc)
      int t = (int)ray, b = 0;
#pragma unroll
      for (int q = 0; q < NSR_ORDER_BINS - 1; ++q) {
        const bool next = b == q && t >= bins[q];
        t -= next ? bins[q] : 0;
        b += next ? 1 : 0;
      }
      ray = __ldg(a.order_bins + (int64_t)b * a.n_rays + t);
    }
    const int total = __ldg(a.counts + ray);
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};  // opacity, depth, rgb, normal
    if (total > 0) {
      const uint32_t mw0 = lane < a.words ? __ldg(a.masks + ray * a.words + lane) : 0u;
      const uint32_t mw1 = lane + 32 < a.words ? __ldg(a.masks + ray * a.words + lane + 32) : 0u;
      const float* rr = a.rays + ray * 6;
      const float ox = __ldg(rr + 0), oy = __ldg(rr + 1), oz = __ldg(rr + 2);
      const float dx = __ldg(rr + 3), dy = __ldg(rr + 4), dz = __ldg(rr + 5);
      const float tmin = __ldg(a.t_min + ray);
      if (lane == 0) {
        float sh[16];
        nsr_sh4(dx, dy, dz, sh);
#pragma unroll
        for (int c = 0; c < 16; ++c) Wp.sh[c] = sh[c];
      }
      float carry = 1.f;
      int cur_w = 0;
      uint32_t cur_m = __shfl_sync(0xffffffffu, mw0, 0);
      for (int b0 = 0; b0 < total; b0 += 32) {
        int k = next_group(lane, a.words, mw0, mw1, cur_w, cur_m);
        const bool ok = k >= 0;
        if (!ok) k = 0;
        const float t0 = nsr_lattice_t((float)k, a.step, tmin), t1 = nsr_lattice_t((float)k + 1.f, a.step, tmin);
        const float mid = nsr_sample_mid(t0, t1);
        float gx = 0.f, gy = 0.f, gz = 0.f;
        if constexpr (FD) {
          float px = 0.f, py = 0.f, pz = 0.f;   // world-space sample point (dead lanes: the box centre)
          if (ok) {
            px = nsr_sample_coord(ox, dx, mid);
            py = nsr_sample_coord(oy, dy, mid);
            pz = nsr_sample_coord(oz, dz, mid);
          }
          {  // centre: sdf and feature
            float x, y, z, e[fd::NINP], out[fd::NOUTP];
            fd::stencil_query(px, py, pz, 0, eps, a.radius, x, y, z);
            fd::encode(g, a.table, x, y, z, n_active, e);
            fd::mlp_eval<fd::NOUTP>(Wf, e, out);
#pragma unroll
            for (int c = 0; c < fd::NOUTP; ++c) Wp.out[lane][c] = out[c];
          }
          float sp = 0.f;   // SDF at the + point of the current axis
#pragma unroll 1
          for (int q = 1; q <= 6; ++q) {   // stencil points +x, -x, +y, -y, +z, -z: SDF only
            float x, y, z, e[fd::NINP], sq[1];
            fd::stencil_query(px, py, pz, q, eps, a.radius, x, y, z);
            fd::encode(g, a.table, x, y, z, n_active, e);
            fd::mlp_eval<1>(Wf, e, sq);
            if (q & 1) {
              sp = sq[0];
            } else {
              const float ga = __fdiv_rn(0.5f * (sp - sq[0]), eps);
              gx = q == 2 ? ga : gx;
              gy = q == 4 ? ga : gy;
              gz = q == 6 ? ga : gz;
            }
          }
        } else {
          float x = 0.5f, y = 0.5f, z = 0.5f;
          if (ok) {   // neus_field_fwd_tc_kernel's unit-cube position of the sample point
            x = (nsr_sample_coord(ox, dx, mid) + a.radius) * inv2r;
            y = (nsr_sample_coord(oy, dy, mid) + a.radius) * inv2r;
            z = (nsr_sample_coord(oz, dz, mid) + a.radius) * inv2r;
          }
          neus_field_rows32<true>(
              S, warp, lane, g, a.table, x, y, z, ok, n_active,
              [&](int r0, int gq, int dr, int col, float v) { Wp.out[r0 + gq + dr][col] = v; },
              [&](float gx_, float gy_, float gz_) {
                gx = gx_ * inv2r;
                gy = gy_ * inv2r;
                gz = gz_ * inv2r;
              });
        }
        __syncwarp();
        const AlphaTerms at = alpha_terms(Wp.out[lane][0], gx, gy, gz, dx, dy, dz, t1 - t0, inv_s, cos_anneal);
        const float alpha = ok ? fminf(fmaxf(at.q, 0.f), 1.f) : 0.f;
        {  // colour network input row [feature | SH4 | normal] (dead lanes: all zero)
          __half* xr = Wp.X[lane];
#pragma unroll
          for (int c = 0; c < 32; ++c) {
            float v = c < kFeat ? Wp.out[lane][c] : c < kFeat + 16 ? Wp.sh[c - kFeat] : c == kFeat + 16 ? at.nx : c == kFeat + 17 ? at.ny : at.nz;
            xr[c] = __float2half_rn(ok ? v : 0.f);
          }
        }
        __syncwarp();
#pragma unroll 1
        for (int m = 0; m < 2; ++m) {
          float acc16[1][2][4];
          radiance_rows16<VANILLA>(acc16, &Wp.X[0][0], m * 16, RW, rbias);
          const int gq = lane >> 2, cq = lane & 3;
          if (cq < 2) {
#pragma unroll
            for (int hh = 0; hh < 2; ++hh)
#pragma unroll
              for (int e = 0; e < 2; ++e) Wp.rgb[m * 16 + gq + hh * 8][cq * 2 + e] = out_value<VANILLA>(acc16[0][0][hh * 2 + e], a.act_mode);
          }
        }
        __syncwarp();
        // neus_composite_fwd_kernel's arithmetic
        const float incl = warp_incl_prod(1.f - alpha, lane);
        float excl = __shfl_up_sync(0xffffffffu, incl, 1);
        if (lane == 0) excl = 1.f;
        const float T = carry * excl;
        const float w = T * alpha;
        if (ok) {
          acc[0] += w;
          acc[1] += w * ((t0 + t1) * 0.5f);
#pragma unroll
          for (int c = 0; c < 3; ++c) acc[2 + c] += w * Wp.rgb[lane][c];
          acc[5] += w * at.nx;
          acc[6] += w * at.ny;
          acc[7] += w * at.nz;
        }
        carry *= __shfl_sync(0xffffffffu, incl, 31);
        __syncwarp();   // Wp is rewritten by the next group
      }
    }
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[c] = warp_sum(acc[c]);
    if (lane == 0) {
      a.opacity[ray] = acc[0];
      a.depth[ray] = acc[1];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        a.comp_rgb[ray * 3 + c] = acc[2 + c];
        a.comp_normal[ray * 3 + c] = acc[5 + c];
      }
    }
  }
}

template <bool VANILLA, bool FD>
int launch(const nsr_grid_t* g, const RenderArgs& a, cudaStream_t st, const char* name) {
  static thread_local bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(neus_render_rays_kernel<VANILLA, FD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kRenderSmem<FD>);
    if (e != cudaSuccess) {
      nsr_set_error("%s: cannot reserve %zu B shared memory: %s", name, kRenderSmem<FD>, cudaGetErrorString(e));
      return 2;
    }
    attr_set = true;
  }
  const int grid = (int)min((int64_t)nsr_sm_count() * kCtasPerSm<FD>, (a.n_rays + kNeusTcWarps - 1) / kNeusTcWarps);
  neus_render_rays_kernel<VANILLA, FD><<<grid, kThreads, kRenderSmem<FD>, st>>>(*g, a);
  NSR_CHECK_LAUNCH(name);
  return 0;
}

// both entry points: field_state is n_active (analytic field) or fd_state (finite-difference field)
template <bool FD>
int render_rays(const char* name, const nsr_grid_t* g, const float* rays, const uint32_t* masks, int32_t words, const float* t_min,
                const int32_t* counts, const int32_t* bin_counts, const int32_t* order_bins, float step, const void* table_h, const float* W1,
                const float* b1, const float* W2, const float* b2, float radius, int32_t n_out, const float* field_state,
                const nsr_radiance_t* rp, int32_t vanilla, const void* rgb_params_h, const float* rgb_bias, const float* inv_s,
                const float* cos_anneal, float* opacity, float* depth, float* comp_rgb, float* comp_normal, uint32_t* ticket, int64_t n_rays,
                void* stream) {
  NSR_REQUIRE(g != nullptr && g->n_levels == 16 && g->n_features == 2, "%s: needs a 16-level F=2 hash grid", name);
  NSR_REQUIRE(n_out >= 1 && n_out <= 16, "%s: n_out must be in [1,16]", name);
  NSR_REQUIRE(rp != nullptr && n_out == kFeat && rp->n_feat == kFeat && rp->n_extra == 3,
              "%s: the colour input must be [feature (13) | SH4 (16) | normal (3)]", name);
  NSR_REQUIRE(rp->act_mode >= 0 && rp->act_mode <= 2, "%s: act_mode must be 0, 1 or 2", name);
  NSR_REQUIRE(words >= 1 && words <= kMaxWords, "%s: words must be in [1, %d]", name, kMaxWords);
  NSR_REQUIRE(step > 0.f, "%s: step must be > 0", name);
  NSR_REQUIRE(rays && masks && t_min && counts && bin_counts && order_bins && table_h && W1 && b1 && W2 && b2 && rgb_params_h && inv_s &&
                  cos_anneal && opacity && depth && comp_rgb && comp_normal && ticket,
              "%s: NULL argument", name);
  NSR_REQUIRE(field_state != nullptr, FD ? "%s: fd_state (device {eps, eps^2, n_active}) is NULL" : "%s: NULL argument", name);
  NSR_REQUIRE(!vanilla || rgb_bias != nullptr, "%s: the VanillaMLP colour network needs its bias", name);
  if (n_rays == 0) return 0;
  RenderArgs a;
  a.rays = rays, a.masks = masks, a.t_min = t_min, a.counts = counts, a.bin_counts = bin_counts, a.order_bins = order_bins;
  a.table = (const __half2*)table_h, a.W1 = W1, a.b1 = b1, a.W2 = W2, a.b2 = b2;
  a.n_active = FD ? nullptr : field_state, a.fd_state = FD ? field_state : nullptr;
  a.rgb_params = (const __half*)rgb_params_h, a.rgb_bias = rgb_bias, a.inv_s = inv_s, a.cos_anneal = cos_anneal;
  a.opacity = opacity, a.depth = depth, a.comp_rgb = comp_rgb, a.comp_normal = comp_normal, a.ticket = ticket;
  a.step = step, a.radius = radius, a.words = words, a.n_out = n_out, a.act_mode = rp->act_mode, a.n_rays = n_rays;
  const cudaStream_t st = (cudaStream_t)stream;
  return vanilla ? launch<true, FD>(g, a, st, name) : launch<false, FD>(g, a, st, name);
}

}  // namespace

extern "C" int nsr_neus_render_rays(const nsr_grid_t* g, const float* rays, const uint32_t* masks, int32_t words, const float* t_min,
                                    const int32_t* counts, const int32_t* bin_counts, const int32_t* order_bins, float step, const void* table_h,
                                    const float* W1, const float* b1, const float* W2, const float* b2, float radius, int32_t n_out,
                                    const float* n_active, const nsr_radiance_t* rp, int32_t vanilla, const void* rgb_params_h,
                                    const float* rgb_bias, const float* inv_s, const float* cos_anneal, float* opacity, float* depth,
                                    float* comp_rgb, float* comp_normal, uint32_t* ticket, int64_t n_rays, void* stream) {
  return render_rays<false>("nsr_neus_render_rays", g, rays, masks, words, t_min, counts, bin_counts, order_bins, step, table_h, W1, b1, W2, b2,
                            radius, n_out, n_active, rp, vanilla, rgb_params_h, rgb_bias, inv_s, cos_anneal, opacity, depth, comp_rgb,
                            comp_normal, ticket, n_rays, stream);
}

extern "C" int nsr_neus_render_rays_fd(const nsr_grid_t* g, const float* rays, const uint32_t* masks, int32_t words, const float* t_min,
                                       const int32_t* counts, const int32_t* bin_counts, const int32_t* order_bins, float step,
                                       const void* table_h, const float* W1, const float* b1, const float* W2, const float* b2, float radius,
                                       int32_t n_out, const float* fd_state, const nsr_radiance_t* rp, int32_t vanilla,
                                       const void* rgb_params_h, const float* rgb_bias, const float* inv_s, const float* cos_anneal,
                                       float* opacity, float* depth, float* comp_rgb, float* comp_normal, uint32_t* ticket, int64_t n_rays,
                                       void* stream) {
  return render_rays<true>("nsr_neus_render_rays_fd", g, rays, masks, words, t_min, counts, bin_counts, order_bins, step, table_h, W1, b1, W2,
                           b2, radius, n_out, fd_state, rp, vanilla, rgb_params_h, rgb_bias, inv_s, cos_anneal, opacity, depth, comp_rgb,
                           comp_normal, ticket, n_rays, stream);
}
