// Persistent per-ray NeRF forward: ONE kernel from occupancy masks to per-ray colour (models/nerf.py:82-109).
//
// A warp owns a ray (rays are handed out through an atomic ticket => rays with 600 samples and rays with none share
// the machine evenly).  It expands the ray's lattice-occupancy mask (written by nsr_march_rays_mask) into sample
// indices in shared memory and then walks the samples 32 at a time:
//     position -> 16-level hash gather -> density MLP -> alpha -> in-warp transmittance scan (carry in a register)
//     -> visibility test T >= early_stop_eps -> SH4 + colour MLP -> weights -> per-ray sums in registers
// and stops at the first chunk after which T < early_stop_eps (early ray termination): samples behind an opaque
// surface are never gathered.  This replaces nerfacc's sigma_fn pre-pass over ALL marched samples + render_visibility +
// three boolean-mask compactions + a second full field evaluation, and our own earlier pre-pass / visibility / compact /
// expand kernels.  Per-ray outputs are plain stores (no atomics: bit-reproducible); kept samples of ray r land at
// offsets_m[r] + j (j < kept[r]) in the per-sample buffers ("loose" layout: a kept prefix per ray).
// The kept set is identical to the two-pass path: same density code, same 32-sample chunking of the scan.
#include "nerf_fused.cuh"

namespace {

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr int kMaxWords = 64;  // mask words per ray held in two registers per lane (<= 2048 lattice points)
// per-warp scratch (halves): A tile [32][40] + SH tile [32][24] + sigma (32 f32) + rgb (32 x 4 f32)
constexpr int kWarpHalves = 32 * NF_LD32 + 32 * 24 + 64 + 256;
constexpr size_t kSmemBytes = (size_t)(NF_W_TOTAL + kWarps * kWarpHalves) * sizeof(__half);

struct RaysFwdArgs {
  const float* rays;           // [n_rays,6]
  const uint32_t* masks;       // [n_rays, words]
  const float* t_min;          // [n_rays]
  const int64_t* offsets_m;    // [n_rays+1] marched offsets (loose layout base of every ray)
  const int32_t* order;        // [n_rays] processing order (longest rays first) or NULL; with bin_counts: [8][n_rays] rays grouped by chunk count
  const int32_t* bin_counts;   // int32[8] (nsr_march_rays_alloc) or NULL
  const int32_t* counts;       // [n_rays] marched samples per ray, or NULL: offsets_m[ray + 1] - offsets_m[ray]
  const __half* dparams;
  const __half* cparams;
  __half* enc_save;            // [cap,32] or NULL
  float* sigmas;               // [cap]
  float* rgbs;                 // [cap,3]
  float* weights;              // [cap]
  float* trans;                // [cap]
  int32_t* kidx_out;           // [cap] lattice index of every kept sample (t = fma(k, step, t_min))
  float* acc_rgb;              // [n_rays,3]
  float* opacity;              // [n_rays]
  float* depth;                // [n_rays]
  int32_t* kept;               // [n_rays]
  int32_t* kept_blocks;        // [ceil(n_rays / 256)] sums of kept over 256-ray blocks (zero on entry) or NULL: lets nsr_pack_kept_scan skip most of its prefix sum
  uint32_t* ticket;            // ray queue head (zero on entry)
  float step, early_stop_eps;
  int words;
  int64_t n_rays;
};

__device__ __forceinline__ float warp_incl_prod(float v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v *= t;
  }
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// The register allocation is sized for kMinBlocks resident CTAs per SM: 2 (128 registers).  (3 CTAs -- 80 registers, 0.5 KB of spills per
// thread, 24 warps per SM -- was markedly slower.)
constexpr int kMinBlocks = 2;
// levels whose 8 corner loads are issued together (8 levels measured no faster and spilled 120 B)
constexpr int kGatherBatch = 4;
__global__ void __launch_bounds__(kThreads, kMinBlocks) nerf_rays_fwd_kernel(const __grid_constant__ nsr_nerf_t P, const RaysFwdArgs a) {
  extern __shared__ __align__(16) __half smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, c = lane & 3;
  __half* At = smem + NF_W_TOTAL + warp * kWarpHalves;
  __half* St = At + 32 * NF_LD32;
  float* s_sig = reinterpret_cast<float*>(St + 32 * 24);
  float* s_rgb = s_sig + 32;
  const __half2* table = reinterpret_cast<const __half2*>(a.dparams + NF_DENSITY_PARAMS);
  nf_stage_weights(smem, a.dparams, a.cparams, true);
  __shared__ int bins[NSR_ORDER_BINS];   // binned queue: ticket t belongs to the first group whose running total exceeds it
  if (threadIdx.x < NSR_ORDER_BINS) bins[threadIdx.x] = a.bin_counts != nullptr ? __ldg(a.bin_counts + threadIdx.x) : 0;
  __syncthreads();

  for (;;) {
    int64_t ray = 0;
    if (lane == 0) ray = atomicAdd(a.ticket, 1u);
    ray = __shfl_sync(0xffffffffu, ray, 0);
    if (ray >= a.n_rays) break;
    if (a.bin_counts != nullptr) {
      int t = (int)ray, b = 0;
#pragma unroll
      for (int q = 0; q < NSR_ORDER_BINS - 1; ++q) {
        const bool next = b == q && t >= bins[q];
        t -= next ? bins[q] : 0;
        b += next ? 1 : 0;
      }
      ray = __ldg(a.order + (int64_t)b * a.n_rays + t);
    } else if (a.order != nullptr) {
      ray = __ldg(a.order + ray);
    }
    // ---- the ray's occupancy mask: lane w holds words w and w+32
    const uint32_t mw0 = lane < a.words ? __ldg(a.masks + ray * a.words + lane) : 0u;
    const uint32_t mw1 = lane + 32 < a.words ? __ldg(a.masks + ray * a.words + lane + 32) : 0u;
    const int64_t base = a.offsets_m[ray];
    const int total = a.counts != nullptr ? __ldg(a.counts + ray) : (int)(a.offsets_m[ray + 1] - base);
    float o_acc = 0.f, d_acc = 0.f, r_acc = 0.f, g_acc = 0.f, b_acc = 0.f;
    int kept = 0;
    if (total > 0) {
      const float* rr = a.rays + ray * 6;
      const float ox = __ldg(rr + 0), oy = __ldg(rr + 1), oz = __ldg(rr + 2);
      const float dx = __ldg(rr + 3), dy = __ldg(rr + 4), dz = __ldg(rr + 5);
      const float tmin = __ldg(a.t_min + ray);
      const float inv = 1.f / (2.f * P.radius);
      float carry = 1.f;
      // SH of the view direction is the same for every sample of the ray: build this lane's SH row once
      uint4 sh0, sh1;
      {
        float s[16];
        nsr_sh4(dx, dy, dz, s);
        sh0 = make_uint4(nsr_pack_h2(s[0], s[1]), nsr_pack_h2(s[2], s[3]), nsr_pack_h2(s[4], s[5]), nsr_pack_h2(s[6], s[7]));
        sh1 = make_uint4(nsr_pack_h2(s[8], s[9]), nsr_pack_h2(s[10], s[11]), nsr_pack_h2(s[12], s[13]), nsr_pack_h2(s[14], s[15]));
      }
      uint4* sp = reinterpret_cast<uint4*>(St + lane * 24);
      sp[0] = sh0;
      sp[1] = sh1;
      int cur_w = 0;
      uint32_t cur_m = __shfl_sync(0xffffffffu, mw0, 0);
      for (int b0 = 0; b0 < total; b0 += 32) {
        const int s_idx = b0 + lane;
        // next 32 set bits of the mask (warp-uniform cursor over the words; lane j takes the j-th of them)
        int k = -1, filled = 0;
        while (filled < 32) {
          if (cur_m == 0u) {
            if (++cur_w >= a.words) break;
            cur_m = cur_w < 32 ? __shfl_sync(0xffffffffu, mw0, cur_w) : __shfl_sync(0xffffffffu, mw1, cur_w - 32);
            continue;
          }
          const int cnt = __popc(cur_m), take = min(cnt, 32 - filled);
          if (lane >= filled && lane < filled + take) k = cur_w * 32 + (int)__fns(cur_m, 0, lane - filled + 1);
          if (take == cnt) {
            cur_m = 0u;
          } else {
            const uint32_t p = __fns(cur_m, 0, take);  // position of the last bit taken
            cur_m &= ~((2u << p) - 1u);
          }
          filled += take;
        }
        const bool valid = k >= 0;
        if (!valid) k = 0;
        // identical expression to nsr_march_rays_expand / march_lattice_kernel: t0 = fma(k, step, t_min)
        const float t0 = __fmaf_rn((float)k, a.step, tmin), t1 = __fmaf_rn((float)k + 1.f, a.step, tmin);
        const float mid = (t0 + t1) * 0.5f;
        uint32_t f[16];
        if (valid) {
          const float x = (fmaf(dx, mid, ox) + P.radius) * inv, y = (fmaf(dy, mid, oy) + P.radius) * inv,
                      z = (fmaf(dz, mid, oz) + P.radius) * inv;
          nf_gather_batched<16, kGatherBatch>(P.grid, table, x, y, z, f);   // 8 kGatherBatch loads per lane in flight
        } else {
#pragma unroll
          for (int l = 0; l < 16; ++l) f[l] = 0u;
        }
        nf_store_row32(At, lane, f);
        if (a.enc_save != nullptr && valid) {  // rows past the kept prefix are written too but never read
          uint4* e = reinterpret_cast<uint4*>(a.enc_save + (base + s_idx) * 32);
          e[0] = make_uint4(f[0], f[1], f[2], f[3]);
          e[1] = make_uint4(f[4], f[5], f[6], f[7]);
          e[2] = make_uint4(f[8], f[9], f[10], f[11]);
          e[3] = make_uint4(f[12], f[13], f[14], f[15]);
        }
        __syncwarp();
        // ---- density network
        uint32_t a_o[2][1][4];
        {
          uint32_t a_in[2][2][4];
          nsr_load_afrag<2, 2>(a_in, At, NF_LD32, 0);
          float acc[2][8][4];
          nsr_zero_acc(acc);
          nsr_gemm_w<2, 2, 8>(acc, a_in, smem + NF_OFF_DW1, NF_LD32);
          uint32_t a_h[2][4][4];
          nsr_acc_to_afrag<2, 8>(acc, a_h, NSR_ACT_RELU);
          float acco[2][2][4];
          nsr_zero_acc(acco);
          nsr_gemm_w<2, 4, 2>(acco, a_h, smem + NF_OFF_DW2, NSR_LD64);
          nsr_acc_to_afrag<2, 2>(acco, a_o, NSR_ACT_NONE);
        }
        if (c == 0) {
#pragma unroll
          for (int m = 0; m < 2; ++m) {
            s_sig[m * 16 + g] = nf_half_lo(a_o[m][0][0]);
            s_sig[m * 16 + g + 8] = nf_half_lo(a_o[m][0][1]);
          }
        }
        // ---- colour network
        {
          uint32_t a_c[2][2][4], a_sh[2][1][4];
          nsr_load_afrag<2, 1>(a_sh, St, 24, 0);
#pragma unroll
          for (int m = 0; m < 2; ++m)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              a_c[m][0][j] = a_o[m][0][j];
              a_c[m][1][j] = a_sh[m][0][j];
            }
          float acc[2][8][4];
          nsr_zero_acc(acc);
          nsr_gemm_w<2, 2, 8>(acc, a_c, smem + NF_OFF_CW1, NF_LD32);
          uint32_t a_h[2][4][4];
          nsr_acc_to_afrag<2, 8>(acc, a_h, NSR_ACT_RELU);
          nsr_zero_acc(acc);
          nsr_gemm_w<2, 4, 8>(acc, a_h, smem + NF_OFF_CW2, NSR_LD64);
          nsr_acc_to_afrag<2, 8>(acc, a_h, NSR_ACT_RELU);
          float acco[2][2][4];
          nsr_zero_acc(acco);
          nsr_gemm_w<2, 4, 2>(acco, a_h, smem + NF_OFF_CW3, NSR_LD64);
          uint32_t a_r[2][1][4];
          nsr_acc_to_afrag<2, 2>(acco, a_r, NSR_ACT_NONE);
          if (c < 2) {
#pragma unroll
            for (int m = 0; m < 2; ++m) {
              float* r0 = s_rgb + (m * 16 + g) * 4 + c * 2;
              float* r1 = s_rgb + (m * 16 + g + 8) * 4 + c * 2;
              r0[0] = nf_half_lo(a_r[m][0][0]);
              r0[1] = nf_half_hi(a_r[m][0][0]);
              r1[0] = nf_half_lo(a_r[m][0][1]);
              r1[1] = nf_half_hi(a_r[m][0][1]);
            }
          }
        }
        __syncwarp();
        // ---- compositing (thread per sample): alpha, exclusive transmittance, visibility, weight
        const float sigma = expf(s_sig[lane] + P.density_bias);
        const float alpha = valid ? 1.f - expf(-sigma * (t1 - t0)) : 0.f;
        const float incl = warp_incl_prod(1.f - alpha, lane);
        float excl = __shfl_up_sync(0xffffffffu, incl, 1);
        if (lane == 0) excl = 1.f;
        const float T = carry * excl;
        const bool keep = valid && (T >= a.early_stop_eps);
        if (keep) {
          const float w = T * alpha;
          const float cr = 1.f / (1.f + expf(-s_rgb[lane * 4 + 0])), cg = 1.f / (1.f + expf(-s_rgb[lane * 4 + 1])),
                      cb = 1.f / (1.f + expf(-s_rgb[lane * 4 + 2]));
          o_acc += w;
          d_acc += w * mid;
          r_acc += w * cr;
          g_acc += w * cg;
          b_acc += w * cb;
          const int64_t p = base + s_idx;
          a.sigmas[p] = sigma;
          a.weights[p] = w;
          a.trans[p] = T;
          a.kidx_out[p] = k;
          a.rgbs[p * 3 + 0] = cr;
          a.rgbs[p * 3 + 1] = cg;
          a.rgbs[p * 3 + 2] = cb;
        }
        kept += __popc(__ballot_sync(0xffffffffu, keep));
        carry *= __shfl_sync(0xffffffffu, incl, 31);
        __syncwarp();
        if (carry < a.early_stop_eps) break;  // early ray termination: everything behind is invisible
      }
    }
    o_acc = warp_sum(o_acc);
    d_acc = warp_sum(d_acc);
    r_acc = warp_sum(r_acc);
    g_acc = warp_sum(g_acc);
    b_acc = warp_sum(b_acc);
    if (lane == 0) {
      a.opacity[ray] = o_acc;
      a.depth[ray] = d_acc;
      a.acc_rgb[ray * 3 + 0] = r_acc;
      a.acc_rgb[ray * 3 + 1] = g_acc;
      a.acc_rgb[ray * 3 + 2] = b_acc;
      a.kept[ray] = kept;
      if (a.kept_blocks != nullptr && kept > 0) atomicAdd(a.kept_blocks + (ray >> 8), kept);
    }
    __syncwarp();
  }
}

// kept prefix of every ray: loose (offsets_m) -> packed (offsets_k), for the exact-size per-sample outputs.
// SCAN = true (nsr_pack_kept_scan): the packed offsets are computed HERE instead of by a one-CTA scan kernel in front: every CTA sums
// the kept counts of the rays before its own eight (n_rays^2 / 16 ints of L2 reads in total: 17 MB at 8192 rays) and writes
// off_k_out[ray] (+ off_k_out[n_rays] by the last CTA) for the kernels behind it.
template <bool SCAN>
__global__ void __launch_bounds__(256) pack_kept_kernel(const int64_t* __restrict__ off_m, const int64_t* __restrict__ off_k,
                                                        const int32_t* __restrict__ kept, int64_t* __restrict__ off_k_out,
                                                        const float* __restrict__ t_min, float step, const int32_t* __restrict__ kidx,
                                                        const float* __restrict__ weights, int32_t* __restrict__ ri_k,
                                                        float* __restrict__ ts_k, float* __restrict__ te_k, float* __restrict__ w_k,
                                                        int64_t* __restrict__ loose_pos, const __grid_constant__ nsr_nerf_t P,
                                                        const float* __restrict__ rays, const uint4* __restrict__ enc_loose,
                                                        uint4* __restrict__ enc_k, float* __restrict__ xyzdir_k, int enc_tiled, int64_t n_rays,
                                                        const int32_t* __restrict__ kept_blocks) {
  const int lane = threadIdx.x & 31;
  const int64_t ray = blockIdx.x * 8ll + (threadIdx.x >> 5);
  int64_t dst, cnt;
  if (SCAN) {
    __shared__ int64_t s_part[8];
    const int64_t ray0 = blockIdx.x * 8ll;
    int64_t sum = 0;
    if (kept_blocks != nullptr) {  // whole 256-ray blocks in front come as sums from the forward kernel: <= 32 + 255 loads instead of n_rays
      const int64_t nb = ray0 >> 8;
      for (int64_t b = threadIdx.x; b < nb; b += 256) sum += __ldg(kept_blocks + b);
      for (int64_t r = (nb << 8) + threadIdx.x; r < ray0; r += 256) sum += __ldg(kept + r);
    } else {
      for (int64_t r = threadIdx.x; r < ray0; r += 256) sum += __ldg(kept + r);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (lane == 0) s_part[threadIdx.x >> 5] = sum;
    __syncthreads();
    int64_t base = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) base += s_part[w];
    for (int64_t r = ray0; r < ray && r < n_rays; ++r) base += __ldg(kept + r);  // the (at most seven) rays of this CTA in front of mine
    if (ray >= n_rays) return;
    dst = base;
    cnt = __ldg(kept + ray);
    if (lane == 0) {
      off_k_out[ray] = dst;
      if (ray == n_rays - 1) off_k_out[n_rays] = dst + cnt;
    }
  } else {
    if (ray >= n_rays) return;
    dst = off_k[ray];
    cnt = off_k[ray + 1] - dst;
  }
  const int64_t src = off_m[ray];
  const float tmin = t_min[ray];
  for (int64_t j = lane; j < cnt; j += 32) {
    const float k = (float)kidx[src + j];
    const float t0 = __fmaf_rn(k, step, tmin), t1 = __fmaf_rn(k + 1.f, step, tmin);
    ri_k[dst + j] = (int32_t)ray;
    ts_k[dst + j] = t0;
    te_k[dst + j] = t1;
    if (w_k) w_k[dst + j] = weights[src + j];
    if (loose_pos) loose_pos[dst + j] = src + j;
    if (xyzdir_k) {  // inputs of the tile backward in packed order: unit-cube position + view direction, encoded features
      float x, y, z, dx, dy, dz;
      nf_sample_position(P, rays, (int)ray, t0, t1, x, y, z, dx, dy, dz);
      float* o = xyzdir_k + (dst + j) * 6;
      o[0] = x; o[1] = y; o[2] = z; o[3] = dx; o[4] = dy; o[5] = dz;
    }
  }
  if (enc_k && !enc_tiled) {  // 64 B rows: 4 lanes per row => every warp iteration moves 8 whole rows with fully used sectors
    for (int64_t v = lane; v < cnt * 4; v += 32) enc_k[dst * 4 + v] = enc_loose[src * 4 + v];
  } else if (enc_k) {
    // canonical tensor-core tile layout for the wgmma backward (csrc/nerf_bwd_tc.cu): packed row R lives in tile R / 128 (8 KB each); inside a
    // tile the 16-byte chunk (row r, k chunk kc) sits at ((r / 8) * 4 + kc) * 128 + (r % 8) * 16 bytes -- ONE cp.async.bulk then fetches a tile
    for (int64_t v = lane; v < cnt * 4; v += 32) {
      const int64_t R = dst + (v >> 2);
      const int kc = (int)(v & 3), r = (int)(R & 127);
      enc_k[(R >> 7) * 512 + ((r >> 3) * 4 + kc) * 8 + (r & 7)] = enc_loose[src * 4 + v];
    }
  }
}

// compositing backward on the loose layout (one warp per ray, reverse chunks, suffix carry): d_sraw, d_rgb (loose), amax
__global__ void __launch_bounds__(256) ray_bwd_loose_kernel(const int64_t* __restrict__ off_m, const int32_t* __restrict__ kept,
                                                            const float* __restrict__ t_min, float step, const int32_t* __restrict__ kidx,
                                                            const float* __restrict__ trans, const float* __restrict__ weights,
                                                            const float* __restrict__ sigmas, const float* __restrict__ rgbs,
                                                            const float* __restrict__ g_rgb, const float* __restrict__ g_opacity,
                                                            const float* __restrict__ g_depth, const float* __restrict__ g_weights,
                                                            float* __restrict__ d_sraw, float* __restrict__ d_rgb, float* __restrict__ amax,
                                                            const int64_t* __restrict__ off_k, int64_t n_rays) {
  const int lane = threadIdx.x & 31;
  const int64_t ray = blockIdx.x * 8ll + (threadIdx.x >> 5);
  if (ray >= n_rays) return;
  const int64_t beg = off_m[ray];
  const int64_t out0 = off_k ? off_k[ray] : beg;  // off_k != NULL: gradients are written in packed row order
  const int n = kept[ray];
  if (n <= 0) return;
  const float tmin = t_min[ray];
  const float gr = g_rgb ? g_rgb[ray * 3 + 0] : 0.f, gg = g_rgb ? g_rgb[ray * 3 + 1] : 0.f, gb = g_rgb ? g_rgb[ray * 3 + 2] : 0.f;
  const float go = g_opacity ? g_opacity[ray] : 0.f, gd = g_depth ? g_depth[ray] : 0.f;
  float carry = 0.f, vmax = 0.f;
  for (int cb = ((n - 1) / 32) * 32; cb >= 0; cb -= 32) {
    const int j = cb + lane;
    const bool ok = j < n;
    const int64_t i = beg + j;
    float w = 0.f, gi = 0.f, delta = 0.f;
    if (ok) {
      w = weights[i];
      const float kf = (float)kidx[i];
      const float t0 = __fmaf_rn(kf, step, tmin), t1 = __fmaf_rn(kf + 1.f, step, tmin);
      delta = t1 - t0;
      gi = gr * rgbs[i * 3 + 0] + gg * rgbs[i * 3 + 1] + gb * rgbs[i * 3 + 2] + go + gd * ((t0 + t1) * 0.5f) + (g_weights ? g_weights[i] : 0.f);
      d_rgb[(out0 + j) * 3 + 0] = w * gr;
      d_rgb[(out0 + j) * 3 + 1] = w * gg;
      d_rgb[(out0 + j) * 3 + 2] = w * gb;
      vmax = fmaxf(vmax, 0.25f * w * fmaxf(fabsf(gr), fmaxf(fabsf(gg), fabsf(gb))));
    }
    const float gw = gi * w;
    float suf = gw;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float t = __shfl_down_sync(0xffffffffu, suf, o);
      if (lane + o < 32) suf += t;
    }
    if (ok) {
      const float ds = delta * (gi * (trans[i] - w) - (carry + suf - gw));
      const float dr = ds * fminf(sigmas[i], 3269017.37f);
      d_sraw[out0 + j] = dr;
      vmax = fmaxf(vmax, fabsf(dr));
    }
    carry += __shfl_sync(0xffffffffu, suf, 0);
  }
  if (amax != nullptr) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
    if (lane == 0 && vmax > 0.f && isfinite(vmax)) atomicMax(reinterpret_cast<int*>(amax), __float_as_int(vmax));
  }
}

}  // namespace

extern "C" int nsr_nerf_rays_fwd(const nsr_nerf_t* f, const float* rays, const uint32_t* masks, int32_t words, const float* t_min,
                                 const int64_t* offsets_m, const int32_t* order, float step, float early_stop_eps, const void* dparams_h, const void* cparams_h,
                                 void* enc_save_h, float* sigmas, float* rgbs, float* weights, float* trans, int32_t* kidx,
                                 float* acc_rgb, float* opacity, float* depth, int32_t* kept, uint32_t* ticket, int64_t n_rays,
                                 const int32_t* counts, const int32_t* bin_counts, int32_t* kept_blocks, void* stream) {
  NSR_REQUIRE(bin_counts == nullptr || (order != nullptr && counts != nullptr), "nsr_nerf_rays_fwd: the binned queue needs order [8][n] and counts");
  NSR_REQUIRE(f != nullptr && f->grid.n_levels == 16 && f->grid.n_features == 2 && f->feature_dim == 16 && f->density_hidden == 1 &&
                  f->color_hidden == 2 && f->contraction == 0,
              "nsr_nerf_rays_fwd: fused path needs L=16, F=2, feature_dim=16, hidden layers 1/2, AABB contraction");
  NSR_REQUIRE(words >= 1 && words <= kMaxWords, "nsr_nerf_rays_fwd: words must be in [1,%d]", kMaxWords);
  NSR_REQUIRE(ticket != nullptr && kept != nullptr, "nsr_nerf_rays_fwd: ticket / kept are required");
  if (n_rays == 0) return 0;
  static thread_local bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(nerf_rays_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes);
    if (e != cudaSuccess) {
      nsr_set_error("nsr_nerf_rays_fwd: cannot reserve %zu B shared memory: %s", kSmemBytes, cudaGetErrorString(e));
      return 2;
    }
    attr_set = true;
  }
  RaysFwdArgs a;
  a.rays = rays; a.masks = masks; a.t_min = t_min; a.offsets_m = offsets_m; a.order = order; a.bin_counts = bin_counts; a.counts = counts; a.kept_blocks = kept_blocks;
  a.dparams = (const __half*)dparams_h; a.cparams = (const __half*)cparams_h; a.enc_save = (__half*)enc_save_h;
  a.sigmas = sigmas; a.rgbs = rgbs; a.weights = weights; a.trans = trans; a.kidx_out = kidx;
  a.acc_rgb = acc_rgb; a.opacity = opacity; a.depth = depth; a.kept = kept; a.ticket = ticket;
  a.step = step; a.early_stop_eps = early_stop_eps; a.words = words; a.n_rays = n_rays;
  const int64_t want = (n_rays + kWarps - 1) / kWarps;
  int grid = (int)min((int64_t)nsr_sm_count() * 2, want > 0 ? want : (int64_t)1);
  nerf_rays_fwd_kernel<<<grid, kThreads, kSmemBytes, (cudaStream_t)stream>>>(*f, a);
  NSR_CHECK_LAUNCH("nsr_nerf_rays_fwd");
  return 0;
}

extern "C" int nsr_pack_kept(const int64_t* offsets_m, const int64_t* offsets_k, const float* t_min, float step, const int32_t* kidx,
                             const float* weights, int32_t* ray_indices_k, float* t_starts_k, float* t_ends_k, float* weights_k,
                             int64_t* loose_pos, const nsr_nerf_t* f, const float* rays, const void* enc_loose_h, void* enc_k_h,
                             float* xyzdir_k, int32_t enc_tiled, int64_t n_rays, void* stream) {
  if (n_rays == 0) return 0;
  NSR_REQUIRE(xyzdir_k == nullptr || (f != nullptr && rays != nullptr), "nsr_pack_kept: xyzdir_k needs the field descriptor and the rays");
  NSR_REQUIRE(enc_k_h == nullptr || enc_loose_h != nullptr, "nsr_pack_kept: enc_k needs the loose encoding buffer");
  nsr_nerf_t dummy;
  memset(&dummy, 0, sizeof(dummy));
  dummy.radius = 1.f;
  pack_kept_kernel<false><<<nsr_blocks(n_rays, 8), 256, 0, (cudaStream_t)stream>>>(offsets_m, offsets_k, nullptr, nullptr, t_min, step, kidx, weights,
                                                                                   ray_indices_k, t_starts_k, t_ends_k, weights_k, loose_pos,
                                                                                   f ? *f : dummy, rays, (const uint4*)enc_loose_h,
                                                                                   (uint4*)enc_k_h, xyzdir_k, enc_tiled, n_rays, nullptr);
  NSR_CHECK_LAUNCH("nsr_pack_kept");
  return 0;
}

extern "C" int nsr_pack_kept_scan(const int64_t* offsets_m, const int32_t* kept, int64_t* offsets_k_out, const float* t_min, float step,
                                  const int32_t* kidx, const float* weights, int32_t* ray_indices_k, float* t_starts_k, float* t_ends_k,
                                  float* weights_k, int64_t* loose_pos, const nsr_nerf_t* f, const float* rays, const void* enc_loose_h,
                                  void* enc_k_h, float* xyzdir_k, int32_t enc_tiled, int64_t n_rays, const int32_t* kept_blocks, void* stream) {
  NSR_REQUIRE(kept != nullptr && offsets_k_out != nullptr, "nsr_pack_kept_scan: kept / offsets_k_out is NULL");
  if (n_rays == 0) {
    cudaMemsetAsync(offsets_k_out, 0, sizeof(int64_t), (cudaStream_t)stream);
    return 0;
  }
  NSR_REQUIRE(xyzdir_k == nullptr || (f != nullptr && rays != nullptr), "nsr_pack_kept_scan: xyzdir_k needs the field descriptor and the rays");
  NSR_REQUIRE(enc_k_h == nullptr || enc_loose_h != nullptr, "nsr_pack_kept_scan: enc_k needs the loose encoding buffer");
  nsr_nerf_t dummy;
  memset(&dummy, 0, sizeof(dummy));
  dummy.radius = 1.f;
  pack_kept_kernel<true><<<nsr_blocks(n_rays, 8), 256, 0, (cudaStream_t)stream>>>(offsets_m, nullptr, kept, offsets_k_out, t_min, step, kidx, weights,
                                                                                  ray_indices_k, t_starts_k, t_ends_k, weights_k, loose_pos,
                                                                                  f ? *f : dummy, rays, (const uint4*)enc_loose_h,
                                                                                  (uint4*)enc_k_h, xyzdir_k, enc_tiled, n_rays, kept_blocks);
  NSR_CHECK_LAUNCH("nsr_pack_kept_scan");
  return 0;
}

extern "C" int nsr_nerf_ray_bwd_loose(const int64_t* offsets_m, const int32_t* kept, const float* t_min, float step, const int32_t* kidx,
                                      const float* trans, const float* weights, const float* sigmas, const float* rgbs, const float* g_rgb,
                                      const float* g_opacity, const float* g_depth, const float* g_weights, float* d_sraw, float* d_rgb,
                                      float* amax, const int64_t* offsets_k, int64_t n_rays, void* stream) {
  if (n_rays == 0) return 0;
  ray_bwd_loose_kernel<<<nsr_blocks(n_rays, 8), 256, 0, (cudaStream_t)stream>>>(offsets_m, kept, t_min, step, kidx, trans, weights, sigmas, rgbs,
                                                                                g_rgb, g_opacity, g_depth, g_weights, d_sraw, d_rgb, amax, offsets_k, n_rays);
  NSR_CHECK_LAUNCH("nsr_nerf_ray_bwd_loose");
  return 0;
}
