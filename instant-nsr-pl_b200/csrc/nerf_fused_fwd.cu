// Fused NeRF forward kernels: sample -> position -> 16-level hash gather -> density MLP -> SH4 -> colour MLP
// -> trunc_exp / sigmoid -> weights -> per-ray sums, in ONE launch (replaces ~25 torch kernels + 2 tcnn module
// calls + 4 nerfacc calls of models/nerf.py:95-109).  A warp owns 32 consecutive samples (consecutive samples
// of a ray share coarse hash cells -> coalesced gathers); the encoded features go registers -> smem tile ->
// tensor-core fragments and never touch HBM (tcnn round-trips them: 64 B write + 64 B read per sample).
#include "nerf_fused.cuh"

namespace {

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
// per-warp scratch (halves): A tile [32][40] + SH tile [32][24] + sigma (32 f32) + rgb (32 x 4 f32)
constexpr int kWarpHalves = 32 * NF_LD32 + 32 * 24 + 64 + 256;
constexpr size_t kSmemBytes = (size_t)(NF_W_TOTAL + kWarps * kWarpHalves) * sizeof(__half);

enum { MODE_DENSITY = 0, MODE_PREPASS = 1, MODE_RENDER = 2 };

struct FwdArgs {
  const float* rays;          // [n_rays,6]           (PREPASS / RENDER)
  const float* positions;     // [n,3] world          (DENSITY)
  const int32_t* ray_indices; // [n]
  const float* t_starts;
  const float* t_ends;
  const float* trans;         // [n] exclusive transmittance carried from the pre-pass (RENDER)
  const __half* dparams;      // [3072 | table]
  const __half* cparams;      // [7168]
  __half* enc_save;           // [n,32] or NULL
  float* out0;                // DENSITY: density[n]; PREPASS: alphas[n]; RENDER: sigmas[n]
  float* rgbs;                // [n,3]
  float* weights;             // [n]
  float* acc_rgb;             // [n_rays,3]
  float* opacity;             // [n_rays]
  float* depth;               // [n_rays]
  int64_t n;                  // sample count (capacity when n_dev is set)
  const int64_t* n_dev;       // optional: the count lives on the device (no host sync / graph capture)
  const __half* table;        // hash table (fp16); FullyFused: dparams + NF_DENSITY_PARAMS
  const float* dbias;         // VanillaMLP: density biases [80]
  const float* cbias;         // VanillaMLP: colour biases [144]   (RENDER)
};
template <int NET>
constexpr size_t fwd_smem() { return kSmemBytes + (NET == NF_NET_VANILLA ? NF_B_TOTAL * sizeof(float) : 0); }

// CT: the field's contraction (NF_AABB / NF_UNBOUNDED_SPHERE), a template parameter so that the AABB build is unchanged
// NET: the network variant (NF_NET_FULLY_FUSED / NF_NET_VANILLA).  VanillaMLP: the accumulators start from the fp32 biases, the density
// and colour outputs stay fp32 (the rounding points of nsr_mlp_vanilla_fwd / nsr_radiance_vanilla_fwd); the feature columns that feed the
// colour network are rounded to fp16 as those kernels' inputs are.
// (VanillaMLP render: the bias accumulators need a few registers more than 128, so that instantiation is sized for one CTA per SM)
template <int MODE, int CT, int NET>
__global__ void __launch_bounds__(kThreads, NET == NF_NET_VANILLA && MODE == MODE_RENDER ? 1 : 2) nerf_fwd_kernel(const __grid_constant__ nsr_nerf_t P, const FwdArgs a) {
  extern __shared__ __align__(16) __half smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, c = lane & 3;
  __half* At = smem + NF_W_TOTAL + warp * kWarpHalves;
  __half* St = At + 32 * NF_LD32;
  float* s_sig = reinterpret_cast<float*>(St + 32 * 24);
  float* s_rgb = s_sig + 32;
  float* bias_sm = reinterpret_cast<float*>(smem + NF_W_TOTAL + kWarps * kWarpHalves);  // VanillaMLP only
  // (FullyFused: the table follows the density network in dparams; deriving it here keeps that build's machine code as it was)
  const __half2* table = reinterpret_cast<const __half2*>(NET == NF_NET_VANILLA ? a.table : a.dparams + NF_DENSITY_PARAMS);
  nf_stage_weights(smem, a.dparams, a.cparams, MODE == MODE_RENDER);
  if (NET == NF_NET_VANILLA) nf_stage_bias(bias_sm, a.dbias, a.cbias, MODE == MODE_RENDER);
  __syncthreads();

  const int64_t n_total = a.n_dev ? min(*a.n_dev, a.n) : a.n;
  const int64_t n_tiles = (n_total + 31) / 32;
  for (int64_t tile = (int64_t)blockIdx.x * kWarps + warp; tile < n_tiles; tile += (int64_t)gridDim.x * kWarps) {
    const int64_t i = tile * 32 + lane;
    const bool valid = i < n_total;
    float x = 0.f, y = 0.f, z = 0.f, dx = 0.f, dy = 0.f, dz = 1.f, t0 = 0.f, t1 = 0.f;
    int ray = -1;
    if (valid) {
      if (MODE == MODE_DENSITY) {
        x = a.positions[i * 3 + 0];
        y = a.positions[i * 3 + 1];
        z = a.positions[i * 3 + 2];
        nf_contract<CT>(P, x, y, z);
      } else {
        ray = a.ray_indices[i];
        t0 = a.t_starts[i];
        t1 = a.t_ends[i];
        nf_sample_position<CT>(P, a.rays, ray, t0, t1, x, y, z, dx, dy, dz);
      }
    }
    uint32_t f[16];
    if (valid) {
      nf_gather<16>(P.grid, table, x, y, z, f);
    } else {
#pragma unroll
      for (int l = 0; l < 16; ++l) f[l] = 0u;
    }
    nf_store_row32(At, lane, f);
    if (MODE == MODE_RENDER) {
      if (a.enc_save != nullptr && valid) {
        uint4* e = reinterpret_cast<uint4*>(a.enc_save + i * 32);
        e[0] = make_uint4(f[0], f[1], f[2], f[3]);
        e[1] = make_uint4(f[4], f[5], f[6], f[7]);
        e[2] = make_uint4(f[8], f[9], f[10], f[11]);
        e[3] = make_uint4(f[12], f[13], f[14], f[15]);
      }
      float s[16];
      nsr_sh4(dx, dy, dz, s);  // tcnn SH takes (d+1)/2 and maps back to d (texture.py:24): net effect is SH(d)
      uint4* sp = reinterpret_cast<uint4*>(St + lane * 24);
      sp[0] = make_uint4(nsr_pack_h2(s[0], s[1]), nsr_pack_h2(s[2], s[3]), nsr_pack_h2(s[4], s[5]), nsr_pack_h2(s[6], s[7]));
      sp[1] = make_uint4(nsr_pack_h2(s[8], s[9]), nsr_pack_h2(s[10], s[11]), nsr_pack_h2(s[12], s[13]), nsr_pack_h2(s[14], s[15]));
    }
    __syncwarp();

    // ---- density network: 32 -> 64 (ReLU) -> 16
    uint32_t a_o[2][1][4];
    {
      uint32_t a_in[2][2][4];
      nsr_load_afrag<2, 2>(a_in, At, NF_LD32, 0);
      float acc[2][8][4];
      nf_init_acc<NET>(acc, bias_sm + NF_B_D1);
      nsr_gemm_w<2, 2, 8>(acc, a_in, smem + NF_OFF_DW1, NF_LD32);
      uint32_t a_h[2][4][4];
      nsr_acc_to_afrag<2, 8>(acc, a_h, NSR_ACT_RELU);
      float acco[2][2][4];
      nf_init_acc<NET>(acco, bias_sm + NF_B_D2);
      nsr_gemm_w<2, 4, 2>(acco, a_h, smem + NF_OFF_DW2, NSR_LD64);
      nsr_acc_to_afrag<2, 2>(acco, a_o, NSR_ACT_NONE);  // fp16 like tcnn's network output (VanillaMLP: the colour network's input)
      if (NET == NF_NET_VANILLA && c == 0) {  // VanillaMLP: the density output stays fp32
#pragma unroll
        for (int m = 0; m < 2; ++m) {
          s_sig[m * 16 + g] = acco[m][0][0];
          s_sig[m * 16 + g + 8] = acco[m][0][2];
        }
      }
    }
    if (NET != NF_NET_VANILLA && c == 0) {
#pragma unroll
      for (int m = 0; m < 2; ++m) {
        s_sig[m * 16 + g] = nf_half_lo(a_o[m][0][0]);
        s_sig[m * 16 + g + 8] = nf_half_lo(a_o[m][0][1]);
      }
    }
    if (MODE == MODE_RENDER) {
      // ---- colour network: [feature(16) | SH(16)] -> 64 -> 64 -> 3 (padded 16)
      uint32_t a_c[2][2][4];
      {
        uint32_t a_sh[2][1][4];
        nsr_load_afrag<2, 1>(a_sh, St, 24, 0);
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            a_c[m][0][j] = a_o[m][0][j];
            a_c[m][1][j] = a_sh[m][0][j];
          }
      }
      float acc[2][8][4];
      nf_init_acc<NET>(acc, bias_sm + NF_B_C1);
      nsr_gemm_w<2, 2, 8>(acc, a_c, smem + NF_OFF_CW1, NF_LD32);
      uint32_t a_h[2][4][4];
      nsr_acc_to_afrag<2, 8>(acc, a_h, NSR_ACT_RELU);
      nf_init_acc<NET>(acc, bias_sm + NF_B_C2);
      nsr_gemm_w<2, 4, 8>(acc, a_h, smem + NF_OFF_CW2, NSR_LD64);
      nsr_acc_to_afrag<2, 8>(acc, a_h, NSR_ACT_RELU);
      float acco[2][2][4];
      nf_init_acc<NET>(acco, bias_sm + NF_B_C3);
      nsr_gemm_w<2, 4, 2>(acco, a_h, smem + NF_OFF_CW3, NSR_LD64);
      if (NET == NF_NET_VANILLA && c < 2) {  // VanillaMLP: fp32 colour output, the sigmoid acts on the un-rounded value
#pragma unroll
        for (int m = 0; m < 2; ++m) {
          float* r0 = s_rgb + (m * 16 + g) * 4 + c * 2;
          float* r1 = s_rgb + (m * 16 + g + 8) * 4 + c * 2;
          r0[0] = acco[m][0][0];
          r0[1] = acco[m][0][1];
          r1[0] = acco[m][0][2];
          r1[1] = acco[m][0][3];
        }
      }
      uint32_t a_r[2][1][4];
      nsr_acc_to_afrag<2, 2>(acco, a_r, NSR_ACT_NONE);
      if (NET != NF_NET_VANILLA && c < 2) {
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

    // ---- per-sample epilogue (thread-per-sample again)
    const float sigma = expf(s_sig[lane] + P.density_bias);  // trunc_exp forward (models/utils.py:59)
    if (MODE == MODE_DENSITY) {
      if (valid) a.out0[i] = sigma;
    } else if (MODE == MODE_PREPASS) {
      if (valid) a.out0[i] = 1.f - expf(-sigma * (t1 - t0));
    } else {
      float w = 0.f, cr = 0.f, cg = 0.f, cb = 0.f;
      if (valid) {
        w = a.trans[i] * (1.f - expf(-sigma * (t1 - t0)));
        cr = 1.f / (1.f + expf(-s_rgb[lane * 4 + 0]));
        cg = 1.f / (1.f + expf(-s_rgb[lane * 4 + 1]));
        cb = 1.f / (1.f + expf(-s_rgb[lane * 4 + 2]));
        a.out0[i] = sigma;
        a.weights[i] = w;
        a.rgbs[i * 3 + 0] = cr;
        a.rgbs[i * 3 + 1] = cg;
        a.rgbs[i * 3 + 2] = cb;
      }
      // segmented (by ray) inclusive scan; rays ascend within the warp
      float v0 = w, v1 = w * ((t0 + t1) * 0.5f), v2 = w * cr, v3 = w * cg, v4 = w * cb;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int kr = __shfl_up_sync(0xffffffffu, ray, o);
        const float u0 = __shfl_up_sync(0xffffffffu, v0, o), u1 = __shfl_up_sync(0xffffffffu, v1, o);
        const float u2 = __shfl_up_sync(0xffffffffu, v2, o), u3 = __shfl_up_sync(0xffffffffu, v3, o);
        const float u4 = __shfl_up_sync(0xffffffffu, v4, o);
        if (lane >= o && kr == ray) {
          v0 += u0; v1 += u1; v2 += u2; v3 += u3; v4 += u4;
        }
      }
      const int next_ray = __shfl_down_sync(0xffffffffu, ray, 1);
      if (valid && (lane == 31 || next_ray != ray)) {
        atomicAdd(a.opacity + ray, v0);
        atomicAdd(a.depth + ray, v1);
        atomicAdd(a.acc_rgb + (size_t)ray * 3 + 0, v2);
        atomicAdd(a.acc_rgb + (size_t)ray * 3 + 1, v3);
        atomicAdd(a.acc_rgb + (size_t)ray * 3 + 2, v4);
      }
    }
    __syncwarp();
  }
}

// ray r: copy its first kept prefix from the marched arrays to the compact arrays
__global__ void __launch_bounds__(256) compact_prefix_kernel(const int64_t* __restrict__ off_m, const int64_t* __restrict__ off_k,
                                                             const int32_t* __restrict__ ri_m, const float* __restrict__ ts_m,
                                                             const float* __restrict__ te_m, const float* __restrict__ tr_m,
                                                             int32_t* __restrict__ ri_k, float* __restrict__ ts_k, float* __restrict__ te_k,
                                                             float* __restrict__ tr_k, int64_t n_rays) {
  const int lane = threadIdx.x & 31;
  const int64_t ray = blockIdx.x * 8ll + (threadIdx.x >> 5);
  if (ray >= n_rays) return;
  const int64_t src = off_m[ray], dst = off_k[ray], cnt = off_k[ray + 1] - dst;
  for (int64_t j = lane; j < cnt; j += 32) {
    ri_k[dst + j] = ri_m[src + j];
    ts_k[dst + j] = ts_m[src + j];
    te_k[dst + j] = te_m[src + j];
    if (tr_k) tr_k[dst + j] = tr_m[src + j];
  }
}

// backward through the compositing, one warp per ray, reverse chunks with a suffix carry
__global__ void __launch_bounds__(256) ray_bwd_kernel(const int64_t* __restrict__ offsets, const float* __restrict__ t_starts,
                                                      const float* __restrict__ t_ends, const float* __restrict__ trans,
                                                      const float* __restrict__ weights, const float* __restrict__ sigmas,
                                                      const float* __restrict__ rgbs, const float* __restrict__ g_rgb,
                                                      const float* __restrict__ g_opacity, const float* __restrict__ g_depth,
                                                      const float* __restrict__ g_weights, float* __restrict__ d_sraw,
                                                      float* __restrict__ d_rgb, float* __restrict__ amax, int64_t n_rays) {
  const int lane = threadIdx.x & 31;
  const int64_t ray = blockIdx.x * 8ll + (threadIdx.x >> 5);
  if (ray >= n_rays) return;
  const int64_t beg = offsets[ray], end = offsets[ray + 1], n = end - beg;
  if (n <= 0) return;
  const float gr = g_rgb ? g_rgb[ray * 3 + 0] : 0.f, gg = g_rgb ? g_rgb[ray * 3 + 1] : 0.f, gb = g_rgb ? g_rgb[ray * 3 + 2] : 0.f;
  const float go = g_opacity ? g_opacity[ray] : 0.f, gd = g_depth ? g_depth[ray] : 0.f;
  float carry = 0.f, vmax = 0.f;
  for (int64_t cb = ((n - 1) / 32) * 32; cb >= 0; cb -= 32) {
    const int64_t i = beg + cb + lane;
    const bool ok = i < end;
    float w = 0.f, gi = 0.f, t0 = 0.f, t1 = 0.f;
    if (ok) {
      w = weights[i];
      t0 = t_starts[i];
      t1 = t_ends[i];
      const float cr = rgbs[i * 3 + 0], cg = rgbs[i * 3 + 1], cbv = rgbs[i * 3 + 2];
      gi = gr * cr + gg * cg + gb * cbv + go + gd * ((t0 + t1) * 0.5f) + (g_weights ? g_weights[i] : 0.f);
      d_rgb[i * 3 + 0] = w * gr;
      d_rgb[i * 3 + 1] = w * gg;
      d_rgb[i * 3 + 2] = w * gb;
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
      // d sigma, then trunc_exp backward (models/utils.py:64-66): sigma = exp(x) => exp(min(x, 15)) = min(sigma, e^15)
      const float ds = (t1 - t0) * (gi * (trans[i] - w) - (carry + suf - gw));
      const float dr = ds * fminf(sigmas[i], 3269017.37f);
      d_sraw[i] = dr;
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

int check_nerf(const nsr_nerf_t* f, const char* name) {
  NSR_REQUIRE(f != nullptr, "%s: field descriptor is NULL", name);
  NSR_REQUIRE(f->grid.n_levels == 16 && f->grid.n_features == 2, "%s: fused path needs a 16-level F=2 hash grid (got L=%d F=%d)", name,
              f->grid.n_levels, f->grid.n_features);
  NSR_REQUIRE(f->feature_dim == 16 && f->density_hidden == 1 && f->color_hidden == 2,
              "%s: fused path needs feature_dim=16, 1 density hidden layer, 2 colour hidden layers", name);
  NSR_REQUIRE(f->radius > 0.f, "%s: radius must be > 0", name);
  NSR_REQUIRE(f->contraction == NF_AABB || f->contraction == NF_UNBOUNDED_SPHERE,
              "%s: contraction type %d not implemented (AABB=0, UN_BOUNDED_SPHERE=2)", name, f->contraction);
  return 0;
}

template <int MODE, int CT, int NET = NF_NET_FULLY_FUSED>
int launch_fwd_ct(const nsr_nerf_t* f, const FwdArgs& a, cudaStream_t st, const char* name) {
  static thread_local bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(nerf_fwd_kernel<MODE, CT, NET>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fwd_smem<NET>());
    if (e != cudaSuccess) {
      nsr_set_error("%s: cannot reserve %zu B shared memory: %s", name, fwd_smem<NET>(), cudaGetErrorString(e));
      return 2;
    }
    attr_set = true;
  }
  const int64_t tiles = (a.n + 31) / 32;
  int grid = (int)min((int64_t)nsr_sm_count() * 2, (tiles + kWarps - 1) / kWarps);
  if (grid < 1) grid = 1;
  if (a.n_dev != nullptr) grid = nsr_sm_count() * 2;  // count unknown on the host: full persistent grid
  nerf_fwd_kernel<MODE, CT, NET><<<grid, kThreads, fwd_smem<NET>(), st>>>(*f, a);
  NSR_CHECK_LAUNCH(name);
  return 0;
}

template <int MODE>
int launch_fwd(const nsr_nerf_t* f, const FwdArgs& a, cudaStream_t st, const char* name) {
  if (int e = check_nerf(f, name)) return e;
  if (a.n == 0) return 0;
  if (f->contraction == NF_UNBOUNDED_SPHERE) return launch_fwd_ct<MODE, NF_UNBOUNDED_SPHERE>(f, a, st, name);
  return launch_fwd_ct<MODE, NF_AABB>(f, a, st, name);
}

// the VanillaMLP field (NeuS learned background): contracted only
template <int MODE>
int launch_bg(const nsr_nerf_t* f, const FwdArgs& a, cudaStream_t st, const char* name) {
  if (int e = check_nerf(f, name)) return e;
  NSR_REQUIRE(f->contraction == NF_UNBOUNDED_SPHERE, "%s: the VanillaMLP field needs contraction = 2 (UN_BOUNDED_SPHERE), got %d", name,
              f->contraction);
  if (a.n == 0) return 0;
  NSR_REQUIRE(a.dparams != nullptr && a.table != nullptr && a.dbias != nullptr && (MODE != MODE_RENDER || (a.cparams != nullptr && a.cbias != nullptr)),
              "%s: weights / table / biases are NULL", name);
  return launch_fwd_ct<MODE, NF_UNBOUNDED_SPHERE, NF_NET_VANILLA>(f, a, st, name);
}

}  // namespace

extern "C" int nsr_nerf_density(const nsr_nerf_t* f, const float* positions, const void* dparams_h, float* density, int64_t n,
                                void* stream) {
  FwdArgs a = {};
  a.positions = positions;
  a.dparams = (const __half*)dparams_h;
  a.table = a.dparams + NF_DENSITY_PARAMS;
  a.out0 = density;
  a.n = n;
  return launch_fwd<MODE_DENSITY>(f, a, (cudaStream_t)stream, "nsr_nerf_density");
}

extern "C" int nsr_nerf_prepass(const nsr_nerf_t* f, const float* rays, const int32_t* ray_indices, const float* t_starts,
                                const float* t_ends, const void* dparams_h, float* alphas, int64_t m, const int64_t* m_dev, void* stream) {
  FwdArgs a = {};
  a.n_dev = m_dev;
  a.rays = rays;
  a.ray_indices = ray_indices;
  a.t_starts = t_starts;
  a.t_ends = t_ends;
  a.dparams = (const __half*)dparams_h;
  a.table = a.dparams + NF_DENSITY_PARAMS;
  a.out0 = alphas;
  a.n = m;
  return launch_fwd<MODE_PREPASS>(f, a, (cudaStream_t)stream, "nsr_nerf_prepass");
}

extern "C" int nsr_nerf_render_fwd(const nsr_nerf_t* f, const float* rays, const int32_t* ray_indices, const float* t_starts,
                                   const float* t_ends, const float* trans, const void* dparams_h, const void* cparams_h,
                                   void* enc_save_h, float* sigmas, float* rgbs, float* weights, float* acc_rgb, float* opacity,
                                   float* depth, int64_t k, const int64_t* k_dev, void* stream) {
  FwdArgs a = {};
  a.n_dev = k_dev;
  a.rays = rays;
  a.ray_indices = ray_indices;
  a.t_starts = t_starts;
  a.t_ends = t_ends;
  a.trans = trans;
  a.dparams = (const __half*)dparams_h;
  a.table = a.dparams + NF_DENSITY_PARAMS;
  a.cparams = (const __half*)cparams_h;
  a.enc_save = (__half*)enc_save_h;
  a.out0 = sigmas;
  a.rgbs = rgbs;
  a.weights = weights;
  a.acc_rgb = acc_rgb;
  a.opacity = opacity;
  a.depth = depth;
  a.n = k;
  return launch_fwd<MODE_RENDER>(f, a, (cudaStream_t)stream, "nsr_nerf_render_fwd");
}

extern "C" int nsr_bg_field_prepass(const nsr_nerf_t* f, const float* rays, const int32_t* ray_indices, const float* t_starts,
                                    const float* t_ends, const void* dmlp_h, const void* table_h, const float* dbias, float* alphas, int64_t m,
                                    const int64_t* m_dev, void* stream) {
  FwdArgs a = {};
  a.n_dev = m_dev;
  a.rays = rays;
  a.ray_indices = ray_indices;
  a.t_starts = t_starts;
  a.t_ends = t_ends;
  a.dparams = (const __half*)dmlp_h;
  a.table = (const __half*)table_h;
  a.dbias = dbias;
  a.out0 = alphas;
  a.n = m;
  return launch_bg<MODE_PREPASS>(f, a, (cudaStream_t)stream, "nsr_bg_field_prepass");
}

extern "C" int nsr_bg_field_render_fwd(const nsr_nerf_t* f, const float* rays, const int32_t* ray_indices, const float* t_starts,
                                       const float* t_ends, const float* trans, const void* dmlp_h, const void* table_h, const float* dbias,
                                       const void* cmlp_h, const float* cbias, void* enc_save_h, float* sigmas, float* rgbs, float* weights,
                                       float* acc_rgb, float* opacity, float* depth, int64_t k, const int64_t* k_dev, void* stream) {
  FwdArgs a = {};
  a.n_dev = k_dev;
  a.rays = rays;
  a.ray_indices = ray_indices;
  a.t_starts = t_starts;
  a.t_ends = t_ends;
  a.trans = trans;
  a.dparams = (const __half*)dmlp_h;
  a.table = (const __half*)table_h;
  a.dbias = dbias;
  a.cparams = (const __half*)cmlp_h;
  a.cbias = cbias;
  a.enc_save = (__half*)enc_save_h;
  a.out0 = sigmas;
  a.rgbs = rgbs;
  a.weights = weights;
  a.acc_rgb = acc_rgb;
  a.opacity = opacity;
  a.depth = depth;
  a.n = k;
  return launch_bg<MODE_RENDER>(f, a, (cudaStream_t)stream, "nsr_bg_field_render_fwd");
}

extern "C" int nsr_compact_prefix(const int64_t* offsets_m, const int64_t* offsets_k, const int32_t* ray_indices_m,
                                  const float* t_starts_m, const float* t_ends_m, const float* trans_m, int32_t* ray_indices_k,
                                  float* t_starts_k, float* t_ends_k, float* trans_k, int64_t n_rays, void* stream) {
  if (n_rays == 0) return 0;
  compact_prefix_kernel<<<nsr_blocks(n_rays, 8), 256, 0, (cudaStream_t)stream>>>(offsets_m, offsets_k, ray_indices_m, t_starts_m, t_ends_m,
                                                                                 trans_m, ray_indices_k, t_starts_k, t_ends_k, trans_k,
                                                                                 n_rays);
  NSR_CHECK_LAUNCH("nsr_compact_prefix");
  return 0;
}

extern "C" int nsr_nerf_ray_bwd(const int64_t* offsets_k, const float* t_starts, const float* t_ends, const float* trans,
                                const float* weights, const float* sigmas, const float* rgbs, const float* g_rgb, const float* g_opacity,
                                const float* g_depth, const float* g_weights, float* d_sraw, float* d_rgb, float* amax, int64_t n_rays,
                                void* stream) {
  if (n_rays == 0) return 0;
  ray_bwd_kernel<<<nsr_blocks(n_rays, 8), 256, 0, (cudaStream_t)stream>>>(offsets_k, t_starts, t_ends, trans, weights, sigmas, rgbs, g_rgb,
                                                                          g_opacity, g_depth, g_weights, d_sraw, d_rgb, amax, n_rays);
  NSR_CHECK_LAUNCH("nsr_nerf_ray_bwd");
  return 0;
}
