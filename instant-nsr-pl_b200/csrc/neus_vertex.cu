// Per-vertex colour of an exported NeuS mesh (NeuSModel.export, models/neus.py:321-329 with export_vertex_color): per vertex
//   SDF field + normal -> n = F.normalize(grad) -> colour network [feature | SH4(-n) | n] -> colour activation
// in ONE kernel, writing rgb [n,3] and nothing else.  The field stages are the per-ray NeuS eval renderer's (neus_render.cu): the
// analytic field of neus_field.cuh (tensor-core encoding tiles, 32 vertices per warp) or the finite-difference field of
// neus_field_fd.cuh (centre with every output, then the six stencil points for the SDF alone, normal 0.5 (s+ - s-) / eps), and the colour
// network is radiance.cuh's 16-row pass.  The only difference from the renderer is the view direction: -n, the colour "seen along the
// normal".  The per-op path this replaces holds sdf [V], grad [V,3] and feature [V,13] in fp32 for every vertex at once.
#include "neus_field.cuh"
#include "neus_field_fd.cuh"
#include "radiance.cuh"

namespace {

constexpr int kThreads = kNeusTcWarps * 32;   // 128: the field's per-warp encoding tiles are sized for this CTA
constexpr int kFeat = 13;                     // colour input [feature 13 | SH4 16 | normal 3] (every NeuS config of the reference)

struct VertexWarpSmem {
  __half X[32][LD32];      // colour network input rows
  float out[32][NOUTP];    // field output rows (sdf, feature)
};
template <bool FD>
constexpr size_t kFieldSmem = FD ? sizeof(fd::FdW) : sizeof(NeusTcSmem);
template <bool FD>
constexpr size_t kVertexSmem = kFieldSmem<FD> + W_TOTAL * sizeof(__half) + N_BIAS * sizeof(float) + kNeusTcWarps * sizeof(VertexWarpSmem);
static_assert(sizeof(NeusTcSmem) % 16 == 0 && sizeof(fd::FdW) % 16 == 0 && (W_TOTAL * sizeof(__half)) % 16 == 0 &&
                  (N_BIAS * sizeof(float)) % 16 == 0, "16-byte aligned");
template <bool FD>
constexpr int kCtasPerSm = FD ? 4 : 2;

struct VertexArgs {
  const float* verts;           // [n, 3] world coordinates
  const __half2* table;
  const float *W1, *b1, *W2, *b2;
  const float* field_state;     // analytic: n_active (device float); FD: {eps, eps^2, n_active}
  const __half* rgb_params;
  const float* rgb_bias;
  float* rgb;                   // [n, 3]
  float radius;
  int32_t n_out, act_mode;
  int64_t n;
};

// A warp takes 32 consecutive vertices per group, groups grid-strided over the warps of the launch.
template <bool VANILLA, bool FD>
__global__ void __launch_bounds__(kThreads, kCtasPerSm<FD>) neus_vertex_rgb_kernel(const __grid_constant__ nsr_grid_t g,
                                                                                   const __grid_constant__ VertexArgs a) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  NeusTcSmem& S = *reinterpret_cast<NeusTcSmem*>(smem_raw);
  fd::FdW& Wf = *reinterpret_cast<fd::FdW*>(smem_raw);
  __half* RW = reinterpret_cast<__half*>(smem_raw + kFieldSmem<FD>);
  float* rbias = reinterpret_cast<float*>(RW + W_TOTAL);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  VertexWarpSmem& Wp = reinterpret_cast<VertexWarpSmem*>(rbias + N_BIAS)[warp];
  if constexpr (FD)
    fd::stage_weights(Wf, a.W1, a.b1, a.W2, a.b2, a.n_out);
  else
    stage_neus_tc_weights(S, a.W1, a.b1, a.W2, a.b2, a.n_out);
  stage_weights(RW, a.rgb_params);
  if (VANILLA) stage_bias(rbias, a.rgb_bias);
  __syncthreads();
  const int n_active = FD ? (int)__ldg(a.field_state + 2) : load_n_active(a.field_state);
  const float eps = FD ? __ldg(a.field_state) : 0.f;
  const float inv2r = 1.f / (2.f * a.radius);
  const int64_t n_groups = (a.n + 31) / 32;

  for (int64_t grp = (int64_t)blockIdx.x * kNeusTcWarps + warp; grp < n_groups; grp += (int64_t)gridDim.x * kNeusTcWarps) {
    const int64_t i = grp * 32 + lane;
    const bool ok = i < a.n;
    float px = 0.f, py = 0.f, pz = 0.f;   // world-space vertex (dead lanes: the box centre)
    if (ok) {
      px = __ldg(a.verts + i * 3 + 0);
      py = __ldg(a.verts + i * 3 + 1);
      pz = __ldg(a.verts + i * 3 + 2);
    }
    float gx = 0.f, gy = 0.f, gz = 0.f;
    if constexpr (FD) {
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
      // neus_field_fwd_tc_kernel's unit-cube position (dead lanes: the cube centre)
      const float x = ok ? (px + a.radius) * inv2r : 0.5f, y = ok ? (py + a.radius) * inv2r : 0.5f, z = ok ? (pz + a.radius) * inv2r : 0.5f;
      neus_field_rows32<true>(
          S, warp, lane, g, a.table, x, y, z, ok, n_active, [&](int r0, int gq, int dr, int col, float v) { Wp.out[r0 + gq + dr][col] = v; },
          [&](float gx_, float gy_, float gz_) {
            gx = gx_ * inv2r;
            gy = gy_ * inv2r;
            gz = gz_ * inv2r;
          });
    }
    __syncwarp();
    // F.normalize(grad): g / max(||g||, 1e-12) in torch's order.  Its CUDA norm reduces a 3-wide row with two threads (block width
    // last_pow2(3)): thread 0 sums x^2 + z^2, thread 1 holds y^2, and a shuffle adds them -- (x^2 + z^2) + y^2, each square rounded on
    // its own, no fused multiply-add.  Any other order changes ||g|| in the last bit for about 12 % of the normals, and that flips
    // fp16 roundings of the colour network's input.  Then a true division.
    const float ss = __fadd_rn(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gz, gz)), __fmul_rn(gy, gy));
    const float nrm = fmaxf(sqrtf(ss), 1e-12f);
    const float nx = __fdiv_rn(gx, nrm), ny = __fdiv_rn(gy, nrm), nz = __fdiv_rn(gz, nrm);
    {  // colour network input row [feature | SH4(-n) | n] (dead lanes: all zero)
      float sh[16];
      nsr_sh4(-nx, -ny, -nz, sh);
      __half* xr = Wp.X[lane];
#pragma unroll
      for (int c = 0; c < 32; ++c) {
        const float v = c < kFeat ? Wp.out[lane][c] : c < kFeat + 16 ? sh[c - kFeat] : c == kFeat + 16 ? nx : c == kFeat + 17 ? ny : nz;
        xr[c] = __float2half_rn(ok ? v : 0.f);
      }
    }
    __syncwarp();
#pragma unroll 1
    for (int m = 0; m < 2; ++m) {
      float acc16[1][2][4];
      radiance_rows16<VANILLA>(acc16, &Wp.X[0][0], m * 16, RW, rbias);
      const int gq = lane >> 2, cq = lane & 3;
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = cq * 2 + e;
          const int64_t r = grp * 32 + m * 16 + gq + hh * 8;
          if (col < 3 && r < a.n) a.rgb[r * 3 + col] = out_value<VANILLA>(acc16[0][0][hh * 2 + e], a.act_mode);
        }
    }
    __syncwarp();   // Wp is rewritten by the next group
  }
}

template <bool VANILLA, bool FD>
int launch(const nsr_grid_t* g, const VertexArgs& a, cudaStream_t st, const char* name) {
  static thread_local bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(neus_vertex_rgb_kernel<VANILLA, FD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kVertexSmem<FD>);
    if (e != cudaSuccess) {
      nsr_set_error("%s: cannot reserve %zu B shared memory: %s", name, kVertexSmem<FD>, cudaGetErrorString(e));
      return 2;
    }
    attr_set = true;
  }
  const int64_t n_groups = (a.n + 31) / 32;
  const int grid = (int)min((int64_t)nsr_sm_count() * kCtasPerSm<FD>, (n_groups + kNeusTcWarps - 1) / kNeusTcWarps);
  neus_vertex_rgb_kernel<VANILLA, FD><<<grid, kThreads, kVertexSmem<FD>, st>>>(*g, a);
  NSR_CHECK_LAUNCH(name);
  return 0;
}

// both entry points: field_state is n_active (analytic field) or fd_state (finite-difference field)
template <bool FD>
int vertex_rgb(const char* name, const nsr_grid_t* g, const float* verts, const void* table_h, const float* W1, const float* b1, const float* W2,
               const float* b2, float radius, int32_t n_out, const float* field_state, const nsr_radiance_t* rp, int32_t vanilla,
               const void* rgb_params_h, const float* rgb_bias, float* rgb, int64_t n, void* stream) {
  NSR_REQUIRE(g != nullptr && g->n_levels == 16 && g->n_features == 2, "%s: needs a 16-level F=2 hash grid", name);
  NSR_REQUIRE(rp != nullptr && n_out == kFeat && rp->n_feat == kFeat && rp->n_extra == 3,
              "%s: the colour input must be [feature (13) | SH4 (16) | normal (3)]", name);
  NSR_REQUIRE(rp->act_mode >= 0 && rp->act_mode <= 2, "%s: act_mode must be 0, 1 or 2", name);
  NSR_REQUIRE(n >= 0, "%s: n must be >= 0", name);
  NSR_REQUIRE(verts && table_h && W1 && b1 && W2 && b2 && rgb_params_h && rgb, "%s: NULL argument", name);
  NSR_REQUIRE(field_state != nullptr, FD ? "%s: fd_state (device {eps, eps^2, n_active}) is NULL" : "%s: n_active is NULL", name);
  NSR_REQUIRE(!vanilla || rgb_bias != nullptr, "%s: the VanillaMLP colour network needs its bias", name);
  if (n == 0) return 0;
  VertexArgs a;
  a.verts = verts, a.table = (const __half2*)table_h, a.W1 = W1, a.b1 = b1, a.W2 = W2, a.b2 = b2, a.field_state = field_state;
  a.rgb_params = (const __half*)rgb_params_h, a.rgb_bias = rgb_bias, a.rgb = rgb;
  a.radius = radius, a.n_out = n_out, a.act_mode = rp->act_mode, a.n = n;
  const cudaStream_t st = (cudaStream_t)stream;
  return vanilla ? launch<true, FD>(g, a, st, name) : launch<false, FD>(g, a, st, name);
}

}  // namespace

extern "C" int nsr_neus_vertex_rgb(const nsr_grid_t* g, const float* verts, const void* table_h, const float* W1, const float* b1,
                                   const float* W2, const float* b2, float radius, int32_t n_out, const float* n_active,
                                   const nsr_radiance_t* rp, int32_t vanilla, const void* rgb_params_h, const float* rgb_bias, float* rgb,
                                   int64_t n, void* stream) {
  return vertex_rgb<false>("nsr_neus_vertex_rgb", g, verts, table_h, W1, b1, W2, b2, radius, n_out, n_active, rp, vanilla, rgb_params_h,
                           rgb_bias, rgb, n, stream);
}

extern "C" int nsr_neus_vertex_rgb_fd(const nsr_grid_t* g, const float* verts, const void* table_h, const float* W1, const float* b1,
                                      const float* W2, const float* b2, float radius, int32_t n_out, const float* fd_state,
                                      const nsr_radiance_t* rp, int32_t vanilla, const void* rgb_params_h, const float* rgb_bias, float* rgb,
                                      int64_t n, void* stream) {
  return vertex_rgb<true>("nsr_neus_vertex_rgb_fd", g, verts, table_h, W1, b1, W2, b2, radius, n_out, fd_state, rp, vanilla, rgb_params_h,
                          rgb_bias, rgb, n, stream);
}
