// Mesh export of the fused NeRF density field (NeRFModel.export, models/nerf.py:153-161), in two kernels:
//   nsr_nerf_density_lattice: VolumeDensity.forward_level on n_planes x-planes of a marching-cubes lattice, written straight into a fp32
//     slab [n_planes, ny, nz] -- 4 B per lattice point against the per-op path's index arithmetic, gathered points, contraction
//     temporaries, fp16 encoding (64 B), network output (32 B) and activation temporaries;
//   nsr_nerf_vertex_rgb: the export's vertex colour texture(feature, (0,0,-1)).clamp(0,1) per mesh vertex, feature being all 16 density
//     network outputs -- the per-op colour pass holds every vertex's features at once.
// Per point both run the per-op field's arithmetic: the contraction in the op order torch runs contract_to_unisphere (below), the gather
// of hashgrid_fwd_kernel (nf_gather: same corner sequence and fmaf chain) and the mma.sync fragment chain 32 -> 64 (ReLU) -> 16 of
// mlp_fwd_kernel; the colour stage is radiance.cuh's 16-row pass, nsr_radiance_fwd's arithmetic.  A warp takes 32 consecutive points
// (lattice: z fastest) per grid-stride step.
#include "nerf_fused.cuh"
#include "radiance.cuh"

namespace {

constexpr int kWarps = 4;
constexpr int kThreads = kWarps * 32;
constexpr int kDensityHalves = NF_OFF_CW1;   // density network W1 [64][40] | W2 [16][72] of nerf_fused.cuh's layout
static_assert(LD32 == NF_LD32, "the density input tile and the colour input tile share one layout");

// world point -> unit-cube position as contract_to_unisphere (models/fields.py) runs in torch on CUDA:
//   scale_anything: (x + r) / (2r) -- a tensor divided by a Python scalar is a multiply by the fp32 reciprocal;
//   UN_BOUNDED_SPHERE: v = 2u - 1, mag = v.norm(dim=-1): torch's CUDA norm of a 3-wide row sums (x^2 + z^2) + y^2 (two threads: x and z,
//   then y through a shuffle), each square rounded on its own; |v| > 1 -> (2 - reciprocal(mag)) * (v / mag) with true divisions; v/4 + 1/2.
// (nf_contract_sphere, which the training and eval kernels use, divides by 2r and sums |v|^2 left to right: not the per-op values.)
template <int CT>
__device__ __forceinline__ void contract_torch(float radius, float inv2r, float& x, float& y, float& z) {
  x = __fmul_rn(__fadd_rn(x, radius), inv2r);
  y = __fmul_rn(__fadd_rn(y, radius), inv2r);
  z = __fmul_rn(__fadd_rn(z, radius), inv2r);
  if (CT == NF_UNBOUNDED_SPHERE) {
    float vx = __fsub_rn(__fmul_rn(x, 2.f), 1.f), vy = __fsub_rn(__fmul_rn(y, 2.f), 1.f), vz = __fsub_rn(__fmul_rn(z, 2.f), 1.f);
    const float mag = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(vx, vx), __fmul_rn(vz, vz)), __fmul_rn(vy, vy)));
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
}

// the warp's 32 rows: hash features (zero for dead lanes) -> tile X -> density network -> its 16 fp16 outputs as A fragments
// (FullyFused: bias-free, ReLU hidden layer, linear fp16 output -- the fragments mlp_fwd_kernel stores)
__device__ __forceinline__ void density_rows32(const nsr_grid_t& g, const __half2* __restrict__ table, const __half* Wd, __half* X, bool ok,
                                               float x, float y, float z, uint32_t (&a_o)[2][1][4]) {
  const int lane = threadIdx.x & 31;
  uint32_t f[16];
  if (ok) {
    nf_gather<16>(g, table, x, y, z, f);
  } else {
#pragma unroll
    for (int l = 0; l < 16; ++l) f[l] = 0u;
  }
  nf_store_row32(X, lane, f);
  __syncwarp();
  uint32_t a_in[2][2][4];
  nsr_load_afrag<2, 2>(a_in, X, NF_LD32, 0);
  float acc[2][8][4];
  nsr_zero_acc(acc);
  nsr_gemm_w<2, 2, 8>(acc, a_in, Wd + NF_OFF_DW1, NF_LD32);
  uint32_t a_h[2][4][4];
  nsr_acc_to_afrag<2, 8>(acc, a_h, NSR_ACT_RELU);
  float acco[2][2][4];
  nsr_zero_acc(acco);
  nsr_gemm_w<2, 4, 2>(acco, a_h, Wd + NF_OFF_DW2, NSR_LD64);
  nsr_acc_to_afrag<2, 2>(acco, a_o, NSR_ACT_NONE);
}

struct LatticeArgs {
  const float *ax, *ay, *az;
  const __half* dparams;   // [density network 3072 | table]
  float* level;            // [n_planes, ny, nz]
  int32_t ny, nz, ix0;
  int64_t n;               // n_planes * ny * nz
};

template <int CT>
__global__ void __launch_bounds__(kThreads) nerf_density_lattice_kernel(const __grid_constant__ nsr_nerf_t P, const __grid_constant__ LatticeArgs a) {
  __shared__ __align__(16) __half Wd[kDensityHalves];
  __shared__ __align__(16) __half Xs[kWarps][32 * NF_LD32];
  __shared__ float raw[kWarps][32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  nsr_stage_matrix(Wd + NF_OFF_DW1, a.dparams, 64, 32, threadIdx.x, kThreads);
  nsr_stage_matrix(Wd + NF_OFF_DW2, a.dparams + 64 * 32, 16, 64, threadIdx.x, kThreads);
  __syncthreads();
  const __half2* table = reinterpret_cast<const __half2*>(a.dparams + NF_DENSITY_PARAMS);
  const float inv2r = 1.f / (2.f * P.radius);
  const int64_t plane = (int64_t)a.ny * a.nz, n_tiles = (a.n + 31) / 32;
  for (int64_t tile = (int64_t)blockIdx.x * kWarps + warp; tile < n_tiles; tile += (int64_t)gridDim.x * kWarps) {
    const int64_t i = tile * 32 + lane;
    const bool ok = i < a.n;
    float x = 0.f, y = 0.f, z = 0.f;
    if (ok) {
      const int64_t r = i % plane;
      x = __ldg(a.ax + a.ix0 + (int)(i / plane));
      y = __ldg(a.ay + (int)(r / a.nz));
      z = __ldg(a.az + (int)(r % a.nz));
      contract_torch<CT>(P.radius, inv2r, x, y, z);
    }
    uint32_t a_o[2][1][4];
    density_rows32(P.grid, table, Wd, Xs[warp], ok, x, y, z, a_o);
    if ((lane & 3) == 0) {   // column 0 (raw density) of rows g and g + 8 of each 16-row tile
#pragma unroll
      for (int m = 0; m < 2; ++m) {
        raw[warp][m * 16 + (lane >> 2)] = nf_half_lo(a_o[m][0][0]);
        raw[warp][m * 16 + (lane >> 2) + 8] = nf_half_lo(a_o[m][0][1]);
      }
    }
    __syncwarp();
    // forward_level: -trunc_exp(raw0 + density_bias) with raw0 the fp16 network output, so the sum is a fp16 tensor (rounded) before
    // trunc_exp takes it to fp32.  (VolumeDensity.forward and nsr_nerf_density add the bias in fp32.)
    if (ok) a.level[i] = -expf(__half2float(__float2half_rn(raw[warp][lane] + P.density_bias)));
    __syncwarp();   // Xs and raw are rewritten by the next tile
  }
}

struct VertexArgs {
  const float* verts;      // [n, 3] world coordinates
  const __half* dparams;   // [density network 3072 | table]
  const __half* cparams;   // colour network [7168]
  float* rgb;              // [n, 3]
  int32_t act_mode;
  int64_t n;
};

template <int CT>
__global__ void __launch_bounds__(kThreads) nerf_vertex_rgb_kernel(const __grid_constant__ nsr_nerf_t P, const __grid_constant__ VertexArgs a) {
  __shared__ __align__(16) __half Wd[kDensityHalves];
  __shared__ __align__(16) __half Wc[W_TOTAL];
  __shared__ __align__(16) __half Xs[kWarps][32 * LD32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  nsr_stage_matrix(Wd + NF_OFF_DW1, a.dparams, 64, 32, threadIdx.x, kThreads);
  nsr_stage_matrix(Wd + NF_OFF_DW2, a.dparams + 64 * 32, 16, 64, threadIdx.x, kThreads);
  stage_weights(Wc, a.cparams);
  __syncthreads();
  const __half2* table = reinterpret_cast<const __half2*>(a.dparams + NF_DENSITY_PARAMS);
  const float inv2r = 1.f / (2.f * P.radius);
  __half* X = Xs[warp];
  // the colour input's direction part: SH4 of the fixed view direction (0, 0, -1), rounded to fp16 as nsr_radiance_fwd rounds it
  uint32_t sh_h[8];
  {
    float s[16];
    nsr_sh4(0.f, 0.f, -1.f, s);
#pragma unroll
    for (int c = 0; c < 8; ++c) sh_h[c] = nsr_pack_h2(s[2 * c], s[2 * c + 1]);
  }
  const int64_t n_groups = (a.n + 31) / 32;
  for (int64_t grp = (int64_t)blockIdx.x * kWarps + warp; grp < n_groups; grp += (int64_t)gridDim.x * kWarps) {
    const int64_t i = grp * 32 + lane;
    const bool ok = i < a.n;
    float x = 0.f, y = 0.f, z = 0.f;
    if (ok) {
      x = __ldg(a.verts + i * 3 + 0);
      y = __ldg(a.verts + i * 3 + 1);
      z = __ldg(a.verts + i * 3 + 2);
      contract_torch<CT>(P.radius, inv2r, x, y, z);
    }
    uint32_t a_o[2][1][4];
    density_rows32(P.grid, table, Wd, X, ok, x, y, z, a_o);
    __syncwarp();   // every lane has read its density input fragments: X becomes the colour input
    // row [feature 16 | SH4(0,0,-1) 16]: the feature is the density network's fp16 output, all 16 columns (the per-op pass widens it to
    // fp32 and nsr_radiance_fwd rounds it back: the same halves)
    nsr_store_afrag<2, 1>(a_o, X, LD32, 0);
    {
      uint4* p = reinterpret_cast<uint4*>(X + lane * LD32 + 16);
      p[0] = make_uint4(sh_h[0], sh_h[1], sh_h[2], sh_h[3]);
      p[1] = make_uint4(sh_h[4], sh_h[5], sh_h[6], sh_h[7]);
    }
    __syncwarp();
#pragma unroll 1
    for (int m = 0; m < 2; ++m) {
      float acc16[1][2][4];
      radiance_rows16<false>(acc16, X, m * 16, Wc, nullptr);
      const int gq = lane >> 2, cq = lane & 3;
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = cq * 2 + e;
          const int64_t r = grp * 32 + m * 16 + gq + hh * 8;
          if (col < 3 && r < a.n) {
            const float v = out_value<false>(acc16[0][0][hh * 2 + e], a.act_mode);
            a.rgb[r * 3 + col] = v < 0.f ? 0.f : (v > 1.f ? 1.f : v);   // .clamp(0, 1) (NaN passes through, as torch's clamp)
          }
        }
    }
    __syncwarp();   // X is rewritten by the next group
  }
}

int check_field(const char* name, const nsr_nerf_t* f, const void* dparams_h) {
  NSR_REQUIRE(f != nullptr && dparams_h != nullptr, "%s: NULL argument", name);
  NSR_REQUIRE(f->grid.n_levels == 16 && f->grid.n_features == 2, "%s: needs a 16-level F=2 hash grid", name);
  NSR_REQUIRE(f->feature_dim == 16 && f->density_hidden == 1, "%s: needs the FullyFused density network 32 -> 64 -> 16", name);
  NSR_REQUIRE(f->contraction == NF_AABB || f->contraction == NF_UNBOUNDED_SPHERE,
              "%s: contraction must be 0 (AABB) or 2 (UN_BOUNDED_SPHERE), got %d", name, f->contraction);
  return 0;
}

int grid_size(int64_t n_tiles) { return (int)min((int64_t)nsr_sm_count() * 8, (n_tiles + kWarps - 1) / kWarps); }

}  // namespace

extern "C" int nsr_nerf_density_lattice(const nsr_nerf_t* f, const float* ax, const float* ay, const float* az, int32_t nx, int32_t ny,
                                        int32_t nz, int32_t ix0, int32_t n_planes, const void* dparams_h, float* level, void* stream) {
  const char* name = "nsr_nerf_density_lattice";
  if (int e = check_field(name, f, dparams_h)) return e;
  NSR_REQUIRE(ax != nullptr && ay != nullptr && az != nullptr && level != nullptr, "%s: NULL argument", name);
  NSR_REQUIRE(nx >= 1 && ny >= 1 && nz >= 1, "%s: empty lattice (%d x %d x %d)", name, nx, ny, nz);
  NSR_REQUIRE(n_planes >= 1 && ix0 >= 0 && ix0 + (int64_t)n_planes <= nx, "%s: planes [%d, %d + %d) outside [0, %d)", name, ix0, ix0,
              n_planes, nx);
  LatticeArgs a;
  a.ax = ax, a.ay = ay, a.az = az, a.dparams = (const __half*)dparams_h, a.level = level;
  a.ny = ny, a.nz = nz, a.ix0 = ix0, a.n = (int64_t)n_planes * ny * nz;
  const int grid = grid_size((a.n + 31) / 32);
  const cudaStream_t st = (cudaStream_t)stream;
  if (f->contraction == NF_AABB)
    nerf_density_lattice_kernel<NF_AABB><<<grid, kThreads, 0, st>>>(*f, a);
  else
    nerf_density_lattice_kernel<NF_UNBOUNDED_SPHERE><<<grid, kThreads, 0, st>>>(*f, a);
  NSR_CHECK_LAUNCH(name);
  return 0;
}

extern "C" int nsr_nerf_vertex_rgb(const nsr_nerf_t* f, const float* verts, const void* dparams_h, const nsr_radiance_t* rp,
                                   const void* cparams_h, float* rgb, int64_t n, void* stream) {
  const char* name = "nsr_nerf_vertex_rgb";
  if (int e = check_field(name, f, dparams_h)) return e;
  NSR_REQUIRE(rp != nullptr && rp->n_feat == 16 && rp->n_extra == 0, "%s: the colour input must be [feature (16) | SH4 (16)]", name);
  NSR_REQUIRE(rp->act_mode >= 0 && rp->act_mode <= 2, "%s: act_mode must be 0, 1 or 2", name);
  NSR_REQUIRE(n >= 0, "%s: n must be >= 0", name);
  NSR_REQUIRE(verts != nullptr && cparams_h != nullptr && rgb != nullptr, "%s: NULL argument", name);
  if (n == 0) return 0;
  VertexArgs a;
  a.verts = verts, a.dparams = (const __half*)dparams_h, a.cparams = (const __half*)cparams_h, a.rgb = rgb, a.act_mode = rp->act_mode, a.n = n;
  const int grid = grid_size((n + 31) / 32);
  const cudaStream_t st = (cudaStream_t)stream;
  if (f->contraction == NF_AABB)
    nerf_vertex_rgb_kernel<NF_AABB><<<grid, kThreads, 0, st>>>(*f, a);
  else
    nerf_vertex_rgb_kernel<NF_UNBOUNDED_SPHERE><<<grid, kThreads, 0, st>>>(*f, a);
  NSR_CHECK_LAUNCH(name);
  return 0;
}
