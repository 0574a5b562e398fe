// Fused NeuS SDF field with FINITE-DIFFERENCE normals and Laplacian: VolumeSDF.forward with grad_type='finite_difference'
// (models/geometry.py:181-199; the Neuralangelo config) -- hash grid with include_xyz and a progressive level mask, the fp32
// VanillaMLP 35 -> 64 (Softplus beta=100) -> n_out, evaluated at the centre and at the six points of the central-difference stencil.
// The math is the hand derivation checked against autograd in oracle/neus_field_fd.py:
//   x_0 = (p + r) / 2r,  x_k = (clamp(p +- eps e_a, -r, r) + r) / 2r  (k = 1..6: +x, -x, +y, -y, +z, -z; fp32, the torch op order)
//   s_k = MLP([2 x_k - 1 | masked hash(x_k)])[0];  grad_a = 0.5 (s_a+ - s_a-) / eps;  lap = sum_a (s_a+ + s_a- - 2 s_0) / eps^2
//   backward: g_out(0) = g_feat + (g_sdf - 6 g_lap / eps^2) e_0;  g_out(a+-)[0] = +-0.5 g_grad_a / eps + g_lap / eps^2
//     then an ordinary first-order MLP + hash backward per evaluation: zb = (W2^T g_out) s;  eb = W1^T zb;  dW1 += zb e^T
//     db1 += zb;  dW2 += g_out h^T;  db2 += g_out;  dtable[c] += w_c eb_l     (levels >= n_active are skipped: their features are 0)
// Layout: a group of 8 lanes owns one sample; lane k evaluates stencil point k (lane 7 idles), so every lane holds one evaluation
// (36 inputs, 64 hidden units) in registers and the stencil is combined with width-8 shuffles.  Everything after the fp16 table
// read is fp32 on the CUDA cores: the 1/eps^2 Laplacian terms cancel across the seven evaluations (1/eps^2 ~ 1e6 at the finest
// level), so neither the SDF values nor the weight-gradient products may go through single fp16 operands.
// Table-gradient merging: per level, every stencil point's corners that are also corners of the centre's cell are summed across
// the group in registers (a width-8 reduce-scatter: lane j ends with centre corner j) and issue ONE RED each; the remaining corners
// of a point one cell away (its far face) are not shared with any other stencil point and are REDed directly.  Points further
// away (eps larger than a cell) share nothing with the centre and RED all 8 corners -- correct for any eps.
// fd_state (device, fp32 [3]) = {eps, eps^2, n_active}: a captured CUDA graph reads the schedule from it on every replay.
#include "neus_field_fd.cuh"

namespace {

using namespace fd;

constexpr int kThreads = 128;
constexpr int G = 8;        // lanes per sample (stencil forms)
constexpr unsigned kFull = 0xffffffffu;

// table index of corner c (runtime) of cell (cx, cy, cz): the arithmetic of nsr_corner_indices for one corner
__device__ __forceinline__ uint32_t corner_index(const LevelInfo& li, uint32_t cx, uint32_t cy, uint32_t cz, int c) {
  const uint32_t bx = c & 1, by = (c >> 1) & 1, bz = (c >> 2) & 1;
  if (li.dense) {
    const uint32_t r = li.res, r2 = li.res * li.res;
    uint32_t i = cx + cy * r + cz * r2 + bx + by * r + bz * r2;
    i = min(i, 2u * li.size - 1u);
    i -= i >= li.size ? li.size : 0u;
    return i + li.offset;
  }
  const uint32_t h = (cx + bx) ^ ((cy + by) * NSR_PRIME_Y) ^ ((cz + bz) * NSR_PRIME_Z);
  return (h & (li.size - 1u)) + li.offset;
}

// ---- forward -------------------------------------------------------------------------------------------------------
// STENCIL = false: one lane per sample, centre only (sdf + feature: the occupancy refresh's SDF-only queries).
template <bool STENCIL>
__global__ void __launch_bounds__(kThreads) neus_fd_fwd_kernel(const __grid_constant__ nsr_grid_t g, const float* __restrict__ points,
                                                             const __half2* __restrict__ table, const float* __restrict__ W1,
                                                             const float* __restrict__ b1, const float* __restrict__ W2,
                                                             const float* __restrict__ b2, float radius, int n_out,
                                                             const float* __restrict__ fd_state, float* __restrict__ sdf,
                                                             float* __restrict__ grad, float* __restrict__ feat, float* __restrict__ lap,
                                                             int64_t n_cap, const int64_t* __restrict__ n_dev) {
  constexpr int GL = STENCIL ? G : 1, kPer = kThreads / GL;
  const int64_t n = n_dev ? min(*n_dev, n_cap) : n_cap;
  __shared__ FdW w;
  stage_weights(w, W1, b1, W2, b2, n_out);
  __syncthreads();
  const float eps = STENCIL ? __ldg(fd_state) : 0.f, eps2 = STENCIL ? __ldg(fd_state + 1) : 1.f;
  const int n_active = (int)__ldg(fd_state + 2);
  const int k = threadIdx.x % GL;
  for (int64_t base = blockIdx.x * (int64_t)kPer; base < n; base += (int64_t)gridDim.x * kPer) {  // uniform per CTA (shuffles below)
    const int64_t i = base + threadIdx.x / GL;
    const bool ok = i < n;
    float px = 0.f, py = 0.f, pz = 0.f;
    if (ok) {
      px = points[i * 3 + 0];
      py = points[i * 3 + 1];
      pz = points[i * 3 + 2];
    }
    float x, y, z, e[NINP];
    stencil_query(px, py, pz, k, eps, radius, x, y, z);
    encode(g, table, x, y, z, n_active, e);
    float out[NOUTP];   // mlp_eval<NOUTP> (neus_field_fd.cuh) written out: the call's inlining renumbers this kernel's registers
#pragma unroll
    for (int o = 0; o < NOUTP; ++o) out[o] = w.b2[o];
#pragma unroll 2
    for (int h = 0; h < NH; ++h) {
      float row[NINP];
#pragma unroll
      for (int v = 0; v < NINP / 4; ++v) *reinterpret_cast<float4*>(&row[4 * v]) = *reinterpret_cast<const float4*>(&w.W1[h][4 * v]);
      float zk = w.b1[h];
#pragma unroll
      for (int j = 0; j < NINP; ++j) zk = fmaf(row[j], e[j], zk);
      float s;
      const float hk = softplus100(zk, s);
      float w2[NOUTP];
#pragma unroll
      for (int v = 0; v < NOUTP / 4; ++v) *reinterpret_cast<float4*>(&w2[4 * v]) = *reinterpret_cast<const float4*>(&w.W2T[h][4 * v]);
#pragma unroll
      for (int o = 0; o < NOUTP; ++o) out[o] = fmaf(w2[o], hk, out[o]);
    }
    float sn[7];
    if (STENCIL) {
#pragma unroll
      for (int j = 1; j < 7; ++j) sn[j] = __shfl_sync(kFull, out[0], j, G);
    }
    if (ok && k == 0) {
      sdf[i] = out[0];
#pragma unroll
      for (int o = 0; o < NOUTP; ++o)
        if (o < n_out) feat[i * n_out + o] = out[o];
      if (STENCIL) {
        if (grad != nullptr) {
          grad[i * 3 + 0] = __fdiv_rn(0.5f * (sn[1] - sn[2]), eps);
          grad[i * 3 + 1] = __fdiv_rn(0.5f * (sn[3] - sn[4]), eps);
          grad[i * 3 + 2] = __fdiv_rn(0.5f * (sn[5] - sn[6]), eps);
        }
        if (lap != nullptr) {
          const float s2 = 2.f * out[0];
          const float t = (((sn[1] + sn[2]) - s2) + ((sn[3] + sn[4]) - s2)) + ((sn[5] + sn[6]) - s2);
          lap[i] = __fdiv_rn(t, eps2);
        }
      }
    }
  }
}

// ---- backward ------------------------------------------------------------------------------------------------------
// Per tile of kThreads evaluations (16 samples x 8 stencil lanes, or 128 samples centre-only): every lane recomputes its
// evaluation, runs the first-order MLP backward in registers, scatters the table gradient, and stages its rows of the
// weight-gradient products in fp32 shared-memory tiles; the whole CTA then accumulates  [dW1 | db1] += ZB^T [E | 1]  and
// dW2 += GO^T H  over the tile's rows in registers (fp32 FMAs), flushed with one atomicAdd per weight per CTA at the end.
constexpr int LDT = kThreads + 4;     // 132 floats: float4 row reads of 8 consecutive lanes' rows hit disjoint banks
constexpr int KE = 40;                // E rows: 35 inputs, the ones column (-> db1), zero padding
constexpr int T_ZB = 0, T_E = T_ZB + NH * LDT, T_H = T_E + KE * LDT, T_GO = T_H + NH * LDT, T_TOTAL = T_GO + NOUTP * LDT;
constexpr size_t kBwdSmem = sizeof(FdW) + (size_t)T_TOTAL * sizeof(float);   // 110.8 KB => two CTAs per SM

template <bool STENCIL>
__global__ void __launch_bounds__(kThreads, 2) neus_fd_bwd_kernel(const __grid_constant__ nsr_grid_t g, const float* __restrict__ points,
                                                                const __half2* __restrict__ table, const float* __restrict__ W1,
                                                                const float* __restrict__ b1, const float* __restrict__ W2,
                                                                const float* __restrict__ b2, float radius, int n_out,
                                                                const float* __restrict__ fd_state, const float* __restrict__ g_out,
                                                                const float* __restrict__ g_sdf, const float* __restrict__ g_grad,
                                                                const float* __restrict__ g_lap, float* __restrict__ grad_table,
                                                                float* __restrict__ dW1, float* __restrict__ db1, float* __restrict__ dW2,
                                                                float* __restrict__ db2, int64_t n_cap, const int64_t* __restrict__ n_dev) {
  constexpr int GL = STENCIL ? G : 1, kPer = kThreads / GL;
  const int64_t n = n_dev ? min(*n_dev, n_cap) : n_cap;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  FdW& w = *reinterpret_cast<FdW*>(smem_raw);
  float* T = reinterpret_cast<float*>(smem_raw + sizeof(FdW));
  const int tid = threadIdx.x, k = tid % GL;
  stage_weights(w, W1, b1, W2, b2, n_out);
  const float eps = STENCIL ? __ldg(fd_state) : 0.f, eps2 = STENCIL ? __ldg(fd_state + 1) : 1.f;
  const int n_active = (int)__ldg(fd_state + 2);
  __syncthreads();

  // weight-gradient accumulators: [dW1 | db1] rows m = mb + 16 i, columns j = jb + 8 c;  dW2 row o, columns kk = jb + 8 i
  const int mb = tid & 15, jb = tid >> 4;
  float acc1[4][5], acc2[8], gsum[NOUTP];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int c = 0; c < 5; ++c) acc1[i][c] = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) acc2[i] = 0.f;
#pragma unroll
  for (int o = 0; o < NOUTP; ++o) gsum[o] = 0.f;

  const int64_t n_tiles = (n + kPer - 1) / kPer;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t i = tile * kPer + tid / GL;
    const bool ok = i < n;
    const bool active = ok && k < 7;
    __syncthreads();  // the previous tile's products are done with the tiles
    float px = 0.f, py = 0.f, pz = 0.f;
    float go[NOUTP];
#pragma unroll
    for (int o = 0; o < NOUTP; ++o) go[o] = 0.f;
    if (ok) {
      px = points[i * 3 + 0];
      py = points[i * 3 + 1];
      pz = points[i * 3 + 2];
    }
    if (active) {
      const float gl = (STENCIL && g_lap != nullptr) ? __fdiv_rn(g_lap[i], eps2) : 0.f;
      if (k == 0) {
        if (g_out != nullptr) {
#pragma unroll
          for (int o = 0; o < NOUTP; ++o)
            if (o < n_out) go[o] = g_out[i * n_out + o];
        }
        if (g_sdf != nullptr) go[0] += g_sdf[i];
        go[0] -= 6.f * gl;
      } else {
        const int a = (k - 1) >> 1;
        const float gg = g_grad != nullptr ? __fdiv_rn(0.5f * g_grad[i * 3 + a], eps) : 0.f;
        go[0] = (((k - 1) & 1) ? -gg : gg) + gl;
      }
    }
    float x, y, z, e[NINP], eb[NINP];
    stencil_query(px, py, pz, k, eps, radius, x, y, z);
    encode(g, table, x, y, z, n_active, e);
#pragma unroll
    for (int j = 0; j < NINP; ++j) eb[j] = 0.f;
#pragma unroll 2
    for (int h = 0; h < NH; ++h) {
      float row[NINP];
#pragma unroll
      for (int v = 0; v < NINP / 4; ++v) *reinterpret_cast<float4*>(&row[4 * v]) = *reinterpret_cast<const float4*>(&w.W1[h][4 * v]);
      float zk = w.b1[h];
#pragma unroll
      for (int j = 0; j < NINP; ++j) zk = fmaf(row[j], e[j], zk);
      float s;
      const float hk = softplus100(zk, s);
      float w2[NOUTP];
#pragma unroll
      for (int v = 0; v < NOUTP / 4; ++v) *reinterpret_cast<float4*>(&w2[4 * v]) = *reinterpret_cast<const float4*>(&w.W2T[h][4 * v]);
      float t = 0.f;
#pragma unroll
      for (int o = 0; o < NOUTP; ++o) t = fmaf(w2[o], go[o], t);
      const float zb = t * s;
#pragma unroll
      for (int j = 3; j < NINP; ++j) eb[j] = fmaf(row[j], zb, eb[j]);   // the points get no gradient: inputs 0..2 are not needed
      T[T_ZB + h * LDT + tid] = active ? zb : 0.f;
      T[T_H + h * LDT + tid] = active ? hk : 0.f;
    }
#pragma unroll
    for (int j = 0; j < KE; ++j) T[T_E + j * LDT + tid] = !active ? 0.f : (j < NIN ? e[j < NINP ? j : 0] : (j == NIN ? 1.f : 0.f));
#pragma unroll
    for (int o = 0; o < NOUTP; ++o) {
      T[T_GO + o * LDT + tid] = go[o];
      gsum[o] += go[o];
    }

    // ---- table gradient
#pragma unroll
    for (int l = 0; l < 16; ++l) {
      if (l >= n_active) break;
      const float eb0 = eb[3 + 2 * l], eb1 = eb[4 + 2 * l];
      const LevelInfo li = nsr_level(g, l);
      uint32_t cx, cy, cz, idx[8];
      float fx, fy, fz;
      nsr_pos_fract(x, li.scale, cx, fx);
      nsr_pos_fract(y, li.scale, cy, fy);
      nsr_pos_fract(z, li.scale, cz, fz);
      nsr_corner_indices(li, cx, cy, cz, idx);
      if (!STENCIL) {
        if (active) {
#pragma unroll
          for (int c = 0; c < 8; ++c) {
            const float wc = nsr_corner_weight(c, fx, fy, fz), v0 = wc * eb0, v1 = wc * eb1;
            if (v0 != 0.f || v1 != 0.f) nsr_red_add_f32x2(grad_table + 2 * (size_t)idx[c], v0, v1);
          }
        }
        continue;
      }
      // this point's cell relative to the centre's (lane 0 of the group)
      const uint32_t ccx = __shfl_sync(kFull, cx, 0, G), ccy = __shfl_sync(kFull, cy, 0, G), ccz = __shfl_sync(kFull, cz, 0, G);
      const int dx = (int)(cx - ccx), dy = (int)(cy - ccy), dz = (int)(cz - ccz);
      // own corner c lands on centre corner c + d when every coordinate stays in {0, 1}: summed across the group below;
      // the others are not shared with any other stencil point (far faces of one-cell moves are disjoint) => direct RED
      float cen[16];
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const int bx = (c & 1) - dx, by = ((c >> 1) & 1) - dy, bz = ((c >> 2) & 1) - dz;
        const bool shared = active && (unsigned)bx <= 1u && (unsigned)by <= 1u && (unsigned)bz <= 1u;
        const float wc = (bx ? fx : 1.f - fx) * (by ? fy : 1.f - fy) * (bz ? fz : 1.f - fz);
        cen[2 * c] = shared ? wc * eb0 : 0.f;
        cen[2 * c + 1] = shared ? wc * eb1 : 0.f;
      }
      if (active) {
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const int bx = (c & 1) + dx, by = ((c >> 1) & 1) + dy, bz = ((c >> 2) & 1) + dz;
          if ((unsigned)bx <= 1u && (unsigned)by <= 1u && (unsigned)bz <= 1u) continue;
          const float wc = nsr_corner_weight(c, fx, fy, fz), v0 = wc * eb0, v1 = wc * eb1;
          if (v0 != 0.f || v1 != 0.f) nsr_red_add_f32x2(grad_table + 2 * (size_t)idx[c], v0, v1);
        }
      }
      // reduce-scatter of the 8 centre corners over the group: lane j ends with corner j
      float r8[8], r4[4], r2[2];
      const bool s2 = (k >> 2) & 1, s1 = (k >> 1) & 1, s0 = k & 1;
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float send = s2 ? cen[q] : cen[q + 8], keep = s2 ? cen[q + 8] : cen[q];
        r8[q] = keep + __shfl_xor_sync(kFull, send, 4);
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float send = s1 ? r8[q] : r8[q + 4], keep = s1 ? r8[q + 4] : r8[q];
        r4[q] = keep + __shfl_xor_sync(kFull, send, 2);
      }
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const float send = s0 ? r4[q] : r4[q + 2], keep = s0 ? r4[q + 2] : r4[q];
        r2[q] = keep + __shfl_xor_sync(kFull, send, 1);
      }
      if (ok && (r2[0] != 0.f || r2[1] != 0.f))
        nsr_red_add_f32x2(grad_table + 2 * (size_t)corner_index(li, ccx, ccy, ccz, k), r2[0], r2[1]);
    }
    __syncthreads();
    // ---- weight-gradient products over the tile's kThreads rows (fp32)
#pragma unroll 1
    for (int r = 0; r < kThreads; r += 4) {
      float4 zv[4], ev[5];
#pragma unroll
      for (int q = 0; q < 4; ++q) zv[q] = *reinterpret_cast<const float4*>(T + T_ZB + (mb + 16 * q) * LDT + r);
#pragma unroll
      for (int c = 0; c < 5; ++c) ev[c] = *reinterpret_cast<const float4*>(T + T_E + (jb + 8 * c) * LDT + r);
#pragma unroll
      for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int c = 0; c < 5; ++c) {
          float a = acc1[q][c];
          a = fmaf(zv[q].x, ev[c].x, a);
          a = fmaf(zv[q].y, ev[c].y, a);
          a = fmaf(zv[q].z, ev[c].z, a);
          a = fmaf(zv[q].w, ev[c].w, a);
          acc1[q][c] = a;
        }
      const float4 gv = *reinterpret_cast<const float4*>(T + T_GO + mb * LDT + r);
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float4 hv = *reinterpret_cast<const float4*>(T + T_H + (jb + 8 * q) * LDT + r);
        float a = acc2[q];
        a = fmaf(gv.x, hv.x, a);
        a = fmaf(gv.y, hv.y, a);
        a = fmaf(gv.z, hv.z, a);
        a = fmaf(gv.w, hv.w, a);
        acc2[q] = a;
      }
    }
  }
  // ---- flush
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int c = 0; c < 5; ++c) {
      const int m = mb + 16 * q, j = jb + 8 * c;
      const float v = acc1[q][c];
      if (v == 0.f) continue;
      if (j < NIN)
        atomicAdd(dW1 + m * NIN + j, v);
      else if (j == NIN)
        atomicAdd(db1 + m, v);
    }
  if (mb < n_out) {
#pragma unroll
    for (int q = 0; q < 8; ++q)
      if (acc2[q] != 0.f) atomicAdd(dW2 + mb * NH + jb + 8 * q, acc2[q]);
  }
#pragma unroll
  for (int o = 0; o < NOUTP; ++o) {
    float v = gsum[o];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(kFull, v, d);
    if ((tid & 31) == 0 && o < n_out && v != 0.f) atomicAdd(db2 + o, v);
  }
}

int check(const nsr_grid_t* g, int n_out, const float* fd_state, const char* name) {
  NSR_REQUIRE(g != nullptr && g->n_levels == 16 && g->n_features == 2, "%s: needs a 16-level F=2 hash grid", name);
  NSR_REQUIRE(n_out >= 1 && n_out <= 16, "%s: n_out must be in [1,16]", name);
  NSR_REQUIRE(fd_state != nullptr, "%s: fd_state (device {eps, eps^2, n_active}) is NULL", name);
  return 0;
}

}  // namespace

extern "C" int nsr_neus_field_fd_fwd(const nsr_grid_t* g, const float* points, const void* table_h, const float* W1, const float* b1,
                                     const float* W2, const float* b2, float radius, int32_t n_out, const float* fd_state, float* sdf,
                                     float* grad, float* feature, float* laplace, int64_t n, const int64_t* n_dev, void* stream) {
  if (int e = check(g, n_out, fd_state, "nsr_neus_field_fd_fwd")) return e;
  if (n == 0) return 0;
  const cudaStream_t st = (cudaStream_t)stream;
  if (grad != nullptr || laplace != nullptr) {
    const int grid = (int)min((int64_t)nsr_sm_count() * 8, (n + kThreads / G - 1) / (kThreads / G));
    neus_fd_fwd_kernel<true><<<grid, kThreads, 0, st>>>(*g, points, (const __half2*)table_h, W1, b1, W2, b2, radius, n_out, fd_state, sdf,
                                                       grad, feature, laplace, n, n_dev);
  } else {
    const int grid = (int)min((int64_t)nsr_sm_count() * 8, (n + kThreads - 1) / kThreads);
    neus_fd_fwd_kernel<false><<<grid, kThreads, 0, st>>>(*g, points, (const __half2*)table_h, W1, b1, W2, b2, radius, n_out, fd_state, sdf,
                                                        nullptr, feature, nullptr, n, n_dev);
  }
  NSR_CHECK_LAUNCH("nsr_neus_field_fd_fwd");
  return 0;
}

extern "C" int nsr_neus_field_fd_bwd(const nsr_grid_t* g, const float* points, const void* table_h, const float* W1, const float* b1,
                                     const float* W2, const float* b2, float radius, int32_t n_out, const float* fd_state, const float* g_out,
                                     const float* g_sdf, const float* g_grad, const float* g_lap, float* grad_table, float* dW1, float* db1,
                                     float* dW2, float* db2, int64_t n, const int64_t* n_dev, void* stream) {
  if (int e = check(g, n_out, fd_state, "nsr_neus_field_fd_bwd")) return e;
  if (n == 0) return 0;
  const bool stencil = g_grad != nullptr || g_lap != nullptr;
  static thread_local bool attr_set = false;
  if (!attr_set) {
    for (const void* fn : {(const void*)neus_fd_bwd_kernel<true>, (const void*)neus_fd_bwd_kernel<false>}) {
      cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBwdSmem);
      if (e != cudaSuccess) {
        nsr_set_error("nsr_neus_field_fd_bwd: cannot reserve %zu B shared memory: %s", kBwdSmem, cudaGetErrorString(e));
        return 2;
      }
    }
    attr_set = true;
  }
  const int per = stencil ? kThreads / G : kThreads;
  const int grid = (int)min((int64_t)nsr_sm_count() * 2, (n + per - 1) / per);
  const cudaStream_t st = (cudaStream_t)stream;
  if (stencil)
    neus_fd_bwd_kernel<true><<<grid, kThreads, kBwdSmem, st>>>(*g, points, (const __half2*)table_h, W1, b1, W2, b2, radius, n_out, fd_state,
                                                               g_out, g_sdf, g_grad, g_lap, grad_table, dW1, db1, dW2, db2, n, n_dev);
  else
    neus_fd_bwd_kernel<false><<<grid, kThreads, kBwdSmem, st>>>(*g, points, (const __half2*)table_h, W1, b1, W2, b2, radius, n_out, fd_state,
                                                                g_out, g_sdf, nullptr, nullptr, grad_table, dW1, db1, dW2, db2, n, n_dev);
  NSR_CHECK_LAUNCH("nsr_neus_field_fd_bwd");
  return 0;
}
