// Fused NeRF backward through both networks and the hash grid (autograd of VolumeRadiance + VolumeDensity +
// HashGrid, models/texture.py:23-30, models/geometry.py:122-130), one launch.
//
// Per 64-sample CTA tile (4 warps x 16 rows, two CTAs per SM): reload the 64 B/sample encoded features saved by the forward,
// recompute every activation on tensor cores (cheaper than storing 416 B/sample of hidden state), run the dgrad
// chain in registers, scatter dL/d(table) straight from the mma accumulator layout (each thread owns 2 samples x 4
// levels) with 8-byte vector REDs into the fp32 gradient table, then split the five weight-gradient GEMMs
// (dW = dPre^T * Act, K = 64 samples) over the 4 warps with register accumulators that persist for the whole
// kernel; one atomicAdd per weight per CTA at the end (tcnn: split-K CUTLASS GEMMs over K = batch + reduction).
// The split backward's network half (nerf_bwd_net_kernel, below) runs the same chain as register-A wgmma on three chain warpgroups and
// hands the weight-gradient GEMMs to a third warpgroup.
#include "nerf_fused.cuh"
#include "wgmma.cuh"

namespace {

constexpr int kWarps = 4;
constexpr int kThreads = kWarps * 32;
constexpr int kRows = kWarps * 16;  // 64-row CTA tile: ~96 KB of smem => 2 CTAs / SM whose phases (MMA / scatter / wgrad) overlap
constexpr int kCtasPerSm = 2;

// smem tile offsets (halves) after the weights
constexpr int T_X0 = 0;                         // [64][40]  encoded features
constexpr int T_H1 = T_X0 + kRows * NF_LD32;    // [64][72]  density hidden (post ReLU)
constexpr int T_CI = T_H1 + kRows * NSR_LD64;   // [64][40]  colour input: out16 | SH16
constexpr int T_G1 = T_CI + kRows * NF_LD32;    // [64][72]
constexpr int T_G2 = T_G1 + kRows * NSR_LD64;   // [64][72]
constexpr int T_DC3 = T_G2 + kRows * NSR_LD64;  // [64][24]  d(rgb pre-activation)
constexpr int T_DG2 = T_DC3 + kRows * 24;       // [64][72]
constexpr int T_DG1 = T_DG2 + kRows * NSR_LD64; // [64][72]
constexpr int T_DO = T_DG1 + kRows * NSR_LD64;  // [64][24]  d(out16)
constexpr int T_DH1 = T_DO + kRows * 24;        // [64][72]
constexpr int T_X0B = T_DH1 + kRows * NSR_LD64; // [64][40]  second encoded-feature buffer (packed mode: cp.async double buffering)
constexpr int T_TOTAL = T_X0B + kRows * NF_LD32;
// packed mode: per-row inputs of two tiles in flight (floats): xyz+dir [64][6], d_sraw [64], d_rgb [64][3]
constexpr int S_XYZ = 0, S_DS = S_XYZ + kRows * 6, S_DRGB = S_DS + kRows, S_ROWF = S_DRGB + kRows * 3;  // 640 floats per buffer
constexpr size_t kSmemBytes = (size_t)(NF_W_TOTAL + T_TOTAL) * sizeof(__half) + 2 * S_ROWF * sizeof(float);
constexpr size_t kSmemBytesVanilla = kSmemBytes + NF_B_TOTAL * sizeof(float);  // + the fp32 biases

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

constexpr int kSlots = 40 / kWarps;  // 40 wgrad pair-tiles split over the warps

struct WgradTile {
  int dy_off, ldy, x_off, ldx, m0, n0;  // smem tiles
  int net, base, in_dim;                // destination in the flat parameter gradient (net 0 density, 1 colour)
};

__device__ __forceinline__ WgradTile wgrad_tile(int t) {
  WgradTile w;
  if (t < 8) {          // density W1 [64][32]
    w = {T_DH1, NSR_LD64, T_X0, NF_LD32, (t / 2) * 16, (t % 2) * 16, 0, 0, 32};
  } else if (t < 12) {  // density W2 [16][64]
    w = {T_DO, 24, T_H1, NSR_LD64, 0, (t - 8) * 16, 0, 64 * 32, 64};
  } else if (t < 20) {  // colour W1 [64][32]
    const int u = t - 12;
    w = {T_DG1, NSR_LD64, T_CI, NF_LD32, (u / 2) * 16, (u % 2) * 16, 1, 0, 32};
  } else if (t < 36) {  // colour W2 [64][64]
    const int u = t - 20;
    w = {T_DG2, NSR_LD64, T_G1, NSR_LD64, (u / 4) * 16, (u % 4) * 16, 1, 64 * 32, 64};
  } else {              // colour W3 [16][64]
    w = {T_DC3, 24, T_G2, NSR_LD64, 0, (t - 36) * 16, 1, 64 * 32 + 64 * 64, 64};
  }
  return w;
}

// mask a dgrad accumulator with the ReLU of the post-activation fragments and pack to fp16 A fragments
__device__ __forceinline__ void relu_mask_pack(const float (&acc)[1][8][4], const uint32_t (&post)[1][4][4], uint32_t (&out)[1][4][4]) {
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const __half2 hv = *reinterpret_cast<const __half2*>(&post[0][k][j]);
      const int nt = 2 * k + (j >> 1), i0 = (j & 1) * 2;
      const float d0 = __low2float(hv) > 0.f ? acc[0][nt][i0] : 0.f;
      const float d1 = __high2float(hv) > 0.f ? acc[0][nt][i0 + 1] : 0.f;
      out[0][k][j] = nsr_pack_h2(d0, d1);
    }
}

// PACKED: enc_save, d_sraw, d_rgb are in packed row order and xyzdir [n,6] holds the unit-cube position and the view direction of
// every row (written by nsr_pack_kept; buffers padded by one tile).  All global inputs of tile t+1 are then fetched with cp.async
// into the second smem buffer while tile t computes: no load of the kernel sits in front of the math any more (ncu before:
// 37 % of the stall samples were long-scoreboard waits on the row_pos -> enc / ray_indices -> rays chains and on the tile's loads).
// The split backward (d(encoding) to memory, REDs in a separate kernel) uses nerf_bwd_net_kernel below instead.
// CT: the field's contraction (NF_AABB / NF_UNBOUNDED_SPHERE) of the positions recomputed from the rays (!PACKED; xyzdir is AABB-only)
// NET: the network variant.  VanillaMLP (!PACKED, contracted): the recompute starts each layer from its fp32 bias and applies the colour
// sigmoid to the un-rounded fp32 output; the table gradient goes to grad_table_sep (the table is not behind the density network there),
// and the bias gradients are the column sums of the five pre-activation-gradient tiles (rows past the live count hold zeros in all of
// them), one atomicAdd per bias per CTA into grad_dbias [80] / grad_cbias [144].
template <bool PACKED, int CT, int NET>
__global__ void __launch_bounds__(kThreads, kCtasPerSm) nerf_bwd_kernel(const __grid_constant__ nsr_nerf_t P, const float* __restrict__ rays,
                                                               const int32_t* __restrict__ ray_indices, const float* __restrict__ t_starts,
                                                               const float* __restrict__ t_ends, const __half* __restrict__ enc_save,
                                                               const __half* __restrict__ dparams, const __half* __restrict__ cparams,
                                                               const float* __restrict__ d_sraw, const float* __restrict__ d_rgb,
                                                               float* __restrict__ grad_dparams, float* __restrict__ grad_cparams,
                                                               float loss_scale, const float* __restrict__ amax_ptr, int64_t n_cap, const int64_t* __restrict__ n_dev,
                                                               const int64_t* __restrict__ row_pos, const float* __restrict__ xyzdir,
                                                               const float* __restrict__ dbias, const float* __restrict__ cbias,
                                                               float* __restrict__ grad_table_sep, float* __restrict__ grad_dbias,
                                                               float* __restrict__ grad_cbias) {
  const int64_t n = n_dev ? min(*n_dev, n_cap) : n_cap;
  extern __shared__ __align__(16) __half smem[];
  __half* T = smem + NF_W_TOTAL;
  float* rowf = reinterpret_cast<float*>(smem + NF_W_TOTAL + T_TOTAL);  // [2][S_ROWF]
  float* bias_sm = rowf + 2 * S_ROWF;                                    // VanillaMLP only
  float bsum[2] = {0.f, 0.f};   // VanillaMLP: this thread's bias columns (threadIdx.x, threadIdx.x + 128) summed over all tiles
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, c = lane & 3;
  const int r0 = warp * 16;
  if (loss_scale <= 0.f) {  // automatic: bring the largest incoming gradient to ~2^8
    const float amax = fmaxf(__ldg(amax_ptr), 1e-30f);
    loss_scale = exp2f(fminf(fmaxf(floorf(log2f(256.f / amax)), -24.f), 60.f));
  }
  const float inv_scale = 1.f / loss_scale;
  nf_stage_weights(smem, dparams, cparams, true);
  if (NET == NF_NET_VANILLA) nf_stage_bias(bias_sm, dbias, cbias, true);
  float* grad_table = NET == NF_NET_VANILLA ? grad_table_sep : grad_dparams + NF_DENSITY_PARAMS;

  float wacc[kSlots][2][4];
#pragma unroll
  for (int s = 0; s < kSlots; ++s)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int i = 0; i < 4; ++i) wacc[s][j][i] = 0.f;

  const int64_t n_tiles = (n + kRows - 1) / kRows;
  // packed mode: asynchronous fetch of one tile's inputs into buffer `buf` (all threads; 16-byte chunks, L1 bypassed)
  auto fetch_tile = [&](int64_t tile, int buf) {
    const int64_t row0 = tile * kRows;
    __half* xb = T + (buf ? T_X0B : T_X0);
    float* rf = rowf + buf * S_ROWF;
    for (int v = threadIdx.x; v < kRows * 4; v += kThreads)  // 64 rows x 4 chunks of the 64-byte encodings
      cp_async16(xb + (v >> 2) * NF_LD32 + (v & 3) * 8, enc_save + (row0 + (v >> 2)) * 32 + (v & 3) * 8);
    for (int v = threadIdx.x; v < kRows * 6 / 4; v += kThreads) cp_async16(rf + S_XYZ + v * 4, xyzdir + row0 * 6 + v * 4);
    if (threadIdx.x < kRows / 4) cp_async16(rf + S_DS + threadIdx.x * 4, d_sraw + row0 + threadIdx.x * 4);
    if (threadIdx.x >= 64 && threadIdx.x < 64 + kRows * 3 / 4)
      cp_async16(rf + S_DRGB + (threadIdx.x - 64) * 4, d_rgb + row0 * 3 + (threadIdx.x - 64) * 4);
    cp_async_commit();
  };
  int buf = 0;
  if (PACKED && (int64_t)blockIdx.x < n_tiles) fetch_tile(blockIdx.x, 0);
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, buf ^= 1) {
    const int64_t row0 = tile * kRows;
    if (PACKED) cp_async_wait_all();  // this tile's inputs have landed (issued one tile ago)
    __syncthreads();  // previous tile's wgrad is done with the smem tiles (first iteration: weights are staged)
    const __half* X0 = T + ((PACKED && buf) ? T_X0B : T_X0);
    const int x0_off = (PACKED && buf) ? T_X0B : T_X0;
    const float* rf = rowf + buf * S_ROWF;
    if (PACKED) {
      if (tile + gridDim.x < n_tiles) fetch_tile(tile + gridDim.x, buf ^ 1);
      if (row0 + kRows > n) {  // last, partial tile: rows >= n hold stale data; zero them so that 0 * garbage never reaches the wgrad sums
        for (int v = threadIdx.x; v < kRows * 4; v += kThreads)
          if (row0 + (v >> 2) >= n) *reinterpret_cast<uint4*>(T + x0_off + (v >> 2) * NF_LD32 + (v & 3) * 8) = make_uint4(0, 0, 0, 0);
        float* rw = rowf + buf * S_ROWF;
        for (int v = threadIdx.x; v < S_ROWF; v += kThreads) {
          const int r = v < S_DS ? v / 6 : (v < S_DRGB ? v - S_DS : (v - S_DRGB) / 3);
          if (row0 + r >= n) rw[v] = 0.f;
        }
        __syncthreads();
      }
    }
    // rows this thread owns in the accumulator layout (g, g+8) and where their per-sample gradients live
    const int64_t ia = row0 + r0 + g, ib = ia + 8;
    const int64_t pa = (!PACKED && row_pos && ia < n) ? row_pos[ia] : ia, pb = (!PACKED && row_pos && ib < n) ? row_pos[ib] : ib;
    // ---- stage this warp's 16 rows: encoded features and SH of the view direction
    if (!PACKED) {
      for (int v = lane; v < 64; v += 32) {
        const int r = v >> 2, q = v & 3;
        const int64_t i = row0 + r0 + r;
        uint4 val = make_uint4(0, 0, 0, 0);
        if (i < n) val = __ldg(reinterpret_cast<const uint4*>(enc_save + (row_pos ? row_pos[i] : i) * 32) + q);
        *reinterpret_cast<uint4*>(T + T_X0 + (r0 + r) * NF_LD32 + q * 8) = val;
      }
    }
    if (lane < 16) {
      const int64_t i = row0 + r0 + lane;
      uint4 s0 = make_uint4(0, 0, 0, 0), s1 = s0;
      if (i < n) {
        float s[16];
        if (PACKED) {
          const float* rr = rf + S_XYZ + (r0 + lane) * 6;
          nsr_sh4(rr[3], rr[4], rr[5], s);
        } else {
          const float* rr = rays + (size_t)ray_indices[i] * 6;
          nsr_sh4(__ldg(rr + 3), __ldg(rr + 4), __ldg(rr + 5), s);
        }
        s0 = make_uint4(nsr_pack_h2(s[0], s[1]), nsr_pack_h2(s[2], s[3]), nsr_pack_h2(s[4], s[5]), nsr_pack_h2(s[6], s[7]));
        s1 = make_uint4(nsr_pack_h2(s[8], s[9]), nsr_pack_h2(s[10], s[11]), nsr_pack_h2(s[12], s[13]), nsr_pack_h2(s[14], s[15]));
      }
      uint4* sp = reinterpret_cast<uint4*>(T + T_CI + (r0 + lane) * NF_LD32 + 16);
      sp[0] = s0;
      sp[1] = s1;
    }
    __syncwarp();

    // ---- forward recompute
    uint32_t a_h1[1][4][4], a_o[1][1][4], a_g1[1][4][4], a_g2[1][4][4];
    float acc[1][8][4], acc16[1][2][4];
    {
      uint32_t a_in[1][2][4];
      nsr_load_afrag<1, 2>(a_in, X0, NF_LD32, r0);
      nf_init_acc<NET>(acc, bias_sm + NF_B_D1);
      nsr_gemm_w<1, 2, 8>(acc, a_in, smem + NF_OFF_DW1, NF_LD32);
      nsr_acc_to_afrag<1, 8>(acc, a_h1, NSR_ACT_RELU);
      nsr_store_afrag<1, 4>(a_h1, T + T_H1, NSR_LD64, r0);
      nf_init_acc<NET>(acc16, bias_sm + NF_B_D2);
      nsr_gemm_w<1, 4, 2>(acc16, a_h1, smem + NF_OFF_DW2, NSR_LD64);
      nsr_acc_to_afrag<1, 2>(acc16, a_o, NSR_ACT_NONE);
      nsr_store_afrag<1, 1>(a_o, T + T_CI, NF_LD32, r0, 0);
    }
    {
      uint32_t a_c[1][2][4], a_sh[1][1][4];
      nsr_load_afrag<1, 1>(a_sh, T + T_CI + 16, NF_LD32, r0);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        a_c[0][0][j] = a_o[0][0][j];
        a_c[0][1][j] = a_sh[0][0][j];
      }
      nf_init_acc<NET>(acc, bias_sm + NF_B_C1);
      nsr_gemm_w<1, 2, 8>(acc, a_c, smem + NF_OFF_CW1, NF_LD32);
      nsr_acc_to_afrag<1, 8>(acc, a_g1, NSR_ACT_RELU);
      nsr_store_afrag<1, 4>(a_g1, T + T_G1, NSR_LD64, r0);
      nf_init_acc<NET>(acc, bias_sm + NF_B_C2);
      nsr_gemm_w<1, 4, 8>(acc, a_g1, smem + NF_OFF_CW2, NSR_LD64);
      nsr_acc_to_afrag<1, 8>(acc, a_g2, NSR_ACT_RELU);
      nsr_store_afrag<1, 4>(a_g2, T + T_G2, NSR_LD64, r0);
      nf_init_acc<NET>(acc16, bias_sm + NF_B_C3);
      nsr_gemm_w<1, 4, 2>(acc16, a_g2, smem + NF_OFF_CW3, NSR_LD64);
    }
    // ---- d(rgb pre-activation) = d_rgb * s (1 - s), s = sigmoid(fp16(raw)) (VanillaMLP: sigmoid(raw)); columns 0..2 only
    uint32_t a_dc3[1][1][4];
    {
      float dp[4] = {0.f, 0.f, 0.f, 0.f};  // (row g: col c*2, c*2+1), (row g+8: col c*2, c*2+1)
      if (c < 2) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int64_t i = hh ? ib : ia, pi = hh ? pb : pa;
          if (i < n) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int col = c * 2 + e;
              if (col < 3) {
                const float raw = NET == NF_NET_VANILLA ? acc16[0][0][hh * 2 + e] : __half2float(__float2half_rn(acc16[0][0][hh * 2 + e]));
                const float s = 1.f / (1.f + expf(-raw));
                const float dr = PACKED ? rf[S_DRGB + (r0 + g + hh * 8) * 3 + col] : d_rgb[pi * 3 + col];
                dp[hh * 2 + e] = dr * s * (1.f - s) * loss_scale;
              }
            }
          }
        }
      }
      a_dc3[0][0][0] = nsr_pack_h2(dp[0], dp[1]);
      a_dc3[0][0][1] = nsr_pack_h2(dp[2], dp[3]);
      a_dc3[0][0][2] = 0u;
      a_dc3[0][0][3] = 0u;
      nsr_store_afrag<1, 1>(a_dc3, T + T_DC3, 24, r0);
    }
    // ---- dgrad chain
    uint32_t a_d[1][4][4];
    nsr_zero_acc(acc);
    nsr_gemm_wt<1, 1, 8>(acc, a_dc3, smem + NF_OFF_CW3, NSR_LD64);
    relu_mask_pack(acc, a_g2, a_d);
    nsr_store_afrag<1, 4>(a_d, T + T_DG2, NSR_LD64, r0);
    nsr_zero_acc(acc);
    nsr_gemm_wt<1, 4, 8>(acc, a_d, smem + NF_OFF_CW2, NSR_LD64);
    relu_mask_pack(acc, a_g1, a_d);
    nsr_store_afrag<1, 4>(a_d, T + T_DG1, NSR_LD64, r0);
    nsr_zero_acc(acc16);
    nsr_gemm_wt<1, 4, 2>(acc16, a_d, smem + NF_OFF_CW1, NF_LD32);  // first 16 input columns = the geometry features
    if (c == 0) {  // density path: d(out0) += d sigma / d raw (trunc_exp backward folded in by nsr_nerf_ray_bwd)
      if (ia < n) acc16[0][0][0] += (PACKED ? rf[S_DS + r0 + g] : d_sraw[pa]) * loss_scale;
      if (ib < n) acc16[0][0][2] += (PACKED ? rf[S_DS + r0 + g + 8] : d_sraw[pb]) * loss_scale;
    }
    uint32_t a_do[1][1][4];
    nsr_acc_to_afrag<1, 2>(acc16, a_do, NSR_ACT_NONE);
    nsr_store_afrag<1, 1>(a_do, T + T_DO, 24, r0);
    nsr_zero_acc(acc);
    nsr_gemm_wt<1, 1, 8>(acc, a_do, smem + NF_OFF_DW2, NSR_LD64);
    relu_mask_pack(acc, a_h1, a_d);
    nsr_store_afrag<1, 4>(a_d, T + T_DH1, NSR_LD64, r0);
    float accE[1][4][4];
    nsr_zero_acc(accE);
    nsr_gemm_wt<1, 4, 4>(accE, a_d, smem + NF_OFF_DW1, NF_LD32);

    // ---- hash-table scatter straight from the accumulator layout: this thread owns samples (g, g+8) x levels (c, 4+c, 8+c, 12+c).
    // Levels 0..7 (nt < 2): consecutive samples of a ray stay in one cell for several steps, so the 8 lanes that hold the
    // same level for 8 consecutive samples first merge runs of equal cells with a segmented shuffle scan and only the
    // last lane of each run issues the 8 REDs (-40 % REDs overall, far less same-address contention in L2).
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int64_t i = hh ? ib : ia;
      const bool ok = i < n;
      float x = 0.f, y = 0.f, z = 0.f, dx, dy, dz;
      if (ok) {
        if (PACKED) {
          const float* rr = rf + S_XYZ + (r0 + g + hh * 8) * 6;
          x = rr[0];
          y = rr[1];
          z = rr[2];
        } else {
          nf_sample_position<CT>(P, rays, ray_indices[i], t_starts[i], t_ends[i], x, y, z, dx, dy, dz);
        }
      }
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        const float d0 = ok ? accE[0][nt][hh * 2] * inv_scale : 0.f, d1 = ok ? accE[0][nt][hh * 2 + 1] * inv_scale : 0.f;
        const LevelInfo li = nsr_level(P.grid, nt * 4 + c);
        uint32_t cx, cy, cz, idx[8];
        float fx, fy, fz;
        nsr_pos_fract(x, li.scale, cx, fx);
        nsr_pos_fract(y, li.scale, cy, fy);
        nsr_pos_fract(z, li.scale, cz, fz);
        if (nt < 2) {
          // segmented inclusive scan over g (lanes c, c+4, ..., c+28) keyed by the cell
          const uint32_t key = ok ? (cx + li.res * (cy + li.res * cz)) : (0xFFFFFFF0u + g);
          const uint32_t key_prev = __shfl_up_sync(0xffffffffu, key, 4);
          const bool head = (g == 0) || (key_prev != key);
          const int next_head = __shfl_down_sync(0xffffffffu, (int)head, 4);
          const bool tail = (g == 7) || next_head;
          float v[16];
#pragma unroll
          for (int cc = 0; cc < 8; ++cc) {
            const float w = nsr_corner_weight(cc, fx, fy, fz);
            v[2 * cc] = w * d0;
            v[2 * cc + 1] = w * d1;
          }
          bool flag = head;
#pragma unroll
          for (int o = 1; o < 8; o <<= 1) {
            const int f_up = __shfl_up_sync(0xffffffffu, (int)flag, 4 * o);
            const bool take = (g >= o) && !flag;
#pragma unroll
            for (int e = 0; e < 16; ++e) {
              const float u = __shfl_up_sync(0xffffffffu, v[e], 4 * o);
              if (take) v[e] += u;
            }
            if (take) flag = f_up;
          }
          if (ok && tail) {
            nsr_corner_indices(li, cx, cy, cz, idx);
            // (pairing x-adjacent corners into one 16-byte RED, nsr_red_corner_pair, wins 27 % in the scatter-only micro-benchmark but
            //  not here: 205 -> 209 us -- at 8 warps/SM the cost is per RED instruction, and the divergent pair test adds instructions)
#pragma unroll
            for (int cc = 0; cc < 8; ++cc)
              if (v[2 * cc] != 0.f || v[2 * cc + 1] != 0.f) nsr_red_add_f32x2(grad_table + 2 * (size_t)idx[cc], v[2 * cc], v[2 * cc + 1]);
          }
        } else if (ok && (d0 != 0.f || d1 != 0.f)) {
          nsr_corner_indices(li, cx, cy, cz, idx);
#pragma unroll
          for (int cc = 0; cc < 8; ++cc) {
            const float w = nsr_corner_weight(cc, fx, fy, fz);
            nsr_red_add_f32x2(grad_table + 2 * (size_t)idx[cc], w * d0, w * d1);
          }
        }
      }
    }
    __syncthreads();
    // ---- weight gradients over the 64 rows of the tile
#pragma unroll
    for (int s = 0; s < kSlots; ++s) {
      const WgradTile w = wgrad_tile(warp + s * kWarps);
      const int xo = (w.x_off == T_X0) ? x0_off : w.x_off;  // the encoded features live in the current double buffer
      nsr_wgrad_tile(wacc[s][0], wacc[s][1], T + w.dy_off, w.ldy, w.m0, T + xo, w.ldx, w.n0, kRows);
    }
    if (NET == NF_NET_VANILLA) {  // bias gradients: column j of [dH1 (64) | dO (16) | dG1 (64) | dG2 (64) | dC3 (16)] over the tile's rows
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int j = threadIdx.x + q * kThreads;
        if (j < NF_B_TOTAL) {
          const __half* col = j < NF_B_D2 ? T + T_DH1 + j : j < NF_B_C1 ? T + T_DO + (j - NF_B_D2) : j < NF_B_C2 ? T + T_DG1 + (j - NF_B_C1)
                                                                                      : j < NF_B_C3 ? T + T_DG2 + (j - NF_B_C2) : T + T_DC3 + (j - NF_B_C3);
          const int ld = (j >= NF_B_D2 && j < NF_B_C1) || j >= NF_B_C3 ? 24 : NSR_LD64;
          float sum = 0.f;
#pragma unroll 8
          for (int r = 0; r < kRows; ++r) sum += __half2float(col[r * ld]);
          bsum[q] += sum;
        }
      }
    }
  }
  if (NET == NF_NET_VANILLA) {
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int j = threadIdx.x + q * kThreads;
      if (j < NF_B_TOTAL && bsum[q] != 0.f) atomicAdd(j < NF_B_C1 ? grad_dbias + j : grad_cbias + (j - NF_B_C1), bsum[q] * inv_scale);
    }
  }
#pragma unroll
  for (int s = 0; s < kSlots; ++s) {
    const WgradTile w = wgrad_tile(warp + s * kWarps);
    float* dst = (w.net == 0 ? grad_dparams : grad_cparams) + w.base;
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int o = w.m0 + g + ((i >> 1) << 3), ii = w.n0 + j * 8 + c * 2 + (i & 1);
        atomicAdd(dst + (size_t)o * w.in_dim + ii, wacc[s][j][i] * inv_scale);
      }
  }
}

// ==== network half of the split backward (nsr_nerf_field_bwd_net / _split) =====================================================
// One CTA per SM, 16 warps, persistent over the CTA's 64-row tiles of packed rows (tile = blockIdx.x + it * gridDim.x):
//   warps 0-11       three chain warpgroups that take the CTA's tiles in turn (group = it % 3).  A group runs the chain of nerf_bwd_kernel
//                    -- forward recompute and dgrad, activations in registers, 16 rows per warp, the same fp16 rounding points, ReLU
//                    masks and loss scale -- but issues each layer as register-A wgmma.mma_async over the group's 64 rows: A is the
//                    warps' m16n8k16 A fragments, B one canonical copy of the weights in shared memory (K-major for the forward, the
//                    same copy MN-major for the dgrad), so the weights are read once per warpgroup and layer, not once per warp.
//                    It writes d(encoding) to global memory and leaves every activation and pre-activation gradient the weight
//                    gradients need in a tile slot, in wgmma's canonical no-swizzle layout.
//                    Each group prefetches its next tile's inputs (cp.async, 7.5 KB) into its own stage while it computes.  Every layer
//                    ends in a wait for its wgmma: three groups keep the tensor cores busy during one another's waits and epilogues.
//   warps 12-15      one warpgroup that runs the five weight-gradient GEMMs of every tile (K = the tile's 64 rows) as wgmma.mma_async
//                    with both operands read from the slot (MN-major descriptors over the K-major tiles: no transposes).  dDW2 and dCW3
//                    (16 outputs) are computed transposed so that M = 64.  The 80 fp32 accumulators per thread live in registers for the
//                    whole kernel; one atomicAdd per weight per CTA at the end.
// Three slots form a ring (tile it -> slot it % 3, so each group fills its own slot): mbarrier FULL[s] hands a slot from its chain group
// to the warpgroup, EMPTY[s] back.  512 threads leave 128 registers per thread; neither role spills at that budget.
// Rows past the live count hold zeros in every slot operand: their encodings and per-row inputs are zeroed in the stage, and every
// layer maps zero inputs to zero.
constexpr int kChainGroups = 3;
constexpr int kNetThreads = (kChainGroups + 1) * 128;
// one tile slot (bytes), canonical [64][K] fp16 tiles
constexpr int SL_X0 = 0;                    // [64][32] encoded features
constexpr int SL_CI = SL_X0 + kRows * 32 * 2;   // [64][32] colour input: out16 | SH16
constexpr int SL_H1 = SL_CI + kRows * 32 * 2;   // [64][64] density hidden (post ReLU)
constexpr int SL_G1 = SL_H1 + kRows * 64 * 2;   // [64][64]
constexpr int SL_G2 = SL_G1 + kRows * 64 * 2;   // [64][64]
constexpr int SL_DC3 = SL_G2 + kRows * 64 * 2;  // [64][16] d(rgb pre-activation), columns 3..15 zero
constexpr int SL_DO = SL_DC3 + kRows * 16 * 2;  // [64][16] d(out16)
constexpr int SL_DG2 = SL_DO + kRows * 16 * 2;  // [64][64]
constexpr int SL_DG1 = SL_DG2 + kRows * 64 * 2; // [64][64]
constexpr int SL_DH1 = SL_DG1 + kRows * 64 * 2; // [64][64]
constexpr int kSlotBytes = SL_DH1 + kRows * 64 * 2;  // 61440
constexpr int kNetSlots = 3;
// CTA map (bytes): weights | slots | one input stage per chain group (encodings [64][40] halves + the per-row floats) | mbarriers
// weights of both networks, canonical [out][in] fp16 tiles
constexpr int NW_DW1 = 0;                      // [64][32]
constexpr int NW_DW2 = NW_DW1 + 64 * 32 * 2;   // [16][64]
constexpr int NW_CW1 = NW_DW2 + 16 * 64 * 2;   // [64][32]
constexpr int NW_CW2 = NW_CW1 + 64 * 32 * 2;   // [64][64]
constexpr int NW_CW3 = NW_CW2 + 64 * 64 * 2;   // [16][64]
constexpr int N_SLOTS = NW_CW3 + 16 * 64 * 2;  // 20480
constexpr int N_STAGE = N_SLOTS + kNetSlots * kSlotBytes;
constexpr int kStageBytes = kRows * NF_LD32 * 2 + S_ROWF * 4;  // 7680
constexpr int N_BARS = N_STAGE + kChainGroups * kStageBytes;
constexpr size_t kNetSmemBytes = N_BARS + 2 * kNetSlots * 8;
static_assert(N_SLOTS % 128 == 0 && kSlotBytes % 128 == 0 && kStageBytes % 16 == 0 && N_BARS % 8 == 0, "alignment");
static_assert(kNetSmemBytes <= 227 * 1024, "shared memory");

// A fragments <-> canonical [rows][K] tile (the fragment layout of nsr_load_afrag / nsr_store_afrag; 128-byte core matrices keep both
// conflict-free)
template <int KT>
__device__ __forceinline__ void canon_load_afrag(uint32_t (&a)[1][KT][4], const uint8_t* tile, int K, int row0, int col0 = 0) {
  const int lane = threadIdx.x & 31, mi = lane >> 3, r = lane & 7;
#pragma unroll
  for (int k = 0; k < KT; ++k) nsr_ldmatrix_x4(a[0][k], tile + nsr_canon_off(row0 + (mi & 1) * 8 + r, col0 + k * 16 + (mi >> 1) * 8, K));
}
template <int KT>
__device__ __forceinline__ void canon_store_afrag(const uint32_t (&a)[1][KT][4], uint8_t* tile, int K, int row0, int col0 = 0) {
  const int lane = threadIdx.x & 31, g = lane >> 2, c = lane & 3;
#pragma unroll
  for (int k = 0; k < KT; ++k) {
    const int col = col0 + k * 16 + c * 2;
    *reinterpret_cast<uint32_t*>(tile + nsr_canon_off(row0 + g, col, K)) = a[0][k][0];
    *reinterpret_cast<uint32_t*>(tile + nsr_canon_off(row0 + g + 8, col, K)) = a[0][k][1];
    *reinterpret_cast<uint32_t*>(tile + nsr_canon_off(row0 + g, col + 8, K)) = a[0][k][2];
    *reinterpret_cast<uint32_t*>(tile + nsr_canon_off(row0 + g + 8, col + 8, K)) = a[0][k][3];
  }
}
__device__ __forceinline__ void group_bar(int grp) { asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory"); }

// row-major [rows][K] fp16 matrix (global) -> canonical smem tile
__device__ __forceinline__ void canon_stage(uint8_t* dst, const __half* __restrict__ src, int rows, int K) {
  const int vec_per_row = K / 8;
  for (int i = threadIdx.x; i < rows * vec_per_row; i += blockDim.x) {
    const int r = i / vec_per_row, kc = i % vec_per_row;
    *reinterpret_cast<uint4*>(dst + nsr_canon_off(r, kc * 8, K)) = __ldg(reinterpret_cast<const uint4*>(src + (size_t)r * K) + kc);
  }
}

// One chain layer over the warpgroup's 64 rows: acc = A . W^T (TB 0, forward: W [N out][K in] read K-major) or acc = A . W (TB 1,
// dgrad: W [K out][ldw in] read MN-major, N <= ldw: the first N input columns).  A = this warp's 16 rows as KT m16n8k16 A fragments,
// W = a canonical weight tile at shared address w with ldw halves per row; acc in the m16n8 C-fragment layout.  Returns with the
// result in acc.
template <int N, int KT, int TB>
__device__ __forceinline__ void chain_gemm(float (&acc)[1][N / 8][4], const uint32_t (&a)[1][KT][4], uint32_t w, int ldw) {
  float(&d)[N / 2] = *reinterpret_cast<float(*)[N / 2]>(&acc[0][0][0]);
#pragma unroll
  for (int kk = 0; kk < KT; ++kk)
#pragma unroll
    for (int i = 0; i < 4; ++i) asm volatile("" ::"r"(a[0][kk][i]) : "memory");  // the A fragments are complete before the fence
  nsr_wg_fence_regs(d);
  nsr_wg_fence();
#pragma unroll
  for (int kk = 0; kk < KT; ++kk) {
    const uint64_t db = TB ? nsr_wg_desc_mn(w, ldw, kk) : nsr_wg_desc(w + 256u * (uint32_t)kk, 128u, (uint32_t)(ldw / 8) * 128u);
    nsr_wgmma_rs<N, TB>(d, a[0][kk], db, kk > 0 ? 1u : 0u);
  }
  nsr_wg_commit();
  nsr_wg_wait0();
  nsr_wg_fence_regs(d);
}

// flush one weight-gradient accumulator (m64nN layout) into dst[m * stride_m + n * stride_n]
template <int R>
__device__ __forceinline__ void net_flush(const float (&w)[R], float* dst, int stride_m, int stride_n, float inv_scale) {
  const int lane = threadIdx.x & 31, m0 = 16 * ((threadIdx.x >> 5) & 3) + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int j = r >> 2, h = (r >> 1) & 1, e = r & 1;
    atomicAdd(dst + (size_t)(m0 + 8 * h) * stride_m + (size_t)(8 * j + c0 + e) * stride_n, w[r] * inv_scale);
  }
}

__global__ void __launch_bounds__(kNetThreads, 1) nerf_bwd_net_kernel(const __half* __restrict__ enc_save, const __half* __restrict__ dparams,
                                                                      const __half* __restrict__ cparams, const float* __restrict__ d_sraw,
                                                                      const float* __restrict__ d_rgb, float* __restrict__ grad_dparams,
                                                                      float* __restrict__ grad_cparams, float loss_scale,
                                                                      const float* __restrict__ amax_ptr, int64_t n_cap,
                                                                      const int64_t* __restrict__ n_dev, const float* __restrict__ xyzdir,
                                                                      uint32_t* __restrict__ denc_out) {
  const int64_t n = n_dev ? min(*n_dev, n_cap) : n_cap;
  extern __shared__ __align__(128) uint8_t smem_net[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (loss_scale <= 0.f) {  // automatic: the same rule as nerf_bwd_kernel
    const float amax = fmaxf(__ldg(amax_ptr), 1e-30f);
    loss_scale = exp2f(fminf(fmaxf(floorf(log2f(256.f / amax)), -24.f), 60.f));
  }
  const float inv_scale = 1.f / loss_scale;
  const uint32_t sbase = nsr_smem_u32(smem_net);
  auto full_bar = [&](int s) { return sbase + N_BARS + 8u * (uint32_t)s; };
  auto empty_bar = [&](int s) { return sbase + N_BARS + 8u * (uint32_t)(kNetSlots + s); };
  if (threadIdx.x == 0) {
    for (int s = 0; s < kNetSlots; ++s) {
      mbar_init(full_bar(s), 128);   // the 128 threads of the chain group that filled the slot
      mbar_init(empty_bar(s), 128);  // the 128 threads of the weight-gradient warpgroup
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  canon_stage(smem_net + NW_DW1, dparams, 64, 32);
  canon_stage(smem_net + NW_DW2, dparams + 64 * 32, 16, 64);
  canon_stage(smem_net + NW_CW1, cparams, 64, 32);
  canon_stage(smem_net + NW_CW2, cparams + 64 * 32, 64, 64);
  canon_stage(smem_net + NW_CW3, cparams + 64 * 32 + 64 * 64, 16, 64);
  nsr_proxy_fence();  // the chain's wgmmas read the weights through the async proxy
  __syncthreads();
  const int64_t n_tiles = (n + kRows - 1) / kRows;
  const int64_t my_tiles = n_tiles > (int64_t)blockIdx.x ? (n_tiles - 1 - blockIdx.x) / gridDim.x + 1 : 0;

  if (warp < 4 * kChainGroups) {
    // ================================ chain groups ================================
    const int grp = warp >> 2, gtid = threadIdx.x & 127, g = lane >> 2, c = lane & 3;
    const int r0 = (warp & 3) * 16;
    __half* sx = reinterpret_cast<__half*>(smem_net + N_STAGE + grp * kStageBytes);  // [64][40] encodings of the group's next tile
    float* rf = reinterpret_cast<float*>(smem_net + N_STAGE + grp * kStageBytes + kRows * NF_LD32 * 2);
    auto fetch_tile = [&](int64_t it) {  // inputs of the CTA's tile `it` -> this group's stage (16-byte chunks, L1 bypassed)
      const int64_t row0 = ((int64_t)blockIdx.x + it * gridDim.x) * kRows;
      for (int v = gtid; v < kRows * 4; v += 128) cp_async16(sx + (v >> 2) * NF_LD32 + (v & 3) * 8, enc_save + (row0 + (v >> 2)) * 32 + (v & 3) * 8);
      if (gtid < kRows * 6 / 4) cp_async16(rf + S_XYZ + gtid * 4, xyzdir + row0 * 6 + gtid * 4);
      if (gtid < kRows / 4) cp_async16(rf + S_DS + gtid * 4, d_sraw + row0 + gtid * 4);
      if (gtid >= 64 && gtid < 64 + kRows * 3 / 4) cp_async16(rf + S_DRGB + (gtid - 64) * 4, d_rgb + row0 * 3 + (gtid - 64) * 4);
      cp_async_commit();
    };
    if (grp < my_tiles) fetch_tile(grp);
    for (int64_t it = grp; it < my_tiles; it += kChainGroups) {
      const int s = (int)(it % kNetSlots);
      const int64_t row0 = ((int64_t)blockIdx.x + it * gridDim.x) * kRows;
      cp_async_wait_all();
      group_bar(grp);  // the group's copies have all landed
      if (row0 + kRows > n) {  // last, partial tile: rows >= n hold stale data; zero them so that 0 * garbage never reaches the wgrad sums
        for (int v = gtid; v < kRows * 4; v += 128)
          if (row0 + (v >> 2) >= n) *reinterpret_cast<uint4*>(sx + (v >> 2) * NF_LD32 + (v & 3) * 8) = make_uint4(0, 0, 0, 0);
        for (int v = gtid; v < S_ROWF; v += 128) {
          const int r = v < S_DS ? v / 6 : (v < S_DRGB ? v - S_DS : (v - S_DRGB) / 3);
          if (row0 + r >= n) rf[v] = 0.f;
        }
        group_bar(grp);
      }
      if (it >= kNetSlots) mbar_wait(empty_bar(s), (uint32_t)((it / kNetSlots - 1) & 1), nullptr, 0);  // tile it - 3's wgrad is done
      uint8_t* slot = smem_net + N_SLOTS + s * kSlotBytes;
      const int64_t ia = row0 + r0 + g, ib = ia + 8;
      // ---- this warp's 16 rows: encoded features (-> slot X0) and SH of the view direction (-> CI columns 16..31); per-row gradients
      uint32_t a_in[1][2][4];
      nsr_load_afrag<1, 2>(a_in, sx, NF_LD32, r0);
      canon_store_afrag<2>(a_in, slot + SL_X0, 32, r0);
      if (lane < 16) {
        uint4 s0 = make_uint4(0, 0, 0, 0), s1 = s0;
        if (row0 + r0 + lane < n) {
          float sh[16];
          const float* rr = rf + S_XYZ + (r0 + lane) * 6;
          nsr_sh4(rr[3], rr[4], rr[5], sh);
          s0 = make_uint4(nsr_pack_h2(sh[0], sh[1]), nsr_pack_h2(sh[2], sh[3]), nsr_pack_h2(sh[4], sh[5]), nsr_pack_h2(sh[6], sh[7]));
          s1 = make_uint4(nsr_pack_h2(sh[8], sh[9]), nsr_pack_h2(sh[10], sh[11]), nsr_pack_h2(sh[12], sh[13]), nsr_pack_h2(sh[14], sh[15]));
        }
        *reinterpret_cast<uint4*>(slot + SL_CI + nsr_canon_off(r0 + lane, 16, 32)) = s0;
        *reinterpret_cast<uint4*>(slot + SL_CI + nsr_canon_off(r0 + lane, 24, 32)) = s1;
      }
      float drgb[2][2], dsr[2];  // (row g / g+8) x (columns 2c, 2c+1 < 3); d sigma_raw of rows g, g+8
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
        for (int e = 0; e < 2; ++e) drgb[hh][e] = (c * 2 + e < 3) ? rf[S_DRGB + (r0 + g + hh * 8) * 3 + c * 2 + e] : 0.f;
        dsr[hh] = rf[S_DS + r0 + g + hh * 8];
      }
      group_bar(grp);  // the whole group is done with the stage: refill it with the group's next tile
      if (it + kChainGroups < my_tiles) fetch_tile(it + kChainGroups);

      // ---- forward recompute
      uint32_t a_h1[1][4][4], a_o[1][1][4], a_g1[1][4][4], a_g2[1][4][4];
      float acc[1][8][4], acc16[1][2][4];
      chain_gemm<64, 2, 0>(acc, a_in, sbase + NW_DW1, 32);
      nsr_acc_to_afrag<1, 8>(acc, a_h1, NSR_ACT_RELU);
      canon_store_afrag<4>(a_h1, slot + SL_H1, 64, r0);
      chain_gemm<16, 4, 0>(acc16, a_h1, sbase + NW_DW2, 64);
      nsr_acc_to_afrag<1, 2>(acc16, a_o, NSR_ACT_NONE);
      canon_store_afrag<1>(a_o, slot + SL_CI, 32, r0);
      __syncwarp();
      {
        uint32_t a_c[1][2][4], a_sh[1][1][4];
        canon_load_afrag<1>(a_sh, slot + SL_CI, 32, r0, 16);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          a_c[0][0][j] = a_o[0][0][j];
          a_c[0][1][j] = a_sh[0][0][j];
        }
        chain_gemm<64, 2, 0>(acc, a_c, sbase + NW_CW1, 32);
      }
      nsr_acc_to_afrag<1, 8>(acc, a_g1, NSR_ACT_RELU);
      canon_store_afrag<4>(a_g1, slot + SL_G1, 64, r0);
      chain_gemm<64, 4, 0>(acc, a_g1, sbase + NW_CW2, 64);
      nsr_acc_to_afrag<1, 8>(acc, a_g2, NSR_ACT_RELU);
      canon_store_afrag<4>(a_g2, slot + SL_G2, 64, r0);
      chain_gemm<16, 4, 0>(acc16, a_g2, sbase + NW_CW3, 64);
      // ---- d(rgb pre-activation) = d_rgb * s (1 - s), s = sigmoid(fp16(raw)); columns 0..2 only
      uint32_t a_dc3[1][1][4];
      {
        float dp[4] = {0.f, 0.f, 0.f, 0.f};  // (row g: col c*2, c*2+1), (row g+8: col c*2, c*2+1)
        if (c < 2) {
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            if ((hh ? ib : ia) < n) {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                if (c * 2 + e < 3) {
                  const float raw = __half2float(__float2half_rn(acc16[0][0][hh * 2 + e]));
                  const float sg = 1.f / (1.f + expf(-raw));
                  dp[hh * 2 + e] = drgb[hh][e] * sg * (1.f - sg) * loss_scale;
                }
              }
            }
          }
        }
        a_dc3[0][0][0] = nsr_pack_h2(dp[0], dp[1]);
        a_dc3[0][0][1] = nsr_pack_h2(dp[2], dp[3]);
        a_dc3[0][0][2] = 0u;
        a_dc3[0][0][3] = 0u;
        canon_store_afrag<1>(a_dc3, slot + SL_DC3, 16, r0);
      }
      // ---- dgrad chain
      uint32_t a_d[1][4][4];
      chain_gemm<64, 1, 1>(acc, a_dc3, sbase + NW_CW3, 64);
      relu_mask_pack(acc, a_g2, a_d);
      canon_store_afrag<4>(a_d, slot + SL_DG2, 64, r0);
      chain_gemm<64, 4, 1>(acc, a_d, sbase + NW_CW2, 64);
      relu_mask_pack(acc, a_g1, a_d);
      canon_store_afrag<4>(a_d, slot + SL_DG1, 64, r0);
      chain_gemm<16, 4, 1>(acc16, a_d, sbase + NW_CW1, 32);  // first 16 input columns = the geometry features
      if (c == 0) {  // density path: d(out0) += d sigma / d raw (trunc_exp backward folded in by nsr_nerf_ray_bwd)
        if (ia < n) acc16[0][0][0] += dsr[0] * loss_scale;
        if (ib < n) acc16[0][0][2] += dsr[1] * loss_scale;
      }
      uint32_t a_do[1][1][4];
      nsr_acc_to_afrag<1, 2>(acc16, a_do, NSR_ACT_NONE);
      canon_store_afrag<1>(a_do, slot + SL_DO, 16, r0);
      chain_gemm<64, 1, 1>(acc, a_do, sbase + NW_DW2, 64);
      relu_mask_pack(acc, a_h1, a_d);
      canon_store_afrag<4>(a_d, slot + SL_DH1, 64, r0);
      // the slot is complete: make this thread's stores visible to the tensor core and hand the slot over
      nsr_proxy_fence();
      mbar_arrive(full_bar(s));
      float accE[1][4][4];
      chain_gemm<32, 4, 1>(accE, a_d, sbase + NW_DW1, 32);
      // ---- d(encoding) -> fp16 pairs [n][16 levels], still multiplied by the loss scale: 4 lanes x 4 bytes = 16 contiguous bytes per (row, nt)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int64_t i = hh ? ib : ia;
        if (i < n) {
#pragma unroll
          for (int nt = 0; nt < 4; ++nt) denc_out[i * 16 + nt * 4 + c] = nsr_pack_h2(accE[0][nt][hh * 2], accE[0][nt][hh * 2 + 1]);
        }
      }
    }
  } else {
    // ================================ weight-gradient warpgroup ================================
    float w_dw1[16], w_dw2t[8], w_cw1[16], w_cw2[32], w_cw3t[8];  // m64 x n32 / n16 / n32 / n64 / n16
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      if (i < 8) w_dw2t[i] = w_cw3t[i] = 0.f;
      if (i < 16) w_dw1[i] = w_cw1[i] = 0.f;
      w_cw2[i] = 0.f;
    }
    for (int64_t it = 0; it < my_tiles; ++it) {
      const int s = (int)(it % kNetSlots);
      mbar_wait(full_bar(s), (uint32_t)((it / kNetSlots) & 1), nullptr, 0);
      const uint32_t sl = sbase + N_SLOTS + (uint32_t)s * kSlotBytes;
      nsr_wg_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {  // K = 64 rows in four k16 steps
        nsr_wgmma_n32<1, 1>(w_dw1, nsr_wg_desc_mn(sl + SL_DH1, 64, kk), nsr_wg_desc_mn(sl + SL_X0, 32, kk), 1u);   // dDW1   += dH1^T . X0
        nsr_wgmma_n16<1, 1>(w_dw2t, nsr_wg_desc_mn(sl + SL_H1, 64, kk), nsr_wg_desc_mn(sl + SL_DO, 16, kk), 1u);   // dDW2^T += H1^T . dO
        nsr_wgmma_n32<1, 1>(w_cw1, nsr_wg_desc_mn(sl + SL_DG1, 64, kk), nsr_wg_desc_mn(sl + SL_CI, 32, kk), 1u);   // dCW1   += dG1^T . CI
        nsr_wgmma_n64<1, 1>(w_cw2, nsr_wg_desc_mn(sl + SL_DG2, 64, kk), nsr_wg_desc_mn(sl + SL_G1, 64, kk), 1u);   // dCW2   += dG2^T . G1
        nsr_wgmma_n16<1, 1>(w_cw3t, nsr_wg_desc_mn(sl + SL_G2, 64, kk), nsr_wg_desc_mn(sl + SL_DC3, 16, kk), 1u);  // dCW3^T += G2^T . dC3
      }
      nsr_wg_commit();
      nsr_wg_wait0();
      nsr_wg_fence_regs(w_dw1);
      nsr_wg_fence_regs(w_dw2t);
      nsr_wg_fence_regs(w_cw1);
      nsr_wg_fence_regs(w_cw2);
      nsr_wg_fence_regs(w_cw3t);
      mbar_arrive(empty_bar(s));
    }
    if (my_tiles > 0) {
      net_flush(w_dw1, grad_dparams, 32, 1, inv_scale);                           // dDW1 [out m][in n]
      net_flush(w_dw2t, grad_dparams + 64 * 32, 1, 64, inv_scale);                // dDW2^T [in m][out n] -> DW2 [out][in]
      net_flush(w_cw1, grad_cparams, 32, 1, inv_scale);                           // dCW1 [out m][in n]
      net_flush(w_cw2, grad_cparams + 64 * 32, 64, 1, inv_scale);                 // dCW2 [out m][in n]
      net_flush(w_cw3t, grad_cparams + 64 * 32 + 64 * 64, 1, 64, inv_scale);      // dCW3^T [in m][out n] -> CW3 [out][in]
    }
  }
}

}  // namespace

namespace {

// Table half of the split backward: rows = kept samples in packed (ray-major) order, thread per row, a warp = 32 consecutive rows.
// Per level: corner weights x d(feature pair); on levels < kMergeLevels runs of rows that sit in the same cell (consecutive samples of
// a ray on the coarse levels) are summed with a segmented shuffle scan over the whole warp and only the run's last lane issues REDs;
// x-adjacent corners that are neighbours in memory (hashed levels: cell x even; dense levels: entry index even) leave as ONE 16-byte
// red.global.add.v4.f32.  48 registers, no shared memory: 64 warps per SM keep the RED path of the SM full (tools/gather_bench.py times
// this form against the plain 8-byte REDs).
constexpr int kMergeLevels = 8;

// The register allocation is sized for 5 resident CTAs per SM (48 registers); budgets for 6 and 8 CTAs spill and measured slower.
__global__ void __launch_bounds__(256, 5) nerf_table_scatter_kernel(const __grid_constant__ nsr_grid_t g, const float* __restrict__ xyz, int stride,
                                                                 const __half2* __restrict__ denc, float loss_scale,
                                                                 const float* __restrict__ amax_ptr, float* __restrict__ grad_table,
                                                                 int64_t n_cap, const int64_t* __restrict__ n_dev, int l_begin, int l_end) {
  const int64_t n = n_dev ? min(*n_dev, n_cap) : n_cap;
  if (loss_scale <= 0.f) {  // the same automatic scale as nerf_bwd_kernel derives from the same amax
    const float amax = fmaxf(__ldg(amax_ptr), 1e-30f);
    loss_scale = exp2f(fminf(fmaxf(floorf(log2f(256.f / amax)), -24.f), 60.f));
  }
  const float inv_scale = 1.f / loss_scale;
  const int lane = threadIdx.x & 31;
  const int64_t n32 = (n + 31) & ~31ll;
  for (int64_t i = blockIdx.x * 256ll + threadIdx.x; i < n32; i += (int64_t)gridDim.x * 256) {
    const bool ok = i < n;
    float x = 0.f, y = 0.f, z = 0.f;
    if (ok) {
      x = xyz[i * stride];
      y = xyz[i * stride + 1];
      z = xyz[i * stride + 2];
    }
    uint2 dq = make_uint2(0u, 0u);   // the row's d(encoding) of the level pair that holds level l: one 8-byte load per pair
#pragma unroll 1
    for (int l = l_begin; l < l_end; ++l) {  // the backward scatters level groups in separate launches (each group's gradient slice stays in L2)
      float2 d = make_float2(0.f, 0.f);
      if (ok) {
        if (l == l_begin || (l & 1) == 0) dq = __ldg(reinterpret_cast<const uint2*>(denc + i * 16 + (l & ~1)));
        const uint32_t h = (l & 1) ? dq.y : dq.x;
        d = __half22float2(*reinterpret_cast<const __half2*>(&h));
        d.x *= inv_scale;
        d.y *= inv_scale;
      }
      const LevelInfo li = nsr_level(g, l);
      uint32_t cx, cy, cz, idx[8];
      float fx, fy, fz;
      nsr_pos_fract(x, li.scale, cx, fx);
      nsr_pos_fract(y, li.scale, cy, fy);
      nsr_pos_fract(z, li.scale, cz, fz);
      float v[16];
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const float w = nsr_corner_weight(c, fx, fy, fz);
        v[2 * c] = w * d.x;
        v[2 * c + 1] = w * d.y;
      }
      bool issue = ok && (d.x != 0.f || d.y != 0.f);
      if (l < kMergeLevels) {  // res^3 < 2^32 on these levels (base 16 .. 32, growth <= 1.45): the cell index is a unique key
        const uint32_t key = ok ? (cx + li.res * (cy + li.res * cz)) : (0xFFFFFF00u + lane);
        const uint32_t prev = __shfl_up_sync(0xffffffffu, key, 1);
        const bool head = lane == 0 || prev != key;
        const uint32_t heads = __ballot_sync(0xffffffffu, head);
        const int my_head = 31 - __clz(heads & (0xffffffffu >> (31 - lane)));  // first lane of my run
        const bool tail = lane == 31 || ((heads >> (lane + 1)) & 1u);
        int maxrun = lane - my_head + 1;  // the longest run of the warp bounds the number of scan steps (warp-uniform)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) maxrun = max(maxrun, __shfl_xor_sync(0xffffffffu, maxrun, o));
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          if (o < maxrun) {
            const bool take = lane - o >= my_head;
#pragma unroll
            for (int e = 0; e < 16; ++e) {
              const float u = __shfl_up_sync(0xffffffffu, v[e], o);
              if (take) v[e] += u;
            }
          }
        }
        issue = ok && tail;
      }
      if (issue) {
        nsr_corner_indices(li, cx, cy, cz, idx);
#pragma unroll
        for (int c = 0; c < 8; c += 2) nsr_red_corner_pair(grad_table, idx[c], idx[c + 1], v[2 * c], v[2 * c + 1], v[2 * c + 2], v[2 * c + 3]);
      }
    }
  }
}

int field_bwd_launch(const nsr_nerf_t* f, const float* rays, const int32_t* ray_indices, const float* t_starts, const float* t_ends,
                     const void* enc_save_h, const void* dparams_h, const void* cparams_h, const float* d_sraw, const float* d_rgb,
                     float* grad_dparams, float* grad_cparams, float loss_scale, const float* amax, int64_t k, const int64_t* k_dev,
                     const int64_t* row_pos, const float* xyzdir, void* stream, const char* who) {
  NSR_REQUIRE(f != nullptr, "%s: field descriptor is NULL", who);
  NSR_REQUIRE(f->grid.n_levels == 16 && f->grid.n_features == 2 && f->feature_dim == 16 && f->density_hidden == 1 && f->color_hidden == 2,
              "%s: fused path needs L=16, F=2, feature_dim=16, hidden layers 1/2", who);
  NSR_REQUIRE(loss_scale > 0.f || amax != nullptr, "%s: loss_scale <= 0 (automatic) needs the amax pointer", who);
  if (k == 0) return 0;
  NSR_REQUIRE(xyzdir == nullptr || row_pos == nullptr, "%s: packed inputs (xyzdir) and row_pos are mutually exclusive", who);
  NSR_REQUIRE(f->contraction == NF_AABB || (f->contraction == NF_UNBOUNDED_SPHERE && xyzdir == nullptr),
              "%s: contraction type %d not implemented here (AABB=0; UN_BOUNDED_SPHERE=2 only without xyzdir)", who, f->contraction);
  static thread_local bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(nerf_bwd_kernel<false, NF_AABB, NF_NET_FULLY_FUSED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(nerf_bwd_kernel<true, NF_AABB, NF_NET_FULLY_FUSED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(nerf_bwd_kernel<false, NF_UNBOUNDED_SPHERE, NF_NET_FULLY_FUSED>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               (int)kSmemBytes);
    if (e != cudaSuccess) {
      nsr_set_error("%s: cannot reserve %zu B shared memory: %s", who, kSmemBytes, cudaGetErrorString(e));
      return 2;
    }
    attr_set = true;
  }
  const int64_t tiles = (k + kRows - 1) / kRows;
  int grid = (int)min((int64_t)nsr_sm_count() * kCtasPerSm, tiles);
  if (k_dev != nullptr) grid = nsr_sm_count() * kCtasPerSm;
#define NSR_BWD_ARGS                                                                                                                        \
  *f, rays, ray_indices, t_starts, t_ends, (const __half*)enc_save_h, (const __half*)dparams_h, (const __half*)cparams_h, d_sraw, d_rgb,    \
      grad_dparams, grad_cparams, loss_scale, amax, k, k_dev, row_pos, xyzdir, nullptr, nullptr, nullptr, nullptr, nullptr
  if (xyzdir != nullptr)
    nerf_bwd_kernel<true, NF_AABB, NF_NET_FULLY_FUSED><<<grid, kThreads, kSmemBytes, (cudaStream_t)stream>>>(NSR_BWD_ARGS);
  else if (f->contraction == NF_UNBOUNDED_SPHERE)
    nerf_bwd_kernel<false, NF_UNBOUNDED_SPHERE, NF_NET_FULLY_FUSED><<<grid, kThreads, kSmemBytes, (cudaStream_t)stream>>>(NSR_BWD_ARGS);
  else
    nerf_bwd_kernel<false, NF_AABB, NF_NET_FULLY_FUSED><<<grid, kThreads, kSmemBytes, (cudaStream_t)stream>>>(NSR_BWD_ARGS);
#undef NSR_BWD_ARGS
  NSR_CHECK_LAUNCH(who);
  return 0;
}

// the VanillaMLP field (NeuS learned background): contracted, positions recomputed from the rays
int bg_field_bwd_launch(const nsr_nerf_t* f, const float* rays, const int32_t* ray_indices, const float* t_starts, const float* t_ends,
                        const void* enc_save_h, const void* dmlp_h, const float* dbias, const void* cmlp_h, const float* cbias, const float* d_sraw,
                        const float* d_rgb, float* grad_dmlp, float* grad_table, float* grad_dbias, float* grad_cmlp, float* grad_cbias,
                        float loss_scale, const float* amax, int64_t k, const int64_t* k_dev, void* stream, const char* who) {
  NSR_REQUIRE(f != nullptr, "%s: field descriptor is NULL", who);
  NSR_REQUIRE(f->grid.n_levels == 16 && f->grid.n_features == 2 && f->feature_dim == 16 && f->density_hidden == 1 && f->color_hidden == 2,
              "%s: fused path needs L=16, F=2, feature_dim=16, hidden layers 1/2", who);
  NSR_REQUIRE(f->contraction == NF_UNBOUNDED_SPHERE, "%s: the VanillaMLP field needs contraction = 2 (UN_BOUNDED_SPHERE), got %d", who,
              f->contraction);
  NSR_REQUIRE(loss_scale > 0.f || amax != nullptr, "%s: loss_scale <= 0 (automatic) needs the amax pointer", who);
  if (k == 0) return 0;
  NSR_REQUIRE(dbias != nullptr && cbias != nullptr && grad_dmlp != nullptr && grad_table != nullptr && grad_dbias != nullptr &&
                  grad_cmlp != nullptr && grad_cbias != nullptr,
              "%s: bias / gradient pointer is NULL", who);
  auto kern = nerf_bwd_kernel<false, NF_UNBOUNDED_SPHERE, NF_NET_VANILLA>;
  static thread_local bool attr_set = false;
  if (!attr_set) {
    const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytesVanilla);
    if (e != cudaSuccess) {
      nsr_set_error("%s: cannot reserve %zu B shared memory: %s", who, kSmemBytesVanilla, cudaGetErrorString(e));
      return 2;
    }
    attr_set = true;
  }
  const int64_t tiles = (k + kRows - 1) / kRows;
  const int grid = k_dev != nullptr ? nsr_sm_count() * kCtasPerSm : (int)min((int64_t)nsr_sm_count() * kCtasPerSm, tiles);
  kern<<<grid, kThreads, kSmemBytesVanilla, (cudaStream_t)stream>>>(*f, rays, ray_indices, t_starts, t_ends, (const __half*)enc_save_h,
                                                                    (const __half*)dmlp_h, (const __half*)cmlp_h, d_sraw, d_rgb, grad_dmlp, grad_cmlp,
                                                                    loss_scale, amax, k, k_dev, nullptr, nullptr, dbias, cbias, grad_table,
                                                                    grad_dbias, grad_cbias);
  NSR_CHECK_LAUNCH(who);
  return 0;
}

// network half of the split backward: nerf_bwd_net_kernel, one CTA per SM
int field_bwd_net_launch(const nsr_nerf_t* f, const void* enc_k_h, const void* dparams_h, const void* cparams_h, const float* d_sraw,
                         const float* d_rgb, float* grad_dparams, float* grad_cparams, float loss_scale, const float* amax, int64_t k,
                         const int64_t* k_dev, const float* xyzdir, void* denc_h, void* stream, const char* who) {
  NSR_REQUIRE(f != nullptr, "%s: field descriptor is NULL", who);
  NSR_REQUIRE(f->grid.n_levels == 16 && f->grid.n_features == 2 && f->feature_dim == 16 && f->density_hidden == 1 && f->color_hidden == 2,
              "%s: fused path needs L=16, F=2, feature_dim=16, hidden layers 1/2", who);
  NSR_REQUIRE(loss_scale > 0.f || amax != nullptr, "%s: loss_scale <= 0 (automatic) needs the amax pointer", who);
  NSR_REQUIRE(denc_h != nullptr && xyzdir != nullptr, "%s: denc / xyzdir is NULL", who);
  NSR_REQUIRE(f->contraction == NF_AABB, "%s: packed inputs (xyzdir) need the AABB contraction (got %d)", who, f->contraction);
  if (k == 0) return 0;
  static thread_local bool attr_set = false;
  if (!attr_set) {
    const cudaError_t e = cudaFuncSetAttribute(nerf_bwd_net_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kNetSmemBytes);
    if (e != cudaSuccess) {
      nsr_set_error("%s: cannot reserve %zu B shared memory: %s", who, kNetSmemBytes, cudaGetErrorString(e));
      return 2;
    }
    attr_set = true;
  }
  const int64_t tiles = (k + kRows - 1) / kRows;
  const int grid = k_dev != nullptr ? nsr_sm_count() : (int)min((int64_t)nsr_sm_count(), tiles);
  nerf_bwd_net_kernel<<<grid, kNetThreads, kNetSmemBytes, (cudaStream_t)stream>>>((const __half*)enc_k_h, (const __half*)dparams_h, (const __half*)cparams_h,
                                                                                  d_sraw, d_rgb, grad_dparams, grad_cparams, loss_scale, amax, k, k_dev,
                                                                                  xyzdir, (uint32_t*)denc_h);
  NSR_CHECK_LAUNCH(who);
  return 0;
}

}  // namespace

extern "C" int nsr_nerf_field_bwd(const nsr_nerf_t* f, const float* rays, const int32_t* ray_indices, const float* t_starts,
                                  const float* t_ends, const void* enc_save_h, const void* dparams_h, const void* cparams_h,
                                  const float* d_sraw, const float* d_rgb, float* grad_dparams, float* grad_cparams, float loss_scale,
                                  const float* amax, int64_t k, const int64_t* k_dev, const int64_t* row_pos, const float* xyzdir,
                                  void* stream) {
  return field_bwd_launch(f, rays, ray_indices, t_starts, t_ends, enc_save_h, dparams_h, cparams_h, d_sraw, d_rgb, grad_dparams, grad_cparams,
                          loss_scale, amax, k, k_dev, row_pos, xyzdir, stream, "nsr_nerf_field_bwd");
}

extern "C" int nsr_bg_field_bwd(const nsr_nerf_t* f, const float* rays, const int32_t* ray_indices, const float* t_starts, const float* t_ends,
                                const void* enc_save_h, const void* dmlp_h, const float* dbias, const void* cmlp_h, const float* cbias,
                                const float* d_sraw, const float* d_rgb, float* grad_dmlp, float* grad_table, float* grad_dbias, float* grad_cmlp,
                                float* grad_cbias, float loss_scale, const float* amax, int64_t k, const int64_t* k_dev, void* stream) {
  return bg_field_bwd_launch(f, rays, ray_indices, t_starts, t_ends, enc_save_h, dmlp_h, dbias, cmlp_h, cbias, d_sraw, d_rgb, grad_dmlp, grad_table,
                             grad_dbias, grad_cmlp, grad_cbias, loss_scale, amax, k, k_dev, stream, "nsr_bg_field_bwd");
}

// The two halves of the split backward as separate entry points (what the Python side calls, so that each half shows up with its own
// duration in bench.py's per-kernel table):
//   nsr_nerf_field_bwd_net   : MLP recompute + dgrad + wgrad over the packed rows; d(encoding) -> denc_h (fp16 [k,32], still multiplied by
//                              the loss scale); grad_dparams receives only the density network's weight gradients
//   nsr_nerf_table_scatter   : levels [level_begin, level_end) of denc_h -> fp32 REDs into grad_table (= grad_dparams + the density network's parameter count); xyz = the
//                              packed unit-cube positions with row stride `stride` floats (6 for the xyzdir buffer of nsr_pack_kept)
extern "C" int nsr_nerf_field_bwd_net(const nsr_nerf_t* f, const void* enc_k_h, const void* dparams_h, const void* cparams_h, const float* d_sraw,
                                      const float* d_rgb, float* grad_dparams, float* grad_cparams, float loss_scale, const float* amax, int64_t k,
                                      const int64_t* k_dev, const float* xyzdir, void* denc_h, void* stream) {
  return field_bwd_net_launch(f, enc_k_h, dparams_h, cparams_h, d_sraw, d_rgb, grad_dparams, grad_cparams, loss_scale, amax, k, k_dev, xyzdir, denc_h,
                              stream, "nsr_nerf_field_bwd_net");
}

extern "C" int nsr_nerf_table_scatter(const nsr_grid_t* g, const float* xyz, int32_t stride, const void* denc_h, float loss_scale, const float* amax,
                                      float* grad_table, int64_t k, const int64_t* k_dev, int32_t level_begin, int32_t level_end, int32_t ctas_per_sm,
                                      void* stream) {
  NSR_REQUIRE(g != nullptr && xyz != nullptr && denc_h != nullptr && grad_table != nullptr, "nsr_nerf_table_scatter: NULL argument");
  NSR_REQUIRE(g->n_levels == 16 && g->n_features == 2, "nsr_nerf_table_scatter: needs L=16, F=2");
  NSR_REQUIRE(loss_scale > 0.f || amax != nullptr, "nsr_nerf_table_scatter: loss_scale <= 0 (automatic) needs the amax pointer");
  NSR_REQUIRE(stride >= 3, "nsr_nerf_table_scatter: stride must be >= 3");
  NSR_REQUIRE((uintptr_t)denc_h % 8 == 0, "nsr_nerf_table_scatter: denc must be 8-byte aligned");
  NSR_REQUIRE(level_begin >= 0 && level_begin <= level_end && level_end <= 16, "nsr_nerf_table_scatter: bad level range [%d, %d)", level_begin, level_end);
  if (k == 0 || level_begin == level_end) return 0;
  const int per_sm = ctas_per_sm >= 1 && ctas_per_sm <= 8 ? ctas_per_sm : 8;   // < 8 leaves room for a kernel running beside it (the exchange)
  const int grid = (int)min((int64_t)nsr_sm_count() * per_sm, (k + 255) / 256);
  nerf_table_scatter_kernel<<<k_dev ? nsr_sm_count() * per_sm : grid, 256, 0, (cudaStream_t)stream>>>(*g, xyz, stride, (const __half2*)denc_h, loss_scale,
                                                                                                  amax, grad_table, k, k_dev, level_begin, level_end);
  NSR_CHECK_LAUNCH("nsr_nerf_table_scatter");
  return 0;
}

// Split form of the same backward (packed inputs only): kernel 1 = MLP recompute + dgrad + wgrad, d(encoding) -> denc_h (fp16 [k,32],
// still multiplied by the loss scale); kernel 2 = nerf_table_scatter_kernel over the same rows (grad_dparams + NF_DENSITY_PARAMS).
extern "C" int nsr_nerf_field_bwd_split(const nsr_nerf_t* f, const void* enc_k_h, const void* dparams_h, const void* cparams_h,
                                        const float* d_sraw, const float* d_rgb, float* grad_dparams, float* grad_cparams, float loss_scale,
                                        const float* amax, int64_t k, const int64_t* k_dev, const float* xyzdir, void* denc_h, void* stream) {
  NSR_REQUIRE((uintptr_t)denc_h % 8 == 0, "nsr_nerf_field_bwd_split: denc must be 8-byte aligned");
  const int rc = field_bwd_net_launch(f, enc_k_h, dparams_h, cparams_h, d_sraw, d_rgb, grad_dparams, grad_cparams, loss_scale, amax, k, k_dev, xyzdir,
                                      denc_h, stream, "nsr_nerf_field_bwd_split");
  if (rc != 0 || k == 0) return rc;
  const int grid = (int)min((int64_t)nsr_sm_count() * 8, (k + 255) / 256);
  nerf_table_scatter_kernel<<<k_dev ? nsr_sm_count() * 8 : grid, 256, 0, (cudaStream_t)stream>>>(f->grid, xyzdir, 6, (const __half2*)denc_h, loss_scale, amax,
                                                                                                 grad_dparams + NF_DENSITY_PARAMS, k, k_dev, 0, 16);
  NSR_CHECK_LAUNCH("nsr_nerf_field_bwd_split (scatter)");
  return 0;
}
