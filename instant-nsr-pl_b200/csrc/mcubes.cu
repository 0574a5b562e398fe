// Isosurface extraction on the GPU (SURVEY 8f-4: models/geometry.py:32-112 -- the reference sweeps the level field on the GPU in
// 2 M-point chunks, copies 512^3 floats to the host and runs PyMCubes on one CPU core).  Here the field never leaves HBM:
//   count    : one thread per grid point: which of its three owned edges (+x, +y, +z) cross the iso-value, how many triangles its
//              cell emits (case table mc_table.inc, generated hole-free by mc_table.py); per-block totals
//   scan     : exclusive scan of the per-block totals (one CTA) -> block offsets, totals (V, F)
//   vertices : recompute the flags, block-level scan -> global vertex ids in (point, axis) order; interpolated positions;
//              vid_map[point] = first vertex id | crossing flags << 29
//   faces    : recompute the case, block-level scan -> triangle slots in (cell, table) order; vertex ids through vid_map
// Field layout [nx, ny, nz], z fastest (torch.meshgrid(indexing='ij').reshape(-1): geometry.py:46-52).  Every pass is a coalesced
// stream over the field (4 B/point; the +y / +x neighbour rows come from L1 / L2), i.e. HBM-bound integer work; nothing is sorted
// and no atomics are used, so vertex and face order are deterministic.
// Slabs: x is the slowest axis, so the planes [a, b) taken in order reproduce the dense (point, axis) vertex order and (cell, table)
// face order.  A slab emits the vertices of the points and the faces of the cells whose x index is in [a, b); its field buffer holds
// the planes [a, min(b + 1, nx - 1)].  The faces of cells on plane b - 1 look up vertex ids on plane b, whose +x flags read plane b + 1:
// plane b is scanned as a TAIL after the slab's own points (its own CTAs, so the slab's vertex count is a block offset) and gets
// vid_map entries but emits nothing.  Vertex ids in vid_map are slab-local (plane b's continue after the slab's last vertex, which is
// where the next slab's numbering starts); faces add the 64-bit vertex base.  The dense grid is the one slab [0, nx) with no tail.
#include "common.cuh"
#include "mc_table.inc"

namespace {

constexpr int kThreads = 256;

struct McDims {
  int32_t nx, ny, nz;  // the whole grid
  int32_t ix0;         // x index of the buffer's first plane (the slab's a)
  int64_t n;           // the slab's own points: (b - a) * ny * nz
  int64_t n_all;       // n + the tail plane's points (0 or ny * nz)
  int64_t nb_main;     // CTAs over the slab's own points; the tail's CTAs follow
};

__device__ __forceinline__ float mc_value(const float* __restrict__ f, int64_t i, int negate) {
  const float v = __ldg(f + i);
  return negate ? -v : v;
}

// crossing flags of the three edges owned by point (ix, iy, iz) (bit a: edge along axis a crosses) and the case index of the cell
// whose minimum corner it is (-1: no such cell); v0 = value at the point
__device__ __forceinline__ void mc_point(const float* __restrict__ f, const McDims& d, int64_t idx, int ix, int iy, int iz, float iso, int negate,
                                         int& vflags, int& cell_case, float (&edge_b)[3], float& v0) {
  const int64_t sx = (int64_t)d.ny * d.nz, sy = d.nz;
  const bool hx = ix + 1 < d.nx, hy = iy + 1 < d.ny, hz = iz + 1 < d.nz;
  v0 = mc_value(f, idx, negate);
  const bool in0 = v0 > iso;
  vflags = 0;
  cell_case = -1;
  float v[8];
  v[0] = v0;
  v[1] = hx ? mc_value(f, idx + sx, negate) : v0;
  v[2] = hy ? mc_value(f, idx + sy, negate) : v0;
  v[4] = hz ? mc_value(f, idx + 1, negate) : v0;
  edge_b[0] = v[1], edge_b[1] = v[2], edge_b[2] = v[4];
  if (hx && ((v[1] > iso) != in0)) vflags |= 1;
  if (hy && ((v[2] > iso) != in0)) vflags |= 2;
  if (hz && ((v[4] > iso) != in0)) vflags |= 4;
  if (hx && hy && hz) {
    v[3] = mc_value(f, idx + sx + sy, negate);
    v[5] = mc_value(f, idx + sx + 1, negate);
    v[6] = mc_value(f, idx + sy + 1, negate);
    v[7] = mc_value(f, idx + sx + sy + 1, negate);
    int c = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) c |= (v[k] > iso) ? (1 << k) : 0;
    cell_case = c;
  }
}

// buffer index of this thread's point (the slab's own points, then the tail plane's), -1 past either range
__device__ __forceinline__ int64_t mc_index(const McDims& d) {
  const int64_t blk = blockIdx.x;
  if (blk < d.nb_main) {
    const int64_t idx = blk * kThreads + threadIdx.x;
    return idx < d.n ? idx : -1;
  }
  const int64_t idx = d.n + (blk - d.nb_main) * kThreads + threadIdx.x;
  return idx < d.n_all ? idx : -1;
}

// grid coordinates of buffer index idx (ix global: the buffer starts at plane ix0)
__device__ __forceinline__ void mc_coords(const McDims& d, int64_t idx, int& ix, int& iy, int& iz) {
  iz = (int)(idx % d.nz);
  const int64_t q = idx / d.nz;
  iy = (int)(q % d.ny);
  ix = (int)(q / d.ny) + d.ix0;
}

// exclusive scan of one int per thread over the 256-thread block; returns the exclusive prefix, total in `total`
__device__ __forceinline__ int block_exclusive_scan(int v, int& total) {
  __shared__ int warp_sums[kThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  __syncthreads();  // the previous call's readers of warp_sums are done
  if (lane == 31) warp_sums[warp] = inc;
  __syncthreads();
  int base = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < kThreads / 32; ++w) {
    const int s = warp_sums[w];
    if (w < warp) base += s;
    tot += s;
  }
  total = tot;
  return base + inc - v;
}

__global__ void __launch_bounds__(kThreads) mc_count_kernel(const float* __restrict__ f, McDims d, float iso, int negate, int32_t* __restrict__ block_v,
                                                            int32_t* __restrict__ block_t) {
  const int64_t idx = mc_index(d);
  int nv = 0, nt = 0;
  if (idx >= 0) {
    int ix, iy, iz, vflags, cc;
    float eb[3], v0;
    mc_coords(d, idx, ix, iy, iz);
    mc_point(f, d, idx, ix, iy, iz, iso, negate, vflags, cc, eb, v0);
    nv = __popc(vflags);
    nt = (cc >= 0 && idx < d.n) ? kMcNumTris[cc] : 0;  // the tail plane's cells belong to the next slab
  }
  int tv, tt;
  block_exclusive_scan(nv, tv);
  block_exclusive_scan(nt, tt);
  if (threadIdx.x == 0) block_v[blockIdx.x] = tv, block_t[blockIdx.x] = tt;
}

// in-place exclusive scan of two int32 arrays of n_blocks entries by ONE 1024-thread CTA (n_blocks = points / 256: 524 k at 512^3);
// totals[0] = vertices before block nb_main (the slab's own; the tail plane's follow), totals[1] = triangles
__global__ void __launch_bounds__(1024) mc_scan_kernel(int32_t* __restrict__ block_v, int32_t* __restrict__ block_t, int64_t n_blocks,
                                                       int64_t nb_main, int64_t* __restrict__ totals) {
  __shared__ int64_t part[2][1024];
  const int t = threadIdx.x;
  const int64_t chunk = (n_blocks + 1023) / 1024, lo = min((int64_t)t * chunk, n_blocks), hi = min(lo + chunk, n_blocks);
  int64_t sv = 0, st = 0;
  for (int64_t i = lo; i < hi; ++i) sv += block_v[i], st += block_t[i];
  part[0][t] = sv, part[1][t] = st;
  __syncthreads();
  if (t < 2) {  // 1024 partial sums per array: a serial pass by one thread each is ~1 us
    int64_t run = 0;
    for (int i = 0; i < 1024; ++i) {
      const int64_t s = part[t][i];
      part[t][i] = run;
      run += s;
    }
    totals[t] = run;
  }
  __syncthreads();
  int64_t rv = part[0][t], rt = part[1][t];
  for (int64_t i = lo; i < hi; ++i) {
    const int32_t a = block_v[i], b = block_t[i];
    if (i == nb_main) totals[0] = rv;  // a tail follows: the slab's own vertices end here
    block_v[i] = (int32_t)rv, block_t[i] = (int32_t)rt;
    rv += a, rt += b;
  }
}

struct McXform {
  float lo[3], ext[3], denom[3];  // world = (index_coordinate / denom) * ext + lo   (geometry.py:65,99-103)
};

__global__ void __launch_bounds__(kThreads) mc_vertices_kernel(const float* __restrict__ f, McDims d, float iso, int negate, McXform X,
                                                               const int32_t* __restrict__ block_v, int32_t* __restrict__ vid_map,
                                                               float* __restrict__ verts, int64_t n_verts) {
  const int64_t idx = mc_index(d);
  int ix = 0, iy = 0, iz = 0, vflags = 0, cc;
  float eb[3] = {0.f, 0.f, 0.f}, v0 = 0.f;
  if (idx >= 0) {
    mc_coords(d, idx, ix, iy, iz);
    mc_point(f, d, idx, ix, iy, iz, iso, negate, vflags, cc, eb, v0);
  }
  int total;
  const int base = block_v[blockIdx.x] + block_exclusive_scan(__popc(vflags), total);
  if (idx < 0) return;
  vid_map[idx] = (int32_t)((uint32_t)base | ((uint32_t)vflags << 29));
  if (idx >= d.n) return;  // tail plane: ids only, its vertices are the next slab's
  int k = 0;
  const float p[3] = {(float)ix, (float)iy, (float)iz};
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    if (!((vflags >> a) & 1)) continue;
    const int64_t vid = base + k++;
    if (vid >= n_verts) continue;  // the field changed between count and emit: never write outside the caller's buffer
    const float t = __fdiv_rn(__fsub_rn(iso, v0), __fsub_rn(eb[a], v0));  // linear interpolation along the edge
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float g = c == a ? __fadd_rn(p[c], t) : p[c];
      verts[vid * 3 + c] = __fadd_rn(__fmul_rn(__fdiv_rn(g, X.denom[c]), X.ext[c]), X.lo[c]);
    }
  }
}

__global__ void __launch_bounds__(kThreads) mc_faces_kernel(const float* __restrict__ f, McDims d, float iso, int negate,
                                                            const int32_t* __restrict__ block_t, const int32_t* __restrict__ vid_map,
                                                            int64_t* __restrict__ faces, int64_t n_faces, int64_t vbase) {
  const int64_t idx = mc_index(d);
  int ix = 0, iy = 0, iz = 0, vflags, cc = -1;
  float eb[3], v0;
  if (idx >= 0 && idx < d.n) {  // the tail's CTAs come after every face slot of the slab: no scan of theirs reaches a face
    mc_coords(d, idx, ix, iy, iz);
    mc_point(f, d, idx, ix, iy, iz, iso, negate, vflags, cc, eb, v0);
  }
  const int nt = cc >= 0 ? kMcNumTris[cc] : 0;
  int total;
  const int64_t base = block_t[blockIdx.x] + block_exclusive_scan(nt, total);
  if (nt == 0) return;
  const int64_t sx = (int64_t)d.ny * d.nz, sy = d.nz;
  for (int t = 0; t < nt; ++t) {
    const int64_t slot = base + t;
    if (slot >= n_faces) return;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const int e = kMcTris[cc][3 * t + j], axis = e >> 2, k = e & 3, a = k & 1, b = k >> 1;
      // owner corner of edge e: axis 0: (0, a, b), axis 1: (a, 0, b), axis 2: (a, b, 0)
      const int ox = axis == 0 ? 0 : a, oy = axis == 0 ? a : (axis == 1 ? 0 : b), oz = axis == 2 ? 0 : b;
      const uint32_t entry = (uint32_t)__ldg(vid_map + idx + ox * sx + oy * sy + oz);
      const uint32_t flags = entry >> 29;
      faces[slot * 3 + j] = vbase + (int64_t)((entry & 0x1fffffffu) + __popc(flags & ((1u << axis) - 1u)));
    }
  }
}

int check_dims(const char* who, int32_t nx, int32_t ny, int32_t nz, int32_t a, int32_t b) {
  NSR_REQUIRE(nx >= 2 && ny >= 2 && nz >= 2, "%s: the field needs at least 2 points per axis (got %d x %d x %d)", who, nx, ny, nz);
  NSR_REQUIRE(0 <= a && a < b && b <= nx, "%s: plane range [%d, %d) is not a non-empty part of [0, %d)", who, a, b, nx);
  NSR_REQUIRE((int64_t)(b - a + (b < nx)) * ny * nz <= ((int64_t)1 << 33), "%s: field too large", who);
  return 0;
}

// the slab [a, b) of an nx x ny x nz grid (see the top of the file); *nb = CTAs of every pass (block_offsets holds 2 * nb entries)
McDims slab_dims(int32_t nx, int32_t ny, int32_t nz, int32_t a, int32_t b, int64_t* nb) {
  const int64_t plane = (int64_t)ny * nz, n = (b - a) * plane, tail = b < nx ? plane : 0;
  const int64_t nb_main = (n + kThreads - 1) / kThreads;
  *nb = nb_main + (tail + kThreads - 1) / kThreads;
  return McDims{nx, ny, nz, a, n, n + tail, nb_main};
}

int mc_count(const char* who, const float* field, int32_t nx, int32_t ny, int32_t nz, int32_t a, int32_t b, float iso, int32_t negate,
             int32_t* block_offsets, int64_t* totals, void* stream) {
  if (int e = check_dims(who, nx, ny, nz, a, b)) return e;
  NSR_REQUIRE(field != nullptr && block_offsets != nullptr && totals != nullptr, "%s: NULL argument", who);
  int64_t nb;
  const McDims d = slab_dims(nx, ny, nz, a, b, &nb);
  mc_count_kernel<<<(unsigned)nb, kThreads, 0, (cudaStream_t)stream>>>(field, d, iso, negate, block_offsets, block_offsets + nb);
  NSR_CHECK_LAUNCH(who);
  mc_scan_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(block_offsets, block_offsets + nb, nb, d.nb_main, totals);
  NSR_CHECK_LAUNCH(who);
  return 0;
}

int mc_emit(const char* who, const float* field, int32_t nx, int32_t ny, int32_t nz, int32_t a, int32_t b, float iso, int32_t negate,
            const int32_t* block_offsets, const float* lo, const float* hi, int32_t* vid_map, float* verts, int64_t n_verts, int64_t* faces,
            int64_t n_faces, int64_t vbase, void* stream) {
  if (int e = check_dims(who, nx, ny, nz, a, b)) return e;
  NSR_REQUIRE(field != nullptr && block_offsets != nullptr && vid_map != nullptr, "%s: NULL argument", who);
  NSR_REQUIRE(lo != nullptr && hi != nullptr, "%s: bounding box is NULL (host float[3] each)", who);
  NSR_REQUIRE((n_verts == 0 || verts != nullptr) && (n_faces == 0 || faces != nullptr), "%s: output buffer is NULL", who);
  int64_t nb;
  const McDims d = slab_dims(nx, ny, nz, a, b, &nb);
  // vid_map ids run on through the tail plane (at most 3 vertices per point)
  NSR_REQUIRE(n_verts + 3 * (d.n_all - d.n) < ((int64_t)1 << 29), "%s: more than 2^29 vertices", who);
  NSR_REQUIRE(n_faces < ((int64_t)1 << 31) && vbase >= 0, "%s: more than 2^31 faces or a negative vertex base", who);
  McXform X;
  const int32_t dims[3] = {nx, ny, nz};
  for (int c = 0; c < 3; ++c) X.lo[c] = lo[c], X.ext[c] = hi[c] - lo[c], X.denom[c] = (float)(dims[c] - 1);
  mc_vertices_kernel<<<(unsigned)nb, kThreads, 0, (cudaStream_t)stream>>>(field, d, iso, negate, X, block_offsets, vid_map, verts, n_verts);
  NSR_CHECK_LAUNCH(who);
  if (n_faces > 0) {
    mc_faces_kernel<<<(unsigned)nb, kThreads, 0, (cudaStream_t)stream>>>(field, d, iso, negate, block_offsets + nb, vid_map, faces, n_faces,
                                                                        vbase);
    NSR_CHECK_LAUNCH(who);
  }
  return 0;
}

}  // namespace

extern "C" int nsr_mc_count(const float* field, int32_t nx, int32_t ny, int32_t nz, float iso, int32_t negate, int32_t* block_offsets,
                            int64_t* totals, void* stream) {
  return mc_count("nsr_mc_count", field, nx, ny, nz, 0, nx, iso, negate, block_offsets, totals, stream);
}

extern "C" int nsr_mc_emit(const float* field, int32_t nx, int32_t ny, int32_t nz, float iso, int32_t negate, const int32_t* block_offsets,
                           const float* lo, const float* hi, int32_t* vid_map, float* verts, int64_t n_verts, int64_t* faces,
                           int64_t n_faces, void* stream) {
  return mc_emit("nsr_mc_emit", field, nx, ny, nz, 0, nx, iso, negate, block_offsets, lo, hi, vid_map, verts, n_verts, faces, n_faces, 0,
                 stream);
}

extern "C" int nsr_mc_count_slab(const float* field, int32_t nx, int32_t ny, int32_t nz, int32_t a, int32_t b, float iso, int32_t negate,
                                 int32_t* block_offsets, int64_t* totals, void* stream) {
  return mc_count("nsr_mc_count_slab", field, nx, ny, nz, a, b, iso, negate, block_offsets, totals, stream);
}

extern "C" int nsr_mc_emit_slab(const float* field, int32_t nx, int32_t ny, int32_t nz, int32_t a, int32_t b, float iso, int32_t negate,
                                const int32_t* block_offsets, const float* lo, const float* hi, int32_t* vid_map, float* verts,
                                int64_t n_verts, int64_t* faces, int64_t n_faces, int64_t vbase, void* stream) {
  return mc_emit("nsr_mc_emit_slab", field, nx, ny, nz, a, b, iso, negate, block_offsets, lo, hi, vid_map, verts, n_verts, faces, n_faces,
                 vbase, stream);
}
