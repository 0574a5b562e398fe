// The SDF of the fused NeuS fields on a marching-cubes lattice (VolumeSDF.forward_level over the isosurface grid: models/geometry.py
// :86-97): n_planes consecutive x-planes of the lattice ax[nx] x ay[ny] x az[nz] ('ij' order, z fastest) are evaluated straight into
// a fp32 slab [n_planes, ny, nz].  One thread per lattice point: the world point (ax[ix], ay[iy], az[iz]) -- the host's per-axis
// vectors, so the points are the torch path's bit for bit -- goes through the finite-difference field's centre query, masked hash
// encoding and SDF-only network (neus_field_fd.cuh): the arithmetic of nsr_neus_field_fd_fwd's sdf.  That is the level of every fused
// SDF geometry: the analytic HashGrid field, the ProgressiveBandHashGrid field under its level mask and the finite-difference field
// (the normal type does not enter the level).  Nothing per point is written but the level: 4 B/point against the per-op path's
// hash features, network input and 13-wide output.
#include "neus_field_fd.cuh"

namespace {

using namespace fd;

constexpr int kThreads = 128;

__global__ void __launch_bounds__(kThreads) neus_sdf_lattice_kernel(const __grid_constant__ nsr_grid_t g, const float* __restrict__ ax,
                                                                  const float* __restrict__ ay, const float* __restrict__ az, int ny, int nz,
                                                                  int ix0, const __half2* __restrict__ table, const float* __restrict__ W1,
                                                                  const float* __restrict__ b1, const float* __restrict__ W2,
                                                                  const float* __restrict__ b2, float radius, int n_out,
                                                                  const float* __restrict__ fd_state, float* __restrict__ level, int64_t n) {
  __shared__ FdW w;
  stage_weights(w, W1, b1, W2, b2, n_out);
  __syncthreads();
  const int n_active = (int)__ldg(fd_state + 2);
  const int64_t plane = (int64_t)ny * nz;
  for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
    const int ix = ix0 + (int)(i / plane);
    const int64_t r = i % plane;
    const int iy = (int)(r / nz), iz = (int)(r % nz);
    float x, y, z, e[NINP], out[1];
    stencil_query(__ldg(ax + ix), __ldg(ay + iy), __ldg(az + iz), 0, 0.f, radius, x, y, z);
    encode(g, table, x, y, z, n_active, e);
    mlp_eval<1>(w, e, out);
    level[i] = out[0];
  }
}

}  // namespace

extern "C" int nsr_neus_sdf_lattice(const nsr_grid_t* g, const float* ax, const float* ay, const float* az, int32_t nx, int32_t ny,
                                    int32_t nz, int32_t ix0, int32_t n_planes, const void* table_h, const float* W1, const float* b1,
                                    const float* W2, const float* b2, float radius, int32_t n_out, const float* fd_state, float* level,
                                    void* stream) {
  const char* name = "nsr_neus_sdf_lattice";
  NSR_REQUIRE(g != nullptr && g->n_levels == 16 && g->n_features == 2, "%s: needs a 16-level F=2 hash grid", name);
  NSR_REQUIRE(n_out >= 1 && n_out <= 16, "%s: n_out must be in [1,16]", name);
  NSR_REQUIRE(fd_state != nullptr, "%s: fd_state (device {eps, eps^2, n_active}) is NULL", name);
  NSR_REQUIRE(ax != nullptr && ay != nullptr && az != nullptr && table_h != nullptr && W1 != nullptr && b1 != nullptr && W2 != nullptr &&
                  b2 != nullptr && level != nullptr,
              "%s: NULL argument", name);
  NSR_REQUIRE(nx >= 1 && ny >= 1 && nz >= 1, "%s: empty lattice (%d x %d x %d)", name, nx, ny, nz);
  NSR_REQUIRE(n_planes >= 1 && ix0 >= 0 && ix0 + (int64_t)n_planes <= nx, "%s: planes [%d, %d + %d) outside [0, %d)", name, ix0, ix0,
              n_planes, nx);
  const int64_t n = (int64_t)n_planes * ny * nz;
  const int grid = (int)min((int64_t)nsr_sm_count() * 8, (n + kThreads - 1) / kThreads);
  neus_sdf_lattice_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(*g, ax, ay, az, ny, nz, ix0, (const __half2*)table_h, W1, b1, W2, b2,
                                                                       radius, n_out, fd_state, level, n);
  NSR_CHECK_LAUNCH(name);
  return 0;
}
