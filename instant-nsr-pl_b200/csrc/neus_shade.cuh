// NeuS SDF -> alpha terms (see neus_shade.cu), shared by the per-sample alpha kernels and the per-ray eval renderer (neus_render.cu).
#pragma once
#include "common.cuh"

namespace {

struct AlphaTerms {
  float nx, ny, nz, inv_norm, true_cos, iter_cos, dist, prev, next, pc, nc, q;
};

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

__device__ __forceinline__ AlphaTerms alpha_terms(float sdf, float gx, float gy, float gz, float dx, float dy, float dz, float dist, float s,
                                                  float a) {
  AlphaTerms t;
  const float nrm = fmaxf(sqrtf(gx * gx + gy * gy + gz * gz), 1e-12f);
  t.inv_norm = 1.f / nrm;
  t.nx = gx * t.inv_norm;
  t.ny = gy * t.inv_norm;
  t.nz = gz * t.inv_norm;
  t.true_cos = dx * t.nx + dy * t.ny + dz * t.nz;
  t.iter_cos = -(fmaxf(-t.true_cos * 0.5f + 0.5f, 0.f) * (1.f - a) + fmaxf(-t.true_cos, 0.f) * a);
  t.dist = dist;
  const float h = t.iter_cos * dist * 0.5f;
  t.prev = sdf - h;
  t.next = sdf + h;
  t.pc = sigmoidf_(t.prev * s);
  t.nc = sigmoidf_(t.next * s);
  t.q = (t.pc - t.nc + 1e-5f) / (t.pc + 1e-5f);
  return t;
}

}  // namespace
