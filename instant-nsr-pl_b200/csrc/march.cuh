// Sample arithmetic of the marchers shared by march.cu (compiled with -fmad=false) and the per-ray eval renderers (neus_render.cu,
// nerf_rays_fwd.cu, compiled with contraction on).  Every op is an explicit IEEE intrinsic, so both compile to the same rounding:
// the renderers' samples are the marcher's bit for bit.
#pragma once
#include "common.cuh"

namespace {

// lattice point k of a ray: t = fma(k, step, t_min); sample k spans [t(k), t(k + 1))
__device__ __forceinline__ float nsr_lattice_t(float k, float step, float t_min) { return __fmaf_rn(k, step, t_min); }

// midpoint of [t0, t1) -> world position o + d * mid (mul, then add: torch's rays_o + rays_d * midpoints)
__device__ __forceinline__ float nsr_sample_mid(float t0, float t1) { return __fmul_rn(__fadd_rn(t0, t1), 0.5f); }  // == (t0 + t1) / 2 exactly
__device__ __forceinline__ float nsr_sample_coord(float o, float d, float mid) { return __fadd_rn(o, __fmul_rn(d, mid)); }

// cone marcher (cone_angle > 0): one step of the recurrence t1 = t0 + min(max(t0 * cone, step), 1e10).  Each step depends on the one
// before, so the chain is never reassociated.
__device__ __forceinline__ float nsr_cone_next(float t0, float cone, float step) {
  return __fadd_rn(t0, fminf(fmaxf(__fmul_rn(t0, cone), step), 1e10f));
}

// advance the chain by the 32 steps of one mask word from t (the word's first t); lane `lane` receives its step [t0, t1).  Every lane runs
// the same chain; the return value is the next word's first t.
__device__ __forceinline__ float nsr_cone_chunk(float t, float cone, float step, int lane, float& t0, float& t1) {
#pragma unroll
  for (int k = 0; k < 32; ++k) {
    const float tn = nsr_cone_next(t, cone, step);
    if (k == lane) {
      t0 = t;
      t1 = tn;
    }
    t = tn;
  }
  return t;
}

}  // namespace
