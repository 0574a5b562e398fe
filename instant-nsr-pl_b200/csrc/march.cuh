// Sample arithmetic of the AABB lattice marcher shared by march.cu (compiled with -fmad=false) and the per-ray NeuS eval renderer
// (neus_render.cu, compiled with contraction on).  Every op is an explicit IEEE intrinsic, so both compile to the same rounding:
// the renderer's samples are the marcher's bit for bit.
#pragma once
#include "common.cuh"

namespace {

// lattice point k of a ray: t = fma(k, step, t_min); sample k spans [t(k), t(k + 1))
__device__ __forceinline__ float nsr_lattice_t(float k, float step, float t_min) { return __fmaf_rn(k, step, t_min); }

// midpoint of [t0, t1) -> world position o + d * mid (mul, then add: torch's rays_o + rays_d * midpoints)
__device__ __forceinline__ float nsr_sample_mid(float t0, float t1) { return __fmul_rn(__fadd_rn(t0, t1), 0.5f); }  // == (t0 + t1) / 2 exactly
__device__ __forceinline__ float nsr_sample_coord(float o, float d, float mid) { return __fadd_rn(o, __fmul_rn(d, mid)); }

}  // namespace
