// Hopper warpgroup MMA (wgmma.mma_async, sm_90a) helpers shared by the tensor-core kernels (mlp_tc.cu, nerf_bwd_tc.cu, nerf_fused_bwd.cu).
//
// Operands live in shared memory in the canonical no-swizzle layout: 8 x 16-byte core matrices.
//   K-major  [rows][K] tile (K contiguous): LBO = byte distance between the two 8-wide K chunks of one k16 step, SBO = distance between
//            8-row groups.
//   MN-major the same physical tile read with M / N along its contiguous dimension: SBO = distance between 8-column chunks, LBO =
//            distance between 8-row k groups.
// The accumulator of one m64nNk16 instruction is N / 2 fp32 registers per thread of the warpgroup: register 4 j + 2 h + e holds
// row 16 * warp + lane / 4 + 8 h, column 8 j + 2 (lane % 4) + e.
#pragma once
#include <stdint.h>

__device__ __forceinline__ uint32_t nsr_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// canonical K-major no-swizzle layout: byte offset of element (row, k) of a [rows][K] fp16 tile
__device__ __forceinline__ int nsr_canon_off(int row, int k, int K) { return ((row >> 3) * (K >> 3) + (k >> 3)) * 128 + (row & 7) * 16 + (k & 7) * 2; }

// 64-bit wgmma shared-memory matrix descriptor: start >> 4 @0, LBO >> 4 @16, SBO >> 4 @32, base offset 0, layout type 0 (no swizzle) @62
__device__ __forceinline__ uint64_t nsr_wg_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) | ((uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32);
}

// MN-major descriptor of a canonical [k rows][C] tile read with M / N along C, k16 step kk: SBO = 128 B (8-column chunks), LBO = (C/8)*128 B
// (8-row k groups); step kk starts 2 LBO further
__device__ __forceinline__ uint64_t nsr_wg_desc_mn(uint32_t addr, int C, int kk) {
  return nsr_wg_desc(addr + 2u * (uint32_t)(C / 8) * 128u * (uint32_t)kk, (uint32_t)(C / 8) * 128u, 128u);
}

__device__ __forceinline__ void nsr_wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void nsr_wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void nsr_wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// generic-proxy shared-memory writes -> visible to the tensor core (async proxy); followed by a barrier
__device__ __forceinline__ void nsr_proxy_fence() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// shared-memory mbarriers (addresses from nsr_smem_u32)
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
// bounded wait: a barrier that is never signalled (a bug) sets *status (if given) and traps instead of hanging the GPU
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, int* status, int code) {
  const long long t0 = clock64();
  for (;;) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}\n"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    if (ok) return;
    if (clock64() - t0 > 4000000000ll) {
      if (status) atomicExch(status, code);
      __trap();
    }
  }
}

// after nsr_wg_wait0: no read of the accumulator registers may be scheduled in front of the wait
template <int R>
__device__ __forceinline__ void nsr_wg_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] * B[16 x N], fp16 operands from shared memory, fp32 accumulate.  TA / TB: 0 = K-major, 1 = MN-major.
template <int TA, int TB>
__device__ __forceinline__ void nsr_wgmma_n16(float (&d)[8], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB)
      : "memory");
}

template <int TA, int TB>
__device__ __forceinline__ void nsr_wgmma_n32(float (&d)[16], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]),
        "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB)
      : "memory");
}

template <int TA, int TB>
__device__ __forceinline__ void nsr_wgmma_n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, "
      "%18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]),
        "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]),
        "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]),
        "+f"(d[31])
      : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB)
      : "memory");
}

// dispatch on N (16 / 32 / 64) for code that is generic over the layer width
template <int N, int TA, int TB>
__device__ __forceinline__ void nsr_wgmma(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t accumulate) {
  if constexpr (N == 16) nsr_wgmma_n16<TA, TB>(d, da, db, accumulate);
  else if constexpr (N == 32) nsr_wgmma_n32<TA, TB>(d, da, db, accumulate);
  else nsr_wgmma_n64<TA, TB>(d, da, db, accumulate);
}

// Register-A form: D[64 x N] (+)= A[64 x 16] * B[16 x N], A from registers, B from shared memory.  Each warp of the warpgroup holds
// its 16 rows of A in the mma.sync m16n8k16 A-fragment layout (a[0]: row g, columns 2c..2c+1; a[1]: row g+8; a[2], a[3]: the same
// rows, columns + 8); the accumulator has the layout above, which is the m16n8 C-fragment layout of each warp's 16 rows.  A registers
// written since the last wgmma need an nsr_wg_fence in front.  TB: 0 = K-major, 1 = MN-major.
template <int TB>
__device__ __forceinline__ void nsr_wgmma_rs_n16(float (&d)[8], const uint32_t (&a)[4], uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %13, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1, %14;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate), "n"(TB)
      : "memory");
}

template <int TB>
__device__ __forceinline__ void nsr_wgmma_rs_n32(float (&d)[16], const uint32_t (&a)[4], uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "{%16, %17, %18, %19}, %20, p, 1, 1, %22;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]),
        "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate), "n"(TB)
      : "memory");
}

template <int TB>
__device__ __forceinline__ void nsr_wgmma_rs_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, "
      "%18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, %38;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]),
        "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]),
        "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]),
        "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate), "n"(TB)
      : "memory");
}

template <int N, int TB>
__device__ __forceinline__ void nsr_wgmma_rs(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t db, uint32_t accumulate) {
  if constexpr (N == 16) nsr_wgmma_rs_n16<TB>(d, a, db, accumulate);
  else if constexpr (N == 32) nsr_wgmma_rs_n32<TB>(d, a, db, accumulate);
  else nsr_wgmma_rs_n64<TB>(d, a, db, accumulate);
}
