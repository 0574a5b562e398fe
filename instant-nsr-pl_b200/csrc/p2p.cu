// Gradient all-reduce (mean) over NVLink peer memory -- the one exchange step of the data-parallel path (SURVEY 8e: what the
// reference gets from Lightning DDP / NCCL, launch.py:98).  Every rank's flat gradient buffer lives in symmetric memory (same
// size, peer-mapped); after the backward
//     barrier  -> every rank's gradients are complete and visible
//     reduce   -> rank r owns chunk r: it sums the chunk over all peers (P2P loads, or ONE multimem.ld_reduce when the buffer has
//                 an NVSwitch multicast mapping: the switch adds the replicas), scales by 1/world and writes the result straight
//                 into every peer's buffer (P2P stores / multimem.st): reduce-scatter and all-gather in one kernel, in place
//     barrier  -> all chunks have landed everywhere
// Chunks are disjoint, so the in-place update is race free.  Barriers are monotonically increasing epochs in a peer-mapped flag
// array (st.release.sys / ld.acquire.sys), with a bounded spin so that a lost peer sets an error flag instead of hanging the GPU.
#include <stdlib.h>
#include "common.cuh"

namespace {

constexpr int kMaxWorld = 16;
constexpr long long kSpinLimit = 1LL << 28;  // ~ a few seconds of polling

// flags layout (int32, per rank, peer-mapped): flags[p] = last epoch signalled by rank p
struct FlagPeers {
  int32_t* p[kMaxWorld];
};

__global__ void p2p_barrier_kernel(const FlagPeers flags, int32_t* __restrict__ epoch, int32_t* __restrict__ err, int rank, int world) {
  __shared__ int e_s;
  if (threadIdx.x == 0) e_s = atomicAdd(epoch, 1) + 1;
  __syncthreads();
  const int e = e_s, p = threadIdx.x;
  if (p < world) {
    __threadfence_system();
    int32_t* dst = flags.p[p] + rank;
    asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(dst), "r"(e) : "memory");
    const int32_t* src = flags.p[rank] + p;
    long long spins = 0;
    int v;
    do {
      asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(src) : "memory");
    } while (v - e < 0 && ++spins < kSpinLimit);
    if (v - e < 0) atomicExch(err, 1);
  }
}

struct Peers {
  float4* p[kMaxWorld];
};

// U independent float4 columns per thread per iteration: all world x U remote loads are in flight before the first add
// (NVLink round trips are ~2-3 us; one load per thread leaves the links mostly idle)
template <int U>
__global__ void __launch_bounds__(256) p2p_allreduce_mean_kernel(const Peers peers, int rank, int world, int64_t n4, float inv) {
  const int64_t chunk = (n4 + world - 1) / world;
  const int64_t lo = rank * chunk, hi = min(n4, lo + chunk);
  const int64_t span = 256ll * U;
  for (int64_t base = lo + blockIdx.x * span; base < hi; base += (int64_t)gridDim.x * span) {
    float4 acc[U];
#pragma unroll
    for (int u = 0; u < U; ++u) acc[u] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int q = 0; q < kMaxWorld; ++q) {
      if (q < world) {  // fixed summation order 0..world-1; the owner broadcasts ONE result, so all replicas stay bit-identical
        float4 v[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int64_t i = base + u * 256 + threadIdx.x;
          // never from a stale cache line: peers wrote this memory over NVLink
          v[u] = i < hi ? __ldcv(peers.p[q] + i) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          acc[u].x += v[u].x;
          acc[u].y += v[u].y;
          acc[u].z += v[u].z;
          acc[u].w += v[u].w;
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = base + u * 256 + threadIdx.x;
      if (i < hi) {
        const float4 r = make_float4(acc[u].x * inv, acc[u].y * inv, acc[u].z * inv, acc[u].w * inv);
#pragma unroll
        for (int q = 0; q < kMaxWorld; ++q)
          if (q < world) peers.p[q][i] = r;
      }
    }
  }
}

// NVSwitch multicast variant: the switch reduces the replicas on the load and broadcasts the store
__global__ void __launch_bounds__(256) p2p_allreduce_mean_multimem_kernel(float* __restrict__ mc, int rank, int world, int64_t n4, float inv) {
  const int64_t chunk = (n4 + world - 1) / world;
  const int64_t lo = rank * chunk, hi = min(n4, lo + chunk);
  for (int64_t i = lo + blockIdx.x * 256ll + threadIdx.x; i < hi; i += (int64_t)gridDim.x * 256) {
    float4 v;
    float* a = mc + i * 4;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "l"(a)
                 : "memory");
    v.x *= inv;
    v.y *= inv;
    v.z *= inv;
    v.w *= inv;
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(a), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
  }
}

// ---- one-launch exchange: entry barrier + reduce-scatter + all-gather + exit barrier in ONE kernel ------------------------------------
// (The step's backward accumulates straight into the symmetric buffer, so this kernel is the whole exchange: no separate barrier
//  launches and no 50 MB copy-in.)
//   entry : CTA 0 publishes "rank's gradients are complete" (epoch e) into every peer's flag array; EVERY CTA waits until all peers have
//           published e (their backward kernels are behind them) -- no grid-wide sync needed, each CTA polls the local flags itself
//   data  : rank r owns chunk r; U 16-byte columns per thread are in flight before the first is consumed
//             multicast: multimem.ld_reduce (the NVSwitch adds the replicas) -> scale -> multimem.st (the switch broadcasts)
//             P2P      : ld.cv from every peer in rank order -> scale -> st to every peer
//   exit  : every CTA fences its stores; the LAST CTA to finish (self-resetting counter) publishes "rank r is done reading and writing"
//           and waits for the same from every peer, so kernel completion == every replica holds the complete mean and nobody still reads
//           this rank's buffer (the next step may zero it).  The epoch lives in device memory => CUDA-graph replay safe.
constexpr int kChannelSlot0 = 32, kChannelSlots = 32;   // flag slots of channel c: [32 + 32 c, 64 + 32 c)
struct XchgArgs {
  float4* peer[kMaxWorld];
  int32_t* flags[kMaxWorld];  // int32[256] per rank; [0, 16) belongs to nsr_p2p_barrier, channel c of this kernel owns [32 + 32 c, 64 + 32 c)
  float* mc;
  int32_t* epoch;    // last completed exchange
  int32_t* counter;  // CTAs that finished their share (returns to 0)
  int32_t* err;
  int rank, world;
  int64_t n4;   // float4 elements of the range
  int64_t o4;   // first float4 of the range
  int slot;     // first flag slot of the channel: entry epochs [slot, slot + 16), exit epochs [slot + 16, slot + 32)
  float inv;
};

__device__ __forceinline__ void xchg_signal_wait(const XchgArgs& a, int slot0, int e) {
  const int p = threadIdx.x;
  if (p < a.world) {
    int32_t* dst = a.flags[p] + slot0 + a.rank;
    asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(dst), "r"(e) : "memory");
  }
}
__device__ __forceinline__ void xchg_wait(const XchgArgs& a, int slot0, int e) {
  const int p = threadIdx.x;
  if (p < a.world) {
    const int32_t* src = a.flags[a.rank] + slot0 + p;
    long long spins = 0;
    int v;
    do {
      asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(src) : "memory");
    } while (v - e < 0 && ++spins < kSpinLimit);
    if (v - e < 0) atomicExch(a.err, 1);
  }
}

template <int U, bool MC>
__global__ void __launch_bounds__(256, U <= 4 ? 4 : (U <= 8 ? 2 : 1)) p2p_exchange_kernel(const XchgArgs a) {
  __shared__ int s_last;
  const int e = *reinterpret_cast<volatile int32_t*>(a.epoch) + 1;  // every CTA reads it before the last one to finish advances it
  if (blockIdx.x == 0) {
    __threadfence_system();
    xchg_signal_wait(a, a.slot, e);
  }
  xchg_wait(a, a.slot, e);
  __syncthreads();
  const int64_t chunk = (a.n4 + a.world - 1) / a.world;
  const int64_t lo = a.o4 + a.rank * chunk, hi = a.o4 + min(a.n4, (a.rank + 1) * chunk);
  const int64_t span = 256ll * U;
  for (int64_t base = lo + blockIdx.x * span; base < hi; base += (int64_t)gridDim.x * span) {
    float4 acc[U];
    if (MC) {
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t i = base + u * 256 + threadIdx.x;
        acc[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (i < hi)
          asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
                       : "=f"(acc[u].x), "=f"(acc[u].y), "=f"(acc[u].z), "=f"(acc[u].w)
                       : "l"(a.mc + i * 4)
                       : "memory");
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t i = base + u * 256 + threadIdx.x;
        if (i < hi)
          asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(a.mc + i * 4), "f"(acc[u].x * a.inv),
                       "f"(acc[u].y * a.inv), "f"(acc[u].z * a.inv), "f"(acc[u].w * a.inv)
                       : "memory");
      }
    } else {
#pragma unroll
      for (int u = 0; u < U; ++u) acc[u] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int q = 0; q < kMaxWorld; ++q) {
        if (q < a.world) {  // fixed summation order 0..world-1; the owner broadcasts ONE result, so all replicas stay bit-identical
          float4 v[U];
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const int64_t i = base + u * 256 + threadIdx.x;
            v[u] = i < hi ? __ldcv(a.peer[q] + i) : make_float4(0.f, 0.f, 0.f, 0.f);
          }
#pragma unroll
          for (int u = 0; u < U; ++u) {
            acc[u].x += v[u].x;
            acc[u].y += v[u].y;
            acc[u].z += v[u].z;
            acc[u].w += v[u].w;
          }
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t i = base + u * 256 + threadIdx.x;
        if (i < hi) {
          const float4 r = make_float4(acc[u].x * a.inv, acc[u].y * a.inv, acc[u].z * a.inv, acc[u].w * a.inv);
#pragma unroll
          for (int q = 0; q < kMaxWorld; ++q)
            if (q < a.world) a.peer[q][i] = r;
        }
      }
    }
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(a.counter, 1) == (int)gridDim.x - 1;
  __syncthreads();
  if (s_last) {
    __threadfence_system();
    xchg_signal_wait(a, a.slot + kMaxWorld, e);
    xchg_wait(a, a.slot + kMaxWorld, e);
    __syncthreads();
    if (threadIdx.x == 0) {
      *a.counter = 0;
      *a.epoch = e;
    }
  }
}

}  // namespace

extern "C" int nsr_p2p_barrier(const uint64_t* flag_ptrs_host, int32_t* epoch_dev, int32_t* err_dev, int32_t rank, int32_t world, void* stream) {
  NSR_REQUIRE(flag_ptrs_host != nullptr && epoch_dev != nullptr && err_dev != nullptr, "nsr_p2p_barrier: NULL argument");
  NSR_REQUIRE(world >= 1 && world <= kMaxWorld && rank >= 0 && rank < world, "nsr_p2p_barrier: bad rank / world (max %d)", kMaxWorld);
  FlagPeers fl;
  for (int q = 0; q < kMaxWorld; ++q) fl.p[q] = q < world ? reinterpret_cast<int32_t*>(flag_ptrs_host[q]) : nullptr;
  p2p_barrier_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(fl, epoch_dev, err_dev, rank, world);
  NSR_CHECK_LAUNCH("nsr_p2p_barrier");
  return 0;
}

extern "C" int nsr_p2p_allreduce_mean(const uint64_t* peer_ptrs_host, void* multicast_ptr, int32_t rank, int32_t world, int64_t n,
                                      void* stream) {
  NSR_REQUIRE(world >= 1 && world <= kMaxWorld && rank >= 0 && rank < world, "nsr_p2p_allreduce_mean: bad rank / world (max %d)", kMaxWorld);
  NSR_REQUIRE(n % 4 == 0, "nsr_p2p_allreduce_mean: n must be a multiple of 4 floats");
  NSR_REQUIRE(multicast_ptr != nullptr || peer_ptrs_host != nullptr, "nsr_p2p_allreduce_mean: no peer pointers");
  if (n == 0 || world == 1) return 0;
  const int64_t n4 = n / 4, chunk = (n4 + world - 1) / world;
  constexpr int kU = 4;
  static const int ctas_per_sm = [] {   // tuning knob (default 4): NSR_P2P_CTAS_PER_SM=1..16
    const char* v = getenv("NSR_P2P_CTAS_PER_SM");
    const int n = v ? atoi(v) : 4;
    return n >= 1 && n <= 16 ? n : 4;
  }();
  const int grid = (int)max((int64_t)1, min((int64_t)nsr_sm_count() * ctas_per_sm, (chunk + 256 * kU - 1) / (256 * kU)));
  const float inv = 1.f / (float)world;
  if (multicast_ptr != nullptr) {
    p2p_allreduce_mean_multimem_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((float*)multicast_ptr, rank, world, n4, inv);
  } else {
    Peers peers;
    for (int q = 0; q < kMaxWorld; ++q) peers.p[q] = q < world ? reinterpret_cast<float4*>(peer_ptrs_host[q]) : nullptr;
    p2p_allreduce_mean_kernel<kU><<<grid, 256, 0, (cudaStream_t)stream>>>(peers, rank, world, n4, inv);
  }
  NSR_CHECK_LAUNCH("nsr_p2p_allreduce_mean");
  return 0;
}

// The whole exchange as ONE launch (see p2p_exchange_kernel) over floats [begin, begin + count) of the symmetric buffer.  flag_ptrs_host: every
// rank's peer-mapped flag array (int32[256], zeroed once at start-up; channel c owns slots [32 + 32 c, 64 + 32 c)); epoch_counter_dev: two local
// int32 {last completed epoch, CTA counter} PER CHANNEL, zeroed once.  Exchanges on different channels may run concurrently (different
// streams); the grid is capped at the number of CTAs that are resident at once (the CTAs poll flags, so they must not wait for each
// other's SMs).
extern "C" int nsr_p2p_exchange_mean_range(const uint64_t* peer_ptrs_host, const uint64_t* flag_ptrs_host, void* multicast_ptr, int32_t* epoch_counter_dev,
                                           int32_t* err_dev, int32_t rank, int32_t world, int64_t begin, int64_t count, int32_t channel,
                                           int32_t ctas_per_sm, void* stream) {
  NSR_REQUIRE(world >= 1 && world <= kMaxWorld && rank >= 0 && rank < world, "nsr_p2p_exchange_mean: bad rank / world (max %d)", kMaxWorld);
  NSR_REQUIRE(begin % 4 == 0 && count % 4 == 0 && begin >= 0 && count >= 0, "nsr_p2p_exchange_mean: begin / count must be multiples of 4 floats");
  NSR_REQUIRE(channel >= 0 && channel < 4, "nsr_p2p_exchange_mean: channel must be 0..3");
  NSR_REQUIRE(peer_ptrs_host != nullptr && flag_ptrs_host != nullptr && epoch_counter_dev != nullptr && err_dev != nullptr,
              "nsr_p2p_exchange_mean: NULL argument");
  if (count == 0 || world == 1) return 0;
  XchgArgs a;
  for (int q = 0; q < kMaxWorld; ++q) {
    a.peer[q] = q < world ? reinterpret_cast<float4*>(peer_ptrs_host[q]) : nullptr;
    a.flags[q] = q < world ? reinterpret_cast<int32_t*>(flag_ptrs_host[q]) : nullptr;
  }
  a.mc = (float*)multicast_ptr;
  a.epoch = epoch_counter_dev;
  a.counter = epoch_counter_dev + 1;
  a.err = err_dev;
  a.rank = rank;
  a.world = world;
  a.n4 = count / 4;
  a.o4 = begin / 4;
  a.slot = kChannelSlot0 + kChannelSlots * channel;
  a.inv = 1.f / (float)world;
  const int64_t chunk = (a.n4 + world - 1) / world;
  static const int env_ctas = [] {   // tuning knob: NSR_P2P_CTAS_PER_SM=1..8 (all CTAs must be resident: 256 threads, <= 64 registers)
    const char* v = getenv("NSR_P2P_CTAS_PER_SM");
    const int n = v ? atoi(v) : 0;
    return n >= 1 && n <= 8 ? n : 0;
  }();
  const int per_sm = ctas_per_sm >= 1 && ctas_per_sm <= 8 ? ctas_per_sm : (env_ctas ? env_ctas : 2);
  static const int env_u = [] {   // tuning knob: 16-byte columns in flight per thread (NSR_P2P_UNROLL = 4 | 8 | 16; default 8)
    const char* v = getenv("NSR_P2P_UNROLL");
    const int n = v ? atoi(v) : 8;
    return n == 4 || n == 16 ? n : 8;
  }();
  // beside a scatter launch (ctas_per_sm == 1) the CTA must fit into the 16 K registers that launch leaves free: P2P form with 4 columns
  const int u = (ctas_per_sm == 1 && multicast_ptr == nullptr) ? 4 : env_u;
  const int grid_u = (int)max((int64_t)1, min((int64_t)nsr_sm_count() * per_sm, (chunk + 256 * u - 1) / (256 * u)));
  cudaStream_t st = (cudaStream_t)stream;
  if (multicast_ptr != nullptr) {
    if (u == 4) p2p_exchange_kernel<4, true><<<grid_u, 256, 0, st>>>(a);
    else if (u == 16) p2p_exchange_kernel<16, true><<<grid_u, 256, 0, st>>>(a);
    else p2p_exchange_kernel<8, true><<<grid_u, 256, 0, st>>>(a);
  } else {
    if (u == 4) p2p_exchange_kernel<4, false><<<grid_u, 256, 0, st>>>(a);
    else if (u == 16) p2p_exchange_kernel<16, false><<<grid_u, 256, 0, st>>>(a);
    else p2p_exchange_kernel<8, false><<<grid_u, 256, 0, st>>>(a);
  }
  NSR_CHECK_LAUNCH("nsr_p2p_exchange_mean");
  return 0;
}

extern "C" int nsr_p2p_exchange_mean(const uint64_t* peer_ptrs_host, const uint64_t* flag_ptrs_host, void* multicast_ptr, int32_t* epoch_counter_dev,
                                     int32_t* err_dev, int32_t rank, int32_t world, int64_t n, void* stream) {
  return nsr_p2p_exchange_mean_range(peer_ptrs_host, flag_ptrs_host, multicast_ptr, epoch_counter_dev, err_dev, rank, world, 0, n, 0, 0, stream);
}
