// Shared device helpers for the parallax_b200 sm_90a kernels.
//
// Conventions
//  * A "world" is up to PX_MAX_RANKS GPUs on one NVSwitch domain.  Peer
//    buffers are passed BY VALUE as a small array of raw device pointers
//    (IPC-mapped symmetric allocations, or plain local allocations when a
//    world is simulated inside one process for single-GPU tests).
//  * Cross-GPU synchronisation uses monotonically increasing 32-bit epochs
//    written with st.release.sys into the peer's signal pad and polled with
//    ld.acquire.sys locally — one NVLink one-way latency per barrier, no
//    remote atomics, no flag reset, replay-safe under CUDA graphs because the
//    epoch counter lives in device memory.
//
// Reference parity: this replaces Horovod's CPU-side coordination
// (horovod/common/operations.cc:1274-1590) + NCCL stream semantics
// (horovod/common/ops/nccl_operations.cc:60-109) with device-side flags.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

#define PX_MAX_RANKS 16
#define PX_NUM_SMS 132            // H100 SXM: grid caps of the grid-stride kernels
#define PX_MAX_BLOCKS 128          // max CTAs of a communicating kernel
#define PX_NUM_CHANNELS 8          // independent barrier channels per pad

struct PeerPtrs {
  void* p[PX_MAX_RANKS];
};

// Signal pad layout (uint32): [channel][block][src_rank]
#define PX_PAD_WORDS (PX_NUM_CHANNELS * PX_MAX_BLOCKS * PX_MAX_RANKS)
// followed by sparse-path flags: pushed[table_slot][src], applied[table_slot][src]
#define PX_PAD_BYTES (PX_PAD_WORDS * 4)

__device__ __forceinline__ void st_release_sys(uint32_t* addr, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* addr) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(addr) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t* addr) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(addr) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_volatile_u32(const uint32_t* addr) {
  uint32_t v;
  asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(addr) : "memory");
  return v;
}

// %globaltimer (ns): the device clock of every profiling stamp
__device__ __forceinline__ unsigned long long px_globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// 16-byte vector load/store.  Peer loads must not go through the
// non-coherent path (data changes between steps; L1 is only invalidated at
// kernel boundaries, which is exactly the granularity we synchronise at).
__device__ __forceinline__ uint4 ld_v4(const void* p) {
  uint4 v;
  asm volatile("ld.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint4 ld_v4_stream(const void* p) {
  uint4 v;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_v4(void* p, const uint4& v) {
  asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};"
               ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void st_v4_stream(void* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};"
               ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// ---- 16-byte pack <-> fp32 lanes -------------------------------------------
template <typename T> struct Vec16;
template <> struct Vec16<float> {
  static constexpr int N = 4;
  __device__ __forceinline__ static void unpack(const uint4& v, float* f) {
    f[0] = __uint_as_float(v.x); f[1] = __uint_as_float(v.y);
    f[2] = __uint_as_float(v.z); f[3] = __uint_as_float(v.w);
  }
  __device__ __forceinline__ static uint4 pack(const float* f) {
    return make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]),
                      __float_as_uint(f[2]), __float_as_uint(f[3]));
  }
};
template <> struct Vec16<__nv_bfloat16> {
  static constexpr int N = 8;
  __device__ __forceinline__ static void unpack(const uint4& v, float* f) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      f[2 * i] = __uint_as_float(w[i] << 16);
      f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    }
  }
  __device__ __forceinline__ static uint4 pack(const float* f) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
      w[i] = *reinterpret_cast<uint32_t*>(&h);
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
  }
};

// ---- cross-GPU block barrier -------------------------------------------------
// Every CTA `b` of rank `r` synchronises with CTA `b` of every peer on
// `channel`.  `epoch_ctr` is a *local* (non-symmetric) array
// [PX_NUM_CHANNELS][PX_MAX_BLOCKS]; all ranks execute the same kernel
// sequence so the counters agree.  On return all global writes made by any
// thread of the peer CTAs before their barrier are visible to this CTA.
// `pads` is a device array of `world` pointers (one signal pad per rank).
__device__ __forceinline__ void px_block_barrier(uint32_t* const* __restrict__ pads,
                                                 uint32_t* epoch_ctr, int channel, int rank,
                                                 int world) {
  const int slot = channel * PX_MAX_BLOCKS + blockIdx.x;
  __syncthreads();
  const uint32_t e = ld_volatile_u32(epoch_ctr + slot) + 1;
  if (threadIdx.x < world) {
    const int peer = threadIdx.x;
    uint32_t* remote = pads[peer] + (size_t)slot * PX_MAX_RANKS + rank;
    __threadfence_system();
    st_release_sys(remote, e);
    const uint32_t* mine = pads[rank] + (size_t)slot * PX_MAX_RANKS + peer;
    while ((int32_t)(ld_acquire_sys(mine) - e) < 0) { }
  }
  __syncthreads();
  if (threadIdx.x == 0) epoch_ctr[slot] = e;
  // no trailing sync needed: the next barrier on this slot starts with one.
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// block-wide sum -> atomicAdd into *out (fp32)
__device__ __forceinline__ void block_atomic_sum(float v, float* out) {
  __shared__ float s_part[32];
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) s_part[wid] = v;
  __syncthreads();
  if (wid == 0) {
    float t = lane < (blockDim.x + 31) / 32 ? s_part[lane] : 0.f;
    t = warp_sum(t);
    if (lane == 0 && t != 0.f) atomicAdd(out, t);
  }
  __syncthreads();
}
