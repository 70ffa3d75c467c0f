// Dense collectives over NVLink peer memory: barrier, two-shot in-place
// all-reduce, staged one-shot all-reduce, broadcast, all-gather.
//
// Reference parity (what these replace): Horovod's fused-bucket path —
// N× cudaMemcpyAsync into the fusion buffer, ncclAllReduce on a private
// stream, N× cudaMemcpyAsync out, then a separate `tf.div(sum, size)` kernel
// (horovod/common/ops/nccl_operations.cc:60-109,
//  horovod/common/ops/cuda_operations.cc:105-121,
//  horovod/tensorflow/__init__.py:76-81); hierarchical reduce-scatter /
// all-gather (nccl_operations.cc:167-363); MPI_Bcast of initial variables
// (mpi_operations.cc:334-358).  Here the bucket already lives contiguously in
// symmetric memory, accumulation is fp32, the 1/N scale and the cast are in
// the epilogue, and an optional Σx² for global-norm clipping rides along.
//
// Peer pointer arrays arrive ROTATED by the launcher: entry p is rank
// (rank+p) % world, so entry 0 is always the local buffer, indices are
// static (no local-memory copy of the parameter struct) and ranks spread
// their first loads over different peers.
#include "common.cuh"

// ---------------------------------------------------------------------------
__global__ void px_barrier_kernel(uint32_t* const* pads, uint32_t* epoch_ctr, int channel,
                                  int rank, int world) {
  px_block_barrier(pads, epoch_ctr, channel, rank, world);
}

// ---------------------------------------------------------------------------
// Two-shot, in place.  Rank r owns slice r: it pulls that slice from every
// peer (reduce-scatter by load), reduces in fp32, scales, and pushes the
// result into every peer's buffer (all-gather by store).  2·(W-1)/W·n bytes
// cross NVLink per rank — the bandwidth-optimal volume.
template <typename T, int W, int UNROLL>
__global__ void __launch_bounds__(512)
px_allreduce_twoshot_kernel(PeerPtrs rot, uint32_t* const* pads, uint32_t* epoch_ctr,
                            int ch_start, int ch_end, size_t n, float scale, float* sumsq_out,
                            int rank) {
  constexpr int VN = Vec16<T>::N;
  px_block_barrier(pads, epoch_ctr, ch_start, rank, W);
  const size_t slice = n / W;               // elements, multiple of VN
  const size_t nvec = slice / VN;
  const size_t base = (size_t)rank * slice;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  float ss = 0.f;
  for (size_t v0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v0 < nvec;
       v0 += stride * UNROLL) {
    uint4 in[UNROLL][W];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const size_t v = v0 + (size_t)u * stride;
      if (v < nvec) {
#pragma unroll
        for (int p = 0; p < W; ++p)
          in[u][p] = ld_v4_stream(reinterpret_cast<const T*>(rot.p[p]) + base + v * VN);
      }
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const size_t v = v0 + (size_t)u * stride;
      if (v < nvec) {
        float acc[VN];
#pragma unroll
        for (int i = 0; i < VN; ++i) acc[i] = 0.f;
#pragma unroll
        for (int p = 0; p < W; ++p) {
          float f[VN];
          Vec16<T>::unpack(in[u][p], f);
#pragma unroll
          for (int i = 0; i < VN; ++i) acc[i] += f[i];
        }
#pragma unroll
        for (int i = 0; i < VN; ++i) { acc[i] *= scale; ss += acc[i] * acc[i]; }
        const uint4 out = Vec16<T>::pack(acc);
#pragma unroll
        for (int p = 0; p < W; ++p)
          st_v4_stream(reinterpret_cast<T*>(rot.p[p]) + base + v * VN, out);
      }
    }
  }
  if (sumsq_out != nullptr) block_atomic_sum(ss, sumsq_out);
  px_block_barrier(pads, epoch_ctr, ch_end, rank, W);
}


// ---------------------------------------------------------------------------
// TMA variant of the two-shot all-reduce (measurement for SURVEY §7.4 / the north star's
// "TMA tiles for the dense reduction"): the reduce-scatter phase pulls every peer's slice with
// `cp.async.bulk` (bulk async copy engine, global -> shared, mbarrier completion) into a
// double-buffered shared-memory stage of W x PX_BULK_BYTES, the CTA sums the W tiles out of shared
// memory in fp32 and stores the reduced tile into every peer (all-gather by store).  Same
// barriers, same bytes over NVLink as `px_allreduce_twoshot_kernel`; only the load path differs
// (TMA engine + SMEM instead of ld.global.v4 into registers).
#define PX_BULK_BYTES 8192
__device__ __forceinline__ uint32_t cvta_smem(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
template <typename T, int W>
__global__ void __launch_bounds__(256)
px_allreduce_twoshot_bulk_kernel(PeerPtrs rot, uint32_t* const* pads, uint32_t* epoch_ctr,
                                 int ch_start, int ch_end, size_t n, float scale, int rank) {
  constexpr int VN = Vec16<T>::N;
  extern __shared__ __align__(128) uint8_t bulk_smem[];       // [2][W][PX_BULK_BYTES]
  __shared__ __align__(8) uint64_t full[2];
  px_block_barrier(pads, epoch_ctr, ch_start, rank, W);
  const size_t slice_bytes = n / W * sizeof(T);               // multiple of 16
  const size_t base_bytes = (size_t)rank * slice_bytes;
  const size_t nchunks = (slice_bytes + PX_BULK_BYTES - 1) / PX_BULK_BYTES;
  if (threadIdx.x == 0) {
    for (int s = 0; s < 2; ++s)
      asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(cvta_smem(&full[s])), "r"(1));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  auto issue = [&](size_t c, int stage) {
    const size_t off = c * PX_BULK_BYTES;
    const uint32_t bytes = (uint32_t)min((size_t)PX_BULK_BYTES, slice_bytes - off);
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::
                 "r"(cvta_smem(&full[stage])), "r"(bytes * W) : "memory");
#pragma unroll
    for (int p = 0; p < W; ++p)
      asm volatile(
          "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
          ::"r"(cvta_smem(bulk_smem + ((size_t)stage * W + p) * PX_BULK_BYTES)),
            "l"(reinterpret_cast<const char*>(rot.p[p]) + base_bytes + off), "r"(bytes),
            "r"(cvta_smem(&full[stage])) : "memory");
  };
  size_t it = 0;
  if (threadIdx.x == 0 && (size_t)blockIdx.x < nchunks) issue(blockIdx.x, 0);
  for (size_t c = blockIdx.x; c < nchunks; c += gridDim.x, ++it) {
    const int stage = (int)(it & 1);
    const size_t cn = c + gridDim.x;
    if (threadIdx.x == 0 && cn < nchunks) issue(cn, stage ^ 1);   // consumed two trips ago
    const uint32_t parity = (uint32_t)((it >> 1) & 1);
    asm volatile(
        "{\n.reg .pred p;\nBW_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra BD_%=;\nbra BW_%=;\nBD_%=:\n}\n" ::"r"(cvta_smem(&full[stage])), "r"(parity)
        : "memory");
    const size_t off = c * PX_BULK_BYTES;
    const int nv = (int)(min((size_t)PX_BULK_BYTES, slice_bytes - off) / 16);
    for (int v = threadIdx.x; v < nv; v += blockDim.x) {
      float acc[VN];
#pragma unroll
      for (int i = 0; i < VN; ++i) acc[i] = 0.f;
#pragma unroll
      for (int p = 0; p < W; ++p) {
        float f[VN];
        Vec16<T>::unpack(*reinterpret_cast<const uint4*>(
                             bulk_smem + ((size_t)stage * W + p) * PX_BULK_BYTES + (size_t)v * 16), f);
#pragma unroll
        for (int i = 0; i < VN; ++i) acc[i] += f[i];
      }
#pragma unroll
      for (int i = 0; i < VN; ++i) acc[i] *= scale;
      const uint4 out = Vec16<T>::pack(acc);
#pragma unroll
      for (int p = 0; p < W; ++p)
        st_v4_stream(reinterpret_cast<char*>(rot.p[p]) + base_bytes + off + (size_t)v * 16, out);
    }
    __syncthreads();            // the stage may be refilled by the async proxy from here on
  }
  px_block_barrier(pads, epoch_ctr, ch_end, rank, W);
}

// ---------------------------------------------------------------------------
// One-shot for latency-bound sizes: copy my input into my double-buffered
// symmetric staging area, barrier, then every rank reads every peer's staging
// and reduces locally in RANK order (bitwise identical on every replica).
// One barrier per call (the staging parity makes an end barrier unnecessary).
template <typename T, int W>
__global__ void __launch_bounds__(512)
px_allreduce_oneshot_kernel(const T* __restrict__ src, T* __restrict__ dst, PeerPtrs stages,
                            char* my_stage_base, size_t stage_half_bytes, uint32_t* const* pads, uint32_t* epoch_ctr,
                            int channel, size_t n, float scale, float* sumsq_out, int rank) {
  constexpr int VN = Vec16<T>::N;
  const size_t nvec = (n + VN - 1) / VN;      // caller guarantees 16B-padded storage
  const int slot = channel * PX_MAX_BLOCKS + blockIdx.x;
  const uint32_t parity = (ld_volatile_u32(epoch_ctr + slot) + 1) & 1u;
  const size_t off = parity ? stage_half_bytes : 0;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  char* my_stage = my_stage_base + off;
  for (size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += stride)
    st_v4(my_stage + v * 16, ld_v4(reinterpret_cast<const char*>(src) + v * 16));
  px_block_barrier(pads, epoch_ctr, channel, rank, W);
  float ss = 0.f;
  for (size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += stride) {
    uint4 in[W];
#pragma unroll
    for (int p = 0; p < W; ++p)
      in[p] = ld_v4_stream(reinterpret_cast<const char*>(stages.p[p]) + off + v * 16);
    float acc[VN];
#pragma unroll
    for (int i = 0; i < VN; ++i) acc[i] = 0.f;
#pragma unroll
    for (int p = 0; p < W; ++p) {
      float f[VN];
      Vec16<T>::unpack(in[p], f);
#pragma unroll
      for (int i = 0; i < VN; ++i) acc[i] += f[i];
    }
#pragma unroll
    for (int i = 0; i < VN; ++i) { acc[i] *= scale; ss += acc[i] * acc[i]; }
    st_v4(reinterpret_cast<char*>(dst) + v * 16, Vec16<T>::pack(acc));
  }
  if (sumsq_out != nullptr) block_atomic_sum(ss, sumsq_out);
}

// ---------------------------------------------------------------------------
// Broadcast root's buffer into every rank's buffer (symmetric, same offset):
// pull model — each non-root rank copies from the root over NVLink.
__global__ void __launch_bounds__(512)
px_broadcast_kernel(const char* __restrict__ root_buf, char* __restrict__ my_buf,
                    uint32_t* const* pads, uint32_t* epoch_ctr, int ch_start, int ch_end,
                    size_t nbytes, int root, int rank, int world) {
  px_block_barrier(pads, epoch_ctr, ch_start, rank, world);
  if (rank != root) {
    const size_t nvec = nbytes / 16;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += stride)
      st_v4(my_buf + v * 16, ld_v4_stream(root_buf + v * 16));
  }
  px_block_barrier(pads, epoch_ctr, ch_end, rank, world);
}

// All-gather by push: rank r's `slice_bytes` at offset r*slice_bytes of its own
// buffer is stored into every peer's buffer at the same offset.
template <int W>
__global__ void __launch_bounds__(512)
px_allgather_kernel(PeerPtrs rot, uint32_t* const* pads, uint32_t* epoch_ctr, int ch_start,
                    int ch_end, size_t slice_bytes, int rank) {
  px_block_barrier(pads, epoch_ctr, ch_start, rank, W);
  const size_t nvec = slice_bytes / 16;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t off = (size_t)rank * slice_bytes;
  const char* src = reinterpret_cast<const char*>(rot.p[0]) + off;
  for (size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += stride) {
    const uint4 x = ld_v4(src + v * 16);
#pragma unroll
    for (int p = 1; p < W; ++p)
      st_v4_stream(reinterpret_cast<char*>(rot.p[p]) + off + v * 16, x);
  }
  px_block_barrier(pads, epoch_ctr, ch_end, rank, W);
}

// ---------------------------------------------------------------------------
// host launchers (C ABI)
// ---------------------------------------------------------------------------
#include "launch.h"

extern "C" {

int px_barrier(void* pads_dev, void* epoch_ctr, int channel, int rank, int world, int blocks,
               cudaStream_t stream) {
  if (blocks < 1) blocks = 1;
  if (blocks > PX_MAX_BLOCKS) blocks = PX_MAX_BLOCKS;
  px_barrier_kernel<<<blocks, 32, 0, stream>>>((uint32_t* const*)pads_dev, (uint32_t*)epoch_ctr,
                                               channel, rank, world);
  return (int)cudaGetLastError();
}

// dtype: 0 = fp32, 1 = bf16.  n must be a multiple of world * (16/sizeof(T)).
int px_allreduce_twoshot(const void* const* bufs, void* pads_dev, void* epoch_ctr, int ch_start,
                         int ch_end, size_t n, int dtype, float scale, float* sumsq_out, int rank,
                         int world, int max_blocks, cudaStream_t stream) {
  const PeerPtrs R = px_rotate(bufs, rank, world);
  const int threads = 512;
  const int vn = dtype == 0 ? 4 : 8;
  if (world < 1 || world > 8) return -3;
  if (n % ((size_t)world * vn) != 0) return -1;
  const int blocks = px_clamp_blocks(n / world / vn, threads * 2, max_blocks);
#define LAUNCH(T, W)                                                                       \
  px_allreduce_twoshot_kernel<T, W, (W <= 4 ? 4 : 2)><<<blocks, threads, 0, stream>>>(       \
      R, (uint32_t* const*)pads_dev, (uint32_t*)epoch_ctr, ch_start, ch_end, n, scale,     \
      sumsq_out, rank)
  if (dtype == 0) { PX_DISPATCH_WORLD(world, LAUNCH, float); }
  else { PX_DISPATCH_WORLD(world, LAUNCH, __nv_bfloat16); }
#undef LAUNCH
  return (int)cudaGetLastError();
}

int px_allreduce_twoshot_bulk(const void* const* bufs, void* pads_dev, void* epoch_ctr,
                              int ch_start, int ch_end, size_t n, int dtype, float scale, int rank,
                              int world, int max_blocks, cudaStream_t stream) {
  if (world < 1 || world > 8) return -3;
  const PeerPtrs R = px_rotate(bufs, rank, world);
  const int vn = dtype == 0 ? 4 : 8;
  if (n % ((size_t)world * vn) != 0) return -1;
  const size_t es = dtype == 0 ? 4 : 2;
  const size_t chunks = (n / world * es + PX_BULK_BYTES - 1) / PX_BULK_BYTES;
  int blocks = (int)(chunks < 1 ? 1 : (chunks > (size_t)max_blocks ? (size_t)max_blocks : chunks));
  if (blocks > PX_MAX_BLOCKS) blocks = PX_MAX_BLOCKS;
  const size_t smem = (size_t)2 * world * PX_BULK_BYTES;
#define LAUNCH(T, W)                                                                          \
  do {                                                                                        \
    cudaFuncSetAttribute(px_allreduce_twoshot_bulk_kernel<T, W>,                              \
                         cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * 8 * PX_BULK_BYTES); \
    px_allreduce_twoshot_bulk_kernel<T, W><<<blocks, 256, smem, stream>>>(                    \
        R, (uint32_t* const*)pads_dev, (uint32_t*)epoch_ctr, ch_start, ch_end, n, scale, rank); \
  } while (0)
  if (dtype == 0) { PX_DISPATCH_WORLD(world, LAUNCH, float); }
  else { PX_DISPATCH_WORLD(world, LAUNCH, __nv_bfloat16); }
#undef LAUNCH
  return (int)cudaGetLastError();
}

int px_allreduce_oneshot(const void* src, void* dst, const void* const* stages,
                         size_t stage_half_bytes, void* pads_dev, void* epoch_ctr, int channel,
                         size_t n, int dtype, float scale, float* sumsq_out, int rank, int world,
                         int max_blocks, cudaStream_t stream) {
  PeerPtrs S{};
  for (int i = 0; i < world; ++i) S.p[i] = const_cast<void*>(stages[i]);
  const int threads = 512;
  const size_t esz = dtype == 0 ? 4 : 2;
  if (world < 1 || world > 8) return -3;
  if (((n * esz + 15) / 16) * 16 > stage_half_bytes) return -2;
  const int blocks = px_clamp_blocks((n * esz + 15) / 16, threads, max_blocks);
#define LAUNCH(T, W)                                                                     \
  px_allreduce_oneshot_kernel<T, W><<<blocks, threads, 0, stream>>>(                     \
      (const T*)src, (T*)dst, S, (char*)S.p[rank], stage_half_bytes, (uint32_t* const*)pads_dev,           \
      (uint32_t*)epoch_ctr, channel, n, scale, sumsq_out, rank)
  if (dtype == 0) { PX_DISPATCH_WORLD(world, LAUNCH, float); }
  else { PX_DISPATCH_WORLD(world, LAUNCH, __nv_bfloat16); }
#undef LAUNCH
  return (int)cudaGetLastError();
}

int px_broadcast(const void* const* bufs, void* pads_dev, void* epoch_ctr, int ch_start,
                 int ch_end, size_t nbytes, int root, int rank, int world, int max_blocks,
                 cudaStream_t stream) {
  if (nbytes % 16) return -1;
  const int blocks = px_clamp_blocks(nbytes / 16, 512 * 4, max_blocks);
  px_broadcast_kernel<<<blocks, 512, 0, stream>>>(
      (const char*)bufs[root], (char*)const_cast<void*>(bufs[rank]), (uint32_t* const*)pads_dev,
      (uint32_t*)epoch_ctr, ch_start, ch_end, nbytes, root, rank, world);
  return (int)cudaGetLastError();
}

int px_allgather(const void* const* bufs, void* pads_dev, void* epoch_ctr, int ch_start,
                 int ch_end, size_t slice_bytes, int rank, int world, int max_blocks,
                 cudaStream_t stream) {
  const PeerPtrs R = px_rotate(bufs, rank, world);
  if (slice_bytes % 16) return -1;
  if (world < 1 || world > 8) return -3;
  const int blocks = px_clamp_blocks(slice_bytes / 16, 512 * 4, max_blocks);
#define LAUNCH(T, W)                                                                  \
  px_allgather_kernel<W><<<blocks, 512, 0, stream>>>(R, (uint32_t* const*)pads_dev,   \
                                                     (uint32_t*)epoch_ctr, ch_start,  \
                                                     ch_end, slice_bytes, rank)
  PX_DISPATCH_WORLD(world, LAUNCH, int);
#undef LAUNCH
  return (int)cudaGetLastError();
}

}  // extern "C"

// ---------------------------------------------------------------------------
// NVLS all-reduce: the buffer is bound to an NVSwitch multicast object.  Rank r
// reduces slice r with ONE multimem.ld_reduce per 16 bytes (the switch pulls
// and sums every GPU's copy: fp32 accumulation for bf16) and broadcasts the
// result to every GPU with ONE multimem.st — (N+1)/N·n bytes cross this GPU's
// links instead of 2(N-1)/N·n, and no SM does the adds.
template <typename T>
__device__ __forceinline__ uint4 mm_ld_reduce(const T* p) {
  uint4 r;
  if (sizeof(T) == 2)
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
  else
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
  return r;
}
__device__ __forceinline__ void mm_st(void* p, const uint4& r) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};"
               ::"l"(p), "r"(r.x), "r"(r.y), "r"(r.z), "r"(r.w) : "memory");
}

template <typename T, int UNROLL>
__global__ void __launch_bounds__(512)
px_allreduce_nvls_kernel(T* __restrict__ mc, uint32_t* const* pads, uint32_t* epoch_ctr,
                         int ch_start, int ch_end, size_t n, float scale, int rank, int world) {
  constexpr int VN = Vec16<T>::N;
  px_block_barrier(pads, epoch_ctr, ch_start, rank, world);
  const size_t slice = n / world;
  const size_t nvec = slice / VN;
  const size_t base = (size_t)rank * slice;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t v0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v0 < nvec;
       v0 += stride * UNROLL) {
    uint4 r[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const size_t v = v0 + (size_t)u * stride;
      if (v < nvec) r[u] = mm_ld_reduce<T>(mc + base + v * VN);
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const size_t v = v0 + (size_t)u * stride;
      if (v < nvec) {
        if (scale != 1.f) {
          float f[VN];
          Vec16<T>::unpack(r[u], f);
#pragma unroll
          for (int i = 0; i < VN; ++i) f[i] *= scale;
          r[u] = Vec16<T>::pack(f);
        }
        mm_st(mc + base + v * VN, r[u]);
      }
    }
  }
  px_block_barrier(pads, epoch_ctr, ch_end, rank, world);
}

extern "C" int px_allreduce_nvls(void* mc_ptr, void* pads_dev, void* epoch_ctr, int ch_start,
                                 int ch_end, size_t n, int dtype, float scale, int rank, int world,
                                 int max_blocks, cudaStream_t stream) {
  const int vn = dtype == 0 ? 4 : 8;
  if (n % ((size_t)world * vn) != 0) return -1;
  const int blocks = px_clamp_blocks(n / world / vn, 512 * 8, max_blocks);
  if (dtype == 0)
    px_allreduce_nvls_kernel<float, 8><<<blocks, 512, 0, stream>>>(
        (float*)mc_ptr, (uint32_t* const*)pads_dev, (uint32_t*)epoch_ctr, ch_start, ch_end, n,
        scale, rank, world);
  else
    px_allreduce_nvls_kernel<__nv_bfloat16, 8><<<blocks, 512, 0, stream>>>(
        (__nv_bfloat16*)mc_ptr, (uint32_t* const*)pads_dev, (uint32_t*)epoch_ctr, ch_start,
        ch_end, n, scale, rank, world);
  return (int)cudaGetLastError();
}
