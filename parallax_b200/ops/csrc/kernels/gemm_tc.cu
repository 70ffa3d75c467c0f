// wgmma / TMA / mbarrier GEMM for the skinny recurrent products of the LSTM
// (M = batch = 128·k rows, huge K or huge N) — hand-written for sm_90a.
//
//   C[M,N] (bf16) = A[M,K] (bf16, K-contiguous) · B[N,K]^T (bf16, K-contiguous)
//                   (+ addend[M,N] bf16)                        "TN" GEMM
//
// Roles (one CTA = 3 warpgroups, 384 threads): warpgroup 0 is the TMA producer
// (one thread issues cp.async.bulk.tensor, 128B swizzle); warpgroups 1 and 2
// are consumers, each owning 64 rows of the 128-row tile and issuing
// wgmma.mma_async m64×BN×16 from shared memory with the fp32 accumulator in
// registers.  STAGES-deep smem ring with full/empty mbarriers; a consumer
// keeps one wgmma group in flight and frees the previous stage when it retires.
//
// Split-K: grid.z CTAs each reduce a K-slice and red.add their fp32 tile into
// an L2-resident workspace; the last CTA to arrive for a tile (atomic ticket)
// converts (+addend) to bf16, stores C and re-zeroes the workspace — so a
// [128, 8192]·[8192, 512] product runs on 4·32 CTAs instead of 4, without a
// second launch.  The reference reaches these products through cuBLAS
// (tensorflow/core/kernels/matmul_op.cc:252-369 → cuda_blas.cc:2229).
#include "wgmma.cuh"
#include "lstm_cell.cuh"

namespace tc {

// Shared main loop.  Producer: thread 0 streams num_kb K-blocks of A (128 rows) and B (BN rows)
// into the ring.  Consumer warpgroup cw (0/1): accumulates rows cw·64 … cw·64+63 of the tile
// into acc.  Accumulator layout (wgmma m64nN f32): acc[j·4 + e] is row
// (warp%4)·16 + lane/4 + 8·(e/2), column j·8 + (lane%4)·2 + e%2 of the warpgroup's 64×BN tile.
template <int BN, int STAGES>
__device__ __forceinline__ void mainloop(const CUtensorMap* tmap_a, const CUtensorMap* tmap_b,
                                         uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar,
                                         int k0, int num_kb, int m0, int n0, float* acc) {
  constexpr int A_BYTES = BM * BK * 2, B_BYTES = BN * BK * 2, STAGE_BYTES = A_BYTES + B_BYTES;
  const int wg = threadIdx.x >> 7;
  if (wg == 0) {
    if (threadIdx.x == 0) {
      for (int kb = 0; kb < num_kb; ++kb) {
        const int s = kb % STAGES;
        const uint32_t ph = (kb / STAGES) & 1;
        mbar_wait(&empty_bar[s], ph ^ 1);
        uint8_t* sa = smem + s * STAGE_BYTES;
        mbar_expect_tx(&full_bar[s], STAGE_BYTES);
        tma_load_2d(sa, tmap_a, &full_bar[s], k0 + kb * BK, m0);
        tma_load_2d(sa + A_BYTES, tmap_b, &full_bar[s], k0 + kb * BK, n0);
      }
    }
    return;
  }
  const int cw = wg - 1;
  const bool leader = (threadIdx.x & 127) == 0;
  for (int kb = 0; kb < num_kb; ++kb) {
    const int s = kb % STAGES;
    mbar_wait(&full_bar[s], (kb / STAGES) & 1);
    const uint32_t sa = smem_u32(smem + s * STAGE_BYTES);
    // this warpgroup's 64 rows start 64·128 B into the A tile (a whole number of swizzle atoms)
    const uint64_t adesc = make_smem_desc(sa + cw * 64 * BK * 2);
    const uint64_t bdesc = make_smem_desc(sa + A_BYTES);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / WG_K; ++k)
      // advance 32 B (= 16 bf16) inside the swizzle atom: +2 in the 16-byte-granular address
      wgmma_bf16<BN>(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2),
                     (kb | k) != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<1>();                               // the group of K-block kb-1 has retired
    if (kb > 0 && leader) mbar_arrive(&empty_bar[(kb - 1) % STAGES]);
  }
  wgmma_wait<0>();
}

struct GemmArgs {
  __nv_bfloat16* C;            // [M, N]
  const __nv_bfloat16* addend; // [M, N] or null
  float* ws;                   // [M, N] fp32, zero between calls (split-K only)
  unsigned int* tickets;       // [(M/128) * (N/BN)] zero between calls (split-K only)
  int M, N, K;                 // K = full reduction length
  int k_per_split;             // multiple of BK
};

__device__ __forceinline__ float2 bf16x2_to_float2(uint32_t w) {
  return make_float2(__uint_as_float(w << 16), __uint_as_float(w & 0xffff0000u));
}
__device__ __forceinline__ uint32_t float2_to_bf16x2(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// CLUSTER = true: the K-splits of one output tile form a thread-block cluster (1,1,splits) and
// reduce their fp32 partial tiles through distributed shared memory — each CTA parks its tile in
// its own SMEM (the drained pipeline stages), cluster barrier, then every CTA sums 1/splits of
// the rows straight out of its peers' SMEM (`ld.shared::cluster`), adds the addend and stores
// bf16.  No L2 `red.add`, no ticket, no read-back pass, no workspace.
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n"
               "barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// Parks this consumer thread's accumulator fragment (see `mainloop`) as rows of a 128×BN fp32
// tile at `park` (row stride BN+4 floats); ROUND: each value rounded to bf16 first.
template <int BN, bool ROUND>
__device__ __forceinline__ void park_acc(float* park, const float* acc) {
  const int t = threadIdx.x - 128, lane = t & 31;
  const int lrow = (t >> 5) * 16 + (lane >> 2);     // tile row of acc[j·4 + 0/1]; +8 for 2/3
  const int lcol = (lane & 3) * 2;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float2 v = make_float2(acc[j * 4 + 2 * h], acc[j * 4 + 2 * h + 1]);
      if (ROUND) v = __bfloat1622float2(__floats2bfloat162_rn(v.x, v.y));
      *reinterpret_cast<float2*>(park + (size_t)(lrow + 8 * h) * (BN + 4) + j * 8 + lcol) = v;
    }
}

template <int BN, int STAGES, bool CLUSTER>
__global__ void __launch_bounds__(THREADS, 1)
px_gemm_tc_kernel(const __grid_constant__ CUtensorMap tmap_a,
                  const __grid_constant__ CUtensorMap tmap_b, GemmArgs g) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // carve: [STAGES][A 16 KB][B BN*128 B] then barriers
  uint8_t* smem = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  constexpr int STAGE_BYTES = BM * BK * 2 + BN * BK * 2;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  __shared__ unsigned int s_last;

  const int n_tile = blockIdx.x, m_tile = blockIdx.y, split = blockIdx.z;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_a) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_b) : "memory");
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  float acc[BN / 2];
  mainloop<BN, STAGES>(&tmap_a, &tmap_b, smem, full_bar, empty_bar, split * g.k_per_split,
                       g.k_per_split / BK, m_tile * BM, n_tile * BN, acc);

  if (threadIdx.x >= 128) {
    // -------------------------------- epilogue --------------------------------
    const int t = threadIdx.x - 128, lane = t & 31;
    const int lrow = (t >> 5) * 16 + (lane >> 2);   // tile row of acc[j·4 + 0/1]; +8 for 2/3
    const int lcol = (lane & 3) * 2;
    const bool splitk = gridDim.z > 1;
    if (CLUSTER) {
      // park the fp32 partial in shared memory; every wgmma of both consumer warpgroups has
      // retired before the stages are overwritten
      consumer_sync();
      park_acc<BN, false>(reinterpret_cast<float*>(smem), acc);
    } else {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = m_tile * BM + lrow + 8 * h;
        if (row >= g.M) continue;
        const size_t base = (size_t)row * g.N + (size_t)n_tile * BN + lcol;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const size_t off = base + j * 8;
          float2 v = make_float2(acc[j * 4 + 2 * h], acc[j * 4 + 2 * h + 1]);
          if (splitk) {
            atomicAdd(reinterpret_cast<float2*>(g.ws + off), v);
          } else {
            if (g.addend) {
              const float2 a = bf16x2_to_float2(*reinterpret_cast<const uint32_t*>(g.addend + off));
              v.x += a.x; v.y += a.y;
            }
            *reinterpret_cast<uint32_t*>(g.C + off) = float2_to_bf16x2(v.x, v.y);
          }
        }
      }
    }
  }
  __syncthreads();
  if (CLUSTER) {
    uint32_t crank, csize;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(crank));
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(csize));
    cluster_sync_all();                               // every split's partial is in its SMEM
    const int rows_per = BM / (int)csize;             // csize divides 128
    const int nvec = rows_per * BN / 4;               // float4 groups this CTA reduces
    const uint32_t my_base = smem_u32(smem);
    for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
      const int rr = (int)crank * rows_per + (v * 4) / BN, cc = (v * 4) % BN;
      const uint32_t off_b = (uint32_t)(((size_t)rr * (BN + 4) + cc) * 4);
      float4 acc4 = make_float4(0.f, 0.f, 0.f, 0.f);
      for (uint32_t p = 0; p < csize; ++p) {
        uint32_t raddr;
        asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(raddr) : "r"(my_base + off_b), "r"(p));
        float4 x;
        asm volatile("ld.shared::cluster.v4.f32 {%0,%1,%2,%3}, [%4];"
                     : "=f"(x.x), "=f"(x.y), "=f"(x.z), "=f"(x.w) : "r"(raddr) : "memory");
        acc4.x += x.x; acc4.y += x.y; acc4.z += x.z; acc4.w += x.w;
      }
      const int row = m_tile * BM + rr;
      if (row < g.M) {
        const size_t off = (size_t)row * g.N + (size_t)n_tile * BN + cc;
        if (g.addend) {
          const uint2 a2 = *reinterpret_cast<const uint2*>(g.addend + off);
          const float2 lo = bf16x2_to_float2(a2.x), hi = bf16x2_to_float2(a2.y);
          acc4.x += lo.x; acc4.y += lo.y; acc4.z += hi.x; acc4.w += hi.y;
        }
        *reinterpret_cast<uint2*>(g.C + off) =
            make_uint2(float2_to_bf16x2(acc4.x, acc4.y), float2_to_bf16x2(acc4.z, acc4.w));
      }
    }
    cluster_sync_all();                               // nobody exits while a peer reads its SMEM
    return;
  }
  if (gridDim.z > 1) {
    // last-arriving split for this tile finalises: ws (+addend) -> bf16 C, ws := 0
    __threadfence();
    __syncthreads();
    const unsigned int tile_id = m_tile * gridDim.x + n_tile;
    if (threadIdx.x == 0) s_last = (atomicAdd(&g.tickets[tile_id], 1u) == gridDim.z - 1) ? 1u : 0u;
    __syncthreads();
    if (s_last) {
      __threadfence();
      for (int idx = threadIdx.x; idx < BM * BN / 8; idx += blockDim.x) {
        const int rr = idx / (BN / 8), cc = (idx % (BN / 8)) * 8;
        const int row = m_tile * BM + rr;
        if (row >= g.M) continue;
        const size_t off = (size_t)row * g.N + (size_t)n_tile * BN + cc;
        float f[8];
        const uint4 lo = __ldcg(reinterpret_cast<const uint4*>(g.ws + off));
        const uint4 hi = __ldcg(reinterpret_cast<const uint4*>(g.ws + off + 4));
        f[0] = __uint_as_float(lo.x); f[1] = __uint_as_float(lo.y); f[2] = __uint_as_float(lo.z);
        f[3] = __uint_as_float(lo.w); f[4] = __uint_as_float(hi.x); f[5] = __uint_as_float(hi.y);
        f[6] = __uint_as_float(hi.z); f[7] = __uint_as_float(hi.w);
        if (g.addend) {
          float a[8];
          Vec16<__nv_bfloat16>::unpack(ld_v4(g.addend + off), a);
#pragma unroll
          for (int j = 0; j < 8; ++j) f[j] += a[j];
        }
        st_v4(g.C + off, Vec16<__nv_bfloat16>::pack(f));
        __stcg(reinterpret_cast<uint4*>(g.ws + off), make_uint4(0, 0, 0, 0));
        __stcg(reinterpret_cast<uint4*>(g.ws + off + 4), make_uint4(0, 0, 0, 0));
      }
      if (threadIdx.x == 0) g.tickets[tile_id] = 0;
    }
  }
}

// ------------------------------------------- LSTM recurrence: cell backward fused into dm
//
// One backward time step of the LSTMP recurrence in place of (dm = dh·W_P^T GEMM, cell kernel):
// dm = dh · W_P^T (A = dh [M, P], Bt = W_P [S, P], both K-contiguous, K = P) with the cell
// backward in the epilogue, so dm never makes a round trip through global memory.  While thread 0
// streams the GEMM operands, warps 1-3 of the producer warpgroup copy the epilogue's operands for
// the CTA's 128×BN tile (act, c_prev, c_new, dc) into shared memory with cp.async, so their load
// latency hides under the GEMM.  The tile of dm is rounded to bf16 (what a bf16 GEMM would
// store), parked in shared memory, and all 384 threads then run the cell backward over it in
// 4-unit vectors, writing the four dgates columns and dc in place.
struct CellBwdArgs {
  float* dc;                    // [M, S] fp32: in dL/dc_new, out dL/dc_prev
  const __nv_bfloat16* act;     // [M, 4S] σ(i) | tanh(j) | σ(f) | σ(o)
  const float* c_prev;          // [M, S]
  const float* c_new;           // [M, S]
  __nv_bfloat16* dgates;        // [M, 4S]
  int S, K;                     // K = P
};

__device__ __forceinline__ void cp_async_16(void* smem_dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(src)
               : "memory");
}

template <int BN>
__host__ __device__ constexpr int dm_cell_stages() { return BN >= 64 ? 2 : 4; }
// epilogue operands in shared memory: act [4][128][BN] bf16, then c_prev, c_new, dc [128][BN] fp32
template <int BN>
__host__ __device__ constexpr int dm_cell_epi_bytes() { return 4 * BM * BN * 2 + 3 * BM * BN * 4; }

template <int BN>
__global__ void __launch_bounds__(THREADS, 1)
px_lstm_dm_cell_bwd_kernel(const __grid_constant__ CUtensorMap tmap_a,
                           const __grid_constant__ CUtensorMap tmap_b, CellBwdArgs g) {
  constexpr int STAGES = dm_cell_stages<BN>();
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  constexpr int STAGE_BYTES = BM * BK * 2 + BN * BK * 2;
  static_assert(BM * (BN + 4) * 4 <= STAGES * STAGE_BYTES, "dm tile must fit the drained stages");
  __nv_bfloat16* s_act = reinterpret_cast<__nv_bfloat16*>(smem + STAGES * STAGE_BYTES);
  float* s_f32 = reinterpret_cast<float*>(s_act + 4 * BM * BN);   // c_prev | c_new | dc
  uint64_t* full_bar =
      reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES + dm_cell_epi_bytes<BN>());
  uint64_t* empty_bar = full_bar + STAGES;
  const int n_tile = blockIdx.x, m_tile = blockIdx.y;
  const int S = g.S, row0 = m_tile * BM, n0 = n_tile * BN;
  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_a) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_b) : "memory");
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x >= 32 && threadIdx.x < 128) {
    const int t = threadIdx.x - 32;
    constexpr int ACH = BN * 2 / 16, FCH = BN * 4 / 16;   // 16-byte chunks per row segment
    for (int i = t; i < 4 * BM * ACH; i += 96) {
      const int q = i / (BM * ACH), r = (i / ACH) % BM, c = i % ACH;
      cp_async_16(s_act + (size_t)(q * BM + r) * BN + c * 8,
                  g.act + (size_t)(row0 + r) * 4 * S + (size_t)q * S + n0 + c * 8);
    }
    for (int i = t; i < 3 * BM * FCH; i += 96) {
      const int a = i / (BM * FCH), r = (i / FCH) % BM, c = i % FCH;
      const float* src = a == 0 ? g.c_prev : (a == 1 ? g.c_new : g.dc);
      cp_async_16(s_f32 + (size_t)(a * BM + r) * BN + c * 4, src + (size_t)(row0 + r) * S + n0 + c * 4);
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
  }
  float acc[BN / 2];
  mainloop<BN, STAGES>(&tmap_a, &tmap_b, smem, full_bar, empty_bar, 0, g.K / BK, row0, n0, acc);
  float* park = reinterpret_cast<float*>(smem);
  if (threadIdx.x >= 128) {
    consumer_sync();                                // both warpgroups' wgmma have retired
    park_acc<BN, true>(park, acc);
  }
  __syncthreads();
  for (int v = threadIdx.x; v < BM * BN / 4; v += THREADS) {
    const int r = v / (BN / 4), c4 = (v % (BN / 4)) * 4;
    const size_t ci = (size_t)(row0 + r) * S + n0 + c4, gi = (size_t)(row0 + r) * 4 * S + n0 + c4;
    const float4 dm4 = *reinterpret_cast<const float4*>(park + (size_t)r * (BN + 4) + c4);
    const float4 cp4 = *reinterpret_cast<const float4*>(s_f32 + (size_t)r * BN + c4);
    const float4 cn4 = *reinterpret_cast<const float4*>(s_f32 + (size_t)(BM + r) * BN + c4);
    const float4 dc4 = *reinterpret_cast<const float4*>(s_f32 + (size_t)(2 * BM + r) * BN + c4);
    float a[4][4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint2 w = *reinterpret_cast<const uint2*>(s_act + (size_t)(q * BM + r) * BN + c4);
      const float2 lo = bf16x2_to_float2(w.x), hi = bf16x2_to_float2(w.y);
      a[q][0] = lo.x; a[q][1] = lo.y; a[q][2] = hi.x; a[q][3] = hi.y;
    }
    const float dmv[4] = {dm4.x, dm4.y, dm4.z, dm4.w}, cp[4] = {cp4.x, cp4.y, cp4.z, cp4.w},
                cn[4] = {cn4.x, cn4.y, cn4.z, cn4.w}, dci[4] = {dc4.x, dc4.y, dc4.z, dc4.w};
    float dg[4][4], dco[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float ae[4] = {a[0][e], a[1][e], a[2][e], a[3][e]};
      float dge[4];
      dco[e] = lstm_cell_bwd_elem(ae, cp[e], cn[e], dmv[e], dci[e], dge);
#pragma unroll
      for (int q = 0; q < 4; ++q) dg[q][e] = dge[q];
    }
#pragma unroll
    for (int q = 0; q < 4; ++q)
      *reinterpret_cast<uint2*>(g.dgates + gi + (size_t)q * S) =
          make_uint2(float2_to_bf16x2(dg[q][0], dg[q][1]), float2_to_bf16x2(dg[q][2], dg[q][3]));
    *reinterpret_cast<float4*>(g.dc + ci) = make_float4(dco[0], dco[1], dco[2], dco[3]);
  }
}

// ------------------------------------------------------------------ host side

template <int BN, int STAGES>
constexpr int smem_bytes() { return STAGES * (BM * BK * 2 + BN * BK * 2) + 1024 + 256; }

// opt a kernel in to `bytes` of dynamic shared memory once
template <auto Kernel>
static void set_smem_once(int bytes) {
  static bool done = false;
  if (done) return;
  cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  done = true;
}

}  // namespace tc

extern "C" {

// C[M,N] = A[M,K] · B[N,K]^T (+ addend).  splits > 1 needs ws (fp32 [M,N], zero)
// and tickets (uint32 [tiles], zero).  Returns 0 or a negative error.
// cluster != 0: the splits of a tile reduce through DSMEM in a (1,1,splits) cluster (splits must
// divide 128 and be <= 16; 16 needs the non-portable cluster size); ws / tickets unused.
int px_gemm_tc(const void* A, const void* B, void* C, const void* addend, float* ws,
               unsigned int* tickets, int M, int N, int K, int splits, int bn, int cluster,
               cudaStream_t stream) {
  using namespace tc;
  if (M % BM || K % BK || (bn != 64 && bn != 128) || N % bn) return -1;
  if (splits < 1 || K % (splits * BK)) return -2;
  if (cluster && (splits < 2 || splits > 16 || (BM % splits) != 0)) return -4;
  if (splits > 1 && !cluster && (!ws || !tickets)) return -3;
  CUtensorMap ta, tb;
  int rc = make_tmap(&ta, A, M, K, BM);
  if (rc) return rc;
  rc = make_tmap(&tb, B, N, K, bn);
  if (rc) return rc;
  GemmArgs g;
  g.C = (__nv_bfloat16*)C; g.addend = (const __nv_bfloat16*)addend; g.ws = ws;
  g.tickets = tickets; g.M = M; g.N = N; g.K = K; g.k_per_split = K / splits;
  dim3 grid(N / bn, M / BM, splits);
  constexpr int STAGES = 4;
  if (cluster) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = dim3(THREADS); cfg.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = 1; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = splits;
    cfg.attrs = at; cfg.numAttrs = 1;
    cudaError_t e;
    if (bn == 128) {
      constexpr int SMEM = smem_bytes<128, STAGES>();
      static bool setc128 = false;
      if (!setc128) {
        cudaFuncSetAttribute(px_gemm_tc_kernel<128, STAGES, true>,
                             cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
        cudaFuncSetAttribute(px_gemm_tc_kernel<128, STAGES, true>,
                             cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
        setc128 = true;
      }
      cfg.dynamicSmemBytes = SMEM;
      e = cudaLaunchKernelEx(&cfg, px_gemm_tc_kernel<128, STAGES, true>, ta, tb, g);
    } else {
      constexpr int SMEM = smem_bytes<64, STAGES>();
      static bool setc64 = false;
      if (!setc64) {
        cudaFuncSetAttribute(px_gemm_tc_kernel<64, STAGES, true>,
                             cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
        cudaFuncSetAttribute(px_gemm_tc_kernel<64, STAGES, true>,
                             cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
        setc64 = true;
      }
      cfg.dynamicSmemBytes = SMEM;
      e = cudaLaunchKernelEx(&cfg, px_gemm_tc_kernel<64, STAGES, true>, ta, tb, g);
    }
    return e == cudaSuccess ? (int)cudaGetLastError() : (int)e;
  }
  if (bn == 128) {
    constexpr int SMEM = smem_bytes<128, STAGES>();
    static bool set128 = false;
    if (!set128) {
      cudaFuncSetAttribute(px_gemm_tc_kernel<128, STAGES, false>,
                           cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
      set128 = true;
    }
    px_gemm_tc_kernel<128, STAGES, false><<<grid, THREADS, SMEM, stream>>>(ta, tb, g);
  } else {
    constexpr int SMEM = smem_bytes<64, STAGES>();
    static bool set64 = false;
    if (!set64) {
      cudaFuncSetAttribute(px_gemm_tc_kernel<64, STAGES, false>,
                           cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
      set64 = true;
    }
    px_gemm_tc_kernel<64, STAGES, false><<<grid, THREADS, SMEM, stream>>>(ta, tb, g);
  }
  return (int)cudaGetLastError();
}


// One backward time step: dm = dh · W_P^T (dh [M, P], W_P [S, P]) with the cell backward in the
// epilogue (see `px_lstm_dm_cell_bwd_kernel`).  bn: 16, 32 or 64 columns of dm per CTA.  Every
// pointer 16-byte aligned.
int px_lstm_dm_cell_bwd(const void* dh, const void* WP, float* dc, const void* act,
                        const float* c_prev, const float* c_new, void* dgates, int M, int S, int P,
                        int bn, cudaStream_t stream) {
  using namespace tc;
  if (M % BM || P % BK || (bn != 16 && bn != 32 && bn != 64) || S % bn) return -1;
  for (const void* q : {dh, WP, (const void*)dc, act, (const void*)c_prev, (const void*)c_new,
                        (const void*)dgates})
    if ((uintptr_t)q % 16) return -1;
  CUtensorMap ta, tb;
  int rc = make_tmap(&ta, dh, M, P, BM);
  if (rc) return rc;
  rc = make_tmap(&tb, WP, S, P, bn);
  if (rc) return rc;
  CellBwdArgs g;
  g.dc = dc; g.act = (const __nv_bfloat16*)act; g.c_prev = c_prev; g.c_new = c_new;
  g.dgates = (__nv_bfloat16*)dgates; g.S = S; g.K = P;
  dim3 grid(S / bn, M / BM);
#define PX_DMB(BN_)                                                                            \
  {                                                                                            \
    constexpr int SMEM = smem_bytes<BN_, dm_cell_stages<BN_>()>() + dm_cell_epi_bytes<BN_>();  \
    set_smem_once<px_lstm_dm_cell_bwd_kernel<BN_>>(SMEM);                                      \
    px_lstm_dm_cell_bwd_kernel<BN_><<<grid, THREADS, SMEM, stream>>>(ta, tb, g);               \
  }
  if (bn == 16) PX_DMB(16) else if (bn == 32) PX_DMB(32) else PX_DMB(64)
#undef PX_DMB
  return (int)cudaGetLastError();
}

}  // extern "C"
