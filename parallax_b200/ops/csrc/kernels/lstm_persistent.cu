// The forward recurrence of an LSTMP layer as ONE persistent cooperative kernel: all T time steps
// of `_LSTMLayerFn.forward` with the recurrent weights resident in shared memory.
//
// Per time step t, with h_t = h_all[t] [B, P], B = 128:
//   phase A  gates = xw[t] + h_t·Wh (fp32, rounded to bf16 as the cuBLAS addmm stores it), the
//            LSTM cell (`lstm_cell_fwd_elem`), act[t], c_all[t+1] and m_all[t] to memory
//   grid barrier: m_t is complete
//   phase B  partial products m_t[:, K-slice]·W_P[K-slice, N-tile] into fixed fp32 slots ws[slice]
//   grid barrier: every slot is written
//   reduce   h_all[t+1] = Σ_slice ws[slice] in slice order (no atomics: the bits do not depend on
//            which CTA finishes first), bf16
//   grid barrier: h_{t+1} is complete
//
// CTA j owns 32 LSTM units for 64 of the 128 rows (rows 64·(j % 2) …, units u0 = 32·(j / 2) …), so a
// step reads half of h_t per CTA (64 KB at P 512; 8 MB over the grid instead of 16 MB with all 128
// rows × 16 units).  Warpgroups 0 and 1 run the products: warpgroup w takes units u0 + 16w …
// u0 + 16w + 15, whose 64 gate columns {g·S + u} are the N side of `wgmma m64n64k16`.  They park
// the fp32 gate tile in shared memory (over h_t, which the product no longer needs), and all 512
// threads run the cell on it, 4 units of one row each, with c in registers across steps.  The
// cell (IEEE divides, five exponentials per unit) is the longest part of a step: on the two
// product warpgroups alone, 8 warps per SM, it took about 4 µs of a step's phase A; with 16 warps
// its latency hides better and its loads and stores are 8- and 16-byte vectors.
// The CTA's slice of Wh (P × 128 bf16, 128 KB at P 512) is copied once, transposed to the K-major
// 128B-swizzled layout of the other wgmma kernels (`wgmma.cuh`) in registers, from 16-byte loads
// along Wh's rows.  The first (P/64)·(S/128) CTAs also hold a 128 × 64 slice of W_P (16 KB) for
// phase B.  h_t (A of phase A, all P/64 K-blocks) and m_t's K-slice (A of phase B) arrive by TMA.
//
// Memory ordering: m_t, ws and h_{t+1} are written by other CTAs of the same launch, so they are
// never read through L1 or the non-coherent path: h and m by TMA (L2) after
// `fence.proxy.async.global` (generic-proxy stores, async-proxy loads), ws by `ld.global.cg`.
// The barriers are `cooperative_groups::this_grid().sync()` (release/acquire fences around an
// arrival counter in the launch's own workspace, so a CUDA-graph replay needs no reset), and the
// launch is cooperative, so every CTA is resident.
#include <cooperative_groups.h>
#include <mutex>

#include "wgmma.cuh"
#include "lstm_cell.cuh"

namespace cg = cooperative_groups;

namespace lstm_fwd {
using namespace tc;

constexpr int UNITS = 32;          // LSTM units per CTA, 16 per warpgroup
constexpr int ROWS = 64;           // rows per CTA: half of the batch
constexpr int GN = 2 * UNITS;      // gate columns per warpgroup: N of the phase-A product
constexpr int PN = 64;             // h columns per phase-B tile
constexpr int PK = 128;            // m columns (K) per phase-B tile: one fp32 slot per K-slice
constexpr int NTHREADS = 512;      // warpgroups 0, 1: products; all four: cell and reduction
constexpr int CELL_U = 4;          // units per thread in the cell: 8 threads per row
constexpr int GATE_LD = 4 * UNITS + 8;   // fp32 row pitch of the parked gate tile (+8: 2-way
                                         // bank conflicts at most on the accumulator stores)
constexpr int MAX_KB = 8;          // P <= 512: h_t fits beside the resident weights

struct Args {
  const __nv_bfloat16* xw;         // [T, B, 4S]  x·Wx + bias
  const __nv_bfloat16* Wh;         // [P, 4S]
  const __nv_bfloat16* WP;         // [S, P]
  __nv_bfloat16* act;              // [T, B, 4S]  σ(i) | tanh(j) | σ(f) | σ(o)
  float* c_all;                    // [T+1, B, S] (row 0: c0, read)
  __nv_bfloat16* m_all;            // [T, B, S]
  __nv_bfloat16* h_all;            // [T+1, B, P] (row 0: h0, read)
  float* ws;                       // [S/PK, B, P] phase-B partial products
  int T, S, P;
  float forget_bias;
};

// the A operand region: h_t's rows (P/64 blocks of 64 rows) or m_t's K-slice (2 blocks of 128),
// and the parked fp32 gate tile
__host__ __device__ constexpr int cmax(int a, int b) { return a > b ? a : b; }
__host__ __device__ constexpr int x_bytes(int P) {
  return cmax(cmax((P / BK) * ROWS * 128, (PK / BK) * BM * 128), ROWS * GATE_LD * 4);
}
// Wh slices of both warpgroups | W_P slice | A operand | mbarriers, after 1024-byte alignment
__host__ __device__ constexpr int smem_bytes(int P) {
  return 2 * (P / BK) * GN * 128 + (PK / BK) * PN * 128 + x_bytes(P) + (MAX_KB + PK / BK) * 8 + 1024;
}
static_assert(smem_bytes(MAX_KB * BK) <= 232448, "P = 512 must fit one CTA's shared memory");

// dst <- the K-major 128B-swizzled image of the [K, N] block src(k, n) = src[k·ld + col(n)] (N
// contiguous in memory, col(n0 .. n0+7) consecutive for n0 % 8 = 0): K-block kb holds N rows of
// 128 B (64 k), chunk c of row n at c ^ (n % 8).  Each thread moves 8×8 blocks: eight 16-byte
// loads along n, transposed in registers.
template <int N, typename Col>
__device__ __forceinline__ void load_transposed(uint8_t* dst, const __nv_bfloat16* src, size_t ld,
                                                int K, Col col) {
  const int nblk = (N / 8) * (K / 8);
  for (int b = threadIdx.x; b < nblk; b += blockDim.x) {
    const int n0 = (b % (N / 8)) * 8, k0 = (b / (N / 8)) * 8;
    uint4 v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
      v[i] = __ldg(reinterpret_cast<const uint4*>(src + (size_t)(k0 + i) * ld + col(n0)));
    const uint32_t* w = reinterpret_cast<const uint32_t*>(v);
    uint8_t* blk = dst + (k0 / BK) * N * 128;
    const int c = (k0 % BK) / 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t sel = (j & 1) ? 0x7632u : 0x5410u;
      uint4 o;
      o.x = __byte_perm(w[0 * 4 + j / 2], w[1 * 4 + j / 2], sel);
      o.y = __byte_perm(w[2 * 4 + j / 2], w[3 * 4 + j / 2], sel);
      o.z = __byte_perm(w[4 * 4 + j / 2], w[5 * 4 + j / 2], sel);
      o.w = __byte_perm(w[6 * 4 + j / 2], w[7 * 4 + j / 2], sel);
      const int n = n0 + j;
      *reinterpret_cast<uint4*>(blk + n * 128 + ((c ^ (n & 7)) << 4)) = o;
    }
  }
}

__device__ __forceinline__ float2 bf16x2_to_float2(uint32_t w) {
  return make_float2(__uint_as_float(w << 16), __uint_as_float(w & 0xffff0000u));
}
__device__ __forceinline__ uint32_t float2_to_bf16x2(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float round_bf16(float x) {
  return __bfloat162float(__float2bfloat16_rn(x));
}

// acc (this warpgroup's 64 × N tile, layout of `tc::mainloop`) = A · B over nkb K-blocks: the
// warpgroup's A rows of K-block kb at a0 + kb·a_stride, its N B rows at b0 + kb·b_stride; K-block
// kb is complete once bar[kb] completes its phase `parity`.
template <int N>
__device__ __forceinline__ void product(float* acc, uint32_t a0, uint32_t a_stride, uint32_t b0,
                                        uint32_t b_stride, uint64_t* bar, int nkb,
                                        uint32_t parity) {
  for (int kb = 0; kb < nkb; ++kb) {
    mbar_wait(&bar[kb], parity);
    const uint64_t adesc = make_smem_desc(a0 + kb * a_stride);
    const uint64_t bdesc = make_smem_desc(b0 + kb * b_stride);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / WG_K; ++k)
      wgmma_bf16<N>(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2),
                    (kb | k) != 0 ? 1u : 0u);
    wgmma_commit();
  }
  wgmma_wait<0>();
}

__global__ void __launch_bounds__(NTHREADS, 1)
px_lstm_fwd_persistent_kernel(const __grid_constant__ CUtensorMap tmap_h,
                              const __grid_constant__ CUtensorMap tmap_m, Args a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const int S = a.S, P = a.P, KB = P / BK;
  const size_t G4 = 4 * (size_t)S;
  uint8_t* sWh = smem;                                // [warpgroup][K-block][64 rows × 128 B]
  uint8_t* sWP = sWh + 2 * KB * GN * 128;
  uint8_t* sX = sWP + (PK / BK) * PN * 128;
  uint64_t* hbar = reinterpret_cast<uint64_t*>(sX + x_bytes(P));
  uint64_t* mbar = hbar + MAX_KB;

  const int row0 = (blockIdx.x & 1) * ROWS, u0 = (blockIdx.x >> 1) * UNITS;
  const int ntn = P / PN;
  const bool proj = (int)blockIdx.x < ntn * (S / PK);      // takes part in phase B
  const int pn0 = (blockIdx.x % ntn) * PN, pk = blockIdx.x / ntn;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_h) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_m) : "memory");
    for (int kb = 0; kb < KB; ++kb) mbar_init(&hbar[kb], 1);
    for (int kb = 0; kb < PK / BK; ++kb) mbar_init(&mbar[kb], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // gate column n = g·16 + u of warpgroup w is column g·S + u0 + 16w + u of Wh (and of xw, act)
  for (int w = 0; w < 2; ++w)
    load_transposed<GN>(sWh + w * KB * GN * 128, a.Wh, G4, P,
                        [=](int n) { return (n / 16) * S + u0 + 16 * w + n % 16; });
  if (proj)
    load_transposed<PN>(sWP, a.WP + (size_t)pk * PK * P, P, PK, [=](int n) { return pn0 + n; });
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // st.shared -> wgmma reads
  __syncthreads();

  // product warpgroups: accumulator element acc[j·4 + 2h + e] is row r + 8h, column j·8 + q2 + e
  // of the warpgroup's tile; in phase A, with j = 2g + uh, gate g of unit 16·wg + uh·8 + q2 + e
  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31, warp = (threadIdx.x >> 5) & 3;
  const int q2 = (lane & 3) * 2;
  const int r = warp * 16 + (lane >> 2);                  // phase A rows r, r + 8 of the CTA's 64
  const int rb = wg * 64 + r;                             // phase B rows rb, rb + 8
  // cell threads: units cu … cu + 3 of the CTA's row crow, i.e. row0 + crow of the batch
  const int crow = threadIdx.x / (UNITS / CELL_U), cu = (threadIdx.x % (UNITS / CELL_U)) * CELL_U;
  const size_t cs_off = (size_t)(row0 + crow) * S + u0 + cu;          // in [B, S]
  const size_t cg_off = (size_t)(row0 + crow) * G4 + u0 + cu;         // in [B, 4S], gate 0
  float c[CELL_U];
  {
    const float4 v = *reinterpret_cast<const float4*>(a.c_all + cs_off);
    c[0] = v.x; c[1] = v.y; c[2] = v.z; c[3] = v.w;
  }
  float* sG = reinterpret_cast<float*>(sX);               // parked gates [row][gate][unit]
  const uint32_t sX_u = smem_u32(sX), sWh_u = smem_u32(sWh) + (wg & 1) * KB * GN * 128;
  const uint32_t sWP_u = smem_u32(sWP);
  cg::grid_group grid = cg::this_grid();
  const int KS = S / PK;
  float acc[32];

  for (int t = 0; t < a.T; ++t) {
    const uint32_t parity = t & 1;
    // ------------------------------------------------------------ phase A: gates and cell
    if (threadIdx.x == 0) {
      asm volatile("fence.proxy.async.global;" ::: "memory");   // h_t: generic stores -> TMA
      for (int kb = 0; kb < KB; ++kb) {
        mbar_expect_tx(&hbar[kb], ROWS * BK * 2);
        tma_load_2d(sX + kb * ROWS * 128, &tmap_h, &hbar[kb], kb * BK, t * BM + row0);
      }
    }
    // this thread's xw[t] quads, loaded under the product: [g] 4 × bf16
    uint2 xv[4];
    const __nv_bfloat16* xr = a.xw + (size_t)t * BM * G4 + cg_off;
#pragma unroll
    for (int g = 0; g < 4; ++g) xv[g] = __ldg(reinterpret_cast<const uint2*>(xr + (size_t)g * S));
    if (wg < 2) {
      product<GN>(acc, sX_u, ROWS * 128, sWh_u, GN * 128, hbar, KB, parity);
      consumer_sync();                                // both warpgroups' wgmma have retired
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < GN / 8; ++j)
          *reinterpret_cast<float2*>(sG + (r + 8 * h) * GATE_LD + (j >> 1) * UNITS + wg * 16 +
                                     (j & 1) * 8 + q2) =
              make_float2(acc[j * 4 + 2 * h], acc[j * 4 + 2 * h + 1]);
    }
    __syncthreads();

    float av[4][CELL_U], mv[CELL_U];
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const float4 v = *reinterpret_cast<const float4*>(sG + crow * GATE_LD + g * UNITS + cu);
      const float2 lo = bf16x2_to_float2(xv[g].x), hi = bf16x2_to_float2(xv[g].y);
      // gate pre-activation rounded to bf16, as the addmm of the per-step path stores it
      av[g][0] = round_bf16(v.x + lo.x);
      av[g][1] = round_bf16(v.y + lo.y);
      av[g][2] = round_bf16(v.z + hi.x);
      av[g][3] = round_bf16(v.w + hi.y);
    }
    // the parked tile is read: later TMA writes into this region come after these reads
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
#pragma unroll
    for (int e = 0; e < CELL_U; ++e) {
      float ae[4];
      c[e] = lstm_cell_fwd_elem(av[0][e], av[1][e], av[2][e], av[3][e], c[e], a.forget_bias, ae,
                                &mv[e]);
#pragma unroll
      for (int g = 0; g < 4; ++g) av[g][e] = ae[g];
    }
    __nv_bfloat16* act = a.act + (size_t)t * BM * G4 + cg_off;
#pragma unroll
    for (int g = 0; g < 4; ++g)
      *reinterpret_cast<uint2*>(act + (size_t)g * S) =
          make_uint2(float2_to_bf16x2(av[g][0], av[g][1]), float2_to_bf16x2(av[g][2], av[g][3]));
    *reinterpret_cast<float4*>(a.c_all + (size_t)(t + 1) * BM * S + cs_off) =
        make_float4(c[0], c[1], c[2], c[3]);
    *reinterpret_cast<uint2*>(a.m_all + (size_t)t * BM * S + cs_off) =
        make_uint2(float2_to_bf16x2(mv[0], mv[1]), float2_to_bf16x2(mv[2], mv[3]));
    grid.sync();                                      // m_t is complete

    // ------------------------------------------------------------ phase B: split-K projection
    if (proj && wg < 2) {
      if (threadIdx.x == 0) {
        asm volatile("fence.proxy.async.global;" ::: "memory");   // m_t: generic -> TMA
        for (int kb = 0; kb < PK / BK; ++kb) {
          mbar_expect_tx(&mbar[kb], BM * BK * 2);
          tma_load_2d(sX + kb * BM * 128, &tmap_m, &mbar[kb], pk * PK + kb * BK, t * BM);
        }
      }
      product<PN>(acc, sX_u + wg * 64 * 128, BM * 128, sWP_u, PN * 128, mbar, PK / BK, parity);
      float* slot = a.ws + (size_t)pk * BM * P;
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < PN / 8; ++j)
          *reinterpret_cast<float2*>(slot + (size_t)(rb + 8 * h) * P + pn0 + j * 8 + q2) =
              make_float2(acc[j * 4 + 2 * h], acc[j * 4 + 2 * h + 1]);
    }
    grid.sync();                                      // every slot is written

    // ------------------------------------------------------------ h_{t+1}: slots in order
    __nv_bfloat16* hn = a.h_all + (size_t)(t + 1) * BM * P;
    const int npairs = BM * P / 2;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < npairs; i += gridDim.x * blockDim.x) {
      float2 s = __ldcg(reinterpret_cast<const float2*>(a.ws) + i);
#pragma unroll 8
      for (int k = 1; k < KS; ++k) {
        const float2 v = __ldcg(reinterpret_cast<const float2*>(a.ws + (size_t)k * BM * P) + i);
        s.x += v.x;
        s.y += v.y;
      }
      reinterpret_cast<uint32_t*>(hn)[i] = float2_to_bf16x2(s.x, s.y);
    }
    if (t + 1 < a.T) grid.sync();                     // h_{t+1} is complete
  }
}

// `grid` when the current device can keep that many CTAs of `Kernel` (NTHREADS threads, smem(P)
// bytes of dynamic shared memory) resident in one cooperative launch, else 0.  Cooperative-launch
// support and occupancy × SMs are queried once per kernel, device and P/64.
template <auto Kernel, int (*Smem)(int)>
int persistent_grid(int grid, int P) {
  static std::mutex mu;
  static int cap[16][MAX_KB + 1];                     // [device][P/64]: resident CTAs, 0 = unknown
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 16) return 0;
  std::lock_guard<std::mutex> lock(mu);
  int& n = cap[dev][P / BK];
  if (n == 0) {
    int coop = 0, sms = 0, per_sm = 0;
    cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    // the limit for the widest P, so that a query for a narrower layer never lowers it
    if (cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             Smem(MAX_KB * BK)) != cudaSuccess ||
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, Kernel, NTHREADS, Smem(P)) !=
            cudaSuccess)
      per_sm = 0;
    n = (coop && per_sm > 0) ? per_sm * sms : -1;
    cudaGetLastError();
  }
  return n >= grid ? grid : 0;
}

// One cooperative launch of `Kernel` on `grid` CTAs of NTHREADS threads.
template <typename... KArgs, typename... Args>
int launch_cooperative(void (*kernel)(KArgs...), int grid, int smem, cudaStream_t stream,
                       Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(NTHREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeCooperative;
  at[0].val.cooperative = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, args...);
  return e == cudaSuccess ? (int)cudaGetLastError() : (int)e;
}

}  // namespace lstm_fwd

// The backward recurrence of the same layer as ONE persistent cooperative kernel: all T steps of
// `_LSTMLayerFn.backward`, t = T-1 … 0, with dh_t = dh_tot[t] [B, P]:
//   phase 1  dm = dh_t·W_P^T (fp32, rounded to bf16 as the per-step kernel rounds it), the cell
//            backward (`lstm_cell_bwd_elem`) with dc in registers, dgates[t] to memory
//   grid barrier: dgates_t is complete
//   phase 2  partial products dgates_t[:, K-slice]·Wh[N-tile, K-slice]^T into fixed fp32 slots
//            ws[slice]
//   grid barrier: every slot is written
//   sum      dh_tot[t-1] = Σ_slice ws[slice] in slice order, + dH[t-1], bf16 (the order of the
//            per-step product's cluster reduction: partials first, then the addend); at t = 0
//            dh_rec = Σ_slice ws[slice], no addend
//   grid barrier: dh_tot[t-1] is complete (not after t = 0)
//
// Same grid as the forward: CTA j owns 32 units for 64 of the 128 rows.  Phase 1 runs on
// warpgroups 0 and 1 (16 units each, `wgmma m64n16k16`, K = P); its B operand, W_P's 32 rows of
// the CTA's units, is already K-contiguous and arrives by TMA once at launch (32 KB at P 512);
// dh_t's 64 rows arrive by TMA every step (64 KB).  All 512 threads run the cell, 4 units of one
// row each (the forward cell's mapping), with act[t], c_all[t] and c_all[t+1] loaded under the
// product.  Phase 2 has (P/64)·(4S/512) work items of 64 dh columns × 512 dgates columns, one per
// CTA at P 512; each item's Wh tile (K-contiguous in Wh, 64 KB) is resident from launch, and its
// dgates_t K-slice (128 rows × 512, 128 KB) arrives by TMA.  All four warpgroups take part:
// warpgroup w multiplies rows 64·(w % 2) … by columns 32·(w / 2) … of the item (m64n32k16).
//
// Memory ordering is the forward's: dgates_t and dh_tot[t-1], written by other CTAs of the launch,
// are read only by TMA after `fence.proxy.async.global`; the slots with `ld.global.cg`.  Inputs of
// the launch (dH, act, c_all, the weights) are read-only in it.
namespace lstm_bwd {
using namespace lstm_fwd;

constexpr int WN = 64;             // dh columns per phase-2 work item
constexpr int WK = 512;            // dgates columns (K) per phase-2 work item: one slot per K-slice
constexpr int DM_LD = UNITS + 8;   // fp32 row pitch of the parked dm tile

struct Args {
  const __nv_bfloat16* dH;         // [T, B, P]
  const __nv_bfloat16* act;        // [T, B, 4S]
  const float* c_all;              // [T+1, B, S]
  float* dc;                       // [B, S]  in dL/dc_T, out dL/dc_0
  __nv_bfloat16* dgates;           // [T, B, 4S]
  __nv_bfloat16* dh_tot;           // [T, B, P] (row T-1 read: dH[T-1] + dh_T)
  __nv_bfloat16* dh_rec;           // [B, P]  dgates[0]·Wh^T
  float* ws;                       // [4S/WK, B, P] phase-2 partial products
  int T, S, P;
};

// W_P's rows of the CTA's units | the A operand: dh_t's rows (P/64 blocks of 64 rows) or a dgates_t
// K-slice (WK/64 blocks of 128 rows), and the parked dm tile
__host__ __device__ constexpr int wp_bytes(int P) { return (P / BK) * UNITS * 128; }
__host__ __device__ constexpr int x_bytes(int P) {
  return cmax(cmax((P / BK) * ROWS * 128, (WK / BK) * BM * 128), ROWS * DM_LD * 4);
}
// Wh tile | W_P slice | A operand | mbarriers, after 1024-byte alignment
__host__ __device__ constexpr int smem_bytes(int P) {
  return (WK / BK) * WN * 128 + wp_bytes(P) + x_bytes(P) + (MAX_KB + WK / BK + 1) * 8 + 1024;
}
static_assert(smem_bytes(MAX_KB * BK) <= 232448, "P = 512 must fit one CTA's shared memory");
static_assert(WN / 2 >= UNITS / 2, "the accumulator holds phase 1's tile too");

__global__ void __launch_bounds__(NTHREADS, 1)
px_lstm_bwd_persistent_kernel(const __grid_constant__ CUtensorMap tmap_dh,
                              const __grid_constant__ CUtensorMap tmap_wp,
                              const __grid_constant__ CUtensorMap tmap_dg,
                              const __grid_constant__ CUtensorMap tmap_wh, Args a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const int S = a.S, P = a.P, KB = P / BK;
  const size_t G4 = 4 * (size_t)S;
  uint8_t* sWh = smem;                                // [K-block][WN rows × 128 B]
  uint8_t* sWP = sWh + (WK / BK) * WN * 128;          // [K-block][UNITS rows × 128 B]
  uint8_t* sX = sWP + wp_bytes(P);
  uint64_t* hbar = reinterpret_cast<uint64_t*>(sX + x_bytes(P));
  uint64_t* gbar = hbar + MAX_KB;
  uint64_t* wbar = gbar + WK / BK;

  const int row0 = (blockIdx.x & 1) * ROWS, u0 = (blockIdx.x >> 1) * UNITS;
  const int ntn = P / WN, NS = (int)(G4 / WK);
  const bool item = (int)blockIdx.x < ntn * NS;       // takes part in phase 2
  const int n0 = (blockIdx.x % ntn) * WN, ks = blockIdx.x / ntn;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_dh) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_wp) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_dg) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_wh) : "memory");
    for (int kb = 0; kb < KB; ++kb) mbar_init(&hbar[kb], 1);
    for (int kb = 0; kb < WK / BK; ++kb) mbar_init(&gbar[kb], 1);
    mbar_init(wbar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    // the resident operands, once: W_P's rows u0 … u0+31 and the work item's Wh tile
    mbar_expect_tx(wbar, wp_bytes(P) + (item ? (WK / BK) * WN * 128 : 0));
    for (int kb = 0; kb < KB; ++kb)
      tma_load_2d(sWP + kb * UNITS * 128, &tmap_wp, wbar, kb * BK, u0);
    if (item)
      for (int kb = 0; kb < WK / BK; ++kb)
        tma_load_2d(sWh + kb * WN * 128, &tmap_wh, wbar, ks * WK + kb * BK, n0);
  }
  __syncthreads();

  // product warpgroups: accumulator element acc[j·4 + 2h + e] is row r + 8h, column j·8 + q2 + e
  // of the warpgroup's tile; in phase 1 unit 16·wg + j·8 + q2 + e of the CTA's 32
  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31, warp = (threadIdx.x >> 5) & 3;
  const int q2 = (lane & 3) * 2;
  const int r = warp * 16 + (lane >> 2);
  // cell threads: units cu … cu + 3 of the CTA's row crow, i.e. row0 + crow of the batch
  const int crow = threadIdx.x / (UNITS / CELL_U), cu = (threadIdx.x % (UNITS / CELL_U)) * CELL_U;
  const size_t cs_off = (size_t)(row0 + crow) * S + u0 + cu;          // in [B, S]
  const size_t cg_off = (size_t)(row0 + crow) * G4 + u0 + cu;         // in [B, 4S], gate 0
  float dc[CELL_U];
  {
    const float4 v = *reinterpret_cast<const float4*>(a.dc + cs_off);
    dc[0] = v.x; dc[1] = v.y; dc[2] = v.z; dc[3] = v.w;
  }
  float* sD = reinterpret_cast<float*>(sX);               // parked dm [row][unit]
  const uint32_t sX_u0 = smem_u32(sX), sWP_u0 = smem_u32(sWP), sWh_u0 = smem_u32(sWh);
  cg::grid_group grid = cg::this_grid();
  float acc[WN / 4];
  mbar_wait(wbar, 0);

  for (int t = a.T - 1; t >= 0; --t) {
    const uint32_t parity = (a.T - 1 - t) & 1;
    // the shared-memory bases, opaque to the compiler for each step: otherwise it hoists every
    // descriptor of the unrolled products out of the time loop (about 100 registers), and spills
    uint32_t sX_u = sX_u0, sWP_u = sWP_u0, sWh_u = sWh_u0;
    asm volatile("" : "+r"(sX_u), "+r"(sWP_u), "+r"(sWh_u));
    // ------------------------------------------------------------ phase 1: dm and the cell
    if (threadIdx.x == 0) {
      asm volatile("fence.proxy.async.global;" ::: "memory");   // dh_t: generic stores -> TMA
      for (int kb = 0; kb < KB; ++kb) {
        mbar_expect_tx(&hbar[kb], ROWS * BK * 2);
        tma_load_2d(sX + kb * ROWS * 128, &tmap_dh, &hbar[kb], kb * BK, t * BM + row0);
      }
    }
    // this thread's cell operands, loaded under the product
    uint2 av[4];
    const __nv_bfloat16* ar = a.act + (size_t)t * BM * G4 + cg_off;
#pragma unroll
    for (int g = 0; g < 4; ++g) av[g] = __ldg(reinterpret_cast<const uint2*>(ar + (size_t)g * S));
    const float4 cp = __ldg(reinterpret_cast<const float4*>(a.c_all + (size_t)t * BM * S + cs_off));
    const float4 cn =
        __ldg(reinterpret_cast<const float4*>(a.c_all + (size_t)(t + 1) * BM * S + cs_off));
    if (wg < 2) {
      product<UNITS / 2>(acc, sX_u, ROWS * 128, sWP_u + wg * (UNITS / 2) * 128, UNITS * 128, hbar,
                         KB, parity);
      consumer_sync();                                // both warpgroups' wgmma have retired
      // dm rounded to bf16, as the per-step kernel's accumulator is
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < UNITS / 16; ++j)
          *reinterpret_cast<float2*>(sD + (r + 8 * h) * DM_LD + wg * 16 + j * 8 + q2) =
              make_float2(round_bf16(acc[j * 4 + 2 * h]), round_bf16(acc[j * 4 + 2 * h + 1]));
    }
    __syncthreads();
    const float4 dm = *reinterpret_cast<const float4*>(sD + crow * DM_LD + cu);
    // the parked tile is read: later TMA writes into this region come after these reads
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    float ag[4][CELL_U];
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const float2 lo = bf16x2_to_float2(av[g].x), hi = bf16x2_to_float2(av[g].y);
      ag[g][0] = lo.x; ag[g][1] = lo.y; ag[g][2] = hi.x; ag[g][3] = hi.y;
    }
    const float dmv[CELL_U] = {dm.x, dm.y, dm.z, dm.w}, cpv[CELL_U] = {cp.x, cp.y, cp.z, cp.w},
                cnv[CELL_U] = {cn.x, cn.y, cn.z, cn.w};
#pragma unroll
    for (int e = 0; e < CELL_U; ++e) {
      const float ae[4] = {ag[0][e], ag[1][e], ag[2][e], ag[3][e]};
      float dge[4];
      dc[e] = lstm_cell_bwd_elem(ae, cpv[e], cnv[e], dmv[e], dc[e], dge);
#pragma unroll
      for (int g = 0; g < 4; ++g) ag[g][e] = dge[g];
    }
    __nv_bfloat16* dg = a.dgates + (size_t)t * BM * G4 + cg_off;
#pragma unroll
    for (int g = 0; g < 4; ++g)
      *reinterpret_cast<uint2*>(dg + (size_t)g * S) =
          make_uint2(float2_to_bf16x2(ag[g][0], ag[g][1]), float2_to_bf16x2(ag[g][2], ag[g][3]));
    grid.sync();                                      // dgates_t is complete

    // ------------------------------------------------------------ phase 2: split-K dh product
    if (item) {
      if (threadIdx.x == 0) {
        asm volatile("fence.proxy.async.global;" ::: "memory");   // dgates_t: generic -> TMA
        for (int kb = 0; kb < WK / BK; ++kb) {
          mbar_expect_tx(&gbar[kb], BM * BK * 2);
          tma_load_2d(sX + kb * BM * 128, &tmap_dg, &gbar[kb], ks * WK + kb * BK, t * BM);
        }
      }
      product<WN / 2>(acc, sX_u + (wg & 1) * 64 * 128, BM * 128,
                      sWh_u + (wg >> 1) * (WN / 2) * 128, WN * 128, gbar, WK / BK, parity);
      float* slot = a.ws + (size_t)ks * BM * P;
      const int rb = (wg & 1) * 64 + r, cb = n0 + (wg >> 1) * (WN / 2);
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < WN / 16; ++j)
          *reinterpret_cast<float2*>(slot + (size_t)(rb + 8 * h) * P + cb + j * 8 + q2) =
              make_float2(acc[j * 4 + 2 * h], acc[j * 4 + 2 * h + 1]);
    }
    grid.sync();                                      // every slot is written

    // ------------------------------------------------------------ dh_{t-1}: slots in order
    __nv_bfloat16* out = t > 0 ? a.dh_tot + (size_t)(t - 1) * BM * P : a.dh_rec;
    const uint32_t* add =
        reinterpret_cast<const uint32_t*>(a.dH + (size_t)(t > 0 ? t - 1 : 0) * BM * P);
    const int npairs = BM * P / 2;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < npairs; i += gridDim.x * blockDim.x) {
      float2 s = __ldcg(reinterpret_cast<const float2*>(a.ws) + i);
#pragma unroll 8
      for (int k = 1; k < NS; ++k) {
        const float2 v = __ldcg(reinterpret_cast<const float2*>(a.ws + (size_t)k * BM * P) + i);
        s.x += v.x;
        s.y += v.y;
      }
      if (t > 0) {
        const float2 d = bf16x2_to_float2(__ldg(add + i));
        s.x += d.x;
        s.y += d.y;
      }
      reinterpret_cast<uint32_t*>(out)[i] = float2_to_bf16x2(s.x, s.y);
    }
    if (t > 0) grid.sync();                           // dh_tot[t-1] is complete
  }
  *reinterpret_cast<float4*>(a.dc + cs_off) = make_float4(dc[0], dc[1], dc[2], dc[3]);
}

}  // namespace lstm_bwd

extern "C" {

// The grid of `px_lstm_fwd_persistent` for a layer of batch B, state S and projection P, or 0 when
// the kernel does not take that shape or the device cannot keep the whole grid resident (the
// caller then runs the per-step kernels).  Shapes: B 128, S a multiple of 128, P a multiple of 64
// up to 512; the grid is 2 · S/32 CTAs of 512 threads, one per SM.
int px_lstm_fwd_persistent_grid(int B, int S, int P) {
  using namespace lstm_fwd;
  if (B != BM || S <= 0 || S % PK || P <= 0 || P % PN || P > MAX_KB * BK) return 0;
  return persistent_grid<px_lstm_fwd_persistent_kernel, smem_bytes>(2 * (S / UNITS), P);
}

// The same for `px_lstm_bwd_persistent`: the shapes and the grid of the forward kernel.
int px_lstm_bwd_persistent_grid(int B, int S, int P) {
  using namespace lstm_fwd;
  if (B != BM || S <= 0 || S % 128 || P <= 0 || P % lstm_bwd::WN || P > MAX_KB * BK) return 0;
  return persistent_grid<lstm_bwd::px_lstm_bwd_persistent_kernel, lstm_bwd::smem_bytes>(
      2 * (S / UNITS), P);
}

// All T backward steps of an LSTMP layer in one cooperative launch (see the kernel).  dH, act and
// c_all as the forward left them; dc [B, S] fp32 holds dL/dc_T and receives dL/dc_0; dh_tot[T-1]
// holds dH[T-1] + dL/dh_T.  Writes dgates [T, B, 4S], dh_tot[0 .. T-2] and dh_rec [B, P] =
// dgates[0]·Wh^T with the layout, dtype and rounding of the per-step kernels.  ws: fp32
// [4S/512, B, P] scratch.  Every pointer 16-byte aligned.  Returns 0, -1 for a shape
// `px_lstm_bwd_persistent_grid` refuses, or a CUDA error.
int px_lstm_bwd_persistent(const void* dH, const void* act, const float* c_all, const void* Wh,
                           const void* WP, float* dc, void* dgates, void* dh_tot, void* dh_rec,
                           float* ws, int T, int B, int S, int P, cudaStream_t stream) {
  using namespace lstm_fwd;
  const int grid = px_lstm_bwd_persistent_grid(B, S, P);
  if (grid <= 0 || T < 1) return -1;
  for (const void* q : {dH, act, (const void*)c_all, Wh, WP, (const void*)dc, (const void*)dgates,
                        (const void*)dh_tot, (const void*)dh_rec, (const void*)ws})
    if ((uintptr_t)q % 16) return -1;
  CUtensorMap tdh, twp, tdg, twh;
  int rc = make_tmap(&tdh, dh_tot, (uint64_t)T * B, P, ROWS);
  if (!rc) rc = make_tmap(&twp, WP, S, P, UNITS);
  if (!rc) rc = make_tmap(&tdg, dgates, (uint64_t)T * B, 4 * (uint64_t)S, BM);
  if (!rc) rc = make_tmap(&twh, Wh, P, 4 * (uint64_t)S, lstm_bwd::WN);
  if (rc) return rc;
  lstm_bwd::Args a;
  a.dH = (const __nv_bfloat16*)dH; a.act = (const __nv_bfloat16*)act; a.c_all = c_all;
  a.dc = dc; a.dgates = (__nv_bfloat16*)dgates; a.dh_tot = (__nv_bfloat16*)dh_tot;
  a.dh_rec = (__nv_bfloat16*)dh_rec; a.ws = ws;
  a.T = T; a.S = S; a.P = P;
  return launch_cooperative(lstm_bwd::px_lstm_bwd_persistent_kernel, grid,
                            lstm_bwd::smem_bytes(P), stream, tdh, twp, tdg, twh, a);
}

// All T forward steps of an LSTMP layer in one cooperative launch (see the kernel).  c_all[0] and
// h_all[0] hold c0 and h0; writes act, c_all[1..T], m_all and h_all[1..T] exactly as the per-step
// kernels do.  ws: fp32 [S/128, B, P] scratch.  Every pointer 16-byte aligned.  Returns 0, -1 for
// a shape `px_lstm_fwd_persistent_grid` refuses, or a CUDA error.
int px_lstm_fwd_persistent(const void* xw, const void* Wh, const void* WP, void* act, float* c_all,
                           void* m_all, void* h_all, float* ws, int T, int B, int S, int P,
                           float forget_bias, cudaStream_t stream) {
  using namespace lstm_fwd;
  const int grid = px_lstm_fwd_persistent_grid(B, S, P);
  if (grid <= 0 || T < 1) return -1;
  for (const void* q : {xw, Wh, WP, (const void*)act, (const void*)c_all, (const void*)m_all,
                        (const void*)h_all, (const void*)ws})
    if ((uintptr_t)q % 16) return -1;
  CUtensorMap th, tm;
  int rc = make_tmap(&th, h_all, (uint64_t)(T + 1) * B, P, ROWS);
  if (rc) return rc;
  rc = make_tmap(&tm, m_all, (uint64_t)T * B, S, BM);
  if (rc) return rc;
  Args a;
  a.xw = (const __nv_bfloat16*)xw; a.Wh = (const __nv_bfloat16*)Wh;
  a.WP = (const __nv_bfloat16*)WP; a.act = (__nv_bfloat16*)act; a.c_all = c_all;
  a.m_all = (__nv_bfloat16*)m_all; a.h_all = (__nv_bfloat16*)h_all; a.ws = ws;
  a.T = T; a.S = S; a.P = P; a.forget_bias = forget_bias;
  return launch_cooperative(px_lstm_fwd_persistent_kernel, grid, smem_bytes(P), stream, th, tm, a);
}

}  // extern "C"
