// Fused linear cross-entropy for dense output layers (sm_90a).
//
// For a chunk of n rows X_c [n, K] (bf16) of the inputs and a dense output layer W [V, K] (bf16,
// K-contiguous: an nn.Linear weight read in place) with an optional bias b [V] (bf16 or fp32):
//
//   px_linear_xent_logits  S = X_c · Wᵀ (+ b) as a TMA + wgmma GEMM in 128 × 256 tiles.  K is
//                          streamed through a STAGES-deep ring of 64-wide K-blocks (a partial last
//                          block is TMA zero-fill), so any K with K % 8 == 0 up to 8192 works.  The
//                          epilogue stores the tile's fp32 logits into the chunk scratch S [n, ldS],
//                          each row's (max, Σexp) over the tile's columns < V into
//                          part [n, V-tiles], and a row's target logit into tgt [n] from the one
//                          tile that holds it.
//   px_linear_xent_rows    one CTA per row: merges the row's partials into lse, writes
//                          nll = lse − s_t (NaN for a target outside [0, V)) and, when G is given,
//                          rewrites the row as G = w · (exp(s − lse) − [v == t]) in bf16.
//
// Every reduction runs in a fixed order and nothing is accumulated with atomics, so two calls on
// the same inputs give the same bits.  The products with G (dX = G·W, dW = Gᵀ·X) run on cuBLAS.
#include "wgmma.cuh"

namespace lx {

using tc::BK;
using tc::BM;
using tc::THREADS;
using tc::WG_K;

constexpr int BN = 256;                       // vocabulary columns per CTA
constexpr int STAGES = 4;
constexpr int A_BYTES = BM * BK * 2;          // 16 KB of X_c
constexpr int B_BYTES = BN * BK * 2;          // 32 KB of W
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 2 * STAGES * 8;
constexpr int K_MAX = 8192;
constexpr int ROW_THREADS = 256;

// d[128] += A(64×16, smem) · B(256×16, smem)^T; scale_d = 0 overwrites d
__device__ __forceinline__ void wgmma_n256(float* d, uint64_t adesc, uint64_t bdesc,
                                           uint32_t scale_d) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
      "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,"
      "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,"
      "%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,"
      "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,"
      "%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, "
      "%128, %129, p, 1, 1, 0, 0;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
struct LogitsArgs {
  float* S;                   // [n, ldS] fp32 logits of the chunk
  float2* part;               // [n, nvt] (max, Σexp) of each row over each V-tile
  float* tgt;                 // [n] the target's logit
  const long long* targets;   // [n]
  const void* bias;           // [V] or null
  int n, V, K, ldS, nvt;
};

template <typename BiasT>
__device__ __forceinline__ float bias_at(const void* b, int v) {
  return static_cast<float>(reinterpret_cast<const BiasT*>(b)[v]);
}

// Grid (row tiles, V-tiles): the row tiles of one V-tile run side by side and share its W block
// through L2.  Roles as in every wgmma kernel here: warpgroup 0 is the TMA producer, warpgroups 1
// and 2 each own 64 rows of the 128-row tile.  Accumulator layout (wgmma m64n256 f32):
// acc[j·4 + e] is row (warp%4)·16 + lane/4 + 8·(e/2), column j·8 + (lane%4)·2 + e%2.
template <typename BiasT>
__global__ void __launch_bounds__(THREADS, 1)
px_linear_xent_logits_kernel(const __grid_constant__ CUtensorMap tmap_x,
                             const __grid_constant__ CUtensorMap tmap_w, LogitsArgs a) {
  using namespace tc;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  const int m0 = blockIdx.x * BM, vt = blockIdx.y, v0 = vt * BN;
  const int num_kb = (a.K + BK - 1) / BK;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_x) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_w) : "memory");
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int wg = threadIdx.x >> 7;
  if (wg == 0) {
    if (threadIdx.x == 0) {
      for (int kb = 0; kb < num_kb; ++kb) {
        const int s = kb % STAGES;
        mbar_wait(&empty_bar[s], ((kb / STAGES) & 1) ^ 1);
        uint8_t* sa = smem + s * STAGE_BYTES;
        // rows past n or V and columns past K arrive as zeros and still count in full
        mbar_expect_tx(&full_bar[s], STAGE_BYTES);
        tma_load_2d(sa, &tmap_x, &full_bar[s], kb * BK, m0);
        tma_load_2d(sa + A_BYTES, &tmap_w, &full_bar[s], kb * BK, v0);
      }
    }
    return;
  }

  const int cw = wg - 1;
  const bool leader = (threadIdx.x & 127) == 0;
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  for (int kb = 0; kb < num_kb; ++kb) {
    const int s = kb % STAGES;
    mbar_wait(&full_bar[s], (kb / STAGES) & 1);
    const uint32_t sa = smem_u32(smem + s * STAGE_BYTES);
    const uint64_t adesc = make_smem_desc(sa + cw * 64 * BK * 2);
    const uint64_t bdesc = make_smem_desc(sa + A_BYTES);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / WG_K; ++k)
      wgmma_n256(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), 1u);
    wgmma_commit();
    wgmma_wait<1>();                               // the group of K-block kb-1 has retired
    if (kb > 0 && leader) mbar_arrive(&empty_bar[(kb - 1) % STAGES]);
  }
  wgmma_wait<0>();

  // ------------------------------------------------------------------------------- epilogue
  const int t = threadIdx.x - 128, lane = t & 31;
  const int lrow = (t >> 5) * 16 + (lane >> 2);
  const int lcol = (lane & 3) * 2;
  if (a.bias) {
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = v0 + j * 8 + lcol + e;
        if (col < a.V) {
          const float b = bias_at<BiasT>(a.bias, col);
          acc[j * 4 + e] += b;
          acc[j * 4 + 2 + e] += b;
        }
      }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = m0 + lrow + 8 * h;
    // the four lanes of a row hold its 256 columns; every tile has at least one column < V
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e)
        if (v0 + j * 8 + lcol + e < a.V) mx = fmaxf(mx, acc[j * 4 + 2 * h + e]);
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
    float se = 0.f;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e)
        if (v0 + j * 8 + lcol + e < a.V) se += __expf(acc[j * 4 + 2 * h + e] - mx);
    se += __shfl_xor_sync(0xffffffffu, se, 1);
    se += __shfl_xor_sync(0xffffffffu, se, 2);
    if (row >= a.n) continue;
    if ((lane & 3) == 0) a.part[(size_t)row * a.nvt + vt] = make_float2(mx, se);
    float* srow = a.S + (size_t)row * a.ldS;
    // ldS is a multiple of 8 >= V, so the pair at an even column < V stays inside the row
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int col = v0 + j * 8 + lcol;
      if (col < a.V)
        *reinterpret_cast<float2*>(srow + col) = make_float2(acc[j * 4 + 2 * h], acc[j * 4 + 2 * h + 1]);
    }
    const long long tt = a.targets[row] - v0;
    if (tt >= 0 && tt < BN && tt < a.V - v0 && ((int)(tt & 7) >> 1) == (lane & 3)) {
      const int jt = (int)(tt >> 3), et = (int)(tt & 1);
      float v = 0.f;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j)
        if (j == jt) v = et ? acc[j * 4 + 2 * h + 1] : acc[j * 4 + 2 * h];
      a.tgt[row] = v;
    }
  }
}

// merge of two (max, Σexp) pairs; m = -inf stands for an empty pair (a thread or warp that
// holds no V-tile), which must not turn exp(-inf - -inf) into a NaN
__device__ __forceinline__ void lse_merge(float& m, float& s, float pm, float ps) {
  if (pm == -INFINITY) return;
  if (pm > m) {
    s = s * __expf(m - pm) + ps;
    m = pm;
  } else {
    s += ps * __expf(pm - m);
  }
}

__global__ void __launch_bounds__(ROW_THREADS)
px_linear_xent_rows_kernel(const float* __restrict__ S, int ldS, const float2* __restrict__ part,
                           int nvt, const float* __restrict__ tgt,
                           const long long* __restrict__ targets,
                           const float* __restrict__ row_w, float* __restrict__ nll,
                           __nv_bfloat16* __restrict__ G, int V) {
  __shared__ float sm[ROW_THREADS / 32], ss[ROW_THREADS / 32];
  __shared__ float s_lse;
  const int row = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float m = -INFINITY, s = 0.f;
  for (int p = tid; p < nvt; p += ROW_THREADS) {
    const float2 q = part[(size_t)row * nvt + p];
    lse_merge(m, s, q.x, q.y);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float pm = __shfl_xor_sync(0xffffffffu, m, o), ps = __shfl_xor_sync(0xffffffffu, s, o);
    lse_merge(m, s, pm, ps);
  }
  if (lane == 0) { sm[warp] = m; ss[warp] = s; }
  __syncthreads();
  const long long t = targets[row];
  const bool valid = t >= 0 && t < V;
  if (tid == 0) {
    float M = sm[0], Sg = ss[0];
    for (int w = 1; w < ROW_THREADS / 32; ++w) lse_merge(M, Sg, sm[w], ss[w]);
    const float lse = M + logf(Sg);
    s_lse = lse;
    nll[row] = valid ? lse - tgt[row] : __int_as_float(0x7fc00000);
  }
  if (!G) return;
  __syncthreads();
  const float lse = s_lse;
  const float w = row_w ? row_w[row] : 1.f;
  const float* srow = S + (size_t)row * ldS;
  __nv_bfloat16* grow = G + (size_t)row * ldS;
  for (int v = tid * 4; v < V; v += ROW_THREADS * 4) {
    const float4 x = *reinterpret_cast<const float4*>(srow + v);
    const float xs[4] = {x.x, x.y, x.z, x.w};
    float g[4];
#pragma unroll
    for (int e = 0; e < 4; ++e)
      g[e] = v + e < V ? w * (__expf(xs[e] - lse) - (v + e == t ? 1.f : 0.f)) : 0.f;
    __nv_bfloat162 lo = __floats2bfloat162_rn(g[0], g[1]), hi = __floats2bfloat162_rn(g[2], g[3]);
    uint2 pk;
    pk.x = *reinterpret_cast<uint32_t*>(&lo);
    pk.y = *reinterpret_cast<uint32_t*>(&hi);
    *reinterpret_cast<uint2*>(grow + v) = pk;
  }
}

template <typename BiasT>
void launch_logits(int grid_m, int nvt, const CUtensorMap& tx, const CUtensorMap& tw,
                   const LogitsArgs& a, cudaStream_t stream) {
  static bool set = false;
  if (!set) {
    cudaFuncSetAttribute(px_linear_xent_logits_kernel<BiasT>,
                         cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    set = true;
  }
  px_linear_xent_logits_kernel<BiasT><<<dim3(grid_m, nvt), THREADS, SMEM_BYTES, stream>>>(tx, tw, a);
}

}  // namespace lx

extern "C" {

// Columns of one logits tile: the partials buffer has ceil(V / this) entries per row.
int px_linear_xent_tile_cols() { return lx::BN; }

// bias_kind: 0 none, 1 bf16, 2 fp32.  X [n, K] and W [V, K] bf16, 16-byte aligned, K % 8 == 0,
// 8 <= K <= 8192; ldS a multiple of 8 >= V; part [n, ceil(V / 256)] float2.
int px_linear_xent_logits(const void* X, int n, int K, const void* W, int V, const void* bias,
                          int bias_kind, const long long* targets, float* S, int ldS, void* part,
                          float* tgt, cudaStream_t stream) {
  if (n < 1 || V < 1 || K < 8 || K > lx::K_MAX || K % 8 || ldS < V || ldS % 8) return -2;
  if ((uintptr_t)X % 16 || (uintptr_t)W % 16 || (bias_kind != 0) != (bias != nullptr)) return -2;
  CUtensorMap tx, tw;
  int rc = tc::make_tmap(&tx, X, n, K, tc::BM);
  if (rc) return rc;
  rc = tc::make_tmap(&tw, W, V, K, lx::BN);
  if (rc) return rc;
  const int nvt = (V + lx::BN - 1) / lx::BN;
  lx::LogitsArgs a{S, reinterpret_cast<float2*>(part), tgt, targets, bias, n, V, K, ldS, nvt};
  const int grid_m = (n + tc::BM - 1) / tc::BM;
  if (bias_kind == 2)
    lx::launch_logits<float>(grid_m, nvt, tx, tw, a, stream);
  else
    lx::launch_logits<__nv_bfloat16>(grid_m, nvt, tx, tw, a, stream);
  return (int)cudaGetLastError();
}

// nll [n] fp32; G [n, ldS] bf16 or null (no gradient); row_w [n] fp32 or null (all ones).
int px_linear_xent_rows(const float* S, int ldS, const void* part, const float* tgt,
                        const long long* targets, const float* row_w, float* nll, void* G, int n,
                        int V, cudaStream_t stream) {
  if (n < 1 || V < 1 || ldS < V || ldS % 8) return -2;
  const int nvt = (V + lx::BN - 1) / lx::BN;
  lx::px_linear_xent_rows_kernel<<<n, lx::ROW_THREADS, 0, stream>>>(
      S, ldS, reinterpret_cast<const float2*>(part), nvt, tgt, targets, row_w, nll,
      reinterpret_cast<__nv_bfloat16*>(G), V);
  return (int)cudaGetLastError();
}

}  // extern "C"
