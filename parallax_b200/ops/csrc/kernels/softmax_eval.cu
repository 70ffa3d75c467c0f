// Full-softmax cross entropy over a partitioned (weight, bias) co-lookup group, evaluated where
// the rows live — no gather of the table, no [N, V] logits buffer, fp32 logits:
//
//   nll[i] = logsumexp_v(x_i · w_v + b_v) − (x_i · w_t + b_t),   t = targets[i]
//
//   px_full_softmax_lse_kernel      wgmma GEMM with a log-sum-exp epilogue.  Work items are
//                                   blocks of BV local rows of one owner, walked in owner order
//                                   rotated by rank; a CTA loads its block (bf16 shadow rows,
//                                   K-major, 128B swizzle) into shared memory once and streams
//                                   every 128-row tile of X through a TMA ring over it, so each
//                                   table byte is read once per call.  The epilogue adds the fp32
//                                   bias, masks padding rows with −inf and merges the block's
//                                   per-row (max, Σexp) into the CTA's slice of a [grid, N]
//                                   workspace (only that CTA touches it: no atomics).  BV is
//                                   128 for K <= 512 and 64 for 512 < K <= 1024 (ev_bv).
//   px_full_softmax_combine_kernel  one row per warp: merge the grid's (max, Σexp) pairs and
//                                   subtract the target logit, whose rows come from the group's
//                                   lookup kernel.
//
// Top-k (px_full_softmax_topk): the same GEMM kernel with a list capacity KC > 0 also keeps, per
// row, the k best (logit, global id) pairs it has seen — logit descending, equal logits by
// ascending id — in the CTA's slice of a [grid, N, k] workspace, and
// px_full_softmax_topk_combine_kernel merges the grid's sorted lists and the (max, Σexp) pairs
// into log-probabilities and int64 ids.
//
// Sampling (px_full_softmax_sample): the top-k instantiations with SAMPLE = true scale the
// biased logits by 1/τ before the (max, Σexp) pairs, so those are of s = l/τ, then replace each s
// by its Gumbel key s − log E (sparse_group.cuh) and keep the n best keys with the same topk_row:
// the n largest keys of a row are n draws without replacement from softmax(s), in draw order.
// The combine recovers s of each kept entry from its key and writes s − lse.
//
// Truncated sampling (top-k / nucleus): each row keeps T = {v : s_v >= θ*}, θ* the largest θ
// with count(θ) >= k or (mass(θ) >= p and count(θ) >= n), where count and mass are the number
// and the softmax mass of the row's s >= θ, compared in the order-preserving uint32 key of fp32
// (−0 taken as +0).  Three kinds of pass of the same GEMM kernel find and apply θ*:
//   px_full_softmax_sample_lse   KC = 0, SAMPLE: the (max, Σexp) pairs of s, merged into each
//                                row's lse and a zeroed threshold state (TruncRow).
//   px_full_softmax_radix        HIST = d: for every real s whose key matches the row's prefix,
//                                count 1 and exp(s − lse) into the bin of its next d-bit digit,
//                                per consumer lane in shared memory, then the quad's sums into the
//                                CTA's slice of a [grid, N, 2^d] workspace (the quad owns its
//                                rows' slices: no atomics); one warp per row then sums the slices
//                                and takes the highest digit whose cumulative (count, mass) from
//                                above satisfies the predicate.  32 / d passes give θ*.
//   px_full_softmax_sample_masked  the sampling kernel with MASK: keys of s below θ* become −inf
//                                after the (max, Σexp) pairs are merged, so log-probabilities
//                                stay those of the untruncated softmax.
//
// Training (px_full_softmax_grad): the log-sum-exp instantiations with GRAD = true take one
// gathered chunk of the table, global ids [v0, v0 + rows), as a one-owner, one-slot table and
// recompute its biased logits s.  The epilogue writes G = g_i · (exp(s − lse_i) − [v == t_i]) in
// bf16 into a [N, ·] chunk buffer and the column sums of G (the bias gradient, fp32) of the
// CTA's block: a CTA streams every X tile over its block, so the sums are complete in the CTA.
// The caller multiplies G into dX = G·W_c and dW_c = Gᵀ·X.
//
// One-sided like the lookup: peers' rows are read over NVLink with 16-byte loads; nothing is
// exchanged, so a rank may evaluate alone.  In sync mode the kernel first waits applied[o] >=
// completed steps on the group header (the lookup's freshness rule).
#include "common.cuh"
#include "sparse_group.cuh"
#include "wgmma.cuh"

#include <type_traits>

namespace tc {

constexpr int EV_STAGES = 4;        // X ring depth (16 KB per stage)
constexpr int EV_KMAX = 1024;
// table rows per work item (= wgmma N) at width K: the resident block of BV rows × K bf16 is at
// most 128 KB, so 128 rows up to K = 512 and 64 rows up to K = 1024.  Fewer rows per block
// halve the FLOP per byte of X each CTA streams, so the wide height is only taken where needed.
constexpr int ev_bv(int K) { return K <= 512 ? 128 : 64; }
constexpr int ev_kmax(int bv) { return 128 * 512 / bv; }   // the widest K a block height takes
constexpr float EV_LOG2E = 1.4426950408889634f;

// one top-k list entry; the order key is (v descending, id ascending).  An empty entry is
// (−inf, INT_MAX), which every real row beats; real logits are never −inf.
struct __align__(8) TopkEntry { float v; int id; };

struct EvalArgs {
  const __nv_bfloat16* const* w;    // [W] bf16 shadow rows of the weight table on every rank
  const void* const* b;             // [W] bias rows on every rank: fp32 master rows, or the bf16
                                    // master of a sparse_weights="bf16" table
  const int* row_cnt;               // [owners][slots] real rows of the partition in each slot
  const uint32_t* applied;          // this rank's group header: applied[W]
  const SparseCtl* ctl;
  float2* ws;                       // [grid][N] running (max, Σexp) per (CTA, row)
  int N, K, kb;                     // kb = ceil(K / 64) K-blocks of 64 columns
  int w_pitch, b_pitch;             // row pitch (elements) of the shadow / bias rows
  int W, rank, replicated, owners, slots, rows_per_part, nblk;
  int wait;
};

// the top-k kernels' arguments (KC > 0); the log-sum-exp kernels take EvalArgs alone
struct TopkArgs : EvalArgs {
  TopkEntry* tk;                    // [grid][N][k] per-CTA lists, sorted by the order key
  const int* part_idx;              // [owners][slots] partition held in each slot (-1: none)
  GroupGeom g;                      // for the global ids of the partitions' rows
  int k;
};

// the sampling kernels' arguments: the lists hold (key, global id) pairs
struct SampleArgs : TopkArgs {
  float inv_tau;                    // fp32(1/τ), finite and > 0
  uint32_t seed;
  int row0;                         // index of X's row 0 within the caller's batch (chunking)
};
// the gradient kernels' arguments (KC == 0): the chunk's rows replace w, b and row_cnt
struct GradArgs : EvalArgs {
  const __nv_bfloat16* wc;          // [rows] bf16 weight rows of the chunk, pitch w_pitch
  const void* bc;                   // [rows] bias rows of the chunk, pitch b_pitch
  int rows;                         // real rows of the chunk
  long long v0;                     // global id of the chunk's row 0
  const float* lse;                 // [N] each row's log-sum-exp from the forward
  const float* g;                   // [N] gradient of each row's NLL
  const long long* targets;         // [N]
  __nv_bfloat16* G;                 // [N][g_pitch] out: g_i · (softmax − onehot) of the chunk
  int g_pitch;                      // >= the chunk's blocks · BV, even
  float* db;                        // [rows] out: column sums of G
};

// truncated sampling: a row's threshold search state.  The keys >= prefix (its bits below the
// current digit zero) that lie above the prefix's range number `above` with softmax mass
// `above_mass`; after the last pass prefix is the key of θ*
struct TruncRow {
  uint32_t prefix, above;
  float above_mass;
  float lse;                        // log-sum-exp of the row's s
};
struct HistBin { uint32_t cnt; float mass; };
constexpr int EV_RADIX_BITS = 4;    // digit width d of a histogram pass

// the tempered log-sum-exp kernels' arguments (KC == 0, SAMPLE)
struct TempArgs : EvalArgs {
  float inv_tau;
};
// the histogram kernels' arguments (KC == 0, HIST = d)
struct HistArgs : TempArgs {
  const TruncRow* rows;             // [N]
  HistBin* hist;                    // [grid][N][2^d] per-CTA bins
  int lo;                           // bit position of the pass's digit
  uint32_t himask;                  // the key bits the prefix has fixed
};
// the masked sampling kernels' arguments (KC > 0, SAMPLE, MASK): keys below rows[].prefix drop
struct MaskArgs : SampleArgs {
  const TruncRow* rows;             // [N]
};

template <int KC, bool SAMPLE = false, bool GRAD = false, int HIST = 0, bool MASK = false>
using EvalParams = typename std::conditional<
    GRAD, GradArgs,
    typename std::conditional<
        KC == 0,
        typename std::conditional<
            HIST != 0, HistArgs,
            typename std::conditional<SAMPLE, TempArgs, EvalArgs>::type>::type,
        typename std::conditional<
            MASK, MaskArgs,
            typename std::conditional<SAMPLE, SampleArgs, TopkArgs>::type>::type>::type>::type;

// order-preserving uint32 key of an fp32 value (not NaN), −0 taken as +0
__device__ __forceinline__ uint32_t ev_key(float f) {
  uint32_t u = __float_as_uint(f);
  if (u == 0x80000000u) u = 0u;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ bool tk_beats(float v, int id, float v2, int id2) {
  return v > v2 || (v == v2 && id < id2);
}

// (m, s) ⊕ (m2, s2) for s = Σ exp(l − m); s == 0 marks an empty pair (m = −inf)
__device__ __forceinline__ void lse_merge(float2& c, float m2, float s2) {
  if (s2 == 0.f) return;
  if (c.y == 0.f) { c = make_float2(m2, s2); return; }
  const float mx = fmaxf(c.x, m2);
  c.y = c.y * exp2f((c.x - mx) * EV_LOG2E) + s2 * exp2f((m2 - mx) * EV_LOG2E);
  c.x = mx;
}

__device__ __forceinline__ bool ev_row_real(const EvalArgs& a, const int* cnt, int lr) {
  return lr < a.slots * a.rows_per_part &&
         (lr % a.rows_per_part) < __ldg(cnt + lr / a.rows_per_part);
}
__device__ __forceinline__ bool ev_row_real(const GradArgs& a, const int*, int lr) {
  return lr < a.rows;
}

// an owner's weight and bias rows; the gradient kernels' one owner is the gathered chunk
__device__ __forceinline__ const __nv_bfloat16* ev_wsrc(const EvalArgs& a, int owner) {
  return a.w[owner];
}
__device__ __forceinline__ const __nv_bfloat16* ev_wsrc(const GradArgs& a, int) { return a.wc; }
__device__ __forceinline__ const void* ev_bsrc(const EvalArgs& a, int owner) { return a.b[owner]; }
__device__ __forceinline__ const void* ev_bsrc(const GradArgs& a, int) { return a.bc; }

// Roles as in gemm_tc.cu: warpgroup 0 produces (thread 0 issues the X TMA loads), warpgroups
// 1 and 2 each own 64 rows of the 128-row X tile and run wgmma m64×BV×16 against the resident
// table block.  All 384 threads load the table block between work items.
// bias element 0 of a 16-byte aligned row, widened to fp32
__device__ __forceinline__ float ev_bias(const float* row) { return __uint_as_float(ld_v4(row).x); }
__device__ __forceinline__ float ev_bias(const __nv_bfloat16* row) {
  return __uint_as_float(ld_v4(row).x << 16);
}

// Top-k epilogue of one row h of the quad's two (all four lanes call it; the row is < N).  A lane
// holds BV/4 of the block's BV logits at acc[j·4 + 2h + e], column j·8 + cq + e; s_gid has their
// global ids.  The list of the CTA is skipped unless the block's row maximum mx can enter it.
// Otherwise up to k rounds of quad-wide arg-max extract, best first, the block's entries that
// beat the list's (k − r)-th entry in round r.  The list is copied to shared memory (lbuf) by the
// four lanes at once, the candidates are staged in cand, and both are merged into the list from
// its tail, so entries ahead of the first insertion are not rewritten.
template <int BV, int KC>
__device__ __forceinline__ void topk_row(const TopkArgs& a, float* acc, int h, int cq, float mx,
                                         const int* s_gid, TopkEntry* cand, TopkEntry* lbuf,
                                         TopkEntry* list, bool first) {
  const TopkEntry none = {-INFINITY, INT_MAX};
  const int k = a.k;
  const unsigned qmask = 0xfu << (threadIdx.x & 28);
  const bool q0 = (threadIdx.x & 3) == 0;
  if (!first && (mx == -INFINITY || mx < list[k - 1].v)) return;
  for (int i = threadIdx.x & 3; i < k; i += 4) lbuf[i] = first ? none : list[i];
  __syncwarp(qmask);
  int m = 0;
  for (; m < k; ++m) {
    float bv = -INFINITY;
    int bc = 0, bid = INT_MAX;
#pragma unroll
    for (int j = 0; j < BV / 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float v = acc[j * 4 + 2 * h + e];
        const int c = j * 8 + cq + e;
        if (v > bv || (v == bv && v != -INFINITY && s_gid[c] < bid)) { bv = v; bc = c; bid = s_gid[c]; }
      }
    float wv = bv;
    int wid = bid;
#pragma unroll
    for (int o = 1; o < 4; o <<= 1) {
      const float v2 = __shfl_xor_sync(qmask, wv, o);
      const int id2 = __shfl_xor_sync(qmask, wid, o);
      if (tk_beats(v2, id2, wv, wid)) { wv = v2; wid = id2; }
    }
    const TopkEntry t = lbuf[k - 1 - m];
    if (wv == -INFINITY || !tk_beats(wv, wid, t.v, t.id)) break;
    if (q0) cand[m] = TopkEntry{wv, wid};
    if (bid == wid && bv == wv) {            // the lane that holds the winner takes it out
#pragma unroll
      for (int j = 0; j < BV / 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (j * 8 + cq + e == bc) acc[j * 4 + 2 * h + e] = -INFINITY;
    }
  }
  __syncwarp(qmask);
  if (q0) {
    // merge from the tail: the worse of (list[i], cand[j]) goes to position o; once every
    // candidate is placed, list[0 .. i] is already where it belongs
    int i = k - 1 - m, j = m - 1;
    for (int o = k - 1; o >= 0 && (j >= 0 || first); --o) {
      const TopkEntry l = i >= 0 ? lbuf[i] : none;
      if (j >= 0 && (i < 0 || tk_beats(l.v, l.id, cand[j].v, cand[j].id))) list[o] = cand[j--];
      else { list[o] = l; --i; }
    }
  }
  __syncwarp(qmask);
}

// BiasT: float (fp32 master bias rows) or __nv_bfloat16 (bf16 master bias rows).  KC: top-k list
// capacity (0: log-sum-exp only; else k <= KC and the top-k epilogue runs).  SAMPLE (KC > 0):
// the lists rank Gumbel keys of the tempered logits instead of the logits.  GRAD (KC == 0): the
// gradient epilogue over one gathered chunk instead of the (max, Σexp) pairs.  SAMPLE with KC == 0:
// the pairs are of s = l/τ.  HIST = d (KC == 0, SAMPLE): the digit histogram of truncated sampling
// instead of the pairs.  MASK (KC > 0, SAMPLE): keys below the row's threshold drop out.  BV:
// the block height, ev_bv(K)
template <typename BiasT, int BV, int KC, bool SAMPLE = false, bool GRAD = false, int HIST = 0,
          bool MASK = false>
__global__ void __launch_bounds__(THREADS, 1)
px_full_softmax_lse_kernel(const __grid_constant__ CUtensorMap tmap_x,
                           EvalParams<KC, SAMPLE, GRAD, HIST, MASK> a) {
  constexpr int X_BYTES = BM * BK * 2;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* sB = smem;                                        // [kb][BV rows][128 B]
  uint8_t* sX = smem + a.kb * BV * 128;                      // [STAGES][128 rows][128 B]
  float* s_bias = reinterpret_cast<float*>(sX + EV_STAGES * X_BYTES);   // [BV], −inf = padding
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(s_bias + BV);
  uint64_t* empty_bar = full_bar + EV_STAGES;
  int* s_gid = reinterpret_cast<int*>(empty_bar + EV_STAGES);      // [BV] (KC > 0)
  TopkEntry* s_cand = reinterpret_cast<TopkEntry*>(s_gid + BV);   // [256 / 4 quads][2][KC]
  float* s_db = reinterpret_cast<float*>(s_gid);                  // [BV] (GRAD)
  HistBin* s_hist = reinterpret_cast<HistBin*>(s_gid);            // [2^d][256 lanes] (HIST)

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_x) : "memory");
    for (int s = 0; s < EV_STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (a.wait && threadIdx.x < a.W) {
    const uint32_t need = a.ctl->step;
    while ((int32_t)(ld_acquire_sys(a.applied + threadIdx.x) - need) < 0) { }
  }
  __syncthreads();

  const int wg = threadIdx.x >> 7;
  const int items = a.owners * a.nblk;
  const int m_tiles = (a.N + BM - 1) / BM;
  const int cpr = a.kb * 8;                     // 16-byte chunks per table row in shared memory
  const int kc = a.K / 8;                       // ... of which real
  uint32_t it = 0;                              // X stages so far: ring slot and parity
  bool first = true;
  for (int item = blockIdx.x; item < items; item += gridDim.x) {
    const int oi = item / a.nblk;
    const int owner = a.replicated ? a.rank : (a.rank + oi) % a.W;
    const int* cnt = a.row_cnt + (a.replicated ? 0 : owner) * a.slots;
    const int r0 = (item % a.nblk) * BV;
    const __nv_bfloat16* src = ev_wsrc(a, owner);
    __syncthreads();                            // every wgmma on the previous block has retired
    // table block -> shared memory, 128B-swizzled K-major (chunk c of row r at c ^ (r % 8));
    // padding rows and columns beyond K are zero.  Eight loads in flight per thread.
    const int total = BV * cpr;
    for (int base = threadIdx.x; base < total; base += 8 * THREADS) {
      uint4 v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int idx = base + u * THREADS;
        const int r = idx / cpr, c = idx % cpr;
        v[u] = make_uint4(0, 0, 0, 0);
        if (idx < total && c < kc && ev_row_real(a, cnt, r0 + r))
          v[u] = ld_v4(src + (size_t)(r0 + r) * a.w_pitch + c * 8);
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int idx = base + u * THREADS;
        if (idx >= total) break;
        const int r = idx / cpr, c = idx % cpr;
        *reinterpret_cast<uint4*>(sB + (c >> 3) * (BV * 128) + r * 128 +
                                  (((c & 7) ^ (r & 7)) << 4)) = v[u];
      }
    }
    if (threadIdx.x < BV) {
      const int lr = r0 + threadIdx.x;
      float bv = -INFINITY;
      if (ev_row_real(a, cnt, lr))
        bv = ev_bias(reinterpret_cast<const BiasT*>(ev_bsrc(a, owner)) + (size_t)lr * a.b_pitch);
      s_bias[threadIdx.x] = bv;
      if constexpr (GRAD) s_db[threadIdx.x] = 0.f;
      if constexpr (KC > 0) {
        int gid = INT_MAX;
        if (bv != -INFINITY) {
          const int slot = lr / a.rows_per_part;
          gid = geom_gid(a.g, __ldg(a.part_idx + (a.replicated ? 0 : owner) * a.slots + slot),
                         lr - slot * a.rows_per_part);
        }
        s_gid[threadIdx.x] = gid;
      }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // st.shared -> wgmma reads
    __syncthreads();

    if (wg == 0) {
      if (threadIdx.x == 0) {
        for (int mt = 0; mt < m_tiles; ++mt)
          for (int kb = 0; kb < a.kb; ++kb, ++it) {
            const int s = it % EV_STAGES;
            mbar_wait(&empty_bar[s], ((it / EV_STAGES) & 1) ^ 1);
            mbar_expect_tx(&full_bar[s], X_BYTES);
            tma_load_2d(sX + s * X_BYTES, &tmap_x, &full_bar[s], kb * BK, mt * BM);
          }
      }
    } else {
      const int cw = wg - 1;
      const bool leader = (threadIdx.x & 127) == 0;
      const int lane = threadIdx.x & 31;
      const int cq = (lane & 3) * 2;
      float colsum[GRAD ? BV / 4 : 1];        // GRAD: the lane's columns of G summed over rows
      if constexpr (GRAD) {
#pragma unroll
        for (int i = 0; i < BV / 4; ++i) colsum[i] = 0.f;
      }
      for (int mt = 0; mt < m_tiles; ++mt) {
        float acc[BV / 2];
        for (int kb = 0; kb < a.kb; ++kb, ++it) {
          const int s = it % EV_STAGES;
          mbar_wait(&full_bar[s], (it / EV_STAGES) & 1);
          const uint64_t adesc = make_smem_desc(smem_u32(sX + s * X_BYTES + cw * 64 * BK * 2));
          const uint64_t bdesc = make_smem_desc(smem_u32(sB + kb * BV * 128));
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / WG_K; ++k)
            wgmma_bf16<BV>(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2),
                           (kb | k) != 0 ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<1>();
          if (kb > 0 && leader) mbar_arrive(&empty_bar[(it - 1) % EV_STAGES]);
        }
        wgmma_wait<0>();
        if (leader) mbar_arrive(&empty_bar[(it - 1) % EV_STAGES]);
        // epilogue: a quad of lanes holds all BV columns of 2 rows (acc[j·4 + 2h + e] is row
        // lane/4 + 8h, column j·8 + (lane%4)·2 + e of the warp's 16 rows)
        const int rbase = mt * BM + cw * 64 + ((threadIdx.x & 127) >> 5) * 16 + (lane >> 2);
        if constexpr (GRAD) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = rbase + 8 * h;
            const bool rv = row < a.N;
            // rows past N (zero-filled X) contribute nothing: g = 0, no store
            const float nl2 = rv ? -__ldg(a.lse + row) * EV_LOG2E : 0.f;
            const float gr = rv ? __ldg(a.g + row) : 0.f;
            const long long tc = rv ? __ldg(a.targets + row) - (a.v0 + r0) : -1;
            __nv_bfloat16* grow = a.G + (size_t)row * a.g_pitch + r0 + cq;
#pragma unroll
            for (int j = 0; j < BV / 8; ++j) {
              float gv[2];
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int c = j * 8 + cq + e;
                const float b = s_bias[c];                  // −inf: padding, p = 0
                float p = exp2f(fmaf(acc[j * 4 + 2 * h + e] + b, EV_LOG2E, nl2));
                if (c == tc && b != -INFINITY) p -= 1.f;
                gv[e] = gr * p;
                colsum[j * 2 + e] += gv[e];
              }
              if (rv)
                *reinterpret_cast<__nv_bfloat162*>(grow + j * 8) =
                    __floats2bfloat162_rn(gv[0], gv[1]);
            }
          }
        } else if constexpr (HIST != 0) {
          // each consumer lane counts its 32 columns of the row into its own bins (bin-major,
          // s_hist[bin][lane]: no atomics, no bank conflicts), then the quad's lane q sums
          // bins q, q + 4, ... over the quad's four lanes into the CTA's slice
          constexpr int NB = 1 << HIST;
          const unsigned qmask = 0xfu << (lane & 28);
          const int tid = threadIdx.x - 128;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = rbase + 8 * h;
            if (row >= a.N) continue;                       // the quad's rows: quad-uniform
            const TruncRow st = a.rows[row];
            HistBin* gb = a.hist + ((size_t)blockIdx.x * a.N + row) * NB;
            bool hit = false;
#pragma unroll
            for (int j = 0; j < BV / 8; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                // s as SAMPLE scales it; padding rows are never candidates
                const float b = s_bias[j * 8 + cq + e];
                const float s = (acc[j * 4 + 2 * h + e] + b) * a.inv_tau;
                hit |= b != -INFINITY && !((ev_key(s) ^ st.prefix) & a.himask);
              }
            if (!__any_sync(qmask, hit)) {                  // no key of the block matches
              if (first)
                for (int i = lane & 3; i < NB; i += 4) gb[i] = HistBin{0u, 0.f};
              continue;
            }
#pragma unroll
            for (int i = 0; i < NB; ++i) s_hist[i * 256 + tid] = HistBin{0u, 0.f};
            const float nl2 = -st.lse * EV_LOG2E;
#pragma unroll
            for (int j = 0; j < BV / 8; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const float b = s_bias[j * 8 + cq + e];
                const float s = (acc[j * 4 + 2 * h + e] + b) * a.inv_tau;
                const uint32_t u = ev_key(s);
                if (b == -INFINITY || ((u ^ st.prefix) & a.himask)) continue;
                HistBin& bin = s_hist[((u >> a.lo) & (NB - 1)) * 256 + tid];
                bin.cnt += 1u;
                bin.mass += exp2f(fmaf(s, EV_LOG2E, nl2));
              }
            __syncwarp(qmask);
            for (int i = lane & 3; i < NB; i += 4) {
              HistBin v = first ? HistBin{0u, 0.f} : gb[i];
#pragma unroll
              for (int l = 0; l < 4; ++l) {
                const HistBin o = s_hist[i * 256 + (tid & ~3) + l];
                v.cnt += o.cnt;
                v.mass += o.mass;
              }
              gb[i] = v;
            }
            __syncwarp(qmask);                              // before the bins are reused
          }
        } else {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float mx = -INFINITY;
#pragma unroll
            for (int j = 0; j < BV / 8; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                float& v = acc[j * 4 + 2 * h + e];
                v += s_bias[j * 8 + cq + e];
                if constexpr (SAMPLE) v *= a.inv_tau;
                mx = fmaxf(mx, v);
              }
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            float sum = 0.f;
            if (mx != -INFINITY) {
              const float ms = mx * EV_LOG2E;
#pragma unroll
              for (int j = 0; j < BV / 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e)
                  sum += exp2f(fmaf(acc[j * 4 + 2 * h + e], EV_LOG2E, -ms));
            }
            sum += __shfl_xor_sync(0xffffffffu, sum, 1);
            sum += __shfl_xor_sync(0xffffffffu, sum, 2);
            const int row = rbase + 8 * h;
            if ((lane & 3) == 0 && row < a.N) {
              float2* p = a.ws + (size_t)blockIdx.x * a.N + row;
              float2 c = first ? make_float2(-INFINITY, 0.f) : *p;
              lse_merge(c, mx, sum);
              *p = c;
            }
            if constexpr (SAMPLE && KC > 0) {
              // keys s − log E in place of s (padding stays −inf), and the quad's key maximum
              const uint32_t rk = sample_row_key(a.seed, (uint32_t)(a.row0 + row));
              [[maybe_unused]] uint32_t thr = 0u;   // MASK: keys of s below θ* become −inf
              if constexpr (MASK) thr = row < a.N ? a.rows[row].prefix : 0u;
              mx = -INFINITY;
#pragma unroll
              for (int j = 0; j < BV / 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  float& v = acc[j * 4 + 2 * h + e];
                  if constexpr (MASK)
                    v = ev_key(v) < thr ? -INFINITY
                                        : v - sample_log_e(rk, (uint32_t)s_gid[j * 8 + cq + e]);
                  else
                    v -= sample_log_e(rk, (uint32_t)s_gid[j * 8 + cq + e]);
                  mx = fmaxf(mx, v);
                }
              mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
              mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            }
            if constexpr (KC > 0) {
              if (row < a.N)
                topk_row<BV, KC>(a, acc, h, cq, mx, s_gid, s_cand + ((threadIdx.x - 128) >> 2) * 2 * KC,
                             s_cand + ((threadIdx.x - 128) >> 2) * 2 * KC + KC,
                             a.tk + ((size_t)blockIdx.x * a.N + row) * a.k, first);
            }
          }
        }
      }
      if constexpr (GRAD) {
        // the 8 lanes of a warp that hold the same columns, then the CTA's 8 consumer warps
#pragma unroll
        for (int i = 0; i < BV / 4; ++i) {
          float v = colsum[i];
          v += __shfl_xor_sync(0xffffffffu, v, 4);
          v += __shfl_xor_sync(0xffffffffu, v, 8);
          v += __shfl_xor_sync(0xffffffffu, v, 16);
          if (lane < 4) atomicAdd(&s_db[(i >> 1) * 8 + cq + (i & 1)], v);
        }
      }
    }
    if constexpr (GRAD) {
      __syncthreads();
      if (threadIdx.x < BV && r0 + (int)threadIdx.x < a.rows) a.db[r0 + threadIdx.x] = s_db[threadIdx.x];
    }
    first = false;
  }
}

// one warp's merge of a row's (max, Σexp) pairs over the grid's ws entries: lane l merges
// entries l, l + 32, ..., then the lanes merge by xor shuffles; every lane returns the result
__device__ __forceinline__ float2 ev_grid_lse(const float2* __restrict__ ws, int grid, int N,
                                             int row, int lane) {
  float2 c = make_float2(-INFINITY, 0.f);
  for (int g = lane; g < grid; g += 32) {
    const float2 p = ws[(size_t)g * N + row];
    lse_merge(c, p.x, p.y);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, c.x, o);
    const float s2 = __shfl_xor_sync(0xffffffffu, c.y, o);
    lse_merge(c, m2, s2);
  }
  return c;
}

// LSE: also write each row's log-sum-exp to lse [N] (the training forward keeps it for backward)
template <typename BiasT, bool LSE = false>
__global__ void __launch_bounds__(256)
px_full_softmax_combine_kernel(const float2* __restrict__ ws, int grid, int N, int K,
                               const __nv_bfloat16* __restrict__ X,
                               const __nv_bfloat16* __restrict__ wt, int wt_pitch,
                               const BiasT* __restrict__ bt, int bt_pitch,
                               const long long* __restrict__ targets, int V,
                               float* __restrict__ nll, float* __restrict__ lse) {
  const int lane = threadIdx.x & 31;
  for (int row = blockIdx.x * 8 + (threadIdx.x >> 5); row < N; row += gridDim.x * 8) {
    const float2 c = ev_grid_lse(ws, grid, N, row, lane);
    float d = 0.f;
    for (int ch = lane; ch < K / 8; ch += 32) {
      float xf[8], wf[8];
      Vec16<__nv_bfloat16>::unpack(*reinterpret_cast<const uint4*>(X + (size_t)row * K + ch * 8), xf);
      Vec16<__nv_bfloat16>::unpack(
          *reinterpret_cast<const uint4*>(wt + (size_t)row * wt_pitch + ch * 8), wf);
#pragma unroll
      for (int e = 0; e < 8; ++e) d = fmaf(xf[e], wf[e], d);
    }
    d = warp_sum(d);
    if (lane == 0) {
      const long long t = targets[row];
      nll[row] = (t >= 0 && t < V) ? c.x + logf(c.y) - (d + (float)bt[(size_t)row * bt_pitch])
                                   : __int_as_float(0x7fc00000);
      if constexpr (LSE) lse[row] = c.x + logf(c.y);
    }
  }
}

// one warp per row: merge the grid's (max, Σexp) pairs, then the grid's sorted top-k lists in k
// rounds of warp-wide arg-max over the lists' heads (lane l holds the heads of lists l, l + 32,
// ...), and write log_probs = logit − lse and the ids of the row's k best entries.
// SAMPLE: the entries are keys s − log E of the lists of the sampling kernels; the entry's s is
// recovered as key + log E with the same noise (seed, row0 + row, id), which is within an ulp of
// the key of the s the kernel scored.  Storing s with each entry instead would widen the entry,
// the lists and topk_row that the top-k kernels share; recomputing costs one hash and two
// logarithms per output.
constexpr int TK_LISTS_PER_LANE = 8;       // grid <= 256

template <bool SAMPLE>
__global__ void __launch_bounds__(256)
px_full_softmax_topk_combine_kernel(const float2* __restrict__ ws,
                                    const TopkEntry* __restrict__ tk, int grid, int N, int k,
                                    float* __restrict__ log_probs, long long* __restrict__ ids,
                                    uint32_t seed, int row0) {
  const int lane = threadIdx.x & 31;
  for (int row = blockIdx.x * 8 + (threadIdx.x >> 5); row < N; row += gridDim.x * 8) {
    const float2 c = ev_grid_lse(ws, grid, N, row, lane);
    const float lse = c.x + logf(c.y);
    int pos[TK_LISTS_PER_LANE];
    TopkEntry head[TK_LISTS_PER_LANE];
#pragma unroll
    for (int s = 0; s < TK_LISTS_PER_LANE; ++s) {
      const int g = lane + 32 * s;
      pos[s] = 0;
      head[s] = g < grid ? tk[((size_t)g * N + row) * k] : TopkEntry{-INFINITY, INT_MAX};
    }
    TopkEntry mine = {-INFINITY, INT_MAX};
    for (int o = 0; o < k; ++o) {
      TopkEntry b = {-INFINITY, INT_MAX};
      int bs = -1;
#pragma unroll
      for (int s = 0; s < TK_LISTS_PER_LANE; ++s)
        if (tk_beats(head[s].v, head[s].id, b.v, b.id)) { b = head[s]; bs = s; }
      TopkEntry w = b;
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        const float v2 = __shfl_xor_sync(0xffffffffu, w.v, off);
        const int id2 = __shfl_xor_sync(0xffffffffu, w.id, off);
        if (tk_beats(v2, id2, w.v, w.id)) w = TopkEntry{v2, id2};
      }
      if (lane == o) mine = w;
      if (bs >= 0 && b.id == w.id) {
#pragma unroll
        for (int s = 0; s < TK_LISTS_PER_LANE; ++s)
          if (s == bs) {
            head[s] = ++pos[s] < k ? tk[((size_t)(lane + 32 * s) * N + row) * k + pos[s]]
                                   : TopkEntry{-INFINITY, INT_MAX};
          }
      }
    }
    if (lane < k) {
      if constexpr (SAMPLE)
        mine.v += sample_log_e(sample_row_key(seed, (uint32_t)(row0 + row)), (uint32_t)mine.id);
      log_probs[(size_t)row * k + lane] = mine.v - lse;
      ids[(size_t)row * k + lane] = mine.id;
    }
  }
}

// truncated sampling, one warp per row: merge the grid's (max, Σexp) pairs of s into the row's
// lse and start its threshold search (prefix 0: every key)
__global__ void __launch_bounds__(256)
px_full_softmax_trunc_init_kernel(const float2* __restrict__ ws, int grid, int N,
                                  TruncRow* __restrict__ rows) {
  const int lane = threadIdx.x & 31;
  for (int row = blockIdx.x * 8 + (threadIdx.x >> 5); row < N; row += gridDim.x * 8) {
    const float2 c = ev_grid_lse(ws, grid, N, row, lane);
    if (lane == 0) rows[row] = TruncRow{0u, 0u, 0.f, c.x + logf(c.y)};
  }
}

// one radix step of the threshold search, one warp per row: sum the grid's bins of the digit at
// bit lo (lane b and b + NB hold bin b), take suffix sums from the highest digit down, and fix
// the highest digit b at which count(θ) >= k or (mass(θ) >= p and count(θ) >= n) holds for θ =
// prefix | b << lo (k = 0 / p = 0: no such clause).  No digit: b = 0, so a row whose predicate
// never holds (fp32 mass short of p) keeps every word.
template <int D>
__global__ void __launch_bounds__(256)
px_full_softmax_select_kernel(const HistBin* __restrict__ hist, int grid, int N,
                              TruncRow* __restrict__ rows, int lo, int k, float p, int n) {
  constexpr int NB = 1 << D;
  static_assert(NB <= 32, "one bin per lane");
  const int lane = threadIdx.x & 31, bin = lane % NB;
  for (int row = blockIdx.x * 8 + (threadIdx.x >> 5); row < N; row += gridDim.x * 8) {
    uint32_t c = 0u;
    float m = 0.f;
    for (int g = lane / NB; g < grid; g += 32 / NB) {
      const HistBin h = hist[((size_t)g * N + row) * NB + bin];
      c += h.cnt;
      m += h.mass;
    }
#pragma unroll
    for (int o = NB; o < 32; o <<= 1) {
      c += __shfl_xor_sync(0xffffffffu, c, o);
      m += __shfl_xor_sync(0xffffffffu, m, o);
    }
#pragma unroll
    for (int o = 1; o < NB; o <<= 1) {           // suffix sums: bins >= bin
      const uint32_t c2 = __shfl_down_sync(0xffffffffu, c, o, NB);
      const float m2 = __shfl_down_sync(0xffffffffu, m, o, NB);
      if (bin + o < NB) { c += c2; m += m2; }
    }
    const TruncRow r = rows[row];
    const uint32_t C = r.above + c;
    const float M = r.above_mass + m;
    const bool ok = (k > 0 && C >= (uint32_t)k) || (p > 0.f && M >= p && C >= (uint32_t)n);
    const uint32_t bal = __ballot_sync(0xffffffffu, ok && lane < NB);
    const int b = bal ? 31 - __clz(bal) : 0;
    const uint32_t ca = __shfl_sync(0xffffffffu, c, (b + 1) & (NB - 1));   // bins above b
    const float ma = __shfl_sync(0xffffffffu, m, (b + 1) & (NB - 1));
    if (lane == 0) {
      TruncRow o = r;
      o.prefix |= (uint32_t)b << lo;
      if (b + 1 < NB) { o.above += ca; o.above_mass += ma; }
      rows[row] = o;
    }
  }
}

// dynamic shared memory of px_full_softmax_lse_kernel<·, bv, kc> at kb K-blocks: alignment
// slack, table block, X ring, bias and barriers; the top-k kernels (kc > 0) add the block's
// global ids, and a candidate list and a copy of the row's list per consumer quad; the gradient
// kernels (grad) the block's column sums; the histogram kernels (bins = 2^d) the bins of one row
// per consumer lane
constexpr int ev_smem_bytes(int bv, int kb, int kc, bool grad = false, int bins = 0) {
  return 1024 + kb * bv * 128 + EV_STAGES * BM * BK * 2 + bv * 4 + 2 * EV_STAGES * 8 +
         (kc > 0 ? bv * 4 + (2 * 128 / 4) * 2 * kc * (int)sizeof(TopkEntry) : 0) +
         (grad ? bv * 4 : 0) + 2 * 128 * bins * (int)sizeof(HistBin);
}
static_assert(ev_kmax(128) == 512 && ev_kmax(64) == EV_KMAX, "block heights");
static_assert(ev_smem_bytes(128, ev_kmax(128) / BK, 0) == 198208,
              "log-sum-exp shared memory at K = 512");
static_assert(ev_smem_bytes(128, ev_kmax(128) / BK, 32) <= 227 * 1024, "top-k shared memory");
static_assert(ev_smem_bytes(128, ev_kmax(128) / BK, 0, false, 1 << EV_RADIX_BITS) <= 227 * 1024,
              "histogram shared memory");
static_assert(ev_smem_bytes(64, ev_kmax(64) / BK, 0) == 197952,
              "log-sum-exp shared memory at K = 1024");
static_assert(ev_smem_bytes(64, ev_kmax(64) / BK, 32) <= 227 * 1024,
              "top-k and masked sampling shared memory at K = 1024");
static_assert(ev_smem_bytes(64, ev_kmax(64) / BK, 0, false, 1 << EV_RADIX_BITS) <= 227 * 1024,
              "histogram shared memory at K = 1024");
static_assert(ev_smem_bytes(64, ev_kmax(64) / BK, 0, true) == 198208,
              "gradient shared memory at K = 1024");

}  // namespace tc

namespace {

// EvalArgs and the X tensor map shared by both entry points; returns 0, a negative argument error
// or a CUDA error code
int ev_setup(tc::EvalArgs& a, CUtensorMap& tx, int& grid, const void* X, int N, int K,
             const void* w_ptrs, int w_pitch, const void* b_ptrs, int b_pitch, int b_bf16,
             const int* row_cnt, int slots, const GroupGeom* g, int rank, const void* hdr_mine,
             const void* ctl, int wait, void* ws, int ws_ctas) {
  using namespace tc;
  if (K < 8 || K % 8 || K > EV_KMAX || w_pitch < K || w_pitch % 8 || b_pitch % (b_bf16 ? 8 : 4)) return -1;
  if (ws_ctas < 1 || slots < 1) return -2;
  const GroupGeom G = *g;
  a = EvalArgs{};
  a.w = (const __nv_bfloat16* const*)w_ptrs; a.b = (const void* const*)b_ptrs;
  a.row_cnt = row_cnt;
  a.applied = reinterpret_cast<const uint32_t*>(hdr_mine) + PX_MAX_RANKS;
  a.ctl = (const SparseCtl*)ctl; a.ws = (float2*)ws;
  a.N = N; a.K = K; a.kb = (K + BK - 1) / BK;
  a.w_pitch = w_pitch; a.b_pitch = b_pitch;
  a.W = G.W; a.rank = rank; a.replicated = G.replicated; a.owners = G.replicated ? 1 : G.W;
  a.slots = slots; a.rows_per_part = G.rows_per_part;
  const int bv = ev_bv(K);
  a.nblk = (slots * G.rows_per_part + bv - 1) / bv;
  a.wait = wait;
  const int items = a.owners * a.nblk;
  grid = items < ws_ctas ? items : ws_ctas;
  return make_tmap(&tx, X, N, K, BM);
}

int ev_combine_blocks(int N) {
  const int blocks = (N + 7) / 8;
  return blocks > PX_NUM_SMS * 8 ? PX_NUM_SMS * 8 : blocks;
}

template <typename BiasT, int KC, bool SAMPLE = false, bool GRAD = false, int HIST = 0,
          bool MASK = false>
void ev_launch(int grid, const CUtensorMap& tx,
               const tc::EvalParams<KC, SAMPLE, GRAD, HIST, MASK>& a, cudaStream_t stream) {
  using namespace tc;
  constexpr int bins = HIST ? 1 << HIST : 0;
  // the block height of a.K; each height's shared memory limit is set at its own widest K
  const int bv = ev_bv(a.K);
  const auto kernel = bv == 128 ? px_full_softmax_lse_kernel<BiasT, 128, KC, SAMPLE, GRAD, HIST, MASK>
                                : px_full_softmax_lse_kernel<BiasT, 64, KC, SAMPLE, GRAD, HIST, MASK>;
  static bool set[2] = {false, false};
  if (!set[bv == 64]) {
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         ev_smem_bytes(bv, ev_kmax(bv) / BK, KC, GRAD, bins));
    set[bv == 64] = true;
  }
  kernel<<<grid, THREADS, ev_smem_bytes(bv, a.kb, KC, GRAD, bins), stream>>>(tx, a);
}

template <typename BiasT>
void ev_nll(int grid, const CUtensorMap& tx, const tc::EvalArgs& a, const void* X,
            const long long* targets, const void* wt, const void* bt, int V, float* nll,
            float* lse, cudaStream_t stream) {
  ev_launch<BiasT, 0>(grid, tx, a, stream);
  (lse ? tc::px_full_softmax_combine_kernel<BiasT, true>
       : tc::px_full_softmax_combine_kernel<BiasT, false>)<<<ev_combine_blocks(a.N), 256, 0,
                                                             stream>>>(
      a.ws, grid, a.N, a.K, (const __nv_bfloat16*)X, (const __nv_bfloat16*)wt, a.w_pitch,
      (const BiasT*)bt, a.b_pitch, targets, V, nll, lse);
}

// the list capacity is k rounded up to 8, 16 or 32
template <typename BiasT, bool SAMPLE, bool MASK = false>
void ev_topk(int grid, const CUtensorMap& tx, const tc::EvalParams<8, SAMPLE, false, 0, MASK>& a,
             cudaStream_t stream) {
  if (a.k <= 8) ev_launch<BiasT, 8, SAMPLE, false, 0, MASK>(grid, tx, a, stream);
  else if (a.k <= 16) ev_launch<BiasT, 16, SAMPLE, false, 0, MASK>(grid, tx, a, stream);
  else ev_launch<BiasT, 32, SAMPLE, false, 0, MASK>(grid, tx, a, stream);
}

// px_full_softmax_topk (SAMPLE = false: inv_tau, seed and row0 unused), px_full_softmax_sample
// and px_full_softmax_sample_masked (MASK: rows holds each row's threshold)
template <bool SAMPLE, bool MASK = false>
int ev_lists(const void* X, int N, int K, const void* w_ptrs, int w_pitch, const void* b_ptrs,
             int b_pitch, int b_bf16, const int* row_cnt, const int* part_idx, int slots,
             const GroupGeom* g, int rank, const void* hdr_mine, const void* ctl, int wait,
             void* ws, int ws_ctas, int k, void* tk, float* log_probs, long long* ids,
             float inv_tau, uint32_t seed, int row0, const void* rows, cudaStream_t stream) {
  using namespace tc;
  if (N <= 0) return 0;
  if (ws_ctas > 32 * TK_LISTS_PER_LANE) return -2;
  MaskArgs a;
  CUtensorMap tx;
  int grid;
  int rc = ev_setup(a, tx, grid, X, N, K, w_ptrs, w_pitch, b_ptrs, b_pitch, b_bf16, row_cnt,
                    slots, g, rank, hdr_mine, ctl, wait, ws, ws_ctas);
  if (rc) return rc;
  a.tk = (TopkEntry*)tk; a.part_idx = part_idx; a.g = *g; a.k = k;
  a.inv_tau = inv_tau; a.seed = seed; a.row0 = row0;
  a.rows = (const TruncRow*)rows;
  (b_bf16 ? ev_topk<__nv_bfloat16, SAMPLE, MASK> : ev_topk<float, SAMPLE, MASK>)(grid, tx, a,
                                                                                 stream);
  px_full_softmax_topk_combine_kernel<SAMPLE><<<ev_combine_blocks(N), 256, 0, stream>>>(
      (const float2*)ws, (const TopkEntry*)tk, grid, N, k, log_probs, ids, seed, row0);
  return (int)cudaGetLastError();
}

// the setup of px_full_softmax_sample_lse and px_full_softmax_radix: ev_setup and inv_tau
int ev_temp_setup(tc::TempArgs& a, CUtensorMap& tx, int& grid, const void* X, int N, int K,
                  const void* w_ptrs, int w_pitch, const void* b_ptrs, int b_pitch, int b_bf16,
                  const int* row_cnt, int slots, const GroupGeom* g, int rank,
                  const void* hdr_mine, const void* ctl, int wait, void* ws, int ws_ctas,
                  float inv_tau) {
  if (!(inv_tau > 0.f) || !isfinite(inv_tau)) return -4;
  const int rc = ev_setup(a, tx, grid, X, N, K, w_ptrs, w_pitch, b_ptrs, b_pitch, b_bf16, row_cnt,
                          slots, g, rank, hdr_mine, ctl, wait, ws, ws_ctas);
  a.inv_tau = inv_tau;
  return rc;
}

}  // namespace

extern "C" {

// nll[N] (fp32) of X [N, K] (bf16, K-contiguous, K % 8 == 0, 8 <= K <= 1024) against a
// (weight, bias) co-lookup group.
//   w_ptrs / b_ptrs: device arrays of every rank's weight shadow (bf16, row pitch w_pitch) and
//                    bias master rows (fp32, or bf16 when b_bf16; row pitch b_pitch elements,
//                    16 bytes apart or a multiple of them);
//   row_cnt:         [owners][slots] real rows of the partition stored in each slot (owners = 1
//                    for a replicated layout, else W);
//   ws:              fp32 [ws_ctas][N][2] scratch, the grid is at most ws_ctas CTAs;
//   targets:         int64 [N]; wt / bt: the targets' rows from the group lookup (same pitches
//                    and types);
//   lse:             null, or fp32 [N] out: each row's log-sum-exp (kept for the backward).
// Returns 0, a negative argument error, or a CUDA error code.
int px_full_softmax_nll(const void* X, int N, int K, const void* w_ptrs, int w_pitch,
                        const void* b_ptrs, int b_pitch, int b_bf16, const int* row_cnt,
                        int slots, const GroupGeom* g, int rank, const void* hdr_mine,
                        const void* ctl, int wait, void* ws, int ws_ctas, const long long* targets,
                        const void* wt, const void* bt, float* nll, float* lse,
                        cudaStream_t stream) {
  using namespace tc;
  if (N <= 0) return 0;
  EvalArgs a;
  CUtensorMap tx;
  int grid;
  int rc = ev_setup(a, tx, grid, X, N, K, w_ptrs, w_pitch, b_ptrs, b_pitch, b_bf16, row_cnt,
                    slots, g, rank, hdr_mine, ctl, wait, ws, ws_ctas);
  if (rc) return rc;
  (b_bf16 ? ev_nll<__nv_bfloat16> : ev_nll<float>)(grid, tx, a, X, targets, wt, bt, g->V, nll,
                                                   lse, stream);
  return (int)cudaGetLastError();
}

// The k largest logits of each row of X [N, K] against a (weight, bias) co-lookup group:
// log_probs fp32 [N, k] (logit − logsumexp of the row) and ids int64 [N, k], logit descending and
// equal logits by ascending id.  Arguments as px_full_softmax_nll, without targets, plus
//   part_idx: [owners][slots] partition held in each slot (-1: none; [1][1] = {0} replicated);
//   k:        1 <= k <= 32; the kernel's list capacity is k rounded up to 8, 16 or 32;
//   tk:       [ws_ctas][N][k] 8-byte (fp32 logit, int32 id) scratch.  ws_ctas <= 256.
// Returns 0, a negative argument error (-3: k out of range), or a CUDA error code.
int px_full_softmax_topk(const void* X, int N, int K, const void* w_ptrs, int w_pitch,
                         const void* b_ptrs, int b_pitch, int b_bf16, const int* row_cnt,
                         const int* part_idx, int slots, const GroupGeom* g, int rank,
                         const void* hdr_mine, const void* ctl, int wait, void* ws, int ws_ctas,
                         int k, void* tk, float* log_probs, long long* ids, cudaStream_t stream) {
  if (k < 1 || k > 32) return -3;
  return ev_lists<false>(X, N, K, w_ptrs, w_pitch, b_ptrs, b_pitch, b_bf16, row_cnt, part_idx,
                         slots, g, rank, hdr_mine, ctl, wait, ws, ws_ctas, k, tk, log_probs, ids,
                         1.f, 0u, 0, nullptr, stream);
}

// n draws without replacement from softmax((X w^T + b) / τ) for each row of X [N, K], in draw
// order (Gumbel-top-k): ids int64 [N, n] are the n largest keys s − log E of the row, s = fp32
// logit · inv_tau and E the noise of (seed, row0 + row, id) (sparse_group.cuh), so a row's draws
// depend on its index in the caller's batch, not on the chunk; log_probs fp32 [N, n] are s − lse
// at those ids.  Arguments as px_full_softmax_topk with k = n (tk holds (key, id) entries), plus
//   inv_tau: fp32(1/τ), finite and > 0;   seed: the call's seed;   row0: batch index of X's row 0.
// Returns 0, a negative argument error (-3: n out of range, -4: inv_tau not finite and > 0), or a
// CUDA error code.
int px_full_softmax_sample(const void* X, int N, int K, const void* w_ptrs, int w_pitch,
                           const void* b_ptrs, int b_pitch, int b_bf16, const int* row_cnt,
                           const int* part_idx, int slots, const GroupGeom* g, int rank,
                           const void* hdr_mine, const void* ctl, int wait, void* ws, int ws_ctas,
                           int n, void* tk, float* log_probs, long long* ids, float inv_tau,
                           unsigned int seed, int row0, cudaStream_t stream) {
  if (n < 1 || n > 32) return -3;
  if (!(inv_tau > 0.f) || !isfinite(inv_tau)) return -4;
  return ev_lists<true>(X, N, K, w_ptrs, w_pitch, b_ptrs, b_pitch, b_bf16, row_cnt, part_idx,
                        slots, g, rank, hdr_mine, ctl, wait, ws, ws_ctas, n, tk, log_probs, ids,
                        inv_tau, seed, row0, nullptr, stream);
}

// Truncated sampling, pass 1: the log-sum-exp of s = fp32 logit · inv_tau of each row of X [N, K]
// into rows [N] (16-byte TruncRow: prefix, above, above_mass, lse), whose threshold search it
// starts.  Arguments as px_full_softmax_nll up to ws_ctas, plus inv_tau (fp32(1/τ)).
// Returns 0, a negative argument error (-4: inv_tau not finite and > 0), or a CUDA error code.
int px_full_softmax_sample_lse(const void* X, int N, int K, const void* w_ptrs, int w_pitch,
                               const void* b_ptrs, int b_pitch, int b_bf16, const int* row_cnt,
                               int slots, const GroupGeom* g, int rank, const void* hdr_mine,
                               const void* ctl, int wait, void* ws, int ws_ctas, float inv_tau,
                               void* rows, cudaStream_t stream) {
  using namespace tc;
  if (N <= 0) return 0;
  TempArgs a;
  CUtensorMap tx;
  int grid;
  int rc = ev_temp_setup(a, tx, grid, X, N, K, w_ptrs, w_pitch, b_ptrs, b_pitch, b_bf16, row_cnt,
                         slots, g, rank, hdr_mine, ctl, wait, ws, ws_ctas, inv_tau);
  if (rc) return rc;
  (b_bf16 ? ev_launch<__nv_bfloat16, 0, true> : ev_launch<float, 0, true>)(grid, tx, a, stream);
  px_full_softmax_trunc_init_kernel<<<ev_combine_blocks(N), 256, 0, stream>>>(
      (const float2*)ws, grid, N, (TruncRow*)rows);
  return (int)cudaGetLastError();
}

// Truncated sampling, one radix pass: the histogram of the d-bit digit at bit lo (d =
// EV_RADIX_BITS; lo = 32 − d, 32 − 2d, ..., 0 in turn) of the keys that match each row's prefix,
// into hist [ws_ctas][N][2^d] 8-byte (count, mass) bins, then the digit of θ* into rows.  After the
// pass at lo = 0, rows[].prefix is the key of θ*.  Arguments as px_full_softmax_sample_lse, hist
// in place of ws, plus
//   k: top_k, 0 for none, else in [n, V];   p: top_p, 0 for none, else in (0, 1];
//   n: the number of samples, in [1, 32].
// Returns 0, a negative argument error (-2: lo not a digit position, -3: n out of range, -4:
// inv_tau not finite and > 0, -5: k out of range, -6: p out of range), or a CUDA error code.
int px_full_softmax_radix(const void* X, int N, int K, const void* w_ptrs, int w_pitch,
                          const void* b_ptrs, int b_pitch, int b_bf16, const int* row_cnt,
                          int slots, const GroupGeom* g, int rank, const void* hdr_mine,
                          const void* ctl, int wait, void* hist, int ws_ctas, float inv_tau,
                          void* rows, int lo, int k, float p, int n, cudaStream_t stream) {
  using namespace tc;
  constexpr int D = EV_RADIX_BITS;
  if (lo < 0 || lo > 32 - D || lo % D) return -2;
  if (n < 1 || n > 32) return -3;
  if (k != 0 && (k < n || k > g->V)) return -5;
  if (!(p >= 0.f && p <= 1.f)) return -6;
  if (N <= 0) return 0;
  HistArgs a;
  CUtensorMap tx;
  int grid;
  int rc = ev_temp_setup(a, tx, grid, X, N, K, w_ptrs, w_pitch, b_ptrs, b_pitch, b_bf16, row_cnt,
                         slots, g, rank, hdr_mine, ctl, wait, nullptr, ws_ctas, inv_tau);
  if (rc) return rc;
  a.rows = (const TruncRow*)rows; a.hist = (HistBin*)hist; a.lo = lo;
  a.himask = lo + D >= 32 ? 0u : ~0u << (lo + D);
  (b_bf16 ? ev_launch<__nv_bfloat16, 0, true, false, D> : ev_launch<float, 0, true, false, D>)(
      grid, tx, a, stream);
  px_full_softmax_select_kernel<D><<<ev_combine_blocks(N), 256, 0, stream>>>(
      (const HistBin*)hist, grid, N, (TruncRow*)rows, lo, k, p, n);
  return (int)cudaGetLastError();
}

// Truncated sampling, last pass: px_full_softmax_sample restricted to each row's T, the words
// whose key of s is >= rows[].prefix after the last radix pass (the −inf keys of the rest are
// set after the (max, Σexp) pairs, so log_probs are those of the untruncated softmax).  Arguments
// and return codes as px_full_softmax_sample, plus rows.  T must hold at least n words.
int px_full_softmax_sample_masked(const void* X, int N, int K, const void* w_ptrs, int w_pitch,
                                  const void* b_ptrs, int b_pitch, int b_bf16, const int* row_cnt,
                                  const int* part_idx, int slots, const GroupGeom* g, int rank,
                                  const void* hdr_mine, const void* ctl, int wait, void* ws,
                                  int ws_ctas, int n, void* tk, float* log_probs, long long* ids,
                                  float inv_tau, unsigned int seed, int row0, const void* rows,
                                  cudaStream_t stream) {
  if (n < 1 || n > 32) return -3;
  if (!(inv_tau > 0.f) || !isfinite(inv_tau)) return -4;
  return ev_lists<true, true>(X, N, K, w_ptrs, w_pitch, b_ptrs, b_pitch, b_bf16, row_cnt,
                              part_idx, slots, g, rank, hdr_mine, ctl, wait, ws, ws_ctas, n, tk,
                              log_probs, ids, inv_tau, seed, row0, rows, stream);
}

// The gradient of the full-softmax NLL over one chunk of the table, global ids [v0, v0 + rows):
//   G  [N][g_pitch] bf16 = g_i · (exp(x_i · w_v + b_v − lse_i) − [v == t_i]),  v in the chunk
//   db [rows] fp32       = Σ_i G[i][v]
// X [N, K] bf16 as px_full_softmax_nll; wc / bc: the chunk's bf16 weight rows and bias rows (fp32,
// or bf16 when b_bf16), row pitches w_pitch / b_pitch elements as px_full_softmax_nll; lse, g fp32
// [N] and targets int64 [N].  Columns of G from rows to rows rounded up to the block height (128
// rows for K <= 512, 64 for 512 < K <= 1024) are written as zero, later ones are not written;
// g_pitch >= rows rounded up to the block height, even.  Grid <= ctas CTAs.
// Returns 0, a negative argument error, or a CUDA error code.
int px_full_softmax_grad(const void* X, int N, int K, const void* wc, int w_pitch, const void* bc,
                         int b_pitch, int b_bf16, int rows, long long v0, const float* lse,
                         const float* g, const long long* targets, void* G, int g_pitch,
                         float* db, int ctas, cudaStream_t stream) {
  using namespace tc;
  if (N <= 0 || rows <= 0) return 0;
  if (K < 8 || K % 8 || K > EV_KMAX || w_pitch < K || w_pitch % 8 || b_pitch % (b_bf16 ? 8 : 4))
    return -1;
  const int bv = ev_bv(K);
  const int nblk = (rows + bv - 1) / bv;
  if (ctas < 1 || g_pitch % 2 || g_pitch < nblk * bv) return -2;
  GradArgs a{};
  a.N = N; a.K = K; a.kb = (K + BK - 1) / BK;
  a.w_pitch = w_pitch; a.b_pitch = b_pitch;
  a.W = 1; a.rank = 0; a.replicated = 1; a.owners = 1; a.slots = 1; a.rows_per_part = rows;
  a.nblk = nblk;
  a.wc = (const __nv_bfloat16*)wc; a.bc = bc; a.rows = rows; a.v0 = v0;
  a.lse = lse; a.g = g; a.targets = targets;
  a.G = (__nv_bfloat16*)G; a.g_pitch = g_pitch; a.db = db;
  CUtensorMap tx;
  int rc = make_tmap(&tx, X, N, K, BM);
  if (rc) return rc;
  const int grid = nblk < ctas ? nblk : ctas;
  (b_bf16 ? ev_launch<__nv_bfloat16, 0, false, true> : ev_launch<float, 0, false, true>)(
      grid, tx, a, stream);
  return (int)cudaGetLastError();
}

}  // extern "C"
