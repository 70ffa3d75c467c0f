// Sparse path, one *group* of co-indexed tables per launch:
//   px_sparse_lookup_kernel  remote-gather lookup (NVLink peer loads), all member tables
//   px_sparse_push_kernel    local aggregation (SMEM dedup) + P2P push + `pushed` flag:
//                            ONE launch per group and step
//   px_sparse_owner_kernel   owner side: cross-source merge + sparse optimizer + `applied`
//                            flag: ONE (cooperative) launch per group and step
// (async / Hogwild mode: the push kernel applies the optimizer remotely, no owner kernel.)
//
// A group is a set of row-partitioned tables that share (V, P, strategy, owner map) and are
// looked up with the SAME ids in one call (LM1B: softmax_w + softmax_b; any single table is a
// group of one).  The ids are deduplicated once and every member table's rows travel together.
//
// What this replaces in the reference (SURVEY §3.3): worker GPU → local-chief CPU
// SparseConditionalAccumulator → gRPC → PS CPU accumulator (sorted two-pointer merge, whole
// value tensor re-allocated per apply, tensorflow/core/kernels/sparse_conditional_accumulator.h
// :192-319) → chief take_grad → serial CPU SparseApplyAdagrad row loop (tensorflow/core/kernels/
// training_ops.cc:1338-1351) → token queues; and for lookups dynamic_partition → per-shard PS CPU
// gather → gRPC → dynamic_stitch (tensorflow/python/ops/embedding_ops.py:151-209,
// gather_functor_gpu.cu.h:32-70, dynamic_partition_op_gpu.cu.cc:60-110).
//
// Step protocol (sync mode); flags are monotonically increasing step numbers in the group's
// symmetric header, written with st.release.sys and polled with ld.acquire.sys:
//   lookup(t)  waits applied[o] >= t-1 for every owner o   (rows fresh, receive rings drained)
//   push(t)    writes rows + local row ids + counts into the owner's ring[src = me], then
//              pushed[me] = t at the owner
//   owner(t)   waits pushed[s] >= t for every source s, links the entries of every touched row
//              into a list (one atomicExch per entry), grid barrier, then the list head sums the
//              (bf16 or fp32) wire rows in fp32 and applies the optimizer once per row; publishes
//              applied[me] = t to every rank.
//
// Wire format ("boundary between workers and servers", graph_transform_lib.py:1315-1370): rows
// cross NVLink in the gradient's own dtype (bf16 gradients stay bf16; the widening cast runs on the
// owner, after the wire) unless the boundary optimisation is switched off, in which case the
// sender widens to fp32 first.
#include "common.cuh"
#include "launch.h"
#include "optim_rules.cuh"
#include "sparse_group.cuh"

#include <algorithm>
#include <climits>
#include <mutex>
#include <string>
#include <unordered_map>

#define PX_SMEM_PARTS 1024

__device__ __forceinline__ void geom_part(const GroupGeom& g, int id, int& p, int& idx) {
  if (g.strategy == 0) { p = id % g.P; idx = id / g.P; }
  else {
    const int thr = g.extras * (g.base + 1);
    if (id < thr) { p = id / (g.base + 1); idx = id - p * (g.base + 1); }
    else { p = (id - g.extras) / max(g.base, 1); idx = id - (p * g.base + g.extras); }
  }
}

__device__ __forceinline__ void geom_map(const GroupGeom& g, int id, int& owner, int& local) {
  if (g.replicated) { owner = 0; local = id; return; }
  int p, idx;
  geom_part(g, id, p, idx);
  owner = __ldg(g.part_owner + p);
  local = __ldg(g.part_slot + p) * g.rows_per_part + idx;
}

// the CTA of a grid of G that owns id: the push kernel hash-partitions ids over its CTAs
__device__ __forceinline__ int hash_cta(int id, int G) {
  uint32_t x = (uint32_t)id * 2654435761u;
  return (int)(((unsigned long long)(x ^ (x >> 15)) * (unsigned)G) >> 32);
}
__device__ __forceinline__ uint32_t hash_slot(int id) {
  uint32_t x = (uint32_t)id * 0x85EBCA6Bu;
  x ^= x >> 13; x *= 0xC2B2AE35u;
  return x ^ (x >> 16);
}

// 4 fp32 <-> 4 bf16 (round to nearest even) in 8 bytes
__device__ __forceinline__ uint2 pack_bf16x4(const float4& v) {
  __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
  return make_uint2(*reinterpret_cast<uint32_t*>(&lo), *reinterpret_cast<uint32_t*>(&hi));
}
__device__ __forceinline__ float4 unpack_bf16x4(const uint2& v) {
  return make_float4(__uint_as_float(v.x << 16), __uint_as_float(v.x & 0xffff0000u),
                     __uint_as_float(v.y << 16), __uint_as_float(v.y & 0xffff0000u));
}

// ---- stochastic rounding of bf16 master rows (sparse_weights="bf16"); `optim.py` holds the same
// hash and rounding in torch arithmetic, and the two agree bit for bit.
// The 16 random bits of element (row, col) are a hash of the table's seed, the global step, the
// row's GLOBAL id and the column only: replicas, world sizes and partitionings round alike.
// sr_mix is in sparse_group.cuh.
__device__ __forceinline__ uint32_t sr_row_key(uint32_t seed, uint32_t step, uint32_t gid) {
  return sr_mix(sr_mix(seed ^ step) ^ gid);
}
// bf16 bits of finite x: the top half of (bits(x) + r), r uniform in [0, 2^16) — x rounds away
// from zero with probability equal to its fraction of an ulp.  Inf stays Inf, NaN stays NaN.
__device__ __forceinline__ uint32_t sr_bf16(float x, uint32_t key, uint32_t col) {
  const uint32_t u = __float_as_uint(x);
  if ((u & 0x7f800000u) == 0x7f800000u) return (u >> 16) | ((u & 0x7fffffu) ? 0x40u : 0u);
  return (u + (sr_mix(key ^ col) >> 16)) >> 16;
}
// 4 elements, columns col .. col+3 of the row with hash key `key`
__device__ __forceinline__ uint2 pack_bf16x4_sr(const float4& v, uint32_t key, uint32_t col) {
  return make_uint2(sr_bf16(v.x, key, col) | (sr_bf16(v.y, key, col + 1) << 16),
                    sr_bf16(v.z, key, col + 2) | (sr_bf16(v.w, key, col + 3) << 16));
}

// 4 master elements (float4 group c) of row `row`: fp32 rows of D4 groups, or bf16 rows padded to
// a multiple of 8 columns (the shadow's layout)
__device__ __forceinline__ size_t bf16_row_groups(int D4) { return (size_t)((D4 + 1) / 2 * 2); }
__device__ __forceinline__ float4 ld_master4(const float* t, size_t row, int D4, int c) {
  return reinterpret_cast<const float4*>(t)[row * D4 + c];
}
__device__ __forceinline__ float4 ld_master4(const __nv_bfloat16* t, size_t row, int D4, int c) {
  return unpack_bf16x4(reinterpret_cast<const uint2*>(t)[row * bf16_row_groups(D4) + c]);
}
// ... and their store; a bf16 row is rounded stochastically with the row's hash key
__device__ __forceinline__ void st_master4(float* t, size_t row, int D4, int c, const float4& w,
                                           uint32_t) {
  reinterpret_cast<float4*>(t)[row * D4 + c] = w;
}
__device__ __forceinline__ void st_master4(__nv_bfloat16* t, size_t row, int D4, int c,
                                           const float4& w, uint32_t key) {
  reinterpret_cast<uint2*>(t)[row * bf16_row_groups(D4) + c] = pack_bf16x4_sr(w, key, 4 * c);
}

// ------------------------------------------------------------------ lookup
struct LookupTable {
  const void* const* srcs;      // device array[W]: fp32 tables or bf16 shadows of every rank
  void* out;                    // [n, D4*4] rows
  int D4;
  int src_bf16;                 // 1: srcs are bf16 shadow copies (out is bf16 too)
  int out_bf16;
};
struct LookupArgs {
  LookupTable t[PX_GRP_MAX];
  int nt;
};

// out_t[i,:] = table_t@owner(ids[i])[local(ids[i]), :] for every member table; LPR lanes per row.
template <typename IdT>
__global__ void __launch_bounds__(256)
px_sparse_lookup_kernel(const IdT* __restrict__ ids, int n, LookupArgs a,
                        int32_t* __restrict__ pend_ids, GroupGeom g, const uint32_t* applied,
                        const SparseCtl* ctl, int lpr, int wait) {
  if (wait) {
    if (threadIdx.x < g.W) {
      const uint32_t need = ctl->step;
      while ((int32_t)(ld_acquire_sys(applied + threadIdx.x) - need) < 0) { }
    }
    __syncthreads();
  }
  const int rows_per_block = blockDim.x / lpr;
  const int sub = threadIdx.x % lpr;
  for (int i = blockIdx.x * rows_per_block + threadIdx.x / lpr; i < n;
       i += gridDim.x * rows_per_block) {
    const long long idl = (long long)ids[i];
    const bool valid = idl >= 0 && idl < g.V;
    const int id = valid ? (int)idl : 0;
    if (pend_ids != nullptr && sub == 0) pend_ids[i] = valid ? id : -1;
    int owner, local;
    geom_map(g, id, owner, local);
#pragma unroll 1
    for (int t = 0; t < a.nt; ++t) {
      const LookupTable& T = a.t[t];
      const char* src = reinterpret_cast<const char*>(T.srcs[owner]);
      if (T.src_bf16) {
        // bf16 shadow → bf16 rows: 8 elements per 16-byte load, half the NVLink/HBM bytes
        const int nv = (T.D4 + 1) / 2;             // 16-byte vectors per row (row padded to 8)
        const uint4* s = reinterpret_cast<const uint4*>(src) + (size_t)local * nv;
        uint4* d = reinterpret_cast<uint4*>(T.out) + (size_t)i * nv;
        for (int c = sub; c < nv; c += lpr)
          st_v4(d + c, valid ? ld_v4(s + c) : make_uint4(0, 0, 0, 0));
      } else {
        const float4* s = reinterpret_cast<const float4*>(src) + (size_t)local * T.D4;
        for (int c = sub; c < T.D4; c += lpr) {
          const uint4 v = valid ? ld_v4(s + c) : make_uint4(0, 0, 0, 0);   // OOB -> zeros
          if (!T.out_bf16) {
            st_v4(reinterpret_cast<float4*>(T.out) + (size_t)i * T.D4 + c, v);
          } else {
            *reinterpret_cast<uint2*>(reinterpret_cast<char*>(T.out) +
                                      ((size_t)i * T.D4 + c) * 8) =
                pack_bf16x4(make_float4(__uint_as_float(v.x), __uint_as_float(v.y),
                                        __uint_as_float(v.z), __uint_as_float(v.w)));
          }
        }
      }
    }
  }
}

// -------------------------------------------------------------------- push
template <typename GradT>
__device__ __forceinline__ float4 ld_grad4(const GradT* base, size_t f4_index) {
  if (sizeof(GradT) == 4) {
    const uint4 v = ld_v4_stream(reinterpret_cast<const float4*>(base) + f4_index);
    return make_float4(__uint_as_float(v.x), __uint_as_float(v.y), __uint_as_float(v.z),
                       __uint_as_float(v.w));
  } else {
    return unpack_bf16x4(*reinterpret_cast<const uint2*>(reinterpret_cast<const char*>(base) +
                                                         f4_index * 8));
  }
}

template <typename WireT>
__device__ __forceinline__ void st_wire4(char* row_base, int c, const float4& v) {
  if (sizeof(WireT) == 4) {
    st_v4_stream(reinterpret_cast<float4*>(row_base) + c,
                 make_uint4(__float_as_uint(v.x), __float_as_uint(v.y), __float_as_uint(v.z),
                            __float_as_uint(v.w)));
  } else {
    const uint2 o = pack_bf16x4(v);
    asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1,%2};"
                 ::"l"(row_base + (size_t)c * 8), "r"(o.x), "r"(o.y) : "memory");
  }
}
template <typename WireT>
__device__ __forceinline__ float4 ld_wire4(const char* row_base, int c) {
  if (sizeof(WireT) == 4) {
    const uint4 v = ld_v4_stream(reinterpret_cast<const float4*>(row_base) + c);
    return make_float4(__uint_as_float(v.x), __uint_as_float(v.y), __uint_as_float(v.z),
                       __uint_as_float(v.w));
  } else {
    uint2 v;
    asm volatile("ld.global.L1::no_allocate.v2.u32 {%0,%1}, [%2];"
                 : "=r"(v.x), "=r"(v.y) : "l"(row_base + (size_t)c * 8) : "memory");
    return unpack_bf16x4(v);
  }
}

// bf16 shadow of 4 elements of one table row (shadow rows are padded to a multiple of 8)
__device__ __forceinline__ void store_shadow4(__nv_bfloat16* shadow, size_t row, int D4, int c,
                                              const float4& w) {
  *reinterpret_cast<uint2*>(reinterpret_cast<char*>(shadow) + (row * ((D4 + 1) / 2 * 2) + c) * 8) =
      pack_bf16x4(w);
}

// optimizer on 4 elements of one table row (+ bf16 shadow refresh); used by the owner kernel on
// local rows and by the async push on remote rows.  MT: the master rows' type; a bf16 master
// (no shadow) is rounded stochastically with the row's hash key `key`.
template <int FAM, typename MT = float>
__device__ __forceinline__ void px_row_apply4(int kind, const PxHP& h, const float4& g,
                                              MT* table, float* slot0, float* slot1,
                                              float* slot2, __nv_bfloat16* shadow, size_t row,
                                              int D4, int c, uint32_t key = 0) {
  const size_t off = row * D4 + c;
  float4* p0 = slot0 ? reinterpret_cast<float4*>(slot0) + off : nullptr;
  float4* p1 = slot1 ? reinterpret_cast<float4*>(slot1) + off : nullptr;
  float4* p2 = (FAM == 1 && slot2) ? reinterpret_cast<float4*>(slot2) + off : nullptr;
  const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 w = ld_master4(table, row, D4, c), s0 = z, s1 = z, s2 = z;
  if (p0) s0 = *p0;
  if (p1) s1 = *p1;
  if (p2) s2 = *p2;
  px_rule4<FAM>(kind, h, g, w, s0, s1, s2);
  st_master4(table, row, D4, c, w, key);
  if (p0) *p0 = s0;
  if (p1) *p1 = s1;
  if (p2) *p2 = s2;
  if (sizeof(MT) == 4 && shadow) store_shadow4(shadow, row, D4, c, w);
}

// same for 8 consecutive elements (two float4 groups 2*c2, 2*c2+1): every load is issued
// before the first store (table / slot pointers may alias as far as the compiler knows, so
// two back-to-back px_row_apply4 calls would serialise load -> store -> load)
template <int FAM, typename MT = float>
__device__ __forceinline__ void px_row_apply8(int kind, const PxHP& h, const float* g,
                                              MT* table, float* slot0, float* slot1,
                                              float* slot2, __nv_bfloat16* shadow, size_t row,
                                              int D4, int c2, uint32_t key = 0) {
  const size_t off = row * D4 + 2 * c2;
  float4* p0 = slot0 ? reinterpret_cast<float4*>(slot0) + off : nullptr;
  float4* p1 = slot1 ? reinterpret_cast<float4*>(slot1) + off : nullptr;
  float4* p2 = (FAM == 1 && slot2) ? reinterpret_cast<float4*>(slot2) + off : nullptr;
  float4* pw = reinterpret_cast<float4*>(table) + off;                        // fp32 master
  uint4* pb = reinterpret_cast<uint4*>(table) + row * ((D4 + 1) / 2) + c2;   // bf16 master
  const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 w[2] = {z, z}, s0[2] = {z, z}, s1[2] = {z, z}, s2[2] = {z, z};
  if constexpr (sizeof(MT) == 4) {
    w[0] = pw[0]; w[1] = pw[1];
  } else {
    float f[8];
    Vec16<__nv_bfloat16>::unpack(*pb, f);
    w[0] = make_float4(f[0], f[1], f[2], f[3]);
    w[1] = make_float4(f[4], f[5], f[6], f[7]);
  }
  if (p0) { s0[0] = p0[0]; s0[1] = p0[1]; }
  if (p1) { s1[0] = p1[0]; s1[1] = p1[1]; }
  if (p2) { s2[0] = p2[0]; s2[1] = p2[1]; }
  px_rule4<FAM>(kind, h, make_float4(g[0], g[1], g[2], g[3]), w[0], s0[0], s1[0], s2[0]);
  px_rule4<FAM>(kind, h, make_float4(g[4], g[5], g[6], g[7]), w[1], s0[1], s1[1], s2[1]);
  if constexpr (sizeof(MT) == 4) {
    pw[0] = w[0]; pw[1] = w[1];
  } else {
    const uint2 lo = pack_bf16x4_sr(w[0], key, 8 * c2), hi = pack_bf16x4_sr(w[1], key, 8 * c2 + 4);
    *pb = make_uint4(lo.x, lo.y, hi.x, hi.y);
  }
  if (p0) { p0[0] = s0[0]; p0[1] = s0[1]; }
  if (p1) { p1[0] = s1[0]; p1[1] = s1[1]; }
  if (p2) { p2[0] = s2[0]; p2[1] = s2[1]; }
  if (sizeof(MT) == 4 && shadow) {
    const float f[8] = {w[0].x, w[0].y, w[0].z, w[0].w, w[1].x, w[1].y, w[1].z, w[1].w};
    st_v4(reinterpret_cast<uint4*>(shadow) + row * ((D4 + 1) / 2) + c2,
          Vec16<__nv_bfloat16>::pack(f));
  }
}

struct PushTable {
  const void* grads;            // [n, D4*4] gradient rows (GradT)
  float* staging;               // [n/2+1, D4*4] fp32 rows for ids carried by several positions
  char* const* rings;           // sync: device array[W] of receive-ring bases
  float* const* tables;         // async: device arrays[W] for the remote optimizer application
  float* const* slot0s;
  float* const* slot1s;
  float* const* slot2s;
  __nv_bfloat16* const* shadows;
  const float* hp;
  int D4, kind;
  float scale;                  // ScaleGradients factor when it runs on the sender
};
struct PushArgs {
  PushTable t[PX_GRP_MAX];
  int nt;
  int32_t* const* ring_ids;     // device array[W]: id rings ([W_src][cap] local rows)
  uint32_t* const* hdrs;        // device array[W]: group headers
  int cap, rank;
};

// destination of one row (all member tables): the owner's ring slot (sync) or the owner's
// table row itself (async)
template <typename WireT, bool ASYNC, int FAM>
__device__ __forceinline__ void emit_row(const PushArgs& a, const GroupGeom& g, int t, int owner,
                                         int local, int k, int c, float4 v) {
  const PushTable& T = a.t[t];
  if (!ASYNC) {
    const size_t row_bytes = (size_t)T.D4 * 4 * sizeof(WireT);
    if (g.replicated) {
      for (int p = 0; p < g.W; ++p) {
        const int q = (a.rank + p) % g.W;
        st_wire4<WireT>(T.rings[q] + ((size_t)a.rank * a.cap + k) * row_bytes, c, v);
      }
    } else {
      st_wire4<WireT>(T.rings[owner] + ((size_t)a.rank * a.cap + k) * row_bytes, c, v);
    }
  } else {
    px_row_apply4<FAM>(T.kind, px_load_hp(T.hp), v, T.tables[owner],
                       T.slot0s ? T.slot0s[owner] : nullptr, T.slot1s ? T.slot1s[owner] : nullptr,
                       T.slot2s ? T.slot2s[owner] : nullptr,
                       T.shadows ? T.shadows[owner] : nullptr, (size_t)local, T.D4, c);
  }
}

__device__ __forceinline__ void emit_id(const PushArgs& a, const GroupGeom& g, int owner,
                                        int local, int k) {
  if (g.replicated) {
    for (int p = 0; p < g.W; ++p) a.ring_ids[p][(size_t)a.rank * a.cap + k] = local;
  } else {
    a.ring_ids[owner][(size_t)a.rank * a.cap + k] = local;
  }
}

// ONE launch: local aggregation + push + flag.
// The id space is partitioned over the CTAs by a hash, so every CTA owns all positions of "its"
// ids: it deduplicates them in a shared-memory hash table ("local aggregation dedups indices in
// SMEM before shipping"), reserves ring slots with one global atomic per (CTA, owner), ships rows
// whose id is unique in the batch straight from the gradient buffer, sums rows sharing an id with
// vector atomics into a local fp32 staging row (O(1) depth for Zipfian batches) and flushes those
// once.  No grid-wide phase is needed; the last CTA publishes the counts and the `pushed` flag.
// Every CTA scans all ids twice; the scans read them from a shared-memory staging chunk filled
// with 16-byte loads issued back to back (a one-id-per-trip global loop is bound by L2 latency,
// and unrolling it instead makes the kernel instruction-fetch bound).
// SMEM layout: keys[H] | cnt[H] | kk[H] (k inside the owner bucket) | dup[H] | ids[PX_ID_CHUNK]
//              | work[PX_ID_CHUNK] (positions of the current chunk that belong to this CTA)
#define PX_ID_CHUNK 4096

// stage ids[base, base+m) into shared memory: 16 ids (4 x int4) per thread in flight
__device__ __forceinline__ void stage_ids(const int32_t* __restrict__ ids, int base, int m,
                                          int32_t* ids_s) {
  int4 q[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int j = (u * blockDim.x + threadIdx.x) * 4;
    q[u] = make_int4(-1, -1, -1, -1);
    if (j + 3 < m) q[u] = __ldg(reinterpret_cast<const int4*>(ids + base + j));
    else {
      if (j < m) q[u].x = __ldg(ids + base + j);
      if (j + 1 < m) q[u].y = __ldg(ids + base + j + 1);
      if (j + 2 < m) q[u].z = __ldg(ids + base + j + 2);
    }
  }
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int j = (u * blockDim.x + threadIdx.x) * 4;
    if (j < PX_ID_CHUNK) *reinterpret_cast<int4*>(ids_s + j) = q[u];
  }
}

// read-only probe of the shared-memory id table: the slot holding id, or -1
__device__ __forceinline__ int find_key(const int32_t* keys, int H, int id) {
  uint32_t h = hash_slot(id) & (H - 1);
  int probes = 0;
  while (keys[h] != id && keys[h] != -1 && ++probes <= H) h = (h + 1) & (H - 1);
  return keys[h] == id ? (int)h : -1;
}

// the factor a row leaves with: ScaleGradients on the sender, × hp[HP_GSCALE] when async
template <bool ASYNC>
__device__ __forceinline__ float row_scale(const PushTable& T) {
  return ASYNC ? T.scale * T.hp[HP_GSCALE] : T.scale;
}

// Row pi of every member table, its id's only position, by the 16 lanes of a half-warp: into ring
// slot k of `owner`, id after it (sync; `rings`: the ring bases), or onto row `local` (async).
template <typename GradT, typename WireT, bool ASYNC, int FAM>
__device__ __forceinline__ void ship_row(const PushArgs& a, const GroupGeom& g,
                                         char* const (*rings)[PX_MAX_RANKS], int pi, int owner,
                                         int local, int k, int sub) {
#pragma unroll 1
  for (int t = 0; t < a.nt; ++t) {
    const PushTable& T = a.t[t];
    const float mul = row_scale<ASYNC>(T);
    if (!ASYNC && sizeof(GradT) == 2 && sizeof(WireT) == 2 && (T.D4 & 1) == 0 &&
        !g.replicated) {
      // bf16 gradient -> bf16 wire: 16-byte copies, four per lane in flight
      const int nv = T.D4 / 2;
      const uint4* src = reinterpret_cast<const uint4*>(T.grads) + (size_t)pi * nv;
      uint4* dst = reinterpret_cast<uint4*>(
          rings[t][owner] + ((size_t)a.rank * a.cap + k) * ((size_t)T.D4 * 8));
#pragma unroll 1
      for (int c = sub; c < nv; c += 64) {
        uint4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u)
          v[u] = c + 16 * u < nv ? ld_v4_stream(src + c + 16 * u) : make_uint4(0, 0, 0, 0);
        if (mul != 1.f) {
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            float f[8];
            Vec16<__nv_bfloat16>::unpack(v[u], f);
#pragma unroll
            for (int q = 0; q < 8; ++q) f[q] *= mul;
            v[u] = Vec16<__nv_bfloat16>::pack(f);
          }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if (c + 16 * u < nv) st_v4_stream(dst + c + 16 * u, v[u]);
      }
      continue;
    }
#pragma unroll 1
    for (int c = sub; c < T.D4; c += 16) {
      float4 v = ld_grad4<GradT>(reinterpret_cast<const GradT*>(T.grads), (size_t)pi * T.D4 + c);
      v.x *= mul; v.y *= mul; v.z *= mul; v.w *= mul;
      emit_row<WireT, ASYNC, FAM>(a, g, t, owner, local, k, c, v);
    }
  }
  if (!ASYNC && sub == 0) emit_id(a, g, owner, local, k);
}

template <typename GradT, typename WireT, bool ASYNC, int FAM>
__global__ void __launch_bounds__(256)
px_sparse_push_kernel(const int32_t* __restrict__ pend_ids, int n, PushArgs a, GroupGeom g,
                      SparseCtl* ctl, int hbits, int dedup) {
  extern __shared__ int32_t smem[];
  const int H = 1 << hbits;
  int32_t* keys = smem;
  int32_t* cnt = smem + H;
  int32_t* kk = smem + 2 * H;
  int32_t* dup = smem + 3 * H;
  int32_t* ids_s = smem + 4 * H;
  __shared__ int s_owner_cnt[PX_MAX_RANKS], s_base_k[PX_MAX_RANKS];
  __shared__ int s_ndup, s_base_dup, s_overflow;
  __shared__ bool s_last;
  // placement maps and ring bases are read for every row: keep them in shared memory (a
  // global load each would put two more memory latencies on every row's critical path)
  __shared__ short s_part_owner[PX_SMEM_PARTS], s_part_slot[PX_SMEM_PARTS];
  __shared__ char* s_ring[PX_GRP_MAX][PX_MAX_RANKS];
  const bool parts_in_smem = !g.replicated && g.P <= PX_SMEM_PARTS;
  if (parts_in_smem)
    for (int p = threadIdx.x; p < g.P; p += blockDim.x) {
      s_part_owner[p] = (short)__ldg(g.part_owner + p);
      s_part_slot[p] = (short)__ldg(g.part_slot + p);
    }
  if (!ASYNC && threadIdx.x < a.nt * PX_MAX_RANKS) {
    const int t = threadIdx.x / PX_MAX_RANKS, r = threadIdx.x % PX_MAX_RANKS;
    s_ring[t][r] = r < g.W ? a.t[t].rings[r] : nullptr;
  }
  auto place = [&](int id, int& owner, int& local) {
    if (parts_in_smem) {
      int p, idx;
      geom_part(g, id, p, idx);
      owner = s_part_owner[p];
      local = s_part_slot[p] * g.rows_per_part + idx;
    } else {
      geom_map(g, id, owner, local);
    }
  };
  auto owner_of = [&](int id) { int owner, local; place(id, owner, local); return owner; };
  const int G = gridDim.x, c_me = blockIdx.x;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  // CTA 0's thread 0 stamps t_push[0] at the start and t_dbg[i] at the end of each phase
  auto stamp_phase = [&](int i) {
    if (c_me == 0 && threadIdx.x == 0) ctl->t_dbg[i] = px_globaltimer();
  };
  if (c_me == 0 && threadIdx.x == 0) ctl->t_push[0] = px_globaltimer();
  for (int h = threadIdx.x; h < H; h += blockDim.x) { keys[h] = -1; cnt[h] = 0; }
  if (threadIdx.x < PX_MAX_RANKS) s_owner_cnt[threadIdx.x] = 0;
  if (threadIdx.x == 0) { s_ndup = 0; s_overflow = 0; }
  __syncthreads();
  // ---- pass 1: insert my ids, count positions per id (raw mode: count my positions per owner)
  for (int base = 0; base < n; base += PX_ID_CHUNK) {
    const int m = min(PX_ID_CHUNK, n - base);
    stage_ids(pend_ids, base, m, ids_s);
    __syncthreads();
#pragma unroll 1
    for (int j = threadIdx.x; j < m; j += blockDim.x) {
      const int id = ids_s[j];
      if (id < 0) continue;
      if (!dedup) {
        if ((base + j) % G == c_me) atomicAdd(&s_owner_cnt[owner_of(id)], 1);
        continue;
      }
      if (hash_cta(id, G) != c_me) continue;
      uint32_t h = hash_slot(id) & (H - 1);
      int probes = 0;
      while (true) {
        const int old = atomicCAS(&keys[h], -1, id);
        if (old == -1 || old == id) { atomicAdd(&cnt[h], 1); break; }
        h = (h + 1) & (H - 1);
        if (++probes >= H) { atomicAdd(&s_overflow, 1); break; }   // table full: raw entry later
      }
    }
    __syncthreads();
  }
  stamp_phase(0);
  if (dedup) {
    // ---- pass 2: one ring slot per unique id, one staging row per duplicated id
    for (int h = threadIdx.x; h < H; h += blockDim.x) {
      const int id = keys[h];
      if (id < 0) continue;
      kk[h] = atomicAdd(&s_owner_cnt[owner_of(id)], 1);
      dup[h] = cnt[h] > 1 ? atomicAdd(&s_ndup, 1) : -1;
    }
    __syncthreads();
    if (s_overflow > 0) {
      // the (statistically never hit) SMEM overflow: positions whose id did not fit travel
      // as raw entries after the deduplicated ones; count them per owner
      for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int id = pend_ids[i];
        if (id < 0) continue;
        if (hash_cta(id, G) != c_me) continue;
        if (find_key(keys, H, id) < 0) atomicAdd(&s_owner_cnt[owner_of(id)], 1);
      }
      __syncthreads();
    }
  }
  if (threadIdx.x < PX_MAX_RANKS) {
    const int m = s_owner_cnt[threadIdx.x];
    s_base_k[threadIdx.x] = m > 0 ? atomicAdd(&ctl->owner_cnt[threadIdx.x], m) : 0;
    s_owner_cnt[threadIdx.x] = 0;              // re-used as the raw-entry cursor below
  }
  if (threadIdx.x == 0) {
    s_base_dup = s_ndup > 0 ? atomicAdd(&ctl->n_dup, s_ndup) : 0;
    if (s_overflow > 0) atomicAdd(&ctl->overflow, s_overflow);
  }
  __syncthreads();
  // raw entries take the slots after the deduplicated ones of this CTA
  if (dedup && s_overflow > 0) {
    for (int h = threadIdx.x; h < H; h += blockDim.x) {
      if (keys[h] >= 0) atomicMax(&s_owner_cnt[owner_of(keys[h])], kk[h] + 1);
    }
    __syncthreads();
  }
  stamp_phase(1);
  // ---- pass 3: ship unique rows, stage duplicated ones.  Per chunk: (a) every thread scans
  // the staged ids and appends its CTA's positions to a work list in shared memory, (b) the
  // list is processed round-robin by half-warps (16 lanes per row, four 16-byte accesses in
  // flight per lane) — balanced whatever the id distribution is.
  int32_t* work = ids_s + PX_ID_CHUNK;
  __shared__ int s_nwork;
  const int sub = lane & 15, half = lane >> 4;
  const unsigned hmask = half ? 0xffff0000u : 0x0000ffffu;
  for (int base = 0; base < n; base += PX_ID_CHUNK) {
    const int m = min(PX_ID_CHUNK, n - base);
    if (threadIdx.x == 0) s_nwork = 0;
    stage_ids(pend_ids, base, m, ids_s);
    __syncthreads();
#pragma unroll 1
    for (int j = threadIdx.x; j < m; j += blockDim.x) {
      const int id = ids_s[j];
      if (id < 0) continue;
      const bool mine = !dedup ? ((base + j) % G == c_me) : hash_cta(id, G) == c_me;
      if (mine) work[atomicAdd(&s_nwork, 1)] = j;
    }
    __syncthreads();
    if (base == 0) stamp_phase(2);
    const int nwork = s_nwork;
#pragma unroll 1
    for (int wi = wid * 2 + half; wi < nwork; wi += nwarps * 2) {
      const int j = work[wi];
      const int pi = base + j;
      const int pid = ids_s[j];
      const int ph = dedup ? find_key(keys, H, pid) : -1;
      int owner, local;
      place(pid, owner, local);
      int k = 0, pcnt = 1;
      if (ph < 0) {                       // raw entry: its own ring slot
        if (sub == 0) k = s_base_k[owner] + atomicAdd(&s_owner_cnt[owner], 1);
        k = __shfl_sync(hmask, k, half * 16);
      } else {
        k = s_base_k[owner] + kk[ph];
        pcnt = cnt[ph];
      }
      if (pcnt == 1) {
        ship_row<GradT, WireT, ASYNC, FAM>(a, g, s_ring, pi, owner, local, k, sub);
      } else {
        const int d = s_base_dup + dup[ph];
#pragma unroll 1
        for (int t = 0; t < a.nt; ++t) {
          const PushTable& T = a.t[t];
          float4* dst = reinterpret_cast<float4*>(T.staging) + (size_t)d * T.D4;
          for (int c = sub; c < T.D4; c += 16)
            atomicAdd(dst + c, ld_grad4<GradT>(reinterpret_cast<const GradT*>(T.grads),
                                               (size_t)pi * T.D4 + c));
        }
      }
    }
    __syncthreads();
  }
  stamp_phase(3);
  // every position of my duplicated ids is staged now (they are all mine)
  // ---- pass 4: flush duplicated ids (warp per id), re-zero the staging rows
  if (dedup && s_ndup > 0) {
    for (int h0 = wid * 32; h0 < H; h0 += nwarps * 32) {
      unsigned dm = __ballot_sync(0xffffffffu, keys[h0 + lane] >= 0 && cnt[h0 + lane] > 1);
      while (dm) {
        const int h = h0 + __ffs(dm) - 1;
        dm &= dm - 1;
        int owner, local;
        place(keys[h], owner, local);
        const int k = s_base_k[owner] + kk[h];
        const int d = s_base_dup + dup[h];
#pragma unroll 1
        for (int t = 0; t < a.nt; ++t) {
          const PushTable& T = a.t[t];
          const float mul = row_scale<ASYNC>(T);
          float4* src = reinterpret_cast<float4*>(T.staging) + (size_t)d * T.D4;
          for (int c = lane; c < T.D4; c += 32) {
            float4 v = __ldcg(src + c);
            __stcg(src + c, make_float4(0.f, 0.f, 0.f, 0.f));
            v.x *= mul; v.y *= mul; v.z *= mul; v.w *= mul;
            emit_row<WireT, ASYNC, FAM>(a, g, t, owner, local, k, c, v);
          }
        }
        if (!ASYNC && lane == 0) emit_id(a, g, owner, local, k);
      }
    }
  }
  stamp_phase(4);
  // ---- completion: last CTA publishes counts + `pushed` (sync) / bumps the step (async).
  // One fence per CTA: the barrier orders every thread's stores before thread 0's
  // system-scope fence (cumulativity), which orders them before the ticket and the flag.
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    s_last = (atomicAdd(&ctl->push_done, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  stamp_phase(5);
  if (!s_last) return;
  __threadfence_system();
  const uint32_t step = ctl->step + 1;
  if (!ASYNC) {
    if (threadIdx.x < g.W) {
      const int o = threadIdx.x;
      const int cn = g.replicated ? ctl->owner_cnt[0] : ctl->owner_cnt[o];
      uint32_t* hdr = a.hdrs[o];
      reinterpret_cast<volatile int32_t*>(hdr + 2 * PX_MAX_RANKS)[a.rank] = cn;   // cnt[src]
      __threadfence_system();
      st_release_sys(hdr + a.rank, step);                                         // pushed[src]
    }
    __syncthreads();
  }
  if (threadIdx.x < PX_MAX_RANKS) ctl->owner_cnt[threadIdx.x] = 0;
  if (threadIdx.x == 0) {
    ctl->n_dup = 0; ctl->push_done = 0;
    ctl->t_push[1] = px_globaltimer();
    if (ASYNC) ctl->step = step;
  }
}

// ------------------------------------------------------------------ owner
struct OwnerTable {
  char* ring;                   // my receive ring: [W_src][cap][D4*4] WireT
  void* table;                  // master rows: fp32 [rows][D4*4], or bf16 [rows][Dps] (w_bf16)
  float* slot0; float* slot1; float* slot2;
  __nv_bfloat16* shadow;        // bf16 copy read by lookups (or null)
  const float* hp;
  int D4, kind;
  float avg;                    // 1/num_workers (average_sparse) × owner-side gradient scale
  int D;                        // true row width, read by family 2 only (the row-wise rule
                                // averages Σg² over it); fills the 8-byte alignment tail
  const int32_t* slot_part;     // bf16 master: partition held in each of my slots (global ids)
  uint32_t seed;                // bf16 master: the table's stochastic-rounding seed
  int w_bf16;                   // 1: bf16 master rows, stochastically rounded; no shadow
};
struct OwnerArgs {
  OwnerTable t[PX_GRP_MAX];
  int nt;
  const int32_t* ring_ids;      // [W_src][cap]
  uint32_t* hdr;                // my group header
  uint32_t* const* hdrs;        // every rank's header (to publish `applied`)
  int32_t* slotmap;             // [rows_local], -1 when idle
  int32_t* next;                // [W_src * cap]
  int cap, rank, use_merge;
  int fixed_cnt;                // >= 0: library-collective arm — every source delivered exactly this
                                // many entries (negative row id = not mine), no flags involved
};

// Σ over the entries linked from list head e of one 4-element group of a wire row, in fp32
template <typename WireT>
__device__ __forceinline__ float4 ld_merged4(const OwnerArgs& a, const OwnerTable& T,
                                             size_t row_bytes, int e, int c) {
  float4 g = ld_wire4<WireT>(T.ring + (size_t)e * row_bytes, c);
  if (a.use_merge) {
    for (int x = __ldcg(a.next + e); x != -1; x = __ldcg(a.next + x)) {
      const float4 o = ld_wire4<WireT>(T.ring + (size_t)x * row_bytes, c);
      g.x += o.x; g.y += o.y; g.z += o.z; g.w += o.w;
    }
  }
  return g;
}

// the same for 8 elements (4-element groups 2*c2, 2*c2+1) of a bf16 wire row into f[8]: one
// 16-byte load per entry
__device__ __forceinline__ void ld_merged8(const OwnerArgs& a, const OwnerTable& T,
                                           size_t row_bytes, int e, int c2, float* f) {
  Vec16<__nv_bfloat16>::unpack(
      ld_v4_stream(reinterpret_cast<const uint4*>(T.ring + (size_t)e * row_bytes) + c2), f);
  if (a.use_merge) {
    for (int x = __ldcg(a.next + e); x != -1; x = __ldcg(a.next + x)) {
      float o[8];
      Vec16<__nv_bfloat16>::unpack(
          ld_v4_stream(reinterpret_cast<const uint4*>(T.ring + (size_t)x * row_bytes) + c2), o);
#pragma unroll
      for (int q = 0; q < 8; ++q) f[q] += o[q];
    }
  }
}

// ---- the entry walk of the owner and owner-norm kernels
// Entries of all sources form ONE index space [0, total): a (source, j) double loop would hand
// every half-warp one entry per source — W entries in sequence for the first few half-warps and
// nothing for the rest.  s_pre[s] is the index of source s's first entry; returns total.
// Every source delivered a.fixed_cnt entries when it is >= 0, else the count in its header word.
__device__ __forceinline__ int owner_prefix(const OwnerArgs& a, const GroupGeom& g, int* s_pre) {
  const uint32_t* cnt = a.hdr + 2 * PX_MAX_RANKS;
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int s = 0; s < g.W; ++s) {
      s_pre[s] = acc;
      acc += a.fixed_cnt >= 0 ? a.fixed_cnt : (int)ld_volatile_u32(cnt + s);
    }
    s_pre[g.W] = acc;
  }
  __syncthreads();
  return s_pre[g.W];
}

// index i -> ring entry e = s * cap + j; the search for source s starts at the s passed in
__device__ __forceinline__ int owner_entry(const OwnerArgs& a, const int* s_pre, int i, int& s) {
  while (i >= s_pre[s + 1]) ++s;
  return s * a.cap + (i - s_pre[s]);
}

// Merge path: every entry pushes itself on the list of its row (at most one entry per source when
// the senders aggregate locally, so lists are <= W long), then a grid barrier on ctl->bar (all
// CTAs are co-resident: cooperative launch).  The `stamp` thread times the barrier in t_dbg[6..7].
__device__ __forceinline__ void owner_link(const OwnerArgs& a, const int* s_pre, int total,
                                           SparseCtl* ctl, bool stamp) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    int s = 0;
    const int e = owner_entry(a, s_pre, i, s);
    const int r = a.ring_ids[e];
    if (r >= 0) a.next[e] = atomicExch(&a.slotmap[r], e);
  }
  if (stamp) ctl->t_dbg[6] = px_globaltimer();
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    atomicAdd(&ctl->bar, 1u);
    while (ld_volatile_u32(&ctl->bar) < gridDim.x) { }
    __threadfence();
  }
  __syncthreads();
  if (stamp) ctl->t_dbg[7] = px_globaltimer();
}

// Sorts the list of ring entries that starts at `first` by ascending entry index (source, then
// position in the source's ring), in place in next[], and returns the new first entry.  The links
// come from atomics in whatever order they ran; in this order every owner of a replicated table
// sums a row's entries alike, so the replicas stay bitwise identical (and a rerun of a step
// gives the same bits).  Bottom-up merge sort, by one lane: O(L log L) for a list of L entries;
// kept out of line so that it does not add to the owner kernels' register budget.
__device__ __noinline__ int owner_sort_list(int32_t* next, int first) {
  int len = 0;
  for (int x = first; x != -1; x = __ldcg(next + x)) ++len;
  for (int run = 1; run < len; run <<= 1) {
    int cur = first, tail = -1;
    first = -1;
    while (cur != -1) {
      // cut two runs of `run` entries off the front: [x ..] and [y ..]
      const int x0 = cur;
      int end = x0;
      for (int k = 1; k < run && __ldcg(next + end) != -1; ++k) end = __ldcg(next + end);
      const int y0 = __ldcg(next + end);
      __stcg(next + end, -1);
      cur = -1;
      if (y0 != -1) {
        end = y0;
        for (int k = 1; k < run && __ldcg(next + end) != -1; ++k) end = __ldcg(next + end);
        cur = __ldcg(next + end);
        __stcg(next + end, -1);
      }
      // merge them onto the tail of the sorted list
      int x = x0, y = y0;
      while (x != -1 || y != -1) {
        int pick;
        if (y == -1 || (x != -1 && x < y)) { pick = x; x = __ldcg(next + x); }
        else { pick = y; y = __ldcg(next + y); }
        if (tail == -1) first = pick;
        else __stcg(next + tail, pick);
        tail = pick;
      }
    }
    __stcg(next + tail, -1);
  }
  return first;
}

// 16 lanes per entry (two entries per warp in flight).  visit(i, s) runs for every entry i (of
// source s); head(e, r) for every row r with an entry of mine (without merge: for every such
// entry e), e being the first entry of the row's list once it is sorted by entry index, after
// which the half-warp resets slotmap[r] for the next step.
template <typename Visit, typename Head>
__device__ __forceinline__ void owner_walk(const OwnerArgs& a, const int* s_pre, int total,
                                           Visit visit, Head head) {
  const int warps = blockDim.x >> 4;
  const unsigned hmask = (threadIdx.x & 16) ? 0xffff0000u : 0x0000ffffu;
  for (int i = blockIdx.x * warps + (threadIdx.x >> 4); i < total; i += gridDim.x * warps) {
    int s = 0;
    const int e = owner_entry(a, s_pre, i, s);
    const int r = a.ring_ids[e];
    visit(i, s);
    if (r < 0) continue;
    if (a.use_merge && __ldcg(a.slotmap + r) != e) continue;          // not the list head
    int first = e;
    if (a.use_merge) {
      if ((threadIdx.x & 15) == 0) first = owner_sort_list(a.next, e);
      __syncwarp(hmask);                    // the sorted links are visible to the half-warp
      first = __shfl_sync(hmask, first, threadIdx.x & 16);
    }
    head(first, r);
    __syncwarp(hmask);
    if (a.use_merge && (threadIdx.x & 15) == 0) a.slotmap[r] = -1;
  }
}

// Family 2 (row-wise Adagrad) on local row r of table T, by the 16 lanes of one half-warp:
//   s[r] += (1/D) Σ_j g_j²        (T.slot0 is a dense [rows_local] fp32 array)
//   w[r, j] -= lr · g_j / (sqrt(s[r]) + eps)
// Pass 1 merges and scales the row and reduces Σg² over the 16 lanes; pass 2 updates the
// row.  Rows of up to PX_RW_REG_F4 · 64 columns keep their gradient and master values in
// registers from pass 1 (every load of the row, and lane 0's load of s[r], is then in flight
// at once); wider rows merge the gradient again from the ring in pass 2 (pass 1 just brought
// it into L2).  Padding columns carry zero gradient and stay unchanged.
#define PX_RW_REG_F4 2

template <typename MT>
__device__ __forceinline__ void px_store_row4(const OwnerTable& T, size_t row, int c,
                                              const float4& w, uint32_t key) {
  st_master4(reinterpret_cast<MT*>(T.table), row, T.D4, c, w, key);
  if (sizeof(MT) == 4 && T.shadow) store_shadow4(T.shadow, row, T.D4, c, w);
}

// the global id of my local row r (a bf16 master's rounding is keyed by it): the inverse of
// geom_map for the partition T.slot_part holds in r's slot
__device__ __forceinline__ uint32_t owner_gid(const GroupGeom& g, const OwnerTable& T, int r) {
  if (g.replicated) return (uint32_t)r;
  const int slot = r / g.rows_per_part, idx = r - slot * g.rows_per_part;
  return (uint32_t)geom_gid(g, __ldg(T.slot_part + slot), idx);
}

__device__ __forceinline__ void px_sgd4(float step, const float4& g, float4& w) {
  w.x = fmaf(-step, g.x, w.x); w.y = fmaf(-step, g.y, w.y);
  w.z = fmaf(-step, g.z, w.z); w.w = fmaf(-step, g.w, w.w);
}

template <typename WireT, typename MT>
__device__ __forceinline__ void px_rowwise_apply(const OwnerArgs& a, const OwnerTable& T, int e,
                                                 int r, int lane, unsigned hmask, uint32_t key) {
  const size_t row_bytes = (size_t)T.D4 * 4 * sizeof(WireT);
  const float gmul = T.avg * T.hp[HP_GSCALE];
  const float s_old = lane == 0 ? T.slot0[r] : 0.f;
  const bool in_regs = T.D4 <= 16 * PX_RW_REG_F4;
  const MT* wtab = reinterpret_cast<const MT*>(T.table);
  const float4* wrow = reinterpret_cast<const float4*>(T.table) + (size_t)r * T.D4;   // fp32
  float4 gk[PX_RW_REG_F4], wk[PX_RW_REG_F4];
  float ss = 0.f;
  if (in_regs) {
#pragma unroll
    for (int k = 0; k < PX_RW_REG_F4; ++k) {
      const int c = lane + 16 * k;
      if (c < T.D4) {
        if constexpr (sizeof(MT) == 4) wk[k] = wrow[c];
        else wk[k] = ld_master4(wtab, (size_t)r, T.D4, c);
        gk[k] = ld_merged4<WireT>(a, T, row_bytes, e, c);
      }
    }
#pragma unroll
    for (int k = 0; k < PX_RW_REG_F4; ++k) {
      if (lane + 16 * k < T.D4) {
        float4& g = gk[k];
        g.x *= gmul; g.y *= gmul; g.z *= gmul; g.w *= gmul;
        ss = fmaf(g.x, g.x, fmaf(g.y, g.y, fmaf(g.z, g.z, fmaf(g.w, g.w, ss))));
      }
    }
  } else {
    for (int c = lane; c < T.D4; c += 16) {
      float4 g = ld_merged4<WireT>(a, T, row_bytes, e, c);
      g.x *= gmul; g.y *= gmul; g.z *= gmul; g.w *= gmul;
      ss = fmaf(g.x, g.x, fmaf(g.y, g.y, fmaf(g.z, g.z, fmaf(g.w, g.w, ss))));
    }
  }
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) ss += __shfl_xor_sync(hmask, ss, o);
  float s = 0.f;
  if (lane == 0) {
    s = s_old + ss / (float)T.D;
    T.slot0[r] = s;
  }
  s = __shfl_sync(hmask, s, threadIdx.x & 16);
  const float step = T.hp[HP_LR] / (sqrtf(s) + T.hp[HP_EPS]);
  if (in_regs) {
#pragma unroll
    for (int k = 0; k < PX_RW_REG_F4; ++k) {
      const int c = lane + 16 * k;
      if (c < T.D4) {
        px_sgd4(step, gk[k], wk[k]);
        px_store_row4<MT>(T, (size_t)r, c, wk[k], key);
      }
    }
  } else {
    for (int c = lane; c < T.D4; c += 16) {
      float4 g = ld_merged4<WireT>(a, T, row_bytes, e, c);
      g.x *= gmul; g.y *= gmul; g.z *= gmul; g.w *= gmul;
      float4 w;
      if constexpr (sizeof(MT) == 4) w = wrow[c];
      else w = ld_master4(wtab, (size_t)r, T.D4, c);
      px_sgd4(step, g, w);
      px_store_row4<MT>(T, (size_t)r, c, w, key);
    }
  }
}

// One warp that waits for every source's `pushed` flag.  Launched right before the owner kernel
// on the comm stream: the owner's (cooperative, whole-GPU) grid then starts with its inputs
// complete instead of spinning with every register file of the device allocated while the
// backward pass on the main stream is starved — measured at N=2: 31 us of owner spinning cost
// 65 us of forward/backward time.
__global__ void px_sparse_wait_kernel(const uint32_t* hdr, const SparseCtl* ctl, int W) {
  if (threadIdx.x < W) {
    const uint32_t need = ctl->step + 1;
    while ((int32_t)(ld_acquire_sys(hdr + threadIdx.x) - need) < 0) { __nanosleep(200); }
  }
}

// ONE launch: wait for every source, merge rows that several sources touched, apply the sparse
// optimizer once per touched row, publish `applied`.  Launched cooperatively when use_merge (one
// grid barrier between linking and applying).  MT: the type of the master rows.
template <typename WireT, int FAM, typename MT = float>
__global__ void __launch_bounds__(256, FAM == 1 ? 2 : 4)
px_sparse_owner_kernel(OwnerArgs a, GroupGeom g, SparseCtl* ctl) {
  __shared__ bool s_last;
  const bool stamp = blockIdx.x == 0 && threadIdx.x == 0;
  if (stamp) ctl->t_own[0] = px_globaltimer();
  if (a.fixed_cnt < 0) {
    if (threadIdx.x < g.W) {
      const uint32_t need = ctl->step + 1;
      while ((int32_t)(ld_acquire_sys(a.hdr + threadIdx.x) - need) < 0) { }
    }
    __syncthreads();
  }
  if (stamp) ctl->t_own[1] = px_globaltimer();
  const int lane = threadIdx.x & 15, warps = blockDim.x >> 4;
  const unsigned hmask = (threadIdx.x & 16) ? 0xffff0000u : 0x0000ffffu;
  __shared__ int s_pre[PX_MAX_RANKS + 1];
  const int total = owner_prefix(a, g, s_pre);
  if (a.use_merge) owner_link(a, s_pre, total, ctl, stamp);
  // the rows of a batch are scattered over a multi-GB table: every touch is a DRAM (and usually
  // a TLB) miss.  Prefetch this half-warp's NEXT entry's table / slot rows into L2 now, so that
  // miss overlaps the work on the current entry.
  auto prefetch_next = [&](int i, int s) {
    const int in = i + gridDim.x * warps;
    if (in >= total) return;
    const int rn = a.ring_ids[owner_entry(a, s_pre, in, s)];
    if (rn < 0) return;
    for (int t = 0; t < a.nt; ++t) {
      const OwnerTable& T = a.t[t];
      const size_t off = (size_t)rn * T.D4 * 16;             // row offset in bytes
      const int lines = (T.D4 * 16 + 127) / 128;
      for (int l = lane; l < lines; l += 16) {
        if constexpr (sizeof(MT) == 4) {
          asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char*>(T.table) + off + l * 128));
        } else if (l < ((T.D4 + 1) / 2 * 16 + 127) / 128) {
          // a bf16 master row is (D4 + 1) / 2 16-byte vectors long
          asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char*>(T.table) +
                                                        (size_t)rn * ((T.D4 + 1) / 2) * 16 + l * 128));
        }
        if (FAM == 2) {
          // one fp32 accumulator per row: its pitch is 4 bytes, not the row's
          if (l == 0)
            asm volatile("prefetch.global.L2 [%0];" ::"l"(T.slot0 + rn));
          continue;
        }
        if (T.slot0)
          asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char*>(T.slot0) + off + l * 128));
        if (T.slot1)
          asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char*>(T.slot1) + off + l * 128));
      }
    }
  };
  auto apply = [&](int e, int r) {
#pragma unroll 1
    for (int t = 0; t < a.nt; ++t) {
      const OwnerTable& T = a.t[t];
      uint32_t key = 0;             // the row's rounding key (bf16 master)
      if constexpr (sizeof(MT) == 2)
        key = sr_row_key(T.seed, (uint32_t)T.hp[HP_STEP], owner_gid(g, T, r));
      if (FAM == 2) {
        px_rowwise_apply<WireT, MT>(a, T, e, r, lane, hmask, key);
        continue;
      }
      const size_t row_bytes = (size_t)T.D4 * 4 * sizeof(WireT);
      const float gmul = T.avg * T.hp[HP_GSCALE];
      const PxHP hp = px_load_hp(T.hp);
      if (sizeof(WireT) == 2 && (T.D4 & 1) == 0) {
        for (int c2 = lane; c2 < T.D4 / 2; c2 += 16) {
          float f[8];
          ld_merged8(a, T, row_bytes, e, c2, f);
#pragma unroll
          for (int q = 0; q < 8; ++q) f[q] *= gmul;
          px_row_apply8<FAM>(T.kind, hp, f, reinterpret_cast<MT*>(T.table), T.slot0, T.slot1, T.slot2, T.shadow,
                             (size_t)r, T.D4, c2, key);
        }
        continue;
      }
      for (int cidx = lane; cidx < T.D4; cidx += 16) {
        float4 gv = ld_merged4<WireT>(a, T, row_bytes, e, cidx);
        gv.x *= gmul; gv.y *= gmul; gv.z *= gmul; gv.w *= gmul;
        px_row_apply4<FAM>(T.kind, hp, gv, reinterpret_cast<MT*>(T.table), T.slot0, T.slot1, T.slot2, T.shadow,
                           (size_t)r, T.D4, cidx, key);
      }
    }
  };
  owner_walk(a, s_pre, total, prefetch_next, apply);
  // ---- completion: publish applied[me] = step to every rank (one fence per CTA, see push)
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    s_last = (atomicAdd(&ctl->apply_done, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence_system();
  const uint32_t step = ctl->step + 1;
  if (a.fixed_cnt < 0 && threadIdx.x < g.W)
    st_release_sys(a.hdrs[threadIdx.x] + PX_MAX_RANKS + a.rank, step);
  __syncthreads();
  if (threadIdx.x == 0) {
    ctl->step = step; ctl->apply_done = 0; ctl->bar = 0;
    ctl->t_own[2] = px_globaltimer();
  }
}

// ---------------------------------------------------------------------------
// Dynamic shared memory of a push launch whose id table has 1 << hbits slots (SMEM layout above)
static constexpr int kPushHbitsMax = 13;
static size_t push_smem_bytes(int hbits) {
  return ((size_t)4 * sizeof(int32_t) << hbits) + 2 * PX_ID_CHUNK * sizeof(int32_t);
}

// The push instantiations, [async][bf16 gradients][async: optimizer family, sync: bf16 wire];
// fp32 gradients never travel narrowed, so that entry is null.
static const void* const kPushKernels[2][2][2] = {
    {{(const void*)px_sparse_push_kernel<float, float, false, 0>, nullptr},
     {(const void*)px_sparse_push_kernel<__nv_bfloat16, float, false, 0>,
      (const void*)px_sparse_push_kernel<__nv_bfloat16, __nv_bfloat16, false, 0>}},
    {{(const void*)px_sparse_push_kernel<float, float, true, 0>,
      (const void*)px_sparse_push_kernel<float, float, true, 1>},
     {(const void*)px_sparse_push_kernel<__nv_bfloat16, float, true, 0>,
      (const void*)px_sparse_push_kernel<__nv_bfloat16, float, true, 1>}}};

// The owner instantiations, [bf16 master][bf16 wire][optimizer family]
#define PX_OWNER_FAMS(WireT, MT)                                                          \
  {(const void*)px_sparse_owner_kernel<WireT, 0, MT>,                                     \
   (const void*)px_sparse_owner_kernel<WireT, 1, MT>,                                     \
   (const void*)px_sparse_owner_kernel<WireT, 2, MT>}
static const void* const kOwnerKernels[2][2][3] = {
    {PX_OWNER_FAMS(float, float), PX_OWNER_FAMS(__nv_bfloat16, float)},
    {PX_OWNER_FAMS(float, __nv_bfloat16), PX_OWNER_FAMS(__nv_bfloat16, __nv_bfloat16)}};
#undef PX_OWNER_FAMS

// The most CTAs of 256 threads of `fn` the device keeps resident at once: the largest grid a
// cooperative launch of `fn` may have.  Cached per kernel.
static int coop_max_blocks(const void* fn) {
  static std::mutex mu;
  static std::unordered_map<const void*, int> cache;
  std::lock_guard<std::mutex> lock(mu);
  int& n = cache[fn];
  if (n == 0) {
    int per_sm = 0, dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, 256, 0);
    n = std::max(per_sm * sms, 1);
  }
  return n;
}

// Launches the owner-side kernel `fn` with parameters `args`, after a one-warp kernel that waits
// for every source's `pushed` flag when the entry counts come from those flags.  With merge, `fn`
// has a grid barrier inside: a cooperative launch of at most PX_NUM_SMS * 4 CTAs, of at most as
// many as `fn` keeps resident, and of at most `coop_cap`.
static int launch_owner_side(const void* fn, void** args, const OwnerArgs& a, const GroupGeom& G,
                             SparseCtl* ctl, int blocks, int coop_cap, cudaStream_t stream) {
  if (a.fixed_cnt < 0 && G.W > 1) px_sparse_wait_kernel<<<1, 32, 0, stream>>>(a.hdr, ctl, G.W);
  blocks = std::max(blocks, 1);
  cudaError_t e;
  if (a.use_merge) {
    blocks = std::min({blocks, PX_NUM_SMS * 4, coop_max_blocks(fn), coop_cap});
    e = cudaLaunchCooperativeKernel(fn, dim3(blocks), dim3(256), args, 0, stream);
  } else {
    e = cudaLaunchKernel(fn, dim3(blocks), dim3(256), args, 0, stream);
  }
  if (e != cudaSuccess) return (int)e;
  return (int)cudaGetLastError();
}

extern "C" {

// The group constants and the layout of the descriptors Python fills through ctypes, as
// `name=value` pairs: `Struct=sizeof(Struct)`, `Struct.field=offsetof(Struct, field)`.
// `ops.lib()` checks its ctypes mirrors against it, so a field changed on one side only fails
// at load.
const char* px_sparse_abi() {
  static const std::string abi = [] {
    std::string s;
    auto put = [&s](const char* k, size_t v) { s += std::string(k) + '=' + std::to_string(v) + ' '; };
#define SIZE(S) put(#S, sizeof(S))
#define FIELD(S, f) put(#S "." #f, offsetof(S, f))
    put("ctl_bytes", sizeof(SparseCtl)); put("hdr_words", PX_GRP_HDR_WORDS);
    put("group_max", PX_GRP_MAX);
    // SparseCtl byte offsets of the u64 device timestamps (t_push, t_own, t_dbg) and of `overflow`
    put("ctl_time_offset", offsetof(SparseCtl, t_push));
    put("ctl_overflow_offset", offsetof(SparseCtl, overflow));
    SIZE(GroupGeom); FIELD(GroupGeom, V); FIELD(GroupGeom, P); FIELD(GroupGeom, W);
    FIELD(GroupGeom, rows_per_part); FIELD(GroupGeom, strategy); FIELD(GroupGeom, replicated);
    FIELD(GroupGeom, extras); FIELD(GroupGeom, base); FIELD(GroupGeom, part_owner);
    FIELD(GroupGeom, part_slot);
    SIZE(LookupTable); FIELD(LookupTable, srcs); FIELD(LookupTable, out); FIELD(LookupTable, D4);
    FIELD(LookupTable, src_bf16); FIELD(LookupTable, out_bf16);
    SIZE(PushTable); FIELD(PushTable, grads); FIELD(PushTable, staging); FIELD(PushTable, rings);
    FIELD(PushTable, tables); FIELD(PushTable, slot0s); FIELD(PushTable, slot1s);
    FIELD(PushTable, slot2s); FIELD(PushTable, shadows); FIELD(PushTable, hp);
    FIELD(PushTable, D4); FIELD(PushTable, kind); FIELD(PushTable, scale);
    SIZE(OwnerTable); FIELD(OwnerTable, ring); FIELD(OwnerTable, table); FIELD(OwnerTable, slot0);
    FIELD(OwnerTable, slot1); FIELD(OwnerTable, slot2); FIELD(OwnerTable, shadow);
    FIELD(OwnerTable, hp); FIELD(OwnerTable, D4); FIELD(OwnerTable, kind); FIELD(OwnerTable, avg);
    FIELD(OwnerTable, D); FIELD(OwnerTable, slot_part); FIELD(OwnerTable, seed);
    FIELD(OwnerTable, w_bf16);
#undef SIZE
#undef FIELD
    return s;
  }();
  return abi.c_str();
}

static inline int pick_lpr(int D4) { int l = 1; while (l < D4 && l < 32) l <<= 1; return l; }

// ids_is64: 1 = int64 ids, 0 = int32.
int px_sparse_lookup(const void* ids, int ids_is64, int n, const LookupTable* tabs, int nt,
                     int32_t* pend_ids, const GroupGeom* g, const void* hdr_mine,
                     const void* ctl, int wait, cudaStream_t stream) {
  if (n <= 0) return 0;
  if (nt < 1 || nt > PX_GRP_MAX) return -4;
  const GroupGeom G = *g;
  LookupArgs a{};
  a.nt = nt;
  int maxv = 1;
  for (int t = 0; t < nt; ++t) {
    a.t[t] = tabs[t];
    const int v = tabs[t].src_bf16 ? (tabs[t].D4 + 1) / 2 : tabs[t].D4;
    if (v > maxv) maxv = v;
  }
  const int lpr = pick_lpr(maxv);
  const int threads = 256, rpb = threads / lpr;
  int blocks = (n + rpb - 1) / rpb;
  if (blocks > PX_NUM_SMS * 8) blocks = PX_NUM_SMS * 8;
  const uint32_t* applied = reinterpret_cast<const uint32_t*>(hdr_mine) + PX_MAX_RANKS;
  if (ids_is64)
    px_sparse_lookup_kernel<long long><<<blocks, threads, 0, stream>>>(
        (const long long*)ids, n, a, pend_ids, G, applied, (const SparseCtl*)ctl, lpr, wait);
  else
    px_sparse_lookup_kernel<int><<<blocks, threads, 0, stream>>>(
        (const int*)ids, n, a, pend_ids, G, applied, (const SparseCtl*)ctl, lpr, wait);
  return (int)cudaGetLastError();
}

static inline int push_hbits(int n, int blocks) {
  // >= 4x the expected ids per CTA, 1024..8192 slots (16 B of SMEM per slot)
  long long want = 4LL * ((n + blocks - 1) / blocks);
  int hb = 10;
  while ((1LL << hb) < want && hb < kPushHbitsMax) ++hb;
  return hb;
}

// grad_dtype / wire_dtype: 0 fp32, 1 bf16.  async: 1 = remote optimizer application (Hogwild).
// All member tables of a group use the same optimizer kind family.
// The kinds the sparse kernels implement: the elementwise families 0 and 1 and the row-wise
// family 2.  Any other kind (the dense-only layer-wise rules among them) is refused, never
// applied as nothing or as another family's rule.
static bool px_sparse_kind(int kind) { return kind >= PX_SGD && kind <= PX_ROWWISE_ADAGRAD; }

int px_sparse_push(const int32_t* pend_ids, int n, const PushTable* tabs, int nt,
                   int grad_dtype, int wire_dtype, int async, void* ring_ids_dev, void* hdrs_dev,
                   int cap, const GroupGeom* g, void* ctl, int rank, int dedup, int max_blocks,
                   cudaStream_t stream) {
  if (nt < 1 || nt > PX_GRP_MAX) return -4;
  GroupGeom G = *g;
  PushArgs a{};
  a.nt = nt; a.ring_ids = (int32_t* const*)ring_ids_dev; a.hdrs = (uint32_t* const*)hdrs_dev;
  a.cap = cap; a.rank = rank;
  const int fam = PX_KIND_FAMILY(tabs[0].kind);
  for (int t = 0; t < nt; ++t) {
    if (!px_sparse_kind(tabs[t].kind)) return -9;
    if (PX_KIND_FAMILY(tabs[t].kind) != fam) return -6;
    a.t[t] = tabs[t];
  }
  int blocks = (n + 15) / 16;
  if (blocks > max_blocks) blocks = max_blocks;
  if (blocks < 1) blocks = 1;
  int hbits = push_hbits(n, blocks);
  if (async && fam == 2) return -7;             // row-wise rules need the merged row
  const void* fn = kPushKernels[async != 0][grad_dtype != 0][async ? fam : wire_dtype != 0];
  if (fn == nullptr) return -5;                 // never narrow fp32 gradients
  static std::once_flag attr;
  std::call_once(attr, [] {
    for (const auto& by_mode : kPushKernels)
      for (const auto& by_grad : by_mode)
        for (const void* k : by_grad)
          if (k) cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)push_smem_bytes(kPushHbitsMax));
  });
  SparseCtl* C = (SparseCtl*)ctl;
  void* args[] = {&pend_ids, &n, &a, &G, &C, &hbits, &dedup};
  cudaLaunchKernel(fn, dim3(blocks), dim3(256), args, push_smem_bytes(hbits), stream);
  return (int)cudaGetLastError();
}

int px_sparse_owner(const OwnerTable* tabs, int nt, int wire_dtype, const int32_t* ring_ids,
                    void* hdr, void* hdrs_dev, int32_t* slotmap, int32_t* next, int cap,
                    const GroupGeom* g, void* ctl, int rank, int use_merge, int blocks,
                    int fixed_cnt, cudaStream_t stream) {
  if (nt < 1 || nt > PX_GRP_MAX) return -4;
  GroupGeom G = *g;
  OwnerArgs a{};
  a.fixed_cnt = fixed_cnt;
  a.nt = nt; a.ring_ids = ring_ids; a.hdr = (uint32_t*)hdr; a.hdrs = (uint32_t* const*)hdrs_dev;
  a.slotmap = slotmap; a.next = next; a.cap = cap; a.rank = rank; a.use_merge = use_merge;
  const int fam = PX_KIND_FAMILY(tabs[0].kind);
  const int w_bf16 = tabs[0].w_bf16 != 0;
  for (int t = 0; t < nt; ++t) {
    if (!px_sparse_kind(tabs[t].kind)) return -9;
    if (PX_KIND_FAMILY(tabs[t].kind) != fam) return -6;
    if ((tabs[t].w_bf16 != 0) != w_bf16) return -8;   // members share one master type
    a.t[t] = tabs[t];
  }
  SparseCtl* C = (SparseCtl*)ctl;
  const void* fn = kOwnerKernels[w_bf16][wire_dtype != 0][fam];
  void* args[] = {&a, &G, &C};
  // Merge grids are also held to the residency of px_sparse_owner_kernel<float, 1> (3 CTAs per
  // SM on the H100): a tuning cap, under which the benchmark numbers were taken.
  return launch_owner_side(fn, args, a, G, C, blocks,
                           coop_max_blocks((const void*)px_sparse_owner_kernel<float, 1>), stream);
}

}  // extern "C"

// ------------------------------------------------------- joint global-norm clip
// ClipByGlobalNorm(include_sparse=True): the norm covers this group's aggregated rows, so
// it is taken on the owner, from the rings, before the (unchanged) owner kernel applies
// them.  The clip factor then reaches the owner kernel through the slot it already
// multiplies by, hp[HP_GSCALE], in a private copy of the group's hyper-parameters.

// Σ over the touched rows of ‖avg · hp[HP_GSCALE] · Σ_entries row‖², i.e. exactly the rows
// px_sparse_owner_kernel would hand to the optimizer, added to *sumsq.  Links and walks the
// entries with the owner kernel's helpers (one grid barrier, cooperative launch), resets the
// slotmap entries it linked and returns ctl->bar / ctl->apply_done to 0; publishes no flag
// and leaves ctl->step alone, so the owner kernel runs next exactly as it would have.
template <typename WireT>
__global__ void __launch_bounds__(256)
px_sparse_owner_norm_kernel(OwnerArgs a, GroupGeom g, SparseCtl* ctl, float* sumsq) {
  __shared__ int s_pre[PX_MAX_RANKS + 1];
  __shared__ double s_part[8];
  const int total = owner_prefix(a, g, s_pre);
  if (a.use_merge) owner_link(a, s_pre, total, ctl, false);
  // fp64 partial sums of 4-element groups
  const int lane = threadIdx.x & 15;
  double acc = 0.0;
  owner_walk(a, s_pre, total, [](int, int) {}, [&](int e, int r) {
#pragma unroll 1
    for (int t = 0; t < a.nt; ++t) {
      const OwnerTable& T = a.t[t];
      const size_t row_bytes = (size_t)T.D4 * 4 * sizeof(WireT);
      const float gmul = T.avg * T.hp[HP_GSCALE];
      for (int cidx = lane; cidx < T.D4; cidx += 16) {
        float4 gv = ld_merged4<WireT>(a, T, row_bytes, e, cidx);
        gv.x *= gmul; gv.y *= gmul; gv.z *= gmul; gv.w *= gmul;
        acc += (double)gv.x * gv.x + (double)gv.y * gv.y + (double)gv.z * gv.z +
               (double)gv.w * gv.w;
      }
    }
  });
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double b = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) b += s_part[w];
    if (b != 0.0) atomicAdd(sumsq, (float)b);
    // every CTA has left the grid barrier once it takes a ticket: the last one resets it
    if (atomicAdd(&ctl->apply_done, 1u) == gridDim.x - 1) { ctl->bar = 0; ctl->apply_done = 0; }
  }
}

// out = hp with out[HP_GSCALE] = hp[HP_GSCALE] · *scale: the hyper-parameters one group
// applies with this step (the shared vector stays untouched for every other reader).
__global__ void px_clip_hp_kernel(const float* hp, const float* scale, float* out) {
  if (threadIdx.x <= HP_FLAGS)
    out[threadIdx.x] = threadIdx.x == HP_GSCALE ? hp[threadIdx.x] * *scale : hp[threadIdx.x];
}

extern "C" {

// `sumsq` += the squared norm of what px_sparse_owner would apply this step (see the kernel).
// Launched after the group's push and before its px_sparse_owner, with the same ring / slotmap
// arguments; waits for every source's `pushed` flag first.
int px_sparse_owner_norm(const OwnerTable* tabs, int nt, int wire_dtype, const int32_t* ring_ids,
                         void* hdr, int32_t* slotmap, int32_t* next, int cap, const GroupGeom* g,
                         void* ctl, int use_merge, int blocks, float* sumsq,
                         cudaStream_t stream) {
  if (nt < 1 || nt > PX_GRP_MAX) return -4;
  GroupGeom G = *g;
  OwnerArgs a{};
  a.fixed_cnt = -1;
  a.nt = nt; a.ring_ids = ring_ids; a.hdr = (uint32_t*)hdr; a.hdrs = nullptr;
  a.slotmap = slotmap; a.next = next; a.cap = cap; a.rank = 0; a.use_merge = use_merge;
  for (int t = 0; t < nt; ++t) a.t[t] = tabs[t];
  const void* fn = wire_dtype == 0 ? (const void*)px_sparse_owner_norm_kernel<float>
                                   : (const void*)px_sparse_owner_norm_kernel<__nv_bfloat16>;
  SparseCtl* C = (SparseCtl*)ctl;
  void* args[] = {&a, &G, &C, &sumsq};
  return launch_owner_side(fn, args, a, G, C, blocks, INT_MAX, stream);
}

int px_clip_hp(const float* hp, const float* scale, float* out, cudaStream_t stream) {
  px_clip_hp_kernel<<<1, 32, 0, stream>>>(hp, scale, out);
  return (int)cudaGetLastError();
}

}  // extern "C"
