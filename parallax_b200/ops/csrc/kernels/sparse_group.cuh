// Geometry and control block of a sparse co-lookup group, shared by the kernels that read
// a group's tables (sparse.cu: lookup / push / owner; softmax_eval.cu: full-softmax eval).
// Python fills GroupGeom through the ctypes class of the same name (`ops.GroupGeom`);
// `px_sparse_abi` in sparse.cu publishes its layout so that `ops.lib()` can check the two agree.
#pragma once
#include "common.cuh"

#define PX_GRP_MAX 4            // member tables per group

struct GroupGeom {
  int V, P, W, rows_per_part;
  int strategy;                 // 0 mod, 1 div
  int replicated;               // 1: every rank holds the full table (AR mode)
  int extras, base;             // div strategy
  const int* part_owner;        // [P] owner rank of partition p (byte-greedy placement)
  const int* part_slot;         // [P] index of partition p among its owner's partitions
};

// the global id of row idx of partition p: the inverse of the (partition, index) split of an id
// (`geom_part` in sparse.cu); a replicated layout is one "mod" partition, so this is the identity
__device__ __forceinline__ int geom_gid(const GroupGeom& g, int p, int idx) {
  if (g.strategy == 0) return idx * g.P + p;
  return p < g.extras ? p * (g.base + 1) + idx : p * g.base + g.extras + idx;
}

// 32-bit integer hash (xor-shift, multiply, twice); `optim.sr_mix` is the same hash in torch.
// It keys the stochastic rounding of bf16 masters (sparse.cu) and the sampling noise below.
__device__ __forceinline__ uint32_t sr_mix(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu;
  return x ^ (x >> 16);
}

// Sampling noise (full-softmax sampling in softmax_eval.cu; `engine.sample_uniform` and
// `engine.sample_log_e` are the same in torch).  Row `row` of a call draws with the keys
// s − log E of its global ids, E = −log1p(−v) ~ Exp(1) (so −log E is Gumbel), where
//   v = min(h · 2^-32 + 2^-33, 1 − 2^-24),  h = sr_mix(sample_row_key(seed, row) ^ gid).
// h and v are bit-identical in torch; E keeps fp32 relative precision down to 1.2e-10, where
// the winner is decided, and the clamp keeps every key finite.
__device__ __forceinline__ uint32_t sample_row_key(uint32_t seed, uint32_t row) {
  return sr_mix(sr_mix(seed) ^ row);
}
__device__ __forceinline__ float sample_log_e(uint32_t row_key, uint32_t gid) {
  const float v = fminf(__fadd_rn(__fmul_rn(__uint2float_rn(sr_mix(row_key ^ gid)), 0x1p-32f),
                                  0x1p-33f), 0x1.fffffep-1f);
  return logf(-log1pf(-v));
}

// per-rank control block of a group (local memory)
struct SparseCtl {
  uint32_t step;                // completed steps
  uint32_t push_done;           // CTA ticket counter (push kernel)
  uint32_t apply_done;          // CTA ticket counter (owner kernel)
  uint32_t bar;                 // grid barrier arrivals (owner kernel)
  int32_t n_dup;                // staging rows handed out this step
  int32_t overflow;             // #positions that fell back to un-deduplicated entries (stat)
  int32_t owner_cnt[PX_MAX_RANKS];
  unsigned long long t_push[2]; // %globaltimer at push start / flag publication
  unsigned long long t_own[3];  // owner kernel: start / all sources arrived / applied published
  unsigned long long t_dbg[8];  // push kernel, CTA 0: end of each internal phase (profiling aid)
};

// group header (symmetric): [pushed[R] | applied[R] | cnt[R]]
#define PX_GRP_HDR_WORDS (3 * PX_MAX_RANKS)
