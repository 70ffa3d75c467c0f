// Fused dense step: reduce-scatter (pull) → fp32 optimizer on the owned slice
// → all-gather of the *updated parameters* (push), in ONE kernel.
//
// What it replaces in the reference:
//   AR / HYBRID dense : ncclAllReduce on the fusion buffer + `tf.div` +
//     one Apply<Optimizer> Eigen kernel per variable on every replica
//     (horovod/common/ops/nccl_operations.cc:60-109,
//      horovod/tensorflow/__init__.py:76-81,
//      tensorflow/core/kernels/training_ops_gpu.cu.cc:28-283)
//   PS dense (sync)   : ConditionalAccumulator.take_grad(num_workers) on the PS
//     CPU, chief applies, token queues, mirror-variable refresh
//     (graph_transform_lib.py:330-582, :584-704)
// Both are the same data movement on an NVSwitch box: the rank that owns
// slice r is that slice's "parameter server".  Owning the slice also means
// only 1/W of the fp32 master weights and optimizer slots live on each GPU.
//
// MODE 0 FUSED        : barrier, reduce, update, push params, barrier
// MODE 1 REDUCE_ONLY  : barrier, reduce → fp32 scratch + Σg² (for global-norm
//                       clipping the norm must be known before any update)
// MODE 2 UPDATE_PUSH  : scratch·clip → update, push params, barrier
// MODE 3 ACCUMULATE   : barrier, reduce → fp32 scratch (= or +=), barrier; no update.  One
//                       micro-batch of a step that accumulates several: the end barrier is
//                       there because peers pull from this rank's gradient bucket, which the
//                       next micro-batch's backward overwrites.
// "Accumulator in" (PX_DS_ACC_IN, modes 0, 1 and 3): the fp32 scratch holds the scaled sum of
// the step's earlier micro-batches and is added to this reduction before anything else, so
// the last micro-batch of a step runs mode 0 or 1 with the flag and mode 2 is unchanged.
// World 1 degenerates to a fused multi-tensor optimizer (also used as the
// local update after a plain all-reduce in "replicated" AR mode).
#include "common.cuh"
#include "launch.h"
#include "optim_rules.cuh"

struct DenseStepArgs {
  PeerPtrs grads;    // rotated, element type T
  PeerPtrs params;   // rotated, element type T
  float* master;     // [slice] fp32 master weights of the owned slice
  float* slot0;      // [slice] or null
  float* slot1;      // [slice] or null
  float* slot2;      // [slice] or null (centered RMSProp)
  float* ema;        // [slice] or null
  float* red;        // [slice] fp32 scratch (modes 1/2/3, accumulator in) or null
  const float* hp;   // device hyper-parameters (8 floats)
  const float* clip; // device scalar multiplier or null
  float* sumsq;      // device scalar accumulator or null
  size_t n;          // bucket elements, multiple of W * VN
  float avg;         // 1/num_workers (or 1)
  float ema_decay;
  int rank, ch_start, ch_end, kind, mode;   // mode | PX_DS_ACC_IN in the ACC kernels
  int use_mc;        // 1: grads.p[0] / params.p[0] are NVSwitch multicast addresses
};

constexpr int PX_DS_ACC_IN = 4;

// NVLS: the switch reduces (fp32 accumulate) / broadcasts; see collectives.cu
template <typename T>
__device__ __forceinline__ uint4 ds_mm_ld_reduce(const T* p) {
  uint4 r;
  if (sizeof(T) == 2)
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
  else
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
  return r;
}
__device__ __forceinline__ void ds_mm_st(void* p, const uint4& r) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};"
               ::"l"(p), "r"(r.x), "r"(r.y), "r"(r.z), "r"(r.w) : "memory");
}

template <int VN>
__device__ __forceinline__ void ld_f32(const float* p, float* f) {
#pragma unroll
  for (int i = 0; i < VN / 4; ++i) {
    const uint4 v = ld_v4(p + 4 * i);
    f[4 * i] = __uint_as_float(v.x); f[4 * i + 1] = __uint_as_float(v.y);
    f[4 * i + 2] = __uint_as_float(v.z); f[4 * i + 3] = __uint_as_float(v.w);
  }
}
template <int VN>
__device__ __forceinline__ void st_f32(float* p, const float* f) {
#pragma unroll
  for (int i = 0; i < VN / 4; ++i)
    st_v4(p + 4 * i, make_uint4(__float_as_uint(f[4 * i]), __float_as_uint(f[4 * i + 1]),
                                __float_as_uint(f[4 * i + 2]), __float_as_uint(f[4 * i + 3])));
}

// Rank-level (not CTA-paired) synchronisation, so the grid is not limited to the
// PX_MAX_BLOCKS barrier slots of `px_block_barrier` and the optimizer phase can use the whole
// GPU's HBM bandwidth:
//  * start: CTA 0 announces "this rank reached the kernel" (all earlier work on the stream —
//    the gradients — is complete) in slot 0 of `ch_start`; EVERY CTA waits until every peer has.
//  * end: the last CTA to finish (ticket) fences, announces "all my parameter stores are out"
//    in slot 0 of `ch_end` and waits for the same from every peer; the kernel — and with it the
//    stream — completes only then.  Slot 1 of `ch_end` holds the ticket counter.
__device__ __forceinline__ void px_rank_signal(uint32_t* const* pads, int slot, int rank, int world,
                                               uint32_t e) {
  if (threadIdx.x < world)
    st_release_sys(pads[threadIdx.x] + (size_t)slot * PX_MAX_RANKS + rank, e);
}
__device__ __forceinline__ void px_rank_wait(uint32_t* const* pads, int slot, int rank, int world,
                                             uint32_t e) {
  if (threadIdx.x < world) {
    const uint32_t* mine = pads[rank] + (size_t)slot * PX_MAX_RANKS + threadIdx.x;
    while ((int32_t)(ld_acquire_sys(mine) - e) < 0) { }
  }
  __syncthreads();
}

// ACC: the instantiation that runs mode 3 and the accumulator-in flag.  A step of one
// micro-batch launches only ACC = false, whose code is that of a kernel without either.  The
// ACC kernels keep one CTA per SM: the accumulator's 8 extra loads in flight spill at the
// 64 registers of two.
template <typename T, int W, int FAM, bool ACC>
__global__ void __launch_bounds__(512, (W == 1 && FAM == 0 && !ACC) ? 2 : 1)
px_dense_step_kernel(DenseStepArgs a, uint32_t* const* pads, uint32_t* epoch_ctr) {
  constexpr int VN = Vec16<T>::N;
  const int mode = ACC ? (a.mode & 3) : a.mode, kind = a.kind;
  const bool acc_in = ACC && (a.mode & PX_DS_ACC_IN);
  const int slot_s = a.ch_start * PX_MAX_BLOCKS, slot_e = a.ch_end * PX_MAX_BLOCKS;
  // profiling aid: %globaltimer stamps of the last launch in the (otherwise unused) epoch slots
  // of the last channel: [0] CTA 0 start, [1] CTA 0 past the start wait, [2] CTA 0 loop done,
  // [3] last CTA fenced, [4] last CTA past the end wait
  unsigned long long* dbg = reinterpret_cast<unsigned long long*>(
      epoch_ctr + (PX_NUM_CHANNELS - 1) * PX_MAX_BLOCKS);
  const bool stamp0 = blockIdx.x == 0 && threadIdx.x == 0;
  if (stamp0) dbg[0] = px_globaltimer();
  uint32_t e_start = 0;
  if (W > 1 && mode != 2) {
    e_start = ld_volatile_u32(epoch_ctr + slot_s) + 1;
    if (blockIdx.x == 0) px_rank_signal(pads, slot_s, a.rank, W, e_start);
    px_rank_wait(pads, slot_s, a.rank, W, e_start);
  }
  if (stamp0) dbg[1] = px_globaltimer();
  const size_t slice = a.n / W;
  const size_t nvec = slice / VN;
  const size_t base = (size_t)a.rank * slice;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const PxHP h = px_load_hp(a.hp);
  float gmul = a.avg * a.hp[HP_GSCALE];
  if (mode == 2) gmul = 1.f;                       // already applied in REDUCE
  if (mode != 1 && a.clip != nullptr) gmul *= *a.clip;
  float ss = 0.f;
  for (size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += stride) {
    const size_t e = v * VN;                        // element offset inside the slice
    // ---- issue EVERY load of this vector before touching any loaded value: the helpers are
    // volatile asm (program order), so a dependent FADD between the peer loads and the
    // master/slot loads would serialise two memory latencies (one of them an NVLink round
    // trip) per vector
    float g[VN];
    uint4 in[W];
    uint4 mcv = make_uint4(0, 0, 0, 0);
    if (mode == 2) {
      ld_f32<VN>(a.red + e, g);
    } else if (a.use_mc) {
      // one switch-side reduction instead of W peer loads
      mcv = ds_mm_ld_reduce<T>(reinterpret_cast<const T*>(a.grads.p[0]) + base + e);
    } else {
#pragma unroll
      for (int p = 0; p < W; ++p)
        in[p] = ld_v4_stream(reinterpret_cast<const T*>(a.grads.p[p]) + base + e);
    }
    float r[ACC ? VN : 1];
    if (acc_in) ld_f32<VN>(a.red + e, r);
    float w[VN], s0[VN], s1[VN], s2[FAM == 1 ? VN : 1], m[VN];
    if (mode != 1 && !(ACC && mode == 3)) {
      ld_f32<VN>(a.master + e, w);
      if (a.slot0) ld_f32<VN>(a.slot0 + e, s0);
      if (a.slot1) ld_f32<VN>(a.slot1 + e, s1);
      if (FAM == 1 && a.slot2) ld_f32<VN>(a.slot2 + e, s2);
      if (a.ema) ld_f32<VN>(a.ema + e, m);
    }
    // ---- math
    if (mode != 2) {
      if (a.use_mc) {
        Vec16<T>::unpack(mcv, g);
      } else {
#pragma unroll
        for (int i = 0; i < VN; ++i) g[i] = 0.f;
#pragma unroll
        for (int p = 0; p < W; ++p) {
          float f[VN];
          Vec16<T>::unpack(in[p], f);
#pragma unroll
          for (int i = 0; i < VN; ++i) g[i] += f[i];
        }
      }
    }
#pragma unroll
    for (int i = 0; i < VN; ++i) g[i] *= gmul;
    if (acc_in) {
#pragma unroll
      for (int i = 0; i < VN; ++i) g[i] += r[ACC ? i : 0];
    }
    if (ACC && mode == 3) {
      st_f32<VN>(a.red + e, g);
      continue;
    }
    if (mode == 1) {
#pragma unroll
      for (int i = 0; i < VN; ++i) ss += g[i] * g[i];
      st_f32<VN>(a.red + e, g);
      continue;
    }
#pragma unroll
    for (int i = 0; i < VN; ++i) {
      const float gi = h.wd != 0.f ? fmaf(h.wd, w[i], g[i]) : g[i];
      px_rule<FAM>(kind, h, gi, w[i], s0[i], s1[i], s2[FAM == 1 ? i : 0]);
    }
    st_f32<VN>(a.master + e, w);
    if (a.slot0) st_f32<VN>(a.slot0 + e, s0);
    if (a.slot1) st_f32<VN>(a.slot1 + e, s1);
    if (FAM == 1 && a.slot2) st_f32<VN>(a.slot2 + e, s2);
    if (a.ema) {
#pragma unroll
      for (int i = 0; i < VN; ++i) m[i] -= (1.f - a.ema_decay) * (m[i] - w[i]);
      st_f32<VN>(a.ema + e, m);
    }
    const uint4 out = Vec16<T>::pack(w);
    if (a.use_mc) {
      ds_mm_st(reinterpret_cast<T*>(a.params.p[0]) + base + e, out);   // switch broadcast
    } else {
#pragma unroll
      for (int p = 0; p < W; ++p)
        st_v4_stream(reinterpret_cast<T*>(a.params.p[p]) + base + e, out);
    }
  }
  if (mode == 1 && a.sumsq != nullptr) block_atomic_sum(ss, a.sumsq);
  if (stamp0) dbg[2] = px_globaltimer();
  if (W > 1) {
    __shared__ bool s_last;
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence_system();          // one fence per CTA (cumulative over the barrier)
      s_last = atomicAdd(epoch_ctr + slot_e + 1, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (s_last) {
      if (threadIdx.x == 0) dbg[3] = px_globaltimer();
      if (mode != 1) {
        const uint32_t e_end = ld_volatile_u32(epoch_ctr + slot_e) + 1;
        px_rank_signal(pads, slot_e, a.rank, W, e_end);
        px_rank_wait(pads, slot_e, a.rank, W, e_end);
        if (threadIdx.x == 0) epoch_ctr[slot_e] = e_end;
      }
      if (threadIdx.x == 0) dbg[4] = px_globaltimer();
      if (threadIdx.x == 0) {
        if (mode != 2) epoch_ctr[slot_s] = e_start;
        epoch_ctr[slot_e + 1] = 0;
      }
    }
  }
}

// device timestamp (ns) — a graph-capturable probe for "exposed communication" measurements
__global__ void px_stamp_kernel(unsigned long long* slot) { *slot = px_globaltimer(); }

// scale = max_norm / max(sqrt(total), max_norm)  (tf.clip_by_global_norm);
// also exports the norm and zeroes the accumulator for the next step.
__global__ void px_clip_scale_kernel(const float* sumsq, float max_norm, float* scale_out,
                                     float* norm_out, float* zero_after) {
  const float norm = sqrtf(*sumsq);
  *scale_out = max_norm / fmaxf(norm, max_norm);
  if (norm_out) *norm_out = norm;
  if (zero_after) *zero_after = 0.f;
}

// Asynchronous PS dense apply (Hogwild): this rank's gradient is applied,
// un-averaged, straight onto every owner's master slice over NVLink, and the
// refreshed values are pulled back into the local parameter mirror.
// Reference: sync=False ⇒ no accumulators, update ops race on the PS
// variables (ps/between_graph_parallel.py:137-146).
template <typename T, int W, int FAM>
__global__ void __launch_bounds__(512)
px_dense_async_kernel(const T* __restrict__ my_grads, T* __restrict__ my_params,
                      PeerPtrs master, PeerPtrs slot0, PeerPtrs slot1, PeerPtrs slot2,
                      const float* hp,
                      const float* clip, size_t n, int kind, int rank) {
  constexpr int VN = Vec16<T>::N;
  const size_t slice = n / W;
  const size_t nvec = n / VN;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const PxHP h = px_load_hp(hp);
  float gmul = hp[HP_GSCALE];
  if (clip != nullptr) gmul *= *clip;
  for (size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += stride) {
    const size_t e = v * VN;
    const int owner = (int)(e / slice);
    const size_t le = e - (size_t)owner * slice;
    float *pm = nullptr, *p0 = nullptr, *p1 = nullptr, *p2 = nullptr;
#pragma unroll
    for (int p = 0; p < W; ++p)     // master/slots arrive in NATURAL rank order
      if (p == owner) {
        pm = reinterpret_cast<float*>(master.p[p]) + le;
        p0 = slot0.p[p] ? reinterpret_cast<float*>(slot0.p[p]) + le : nullptr;
        p1 = slot1.p[p] ? reinterpret_cast<float*>(slot1.p[p]) + le : nullptr;
        p2 = (FAM == 1 && slot2.p[p]) ? reinterpret_cast<float*>(slot2.p[p]) + le : nullptr;
      }
    float g[VN], w[VN], s0[VN], s1[VN], s2[FAM == 1 ? VN : 1];
    Vec16<T>::unpack(ld_v4(my_grads + e), g);
    ld_f32<VN>(pm, w);
    if (p0) ld_f32<VN>(p0, s0);
    if (p1) ld_f32<VN>(p1, s1);
    if (FAM == 1 && p2) ld_f32<VN>(p2, s2);
#pragma unroll
    for (int i = 0; i < VN; ++i) {
      float gi = g[i] * gmul;
      if (h.wd != 0.f) gi = fmaf(h.wd, w[i], gi);
      px_rule<FAM>(kind, h, gi, w[i], s0[i], s1[i], s2[FAM == 1 ? i : 0]);
    }
    st_f32<VN>(pm, w);
    if (p0) st_f32<VN>(p0, s0);
    if (p1) st_f32<VN>(p1, s1);
    if (FAM == 1 && p2) st_f32<VN>(p2, s2);
    st_v4(my_params + e, Vec16<T>::pack(w));
  }
}

// Σx² of a local buffer (used for clipping in the async path)
template <typename T>
__global__ void __launch_bounds__(512)
px_sumsq_kernel(const T* __restrict__ x, size_t n, float mul, float* out) {
  constexpr int VN = Vec16<T>::N;
  const size_t nvec = n / VN;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  float ss = 0.f;
  for (size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += stride) {
    float f[VN];
    Vec16<T>::unpack(ld_v4(x + v * VN), f);
#pragma unroll
    for (int i = 0; i < VN; ++i) ss += f[i] * f[i] * mul * mul;
  }
  block_atomic_sum(ss, out);
}

// ---------------------------------------------------------------------------------------------
// Layer-wise rules (family 3: LARS, LAMB).  A bucket's step scales every tensor's update by a
// trust ratio of two norms over the WHOLE tensor, which may straddle several owners' slices:
//   MODE 1 (unchanged)  : reduce → `red` (+ Σg² under a clip rule)
//   px_lw_norm_kernel   : per chunk of this slice, Σw² and Σx² (x = g for LARS, r for LAMB)
//                         → partials[chunk]; no atomics
//   px_lw_combine_kernel: per segment (tensor), its chunks' partials in chunk order → sums
//   one-shot all-reduce : sums → total, bitwise identical on every rank (W > 1 only)
//   px_lw_update_kernel : trust ratio per segment, rule, EMA, push of the parameters, end barrier
// The chunk table is built once per bucket and rank on the host (nvlink_backend.py): a chunk
// lies inside one tensor, in units of the bucket's 16-byte vectors relative to the slice start;
// padding vectors belong to no chunk and are never touched.  `ne` counts the chunk's elements
// that belong to the tensor: the tail of a tensor's last vector is left out of its sums.
struct LwChunk { int v0, nv, seg, ne; };

struct LayerwiseArgs {
  const float* red;      // [slice] reduced gradient (1/W and micro-batch weights applied)
  float* master;         // [slice]
  float* slot0;          // LARS momentum / LAMB m
  float* slot1;          // LAMB v or null
  float* ema;            // [slice] or null
  const float* hp;       // device hyper-parameters (10 floats)
  const float* clip;     // device scalar multiplier or null
  const LwChunk* chunks; // [nchunks]
  const int* seg_flags;  // [nseg] PX_LW_* bits
  const int* seg_chunks; // [nseg, 2] first / end chunk of each segment in this slice
  float* partials;       // [nchunks, 2]
  float* sums;           // [nseg, 2] this rank's Σw², Σx² (zero outside the slice)
  const float* total;    // [nseg, 2] sums over every rank
  int nchunks, nseg, kind;
};

__device__ __forceinline__ float2 lw_block_sum2(float a, float b) {
  __shared__ float2 s_part[32];
  a = warp_sum(a); b = warp_sum(b);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) s_part[wid] = make_float2(a, b);
  __syncthreads();
  float2 t = make_float2(0.f, 0.f);
  if (wid == 0) {
    if (lane < (int)(blockDim.x + 31) / 32) t = s_part[lane];
    t.x = warp_sum(t.x); t.y = warp_sum(t.y);
  }
  __syncthreads();          // s_part is reused by the next chunk
  return t;
}

template <int VN>
__global__ void __launch_bounds__(512)
px_lw_norm_kernel(LayerwiseArgs a) {
  // the decay is read per chunk, next to its flag: held across the chunk loop (and the
  // sqrt / division slow-path calls inside it), ptxas spilled it at the fp32 width
  const float b1 = a.hp[HP_A], b2 = a.hp[HP_B], eps = a.hp[HP_EPS];
  const float bc1 = a.hp[HP_BC1], bc2 = a.hp[HP_BC2];
  const float gmul = a.clip != nullptr ? *a.clip : 1.f;
  for (int c = blockIdx.x; c < a.nchunks; c += gridDim.x) {
    const LwChunk ch = a.chunks[c];
    const float wd = (a.seg_flags[ch.seg] & PX_LW_DECAY) ? a.hp[HP_WD] : 0.f;
    float sw = 0.f, sx = 0.f;
    for (int v = threadIdx.x; v < ch.nv; v += blockDim.x) {
      const size_t e = (size_t)(ch.v0 + v) * VN;
      const int lim = ch.ne - v * VN;
      float g[VN], w[VN], s0[VN], s1[VN];
      ld_f32<VN>(a.red + e, g);
      ld_f32<VN>(a.master + e, w);
      if (a.kind == PX_LAMB) {
        ld_f32<VN>(a.slot0 + e, s0);
        ld_f32<VN>(a.slot1 + e, s1);
      }
#pragma unroll
      for (int i = 0; i < VN; ++i) {
        float x = g[i] * gmul;
        if (a.kind == PX_LAMB) x = px_lamb_r(b1, b2, eps, bc1, bc2, wd, x, w[i], s0[i], s1[i]);
        if (i < lim) {
          sw = fmaf(w[i], w[i], sw);
          sx = fmaf(x, x, sx);
        }
      }
    }
    const float2 t = lw_block_sum2(sw, sx);
    if (threadIdx.x == 0) { a.partials[2 * c] = t.x; a.partials[2 * c + 1] = t.y; }
  }
}

// one thread per segment: its chunks' partials in chunk order (fixed, so the sums — and with
// them the parameters — are reproducible run to run)
__global__ void __launch_bounds__(256)
px_lw_combine_kernel(LayerwiseArgs a) {
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < a.nseg; s += gridDim.x * blockDim.x) {
    double sw = 0.0, sx = 0.0;
    for (int c = a.seg_chunks[2 * s]; c < a.seg_chunks[2 * s + 1]; ++c) {
      sw += a.partials[2 * c];
      sx += a.partials[2 * c + 1];
    }
    a.sums[2 * s] = (float)sw;
    a.sums[2 * s + 1] = (float)sx;
  }
}

__device__ __forceinline__ float px_lw_trust(int kind, const PxHP& h, int flags, float sw,
                                             float sx) {
  const float wn = sqrtf(sw), xn = sqrtf(sx);
  if (!(flags & PX_LW_ADAPT) || !(wn > 0.f && xn > 0.f)) return 1.f;
  return kind == PX_LARS ? h.b * wn / (xn + h.wd * wn + h.eps) : wn / xn;
}

template <typename T, int W>
__global__ void __launch_bounds__(512)
px_lw_update_kernel(LayerwiseArgs a, PeerPtrs params, size_t n, float ema_decay, int rank,
                    int ch_end, int use_mc, uint32_t* const* pads, uint32_t* epoch_ctr) {
  constexpr int VN = Vec16<T>::N;
  const PxHP h = px_load_hp(a.hp);
  const float bc1 = a.hp[HP_BC1], bc2 = a.hp[HP_BC2];
  const float gmul = a.clip != nullptr ? *a.clip : 1.f;
  const size_t base = (size_t)rank * (n / W);
  for (int c = blockIdx.x; c < a.nchunks; c += gridDim.x) {
    const LwChunk ch = a.chunks[c];
    const int flags = a.seg_flags[ch.seg];
    const float lr_t = h.lr * px_lw_trust(a.kind, h, flags, a.total[2 * ch.seg],
                                          a.total[2 * ch.seg + 1]);
    const float wd = (flags & PX_LW_DECAY) ? h.wd : 0.f;
    for (int v = threadIdx.x; v < ch.nv; v += blockDim.x) {
      const size_t e = (size_t)(ch.v0 + v) * VN;
      float g[VN], w[VN], s0[VN], s1[VN], m[VN];
      ld_f32<VN>(a.red + e, g);
      ld_f32<VN>(a.master + e, w);
      ld_f32<VN>(a.slot0 + e, s0);
      if (a.kind == PX_LAMB) ld_f32<VN>(a.slot1 + e, s1);
      if (a.ema) ld_f32<VN>(a.ema + e, m);
#pragma unroll
      for (int i = 0; i < VN; ++i) {
        const float gi = g[i] * gmul;
        if (a.kind == PX_LARS) {
          s0[i] = fmaf(h.a, s0[i], gi);
          w[i] = fmaf(-lr_t, (flags & PX_LW_NESTEROV) ? fmaf(h.a, s0[i], gi) : s0[i], w[i]);
        } else {
          const float r = px_lamb_r(h.a, h.b, h.eps, bc1, bc2, wd, gi, w[i], s0[i], s1[i]);
          w[i] = fmaf(-lr_t, r, w[i]);
        }
      }
      st_f32<VN>(a.master + e, w);
      st_f32<VN>(a.slot0 + e, s0);
      if (a.kind == PX_LAMB) st_f32<VN>(a.slot1 + e, s1);
      if (a.ema) {
#pragma unroll
        for (int i = 0; i < VN; ++i) m[i] -= (1.f - ema_decay) * (m[i] - w[i]);
        st_f32<VN>(a.ema + e, m);
      }
      const uint4 out = Vec16<T>::pack(w);
      if (use_mc) {
        ds_mm_st(reinterpret_cast<T*>(params.p[0]) + base + e, out);
      } else {
#pragma unroll
        for (int p = 0; p < W; ++p) st_v4_stream(reinterpret_cast<T*>(params.p[p]) + base + e, out);
      }
    }
  }
  // MODE 2's end barrier: the last CTA announces that this rank's parameter stores are out and
  // waits for the same from every peer
  if (W > 1) {
    const int slot_e = ch_end * PX_MAX_BLOCKS;
    __shared__ bool s_last;
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence_system();
      s_last = atomicAdd(epoch_ctr + slot_e + 1, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (s_last) {
      const uint32_t e_end = ld_volatile_u32(epoch_ctr + slot_e) + 1;
      px_rank_signal(pads, slot_e, rank, W, e_end);
      px_rank_wait(pads, slot_e, rank, W, e_end);
      if (threadIdx.x == 0) {
        epoch_ctr[slot_e] = e_end;
        epoch_ctr[slot_e + 1] = 0;
      }
    }
  }
}

extern "C" {

// dtype 0 fp32 / 1 bf16.  grads/params: `world` pointers in natural order.
int px_dense_step(const void* const* grads, const void* const* params, float* master,
                  float* slot0, float* slot1, float* slot2, float* ema, float* red, const float* hp,
                  const float* clip, float* sumsq, size_t n, float avg, float ema_decay,
                  int kind, int mode, int acc_in, int dtype, void* pads_dev, void* epoch_ctr,
                  int ch_start, int ch_end, int rank, int world, int max_blocks, int use_mc,
                  cudaStream_t stream) {
  if (world < 1 || world > 8) return -3;
  const int vn = dtype == 0 ? 4 : 8;
  if (n % ((size_t)world * vn) != 0) return -1;
  // mode 3 and the accumulator need the fp32 scratch; the clip multiplier belongs to mode 2
  const bool acc = mode == 3 || acc_in;
  if (mode < 0 || mode > 3 || (acc && (red == nullptr || clip != nullptr || mode == 2)))
    return -2;
  // modes 0 and 2 apply an elementwise rule: the layer-wise and row-wise kinds have none here
  if ((mode == 0 || mode == 2) && (kind < 0 || kind > PX_CENTERED_RMSPROP)) return -4;
  DenseStepArgs a;
  a.use_mc = use_mc;
  if (use_mc) {            // entry 0 = multicast address; no peer pointers needed
    a.grads = PeerPtrs{}; a.params = PeerPtrs{};
    a.grads.p[0] = const_cast<void*>(grads[0]);
    a.params.p[0] = const_cast<void*>(params[0]);
  } else {
  a.grads = px_rotate(grads, rank, world);
  a.params = px_rotate(params, rank, world);
  }
  a.master = master; a.slot0 = slot0; a.slot1 = slot1; a.slot2 = slot2; a.ema = ema; a.red = red;
  a.hp = hp; a.clip = clip; a.sumsq = sumsq; a.n = n; a.avg = avg; a.ema_decay = ema_decay;
  a.rank = rank; a.ch_start = ch_start; a.ch_end = ch_end; a.kind = kind;
  a.mode = mode | (acc_in ? PX_DS_ACC_IN : 0);
  const int threads = 512;
  // rank-level barriers: the grid is sized for HBM bandwidth, not by barrier slots
  size_t b = (n / world / vn + threads - 1) / threads;
  const size_t cap = world == 1 ? PX_NUM_SMS * 4 : (size_t)(max_blocks > 0 ? max_blocks : PX_NUM_SMS);
  int blocks = (int)(b < 1 ? 1 : (b > cap ? cap : b));
#define LAUNCH_FAM(T, W, FAM)                                                              \
  do {                                                                                     \
    if (acc)                                                                               \
      px_dense_step_kernel<T, W, FAM, true><<<blocks, threads, 0, stream>>>(               \
          a, (uint32_t* const*)pads_dev, (uint32_t*)epoch_ctr);                            \
    else                                                                                   \
      px_dense_step_kernel<T, W, FAM, false><<<blocks, threads, 0, stream>>>(              \
          a, (uint32_t* const*)pads_dev, (uint32_t*)epoch_ctr);                            \
  } while (0)
#define LAUNCH(T, W)                                                                       \
  do {                                                                                     \
    if (PX_KIND_FAMILY(kind) == 0) LAUNCH_FAM(T, W, 0);                                    \
    else LAUNCH_FAM(T, W, 1);                                                              \
  } while (0)
  if (dtype == 0) { PX_DISPATCH_WORLD(world, LAUNCH, float); }
  else { PX_DISPATCH_WORLD(world, LAUNCH, __nv_bfloat16); }
#undef LAUNCH
#undef LAUNCH_FAM
  return (int)cudaGetLastError();
}

int px_stamp(void* slot, cudaStream_t stream) {
  px_stamp_kernel<<<1, 1, 0, stream>>>((unsigned long long*)slot);
  return (int)cudaGetLastError();
}

int px_clip_scale(const float* sumsq, float max_norm, float* scale_out, float* norm_out,
                  float* zero_after, cudaStream_t stream) {
  px_clip_scale_kernel<<<1, 1, 0, stream>>>(sumsq, max_norm, scale_out, norm_out, zero_after);
  return (int)cudaGetLastError();
}

int px_dense_async(const void* my_grads, void* my_params, const void* const* master,
                   const void* const* slot0, const void* const* slot1,
                   const void* const* slot2, const float* hp,
                   const float* clip, size_t n, int kind, int dtype, int rank, int world,
                   int max_blocks, cudaStream_t stream) {
  if (world < 1 || world > 8) return -3;
  const int vn = dtype == 0 ? 4 : 8;
  if (n % ((size_t)world * vn) != 0) return -1;
  if (kind < 0 || kind > PX_CENTERED_RMSPROP) return -4;     // elementwise rules only
  PeerPtrs M{}, S0{}, S1{}, S2{};
  for (int i = 0; i < world; ++i) {
    M.p[i] = const_cast<void*>(master[i]);
    S0.p[i] = slot0 ? const_cast<void*>(slot0[i]) : nullptr;
    S1.p[i] = slot1 ? const_cast<void*>(slot1[i]) : nullptr;
    S2.p[i] = slot2 ? const_cast<void*>(slot2[i]) : nullptr;
  }
  const int blocks = px_clamp_blocks(n / vn, 512, max_blocks);
#define LAUNCH(T, W)                                                                   \
  do {                                                                                 \
    if (PX_KIND_FAMILY(kind) == 0)                                                     \
      px_dense_async_kernel<T, W, 0><<<blocks, 512, 0, stream>>>(                      \
          (const T*)my_grads, (T*)my_params, M, S0, S1, S2, hp, clip, n, kind, rank);  \
    else                                                                               \
      px_dense_async_kernel<T, W, 1><<<blocks, 512, 0, stream>>>(                      \
          (const T*)my_grads, (T*)my_params, M, S0, S1, S2, hp, clip, n, kind, rank);  \
  } while (0)
  if (dtype == 0) { PX_DISPATCH_WORLD(world, LAUNCH, float); }
  else { PX_DISPATCH_WORLD(world, LAUNCH, __nv_bfloat16); }
#undef LAUNCH
  return (int)cudaGetLastError();
}

// n must be a multiple of 16/sizeof(T): the kernel reads whole 16-byte vectors only
int px_sumsq(const void* x, size_t n, int dtype, float mul, float* out, cudaStream_t stream) {
  const int vn = dtype == 0 ? 4 : 8;
  if (n % vn != 0) return -1;
  const int blocks = px_clamp_blocks(n / vn, 512 * 4, PX_NUM_SMS * 2);
  if (dtype == 0) px_sumsq_kernel<float><<<blocks, 512, 0, stream>>>((const float*)x, n, mul, out);
  else px_sumsq_kernel<__nv_bfloat16><<<blocks, 512, 0, stream>>>((const __nv_bfloat16*)x, n, mul, out);
  return (int)cudaGetLastError();
}

// Layer-wise passes of one bucket (kind PX_LARS / PX_LAMB, sharded update).  `chunks`,
// `seg_flags`, `seg_chunks`: the bucket's segment map for this rank (device); `red`, `master`,
// slots and `ema` are this rank's slices.
//   px_layerwise_norm  : norm pass and per-segment combine → sums [nseg, 2]
//   px_layerwise_update: trust ratios from `total` (the all-reduced sums; `sums` itself at
//                        W = 1), the update, the push to `params` and the end barrier
static int lw_args(LayerwiseArgs& a, int kind, const float* red, float* master, float* slot0,
                   float* slot1, float* ema, const float* hp, const float* clip,
                   const void* chunks, int nchunks, const int* seg_flags, const int* seg_chunks,
                   int nseg, float* partials, float* sums, const float* total) {
  if (kind != PX_LARS && kind != PX_LAMB) return -4;
  if (red == nullptr || master == nullptr || slot0 == nullptr ||
      (kind == PX_LAMB && slot1 == nullptr) || nchunks < 0 || nseg < 0) return -2;
  a.red = red; a.master = master; a.slot0 = slot0; a.slot1 = slot1; a.ema = ema; a.hp = hp;
  a.clip = clip; a.chunks = (const LwChunk*)chunks; a.nchunks = nchunks; a.seg_flags = seg_flags;
  a.seg_chunks = seg_chunks; a.nseg = nseg; a.partials = partials; a.sums = sums;
  a.total = total; a.kind = kind;
  return 0;
}

int px_layerwise_norm(const float* red, const float* master, const float* slot0,
                      const float* slot1, const float* hp, const float* clip, const void* chunks,
                      int nchunks, const int* seg_flags, const int* seg_chunks, int nseg,
                      float* partials, float* sums, int kind, int dtype, int max_blocks,
                      cudaStream_t stream) {
  LayerwiseArgs a;
  const int rc = lw_args(a, kind, red, const_cast<float*>(master), const_cast<float*>(slot0),
                         const_cast<float*>(slot1), nullptr, hp, clip, chunks, nchunks,
                         seg_flags, seg_chunks, nseg, partials, sums, nullptr);
  if (rc != 0) return rc;
  if (nseg == 0) return 0;
  const int cap = max_blocks > 0 ? max_blocks : PX_NUM_SMS * 4;
  const int blocks = nchunks < 1 ? 1 : (nchunks > cap ? cap : nchunks);
  if (nchunks > 0) {
    if (dtype == 0) px_lw_norm_kernel<4><<<blocks, 512, 0, stream>>>(a);
    else px_lw_norm_kernel<8><<<blocks, 512, 0, stream>>>(a);
  }
  px_lw_combine_kernel<<<(nseg + 255) / 256, 256, 0, stream>>>(a);
  return (int)cudaGetLastError();
}

int px_layerwise_update(const void* const* params, const float* red, float* master, float* slot0,
                        float* slot1, float* ema, const float* hp, const float* clip,
                        const void* chunks, int nchunks, const int* seg_flags, int nseg,
                        const float* total, size_t n, float ema_decay, int kind, int dtype,
                        void* pads_dev, void* epoch_ctr, int ch_end, int rank, int world,
                        int max_blocks, int use_mc, cudaStream_t stream) {
  if (world < 1 || world > 8) return -3;
  const int vn = dtype == 0 ? 4 : 8;
  if (n % ((size_t)world * vn) != 0) return -1;
  LayerwiseArgs a;
  const int rc = lw_args(a, kind, red, master, slot0, slot1, ema, hp, clip, chunks, nchunks,
                         seg_flags, nullptr, nseg, nullptr, nullptr, total);
  if (rc != 0) return rc;
  PeerPtrs P{};
  if (use_mc) P.p[0] = const_cast<void*>(params[0]);
  else P = px_rotate(params, rank, world);
  const int cap = world == 1 ? PX_NUM_SMS * 4 : (max_blocks > 0 ? max_blocks : PX_NUM_SMS);
  const int blocks = nchunks < 1 ? 1 : (nchunks > cap ? cap : nchunks);
#define LAUNCH(T, W)                                                                       \
  px_lw_update_kernel<T, W><<<blocks, 512, 0, stream>>>(a, P, n, ema_decay, rank, ch_end,  \
                                                        use_mc, (uint32_t* const*)pads_dev, \
                                                        (uint32_t*)epoch_ctr)
  if (dtype == 0) { PX_DISPATCH_WORLD(world, LAUNCH, float); }
  else { PX_DISPATCH_WORLD(world, LAUNCH, __nv_bfloat16); }
#undef LAUNCH
  return (int)cudaGetLastError();
}

}  // extern "C"
