// Fused attention decoder of the NMT models (`models/nmt/model.py: Decoder`,
// `ops/fused.py: nmt_attention_decoder`).
//
// Per time step and layer the node runs one cuBLAS product with an fp32 output (the gate
// pre-activations of [x_t | h_{t-1}]) and `px_nmt_lstm_cell_fwd`; per step the attention is
// `px_nmt_attn_fwd` (after the cuBLAS query projection for the Bahdanau kinds).  Backward mirrors
// it with `px_nmt_lstm_cell_bwd` and `px_nmt_attn_bwd`.  With layer-normalised LSTM cells the cell
// kernels are `px_nmt_ln_lstm_cell_fwd` / `bwd`, built on the row code of `ln_lstm_cell.cuh`.
//
// Every kernel runs one CTA of NA_THREADS threads per batch row.  All math is fp32; what is
// stored is bf16 or fp32 (the compute dtype) or fp32 where the backward pass consumes it.
// Attention never materialises [B, S, U]: a warp scores one source position at a time from the
// keys row and the query held in shared memory.  Reductions go through warp shuffles and then
// the warp partials in warp order, so two runs give the same bits.  d_keys and d_values are
// accumulated over the time steps in fp32 by the CTA that owns the row, and the per-row partials
// of the attention parameters' gradients are summed over rows in row order by
// `px_nmt_attn_param_grad`: no atomics anywhere.
#include "common.cuh"
#include "lstm_cell.cuh"   // lstm_cell_fwd_elem / lstm_cell_bwd_elem, sigmoidf_, tanhf_
#include "ln_lstm_cell.cuh"   // ln_lstm_cell_fwd_row / ln_lstm_cell_bwd_row

#define NA_THREADS 256
#define NA_WARPS (NA_THREADS / 32)
#define NA_MAX_U 1024   // units (keys and query width)
#define NA_MAX_M 2048   // memory width (values and context)
#define NA_MAX_S 1024   // source positions
static_assert(NA_THREADS == LN_ROW_THREADS, "the LN-LSTM cell kernels run the shared row code");

namespace {

template <typename T> __device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<__nv_bfloat16>(__nv_bfloat16 v) {
  return __bfloat162float(v);
}
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) {
  return __float2bfloat16_rn(v);
}
// value as stored in T, back in fp32
template <typename T> __device__ __forceinline__ float round_t(float v) {
  return to_f<T>(from_f<T>(v));
}

// 16-byte vectors: Vec16<T>::N elements
template <typename T>
__device__ __forceinline__ void ldv(const T* p, float* f) {
  Vec16<T>::unpack(*reinterpret_cast<const uint4*>(p), f);
}
template <typename T>
__device__ __forceinline__ void stv(T* p, const float* f) {
  *reinterpret_cast<uint4*>(p) = Vec16<T>::pack(f);
}
// 4-element groups (16 bytes of fp32, 8 of bf16)
template <typename T> __device__ __forceinline__ void ld4(const T* p, float* f);
template <> __device__ __forceinline__ void ld4<float>(const float* p, float* f) {
  const float4 v = *reinterpret_cast<const float4*>(p);
  f[0] = v.x; f[1] = v.y; f[2] = v.z; f[3] = v.w;
}
template <> __device__ __forceinline__ void ld4<__nv_bfloat16>(const __nv_bfloat16* p, float* f) {
  const uint2 v = *reinterpret_cast<const uint2*>(p);
  f[0] = __uint_as_float(v.x << 16); f[1] = __uint_as_float(v.x & 0xffff0000u);
  f[2] = __uint_as_float(v.y << 16); f[3] = __uint_as_float(v.y & 0xffff0000u);
}
template <typename T> __device__ __forceinline__ void st4(T* p, const float* f);
template <> __device__ __forceinline__ void st4<float>(float* p, const float* f) {
  *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
}
template <> __device__ __forceinline__ void st4<__nv_bfloat16>(__nv_bfloat16* p, const float* f) {
  __nv_bfloat162 a = __floats2bfloat162_rn(f[0], f[1]), b = __floats2bfloat162_rn(f[2], f[3]);
  *reinterpret_cast<uint2*>(p) =
      make_uint2(*reinterpret_cast<uint32_t*>(&a), *reinterpret_cast<uint32_t*>(&b));
}

// Block-wide sum or max; every thread gets the same bits (warp partials added in warp order).
template <bool MAX>
__device__ __forceinline__ float block_reduce(float v, float* s_red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float w = __shfl_xor_sync(0xffffffffu, v, o);
    v = MAX ? fmaxf(v, w) : v + w;
  }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) s_red[w] = v;
  __syncthreads();
  float t = s_red[0];
#pragma unroll
  for (int i = 1; i < NA_WARPS; ++i) t = MAX ? fmaxf(t, s_red[i]) : t + s_red[i];
  __syncthreads();
  return t;
}

// The query side of a row in shared memory: q (Luong) or pq + b (Bahdanau) in s_q, v' in s_v.
template <typename T, bool BAH>
__device__ __forceinline__ void load_query(const T* q, int q_ld, const float* pq, const float* vp,
                                           const T* bias, int U, float* s_q, float* s_v) {
  const int b = blockIdx.x;
  for (int u = threadIdx.x; u < U; u += NA_THREADS) {
    if (BAH) {
      s_q[u] = pq[(size_t)b * U + u] + (bias != nullptr ? to_f<T>(bias[u]) : 0.f);
      s_v[u] = vp[u];
    } else {
      s_q[u] = to_f<T>(q[(size_t)b * q_ld + u]);
    }
  }
}

// Σ_u f(k_u) over one keys row by one warp: q·k (Luong) or v'·tanh(k + pq + b) (Bahdanau).
template <typename T, bool BAH>
__device__ __forceinline__ float score_row(const T* krow, const float* s_q, const float* s_v,
                                           int U) {
  constexpr int V = Vec16<T>::N;
  const int lane = threadIdx.x & 31;
  float acc = 0.f;
  for (int u0 = lane * V; u0 < U; u0 += 32 * V) {
    float k[V];
    ldv(krow + u0, k);
#pragma unroll
    for (int i = 0; i < V; ++i)
      acc += BAH ? s_v[u0 + i] * tanhf_(k[i] + s_q[u0 + i]) : s_q[u0 + i] * k[i];
  }
  return warp_sum(acc);
}

// Attention forward of one step for row blockIdx.x:
//   score_s = g·(q·k_s) (luong, g = 1 when null) or v'·tanh(k_s + pq + b) (bahdanau kinds);
//   pad[b, s] -> −inf; a = softmax(score); ctx = Σ_s a_s values_s.
// Writes ctx (T, row stride ctx_ld), the alignments (fp32 [B, S]) and, when `feed` is set, the
// next step's layer-0 input ctx ⊙ fmask (T, row strides feed_ld / fmask_ld; fmask nullable).
template <typename T, bool BAH>
__global__ void __launch_bounds__(NA_THREADS)
px_nmt_attn_fwd_kernel(const T* __restrict__ q, int q_ld, const float* __restrict__ pq,
                       const T* __restrict__ keys, const T* __restrict__ values,
                       const unsigned char* __restrict__ pad, const T* __restrict__ g,
                       const float* __restrict__ vp, const T* __restrict__ bias,
                       T* __restrict__ ctx, int ctx_ld, const T* __restrict__ fmask,
                       int fmask_ld, T* __restrict__ feed, int feed_ld,
                       float* __restrict__ align, int S, int U, int M) {
  __shared__ __align__(16) float s_q[NA_MAX_U], s_v[BAH ? NA_MAX_U : 1], s_a[NA_MAX_S], s_red[NA_WARPS];
  const int b = blockIdx.x, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  load_query<T, BAH>(q, q_ld, pq, vp, bias, U, s_q, s_v);
  __syncthreads();
  const float scale = (!BAH && g != nullptr) ? to_f<T>(*g) : 1.f;
  for (int s = w; s < S; s += NA_WARPS) {
    const float sc = score_row<T, BAH>(keys + ((size_t)b * S + s) * U, s_q, s_v, U);
    if (lane == 0) s_a[s] = pad[(size_t)b * S + s] ? -INFINITY : sc * scale;
  }
  __syncthreads();
  float mx = -INFINITY;
  for (int s = threadIdx.x; s < S; s += NA_THREADS) mx = fmaxf(mx, s_a[s]);
  mx = block_reduce<true>(mx, s_red);
  float sum = 0.f;
  for (int s = threadIdx.x; s < S; s += NA_THREADS) {
    const float e = __expf(s_a[s] - mx);
    s_a[s] = e;
    sum += e;
  }
  sum = block_reduce<false>(sum, s_red);   // also orders the s_a writes before the reads below
  const float inv = 1.f / sum;
  for (int s = threadIdx.x; s < S; s += NA_THREADS) {
    const float a = s_a[s] * inv;
    s_a[s] = a;
    align[(size_t)b * S + s] = a;
  }
  __syncthreads();
  constexpr int V = Vec16<T>::N;
  const T* vrow = values + (size_t)b * S * M;
  for (int m0 = threadIdx.x * V; m0 < M; m0 += NA_THREADS * V) {
    float acc[V], v[V];
#pragma unroll
    for (int i = 0; i < V; ++i) acc[i] = 0.f;
    for (int s = 0; s < S; ++s) {
      const float a = s_a[s];
      if (a == 0.f) continue;        // masked positions (their values rows are zero)
      ldv(vrow + (size_t)s * M + m0, v);
#pragma unroll
      for (int i = 0; i < V; ++i) acc[i] += a * v[i];
    }
    stv(ctx + (size_t)b * ctx_ld + m0, acc);
    if (feed != nullptr) {
      float f[V];
#pragma unroll
      for (int i = 0; i < V; ++i)
        f[i] = round_t<T>(acc[i]) *
               (fmask != nullptr ? to_f<T>(fmask[(size_t)b * fmask_ld + m0 + i]) : 1.f);
      stv(feed + (size_t)b * feed_ld + m0, f);
    }
  }
}

// Attention backward of one step for row blockIdx.x.  d_ctx = dA ⊙ dA_mask + dO (each term
// nullable; dA fp32, the others T, all through row strides).  From the saved alignments a:
//   d_values[b] += a ⊗ d_ctx;  d_a_s = d_ctx·values_s;  d_score = a ⊙ (d_a − Σ a·d_a);
//   luong:    dq = g·Σ_s d_score_s k_s (fp32 [B, U]);  d_keys[b] += g·d_score ⊗ q;
//             part_g[b] += Σ_s d_score_s (q·k_s)  (scaled_luong);
//   bahdanau: d_pre = d_score_s v' (1 − tanh²);  dpq = Σ_s d_pre (T [B, U]);  d_keys[b] += d_pre;
//             part_v[b] += Σ_s d_score_s tanh(·);  part_b[b] += dpq  (normed_bahdanau).
// d_keys, d_values and the partials are fp32 and only ever touched by this row's CTA.
template <typename T, bool BAH>
__global__ void __launch_bounds__(NA_THREADS)
px_nmt_attn_bwd_kernel(const float* __restrict__ dA, int dA_ld, const T* __restrict__ dA_mask,
                       int dA_mask_ld, const T* __restrict__ dO, int dO_ld,
                       const float* __restrict__ align, const T* __restrict__ q, int q_ld,
                       const float* __restrict__ pq, const T* __restrict__ keys,
                       const T* __restrict__ values, const T* __restrict__ g,
                       const float* __restrict__ vp, const T* __restrict__ bias,
                       float* __restrict__ dq, T* __restrict__ dpq, float* __restrict__ dkeys,
                       float* __restrict__ dvalues, float* __restrict__ part_g,
                       float* __restrict__ part_v, float* __restrict__ part_b, int S, int U,
                       int M) {
  __shared__ __align__(16) float s_dc[NA_MAX_M], s_q[NA_MAX_U], s_v[BAH ? NA_MAX_U : 4];
  __shared__ float s_a[NA_MAX_S], s_d[NA_MAX_S], s_raw[BAH ? 1 : NA_MAX_S], s_red[NA_WARPS];
  const int b = blockIdx.x, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  load_query<T, BAH>(q, q_ld, pq, vp, bias, U, s_q, s_v);
  for (int m = threadIdx.x; m < M; m += NA_THREADS) {
    float d = 0.f;
    if (dA != nullptr)
      d = dA[(size_t)b * dA_ld + m] *
          (dA_mask != nullptr ? to_f<T>(dA_mask[(size_t)b * dA_mask_ld + m]) : 1.f);
    if (dO != nullptr) d += to_f<T>(dO[(size_t)b * dO_ld + m]);
    s_dc[m] = d;
  }
  for (int s = threadIdx.x; s < S; s += NA_THREADS) s_a[s] = align[(size_t)b * S + s];
  __syncthreads();
  const bool want_raw = !BAH && g != nullptr;
  constexpr int V = Vec16<T>::N;
  const T* vrow = values + (size_t)b * S * M;
  const T* krow = keys + (size_t)b * S * U;
  for (int s = w; s < S; s += NA_WARPS) {
    float acc = 0.f;
    if (s_a[s] != 0.f) {
      for (int m0 = lane * V; m0 < M; m0 += 32 * V) {
        float v[V];
        ldv(vrow + (size_t)s * M + m0, v);
#pragma unroll
        for (int i = 0; i < V; ++i) acc += s_dc[m0 + i] * v[i];
      }
    }
    acc = warp_sum(acc);
    const float raw = want_raw ? score_row<T, false>(krow + (size_t)s * U, s_q, s_v, U) : 0.f;
    if (lane == 0) {
      s_d[s] = acc;
      if (!BAH) s_raw[s] = raw;
    }
  }
  // d_values: columns of 4 per thread, every source position
  for (int m0 = threadIdx.x * 4; m0 < M; m0 += NA_THREADS * 4) {
    float dc[4], d[4];
    ld4(s_dc + m0, dc);
    for (int s = 0; s < S; ++s) {
      const float a = s_a[s];
      if (a == 0.f) continue;
      float* p = dvalues + ((size_t)b * S + s) * M + m0;
      ld4(p, d);
#pragma unroll
      for (int i = 0; i < 4; ++i) d[i] += a * dc[i];
      st4(p, d);
    }
  }
  __syncthreads();
  float dot = 0.f;
  for (int s = threadIdx.x; s < S; s += NA_THREADS) dot += s_a[s] * s_d[s];
  dot = block_reduce<false>(dot, s_red);
  float gs = 0.f;
  const float scale = (!BAH && g != nullptr) ? to_f<T>(*g) : 1.f;
  for (int s = threadIdx.x; s < S; s += NA_THREADS) {
    const float ds = s_a[s] * (s_d[s] - dot);
    if (want_raw) gs += ds * s_raw[s];
    s_d[s] = ds * scale;        // luong: d(q·k_s); bahdanau: d_score_s
  }
  if (want_raw) {
    gs = block_reduce<false>(gs, s_red);
    if (threadIdx.x == 0) part_g[b] += gs;
  } else {
    __syncthreads();
  }
  for (int u0 = threadIdx.x * 4; u0 < U; u0 += NA_THREADS * 4) {
    float qq[4], vv[4], acc[4] = {0.f, 0.f, 0.f, 0.f}, accv[4] = {0.f, 0.f, 0.f, 0.f};
    ld4(s_q + u0, qq);
    if (BAH) ld4(s_v + u0, vv);
    for (int s = 0; s < S; ++s) {
      const float ds = s_d[s];
      if (s_a[s] == 0.f) continue;
      float k[4], dk[4];
      ld4(krow + (size_t)s * U + u0, k);
      float* p = dkeys + ((size_t)b * S + s) * U + u0;
      ld4(p, dk);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (BAH) {
          const float th = tanhf_(k[i] + qq[i]);
          const float dpre = ds * vv[i] * (1.f - th * th);
          acc[i] += dpre;
          accv[i] += ds * th;
          dk[i] += dpre;
        } else {
          acc[i] += ds * k[i];
          dk[i] += ds * qq[i];
        }
      }
      st4(p, dk);
    }
    if (BAH) {
      st4(dpq + (size_t)b * U + u0, acc);
      float pv[4];
      ld4(part_v + (size_t)b * U + u0, pv);
#pragma unroll
      for (int i = 0; i < 4; ++i) pv[i] += accv[i];
      st4(part_v + (size_t)b * U + u0, pv);
      if (part_b != nullptr) {
        ld4(part_b + (size_t)b * U + u0, pv);
#pragma unroll
        for (int i = 0; i < 4; ++i) pv[i] += acc[i];
        st4(part_b + (size_t)b * U + u0, pv);
      }
    } else {
      st4(dq + (size_t)b * U + u0, acc);
    }
  }
}

// Column sums of per-row partials [B, n] over the rows, in row order.
__global__ void __launch_bounds__(256)
px_nmt_attn_param_grad_kernel(const float* __restrict__ part, int B, int n,
                              float* __restrict__ out) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= n) return;
  float s = 0.f;
  for (int b = 0; b < B; ++b) s += part[(size_t)b * n + col];
  out[col] = s;
}

// torch.nn.LSTM cell of one step for row blockIdx.x (gate order i, f, g, o):
//   pre = P + gx (nullable) + b_ih + b_hh (all fp32 but the biases);  c' = σf·c + σi·tanh g;
//   h = σo·tanh c'.  Writes c' (fp32), h (T) into h_out, the layer output y = h + resid
//   (resid nullable: the residual connection) into y, and, when `xn` is set, the next layer's
//   input y ⊙ mask (mask nullable: dropout) into xn.  Every T tensor goes through a row stride.
template <typename T>
__global__ void __launch_bounds__(NA_THREADS)
px_nmt_lstm_cell_fwd_kernel(const float* __restrict__ P, const float* __restrict__ gx,
                            const T* __restrict__ b_ih, const T* __restrict__ b_hh,
                            const float* __restrict__ c_prev, float* __restrict__ c_new,
                            T* __restrict__ h_out, int h_ld, const T* __restrict__ resid,
                            int resid_ld, T* __restrict__ y, int y_ld, const T* __restrict__ mask,
                            int mask_ld, T* __restrict__ xn, int xn_ld, int U) {
  const int b = blockIdx.x;
  const float* pr = P + (size_t)b * 4 * U;
  const float* gr = gx != nullptr ? gx + (size_t)b * 4 * U : nullptr;
  for (int u = threadIdx.x; u < U; u += NA_THREADS) {
    float pre[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int j = k * U + u;
      pre[k] = pr[j] + (gr != nullptr ? gr[j] : 0.f) + to_f<T>(b_ih[j]) + to_f<T>(b_hh[j]);
    }
    float a[4], m;
    const float c = lstm_cell_fwd_elem(pre[0], pre[2], pre[1], pre[3], c_prev[(size_t)b * U + u],
                                       0.f, a, &m);
    c_new[(size_t)b * U + u] = c;
    const T h = from_f<T>(m);
    h_out[(size_t)b * h_ld + u] = h;
    float yv = to_f<T>(h);
    if (resid != nullptr) yv = round_t<T>(yv + to_f<T>(resid[(size_t)b * resid_ld + u]));
    y[(size_t)b * y_ld + u] = from_f<T>(yv);
    if (xn != nullptr)
      xn[(size_t)b * xn_ld + u] =
          from_f<T>(mask != nullptr ? yv * to_f<T>(mask[(size_t)b * mask_ld + u]) : yv);
  }
}

// Backward of the cell above for row blockIdx.x.  The gradient of the layer output is
//   dy = dA ⊙ dA_mask + dR + dO  (dA fp32, dR fp32 [B, U], dO T; each nullable),
// written to dY (fp32 [B, U], nullable) for a residual connection below; dh = dy + drec (fp32,
// nullable: the recurrent term from step t+1).  Recomputes the gates from P, gx and the biases,
// takes the fp32 carry dc (dL/dc') in place to dL/dc, and writes the gate gradients dG (T,
// [B, 4U], gate order i, f, g, o).
template <typename T>
__global__ void __launch_bounds__(NA_THREADS)
px_nmt_lstm_cell_bwd_kernel(const float* __restrict__ P, const float* __restrict__ gx,
                            const T* __restrict__ b_ih, const T* __restrict__ b_hh,
                            const float* __restrict__ c_prev, const float* __restrict__ c_new,
                            const float* __restrict__ dA, int dA_ld, const T* __restrict__ dA_mask,
                            int dA_mask_ld, const float* __restrict__ dR, const T* __restrict__ dO,
                            int dO_ld, const float* __restrict__ drec, int drec_ld,
                            float* __restrict__ dc, T* __restrict__ dG, float* __restrict__ dY,
                            int U) {
  const int b = blockIdx.x;
  const float* pr = P + (size_t)b * 4 * U;
  const float* gr = gx != nullptr ? gx + (size_t)b * 4 * U : nullptr;
  for (int u = threadIdx.x; u < U; u += NA_THREADS) {
    float dy = 0.f;
    if (dA != nullptr)
      dy = dA[(size_t)b * dA_ld + u] *
           (dA_mask != nullptr ? to_f<T>(dA_mask[(size_t)b * dA_mask_ld + u]) : 1.f);
    if (dR != nullptr) dy += dR[(size_t)b * U + u];
    if (dO != nullptr) dy += to_f<T>(dO[(size_t)b * dO_ld + u]);
    if (dY != nullptr) dY[(size_t)b * U + u] = dy;
    const float dh = dy + (drec != nullptr ? drec[(size_t)b * drec_ld + u] : 0.f);
    float pre[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int j = k * U + u;
      pre[k] = pr[j] + (gr != nullptr ? gr[j] : 0.f) + to_f<T>(b_ih[j]) + to_f<T>(b_hh[j]);
    }
    const float cp = c_prev[(size_t)b * U + u];
    float a[4], m, dg[4];
    lstm_cell_fwd_elem(pre[0], pre[2], pre[1], pre[3], cp, 0.f, a, &m);
    dc[(size_t)b * U + u] =
        lstm_cell_bwd_elem(a, cp, c_new[(size_t)b * U + u], dh, dc[(size_t)b * U + u], dg);
    T* o = dG + (size_t)b * 4 * U + u;
    o[0] = from_f<T>(dg[0]);          // i
    o[U] = from_f<T>(dg[2]);          // f
    o[2 * U] = from_f<T>(dg[1]);      // g
    o[3 * U] = from_f<T>(dg[3]);      // o
  }
}

// Layer-normalised LSTM cell (`LayerNormLSTM.cell`, gates i, j, f, o; ln_lstm_cell.cuh) of one
// step for row blockIdx.x: pre = P + gx (nullable), both fp32 [B, 4U].  Writes c' (fp32, the
// carried state), h, y and xn exactly as px_nmt_lstm_cell_fwd_kernel does, and, when `stats` is
// set, the row's LL_NSTAT LayerNorm statistics.
template <typename T>
__global__ void __launch_bounds__(NA_THREADS)
px_nmt_ln_lstm_cell_fwd_kernel(const float* __restrict__ P, const float* __restrict__ gx,
                               const float* __restrict__ c_prev, float* __restrict__ c_new,
                               T* __restrict__ h_out, int h_ld, const T* __restrict__ resid,
                               int resid_ld, T* __restrict__ y, int y_ld,
                               const T* __restrict__ mask, int mask_ld, T* __restrict__ xn,
                               int xn_ld, float* __restrict__ stats, LnLstmParams<T> p, int U) {
  __shared__ float s_red[4 * NA_WARPS];
  const int b = blockIdx.x, j = threadIdx.x * 8;
  float hv[8], c2[8], st[LL_NSTAT];
  ln_lstm_cell_fwd_row<T>(P + (size_t)b * 4 * U, gx != nullptr ? gx + (size_t)b * 4 * U : nullptr,
                          c_prev + (size_t)b * U, p, U, s_red, hv, c2, st);
  if (stats != nullptr && threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < LL_NSTAT; ++k) stats[(size_t)b * LL_NSTAT + k] = st[k];
  }
  if (j >= U) return;
  st8(c_new + (size_t)b * U + j, c2);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int u = j + i;
    const T h = from_f<T>(hv[i]);
    h_out[(size_t)b * h_ld + u] = h;
    float yv = to_f<T>(h);
    if (resid != nullptr) yv = round_t<T>(yv + to_f<T>(resid[(size_t)b * resid_ld + u]));
    y[(size_t)b * y_ld + u] = from_f<T>(yv);
    if (xn != nullptr)
      xn[(size_t)b * xn_ld + u] =
          from_f<T>(mask != nullptr ? yv * to_f<T>(mask[(size_t)b * mask_ld + u]) : yv);
  }
}

// Backward of the cell above for row blockIdx.x, with the layer-output gradient dy, dY, drec and
// the in-place fp32 carry dc as in px_nmt_lstm_cell_bwd_kernel.  Recomputes the cell from P, gx
// and the saved statistics, writes the pre-LayerNorm gate gradients dG (T, [B, 4U], gate order
// i, j, f, o) and adds the row's dy·x̂ and dy of the five LayerNorms to acc[b] = [Σ dy·x̂ (5U) |
// Σ dy (5U)] (set instead of added when `first`).
template <typename T>
__global__ void __launch_bounds__(NA_THREADS)
px_nmt_ln_lstm_cell_bwd_kernel(const float* __restrict__ P, const float* __restrict__ gx,
                               const float* __restrict__ stats, const float* __restrict__ c_prev,
                               const float* __restrict__ dA, int dA_ld,
                               const T* __restrict__ dA_mask, int dA_mask_ld,
                               const float* __restrict__ dR, const T* __restrict__ dO, int dO_ld,
                               const float* __restrict__ drec, int drec_ld,
                               float* __restrict__ dc, T* __restrict__ dG, float* __restrict__ dY,
                               float* __restrict__ acc, int first, LnLstmParams<T> p, int U) {
  __shared__ float s_red[8 * NA_WARPS];
  const int b = blockIdx.x, j = threadIdx.x * 8;
  const bool on = j < U;
  float st[LL_NSTAT];
#pragma unroll
  for (int k = 0; k < LL_NSTAT; ++k) st[k] = stats[(size_t)b * LL_NSTAT + k];
  float dh[8], dcv[8];
  if (on) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int u = j + i;
      float dy = 0.f;
      if (dA != nullptr)
        dy = dA[(size_t)b * dA_ld + u] *
             (dA_mask != nullptr ? to_f<T>(dA_mask[(size_t)b * dA_mask_ld + u]) : 1.f);
      if (dR != nullptr) dy += dR[(size_t)b * U + u];
      if (dO != nullptr) dy += to_f<T>(dO[(size_t)b * dO_ld + u]);
      if (dY != nullptr) dY[(size_t)b * U + u] = dy;
      dh[i] = dy + (drec != nullptr ? drec[(size_t)b * drec_ld + u] : 0.f);
    }
    ld8(dc + (size_t)b * U + j, dcv);
  }
  float dp[4][8], dcp[8];
  ln_lstm_cell_bwd_row<T>(P + (size_t)b * 4 * U, gx != nullptr ? gx + (size_t)b * 4 * U : nullptr,
                          st, c_prev + (size_t)b * U, p, U, dh, dcv, s_red, dp, dcp,
                          acc + (size_t)b * 10 * U, first);
  if (!on) return;
  st8(dc + (size_t)b * U + j, dcp);
  T* o = dG + (size_t)b * 4 * U + j;
#pragma unroll
  for (int k = 0; k < 4; ++k) st8(o + k * U, dp[k]);
}

// Vector loads need U and M in whole 16-byte vectors and 4-column groups, and every row start
// (row strides included) on a 16-byte boundary.
inline bool attn_shape_ok(int B, int S, int U, int M, int dtype) {
  const int V = dtype == 0 ? 4 : 8;
  return B > 0 && S > 0 && S <= NA_MAX_S && U > 0 && U <= NA_MAX_U && U % V == 0 && M > 0 &&
         M <= NA_MAX_M && M % V == 0;
}

inline bool aligned16(const void* p) { return p == nullptr || ((uintptr_t)p & 15) == 0; }

inline bool ld_ok(int ld, int dtype) { return ld % (dtype == 0 ? 4 : 8) == 0; }

}  // namespace

extern "C" {

// Size limits of the attention kernels: units (U, keys and query width), memory width (M) and
// source positions (S).  U and M must also be multiples of 8 (16 bytes of bf16; 4 for fp32).
int px_nmt_max_units() { return NA_MAX_U; }
int px_nmt_max_memory() { return NA_MAX_M; }
int px_nmt_max_source() { return NA_MAX_S; }

// kind: 0 luong (g nullable: scaled_luong's scale), 1 bahdanau (bias nullable: normed's b)
int px_nmt_attn_fwd(const void* q, int q_ld, const float* pq, const void* keys,
                    const void* values, const unsigned char* pad, const void* g,
                    const float* vp, const void* bias, void* ctx, int ctx_ld, const void* fmask,
                    int fmask_ld, void* feed, int feed_ld, float* align, int B, int S, int U,
                    int M, int kind, int dtype, cudaStream_t stream) {
  if (!attn_shape_ok(B, S, U, M, dtype) || !ld_ok(ctx_ld, dtype) || !ld_ok(feed_ld, dtype) ||
      !aligned16(keys) || !aligned16(values) || !aligned16(ctx) || !aligned16(feed) ||
      (kind == 1 && (pq == nullptr || vp == nullptr)) || (kind == 0 && q == nullptr))
    return -2;
#define NA_FWD(T, K)                                                                            \
  px_nmt_attn_fwd_kernel<T, K><<<B, NA_THREADS, 0, stream>>>(                                   \
      (const T*)q, q_ld, pq, (const T*)keys, (const T*)values, pad, (const T*)g, vp,            \
      (const T*)bias, (T*)ctx, ctx_ld, (const T*)fmask, fmask_ld, (T*)feed, feed_ld, align, S, \
      U, M)
  if (dtype == 0) {
    if (kind == 1) NA_FWD(float, true); else NA_FWD(float, false);
  } else {
    if (kind == 1) NA_FWD(__nv_bfloat16, true); else NA_FWD(__nv_bfloat16, false);
  }
#undef NA_FWD
  return (int)cudaGetLastError();
}

int px_nmt_attn_bwd(const float* dA, int dA_ld, const void* dA_mask, int dA_mask_ld,
                    const void* dO, int dO_ld, const float* align, const void* q, int q_ld,
                    const float* pq, const void* keys, const void* values, const void* g,
                    const float* vp, const void* bias, float* dq, void* dpq, float* dkeys,
                    float* dvalues, float* part_g, float* part_v, float* part_b, int B, int S,
                    int U, int M, int kind, int dtype, cudaStream_t stream) {
  if (!attn_shape_ok(B, S, U, M, dtype) || !aligned16(keys) || !aligned16(values) ||
      !aligned16(dq) || !aligned16(dpq) || !aligned16(dkeys) || !aligned16(dvalues) ||
      !aligned16(part_v) || !aligned16(part_b) ||
      (kind == 1 && (pq == nullptr || vp == nullptr || dpq == nullptr || part_v == nullptr)) ||
      (kind == 0 && (q == nullptr || dq == nullptr || (g != nullptr && part_g == nullptr))))
    return -2;
#define NA_BWD(T, K)                                                                           \
  px_nmt_attn_bwd_kernel<T, K><<<B, NA_THREADS, 0, stream>>>(                                  \
      dA, dA_ld, (const T*)dA_mask, dA_mask_ld, (const T*)dO, dO_ld, align, (const T*)q, q_ld, \
      pq, (const T*)keys, (const T*)values, (const T*)g, vp, (const T*)bias, dq, (T*)dpq,      \
      dkeys, dvalues, part_g, part_v, part_b, S, U, M)
  if (dtype == 0) {
    if (kind == 1) NA_BWD(float, true); else NA_BWD(float, false);
  } else {
    if (kind == 1) NA_BWD(__nv_bfloat16, true); else NA_BWD(__nv_bfloat16, false);
  }
#undef NA_BWD
  return (int)cudaGetLastError();
}

int px_nmt_attn_param_grad(const float* part, int B, int n, float* out, cudaStream_t stream) {
  if (B <= 0 || n <= 0) return -2;
  px_nmt_attn_param_grad_kernel<<<(n + 255) / 256, 256, 0, stream>>>(part, B, n, out);
  return (int)cudaGetLastError();
}

int px_nmt_lstm_cell_fwd(const float* P, const float* gx, const void* b_ih, const void* b_hh,
                         const float* c_prev, float* c_new, void* h_out, int h_ld,
                         const void* resid, int resid_ld, void* y, int y_ld, const void* mask,
                         int mask_ld, void* xn, int xn_ld, int B, int U, int dtype,
                         cudaStream_t stream) {
  if (B <= 0 || U <= 0) return -2;
#define NL_FWD(T)                                                                             \
  px_nmt_lstm_cell_fwd_kernel<T><<<B, NA_THREADS, 0, stream>>>(                               \
      P, gx, (const T*)b_ih, (const T*)b_hh, c_prev, c_new, (T*)h_out, h_ld, (const T*)resid, \
      resid_ld, (T*)y, y_ld, (const T*)mask, mask_ld, (T*)xn, xn_ld, U)
  if (dtype == 0) NL_FWD(float); else NL_FWD(__nv_bfloat16);
#undef NL_FWD
  return (int)cudaGetLastError();
}

int px_nmt_lstm_cell_bwd(const float* P, const float* gx, const void* b_ih, const void* b_hh,
                         const float* c_prev, const float* c_new, const float* dA, int dA_ld,
                         const void* dA_mask, int dA_mask_ld, const float* dR, const void* dO,
                         int dO_ld, const float* drec, int drec_ld, float* dc, void* dG,
                         float* dY, int B, int U, int dtype, cudaStream_t stream) {
  if (B <= 0 || U <= 0) return -2;
#define NL_BWD(T)                                                                               \
  px_nmt_lstm_cell_bwd_kernel<T><<<B, NA_THREADS, 0, stream>>>(                                 \
      P, gx, (const T*)b_ih, (const T*)b_hh, c_prev, c_new, dA, dA_ld, (const T*)dA_mask,       \
      dA_mask_ld, dR, (const T*)dO, dO_ld, drec, drec_ld, dc, (T*)dG, dY, U)
  if (dtype == 0) NL_BWD(float); else NL_BWD(__nv_bfloat16);
#undef NL_BWD
  return (int)cudaGetLastError();
}

// ln: host array of 10 device pointers (γ of LN_i, LN_j, LN_f, LN_o, LN_c, then their β);
// eps: host array of the 5 LayerNorms' eps.
int px_nmt_ln_lstm_cell_fwd(const float* P, const float* gx, const float* c_prev, float* c_new,
                            void* h_out, int h_ld, const void* resid, int resid_ld, void* y,
                            int y_ld, const void* mask, int mask_ld, void* xn, int xn_ld,
                            float* stats, const void* const* ln, const float* eps,
                            float forget_bias, int B, int U, int dtype, cudaStream_t stream) {
  if (B <= 0 || U <= 0 || U % 8 || U > LL_MAX_UNITS) return -2;
#define NL_FWD(T)                                                                             \
  px_nmt_ln_lstm_cell_fwd_kernel<T><<<B, NA_THREADS, 0, stream>>>(                            \
      P, gx, c_prev, c_new, (T*)h_out, h_ld, (const T*)resid, resid_ld, (T*)y, y_ld,          \
      (const T*)mask, mask_ld, (T*)xn, xn_ld, stats, ln_lstm_params<T>(ln, eps, forget_bias), U)
  if (dtype == 0) NL_FWD(float); else NL_FWD(__nv_bfloat16);
#undef NL_FWD
  return (int)cudaGetLastError();
}

int px_nmt_ln_lstm_cell_bwd(const float* P, const float* gx, const float* stats,
                            const float* c_prev, const float* dA, int dA_ld, const void* dA_mask,
                            int dA_mask_ld, const float* dR, const void* dO, int dO_ld,
                            const float* drec, int drec_ld, float* dc, void* dG, float* dY,
                            float* acc, int first, const void* const* ln, const float* eps,
                            float forget_bias, int B, int U, int dtype, cudaStream_t stream) {
  if (B <= 0 || U <= 0 || U % 8 || U > LL_MAX_UNITS) return -2;
#define NL_BWD(T)                                                                               \
  px_nmt_ln_lstm_cell_bwd_kernel<T><<<B, NA_THREADS, 0, stream>>>(                              \
      P, gx, stats, c_prev, dA, dA_ld, (const T*)dA_mask, dA_mask_ld, dR, (const T*)dO, dO_ld,  \
      drec, drec_ld, dc, (T*)dG, dY, acc, first, ln_lstm_params<T>(ln, eps, forget_bias), U)
  if (dtype == 0) NL_BWD(float); else NL_BWD(__nv_bfloat16);
#undef NL_BWD
  return (int)cudaGetLastError();
}

}  // extern "C"
