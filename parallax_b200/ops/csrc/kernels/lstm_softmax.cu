// Fused model-side kernels for the LM1B hot path.
//
//  * LSTM cell forward / backward (all gate non-linearities, cell update and
//    output gate in one pass each) — replaces ~8 + ~15 Eigen/ATen elementwise
//    launches per time step (reference: cwise_op_gpu_*.cu.cc sigmoid/tanh/mul/
//    add functors driven by `examples/lm1b/language_model.py:76-87`).
//  * Sampled-softmax loss forward+backward in ONE pass over the logits:
//    bias − log Q correction, accidental-hit masking, row log-sum-exp, loss,
//    and the softmax probabilities (= d loss / d logits) written back in place
//    (reference: tf.nn.sampled_softmax_loss → softmax_op_gpu.cu.cc:72,
//    sparse_xent_op_gpu.cu.cc, ≈15 elementwise passes over a [B·T, 8193] fp32
//    tensor).
#include "common.cuh"
#include "lstm_cell.cuh"

template <typename T> __device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// gates: [B, 4S] pre-activation (i | j | f | o);  c_prev/c_new: [B, S] fp32
// act:   [B, 4S] activated gates (σ(i) | tanh(j) | σ(f+1) | σ(o)) for backward
// m:     [B, S]  σ(o)·tanh(c_new)
template <typename T>
__global__ void __launch_bounds__(256)
px_lstm_cell_fwd_kernel(const T* __restrict__ gates, const float* __restrict__ c_prev,
                        T* __restrict__ act, float* __restrict__ c_new, T* __restrict__ m,
                        int B, int S, float forget_bias) {
  const int total = B * S;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += gridDim.x * blockDim.x) {
    const int b = idx / S, s = idx - b * S;
    const size_t g0 = (size_t)b * 4 * S + s;
    float a[4], mv;
    c_new[idx] = lstm_cell_fwd_elem(to_f(gates[g0]), to_f(gates[g0 + S]), to_f(gates[g0 + 2 * S]),
                                    to_f(gates[g0 + 3 * S]), c_prev[idx], forget_bias, a, &mv);
    m[idx] = from_f<T>(mv);
#pragma unroll
    for (int g = 0; g < 4; ++g) act[g0 + g * S] = from_f<T>(a[g]);
  }
}

// dm: [B,S]; dc (in: dL/dc_new from the future, out: dL/dc_prev) fp32 [B,S]
// dgates: [B,4S]
template <typename T>
__global__ void __launch_bounds__(256)
px_lstm_cell_bwd_kernel(const T* __restrict__ dm, float* __restrict__ dc,
                        const T* __restrict__ act, const float* __restrict__ c_prev,
                        const float* __restrict__ c_new, T* __restrict__ dgates, int B, int S) {
  const int total = B * S;
  // gate g of unit s lives at column g*S + s
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += gridDim.x * blockDim.x) {
    const int b = idx / S, s = idx - b * S;
    const size_t g0 = (size_t)b * 4 * S + s;
    float a[4], dg[4];
#pragma unroll
    for (int g = 0; g < 4; ++g) a[g] = to_f(act[g0 + g * S]);
    dc[idx] = lstm_cell_bwd_elem(a, c_prev[idx], c_new[idx], to_f(dm[idx]), dc[idx], dg);
#pragma unroll
    for (int g = 0; g < 4; ++g) dgates[g0 + g * S] = from_f<T>(dg[g]);
  }
}

// ---------------------------------------------------------------------------
// One CTA per row.  logits[N,S] (in: h·w_s ; out: p_ij = softmax prob of the
// sampled class j among {true, sampled}).  Row is held in registers
// (ITEMS × 256 threads ≥ S).
// DOT: the true-class logit h_row · w_true_row (P elements) is computed here as well
// (one launch instead of two casts, a multiply and a row reduction before this kernel).
template <typename T, int ITEMS, bool DOT>
__global__ void __launch_bounds__(256)
px_sampled_softmax_kernel(T* __restrict__ logits, const float* __restrict__ true_dot,
                          const float* __restrict__ adj_true,   // b_true - logq_true  [N]
                          const float* __restrict__ adj_samp,   // b_samp - logq_samp  [S]
                          const long long* __restrict__ targets, const long long* __restrict__ sampled,
                          float* __restrict__ loss, float* __restrict__ dtrue, int N, int S,
                          const T* __restrict__ h, const T* __restrict__ w_true, int P) {
  const int row = blockIdx.x;
  if (row >= N) return;
  __shared__ float s_red[8];
  __shared__ float s_bcast;
  T* x = logits + (size_t)row * S;
  const long long tgt = targets[row];
  float tl;
  if (DOT) {
    __shared__ float s_dot[8];
    const T* hr = h + (size_t)row * P;
    const T* wr = w_true + (size_t)row * P;
    float part = 0.f;
    for (int k = threadIdx.x; k < P; k += 256) part += to_f(hr[k]) * to_f(wr[k]);
    part = warp_sum(part);
    if ((threadIdx.x & 31) == 0) s_dot[threadIdx.x >> 5] = part;
    __syncthreads();
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += s_dot[k];          // same order in every thread
    tl = t + adj_true[row];
  } else {
    tl = true_dot[row] + adj_true[row];
  }
  float v[ITEMS];
  float mx = tl;
#pragma unroll
  for (int k = 0; k < ITEMS; ++k) {
    const int j = k * 256 + threadIdx.x;
    float a = -INFINITY;
    if (j < S) {
      a = to_f(x[j]) + adj_samp[j];
      if (sampled[j] == tgt) a = -INFINITY;        // remove accidental hits
    }
    v[k] = a;
    mx = fmaxf(mx, a);
  }
  // block max
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < 8 ? s_red[threadIdx.x] : -INFINITY;
    for (int o = 4; o > 0; o >>= 1) t = fmaxf(t, __shfl_xor_sync(0xffffffffu, t, o));
    if (threadIdx.x == 0) s_bcast = t;
  }
  __syncthreads();
  mx = s_bcast;
  float sum = 0.f;
#pragma unroll
  for (int k = 0; k < ITEMS; ++k) { v[k] = __expf(v[k] - mx); sum += v[k]; }
  sum = warp_sum(sum);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = sum;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < 8 ? s_red[threadIdx.x] : 0.f;
    t = warp_sum(t);
    if (threadIdx.x == 0) s_bcast = t + __expf(tl - mx);
  }
  __syncthreads();
  const float denom = s_bcast;
  const float inv = 1.f / denom;
#pragma unroll
  for (int k = 0; k < ITEMS; ++k) {
    const int j = k * 256 + threadIdx.x;
    if (j < S) x[j] = from_f<T>(v[k] * inv);
  }
  if (threadIdx.x == 0) {
    loss[row] = (mx + __logf(denom)) - tl;
    dtrue[row] = __expf(tl - mx) * inv - 1.f;
  }
}

// 16-byte vectors of T (4 floats / 8 bf16)
template <typename T> struct PxVec16;
template <> struct PxVec16<float> {
  static constexpr int N = 4;
  float v[4];
  __device__ __forceinline__ void load(const float* p) {
    const float4 t = *reinterpret_cast<const float4*>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  }
  __device__ __forceinline__ void store(float* p) const {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  }
};
template <> struct PxVec16<__nv_bfloat16> {
  static constexpr int N = 8;
  float v[8];
  __device__ __forceinline__ void load(const __nv_bfloat16* p) {
    const uint4 t = *reinterpret_cast<const uint4*>(p);
    const unsigned w[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      v[2 * i] = __uint_as_float(w[i] << 16);
      v[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    }
  }
  __device__ __forceinline__ void store(__nv_bfloat16* p) const {
    unsigned w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const __nv_bfloat162 b = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
      w[i] = *reinterpret_cast<const unsigned*>(&b);
    }
    *reinterpret_cast<uint4*>(p) = make_uint4(w[0], w[1], w[2], w[3]);
  }
};

template <typename T>
__global__ void __launch_bounds__(256)
px_ssm_bwd_kernel(T* __restrict__ G, const T* __restrict__ inputs, const T* __restrict__ w_true,
                  const float* __restrict__ g, int g_stride, const float* __restrict__ row_w,
                  const float* __restrict__ dtrue, float inv_n, T* __restrict__ gi,
                  T* __restrict__ d_w_true, void* __restrict__ d_b_true, int db_bf16,
                  T* __restrict__ grow_out, int N, int P) {
  constexpr int V = PxVec16<T>::N;
  const int per_row = P / V;
  const long long total = (long long)N * per_row;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int row = (int)(idx / per_row);
    const int col = (int)(idx - (long long)row * per_row);
    float grow = g[(size_t)row * g_stride] * inv_n;
    if (row_w != nullptr) grow *= row_w[row];
    const float gt = grow * dtrue[row];
    const size_t off = (size_t)row * P + (size_t)col * V;
    PxVec16<T> a, x, w, o;
    a.load(G + off);
    x.load(inputs + off);
    w.load(w_true + off);
#pragma unroll
    for (int i = 0; i < V; ++i) o.v[i] = a.v[i] * grow + gt * w.v[i];
    o.store(G + off);
#pragma unroll
    for (int i = 0; i < V; ++i) o.v[i] = x.v[i] * grow;
    o.store(gi + off);
#pragma unroll
    for (int i = 0; i < V; ++i) o.v[i] = x.v[i] * gt;
    o.store(d_w_true + off);
    if (col == 0) {
      if (db_bf16) reinterpret_cast<__nv_bfloat16*>(d_b_true)[row] = __float2bfloat16_rn(gt);
      else reinterpret_cast<float*>(d_b_true)[row] = gt;
      grow_out[row] = from_f<T>(grow);
    }
  }
}

extern "C" {

int px_lstm_cell_fwd(const void* gates, const float* c_prev, void* act, float* c_new, void* m,
                     int B, int S, float forget_bias, int dtype, cudaStream_t stream) {
  int blocks = (B * S + 255) / 256;
  if (blocks > PX_NUM_SMS * 8) blocks = PX_NUM_SMS * 8;
  if (dtype == 0)
    px_lstm_cell_fwd_kernel<float><<<blocks, 256, 0, stream>>>(
        (const float*)gates, c_prev, (float*)act, c_new, (float*)m, B, S, forget_bias);
  else
    px_lstm_cell_fwd_kernel<__nv_bfloat16><<<blocks, 256, 0, stream>>>(
        (const __nv_bfloat16*)gates, c_prev, (__nv_bfloat16*)act, c_new, (__nv_bfloat16*)m, B, S,
        forget_bias);
  return (int)cudaGetLastError();
}

int px_lstm_cell_bwd(const void* dm, float* dc, const void* act, const float* c_prev,
                     const float* c_new, void* dgates, int B, int S, int dtype, cudaStream_t stream) {
  int blocks = (B * S + 255) / 256;
  if (blocks > PX_NUM_SMS * 8) blocks = PX_NUM_SMS * 8;
  if (dtype == 0)
    px_lstm_cell_bwd_kernel<float><<<blocks, 256, 0, stream>>>(
        (const float*)dm, dc, (const float*)act, c_prev, c_new, (float*)dgates, B, S);
  else
    px_lstm_cell_bwd_kernel<__nv_bfloat16><<<blocks, 256, 0, stream>>>(
        (const __nv_bfloat16*)dm, dc, (const __nv_bfloat16*)act, c_prev, c_new,
        (__nv_bfloat16*)dgates, B, S);
  return (int)cudaGetLastError();
}

int px_sampled_softmax(void* logits, const float* true_dot, const float* adj_true,
                       const float* adj_samp, const long long* targets, const long long* sampled,
                       float* loss, float* dtrue, int N, int S, int dtype, cudaStream_t stream) {
  if (S > 256 * 64) return -2;
#define SS(T, I)                                                                          \
  px_sampled_softmax_kernel<T, I, false><<<N, 256, 0, stream>>>(                          \
      (T*)logits, true_dot, adj_true, adj_samp, targets, sampled, loss, dtrue, N, S,      \
      (const T*)nullptr, (const T*)nullptr, 0)
#define SSD(T)                                                      \
  if (S <= 256 * 4) SS(T, 4); else if (S <= 256 * 8) SS(T, 8);      \
  else if (S <= 256 * 16) SS(T, 16); else if (S <= 256 * 32) SS(T, 32); else SS(T, 64)
  if (dtype == 0) { SSD(float); } else { SSD(__nv_bfloat16); }
#undef SSD
#undef SS
  return (int)cudaGetLastError();
}

// Same, with the true-class dot product h[n]·w_true[n] computed in the kernel.
int px_sampled_softmax_dot(void* logits, const void* h, const void* w_true, int P,
                           const float* adj_true, const float* adj_samp,
                           const long long* targets, const long long* sampled, float* loss,
                           float* dtrue, int N, int S, int dtype, cudaStream_t stream) {
  if (S > 256 * 64) return -2;
#define SS(T, I)                                                                          \
  px_sampled_softmax_kernel<T, I, true><<<N, 256, 0, stream>>>(                           \
      (T*)logits, nullptr, adj_true, adj_samp, targets, sampled, loss, dtrue, N, S,       \
      (const T*)h, (const T*)w_true, P)
#define SSD(T)                                                      \
  if (S <= 256 * 4) SS(T, 4); else if (S <= 256 * 8) SS(T, 8);      \
  else if (S <= 256 * 16) SS(T, 16); else if (S <= 256 * 32) SS(T, 32); else SS(T, 64)
  if (dtype == 0) { SSD(float); } else { SSD(__nv_bfloat16); }
#undef SSD
#undef SS
  return (int)cudaGetLastError();
}

// Backward glue of the sampled-softmax head in one pass (was ~13 elementwise launches):
//   grow[n] = g[n*g_stride] * inv_n * (row_w ? row_w[n] : 1)       per-row upstream gradient
//   G (in: probs @ w_samp) -> d_inputs = G*grow + (grow*dtrue) * w_true
//   gi = inputs * grow              (operand of d_w_samp = probs^T @ gi)
//   d_w_true = (grow*dtrue) * inputs
//   d_b_true[n] = grow*dtrue ;  grow_out[n] = grow   (operand of d_b_samp = probs^T @ grow)
int px_ssm_bwd(void* G, const void* inputs, const void* w_true, const float* g, int g_stride,
               const float* row_w, const float* dtrue, float inv_n, void* gi, void* d_w_true,
               void* d_b_true, int db_bf16, void* grow_out, int N, int P, int dtype,
               cudaStream_t stream) {
  const int vec = dtype == 0 ? 4 : 8;
  if (P % vec) return -2;
  const long long total = (long long)N * (P / vec);
  int blocks = (int)((total + 255) / 256);
  if (blocks > PX_NUM_SMS * 8) blocks = PX_NUM_SMS * 8;
  if (blocks < 1) blocks = 1;
  if (dtype == 0)
    px_ssm_bwd_kernel<float><<<blocks, 256, 0, stream>>>(
        (float*)G, (const float*)inputs, (const float*)w_true, g, g_stride, row_w, dtrue, inv_n,
        (float*)gi, (float*)d_w_true, d_b_true, db_bf16, (float*)grow_out, N, P);
  else
    px_ssm_bwd_kernel<__nv_bfloat16><<<blocks, 256, 0, stream>>>(
        (__nv_bfloat16*)G, (const __nv_bfloat16*)inputs, (const __nv_bfloat16*)w_true, g,
        g_stride, row_w, dtrue, inv_n, (__nv_bfloat16*)gi, (__nv_bfloat16*)d_w_true, d_b_true,
        db_bf16, (__nv_bfloat16*)grow_out, N, P);
  return (int)cudaGetLastError();
}

}  // extern "C"
