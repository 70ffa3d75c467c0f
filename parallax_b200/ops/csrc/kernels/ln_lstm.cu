// Fused layer-normalised LSTM sequence layer for the NMT models (`models/nmt/model.py:
// LayerNormLSTM`, `ops/fused.py: ln_lstm_layer`).
//
// Before the loop one cuBLAS product gives the input side gx = x·W_xᵀ (fp32) of all T steps.
// Per time step the layer runs two launches forward (the cuBLAS product P = h·W_hᵀ in fp32, then
// `px_ln_lstm_fwd`) and two backward (`px_ln_lstm_bwd`, then dpre·W_h in fp32), in place of the
// composition's ~22 forward PyTorch ops per step.  After the loop dW and dx are one GEMM each
// over all T·B rows and `px_ln_lstm_param_grad` sums the γ/β accumulators.
//
// One CTA per batch row; the cell math is `ln_lstm_cell.cuh`.  The γ/β gradients are
// accumulated per row over the time steps by the CTA that owns the row and summed over rows, in
// row order, after the loop: no atomics, so the same operands give the same bits.
#include "common.cuh"
#include "ln_lstm_cell.cuh"

namespace {

// Forward of step t for row blockIdx.x.  live = lengths[b] > t (all rows when lengths is null):
//   c_new = live ? c' : c_prev,  h_next = live ? h' : h,  out_t = live ? h' : 0.
// gx, h, h_next and out go through row strides (gx_ld, h_ld, hn_ld, out_ld elements).
// stats (nullable) gets the row's LL_NSTAT LayerNorm statistics.
template <typename T>
__global__ void __launch_bounds__(LN_ROW_THREADS)
px_ln_lstm_fwd_kernel(const float* __restrict__ P, const float* __restrict__ gx, int gx_ld,
                      const float* __restrict__ c_prev, float* __restrict__ c_new,
                      const T* __restrict__ h, int h_ld, T* __restrict__ h_next, int hn_ld,
                      T* __restrict__ out, int out_ld, float* __restrict__ stats,
                      LnLstmParams<T> p, const long long* __restrict__ lengths, int t, int n) {
  __shared__ float s_red[4 * (LN_ROW_THREADS / 32)];
  const int b = blockIdx.x, j = threadIdx.x * 8;
  float hv[8], c2[8], st[LL_NSTAT];
  ln_lstm_cell_fwd_row<T>(P + (size_t)b * 4 * n, gx + (size_t)b * gx_ld, c_prev + (size_t)b * n,
                          p, n, s_red, hv, c2, st);
  if (stats != nullptr && threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < LL_NSTAT; ++k) stats[(size_t)b * LL_NSTAT + k] = st[k];
  }
  if (j >= n) return;
  const bool live = lengths == nullptr || lengths[b] > (long long)t;
  float o8[8];
  if (live) {
#pragma unroll
    for (int i = 0; i < 8; ++i) o8[i] = hv[i];
    st8(c_new + (size_t)b * n + j, c2);
  } else {
    ld8(h + (size_t)b * h_ld + j, hv);
    ld8(c_prev + (size_t)b * n + j, c2);
    st8(c_new + (size_t)b * n + j, c2);
#pragma unroll
    for (int i = 0; i < 8; ++i) o8[i] = 0.f;
  }
  st8(h_next + (size_t)b * hn_ld + j, hv);
  st8(out + (size_t)b * out_ld + j, o8);
}

// Backward of step t for row blockIdx.x, from the saved P, gx, stats and c_prev.  The carries
// are fp32 [B, n] and updated in place:
//   dh_t = carry_h + drec (drec = dpre_{t+1}·W_h, null at the first backward step);
//   live: the cell gets dh' = d_out_t + dh_t and dc' = carry_c; carry_h = 0, carry_c = dL/dc;
//   finished: the cell gets nothing; carry_h = dh_t, carry_c unchanged.
// Writes dpre (T, row stride dpre_ld: the pre-LayerNorm gate gradient, gate order i, j, f, o)
// and adds the row's LayerNorm terms to acc[b] = [Σ dy·x̂ (5n) | Σ dy (5n)].
template <typename T>
__global__ void __launch_bounds__(LN_ROW_THREADS)
px_ln_lstm_bwd_kernel(const float* __restrict__ P, const float* __restrict__ gx, int gx_ld,
                      const float* __restrict__ stats, const float* __restrict__ c_prev,
                      const T* __restrict__ dout, int dout_ld, const float* __restrict__ drec,
                      float* __restrict__ carry_h, float* __restrict__ carry_c,
                      T* __restrict__ dpre, int dpre_ld, float* __restrict__ acc, int first,
                      LnLstmParams<T> p, const long long* __restrict__ lengths, int t, int n) {
  __shared__ float s_red[8 * (LN_ROW_THREADS / 32)];
  const int b = blockIdx.x, j = threadIdx.x * 8;
  const bool on = j < n;
  const bool live = lengths == nullptr || lengths[b] > (long long)t;
  float st[LL_NSTAT];
#pragma unroll
  for (int k = 0; k < LL_NSTAT; ++k) st[k] = stats[(size_t)b * LL_NSTAT + k];
  float dh[8], dc[8], dht[8];
  if (on) {
    ld8(carry_h + (size_t)b * n + j, dht);
    if (drec != nullptr) {
      float r[8];
      ld8(drec + (size_t)b * n + j, r);
#pragma unroll
      for (int i = 0; i < 8; ++i) dht[i] += r[i];
    }
    if (live) {
      ld8(carry_c + (size_t)b * n + j, dc);
      if (dout != nullptr) {
        ld8(dout + (size_t)b * dout_ld + j, dh);
#pragma unroll
        for (int i = 0; i < 8; ++i) dh[i] += dht[i];
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) dh[i] = dht[i];
      }
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) { dh[i] = 0.f; dc[i] = 0.f; }
    }
  }
  float dp[4][8], dcp[8];
  ln_lstm_cell_bwd_row<T>(P + (size_t)b * 4 * n, gx + (size_t)b * gx_ld, st,
                          c_prev + (size_t)b * n, p, n, dh, dc, s_red, dp, dcp,
                          acc + (size_t)b * 10 * n, first);
  if (!on) return;
  T* o = dpre + (size_t)b * dpre_ld + j;
#pragma unroll
  for (int k = 0; k < 4; ++k) st8(o + k * n, dp[k]);
  if (live) {
#pragma unroll
    for (int i = 0; i < 8; ++i) dht[i] = 0.f;
    st8(carry_c + (size_t)b * n + j, dcp);
  }
  st8(carry_h + (size_t)b * n + j, dht);
}

// γ/β gradients: column sums of the per-row accumulators [B, 10n] over the rows, in row order,
// into out = [γ_i, γ_j, γ_f, γ_o, γ_c, β_i, β_j, β_f, β_o, β_c] (n each).
template <typename T>
__global__ void __launch_bounds__(256)
px_ln_lstm_param_grad_kernel(const float* __restrict__ acc, int B, int n, T* __restrict__ out) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= 10 * n) return;
  float s = 0.f;
  for (int b = 0; b < B; ++b) s += acc[(size_t)b * 10 * n + col];
  out[col] = from_f32<T>(s);
}

// Row strides must keep every 8-unit group on a 16-byte boundary.
inline bool ll_shape_ok(int B, int n) {
  return B > 0 && n > 0 && n % 8 == 0 && n <= LL_MAX_UNITS;
}

}  // namespace

extern "C" {

// Largest n (units) the cell kernels take: 8 units per thread, one 256-thread CTA per row.
int px_ln_lstm_max_units() { return LL_MAX_UNITS; }

// ln: host array of 10 device pointers (γ of LN_i, LN_j, LN_f, LN_o, LN_c, then their β);
// eps: host array of the 5 LayerNorms' eps.
int px_ln_lstm_fwd(const float* P, const float* gx, int gx_ld, const float* c_prev, float* c_new,
                   const void* h, int h_ld, void* h_next, int hn_ld, void* out, int out_ld,
                   float* stats, const void* const* ln, const float* eps, float forget_bias,
                   const long long* lengths, int t, int B, int n, int dtype,
                   cudaStream_t stream) {
  if (!ll_shape_ok(B, n) || gx_ld % 8 || h_ld % 8 || hn_ld % 8 || out_ld % 8) return -2;
#define LL_FWD(T)                                                                             \
  px_ln_lstm_fwd_kernel<T><<<B, LN_ROW_THREADS, 0, stream>>>(                                 \
      P, gx, gx_ld, c_prev, c_new, (const T*)h, h_ld, (T*)h_next, hn_ld, (T*)out, out_ld,     \
      stats, ln_lstm_params<T>(ln, eps, forget_bias), lengths, t, n)
  if (dtype == 0) LL_FWD(float); else LL_FWD(__nv_bfloat16);
#undef LL_FWD
  return (int)cudaGetLastError();
}

int px_ln_lstm_bwd(const float* P, const float* gx, int gx_ld, const float* stats,
                   const float* c_prev, const void* dout, int dout_ld, const float* drec,
                   float* carry_h, float* carry_c, void* dpre, int dpre_ld, float* acc, int first,
                   const void* const* ln, const float* eps, float forget_bias,
                   const long long* lengths, int t, int B, int n, int dtype,
                   cudaStream_t stream) {
  if (!ll_shape_ok(B, n) || gx_ld % 8 || dout_ld % 8 || dpre_ld % 8) return -2;
#define LL_BWD(T)                                                                             \
  px_ln_lstm_bwd_kernel<T><<<B, LN_ROW_THREADS, 0, stream>>>(                                 \
      P, gx, gx_ld, stats, c_prev, (const T*)dout, dout_ld, drec, carry_h, carry_c, (T*)dpre, \
      dpre_ld, acc, first, ln_lstm_params<T>(ln, eps, forget_bias), lengths, t, n)
  if (dtype == 0) LL_BWD(float); else LL_BWD(__nv_bfloat16);
#undef LL_BWD
  return (int)cudaGetLastError();
}

int px_ln_lstm_param_grad(const float* acc, int B, int n, void* out, int dtype,
                          cudaStream_t stream) {
  if (!ll_shape_ok(B, n)) return -2;
  const int blocks = (10 * n + 255) / 256;
  if (dtype == 0)
    px_ln_lstm_param_grad_kernel<float><<<blocks, 256, 0, stream>>>(acc, B, n, (float*)out);
  else
    px_ln_lstm_param_grad_kernel<__nv_bfloat16><<<blocks, 256, 0, stream>>>(
        acc, B, n, (__nv_bfloat16*)out);
  return (int)cudaGetLastError();
}

}  // extern "C"
