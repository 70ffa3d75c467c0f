// Per-row math of the layer-normalised LSTM cell (`models/nmt/model.py: LayerNormLSTM.cell`),
// shared by the sequence layer (ln_lstm.cu) and the NMT attention decoder's cell kernels
// (nmt_decoder.cu), so that both compute the same bits:
//
//   [i, j, f, o] = pre = [x | h]·Wᵀ (4 column blocks of n);  each block gets its own LayerNorm;
//   c' = c·σ(LN_f(f) + forget_bias) + σ(LN_i(i))·tanh(LN_j(j));
//   h' = tanh(LN_c(c'))·σ(LN_o(o)).
//
// The state carried to the next step is the un-normalised c', as `LayerNormLSTM.cell` carries
// it: `ln_lstm_cell_fwd_row` returns it in `c2` and `ln_lstm_cell_bwd_row` takes its gradient
// in `dc`.  Those two arguments are the only places that choice is made.
//
// One CTA of LN_ROW_THREADS threads per row; thread i owns the 8 units [8i, 8i + 8) of each
// block, so n <= LL_MAX_UNITS.  Every thread of the CTA must call these functions (they
// synchronise), including threads past n.  LayerNorm statistics are two-pass, as nn.LayerNorm
// computes them; all math is fp32.
#pragma once
#include "ln_row.cuh"
#include "lstm_cell.cuh"   // lstm_cell_fwd_elem, lstm_cell_bwd_elem, sigmoidf_, tanhf_

#define LL_MAX_UNITS (8 * LN_ROW_THREADS)
#define LL_NSTAT 10   // (mean, rstd) of LN_i, LN_j, LN_f, LN_o, LN_c

// γ, β and eps of the five LayerNorms (0-3: the gates i, j, f, o; 4: c) and the forget bias
template <typename T>
struct LnLstmParams {
  const T* g[5];
  const T* b[5];
  float eps[5];
  float forget_bias;
};

// ln: 10 device pointers (γ_0..γ_4, β_0..β_4), eps: 5 floats, both host arrays
template <typename T>
inline LnLstmParams<T> ln_lstm_params(const void* const* ln, const float* eps, float forget_bias) {
  LnLstmParams<T> p;
  for (int k = 0; k < 5; ++k) {
    p.g[k] = (const T*)ln[k];
    p.b[k] = (const T*)ln[5 + k];
    p.eps[k] = eps[k];
  }
  p.forget_bias = forget_bias;
  return p;
}

namespace {

// pre[k] = pr[k·n + j, +8) (+ gr, nullable) for this thread's 8 units
__device__ __forceinline__ void ll_load_pre(const float* pr, const float* gr, int n, int j,
                                            float (&v)[4][8]) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    ld8(pr + k * n + j, v[k]);
    if (gr != nullptr) {
      float a[8];
      ld8(gr + k * n + j, a);
#pragma unroll
      for (int i = 0; i < 8; ++i) v[k][i] += a[i];
    }
  }
}

// Forward of one row: pr, gr (nullable) the fp32 gate pre-activation terms [4n], c_prev the
// fp32 state row.  Returns this thread's h'[8] and carried state c2[8] (unset past n) and, in
// every thread, st[LL_NSTAT] = (mean, rstd) of the five LayerNorms.
template <typename T>
__device__ __forceinline__ void ln_lstm_cell_fwd_row(const float* pr, const float* gr,
                                                     const float* c_prev,
                                                     const LnLstmParams<T>& p, int n,
                                                     float* s_red, float* h, float* c2,
                                                     float* st) {
  const int j = threadIdx.x * 8;
  const bool on = j < n;
  float v[4][8];
  float s[4] = {0.f, 0.f, 0.f, 0.f};
  if (on) {
    ll_load_pre(pr, gr, n, j, v);
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int i = 0; i < 8; ++i) s[k] += v[k][i];
  }
  row_sum<4>(s, s_red);
  float q[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int k = 0; k < 4; ++k) st[2 * k] = s[k] / (float)n;
  if (on) {
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float d = v[k][i] - st[2 * k];
        q[k] += d * d;
      }
  }
  row_sum<4>(q, s_red);
#pragma unroll
  for (int k = 0; k < 4; ++k) st[2 * k + 1] = 1.f / sqrtf(q[k] / (float)n + p.eps[k]);
  float so[8], sc = 0.f;
  if (on) {
    float cp[8], g[4][8], b[4][8];
    ld8(c_prev + j, cp);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      ld8_scalar(p.g[k] + j, g[k]);
      ld8_scalar(p.b[k] + j, b[k]);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float a[4], pre[4], m;
#pragma unroll
      for (int k = 0; k < 4; ++k) pre[k] = (v[k][i] - st[2 * k]) * st[2 * k + 1] * g[k][i] + b[k][i];
      c2[i] = lstm_cell_fwd_elem(pre[0], pre[1], pre[2], pre[3], cp[i], p.forget_bias, a, &m);
      so[i] = a[3];
      sc += c2[i];
    }
  }
  row_sum<1>(&sc, s_red);
  st[8] = sc / (float)n;
  float qc = 0.f;
  if (on) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float d = c2[i] - st[8];
      qc += d * d;
    }
  }
  row_sum<1>(&qc, s_red);
  st[9] = 1.f / sqrtf(qc / (float)n + p.eps[4]);
  if (on) {
    float g[8], b[8];
    ld8_scalar(p.g[4] + j, g);
    ld8_scalar(p.b[4] + j, b);
#pragma unroll
    for (int i = 0; i < 8; ++i) h[i] = tanhf_((c2[i] - st[8]) * st[9] * g[i] + b[i]) * so[i];
  }
}

// Backward of one row from the forward's inputs and its saved statistics st.  dh: dL/dh',
// dc: dL/dc' from the later steps (both fp32, this thread's 8 units).  Writes dpre[4][8] (the
// gradient of the pre-LayerNorm gate terms, the operand of the products with W), dc_prev[8]
// = dL/dc, and adds dy·x̂ and dy of the five LayerNorms to the row's accumulator acc =
// [Σ dy·x̂ (5n) | Σ dy (5n)], column blocks i, j, f, o, c (set instead of added when `first`).
template <typename T>
__device__ __forceinline__ void ln_lstm_cell_bwd_row(const float* pr, const float* gr,
                                                     const float* __restrict__ st,
                                                     const float* c_prev,
                                                     const LnLstmParams<T>& p, int n,
                                                     const float* dh, const float* dc,
                                                     float* s_red, float (&dpre)[4][8],
                                                     float* dc_prev, float* acc, int first) {
  const int j = threadIdx.x * 8;
  const bool on = j < n;
  float xh[4][8], act[4][8], g[4][8], cp[8], cn[8], xc[8], dyc[8];
  float s[2] = {0.f, 0.f};   // Σ dx̂_c, Σ dx̂_c·x̂_c
  if (on) {
    ll_load_pre(pr, gr, n, j, xh);
    ld8(c_prev + j, cp);
    float b[4][8], gc[8], bc[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      ld8_scalar(p.g[k] + j, g[k]);
      ld8_scalar(p.b[k] + j, b[k]);
    }
    ld8_scalar(p.g[4] + j, gc);
    ld8_scalar(p.b[4] + j, bc);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float pre[4], a[4], m;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        xh[k][i] = (xh[k][i] - st[2 * k]) * st[2 * k + 1];
        pre[k] = xh[k][i] * g[k][i] + b[k][i];
      }
      cn[i] = lstm_cell_fwd_elem(pre[0], pre[1], pre[2], pre[3], cp[i], p.forget_bias, a, &m);
#pragma unroll
      for (int k = 0; k < 4; ++k) act[k][i] = a[k];
      xc[i] = (cn[i] - st[8]) * st[9];
      const float tc = tanhf_(xc[i] * gc[i] + bc[i]);
      dyc[i] = dh[i] * act[3][i] * (1.f - tc * tc);
      dpre[3][i] = dh[i] * tc * act[3][i] * (1.f - act[3][i]);   // LN_o's output gradient
      const float dx = dyc[i] * gc[i];
      s[0] += dx;
      s[1] += dx * xc[i];
    }
  }
  row_sum<2>(s, s_red);
  const float ac = s[0] / (float)n, bcm = s[1] / (float)n;
  float s8[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};   // per gate Σ dx̂, Σ dx̂·x̂
  if (on) {
    float gc[8];
    ld8_scalar(p.g[4] + j, gc);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      // dL/dc' through LN_c, plus the carried dc; the gate formulas of the plain LSTM cell
      // with no h-path term (dmv = 0) give the i, j, f gradients and dL/dc
      const float dc2 = st[9] * (dyc[i] * gc[i] - ac - xc[i] * bcm) + dc[i];
      const float a[4] = {act[0][i], act[1][i], act[2][i], act[3][i]};
      float dg[4];
      dc_prev[i] = lstm_cell_bwd_elem(a, cp[i], cn[i], 0.f, dc2, dg);
      dpre[0][i] = dg[0];
      dpre[1][i] = dg[1];
      dpre[2][i] = dg[2];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float dx = dpre[k][i] * g[k][i];
        s8[2 * k] += dx;
        s8[2 * k + 1] += dx * xh[k][i];
      }
    }
  }
  row_sum<8>(s8, s_red);
  if (on) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      acc_add(acc + k * n + j, acc + (5 + k) * n + j, xh[k], dpre[k], first);
      const float a = s8[2 * k] / (float)n, c = s8[2 * k + 1] / (float)n;
#pragma unroll
      for (int i = 0; i < 8; ++i)
        dpre[k][i] = st[2 * k + 1] * (dpre[k][i] * g[k][i] - a - xh[k][i] * c);
    }
    acc_add(acc + 4 * n + j, acc + 9 * n + j, xc, dyc, first);
  }
}

}  // namespace
