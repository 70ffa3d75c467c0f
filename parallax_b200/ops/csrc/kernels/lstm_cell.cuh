// Per-element LSTM cell math, shared by the standalone cell kernels (lstm_softmax.cu) and the
// cell stages fused into the recurrent projection products (gemm_tc.cu), so that both compute
// the same bits.
#pragma once
#include "common.cuh"

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + __expf(-x)); }
__device__ __forceinline__ float tanhf_(float x) {
  // accurate enough for bf16 activations, exact limits for |x| large
  const float e = __expf(-2.f * fabsf(x));
  const float t = (1.f - e) / (1.f + e);
  return copysignf(t, x);
}

// Forward cell of one unit from its four gate pre-activations (i, j, f, o) and c_prev:
// a[0..3] = σ(i), tanh(j), σ(f + forget_bias), σ(o); returns c_new; *m_out = σ(o)·tanh(c_new).
// c_new is one explicit fma so that every kernel using this rounds it identically.
__device__ __forceinline__ float lstm_cell_fwd_elem(float gi, float gj, float gf, float go,
                                                    float c_prev, float forget_bias, float* a,
                                                    float* m_out) {
  a[0] = sigmoidf_(gi);
  a[1] = tanhf_(gj);
  a[2] = sigmoidf_(gf + forget_bias);
  a[3] = sigmoidf_(go);
  const float c = __fmaf_rn(a[2], c_prev, __fmul_rn(a[0], a[1]));
  *m_out = a[3] * tanhf_(c);
  return c;
}

// Backward cell of one unit: activations a (σ(i), tanh(j), σ(f), σ(o)), c_prev, c_new, dL/dm
// and dL/dc_new (dc) -> the four gate gradients dg; returns dL/dc_prev.
__device__ __forceinline__ float lstm_cell_bwd_elem(const float* a, float c_prev, float c_new,
                                                    float dmv, float dc, float* dg) {
  const float si = a[0], tj = a[1], sf = a[2], so = a[3];
  const float tc = tanhf_(c_new);
  const float dcv = dc + dmv * so * (1.f - tc * tc);
  dg[0] = dcv * tj * si * (1.f - si);
  dg[1] = dcv * si * (1.f - tj * tj);
  dg[2] = dcv * c_prev * sf * (1.f - sf);
  dg[3] = dmv * tc * so * (1.f - so);
  return dcv * sf;
}
