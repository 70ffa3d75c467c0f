// Row helpers of the one-CTA-per-row LayerNorm cell kernels (ln_gru.cu, ln_lstm.cu,
// nmt_decoder.cu).  A CTA of LN_ROW_THREADS threads owns one batch row; thread i holds the
// 8-unit groups i, i + LN_ROW_THREADS, … in registers.  Row sums go through warp shuffles and
// then the warp partials in warp order, so every thread sees the same bits and two runs give
// the same bits.
#pragma once
#include "common.cuh"

#define LN_ROW_THREADS 256

namespace {

template <typename T>
__device__ __forceinline__ void ld8(const T* p, float* f) {
  constexpr int N = Vec16<T>::N;
#pragma unroll
  for (int i = 0; i < 8 / N; ++i) Vec16<T>::unpack(*reinterpret_cast<const uint4*>(p + i * N), f + i * N);
}
template <typename T>
__device__ __forceinline__ void st8(T* p, const float* f) {
  constexpr int N = Vec16<T>::N;
#pragma unroll
  for (int i = 0; i < 8 / N; ++i) *reinterpret_cast<uint4*>(p + i * N) = Vec16<T>::pack(f + i * N);
}
// LayerNorm parameters are read one element at a time: they may be views into a parameter
// bucket at any 2-byte offset
template <typename T>
__device__ __forceinline__ void ld8_scalar(const T* p, float* f) {
#pragma unroll
  for (int i = 0; i < 8; ++i) f[i] = (float)p[i];
}
template <>
__device__ __forceinline__ void ld8_scalar<__nv_bfloat16>(const __nv_bfloat16* p, float* f) {
#pragma unroll
  for (int i = 0; i < 8; ++i) f[i] = __bfloat162float(p[i]);
}

template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) {
  return __float2bfloat16_rn(v);
}

// acc_g += dy·x̂, acc_b += dy for 8 columns (set instead of added when `first`)
__device__ __forceinline__ void acc_add(float* acc_g, float* acc_b, const float* x,
                                        const float* dy, int first) {
  float pg[8], pb[8];
  if (first) {
#pragma unroll
    for (int i = 0; i < 8; ++i) { pg[i] = 0.f; pb[i] = 0.f; }
  } else {
    ld8(acc_g, pg);
    ld8(acc_b, pb);
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) { pg[i] += dy[i] * x[i]; pb[i] += dy[i]; }
  st8(acc_g, pg);
  st8(acc_b, pb);
}

// K row sums over the CTA; every thread gets the same bits.  s_red holds K · warps floats.
template <int K>
__device__ __forceinline__ void row_sum(float* v, float* s_red) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    v[k] = warp_sum(v[k]);
    if (lane == 0) s_red[k * (LN_ROW_THREADS / 32) + w] = v[k];
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < K; ++k) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < LN_ROW_THREADS / 32; ++i) t += s_red[k * (LN_ROW_THREADS / 32) + i];
    v[k] = t;
  }
  __syncthreads();
}

}  // namespace
