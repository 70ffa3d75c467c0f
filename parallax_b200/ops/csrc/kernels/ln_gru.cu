// Fused layer-normalised GRU cell for the skip-thoughts encoder and decoders
// (`models/skip_thoughts/gru_cell.py`, `ops/fused.py: ln_gru_layer`).
//
// Per time step the layer runs two launches forward (the cuBLAS product hh = h·w_hu in fp32,
// then `px_ln_gru_fwd`) and two backward (`px_ln_gru_bwd`, then d(hh)·w_hu^T in fp32), in place
// of the composition's ~12 forward and ~30 backward elementwise / LayerNorm kernels per step.
//
// One CTA per batch row.  Thread i owns the 8-unit groups i, i + 256, …  (n % 8 == 0, at most
// LG_MAX_G groups per thread, so n <= 8 · 256 · LG_MAX_G = 4096): a group's hh values
// (z, r and candidate columns) stay in registers between the row reductions.  Row sums go
// through warp shuffles and then the 8 warp partials in warp order, so every thread sees the
// same bits and two runs give the same bits.  The γ/β gradients are accumulated per row over
// the time steps by the CTA that owns the row (no atomics) and summed over rows, in row order,
// by `px_ln_gru_param_grad` after the loop.
#include "common.cuh"
#include "ln_row.cuh"      // ld8, st8, ld8_scalar, from_f32, acc_add, row_sum
#include "lstm_cell.cuh"   // sigmoidf_, tanhf_

#define LG_THREADS LN_ROW_THREADS
#define LG_MAX_G 2
#define LG_MAX_UNITS (8 * LG_THREADS * LG_MAX_G)

namespace {

// Mean and 1/sqrt(biased var + eps) of the two LayerNorms of a row (over the 2n z|r columns and
// the n candidate columns), two-pass, as nn.LayerNorm computes them.
template <int G>
__device__ __forceinline__ void ln_stats(const float (&vz)[G][8], const float (&vr)[G][8],
                                         const float (&vu)[G][8], int n, float eps_wh,
                                         float eps_u, float* s_red, float* st) {
  float s[2] = {0.f, 0.f};
#pragma unroll
  for (int g = 0; g < G; ++g) {
    if ((threadIdx.x + g * LG_THREADS) * 8 >= n) continue;
#pragma unroll
    for (int i = 0; i < 8; ++i) { s[0] += vz[g][i] + vr[g][i]; s[1] += vu[g][i]; }
  }
  row_sum<2>(s, s_red);
  const float m1 = s[0] / (float)(2 * n), m2 = s[1] / (float)n;
  float q[2] = {0.f, 0.f};
#pragma unroll
  for (int g = 0; g < G; ++g) {
    if ((threadIdx.x + g * LG_THREADS) * 8 >= n) continue;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float a = vz[g][i] - m1, b = vr[g][i] - m1, c = vu[g][i] - m2;
      q[0] += a * a + b * b;
      q[1] += c * c;
    }
  }
  row_sum<2>(q, s_red);
  st[0] = m1;
  st[1] = 1.f / sqrtf(q[0] / (float)(2 * n) + eps_wh);
  st[2] = m2;
  st[3] = 1.f / sqrtf(q[1] / (float)n + eps_u);
}

// Forward cell of step t for row blockIdx.x:
//   [z, r] = σ(LN_wh(hh[:2n]) + gx_t),  ĥ = tanh(r ⊙ LN_u(hh[2n:]) + cx_t),
//   h' = (1 − z) ⊙ h + z ⊙ ĥ;  live = lengths[b] > t (all rows when lengths is null):
//   h_next = live ? h' : h,  out_t = live ? h' : 0.
// gx/cx/out are [B, T, ·] tensors read and written in place: row b of step t is at
// base + b·ld.  stats (nullable) gets (mean_wh, rstd_wh, mean_u, rstd_u) of the row.
template <typename T, int G>
__global__ void __launch_bounds__(LG_THREADS)
px_ln_gru_fwd_kernel(const float* __restrict__ hh, const T* __restrict__ gx, int gx_ld,
                     const T* __restrict__ cx, int cx_ld, const T* __restrict__ h,
                     T* __restrict__ h_next, T* __restrict__ out, int out_ld,
                     float* __restrict__ stats, const T* __restrict__ g_wh,
                     const T* __restrict__ b_wh, const T* __restrict__ g_u,
                     const T* __restrict__ b_u, const long long* __restrict__ lengths, int t,
                     int n, float eps_wh, float eps_u) {
  __shared__ float s_red[2 * (LG_THREADS / 32)];
  const int b = blockIdx.x;
  const float* hr = hh + (size_t)b * 3 * n;
  float vz[G][8], vr[G][8], vu[G][8];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const int j = (threadIdx.x + g * LG_THREADS) * 8;
    if (j >= n) continue;
    ld8(hr + j, vz[g]);
    ld8(hr + n + j, vr[g]);
    ld8(hr + 2 * n + j, vu[g]);
  }
  float st[4];
  ln_stats<G>(vz, vr, vu, n, eps_wh, eps_u, s_red, st);
  if (stats != nullptr && threadIdx.x == 0) {
    *reinterpret_cast<float4*>(stats + 4 * (size_t)b) = make_float4(st[0], st[1], st[2], st[3]);
  }
  const bool live = lengths == nullptr || lengths[b] > (long long)t;
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const int j = (threadIdx.x + g * LG_THREADS) * 8;
    if (j >= n) continue;
    float gxz[8], gxr[8], c8[8], h8[8], gz[8], bz[8], gr[8], br[8], gu[8], bu[8];
    ld8(gx + (size_t)b * gx_ld + j, gxz);
    ld8(gx + (size_t)b * gx_ld + n + j, gxr);
    ld8(cx + (size_t)b * cx_ld + j, c8);
    ld8(h + (size_t)b * n + j, h8);
    ld8_scalar(g_wh + j, gz);
    ld8_scalar(b_wh + j, bz);
    ld8_scalar(g_wh + n + j, gr);
    ld8_scalar(b_wh + n + j, br);
    ld8_scalar(g_u + j, gu);
    ld8_scalar(b_u + j, bu);
    float hn[8], o8[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float z = sigmoidf_((vz[g][i] - st[0]) * st[1] * gz[i] + bz[i] + gxz[i]);
      const float r = sigmoidf_((vr[g][i] - st[0]) * st[1] * gr[i] + br[i] + gxr[i]);
      const float un = (vu[g][i] - st[2]) * st[3] * gu[i] + bu[i];
      const float c = tanhf_(r * un + c8[i]);
      const float hp = (1.f - z) * h8[i] + z * c;
      hn[i] = live ? hp : h8[i];
      o8[i] = live ? hp : 0.f;
    }
    st8(h_next + (size_t)b * n + j, hn);
    st8(out + (size_t)b * out_ld + j, o8);
  }
}

// Backward cell of step t for row blockIdx.x, from the saved hh and stats:
//   dh' = live ? d_out_t + dh_carry : 0,  dh_carry = carry + drec (drec = d(hh)_{t+1}·w_hu^T,
//   null at the first backward step);  direct term of dh_t = live ? dh'·(1 − z) : dh_carry,
//   written back to carry.  Writes d(hh) (the operand of the next product), dgx_t, dcx_t,
//   and adds dy·x̂ and dy of both LayerNorms to the row's accumulator acc[b] = [Σ dy·x̂ (3n) |
//   Σ dy (3n)] (overwritten when `first`).
template <typename T, int G>
__global__ void __launch_bounds__(LG_THREADS)
px_ln_gru_bwd_kernel(const float* __restrict__ hh, const float* __restrict__ stats,
                     const T* __restrict__ gx, int gx_ld, const T* __restrict__ cx, int cx_ld,
                     const T* __restrict__ h, const T* __restrict__ dout, int dout_ld,
                     const float* __restrict__ drec, float* __restrict__ carry,
                     T* __restrict__ dhh, T* __restrict__ dgx, int dgx_ld, T* __restrict__ dcx,
                     int dcx_ld, float* __restrict__ acc, int first, const T* __restrict__ g_wh,
                     const T* __restrict__ b_wh, const T* __restrict__ g_u,
                     const T* __restrict__ b_u, const long long* __restrict__ lengths, int t,
                     int n) {
  __shared__ float s_red[4 * (LG_THREADS / 32)];
  const int b = blockIdx.x;
  const float* hr = hh + (size_t)b * 3 * n;
  const float4 st = *reinterpret_cast<const float4*>(stats + 4 * (size_t)b);
  const bool live = lengths == nullptr || lengths[b] > (long long)t;
  // xz/xr/xu: hh, then the normalised x̂;  dz/dr/du: the LayerNorm output gradients dy
  float xz[G][8], xr[G][8], xu[G][8], dz[G][8], dr[G][8], du[G][8];
  float s[4] = {0.f, 0.f, 0.f, 0.f};   // Σ dx̂_zr, Σ dx̂_zr·x̂_zr, Σ dx̂_u, Σ dx̂_u·x̂_u
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const int j = (threadIdx.x + g * LG_THREADS) * 8;
    if (j >= n) continue;
    ld8(hr + j, xz[g]);
    ld8(hr + n + j, xr[g]);
    ld8(hr + 2 * n + j, xu[g]);
    float gxz[8], gxr[8], c8[8], h8[8], gz[8], bz[8], gr[8], br[8], gu[8], bu[8];
    float dc8[8], do8[8], dr8[8];
    ld8(gx + (size_t)b * gx_ld + j, gxz);
    ld8(gx + (size_t)b * gx_ld + n + j, gxr);
    ld8(cx + (size_t)b * cx_ld + j, c8);
    ld8(h + (size_t)b * n + j, h8);
    ld8_scalar(g_wh + j, gz);
    ld8_scalar(b_wh + j, bz);
    ld8_scalar(g_wh + n + j, gr);
    ld8_scalar(b_wh + n + j, br);
    ld8_scalar(g_u + j, gu);
    ld8_scalar(b_u + j, bu);
    ld8(carry + (size_t)b * n + j, dc8);
    if (drec != nullptr) {
      ld8(drec + (size_t)b * n + j, dr8);
#pragma unroll
      for (int i = 0; i < 8; ++i) dc8[i] += dr8[i];
    }
    if (dout != nullptr) ld8(dout + (size_t)b * dout_ld + j, do8);
    float dgz[8], dgr[8], dcp[8], direct[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      xz[g][i] = (xz[g][i] - st.x) * st.y;
      xr[g][i] = (xr[g][i] - st.x) * st.y;
      xu[g][i] = (xu[g][i] - st.z) * st.w;
      const float z = sigmoidf_(xz[g][i] * gz[i] + bz[i] + gxz[i]);
      const float r = sigmoidf_(xr[g][i] * gr[i] + br[i] + gxr[i]);
      const float un = xu[g][i] * gu[i] + bu[i];
      const float c = tanhf_(r * un + c8[i]);
      const float gh = live ? (dout != nullptr ? do8[i] : 0.f) + dc8[i] : 0.f;
      direct[i] = live ? gh * (1.f - z) : dc8[i];
      const float dcpre = gh * z * (1.f - c * c);
      dz[g][i] = gh * (c - h8[i]) * z * (1.f - z);
      dr[g][i] = dcpre * un * r * (1.f - r);
      du[g][i] = dcpre * r;
      dgz[i] = dz[g][i];
      dgr[i] = dr[g][i];
      dcp[i] = dcpre;
      const float az = dz[g][i] * gz[i], ar = dr[g][i] * gr[i], au = du[g][i] * gu[i];
      s[0] += az + ar;
      s[1] += az * xz[g][i] + ar * xr[g][i];
      s[2] += au;
      s[3] += au * xu[g][i];
    }
    st8(carry + (size_t)b * n + j, direct);
    st8(dgx + (size_t)b * dgx_ld + j, dgz);
    st8(dgx + (size_t)b * dgx_ld + n + j, dgr);
    st8(dcx + (size_t)b * dcx_ld + j, dcp);
  }
  row_sum<4>(s, s_red);
  const float a1 = s[0] / (float)(2 * n), c1 = s[1] / (float)(2 * n);
  const float a2 = s[2] / (float)n, c2 = s[3] / (float)n;
  float* ar = acc + (size_t)b * 6 * n;
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const int j = (threadIdx.x + g * LG_THREADS) * 8;
    if (j >= n) continue;
    float gz[8], gr[8], gu[8], o[8];
    ld8_scalar(g_wh + j, gz);
    ld8_scalar(g_wh + n + j, gr);
    ld8_scalar(g_u + j, gu);
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i] = st.y * (dz[g][i] * gz[i] - a1 - xz[g][i] * c1);
    st8(dhh + (size_t)b * 3 * n + j, o);
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i] = st.y * (dr[g][i] * gr[i] - a1 - xr[g][i] * c1);
    st8(dhh + (size_t)b * 3 * n + n + j, o);
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i] = st.w * (du[g][i] * gu[i] - a2 - xu[g][i] * c2);
    st8(dhh + (size_t)b * 3 * n + 2 * n + j, o);
    // the row's γ/β accumulators: columns [0, 3n) Σ dy·x̂, [3n, 6n) Σ dy, in hh's column order
    acc_add(ar + j, ar + 3 * n + j, xz[g], dz[g], first);
    acc_add(ar + n + j, ar + 4 * n + j, xr[g], dr[g], first);
    acc_add(ar + 2 * n + j, ar + 5 * n + j, xu[g], du[g], first);
  }
}

// γ/β gradients: column sums of the per-row accumulators over the B rows, in row order.
template <typename T>
__global__ void __launch_bounds__(256)
px_ln_gru_param_grad_kernel(const float* __restrict__ acc, int B, int n, T* __restrict__ dg_wh,
                            T* __restrict__ db_wh, T* __restrict__ dg_u, T* __restrict__ db_u) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= 6 * n) return;
  float s = 0.f;
  for (int b = 0; b < B; ++b) s += acc[(size_t)b * 6 * n + col];
  const int k = col < 3 * n ? col : col - 3 * n;
  T* dst = col < 3 * n ? (k < 2 * n ? dg_wh + k : dg_u + (k - 2 * n))
                       : (k < 2 * n ? db_wh + k : db_u + (k - 2 * n));
  *dst = from_f32<T>(s);
}

inline bool lg_shape_ok(int B, int n) {
  return B > 0 && n > 0 && n % 8 == 0 && n <= LG_MAX_UNITS;
}

}  // namespace

extern "C" {

// Largest n (units) the cell kernels take: 8 units per group, LG_MAX_G groups per thread.
int px_ln_gru_max_units() { return LG_MAX_UNITS; }

int px_ln_gru_fwd(const float* hh, const void* gx, int gx_ld, const void* cx, int cx_ld,
                  const void* h, void* h_next, void* out, int out_ld, float* stats,
                  const void* g_wh, const void* b_wh, const void* g_u, const void* b_u,
                  const long long* lengths, int t, int B, int n, float eps_wh, float eps_u,
                  int dtype, cudaStream_t stream) {
  if (!lg_shape_ok(B, n)) return -2;
  const int G = (n / 8 + LG_THREADS - 1) / LG_THREADS;
#define LG_FWD(T, GG)                                                                         \
  px_ln_gru_fwd_kernel<T, GG><<<B, LG_THREADS, 0, stream>>>(                                  \
      hh, (const T*)gx, gx_ld, (const T*)cx, cx_ld, (const T*)h, (T*)h_next, (T*)out, out_ld, \
      stats, (const T*)g_wh, (const T*)b_wh, (const T*)g_u, (const T*)b_u, lengths, t, n,     \
      eps_wh, eps_u)
  if (dtype == 0) {
    if (G == 1) LG_FWD(float, 1); else LG_FWD(float, 2);
  } else {
    if (G == 1) LG_FWD(__nv_bfloat16, 1); else LG_FWD(__nv_bfloat16, 2);
  }
#undef LG_FWD
  return (int)cudaGetLastError();
}

int px_ln_gru_bwd(const float* hh, const float* stats, const void* gx, int gx_ld, const void* cx,
                  int cx_ld, const void* h, const void* dout, int dout_ld, const float* drec,
                  float* carry, void* dhh, void* dgx, int dgx_ld, void* dcx, int dcx_ld,
                  float* acc, int first, const void* g_wh, const void* b_wh, const void* g_u,
                  const void* b_u, const long long* lengths, int t, int B, int n, int dtype,
                  cudaStream_t stream) {
  if (!lg_shape_ok(B, n)) return -2;
  const int G = (n / 8 + LG_THREADS - 1) / LG_THREADS;
#define LG_BWD(T, GG)                                                                           \
  px_ln_gru_bwd_kernel<T, GG><<<B, LG_THREADS, 0, stream>>>(                                    \
      hh, stats, (const T*)gx, gx_ld, (const T*)cx, cx_ld, (const T*)h, (const T*)dout, dout_ld, \
      drec, carry, (T*)dhh, (T*)dgx, dgx_ld, (T*)dcx, dcx_ld, acc, first, (const T*)g_wh,       \
      (const T*)b_wh, (const T*)g_u, (const T*)b_u, lengths, t, n)
  if (dtype == 0) {
    if (G == 1) LG_BWD(float, 1); else LG_BWD(float, 2);
  } else {
    if (G == 1) LG_BWD(__nv_bfloat16, 1); else LG_BWD(__nv_bfloat16, 2);
  }
#undef LG_BWD
  return (int)cudaGetLastError();
}

int px_ln_gru_param_grad(const float* acc, int B, int n, void* dg_wh, void* db_wh, void* dg_u,
                         void* db_u, int dtype, cudaStream_t stream) {
  if (!lg_shape_ok(B, n)) return -2;
  const int blocks = (6 * n + 255) / 256;
  if (dtype == 0)
    px_ln_gru_param_grad_kernel<float><<<blocks, 256, 0, stream>>>(
        acc, B, n, (float*)dg_wh, (float*)db_wh, (float*)dg_u, (float*)db_u);
  else
    px_ln_gru_param_grad_kernel<__nv_bfloat16><<<blocks, 256, 0, stream>>>(
        acc, B, n, (__nv_bfloat16*)dg_wh, (__nv_bfloat16*)db_wh, (__nv_bfloat16*)dg_u,
        (__nv_bfloat16*)db_u);
  return (int)cudaGetLastError();
}

}  // extern "C"
