// Optimizer update rules shared by the fused dense step and the sparse owner / async kernels.
//
// The reference recognises TF's update ops in the user graph and runs TF's kernels
// (graph_transform_lib.py:56-98 dense_var_update_op_types / sparse_var_update_op_types,
// tensorflow/core/kernels/training_ops_gpu.cu.cc:28-283, training_ops.cc:1276-1382).  All of them
// are available here as device rules, split in two template *families* so that the code (and
// register allocation) of the five hot rules is not touched by the long tail:
//   family 0: sgd, momentum(+nesterov), adagrad, adam, rmsprop          (<= 2 slots)
//   family 1: adadelta, ftrl, proximal sgd, proximal adagrad, adagrad-DA, centered rmsprop
//             (<= 3 slots; needs l1/l2/lr_power and the global step)
//   family 2: row-wise adagrad — one accumulator per table row, fed by the row's mean g²;
//             sparse owner kernel only (`px_sparse_owner_kernel<.., 2>` in sparse.cu), since
//             the rule needs the whole row before it can update any element of it
// Numerics oracle: `parallax_b200/optim.py::apply_dense_` / `apply_sparse_rows_`.
#pragma once
#include <cuda_runtime.h>

enum {
  PX_SGD = 0, PX_MOMENTUM = 1, PX_ADAGRAD = 2, PX_ADAM = 3, PX_RMSPROP = 4,
  PX_ADADELTA = 5, PX_FTRL = 6, PX_PROX_SGD = 7, PX_PROX_ADAGRAD = 8, PX_ADAGRAD_DA = 9,
  PX_CENTERED_RMSPROP = 10, PX_ROWWISE_ADAGRAD = 11
};
#define PX_KIND_FAMILY(kind) \
  ((kind) <= PX_RMSPROP ? 0 : (kind) <= PX_CENTERED_RMSPROP ? 1 : 2)

// device hyper-parameter vector (8 floats), see optim.py
enum { HP_LR = 0, HP_A, HP_B, HP_EPS, HP_WD, HP_STEP, HP_GSCALE, HP_FLAGS };

struct PxHP { float lr, a, b, eps, wd, step, flags; };
__device__ __forceinline__ PxHP px_load_hp(const float* hp) {
  PxHP h;
  h.lr = hp[HP_LR]; h.a = hp[HP_A]; h.b = hp[HP_B]; h.eps = hp[HP_EPS]; h.wd = hp[HP_WD];
  h.step = hp[HP_STEP]; h.flags = hp[HP_FLAGS];
  return h;
}

__device__ __forceinline__ float px_sign(float x) { return x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f); }

// prox step of the proximal optimizers: soft threshold by lr·l1, shrink by 1 + lr·l2
__device__ __forceinline__ float px_prox(float w, float g, float lr_t, float l1, float l2) {
  const float prox = fmaf(-lr_t, g, w);
  return px_sign(prox) * fmaxf(fabsf(prox) - lr_t * l1, 0.f) / fmaf(lr_t, l2, 1.f);
}

template <int FAM>
__device__ __forceinline__ void px_rule(int kind, const PxHP& h, float g, float& w, float& s0,
                                        float& s1, float& s2) {
  if (FAM == 0) {
    switch (kind) {
      case PX_SGD: w = fmaf(-h.lr, g, w); break;
      case PX_MOMENTUM:
        s0 = fmaf(h.a, s0, g);
        w = h.flags != 0.f ? fmaf(-h.lr, fmaf(h.a, s0, g), w) : fmaf(-h.lr, s0, w);
        break;
      case PX_ADAGRAD:
        s0 = fmaf(g, g, s0);
        w = fmaf(-h.lr * g, rsqrtf(s0), w);
        break;
      case PX_ADAM:
        s0 = fmaf(h.a, s0, (1.f - h.a) * g);
        s1 = fmaf(h.b, s1, (1.f - h.b) * g * g);
        w -= h.lr * s0 / (sqrtf(s1) + h.eps);
        break;
      case PX_RMSPROP:
        s0 = fmaf(h.a, s0, (1.f - h.a) * g * g);
        s1 = fmaf(h.b, s1, h.lr * g * rsqrtf(s0 + h.eps));
        w -= s1;
        break;
    }
  } else {
    switch (kind) {
      case PX_ADADELTA: {           // s0 accum, s1 accum_update; a = rho
        s0 = fmaf(h.a, s0, (1.f - h.a) * g * g);
        const float upd = sqrtf(s1 + h.eps) * rsqrtf(s0 + h.eps) * g;
        s1 = fmaf(h.a, s1, (1.f - h.a) * upd * upd);
        w = fmaf(-h.lr, upd, w);
        break;
      }
      case PX_FTRL: {               // s0 accum, s1 linear; a = lr_power (<=0), b = l1, eps = l2
        const float na = fmaf(g, g, s0);
        float pn, po;
        if (h.a == -0.5f) { pn = sqrtf(na); po = sqrtf(s0); }
        else { pn = powf(na, -h.a); po = powf(s0, -h.a); }
        s1 += g - (pn - po) / h.lr * w;
        const float quad = pn / h.lr + 2.f * h.eps;
        w = fabsf(s1) > h.b ? (px_sign(s1) * h.b - s1) / quad : 0.f;
        s0 = na;
        break;
      }
      case PX_PROX_SGD:             // a = l1, b = l2
        w = px_prox(w, g, h.lr, h.a, h.b);
        break;
      case PX_PROX_ADAGRAD:         // s0 accumulator
        s0 = fmaf(g, g, s0);
        w = px_prox(w, g, h.lr * rsqrtf(s0), h.a, h.b);
        break;
      case PX_ADAGRAD_DA: {         // s0 Σg, s1 Σg²; a = l1, b = l2; step = global step
        s0 += g;
        s1 = fmaf(g, g, s1);
        const float t = h.step;
        const float tmp = h.a > 0.f ? px_sign(s0) * fmaxf(fabsf(s0) - h.a * t, 0.f) : s0;
        w = -h.lr * tmp / (h.b * t * h.lr + sqrtf(s1));
        break;
      }
      case PX_CENTERED_RMSPROP:     // s0 ms, s1 mg, s2 mom; a = decay, b = momentum
        s0 = fmaf(h.a, s0, (1.f - h.a) * g * g);
        s1 = fmaf(h.a, s1, (1.f - h.a) * g);
        s2 = fmaf(h.b, s2, h.lr * g * rsqrtf(s0 - s1 * s1 + h.eps));
        w -= s2;
        break;
    }
  }
}

// four lanes of a row at once (sparse kernels)
template <int FAM>
__device__ __forceinline__ void px_rule4(int kind, const PxHP& h, const float4& g, float4& w,
                                         float4& s0, float4& s1, float4& s2) {
  px_rule<FAM>(kind, h, g.x, w.x, s0.x, s1.x, s2.x);
  px_rule<FAM>(kind, h, g.y, w.y, s0.y, s1.y, s2.y);
  px_rule<FAM>(kind, h, g.z, w.z, s0.z, s1.z, s2.z);
  px_rule<FAM>(kind, h, g.w, w.w, s0.w, s1.w, s2.w);
}
