// sam_road_b200 :: per-element loss terms of the reference's criteria (model.py:350-354), shared by the
// validation accumulator (metrics.cu) and the training step (train.cu) so that both score a logit alike.
#pragma once

#include <cuda_runtime.h>

namespace srb {

// torch's CUDA log_sigmoid: min(0, x) - log1p(exp(-|x|))
__device__ __forceinline__ float log_sigmoid_f32(float x) {
  return __fsub_rn(fminf(0.0f, x), log1pf(expf(-fabsf(x))));
}

// F.binary_cross_entropy_with_logits(x, y, reduction='none') = (1 - y) * x - log_sigmoid(x), one rounding
// per torch op
__device__ __forceinline__ float bce_term(float x, float y) {
  return __fsub_rn(__fmul_rn(__fsub_rn(1.0f, y), x), log_sigmoid_f32(x));
}

// torchvision.ops.sigmoid_focal_loss(x, y, alpha=0.25, gamma=2, reduction='none') in its order
__device__ __forceinline__ float focal_term(float x, float y) {
  const float p = __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-x)));
  const float one_y = __fsub_rn(1.0f, y);
  const float p_t = __fadd_rn(__fmul_rn(p, y), __fmul_rn(__fsub_rn(1.0f, p), one_y));
  const float m = __fsub_rn(1.0f, p_t);
  const float loss = __fmul_rn(bce_term(x, y), __fmul_rn(m, m));
  const float alpha_t = __fadd_rn(__fmul_rn(0.25f, y), __fmul_rn(0.75f, one_y));
  return __fmul_rn(alpha_t, loss);
}

// d bce_term / dx = sigmoid(x) - y
__device__ __forceinline__ float bce_grad(float x, float y) { return 1.0f / (1.0f + expf(-x)) - y; }

// d focal_term / dx in closed form: with p = sigmoid(x), ce = bce_term, p_t = p y + (1 - p)(1 - y),
// m = 1 - p_t:  alpha_t * (m^2 (p - y) - 2 m ce dp_t/dx),  dp_t/dx = p (1 - p)(2y - 1)
__device__ __forceinline__ float focal_grad(float x, float y) {
  const float p = 1.0f / (1.0f + expf(-x));
  const float p_t = p * y + (1.0f - p) * (1.0f - y);
  const float m = 1.0f - p_t;
  const float alpha_t = 0.25f * y + 0.75f * (1.0f - y);
  const float dpt = p * (1.0f - p) * (2.0f * y - 1.0f);
  return alpha_t * (m * m * (p - y) - 2.0f * m * bce_term(x, y) * dpt);
}

}  // namespace srb
