// Element updates shared by the multi-tensor optimizer (multi_tensor.cu) and the fused optimizer tail
// (comm/fused_step.cu): both must train bit for bit alike.
#pragma once
#include "../common.cuh"

namespace ub {

// Adam(W) on one element: m, v are the moments; `h` is an AdamHyper or any type with its fields (the fused tail reads
// them from its parameter group in place).  step_size = lr * sqrt(1-b2^t)/(1-b1^t), decay_mul = 1 - step_size * wd.
// Every fused multiply-add is spelled out: left to contraction, the compiler fused v = b2 v + (1-b2) g g one way in the
// vectorised loop of multi_tensor.cu and the other way in its scalar loop and in the fused tail, so the three paths
// rounded v differently.  The forms below are the ones the vectorised loop had.
struct AdamHyper {
  float beta1, beta2, eps, step_size, decay_mul;
};
template <typename Hyper>
UB_DEVICE void adam_math(float& p, float& m, float& v, float g, const Hyper& h) {
  m = fmaf(m, h.beta1, (1.f - h.beta1) * g);
  v = fmaf(g, (1.f - h.beta2) * g, h.beta2 * v);
  p = fmaf(p, h.decay_mul, -(h.step_size * (m / (sqrtf(v) + h.eps))));
}

// bf16 bits of x stochastically rounded with 16 random bits
UB_DEVICE uint16_t bf16_sr_bits(float x, uint32_t rnd16) {
  uint32_t bits = __float_as_uint(x);
  // leave inf/nan untouched; otherwise add 16 random low bits and truncate
  if ((bits & 0x7f800000u) != 0x7f800000u) bits += rnd16;
  return (uint16_t)(bits >> 16);
}

// exponential moving average of the parameter p, one_minus = 1 - decay
UB_DEVICE float ema_step(float e, float p, float one_minus) { return fmaf(e - p, -one_minus, e); }

}  // namespace ub
