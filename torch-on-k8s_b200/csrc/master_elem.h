// Per-element pieces of the fp32 master-weight steps, shared by SGD / Adam (optim.cu), LAMB (lamb.cu)
// and LARS (lars.cu): the half-precision conversions, the gradient as the optimizer reads it, the
// roundings of torch's Adam moment update and torch's SGD element step.  optim.cu's header comment
// says how each rounding was settled.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace tok {
namespace {

template <typename T> __device__ __forceinline__ float widen(uint16_t bits);
template <> __device__ __forceinline__ float widen<__nv_bfloat16>(uint16_t bits) {
  return __uint_as_float((uint32_t)bits << 16);
}
template <> __device__ __forceinline__ float widen<__half>(uint16_t bits) {
  return __half2float(__ushort_as_half(bits));
}

template <typename T> __device__ __forceinline__ uint16_t narrow(float v);
template <> __device__ __forceinline__ uint16_t narrow<__nv_bfloat16>(float v) {
  return __bfloat16_as_ushort(__float2bfloat16_rn(v));   // what c10::BFloat16(float) does on sm_80+
}
template <> __device__ __forceinline__ uint16_t narrow<__half>(float v) {
  return __half_as_ushort(__float2half_rn(v));
}

// The gradient element as the optimizer reads it: f32(grad); with kUnscale that times the inverse loss
// scale, rounded once, as GradScaler.unscale_ stores master.grad; with kClip that times the clip
// coefficient, rounded once, as torch's clip_grad_norm_ multiplies master.grad (_foreach_mul_) before
// the optimizer step reads it.
template <typename T, bool kClip, bool kUnscale>
__device__ __forceinline__ float grad_in(uint16_t bits, float coef, float inv_scale) {
  const float g = kUnscale ? __fmul_rn(widen<T>(bits), inv_scale) : widen<T>(bits);
  return kClip ? __fmul_rn(g, coef) : g;
}

// at::native::lerp: |w| < 0.5 ? m + w*(g-m) : g - (g-m)*(1-w), each branch one FMA (the probe).
__device__ __forceinline__ float lerp(float m, float g, float w) {
  const float d = __fsub_rn(g, m);
  return fabsf(w) < 0.5f ? __fmaf_rn(w, d, m) : __fmaf_rn(-d, __fsub_rn(1.0f, w), g);
}

// _foreach_mul_(v, beta2) then _foreach_addcmul_(v, g, g, value): fma(value, g*g, v), or fma(g, g, v)
// when value == 1 (ATen's pointwise_op_impl).
__device__ __forceinline__ float second_moment(float v, float g, float beta2, float value) {
  v = __fmul_rn(v, beta2);
  return value == 1.0f ? __fmaf_rn(g, g, v) : __fmaf_rn(value, __fmul_rn(g, g), v);
}

__device__ __forceinline__ float add_alpha(float a, float b, float alpha) {
  return __fmaf_rn(alpha, b, a);   // a + alpha * b, one rounding (optim.cu's header comment)
}

// torch.optim.SGD's foreach step on one element of the masters: returns the new master w and updates
// the momentum buffer m in place (m is neither read nor written without use_mu, nor read when fresh).
__device__ __forceinline__ float sgd_update(float g, float w, float& m, float neg_lr, float mu,
                                            float damp_alpha, float wd, bool use_wd, bool use_mu,
                                            bool nesterov, bool fresh) {
  if (use_wd) g = add_alpha(g, w, wd);
  if (use_mu) {
    m = fresh ? g : add_alpha(__fmul_rn(m, mu), g, damp_alpha);
    g = nesterov ? add_alpha(g, m, mu) : m;
  }
  return add_alpha(w, g, neg_lr);
}

__device__ __forceinline__ bool aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

}  // namespace
}  // namespace tok
