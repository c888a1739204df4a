// Optimizer steps on fp32 master weights for bf16 / f16 parameters, one launch per gradient bucket:
// SGD (sgd_master_kernel) and Adam / AdamW (adam_master_kernel).
//
// SGD.  For every element of every segment (one parameter: its gradient inside the bucket, the half-
// precision parameter, the fp32 master w and the fp32 momentum buffer m) the kernel evaluates what
// torch.optim.SGD's foreach path evaluates on the masters, followed by param.copy_(master):
//
//   g = f32(grad)
//   g = g + wd * w                              _foreach_add(grads, params, alpha=wd)   (wd != 0)
//   m = g                                       clone                                   (first step)
//   m = m * mu;  m = m + (1 - dampening) * g    _foreach_mul_, _foreach_add_(alpha)     (later steps)
//   g = g + mu * m   (nesterov)  or  g = m      _foreach_add_(alpha=mu)
//   w = w + (-lr) * g                           _foreach_add_(params, grads, alpha=-lr)
//   param = half(w)                             round to nearest even
//
// Every _foreach_* call rounds its result to fp32, and so does this kernel.  ATen's alpha functor
// computes `a + alpha * b` in float; built with nvcc's default contraction, it is one FMA.  That was
// settled on an H100 by tools/foreach_fma_probe.py (profiles/h100_foreach_fma_probe.json): on 2^24
// random fp32 pairs for each of 4 alphas, _foreach_add_ matched the singly rounded a + alpha*b in
// every element and differed from the separately rounded multiply and add in 6.7 M of them.  add_alpha pins it with __fmaf_rn so no compiler choice can
// change it.  The hyperparameters arrive as the floats ATen's Scalar conversion produces (the host
// rounds the double values, 1 - dampening included, once).
//
// Adam / AdamW.  Per element, with w the master, m exp_avg, v exp_avg_sq and vmax max_exp_avg_sq, the
// kernel evaluates torch.optim.Adam's _multi_tensor_adam on the masters, then param.copy_(master):
//
//   g = f32(grad)
//   g = g + wd * w              _foreach_add(grads, params, alpha=wd)     (Adam, wd != 0)   one FMA
//   w = w * decay               _foreach_mul_(params, 1 - lr * wd)        (AdamW, wd != 0)
//   m = lerp(m, g, 1 - beta1)   _foreach_lerp_                            see lerp() below
//   v = v * beta2               _foreach_mul_
//   v = v + value * (g * g)     _foreach_addcmul_(v, g, g, 1 - beta2)     fma(value, g*g, v), or
//                                                                         fma(g, g, v) if value == 1
//   vmax = maximum(vmax, v)     _foreach_maximum_                         (amsgrad) NaN propagates
//   d = sqrt(amsgrad ? vmax : v) / bc2_sqrt + eps                         three roundings
//   w = w + step_size * (m / d) _foreach_addcdiv_                         fma(s, m/d, w)
//   param = half(w)
//
// The host computes bc1 = 1 - beta1^step, step_size = (lr / bc1) * -1, bc2_sqrt = (1 - beta2^step)^0.5
// and decay = 1 - lr * wd in double with libm's pow, as torch's Python does, and rounds each to float
// once.  How ATen rounds each op on CUDA fp32 was settled on an H100 by tools/foreach_adam_probe.py
// (profiles/h100_foreach_adam_probe.json), 2^24 random elements per case, torch 2.11: lerp is one FMA
// per branch (0 mismatches against the FMA form, 1.2-3.4 M against a multiply and an add); addcmul and
// addcdiv are the FMAs of ATen's pointwise_op_impl (0 against them, 1.2-2.0 M against a multiply and an
// add); the division by the bias-correction scalar list is a true division (0 against it, 1.0-5.6 M
// against a multiply by the reciprocal); sqrt is correctly rounded; maximum propagates NaN from either
// operand (335 k mismatches against fmaxf).  Every rounding below is pinned with an intrinsic.
//
// Clipped steps (tok_*_master_step_clipped) are the same kernels instantiated with kClip: the first
// operation on every gradient element is g = f32(grad) * coef, one rounding, with coef the 0-d fp32
// tensor clip_grad_norm_ forms on the device (grad_norm.cu computes the norms it is formed from).  The
// unclipped instantiations compile to the SASS they had before the flag existed.
//
// Unscaled steps (tok_*_master_step_unscaled, dynamic loss scaling) add kUnscale: the first operation
// becomes g = f32(grad) * inv_scale, one rounding, as torch's _amp_foreach_non_finite_check_and_unscale_
// stores master.grad (its `inv_scale == 1 ? val : val * inv_scale` is the same bits for every value it
// does not flag as non-finite).  With a clip coefficient as well, g = g * coef follows as a second
// rounding: GradScaler.unscale_ and clip_grad_norm_ each store master.grad, and one multiply by
// inv_scale * coef would differ whenever inv_scale is not a power of two.  The plain and clipped
// instantiations compile to the SASS they had before this flag existed.
//
// Both kernels split work over (segment, chunk) pairs: block b takes chunk b of the whole table and
// finds its segment by binary search over the entries' first-chunk indices.  Inside a chunk, 8
// elements at a time go through 16-byte vector loads and stores where the parameter and every fp32
// array share an alignment phase; the gradient is a vector load when its phase agrees too (DDP does
// not pad bucket views, so it often does not), otherwise 8 scalar loads.  The chunk's unaligned head
// and tail are scalar.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "master_elem.h"
#include "norm_reduce.h"
#include "tok_internal.h"

namespace tok {
namespace {

constexpr int kSgdThreads = 256;            // threads per CTA of both kernels
constexpr int64_t kChunk = TOK_SGD_CHUNK;   // elements per (segment, chunk) work item
static_assert(kChunk % 8 == 0, "a chunk must start at a vector boundary of every array");

__device__ __forceinline__ float lane(const float4& v, int k) {
  return k == 0 ? v.x : k == 1 ? v.y : k == 2 ? v.z : v.w;
}

__device__ __forceinline__ bool aligned16(const void* p, int64_t i, int esz) {
  return (((uintptr_t)p + (uintptr_t)(i * esz)) & 15u) == 0;
}

// 8 gradient elements from i on: one 16-byte load when the gradient is aligned there, else 8.
__device__ __forceinline__ void load_grad8(const void* grad, int64_t i, bool vec, uint16_t gb[8]) {
  if (vec) {
    const uint4 q = __ldg((const uint4*)((const uint16_t*)grad + i));
    const uint32_t w4[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      gb[2 * k] = (uint16_t)(w4[k] & 0xffffu);
      gb[2 * k + 1] = (uint16_t)(w4[k] >> 16);
    }
  } else {
#pragma unroll
    for (int k = 0; k < 8; ++k) gb[k] = __ldg((const uint16_t*)grad + i + k);
  }
}

__device__ __forceinline__ void store_param8(void* param, int64_t i, const uint16_t out[8]) {
  *(uint4*)((uint16_t*)param + i) =
      make_uint4(out[0] | ((uint32_t)out[1] << 16), out[2] | ((uint32_t)out[3] << 16),
                 out[4] | ((uint32_t)out[5] << 16), out[6] | ((uint32_t)out[7] << 16));
}

// Chunk blockIdx.x of the table in `a` (a Step: SgdArgs or AdamArgs).  Thread 0 finds the last entry
// whose first chunk is <= the block's and copies it to shared memory; then the block walks the
// chunk's elements: Step::vector for 8 at a time from the first element at which the parameter is
// 16-byte aligned, if Step::vectorizable says every fp32 array is aligned there too, and
// Step::scalar for the rest.  With kUnscale, every gradient element is multiplied by `inv_scale` (the
// inverse loss scale) before anything else reads it, and with kClip then by `coef` (the clip
// coefficient); without the flags, those arguments are unused.
template <typename T, bool kClip, bool kUnscale, typename Step>
__device__ __forceinline__ void walk_chunk(const Step& a, float coef, float inv_scale) {
  __shared__ typename Step::Segment s;
  const int64_t c = blockIdx.x;
  find_segment(a.seg, a.count, c, s);
  const int64_t start = (c - s.chunk0) * kChunk;
  const int64_t end = min(start + kChunk, s.numel);
  if (start >= end) return;
  int64_t head = ((16 - (((uintptr_t)s.param + (uintptr_t)(start * 2)) & 15u)) & 15u) / 2;
  const bool vec = ((uintptr_t)s.param & 1u) == 0 && a.vectorizable(s, start + head);
  if (!vec || head > end - start) head = end - start;
  const int64_t nvec = (end - start - head) / 8;
  const int64_t vbeg = start + head, tail = vbeg + 8 * nvec;
  const bool grad_vec = aligned16(s.grad, vbeg, 2);
  for (int64_t v = threadIdx.x; v < nvec; v += kSgdThreads)
    a.template vector<T, kClip, kUnscale>(s, vbeg + 8 * v, grad_vec, coef, inv_scale);
  const int64_t nscalar = head + (end - tail);
  for (int64_t j = threadIdx.x; j < nscalar; j += kSgdThreads)
    a.template scalar<T, kClip, kUnscale>(s, j < head ? start + j : tail + (j - head), coef,
                                          inv_scale);
}

// ---- SGD ----------------------------------------------------------------------------------------
struct SgdArgs {
  using Segment = tok_sgd_segment_t;
  const tok_sgd_segment_t* seg;
  int count;
  float neg_lr;        // float(-lr)
  float mu;            // float(momentum)
  float damp_alpha;    // float(1 - dampening)
  float wd;            // float(weight_decay)
  bool use_wd;         // weight_decay != 0 (decided on the double, as torch decides it)
  bool use_mu;         // momentum != 0
  bool nesterov;
  bool fresh;          // momentum buffers hold nothing yet: m = g

  // One element: returns the new master; updates m in place.
  __device__ __forceinline__ float step(float g, float w, float& m) const {
    return sgd_update(g, w, m, neg_lr, mu, damp_alpha, wd, use_wd, use_mu, nesterov, fresh);
  }

  __device__ __forceinline__ bool vectorizable(const tok_sgd_segment_t& s, int64_t i) const {
    return aligned16(s.master, i, 4) && (!use_mu || aligned16(s.momentum, i, 4));
  }

  template <typename T, bool kClip, bool kUnscale>
  __device__ __forceinline__ void scalar(const tok_sgd_segment_t& s, int64_t i, float coef,
                                         float inv_scale) const {
    const float g = grad_in<T, kClip, kUnscale>(__ldg((const uint16_t*)s.grad + i), coef, inv_scale);
    float m = (use_mu && !fresh) ? s.momentum[i] : 0.0f;
    const float w = step(g, s.master[i], m);
    s.master[i] = w;
    if (use_mu) s.momentum[i] = m;
    ((uint16_t*)s.param)[i] = narrow<T>(w);
  }

  template <typename T, bool kClip, bool kUnscale>
  __device__ __forceinline__ void vector(const tok_sgd_segment_t& s, int64_t i, bool grad_vec,
                                         float coef, float inv_scale) const {
    // The gradient load is load_grad8 written out: called through the helper, ptxas schedules this
    // kernel differently (46 registers instead of 48); written out, its SASS is what it was before
    // the Adam kernel shared this file.
    uint16_t gb[8];
    if (grad_vec) {
      const uint4 q = __ldg((const uint4*)((const uint16_t*)s.grad + i));
      const uint32_t w4[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        gb[2 * k] = (uint16_t)(w4[k] & 0xffffu);
        gb[2 * k + 1] = (uint16_t)(w4[k] >> 16);
      }
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) gb[k] = __ldg((const uint16_t*)s.grad + i + k);
    }
    float4* wp = (float4*)(s.master + i);
    float4* mp = (float4*)(s.momentum + i);
    const float4 w0 = wp[0], w1 = wp[1];
    float4 m0 = make_float4(0.f, 0.f, 0.f, 0.f), m1 = m0;
    if (use_mu && !fresh) {
      m0 = mp[0];
      m1 = mp[1];
    }
    float w[8], m[8];
    uint16_t out[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      m[k] = k < 4 ? lane(m0, k) : lane(m1, k - 4);
      w[k] = step(grad_in<T, kClip, kUnscale>(gb[k], coef, inv_scale),
                  k < 4 ? lane(w0, k) : lane(w1, k - 4), m[k]);
      out[k] = narrow<T>(w[k]);
    }
    wp[0] = make_float4(w[0], w[1], w[2], w[3]);
    wp[1] = make_float4(w[4], w[5], w[6], w[7]);
    if (use_mu) {
      mp[0] = make_float4(m[0], m[1], m[2], m[3]);
      mp[1] = make_float4(m[4], m[5], m[6], m[7]);
    }
    store_param8(s.param, i, out);
  }
};

template <typename T>
__global__ void __launch_bounds__(kSgdThreads) sgd_master_kernel(const SgdArgs a) {
  walk_chunk<T, false, false>(a, 1.0f, 1.0f);
}

template <typename T>
__global__ void __launch_bounds__(kSgdThreads)
    sgd_master_clipped_kernel(const SgdArgs a, const float* __restrict__ grad_coef) {
  walk_chunk<T, true, false>(a, __ldg(grad_coef), 1.0f);
}

template <typename T, bool kClip>
__global__ void __launch_bounds__(kSgdThreads)
    sgd_master_unscaled_kernel(const SgdArgs a, const float* __restrict__ inv_scale,
                               const float* __restrict__ grad_coef) {
  walk_chunk<T, kClip, true>(a, kClip ? __ldg(grad_coef) : 1.0f, __ldg(inv_scale));
}

// ---- Adam / AdamW -------------------------------------------------------------------------------
struct AdamArgs {
  using Segment = tok_adam_segment_t;
  const tok_adam_segment_t* seg;
  int count;
  float step_size;     // float((lr / (1 - beta1^step)) * -1)
  float bc2_sqrt;      // float((1 - beta2^step)^0.5)
  float eps;
  float wd;            // float(weight_decay): the L2 term (Adam)
  float decay;         // float(1 - lr * weight_decay): the decoupled decay (AdamW)
  float lerp_w;        // float(1 - beta1)
  float beta2;         // float(beta2)
  float sq_value;      // float(1 - beta2)
  bool use_wd;         // weight_decay != 0
  bool decoupled;
  bool amsgrad;

  // One element: returns the new master; updates m, v and vmax in place.  step_size <= 0 (lr >= 0), so
  // addcdiv's `s == 1` branch (w + m/d) cannot occur.
  __device__ __forceinline__ float step(float g, float w, float& m, float& v, float& vmax) const {
    if (use_wd) {
      if (decoupled) w = __fmul_rn(w, decay);
      else g = add_alpha(g, w, wd);
    }
    m = lerp(m, g, lerp_w);
    v = second_moment(v, g, beta2, sq_value);
    float d = v;
    if (amsgrad) d = vmax = (isnan(vmax) || vmax > v) ? vmax : v;   // ATen's maximum
    d = __fadd_rn(__fdiv_rn(__fsqrt_rn(d), bc2_sqrt), eps);
    return __fmaf_rn(step_size, __fdiv_rn(m, d), w);
  }

  __device__ __forceinline__ bool vectorizable(const tok_adam_segment_t& s, int64_t i) const {
    return aligned16(s.master, i, 4) && aligned16(s.exp_avg, i, 4) &&
           aligned16(s.exp_avg_sq, i, 4) && (!amsgrad || aligned16(s.max_exp_avg_sq, i, 4));
  }

  template <typename T, bool kClip, bool kUnscale>
  __device__ __forceinline__ void scalar(const tok_adam_segment_t& s, int64_t i, float coef,
                                         float inv_scale) const {
    const float g = grad_in<T, kClip, kUnscale>(__ldg((const uint16_t*)s.grad + i), coef, inv_scale);
    float m = s.exp_avg[i], v = s.exp_avg_sq[i];
    float vmax = amsgrad ? s.max_exp_avg_sq[i] : 0.0f;
    const float w = step(g, s.master[i], m, v, vmax);
    s.master[i] = w;
    s.exp_avg[i] = m;
    s.exp_avg_sq[i] = v;
    if (amsgrad) s.max_exp_avg_sq[i] = vmax;
    ((uint16_t*)s.param)[i] = narrow<T>(w);
  }

  template <typename T, bool kClip, bool kUnscale>
  __device__ __forceinline__ void vector(const tok_adam_segment_t& s, int64_t i, bool grad_vec,
                                         float coef, float inv_scale) const {
    uint16_t gb[8];
    load_grad8(s.grad, i, grad_vec, gb);
    float4* wp = (float4*)(s.master + i);
    float4* mp = (float4*)(s.exp_avg + i);
    float4* vp = (float4*)(s.exp_avg_sq + i);
    float4* xp = (float4*)(s.max_exp_avg_sq + i);
    const float4 w0 = wp[0], w1 = wp[1], m0 = mp[0], m1 = mp[1], v0 = vp[0], v1 = vp[1];
    float4 x0 = make_float4(0.f, 0.f, 0.f, 0.f), x1 = x0;
    if (amsgrad) {
      x0 = xp[0];
      x1 = xp[1];
    }
    float w[8], m[8], v[8], x[8];
    uint16_t out[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      m[k] = k < 4 ? lane(m0, k) : lane(m1, k - 4);
      v[k] = k < 4 ? lane(v0, k) : lane(v1, k - 4);
      x[k] = k < 4 ? lane(x0, k) : lane(x1, k - 4);
      w[k] = step(grad_in<T, kClip, kUnscale>(gb[k], coef, inv_scale),
                  k < 4 ? lane(w0, k) : lane(w1, k - 4), m[k], v[k], x[k]);
      out[k] = narrow<T>(w[k]);
    }
    wp[0] = make_float4(w[0], w[1], w[2], w[3]);
    wp[1] = make_float4(w[4], w[5], w[6], w[7]);
    mp[0] = make_float4(m[0], m[1], m[2], m[3]);
    mp[1] = make_float4(m[4], m[5], m[6], m[7]);
    vp[0] = make_float4(v[0], v[1], v[2], v[3]);
    vp[1] = make_float4(v[4], v[5], v[6], v[7]);
    if (amsgrad) {
      xp[0] = make_float4(x[0], x[1], x[2], x[3]);
      xp[1] = make_float4(x[4], x[5], x[6], x[7]);
    }
    store_param8(s.param, i, out);
  }
};

template <typename T>
__global__ void __launch_bounds__(kSgdThreads) adam_master_kernel(const AdamArgs a) {
  walk_chunk<T, false, false>(a, 1.0f, 1.0f);
}

template <typename T>
__global__ void __launch_bounds__(kSgdThreads)
    adam_master_clipped_kernel(const AdamArgs a, const float* __restrict__ grad_coef) {
  walk_chunk<T, true, false>(a, __ldg(grad_coef), 1.0f);
}

template <typename T, bool kClip>
__global__ void __launch_bounds__(kSgdThreads)
    adam_master_unscaled_kernel(const AdamArgs a, const float* __restrict__ inv_scale,
                                const float* __restrict__ grad_coef) {
  walk_chunk<T, kClip, true>(a, kClip ? __ldg(grad_coef) : 1.0f, __ldg(inv_scale));
}

// The table and dtype checks both entry points share; 0 when they pass.
int check_table(const char* who, const void* segments, int count, int64_t chunks, int dtype) {
  if (!segments) return fail(TOK_ERR_INVALID, "%s: null segment table", who);
  if (count <= 0 || chunks <= 0 || chunks > 0x7fffffffLL)
    return fail(TOK_ERR_INVALID, "%s: %d segments in %lld chunks", who, count, (long long)chunks);
  if (dtype != TOK_BF16 && dtype != TOK_F16)
    return fail(TOK_ERR_INVALID, "%s: parameters must be bf16 or f16 (dtype %d)", who, dtype);
  return 0;
}

int launched(const char* who) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(TOK_ERR_CUDA, "%s launch: %s", who, cudaGetErrorString(e));
  return TOK_OK;
}

// The SGD entry points: checks, the float hyperparameters, and one launch of the plain kernel, with a
// coefficient the clipped one, or with `unscale` the unscaled one (clipped too when grad_coef is set).
int sgd_step(const char* who, const tok_sgd_segment_t* segments, int count, int64_t chunks,
             int dtype, double lr, double momentum, double dampening, double weight_decay,
             int nesterov, int fresh, const float* grad_coef, bool clip, const float* inv_scale,
             bool unscale, void* cuda_stream) {
  if (const int rc = check_table(who, segments, count, chunks, dtype)) return rc;
  if (!(lr >= 0.0) || !isfinite(lr)) return fail(TOK_ERR_INVALID, "%s: lr %g", who, lr);
  if (!(momentum >= 0.0) || !isfinite(momentum))
    return fail(TOK_ERR_INVALID, "%s: momentum %g", who, momentum);
  if (!isfinite(dampening)) return fail(TOK_ERR_INVALID, "%s: dampening %g", who, dampening);
  if (!(weight_decay >= 0.0) || !isfinite(weight_decay))
    return fail(TOK_ERR_INVALID, "%s: weight_decay %g", who, weight_decay);
  if (nesterov && (momentum <= 0.0 || dampening != 0.0))
    return fail(TOK_ERR_INVALID, "%s: nesterov needs a momentum and zero dampening", who);
  if (clip && !grad_coef) return fail(TOK_ERR_INVALID, "%s: null grad_coef", who);
  if (unscale && !inv_scale) return fail(TOK_ERR_INVALID, "%s: null inv_scale", who);
  if (!device_ready()) return fail(TOK_ERR_NO_DEVICE, "%s needs a CUDA GPU (no CPU fallback)", who);
  SgdArgs a{};
  a.seg = segments;
  a.count = count;
  a.neg_lr = (float)(-lr);
  a.mu = (float)momentum;
  a.damp_alpha = (float)(1.0 - dampening);
  a.wd = (float)weight_decay;
  a.use_wd = weight_decay != 0.0;
  a.use_mu = momentum != 0.0;
  a.nesterov = nesterov != 0;
  a.fresh = fresh != 0;
  const dim3 grid((unsigned)chunks);
  const cudaStream_t st = (cudaStream_t)cuda_stream;
  if (unscale) {
    if (dtype == TOK_BF16 && grad_coef)
      sgd_master_unscaled_kernel<__nv_bfloat16, true><<<grid, kSgdThreads, 0, st>>>(a, inv_scale,
                                                                                   grad_coef);
    else if (dtype == TOK_BF16)
      sgd_master_unscaled_kernel<__nv_bfloat16, false><<<grid, kSgdThreads, 0, st>>>(a, inv_scale,
                                                                                    grad_coef);
    else if (grad_coef)
      sgd_master_unscaled_kernel<__half, true><<<grid, kSgdThreads, 0, st>>>(a, inv_scale, grad_coef);
    else
      sgd_master_unscaled_kernel<__half, false><<<grid, kSgdThreads, 0, st>>>(a, inv_scale,
                                                                             grad_coef);
  } else if (clip) {
    if (dtype == TOK_BF16)
      sgd_master_clipped_kernel<__nv_bfloat16><<<grid, kSgdThreads, 0, st>>>(a, grad_coef);
    else
      sgd_master_clipped_kernel<__half><<<grid, kSgdThreads, 0, st>>>(a, grad_coef);
  } else if (dtype == TOK_BF16) {
    sgd_master_kernel<__nv_bfloat16><<<grid, kSgdThreads, 0, st>>>(a);
  } else {
    sgd_master_kernel<__half><<<grid, kSgdThreads, 0, st>>>(a);
  }
  return launched(who);
}

// The Adam entry points, likewise.
int adam_step(const char* who, const tok_adam_segment_t* segments, int count, int64_t chunks,
              int dtype, double lr, double beta1, double beta2, double eps, double weight_decay,
              int decoupled, int amsgrad, double step, const float* grad_coef, bool clip,
              const float* inv_scale, bool unscale, void* cuda_stream) {
  if (const int rc = check_table(who, segments, count, chunks, dtype)) return rc;
  if (!(lr >= 0.0) || !isfinite(lr)) return fail(TOK_ERR_INVALID, "%s: lr %g", who, lr);
  if (!(beta1 >= 0.0 && beta1 < 1.0))
    return fail(TOK_ERR_INVALID, "%s: beta1 %g outside [0, 1)", who, beta1);
  if (!(beta2 >= 0.0 && beta2 < 1.0))
    return fail(TOK_ERR_INVALID, "%s: beta2 %g outside [0, 1)", who, beta2);
  if (!(eps >= 0.0) || !isfinite(eps)) return fail(TOK_ERR_INVALID, "%s: eps %g", who, eps);
  if (!(weight_decay >= 0.0) || !isfinite(weight_decay))
    return fail(TOK_ERR_INVALID, "%s: weight_decay %g", who, weight_decay);
  if (!(step >= 1.0) || !isfinite(step)) return fail(TOK_ERR_INVALID, "%s: step %g", who, step);
  if (clip && !grad_coef) return fail(TOK_ERR_INVALID, "%s: null grad_coef", who);
  if (unscale && !inv_scale) return fail(TOK_ERR_INVALID, "%s: null inv_scale", who);
  if (!device_ready()) return fail(TOK_ERR_NO_DEVICE, "%s needs a CUDA GPU (no CPU fallback)", who);
  // torch's Python, in double: bias_correction1 = 1 - beta1 ** step; step_size = (lr / bc1) * -1;
  // bias_correction2_sqrt = (1 - beta2 ** step) ** 0.5 — CPython's float ** is libm's pow
  const double bc1 = 1.0 - pow(beta1, step);
  AdamArgs a{};
  a.seg = segments;
  a.count = count;
  a.step_size = (float)((lr / bc1) * -1.0);
  a.bc2_sqrt = (float)pow(1.0 - pow(beta2, step), 0.5);
  a.eps = (float)eps;
  a.wd = (float)weight_decay;
  a.decay = (float)(1.0 - lr * weight_decay);
  a.lerp_w = (float)(1.0 - beta1);
  a.beta2 = (float)beta2;
  a.sq_value = (float)(1.0 - beta2);
  a.use_wd = weight_decay != 0.0;
  a.decoupled = decoupled != 0;
  a.amsgrad = amsgrad != 0;
  const dim3 grid((unsigned)chunks);
  const cudaStream_t st = (cudaStream_t)cuda_stream;
  if (unscale) {
    if (dtype == TOK_BF16 && grad_coef)
      adam_master_unscaled_kernel<__nv_bfloat16, true><<<grid, kSgdThreads, 0, st>>>(a, inv_scale,
                                                                                    grad_coef);
    else if (dtype == TOK_BF16)
      adam_master_unscaled_kernel<__nv_bfloat16, false><<<grid, kSgdThreads, 0, st>>>(a, inv_scale,
                                                                                     grad_coef);
    else if (grad_coef)
      adam_master_unscaled_kernel<__half, true><<<grid, kSgdThreads, 0, st>>>(a, inv_scale,
                                                                             grad_coef);
    else
      adam_master_unscaled_kernel<__half, false><<<grid, kSgdThreads, 0, st>>>(a, inv_scale,
                                                                              grad_coef);
  } else if (clip) {
    if (dtype == TOK_BF16)
      adam_master_clipped_kernel<__nv_bfloat16><<<grid, kSgdThreads, 0, st>>>(a, grad_coef);
    else
      adam_master_clipped_kernel<__half><<<grid, kSgdThreads, 0, st>>>(a, grad_coef);
  } else if (dtype == TOK_BF16) {
    adam_master_kernel<__nv_bfloat16><<<grid, kSgdThreads, 0, st>>>(a);
  } else {
    adam_master_kernel<__half><<<grid, kSgdThreads, 0, st>>>(a);
  }
  return launched(who);
}

}  // namespace
}  // namespace tok

using namespace tok;

extern "C" int tok_sgd_master_step(const tok_sgd_segment_t* segments, int count, int64_t chunks,
                                   int dtype, double lr, double momentum, double dampening,
                                   double weight_decay, int nesterov, int fresh,
                                   void* cuda_stream) {
  return sgd_step("tok_sgd_master_step", segments, count, chunks, dtype, lr, momentum, dampening,
                  weight_decay, nesterov, fresh, nullptr, false, nullptr, false, cuda_stream);
}

extern "C" int tok_sgd_master_step_clipped(const tok_sgd_segment_t* segments, int count,
                                           int64_t chunks, int dtype, double lr, double momentum,
                                           double dampening, double weight_decay, int nesterov,
                                           int fresh, const float* grad_coef, void* cuda_stream) {
  return sgd_step("tok_sgd_master_step_clipped", segments, count, chunks, dtype, lr, momentum,
                  dampening, weight_decay, nesterov, fresh, grad_coef, true, nullptr, false,
                  cuda_stream);
}

extern "C" int tok_sgd_master_step_unscaled(const tok_sgd_segment_t* segments, int count,
                                            int64_t chunks, int dtype, double lr, double momentum,
                                            double dampening, double weight_decay, int nesterov,
                                            int fresh, const float* inv_scale,
                                            const float* grad_coef, void* cuda_stream) {
  return sgd_step("tok_sgd_master_step_unscaled", segments, count, chunks, dtype, lr, momentum,
                  dampening, weight_decay, nesterov, fresh, grad_coef, false, inv_scale, true,
                  cuda_stream);
}

extern "C" int tok_adam_master_step(const tok_adam_segment_t* segments, int count, int64_t chunks,
                                    int dtype, double lr, double beta1, double beta2, double eps,
                                    double weight_decay, int decoupled, int amsgrad, double step,
                                    void* cuda_stream) {
  return adam_step("tok_adam_master_step", segments, count, chunks, dtype, lr, beta1, beta2, eps,
                   weight_decay, decoupled, amsgrad, step, nullptr, false, nullptr, false,
                   cuda_stream);
}

extern "C" int tok_adam_master_step_clipped(const tok_adam_segment_t* segments, int count,
                                            int64_t chunks, int dtype, double lr, double beta1,
                                            double beta2, double eps, double weight_decay,
                                            int decoupled, int amsgrad, double step,
                                            const float* grad_coef, void* cuda_stream) {
  return adam_step("tok_adam_master_step_clipped", segments, count, chunks, dtype, lr, beta1,
                   beta2, eps, weight_decay, decoupled, amsgrad, step, grad_coef, true, nullptr,
                   false, cuda_stream);
}

extern "C" int tok_adam_master_step_unscaled(const tok_adam_segment_t* segments, int count,
                                             int64_t chunks, int dtype, double lr, double beta1,
                                             double beta2, double eps, double weight_decay,
                                             int decoupled, int amsgrad, double step,
                                             const float* inv_scale, const float* grad_coef,
                                             void* cuda_stream) {
  return adam_step("tok_adam_master_step_unscaled", segments, count, chunks, dtype, lr, beta1,
                   beta2, eps, weight_decay, decoupled, amsgrad, step, grad_coef, false, inv_scale,
                   true, cuda_stream);
}
