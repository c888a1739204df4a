// LAMB (You et al., 2019) on fp32 master weights for bf16 / f16 parameters (optim.py's
// MasterWeightLAMB): apex FusedLAMB's algorithm in its defaults (adam_w_mode, bias correction,
// grad_averaging, use_nvlamb=False), bit for bit with this torch loop on the masters W, M exp_avg,
// V exp_avg_sq and G the fp32 master.grad, for the parameters of one param group that share a step:
//
//   _foreach_lerp_(M, G, 1 - beta1)                       lerp(): one FMA per branch
//   _foreach_mul_(V, beta2); _foreach_addcmul_(V, G, G, 1 - beta2)    second_moment()
//   D = _foreach_sqrt(V) / bc2_sqrt + eps                 sqrt, true division, add: three roundings
//   U = M / bc1 / D                                       two true divisions
//   U = U + wd * W                 (wd != 0)              _foreach_add_(alpha=wd): one FMA
//   c = where(|W| > 0 & |U| > 0, |W| / |U|, 1) * lr  (wd != 0; |.| = _foreach_norm, W before the step)
//   c = lr                         (wd == 0: no trust ratio, FusedLAMB's use_nvlamb=False)
//   W = W - U * c                                         two roundings: U*c, then the subtraction
//   param = half(W)                                       round to nearest even
//
// The roundings of lerp, addcmul, the scalar-list division and sqrt are the ones optim.cu's Adam
// kernel pins (tools/foreach_adam_probe.py); the alpha add is one FMA (tools/foreach_fma_probe.py).
// bc1 = 1 - beta1^step and bc2_sqrt = (1 - beta2^step)^0.5 are computed in double, as torch's Adam
// computes them in Python, and rounded to float once, as ATen rounds a scalar list.  The ratio and
// `* lr` are 0-d fp32 tensor ops: one true division, one multiply by float(lr).
//
// Two launches over the table, one 512-thread CTA per TOK_NORM_CHUNK (65,536) elements of a segment,
// _foreach_norm's geometry:
//
//   1. lamb_moments_kernel reads g, w, m and v, writes m and v, and forms u in registers.  When wd != 0
//      it also accumulates the chunk's sums of w^2 and u^2 exactly as LpNormFunctor accumulates an fp32
//      tensor (grad_norm.cu's header comment): the float4 mapping when numel % 4 == 0, the strided
//      scalar mapping otherwise, in storage order (the masters and moments are dense, so channels_last
//      tensors are taken as torch's multi_tensor_apply takes them), and the same block tree.  It
//      writes the two partials of every chunk to caller scratch.
//   2. lamb_apply_kernel: every CTA of a segment first runs lpnorm_cleanup over that segment's
//      partials (cleanup_sum and a correctly rounded sqrt, as norm_finish_kernel), so each derives the
//      same c without a third launch or a coefficient buffer.  Then it recomputes u from the new m and
//      v and the unchanged w with the same inline function, lamb_update, and writes w and param.  It
//      reads no gradient, so it has no clip or unscale variants.
//
// Per bf16 element that is 22 bytes for the first kernel and 18 for the second.  Storing u instead of
// recomputing it would move the same bytes and need numel fp32 of scratch.
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

constexpr int64_t kLambChunk = TOK_NORM_CHUNK;   // _foreach_norm's chunk
constexpr int kLambIlp = 4;                      // ATen's kILP: accumulators per thread
static_assert(kLambChunk % (kLambIlp * kNormThreads) == 0, "a chunk is whole strided rounds");

struct LambArgs {
  const tok_lamb_segment_t* seg;
  int count;
  int64_t chunks;
  float* partials;   // [0, chunks): sums of w^2 per chunk; [chunks, 2 chunks): sums of u^2
  float lr;          // float(lr)
  float lerp_w;      // float(1 - beta1)
  float beta2;       // float(beta2)
  float sq_value;    // float(1 - beta2)
  float bc1;         // float(1 - beta1^step)
  float bc2_sqrt;    // float((1 - beta2^step)^0.5)
  float eps;
  float wd;          // float(weight_decay)
  bool use_wd;       // weight_decay != 0, decided on the double: trust ratio and decay term
};

// u from the updated moments and the master before this step: D, U and the decay term.  Both kernels
// call it, so the u whose norm kernel 1 takes is the u kernel 2 applies.
__device__ __forceinline__ float lamb_update(const LambArgs& a, float m, float v, float w) {
  const float d = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), a.bc2_sqrt), a.eps);
  const float u = __fdiv_rn(__fdiv_rn(m, a.bc1), d);
  return a.use_wd ? __fmaf_rn(a.wd, w, u) : u;
}

template <typename T, bool kClip, bool kUnscale>
__global__ void __launch_bounds__(kNormThreads)
    lamb_moments_kernel(const LambArgs a, const float* __restrict__ inv_scale,
                        const float* __restrict__ grad_coef) {
  __shared__ tok_lamb_segment_t s;
  __shared__ float red[32];
  const int64_t c = blockIdx.x;
  find_segment(a.seg, a.count, c, s);
  const float inv = kUnscale ? __ldg(inv_scale) : 1.0f;
  const float coef = kClip ? __ldg(grad_coef) : 1.0f;
  const int64_t start = (c - s.chunk0) * kLambChunk;
  const int64_t n = min(s.numel - start, kLambChunk);   // this chunk's elements
  const uint16_t* gp = (const uint16_t*)s.grad + start;
  const float* wp = s.master + start;
  float* mp = s.exp_avg + start;
  float* vp = s.exp_avg_sq + start;
  float wacc[kLambIlp] = {0.0f, 0.0f, 0.0f, 0.0f}, uacc[kLambIlp] = {0.0f, 0.0f, 0.0f, 0.0f};
  if (s.numel % kLambIlp == 0) {
    // LpNormFunctor's vector path: group q (elements 4q .. 4q+3) belongs to thread q % 512, and
    // accumulator k takes lane k
    const int64_t groups = n / kLambIlp;
    const bool gvec = ((uintptr_t)gp & 7u) == 0;
    const bool vec = aligned16(wp) && aligned16(mp) && aligned16(vp);
    for (int64_t q = threadIdx.x; q < groups; q += kNormThreads) {
      const int64_t i = kLambIlp * q;
      uint16_t gb[kLambIlp];
      if (gvec) {
        const uint2 r = __ldg((const uint2*)(gp + i));
        gb[0] = (uint16_t)(r.x & 0xffffu);
        gb[1] = (uint16_t)(r.x >> 16);
        gb[2] = (uint16_t)(r.y & 0xffffu);
        gb[3] = (uint16_t)(r.y >> 16);
      } else {
#pragma unroll
        for (int k = 0; k < kLambIlp; ++k) gb[k] = __ldg(gp + i + k);
      }
      float w[kLambIlp], m[kLambIlp], v[kLambIlp];
      if (vec) {
        const float4 w4 = __ldg((const float4*)(wp + i)), m4 = *(const float4*)(mp + i),
                     v4 = *(const float4*)(vp + i);
        w[0] = w4.x; w[1] = w4.y; w[2] = w4.z; w[3] = w4.w;
        m[0] = m4.x; m[1] = m4.y; m[2] = m4.z; m[3] = m4.w;
        v[0] = v4.x; v[1] = v4.y; v[2] = v4.z; v[3] = v4.w;
      } else {
#pragma unroll
        for (int k = 0; k < kLambIlp; ++k) {
          w[k] = wp[i + k];
          m[k] = mp[i + k];
          v[k] = vp[i + k];
        }
      }
#pragma unroll
      for (int k = 0; k < kLambIlp; ++k) {
        const float g = grad_in<T, kClip, kUnscale>(gb[k], coef, inv);
        m[k] = lerp(m[k], g, a.lerp_w);
        v[k] = second_moment(v[k], g, a.beta2, a.sq_value);
        const float u = lamb_update(a, m[k], v[k], w[k]);
        wacc[k] = __fmaf_rn(w[k], w[k], wacc[k]);
        uacc[k] = __fmaf_rn(u, u, uacc[k]);
      }
      if (vec) {
        *(float4*)(mp + i) = make_float4(m[0], m[1], m[2], m[3]);
        *(float4*)(vp + i) = make_float4(v[0], v[1], v[2], v[3]);
      } else {
#pragma unroll
        for (int k = 0; k < kLambIlp; ++k) {
          mp[i + k] = m[k];
          vp[i + k] = v[k];
        }
      }
    }
  } else {
    // LpNormFunctor's scalar path: element i0 + t + 512 * k feeds accumulator k
    for (int64_t i0 = 0; i0 < n; i0 += kLambIlp * kNormThreads) {
#pragma unroll
      for (int k = 0; k < kLambIlp; ++k) {
        const int64_t i = i0 + threadIdx.x + (int64_t)k * kNormThreads;
        if (i >= n) continue;
        const float w = wp[i];
        const float g = grad_in<T, kClip, kUnscale>(__ldg(gp + i), coef, inv);
        const float m = lerp(mp[i], g, a.lerp_w);
        const float v = second_moment(vp[i], g, a.beta2, a.sq_value);
        mp[i] = m;
        vp[i] = v;
        const float u = lamb_update(a, m, v, w);
        wacc[k] = __fmaf_rn(w, w, wacc[k]);
        uacc[k] = __fmaf_rn(u, u, uacc[k]);
      }
    }
  }
  if (!a.use_wd) return;   // no trust ratio: nothing reads the partials
  float wsum = 0.0f, usum = 0.0f;
#pragma unroll
  for (int k = 0; k < kLambIlp; ++k) {
    wsum = __fadd_rn(wsum, wacc[k]);
    usum = __fadd_rn(usum, uacc[k]);
  }
  wsum = block_sum(wsum, red);
  usum = block_sum(usum, red);
  if (threadIdx.x == 0) {
    a.partials[c] = wsum;
    a.partials[a.chunks + c] = usum;
  }
}

template <typename T>
__global__ void __launch_bounds__(kNormThreads) lamb_apply_kernel(const LambArgs a) {
  __shared__ tok_lamb_segment_t s;
  __shared__ float red[32];
  __shared__ float ratio_lr;
  const int64_t c = blockIdx.x;
  find_segment(a.seg, a.count, c, s);
  float lr_c = a.lr;   // `* lr`, or with the trust ratio `where(...) * lr`
  if (a.use_wd) {
    const int64_t nchunks = (s.numel + kLambChunk - 1) / kLambChunk;
    const float wsq = cleanup_sum(a.partials + s.chunk0, nchunks, red);
    const float usq = cleanup_sum(a.partials + a.chunks + s.chunk0, nchunks, red);
    if (threadIdx.x == 0) {
      const float wn = __fsqrt_rn(wsq), un = __fsqrt_rn(usq);
      ratio_lr = __fmul_rn((wn > 0.0f && un > 0.0f) ? __fdiv_rn(wn, un) : 1.0f, a.lr);
    }
    __syncthreads();
    lr_c = ratio_lr;
  }
  const int64_t start = (c - s.chunk0) * kLambChunk;
  const int64_t n = min(s.numel - start, kLambChunk);
  float* wp = s.master + start;
  const float* mp = s.exp_avg + start;
  const float* vp = s.exp_avg_sq + start;
  uint16_t* pp = (uint16_t*)s.param + start;
  // 4 elements at a time where every array allows 16-byte (param: 8-byte) accesses, then the rest
  const bool vec = aligned16(wp) && aligned16(mp) && aligned16(vp) && ((uintptr_t)pp & 7u) == 0;
  const int64_t nvec = vec ? n / 4 : 0;
  for (int64_t q = threadIdx.x; q < nvec; q += kNormThreads) {
    const int64_t i = 4 * q;
    const float4 w4 = *(const float4*)(wp + i), m4 = __ldg((const float4*)(mp + i)),
                 v4 = __ldg((const float4*)(vp + i));
    const float w[4] = {w4.x, w4.y, w4.z, w4.w}, m[4] = {m4.x, m4.y, m4.z, m4.w},
                v[4] = {v4.x, v4.y, v4.z, v4.w};
    float o[4];
    uint16_t h[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      o[k] = __fsub_rn(w[k], __fmul_rn(lamb_update(a, m[k], v[k], w[k]), lr_c));
      h[k] = narrow<T>(o[k]);
    }
    *(float4*)(wp + i) = make_float4(o[0], o[1], o[2], o[3]);
    *(uint2*)(pp + i) = make_uint2(h[0] | ((uint32_t)h[1] << 16), h[2] | ((uint32_t)h[3] << 16));
  }
  for (int64_t i = 4 * nvec + threadIdx.x; i < n; i += kNormThreads) {
    const float w = wp[i];
    const float o = __fsub_rn(w, __fmul_rn(lamb_update(a, mp[i], vp[i], w), lr_c));
    wp[i] = o;
    pp[i] = narrow<T>(o);
  }
}

int launched(const char* who) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(TOK_ERR_CUDA, "%s launch: %s", who, cudaGetErrorString(e));
  return TOK_OK;
}

template <typename T>
void launch_moments(const LambArgs& a, const float* inv_scale, const float* grad_coef,
                    cudaStream_t st) {
  const unsigned grid = (unsigned)a.chunks;
  if (inv_scale && grad_coef)
    lamb_moments_kernel<T, true, true><<<grid, kNormThreads, 0, st>>>(a, inv_scale, grad_coef);
  else if (inv_scale)
    lamb_moments_kernel<T, false, true><<<grid, kNormThreads, 0, st>>>(a, inv_scale, grad_coef);
  else if (grad_coef)
    lamb_moments_kernel<T, true, false><<<grid, kNormThreads, 0, st>>>(a, inv_scale, grad_coef);
  else
    lamb_moments_kernel<T, false, false><<<grid, kNormThreads, 0, st>>>(a, inv_scale, grad_coef);
  lamb_apply_kernel<T><<<grid, kNormThreads, 0, st>>>(a);
}

}  // namespace
}  // namespace tok

using namespace tok;

extern "C" int tok_lamb_master_step(const tok_lamb_segment_t* segments, int count, int64_t chunks,
                                    int dtype, double lr, double beta1, double beta2, double eps,
                                    double weight_decay, double step, float* partials,
                                    const float* inv_scale, const float* grad_coef,
                                    void* cuda_stream) {
  const char* who = "tok_lamb_master_step";
  if (!segments) return fail(TOK_ERR_INVALID, "%s: null segment table", who);
  if (count <= 0 || chunks < 0 || chunks > 0x7fffffffLL)
    return fail(TOK_ERR_INVALID, "%s: %d segments in %lld chunks", who, count, (long long)chunks);
  if (dtype != TOK_BF16 && dtype != TOK_F16)
    return fail(TOK_ERR_INVALID, "%s: parameters must be bf16 or f16 (dtype %d)", who, dtype);
  if (!(lr >= 0.0) || !isfinite(lr)) return fail(TOK_ERR_INVALID, "%s: lr %g", who, lr);
  if (!(beta1 >= 0.0 && beta1 < 1.0))
    return fail(TOK_ERR_INVALID, "%s: beta1 %g outside [0, 1)", who, beta1);
  if (!(beta2 >= 0.0 && beta2 < 1.0))
    return fail(TOK_ERR_INVALID, "%s: beta2 %g outside [0, 1)", who, beta2);
  if (!(eps >= 0.0) || !isfinite(eps)) return fail(TOK_ERR_INVALID, "%s: eps %g", who, eps);
  if (!(weight_decay >= 0.0) || !isfinite(weight_decay))
    return fail(TOK_ERR_INVALID, "%s: weight_decay %g", who, weight_decay);
  if (!(step >= 1.0) || !isfinite(step)) return fail(TOK_ERR_INVALID, "%s: step %g", who, step);
  if (chunks > 0 && !partials) return fail(TOK_ERR_INVALID, "%s: null partials", who);
  if (!device_ready()) return fail(TOK_ERR_NO_DEVICE, "%s needs a CUDA GPU (no CPU fallback)", who);
  if (chunks == 0) return TOK_OK;
  LambArgs a{};
  a.seg = segments;
  a.count = count;
  a.chunks = chunks;
  a.partials = partials;
  a.lr = (float)lr;
  a.lerp_w = (float)(1.0 - beta1);
  a.beta2 = (float)beta2;
  a.sq_value = (float)(1.0 - beta2);
  // torch's Python, in double: 1 - beta1 ** step and (1 - beta2 ** step) ** 0.5 (libm's pow)
  a.bc1 = (float)(1.0 - pow(beta1, step));
  a.bc2_sqrt = (float)pow(1.0 - pow(beta2, step), 0.5);
  a.eps = (float)eps;
  a.wd = (float)weight_decay;
  a.use_wd = weight_decay != 0.0;
  const cudaStream_t st = (cudaStream_t)cuda_stream;
  if (dtype == TOK_BF16)
    launch_moments<__nv_bfloat16>(a, inv_scale, grad_coef, st);
  else
    launch_moments<__half>(a, inv_scale, grad_coef, st);
  return launched(who);
}
