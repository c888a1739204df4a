// LARS (You et al., 2017) on fp32 master weights for bf16 / f16 parameters (optim.py's
// MasterWeightLARS): apex LARC's algorithm, in its clip and scale modes, around torch.optim.SGD, bit
// for bit with this torch loop on the masters W, momentum buffers B and G the fp32 master.grad, for the
// parameters of one param group that share a momentum state:
//
//   wn, gn = _foreach_norm(W), _foreach_norm(G)         W before this step's update
//   r = tc * wn / (gn + wn * wd + eps)                  tc*wn, wn*wd: fp32 multiplies by float(scalar);
//                                                       two fp32 adds; one true division
//   r = clamp(r / lr, max=1)         (clip)             r * float(1.0 / lr): ATen's division by a
//                                                       CPU scalar; clamp keeps NaN, so not fminf
//   g = where(wn != 0 & gn != 0, (g + wd * w) * r, g)   three roundings: wd*w, the add, the multiply
//   SGD(W, lr, momentum, dampening, weight_decay=0, nesterov).step()      sgd_update(), use_wd false
//   param = half(W)                                     round to nearest even
//
// The ratio's roundings are those ATen gives 0-d fp32 CUDA tensors and Python scalars: a tensor times a
// Python float is one multiply by the float; `r / lr` with a Python float is div_true_kernel_cuda's
// multiply by the reciprocal, which the host takes in double and rounds to float once.  That was
// settled on an H100 by tools/scalar_div_probe.py (profiles/h100_scalar_div_probe.txt): over 4,000
// ratios at each of 5 learning rates, r * float(1.0 / lr) matched torch in every one, while
// r * (1.0f / float(lr)) missed up to 3,989 and r / float(lr) up to 3,020.  The reciprocal is inf at
// lr = 0, so a clipped ratio of a non-zero tensor is 1 there.  The decay term is always evaluated,
// also at wd = 0: g + 0 * w turns g = -0 into +0 and w = +-inf into NaN, as the torch expression does.  The SGD part is optim.cu's SGD
// element step without weight decay.
//
// Two launches over the table, one 512-thread CTA per TOK_NORM_CHUNK (65,536) elements of a segment,
// _foreach_norm's geometry:
//
//   1. lars_norms_kernel reads g through grad_in (unscaled and clipped as the other steps read it) and
//      w, and accumulates each chunk's sums of w^2 and g^2 as LpNormFunctor accumulates an fp32 tensor
//      (grad_norm.cu's header comment): the float4 mapping when numel % 4 == 0, the strided scalar
//      mapping otherwise, in storage order, so the gradient's norm is its fp32 copy's wherever the
//      bf16 view sits, and the dense master's is lamb.cu's.  It writes both partials of every chunk.
//   2. lars_apply_kernel: every CTA of a segment runs lpnorm_cleanup over that segment's partials
//      (cleanup_sum and a correctly rounded sqrt), so each derives the same wn, gn and r without a third
//      launch.  Then it reads g again through the same grad_in, applies the transform and the SGD step
//      and writes w, the momentum and param, 4 elements at a time where the master, momentum and
//      parameter allow 16-byte (parameter: 8-byte) accesses, the rest one at a time.
//
// Per bf16 element that is 6 bytes for the first kernel and 20 (10 read, 10 written) for the second.
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

constexpr int64_t kLarsChunk = TOK_NORM_CHUNK;   // _foreach_norm's chunk
constexpr int kLarsIlp = 4;                      // ATen's kILP: accumulators per thread
static_assert(kLarsChunk % (kLarsIlp * kNormThreads) == 0, "a chunk is whole strided rounds");

struct LarsArgs {
  const tok_lars_segment_t* seg;
  int count;
  int64_t chunks;
  float* partials;    // [0, chunks): sums of w^2 per chunk; [chunks, 2 chunks): sums of g^2
  float neg_lr;       // float(-lr)
  float inv_lr;       // float(1.0 / lr)
  float mu;           // float(momentum)
  float damp_alpha;   // float(1 - dampening)
  float tc;           // float(trust_coefficient)
  float wd;           // float(weight_decay)
  float eps;          // float(eps)
  bool use_mu;        // momentum != 0
  bool nesterov;
  bool fresh;         // momentum buffers hold nothing yet: m = g
  bool clip;          // LARC's clip mode: min(r / lr, 1)
};

// The trust ratio from the two squared norms, in thread 0; `apply` is LARC's zero-norm guard.
__device__ __forceinline__ float lars_ratio(const LarsArgs& a, float wsq, float gsq, bool& apply) {
  const float wn = __fsqrt_rn(wsq), gn = __fsqrt_rn(gsq);
  apply = wn != 0.0f && gn != 0.0f;   // NaN norms pass, as (a != 0) & (b != 0) lets them
  float r = __fdiv_rn(__fmul_rn(wn, a.tc), __fadd_rn(__fadd_rn(gn, __fmul_rn(wn, a.wd)), a.eps));
  if (a.clip) {
    r = __fmul_rn(r, a.inv_lr);
    r = isnan(r) ? r : fminf(r, 1.0f);   // ATen's clamp_max
  }
  return r;
}

// One element: LARC's gradient transform, then the SGD step; returns the new master, updates m.
__device__ __forceinline__ float lars_update(const LarsArgs& a, float g, float w, float& m,
                                             bool apply, float r) {
  if (apply) g = __fmul_rn(__fadd_rn(g, __fmul_rn(w, a.wd)), r);
  return sgd_update(g, w, m, a.neg_lr, a.mu, a.damp_alpha, 0.0f, false, a.use_mu, a.nesterov,
                    a.fresh);
}

template <typename T, bool kClip, bool kUnscale>
__global__ void __launch_bounds__(kNormThreads)
    lars_norms_kernel(const LarsArgs a, const float* __restrict__ inv_scale,
                      const float* __restrict__ grad_coef) {
  __shared__ tok_lars_segment_t s;
  __shared__ float red[32];
  const int64_t c = blockIdx.x;
  find_segment(a.seg, a.count, c, s);
  const float inv = kUnscale ? __ldg(inv_scale) : 1.0f;
  const float coef = kClip ? __ldg(grad_coef) : 1.0f;
  const int64_t start = (c - s.chunk0) * kLarsChunk;
  const int64_t n = min(s.numel - start, kLarsChunk);   // this chunk's elements
  const uint16_t* gp = (const uint16_t*)s.grad + start;
  const float* wp = s.master + start;
  float wacc[kLarsIlp] = {0.0f, 0.0f, 0.0f, 0.0f}, gacc[kLarsIlp] = {0.0f, 0.0f, 0.0f, 0.0f};
  if (s.numel % kLarsIlp == 0) {
    // LpNormFunctor's vector path: group q (elements 4q .. 4q+3) belongs to thread q % 512, and
    // accumulator k takes lane k
    const int64_t groups = n / kLarsIlp;
    const bool gvec = ((uintptr_t)gp & 7u) == 0;
    const bool wvec = aligned16(wp);
    for (int64_t q = threadIdx.x; q < groups; q += kNormThreads) {
      const int64_t i = kLarsIlp * q;
      uint16_t gb[kLarsIlp];
      if (gvec) {
        const uint2 r = __ldg((const uint2*)(gp + i));
        gb[0] = (uint16_t)(r.x & 0xffffu);
        gb[1] = (uint16_t)(r.x >> 16);
        gb[2] = (uint16_t)(r.y & 0xffffu);
        gb[3] = (uint16_t)(r.y >> 16);
      } else {
#pragma unroll
        for (int k = 0; k < kLarsIlp; ++k) gb[k] = __ldg(gp + i + k);
      }
      float w[kLarsIlp];
      if (wvec) {
        const float4 w4 = __ldg((const float4*)(wp + i));
        w[0] = w4.x; w[1] = w4.y; w[2] = w4.z; w[3] = w4.w;
      } else {
#pragma unroll
        for (int k = 0; k < kLarsIlp; ++k) w[k] = __ldg(wp + i + k);
      }
#pragma unroll
      for (int k = 0; k < kLarsIlp; ++k) {
        const float g = grad_in<T, kClip, kUnscale>(gb[k], coef, inv);
        wacc[k] = __fmaf_rn(w[k], w[k], wacc[k]);
        gacc[k] = __fmaf_rn(g, g, gacc[k]);
      }
    }
  } else {
    // LpNormFunctor's scalar path: element i0 + t + 512 * k feeds accumulator k
    for (int64_t i0 = 0; i0 < n; i0 += kLarsIlp * kNormThreads) {
#pragma unroll
      for (int k = 0; k < kLarsIlp; ++k) {
        const int64_t i = i0 + threadIdx.x + (int64_t)k * kNormThreads;
        if (i >= n) continue;
        const float w = __ldg(wp + i);
        const float g = grad_in<T, kClip, kUnscale>(__ldg(gp + i), coef, inv);
        wacc[k] = __fmaf_rn(w, w, wacc[k]);
        gacc[k] = __fmaf_rn(g, g, gacc[k]);
      }
    }
  }
  float wsum = 0.0f, gsum = 0.0f;
#pragma unroll
  for (int k = 0; k < kLarsIlp; ++k) {
    wsum = __fadd_rn(wsum, wacc[k]);
    gsum = __fadd_rn(gsum, gacc[k]);
  }
  wsum = block_sum(wsum, red);
  gsum = block_sum(gsum, red);
  if (threadIdx.x == 0) {
    a.partials[c] = wsum;
    a.partials[a.chunks + c] = gsum;
  }
}

template <typename T, bool kClip, bool kUnscale>
__global__ void __launch_bounds__(kNormThreads)
    lars_apply_kernel(const LarsArgs a, const float* __restrict__ inv_scale,
                      const float* __restrict__ grad_coef) {
  __shared__ tok_lars_segment_t s;
  __shared__ float red[32];
  __shared__ float ratio;
  __shared__ bool guard;
  const int64_t c = blockIdx.x;
  find_segment(a.seg, a.count, c, s);
  const float inv = kUnscale ? __ldg(inv_scale) : 1.0f;
  const float coef = kClip ? __ldg(grad_coef) : 1.0f;
  const int64_t nchunks = (s.numel + kLarsChunk - 1) / kLarsChunk;
  const float wsq = cleanup_sum(a.partials + s.chunk0, nchunks, red);
  const float gsq = cleanup_sum(a.partials + a.chunks + s.chunk0, nchunks, red);
  if (threadIdx.x == 0) {
    bool apply;
    ratio = lars_ratio(a, wsq, gsq, apply);
    guard = apply;
  }
  __syncthreads();
  const float r = ratio;
  const bool apply = guard;
  const int64_t start = (c - s.chunk0) * kLarsChunk;
  const int64_t n = min(s.numel - start, kLarsChunk);
  const uint16_t* gp = (const uint16_t*)s.grad + start;
  float* wp = s.master + start;
  float* mp = a.use_mu ? s.momentum + start : nullptr;
  uint16_t* pp = (uint16_t*)s.param + start;
  const bool read_m = a.use_mu && !a.fresh;
  const bool vec = aligned16(wp) && (!a.use_mu || aligned16(mp)) && ((uintptr_t)pp & 7u) == 0;
  const bool gvec = ((uintptr_t)gp & 7u) == 0;
  const int64_t nvec = vec ? n / 4 : 0;
  for (int64_t q = threadIdx.x; q < nvec; q += kNormThreads) {
    const int64_t i = 4 * q;
    uint16_t gb[4];
    if (gvec) {
      const uint2 g2 = __ldg((const uint2*)(gp + i));
      gb[0] = (uint16_t)(g2.x & 0xffffu);
      gb[1] = (uint16_t)(g2.x >> 16);
      gb[2] = (uint16_t)(g2.y & 0xffffu);
      gb[3] = (uint16_t)(g2.y >> 16);
    } else {
#pragma unroll
      for (int k = 0; k < 4; ++k) gb[k] = __ldg(gp + i + k);
    }
    const float4 w4 = *(const float4*)(wp + i);
    const float4 m4 = read_m ? *(const float4*)(mp + i) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float w[4] = {w4.x, w4.y, w4.z, w4.w};
    float m[4] = {m4.x, m4.y, m4.z, m4.w}, o[4];
    uint16_t h[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      o[k] = lars_update(a, grad_in<T, kClip, kUnscale>(gb[k], coef, inv), w[k], m[k], apply, r);
      h[k] = narrow<T>(o[k]);
    }
    *(float4*)(wp + i) = make_float4(o[0], o[1], o[2], o[3]);
    if (a.use_mu) *(float4*)(mp + i) = make_float4(m[0], m[1], m[2], m[3]);
    *(uint2*)(pp + i) = make_uint2(h[0] | ((uint32_t)h[1] << 16), h[2] | ((uint32_t)h[3] << 16));
  }
  for (int64_t i = 4 * nvec + threadIdx.x; i < n; i += kNormThreads) {
    float m = read_m ? mp[i] : 0.0f;
    const float o =
        lars_update(a, grad_in<T, kClip, kUnscale>(__ldg(gp + i), coef, inv), wp[i], m, apply, r);
    wp[i] = o;
    if (a.use_mu) mp[i] = m;
    pp[i] = narrow<T>(o);
  }
}

int launched(const char* who) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(TOK_ERR_CUDA, "%s launch: %s", who, cudaGetErrorString(e));
  return TOK_OK;
}

template <typename T, bool kClip, bool kUnscale>
void launch_pair(const LarsArgs& a, const float* inv_scale, const float* grad_coef,
                 cudaStream_t st) {
  const unsigned grid = (unsigned)a.chunks;
  lars_norms_kernel<T, kClip, kUnscale><<<grid, kNormThreads, 0, st>>>(a, inv_scale, grad_coef);
  lars_apply_kernel<T, kClip, kUnscale><<<grid, kNormThreads, 0, st>>>(a, inv_scale, grad_coef);
}

template <typename T>
void launch(const LarsArgs& a, const float* inv_scale, const float* grad_coef, cudaStream_t st) {
  if (inv_scale && grad_coef)
    launch_pair<T, true, true>(a, inv_scale, grad_coef, st);
  else if (inv_scale)
    launch_pair<T, false, true>(a, inv_scale, grad_coef, st);
  else if (grad_coef)
    launch_pair<T, true, false>(a, inv_scale, grad_coef, st);
  else
    launch_pair<T, false, false>(a, inv_scale, grad_coef, st);
}

}  // namespace
}  // namespace tok

using namespace tok;

extern "C" int tok_lars_master_step(const tok_lars_segment_t* segments, int count, int64_t chunks,
                                    int dtype, double lr, double momentum, double dampening,
                                    double weight_decay, int nesterov, int fresh,
                                    double trust_coefficient, int clip, double eps,
                                    float* partials, const float* inv_scale,
                                    const float* grad_coef, void* cuda_stream) {
  const char* who = "tok_lars_master_step";
  if (!segments) return fail(TOK_ERR_INVALID, "%s: null segment table", who);
  if (count <= 0 || chunks < 0 || chunks > 0x7fffffffLL)
    return fail(TOK_ERR_INVALID, "%s: %d segments in %lld chunks", who, count, (long long)chunks);
  if (dtype != TOK_BF16 && dtype != TOK_F16)
    return fail(TOK_ERR_INVALID, "%s: parameters must be bf16 or f16 (dtype %d)", who, dtype);
  const struct { const char* name; double value; } hyper[] = {
      {"lr", lr}, {"momentum", momentum}, {"dampening", dampening},
      {"weight_decay", weight_decay}, {"trust_coefficient", trust_coefficient}, {"eps", eps}};
  for (const auto& h : hyper)
    if (!(h.value >= 0.0) || !isfinite(h.value))
      return fail(TOK_ERR_INVALID, "%s: %s %g", who, h.name, h.value);
  if (nesterov && (momentum <= 0.0 || dampening != 0.0))
    return fail(TOK_ERR_INVALID, "%s: nesterov needs a momentum and zero dampening", who);
  if (chunks > 0 && !partials) return fail(TOK_ERR_INVALID, "%s: null partials", who);
  if (!device_ready()) return fail(TOK_ERR_NO_DEVICE, "%s needs a CUDA GPU (no CPU fallback)", who);
  if (chunks == 0) return TOK_OK;
  LarsArgs a{};
  a.seg = segments;
  a.count = count;
  a.chunks = chunks;
  a.partials = partials;
  a.neg_lr = (float)(-lr);
  a.inv_lr = (float)(1.0 / lr);   // the reciprocal in double, rounded once; inf at lr = 0
  a.mu = (float)momentum;
  a.damp_alpha = (float)(1.0 - dampening);
  a.tc = (float)trust_coefficient;
  a.wd = (float)weight_decay;
  a.eps = (float)eps;
  a.use_mu = momentum != 0.0;
  a.nesterov = nesterov != 0;
  a.fresh = fresh != 0;
  a.clip = clip != 0;
  const cudaStream_t st = (cudaStream_t)cuda_stream;
  if (dtype == TOK_BF16)
    launch<__nv_bfloat16>(a, inv_scale, grad_coef, st);
  else
    launch<__half>(a, inv_scale, grad_coef, st);
  return launched(who);
}
