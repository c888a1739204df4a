// SGD step on fp32 master weights for bf16 / f16 parameters, one launch per gradient bucket.
//
// For every element of every segment (one parameter: its gradient inside the bucket, the half-
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
// Work is split over (segment, chunk) pairs: block b takes chunk b of the whole table and finds its
// segment by binary search over the entries' first-chunk indices.  Inside a chunk, 8 elements at a
// time go through 16-byte vector loads and stores where the parameter, master and momentum pointers
// share an alignment phase; the gradient is a vector load when its phase agrees too (DDP does not pad
// bucket views, so it often does not), otherwise 8 scalar loads.  The chunk's unaligned head and tail
// are scalar.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "tok_internal.h"

namespace tok {
namespace {

constexpr int kSgdThreads = 256;
constexpr int64_t kChunk = TOK_SGD_CHUNK;   // elements per (segment, chunk) work item
static_assert(kChunk % 8 == 0, "a chunk must start at a vector boundary of every array");

struct SgdArgs {
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
};

__device__ __forceinline__ float add_alpha(float a, float b, float alpha) {
  return __fmaf_rn(alpha, b, a);   // a + alpha * b, one rounding (see the header comment)
}

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

// One element: returns the new master; updates m in place.
__device__ __forceinline__ float sgd(const SgdArgs& a, float g, float w, float& m) {
  if (a.use_wd) g = add_alpha(g, w, a.wd);
  if (a.use_mu) {
    m = a.fresh ? g : add_alpha(__fmul_rn(m, a.mu), g, a.damp_alpha);
    g = a.nesterov ? add_alpha(g, m, a.mu) : m;
  }
  return add_alpha(w, g, a.neg_lr);
}

template <typename T>
__device__ __forceinline__ void scalar_step(const SgdArgs& a, const tok_sgd_segment_t& s,
                                            int64_t i) {
  const float g = widen<T>(__ldg((const uint16_t*)s.grad + i));
  float m = (a.use_mu && !a.fresh) ? s.momentum[i] : 0.0f;
  const float w = sgd(a, g, s.master[i], m);
  s.master[i] = w;
  if (a.use_mu) s.momentum[i] = m;
  ((uint16_t*)s.param)[i] = narrow<T>(w);
}

__device__ __forceinline__ float lane(const float4& v, int k) {
  return k == 0 ? v.x : k == 1 ? v.y : k == 2 ? v.z : v.w;
}

template <typename T>
__device__ __forceinline__ void vector_step(const SgdArgs& a, const tok_sgd_segment_t& s,
                                            int64_t i, bool grad_vec) {
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
  if (a.use_mu && !a.fresh) {
    m0 = mp[0];
    m1 = mp[1];
  }
  float w[8], m[8];
  uint16_t out[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    m[k] = k < 4 ? lane(m0, k) : lane(m1, k - 4);
    w[k] = sgd(a, widen<T>(gb[k]), k < 4 ? lane(w0, k) : lane(w1, k - 4), m[k]);
    out[k] = narrow<T>(w[k]);
  }
  wp[0] = make_float4(w[0], w[1], w[2], w[3]);
  wp[1] = make_float4(w[4], w[5], w[6], w[7]);
  if (a.use_mu) {
    mp[0] = make_float4(m[0], m[1], m[2], m[3]);
    mp[1] = make_float4(m[4], m[5], m[6], m[7]);
  }
  *(uint4*)((uint16_t*)s.param + i) =
      make_uint4(out[0] | ((uint32_t)out[1] << 16), out[2] | ((uint32_t)out[3] << 16),
                 out[4] | ((uint32_t)out[5] << 16), out[6] | ((uint32_t)out[7] << 16));
}

__device__ __forceinline__ bool aligned16(const void* p, int64_t i, int esz) {
  return (((uintptr_t)p + (uintptr_t)(i * esz)) & 15u) == 0;
}

template <typename T>
__global__ void __launch_bounds__(kSgdThreads) sgd_master_kernel(const SgdArgs a) {
  __shared__ tok_sgd_segment_t s;
  const int64_t c = blockIdx.x;
  if (threadIdx.x == 0) {
    int lo = 0, hi = a.count - 1;   // last entry whose first chunk is <= c
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (a.seg[mid].chunk0 <= c) lo = mid; else hi = mid - 1;
    }
    s = a.seg[lo];
  }
  __syncthreads();
  const int64_t start = (c - s.chunk0) * kChunk;
  const int64_t end = min(start + kChunk, s.numel);
  if (start >= end) return;
  // first element at which the parameter is 16-byte aligned; the vector path needs the master and
  // the momentum aligned there too
  int64_t head = ((16 - (((uintptr_t)s.param + (uintptr_t)(start * 2)) & 15u)) & 15u) / 2;
  const bool vec = ((uintptr_t)s.param & 1u) == 0 && aligned16(s.master, start + head, 4) &&
                   (!a.use_mu || aligned16(s.momentum, start + head, 4));
  if (!vec || head > end - start) head = end - start;
  const int64_t nvec = (end - start - head) / 8;
  const int64_t vbeg = start + head, tail = vbeg + 8 * nvec;
  const bool grad_vec = aligned16(s.grad, vbeg, 2);
  for (int64_t v = threadIdx.x; v < nvec; v += kSgdThreads)
    vector_step<T>(a, s, vbeg + 8 * v, grad_vec);
  const int64_t nscalar = head + (end - tail);
  for (int64_t j = threadIdx.x; j < nscalar; j += kSgdThreads)
    scalar_step<T>(a, s, j < head ? start + j : tail + (j - head));
}

}  // namespace
}  // namespace tok

using namespace tok;

extern "C" int tok_sgd_master_step(const tok_sgd_segment_t* segments, int count, int64_t chunks,
                                   int dtype, double lr, double momentum, double dampening,
                                   double weight_decay, int nesterov, int fresh,
                                   void* cuda_stream) {
  const char* who = "tok_sgd_master_step";
  if (!segments) return fail(TOK_ERR_INVALID, "%s: null segment table", who);
  if (count <= 0 || chunks <= 0 || chunks > 0x7fffffffLL)
    return fail(TOK_ERR_INVALID, "%s: %d segments in %lld chunks", who, count, (long long)chunks);
  if (dtype != TOK_BF16 && dtype != TOK_F16)
    return fail(TOK_ERR_INVALID, "%s: parameters must be bf16 or f16 (dtype %d)", who, dtype);
  if (!(lr >= 0.0) || !isfinite(lr)) return fail(TOK_ERR_INVALID, "%s: lr %g", who, lr);
  if (!(momentum >= 0.0) || !isfinite(momentum))
    return fail(TOK_ERR_INVALID, "%s: momentum %g", who, momentum);
  if (!isfinite(dampening)) return fail(TOK_ERR_INVALID, "%s: dampening %g", who, dampening);
  if (!(weight_decay >= 0.0) || !isfinite(weight_decay))
    return fail(TOK_ERR_INVALID, "%s: weight_decay %g", who, weight_decay);
  if (nesterov && (momentum <= 0.0 || dampening != 0.0))
    return fail(TOK_ERR_INVALID, "%s: nesterov needs a momentum and zero dampening", who);
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
  if (dtype == TOK_BF16)
    sgd_master_kernel<__nv_bfloat16><<<grid, kSgdThreads, 0, (cudaStream_t)cuda_stream>>>(a);
  else
    sgd_master_kernel<__half><<<grid, kSgdThreads, 0, (cudaStream_t)cuda_stream>>>(a);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(TOK_ERR_CUDA, "%s launch: %s", who, cudaGetErrorString(e));
  return TOK_OK;
}
