// Per-tensor L2 norms of bf16 / f16 gradients for gradient clipping (optim.py's max_grad_norm), two
// launches per table: the bits torch._foreach_norm(f32(grads), 2) gives, wherever each gradient sits
// inside its bucket.
//
// ATen's _foreach_norm on fp32 CUDA tensors (ForeachReduceOp.cu, read off the sm_90 SASS of torch 2.11's
// LpNormFunctor<float, L2> and lpnorm_cleanup<float, L2, apply_root=true>, and settled element by
// element on an H100 by tools/foreach_norm_probe.py, profiles/h100_foreach_norm_probe.json):
//
//   * The tensor is cut into chunks of 65,536 elements (kChunkSize); one 512-thread block per chunk.
//   * A thread keeps 4 fp32 accumulators (kILP) and adds each element's square with one FMA,
//     acc = fma(x, x, acc).  Which elements feed which accumulator depends on the fp32 tensor: when
//     its length is a multiple of 4 (and it is 16-byte aligned, which a fresh p.grad.float() always
//     is) thread t of the chunk reads the float4 at 4*(t + 512*j) and accumulator ii takes lane ii;
//     otherwise accumulator ii takes element i0 + t + 512*ii for i0 = 0, 2048, 4096, ...
//   * The accumulators merge as ((0 + a0) + a1) + a2) + a3, then the block sums with ATen's
//     BlockReduceSum: a shfl_down tree (16, 8, 4, 2, 1) in every warp, the 16 warp sums through shared
//     memory into warp 0 (lanes 16..31 hold 0), the same tree again.  Thread 0 writes the chunk's
//     partial.
//   * lpnorm_cleanup, one 512-thread block per tensor: thread t adds partials t, t + 512, ... in
//     order (a tensor with more than 512 chunks gives a thread several), the same block tree, and a
//     correctly rounded sqrt.
//
// So the norm of a bf16 gradient inside a bucket depends on the gradient's length, never on its
// offset: this kernel reproduces the mapping of the fp32 copy whatever the bf16 view's alignment.
// Only the physical loads differ: 4 bf16 of a float4 group are one 8-byte load when the view allows
// it, and each thread issues 8 groups' loads before their FMAs (in the same order) run.
//
// Dynamic loss scaling (optim.py's loss_scale) adds two entry points over the same table:
//
//   * tok_grad_norms_unscaled: the partial kernel instantiated with kUnscale, so each element is
//     __fmul_rn(f32(g), inv_scale) before its FMA square — the one rounding
//     _amp_foreach_non_finite_check_and_unscale_ applies to master.grad, whose norm clip_grad_norm_
//     then takes.  The same pass votes on the raw values and sets *found_inf = 1 when one is inf or
//     NaN, so clipping with loss scaling reads every gradient once.  The plain instantiation compiles
//     to the SASS it had before the flag existed.
//   * tok_grad_nonfinite: only the vote, for steps without clipping.  One 512-thread block per
//     (segment, chunk), 16-byte loads from the first aligned element, scalar loads for the head and
//     tail, one __syncthreads_or per block and at most one store.  A 2-byte value is inf or NaN exactly
//     when its exponent bits are all set, which is when its fp32 widening is, so the bits are tested
//     without converting them.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "norm_reduce.h"
#include "tok_internal.h"

namespace tok {
namespace {

constexpr int64_t kNormChunk = TOK_NORM_CHUNK;  // ATen's kChunkSize for multi_tensor_apply
constexpr int kIlp = 4;                        // ATen's kILP
constexpr int kAhead = 8;                      // float4 groups loaded before their FMAs run
static_assert(kNormChunk % (kIlp * kNormThreads) == 0, "a chunk is whole strided rounds");

template <typename T> __device__ __forceinline__ float to_f32(uint16_t bits);
template <> __device__ __forceinline__ float to_f32<__nv_bfloat16>(uint16_t bits) {
  return __uint_as_float((uint32_t)bits << 16);
}
template <> __device__ __forceinline__ float to_f32<__half>(uint16_t bits) {
  return __half2float(__ushort_as_half(bits));
}

// The exponent bits of T: a value is inf or NaN when all of them are set.
template <typename T> constexpr uint32_t kExpBits = 0;
template <> constexpr uint32_t kExpBits<__nv_bfloat16> = 0x7f80u;
template <> constexpr uint32_t kExpBits<__half> = 0x7c00u;

template <typename T> __device__ __forceinline__ bool nonfinite(uint32_t bits) {
  return (bits & kExpBits<T>) == kExpBits<T>;
}

// Either of the two values packed in a 32-bit word.
template <typename T> __device__ __forceinline__ bool nonfinite2(uint32_t w) {
  return nonfinite<T>(w & 0xffffu) | nonfinite<T>(w >> 16);
}

// The block of one (segment, chunk): the chunk's sum of squares, as LpNormFunctor forms it, into
// partials[blockIdx.x].  With kUnscale each element is first multiplied by inv_scale (one rounding),
// and *found_inf becomes 1 when any raw element of the chunk is inf or NaN.
template <typename T, bool kUnscale>
__device__ __forceinline__ void norm_partial(const tok_norm_segment_t* __restrict__ seg, int count,
                                             float* __restrict__ partials, float inv_scale,
                                             float* __restrict__ found_inf) {
  __shared__ tok_norm_segment_t s;
  __shared__ float red[32];
  const int64_t c = blockIdx.x;
  find_segment(seg, count, c, s);
  const int64_t start = (c - s.chunk0) * kNormChunk;
  const int64_t n = min(s.numel - start, kNormChunk);   // this chunk's elements
  const uint16_t* x = (const uint16_t*)s.grad + start;
  float acc[kIlp] = {0.0f, 0.0f, 0.0f, 0.0f};
  bool bad = false;   // kUnscale: a raw inf or NaN seen by this thread
  if (s.numel % kIlp == 0) {
    // ATen's vector path: group g (elements 4g .. 4g+3) belongs to thread g % 512
    const int64_t groups = n / kIlp;
    const bool vec8 = ((uintptr_t)s.grad & 7u) == 0;   // start is a multiple of 4 elements
    for (int64_t g0 = threadIdx.x; g0 < groups; g0 += kAhead * kNormThreads) {
      uint32_t b[kAhead][2];   // the group's 4 values as bf16 / f16 pairs, low half first
#pragma unroll
      for (int u = 0; u < kAhead; ++u) {
        const int64_t g = g0 + (int64_t)u * kNormThreads;
        if (g >= groups) continue;
        if (vec8) {
          const uint2 q = __ldg((const uint2*)(x + kIlp * g));
          b[u][0] = q.x;
          b[u][1] = q.y;
        } else {
          const uint16_t* e = x + kIlp * g;
          b[u][0] = __ldg(e) | ((uint32_t)__ldg(e + 1) << 16);
          b[u][1] = __ldg(e + 2) | ((uint32_t)__ldg(e + 3) << 16);
        }
      }
#pragma unroll
      for (int u = 0; u < kAhead; ++u) {
        if (g0 + (int64_t)u * kNormThreads >= groups) continue;
#pragma unroll
        for (int k = 0; k < kIlp; ++k) {
          const uint16_t raw = (uint16_t)(b[u][k >> 1] >> (16 * (k & 1)));
          float f = to_f32<T>(raw);
          if (kUnscale) {
            bad |= nonfinite<T>(raw);
            f = __fmul_rn(f, inv_scale);
          }
          acc[k] = __fmaf_rn(f, f, acc[k]);
        }
      }
    }
  } else {
    // ATen's scalar path: element i0 + t + 512 * ii feeds accumulator ii
    for (int64_t i0 = 0; i0 < n; i0 += kIlp * kNormThreads) {
      uint16_t b[kIlp];
#pragma unroll
      for (int k = 0; k < kIlp; ++k) {
        const int64_t i = i0 + threadIdx.x + (int64_t)k * kNormThreads;
        b[k] = i < n ? __ldg(x + i) : (uint16_t)0;
      }
#pragma unroll
      for (int k = 0; k < kIlp; ++k) {
        if (i0 + threadIdx.x + (int64_t)k * kNormThreads >= n) continue;
        float f = to_f32<T>(b[k]);
        if (kUnscale) {
          bad |= nonfinite<T>(b[k]);
          f = __fmul_rn(f, inv_scale);
        }
        acc[k] = __fmaf_rn(f, f, acc[k]);
      }
    }
  }
  float val = 0.0f;
#pragma unroll
  for (int k = 0; k < kIlp; ++k) val = __fadd_rn(val, acc[k]);
  if (kUnscale && __syncthreads_or(bad) && threadIdx.x == 0) *found_inf = 1.0f;
  val = block_sum(val, red);
  if (threadIdx.x == 0) partials[c] = val;
}

template <typename T>
__global__ void __launch_bounds__(kNormThreads)
    norm_partial_kernel(const tok_norm_segment_t* __restrict__ seg, int count,
                        float* __restrict__ partials) {
  norm_partial<T, false>(seg, count, partials, 1.0f, nullptr);
}

template <typename T>
__global__ void __launch_bounds__(kNormThreads)
    norm_partial_unscaled_kernel(const tok_norm_segment_t* __restrict__ seg, int count,
                                 const float* __restrict__ inv_scale, float* __restrict__ partials,
                                 float* __restrict__ found_inf) {
  norm_partial<T, true>(seg, count, partials, __ldg(inv_scale), found_inf);
}

// One block per segment: lpnorm_cleanup over the segment's partials, sqrt into norms[slot].
__global__ void __launch_bounds__(kNormThreads)
    norm_finish_kernel(const tok_norm_segment_t* __restrict__ seg,
                       const float* __restrict__ partials, float* __restrict__ norms) {
  __shared__ float red[32];
  const tok_norm_segment_t s = seg[blockIdx.x];
  const float val = cleanup_sum(partials + s.chunk0, (s.numel + kNormChunk - 1) / kNormChunk, red);
  if (threadIdx.x == 0) norms[s.slot] = __fsqrt_rn(val);
}

constexpr int kVoteThreads = 512;
constexpr int kVoteAhead = 4;   // 16-byte loads in flight per thread

// One block per (segment, chunk): *found_inf = 1 when an element of the chunk is inf or NaN.
template <typename T>
__global__ void __launch_bounds__(kVoteThreads)
    nonfinite_kernel(const tok_norm_segment_t* __restrict__ seg, int count,
                     float* __restrict__ found_inf) {
  __shared__ tok_norm_segment_t s;
  const int64_t c = blockIdx.x;
  find_segment(seg, count, c, s);
  const int64_t start = (c - s.chunk0) * kNormChunk;
  const int64_t n = min(s.numel - start, kNormChunk);
  const uint16_t* x = (const uint16_t*)s.grad + start;
  // the scalar head up to the first 16-byte boundary (2-byte values: the address is even), the
  // 8-element vectors, the scalar tail
  int64_t head = (int64_t)(((16u - ((uintptr_t)x & 15u)) & 15u) >> 1);
  if (((uintptr_t)x & 1u) != 0 || head > n) head = n;
  const int64_t nvec = (n - head) >> 3;
  const uint4* v = (const uint4*)(x + head);
  bool bad = false;
  for (int64_t i0 = threadIdx.x; i0 < nvec; i0 += kVoteAhead * kVoteThreads) {
    uint4 q[kVoteAhead];
#pragma unroll
    for (int u = 0; u < kVoteAhead; ++u) {
      const int64_t i = i0 + (int64_t)u * kVoteThreads;
      q[u] = i < nvec ? __ldg(v + i) : make_uint4(0u, 0u, 0u, 0u);
    }
#pragma unroll
    for (int u = 0; u < kVoteAhead; ++u)
      bad |= nonfinite2<T>(q[u].x) | nonfinite2<T>(q[u].y) | nonfinite2<T>(q[u].z) |
             nonfinite2<T>(q[u].w);
  }
  const int64_t tail = head + (nvec << 3);
  const int64_t nscalar = head + (n - tail);
  for (int64_t j = threadIdx.x; j < nscalar; j += kVoteThreads)
    bad |= nonfinite<T>(__ldg(x + (j < head ? j : tail + (j - head))));
  if (__syncthreads_or(bad) && threadIdx.x == 0) *found_inf = 1.0f;
}

// The table checks every entry point here shares; 0 when they pass.
int check_norm_table(const char* who, const tok_norm_segment_t* segments, int count, int64_t chunks,
                     int dtype) {
  if (!segments) return fail(TOK_ERR_INVALID, "%s: null segment table", who);
  if (count <= 0 || chunks < 0 || chunks > 0x7fffffffLL)
    return fail(TOK_ERR_INVALID, "%s: %d segments in %lld chunks", who, count, (long long)chunks);
  if (dtype != TOK_BF16 && dtype != TOK_F16)
    return fail(TOK_ERR_INVALID, "%s: gradients must be bf16 or f16 (dtype %d)", who, dtype);
  return 0;
}

int launched(const char* who) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(TOK_ERR_CUDA, "%s launch: %s", who, cudaGetErrorString(e));
  return TOK_OK;
}

}  // namespace
}  // namespace tok

using namespace tok;

extern "C" int tok_grad_norms(const tok_norm_segment_t* segments, int count, int64_t chunks,
                              int dtype, float* partials, float* norms, void* cuda_stream) {
  const char* who = "tok_grad_norms";
  if (const int rc = check_norm_table(who, segments, count, chunks, dtype)) return rc;
  if (!norms) return fail(TOK_ERR_INVALID, "%s: null norms", who);
  if (chunks > 0 && !partials) return fail(TOK_ERR_INVALID, "%s: null partials", who);
  if (!device_ready()) return fail(TOK_ERR_NO_DEVICE, "%s needs a CUDA GPU (no CPU fallback)", who);
  const cudaStream_t st = (cudaStream_t)cuda_stream;
  if (chunks > 0) {
    if (dtype == TOK_BF16)
      norm_partial_kernel<__nv_bfloat16><<<(unsigned)chunks, kNormThreads, 0, st>>>(segments, count,
                                                                                   partials);
    else
      norm_partial_kernel<__half><<<(unsigned)chunks, kNormThreads, 0, st>>>(segments, count,
                                                                            partials);
  }
  norm_finish_kernel<<<(unsigned)count, kNormThreads, 0, st>>>(segments, partials, norms);
  return launched(who);
}

extern "C" int tok_grad_norms_unscaled(const tok_norm_segment_t* segments, int count, int64_t chunks,
                                       int dtype, const float* inv_scale, float* partials,
                                       float* norms, float* found_inf, void* cuda_stream) {
  const char* who = "tok_grad_norms_unscaled";
  if (const int rc = check_norm_table(who, segments, count, chunks, dtype)) return rc;
  if (!inv_scale) return fail(TOK_ERR_INVALID, "%s: null inv_scale", who);
  if (!norms) return fail(TOK_ERR_INVALID, "%s: null norms", who);
  if (!found_inf) return fail(TOK_ERR_INVALID, "%s: null found_inf", who);
  if (chunks > 0 && !partials) return fail(TOK_ERR_INVALID, "%s: null partials", who);
  if (!device_ready()) return fail(TOK_ERR_NO_DEVICE, "%s needs a CUDA GPU (no CPU fallback)", who);
  const cudaStream_t st = (cudaStream_t)cuda_stream;
  if (chunks > 0) {
    if (dtype == TOK_BF16)
      norm_partial_unscaled_kernel<__nv_bfloat16><<<(unsigned)chunks, kNormThreads, 0, st>>>(
          segments, count, inv_scale, partials, found_inf);
    else
      norm_partial_unscaled_kernel<__half><<<(unsigned)chunks, kNormThreads, 0, st>>>(
          segments, count, inv_scale, partials, found_inf);
  }
  norm_finish_kernel<<<(unsigned)count, kNormThreads, 0, st>>>(segments, partials, norms);
  return launched(who);
}

extern "C" int tok_grad_nonfinite(const tok_norm_segment_t* segments, int count, int64_t chunks,
                                  int dtype, float* found_inf, void* cuda_stream) {
  const char* who = "tok_grad_nonfinite";
  if (const int rc = check_norm_table(who, segments, count, chunks, dtype)) return rc;
  if (!found_inf) return fail(TOK_ERR_INVALID, "%s: null found_inf", who);
  if (!device_ready()) return fail(TOK_ERR_NO_DEVICE, "%s needs a CUDA GPU (no CPU fallback)", who);
  if (chunks == 0) return TOK_OK;
  const cudaStream_t st = (cudaStream_t)cuda_stream;
  if (dtype == TOK_BF16)
    nonfinite_kernel<__nv_bfloat16><<<(unsigned)chunks, kVoteThreads, 0, st>>>(segments, count,
                                                                              found_inf);
  else
    nonfinite_kernel<__half><<<(unsigned)chunks, kVoteThreads, 0, st>>>(segments, count, found_inf);
  return launched(who);
}
