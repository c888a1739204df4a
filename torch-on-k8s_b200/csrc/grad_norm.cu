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
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "tok_internal.h"

namespace tok {
namespace {

constexpr int kNormThreads = 512;              // ATen's kBlockSize, and lpnorm_cleanup's block
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

// ATen's BlockReduceSum for a 512-thread block; the sum is valid in thread 0.
__device__ __forceinline__ float block_sum(float val, float* shared) {
  const int lid = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) val = __fadd_rn(val, __shfl_down_sync(0xffffffffu, val, off));
  __syncthreads();
  if (lid == 0) shared[wid] = val;
  __syncthreads();
  val = threadIdx.x < kNormThreads / 32 ? shared[lid] : 0.0f;
  if (wid == 0) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1)
      val = __fadd_rn(val, __shfl_down_sync(0xffffffffu, val, off));
  }
  return val;
}

// One block per (segment, chunk): the chunk's sum of squares, as LpNormFunctor forms it, into
// partials[blockIdx.x].
template <typename T>
__global__ void __launch_bounds__(kNormThreads)
    norm_partial_kernel(const tok_norm_segment_t* __restrict__ seg, int count,
                        float* __restrict__ partials) {
  __shared__ tok_norm_segment_t s;
  __shared__ float red[32];
  const int64_t c = blockIdx.x;
  if (threadIdx.x == 0) {
    int lo = 0, hi = count - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (seg[mid].chunk0 <= c) lo = mid; else hi = mid - 1;
    }
    s = seg[lo];
  }
  __syncthreads();
  const int64_t start = (c - s.chunk0) * kNormChunk;
  const int64_t n = min(s.numel - start, kNormChunk);   // this chunk's elements
  const uint16_t* x = (const uint16_t*)s.grad + start;
  float acc[kIlp] = {0.0f, 0.0f, 0.0f, 0.0f};
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
          const float f = to_f32<T>((uint16_t)(b[u][k >> 1] >> (16 * (k & 1))));
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
        const float f = to_f32<T>(b[k]);
        acc[k] = __fmaf_rn(f, f, acc[k]);
      }
    }
  }
  float val = 0.0f;
#pragma unroll
  for (int k = 0; k < kIlp; ++k) val = __fadd_rn(val, acc[k]);
  val = block_sum(val, red);
  if (threadIdx.x == 0) partials[c] = val;
}

// One block per segment: lpnorm_cleanup over the segment's partials, sqrt into norms[slot].
__global__ void __launch_bounds__(kNormThreads)
    norm_finish_kernel(const tok_norm_segment_t* __restrict__ seg,
                       const float* __restrict__ partials, float* __restrict__ norms) {
  __shared__ float red[32];
  const tok_norm_segment_t s = seg[blockIdx.x];
  const int64_t nchunks = (s.numel + kNormChunk - 1) / kNormChunk;
  float val = 0.0f;
  for (int64_t i = threadIdx.x; i < nchunks; i += kNormThreads)
    val = __fadd_rn(val, partials[s.chunk0 + i]);
  val = block_sum(val, red);
  if (threadIdx.x == 0) norms[s.slot] = __fsqrt_rn(val);
}

}  // namespace
}  // namespace tok

using namespace tok;

extern "C" int tok_grad_norms(const tok_norm_segment_t* segments, int count, int64_t chunks,
                              int dtype, float* partials, float* norms, void* cuda_stream) {
  const char* who = "tok_grad_norms";
  if (!segments) return fail(TOK_ERR_INVALID, "%s: null segment table", who);
  if (count <= 0 || chunks < 0 || chunks > 0x7fffffffLL)
    return fail(TOK_ERR_INVALID, "%s: %d segments in %lld chunks", who, count, (long long)chunks);
  if (dtype != TOK_BF16 && dtype != TOK_F16)
    return fail(TOK_ERR_INVALID, "%s: gradients must be bf16 or f16 (dtype %d)", who, dtype);
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
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(TOK_ERR_CUDA, "%s launch: %s", who, cudaGetErrorString(e));
  return TOK_OK;
}
