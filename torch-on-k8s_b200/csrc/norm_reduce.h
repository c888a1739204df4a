// ATen's block reductions for the fp32 L2 norms of torch._foreach_norm, shared by the gradient norms
// (grad_norm.cu) and the trust ratios of LAMB (lamb.cu) and LARS (lars.cu).  See grad_norm.cu's header comment for how they
// were read off torch 2.11's LpNormFunctor and lpnorm_cleanup.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace tok {
namespace {

constexpr int kNormThreads = 512;   // ATen's kBlockSize, and lpnorm_cleanup's block

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

// lpnorm_cleanup's sum over one tensor's `nchunks` chunk partials: thread t adds partials t, t + 512,
// ... in order, then block_sum.  Valid in thread 0; the norm is its correctly rounded sqrt.
__device__ __forceinline__ float cleanup_sum(const float* __restrict__ partials, int64_t nchunks,
                                             float* shared) {
  float val = 0.0f;
  for (int64_t i = threadIdx.x; i < nchunks; i += kNormThreads) val = __fadd_rn(val, partials[i]);
  return block_sum(val, shared);
}

// The segment of chunk c in a table of `count` segments with first-chunk indices `chunk0`: thread 0
// finds the last segment whose first chunk is <= c and copies it to `s`, then the block syncs.
template <typename Seg>
__device__ __forceinline__ void find_segment(const Seg* seg, int count, int64_t c, Seg& s) {
  if (threadIdx.x == 0) {
    int lo = 0, hi = count - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (seg[mid].chunk0 <= c) lo = mid; else hi = mid - 1;
    }
    s = seg[lo];
  }
  __syncthreads();
}

}  // namespace
}  // namespace tok
