// Exponential moving average of the fp32 master weights (optim.py's ema_decay), one launch per gradient
// bucket, behind that bucket's step.  For every element of every segment (one parameter: its fp32
// master w and its fp32 average e) the kernel evaluates what torch.optim.swa_utils.AveragedModel with
// get_ema_multi_avg_fn(decay) evaluates on the masters:
//
//   e = w                        p_averaged.copy_(p_model)                   (copy: the first update)
//   e = lerp(e, w, weight)       torch._foreach_lerp_(ema, masters, 1 - decay)   (later updates)
//
// with weight = float(1.0 - decay): Python forms 1 - decay in double and ATen rounds the Scalar to
// float once.  lerp is master_elem.h's, ATen's two branches of one FMA each, pinned on an H100 by
// tools/foreach_adam_probe.py.  The first update must be a copy: a lerp with weight 1 would turn
// inf - inf into NaN.
//
// Work is split as in optim.cu: block b takes chunk b (TOK_SGD_CHUNK elements) of the whole table and
// finds its segment by binary search.  Inside a chunk, 4 elements at a time go through 16-byte loads
// and stores when the master and the average share an alignment phase there; the chunk's unaligned
// head and tail, and every element of a chunk whose phases differ, are scalar.  Nothing outside the
// segments is read or written.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "master_elem.h"
#include "norm_reduce.h"
#include "tok_internal.h"

namespace tok {
namespace {

constexpr int kEmaThreads = 256;
constexpr int64_t kEmaChunk = TOK_SGD_CHUNK;
static_assert(kEmaChunk % 4 == 0, "a chunk must start at a vector boundary of both arrays");

template <bool kCopy>
__device__ __forceinline__ float ema_elem(float e, float w, float weight) {
  return kCopy ? w : lerp(e, w, weight);
}

template <bool kCopy>
__global__ void __launch_bounds__(kEmaThreads)
    ema_master_kernel(const tok_ema_segment_t* __restrict__ seg, int count, float weight) {
  __shared__ tok_ema_segment_t s;
  const int64_t c = blockIdx.x;
  find_segment(seg, count, c, s);
  const int64_t start = (c - s.chunk0) * kEmaChunk;
  const int64_t end = min(start + kEmaChunk, s.numel);
  if (start >= end) return;
  const float* __restrict__ w = s.master;
  float* __restrict__ e = s.ema;
  // elements from `start` until the average is 16-byte aligned; the master must agree there
  int64_t head = ((16 - (((uintptr_t)e + (uintptr_t)(start * 4)) & 15u)) & 15u) / 4;
  const bool vec = (((uintptr_t)w + (uintptr_t)((start + head) * 4)) & 15u) == 0;
  if (!vec || head > end - start) head = end - start;
  const int64_t nvec = (end - start - head) / 4;
  const int64_t vbeg = start + head, tail = vbeg + 4 * nvec;
  for (int64_t v = threadIdx.x; v < nvec; v += kEmaThreads) {
    const float4 wv = __ldg((const float4*)(w + vbeg) + v);
    float4 ev = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!kCopy) ev = ((const float4*)(e + vbeg))[v];
    ev.x = ema_elem<kCopy>(ev.x, wv.x, weight);
    ev.y = ema_elem<kCopy>(ev.y, wv.y, weight);
    ev.z = ema_elem<kCopy>(ev.z, wv.z, weight);
    ev.w = ema_elem<kCopy>(ev.w, wv.w, weight);
    ((float4*)(e + vbeg))[v] = ev;
  }
  const int64_t nscalar = head + (end - tail);
  for (int64_t j = threadIdx.x; j < nscalar; j += kEmaThreads) {
    const int64_t i = j < head ? start + j : tail + (j - head);
    e[i] = ema_elem<kCopy>(kCopy ? 0.0f : e[i], __ldg(w + i), weight);
  }
}

}  // namespace
}  // namespace tok

using namespace tok;

extern "C" int tok_ema_master_update(const tok_ema_segment_t* segments, int count, int64_t chunks,
                                     double decay, int copy, void* cuda_stream) {
  const char* who = "tok_ema_master_update";
  if (!segments) return fail(TOK_ERR_INVALID, "%s: null segment table", who);
  if (count <= 0 || chunks <= 0 || chunks > 0x7fffffffLL)
    return fail(TOK_ERR_INVALID, "%s: %d segments in %lld chunks", who, count, (long long)chunks);
  if (!(decay >= 0.0 && decay <= 1.0))
    return fail(TOK_ERR_INVALID, "%s: decay %g outside [0, 1]", who, decay);
  if (!device_ready()) return fail(TOK_ERR_NO_DEVICE, "%s needs a CUDA GPU (no CPU fallback)", who);
  const float weight = (float)(1.0 - decay);   // Python's 1 - decay, rounded once as ATen's Scalar
  const cudaStream_t st = (cudaStream_t)cuda_stream;
  if (copy)
    ema_master_kernel<true><<<(unsigned)chunks, kEmaThreads, 0, st>>>(segments, count, weight);
  else
    ema_master_kernel<false><<<(unsigned)chunks, kEmaThreads, 0, st>>>(segments, count, weight);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(TOK_ERR_CUDA, "%s launch: %s", who, cudaGetErrorString(e));
  return TOK_OK;
}
