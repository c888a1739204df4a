// ResNet's stem max pool (kernel 3, stride 2, padding 1, dilation 1, no ceil mode), NHWC bf16, with
// one position byte per pooled element instead of ATen's int64 index.
//
// The activation of a channels_last [N, C, H, W] tensor is [N, H, W, C] in memory; the pooled output
// is [N, OH, OW, C] with OH = (H - 1) / 2 + 1, OW = (W - 1) / 2 + 1, and the positions are uint8
// [N, OH, OW, C].  Output (oh, ow) pools the window of input rows 2*oh - 1 + kh and columns
// 2*ow - 1 + kw, kh, kw in 0..2, clipped to the image; its position byte is kh * 3 + kw of the
// element ATen's max_pool_forward_nhwc records, or kPosNone when ATen records a plane index outside
// the window.
//
// Forward, as ATen's max_pool_forward_nhwc: the running maximum starts at -inf with index 0 (the
// plane's element (0, 0)), the window is scanned row by row (ih, then iw), and an element replaces
// the maximum when (val > max || isnan(val)).  So the first of equal maxima wins (+0 and -0
// compare equal), the last NaN wins, and the output is the winning element's bits (NaN payload and
// sign included).  A window in which nothing beats -inf (all -inf) keeps index 0: that element lies
// in the window of output (0, 0) only, at position 4, and outside every other window (kPosNone).
//
// Backward, as ATen's max_pool_backward_nhwc: each input element gathers from the outputs whose
// window covers it, oh ascending, then ow.  An element covered by one window only gets that
// output's gradient bits when it is the recorded position and +0 otherwise (ATen zero-fills the
// gradient and copies the bf16 value).  An element covered by more windows gets
// bf16(0.0f + g1 + g2 ...) over the outputs that recorded it, a float sum in that order, rounded
// to nearest even by the same conversion (a NaN comes out as the canonical 0x7fff).
//
// Each thread owns one 16-byte vector (8 channels) of one output (forward) or input (backward)
// column and walks a run of rows, keeping in registers what the next row shares with this one: the
// forward's window row 2*oh + 1 is the next window's first row, and the backward's output row k
// serves input rows 2k - 1, 2k and 2k + 1.  Neighbouring columns share their loads through L1.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "tok_internal.h"

namespace tok {
namespace {

constexpr int kVec = 8;             // bf16 per 16-byte vector
constexpr int kPoolThreads = 256;
constexpr int kPoolBlocksPerSm = 4;  // 64 registers: half the SM's threads resident
constexpr int kRowRun = 8;          // output rows per thread (forward: pooled rows; backward: k)
constexpr uint32_t kPosNone = 0xff; // the recorded element is outside the window
constexpr uint32_t kNegInf = 0xff800000u;

struct PoolGeom {
  int n, h, w, oh, ow, vecs, runs;  // runs = ceil(oh / kRowRun)
};

__device__ __forceinline__ uint32_t word(const uint4& q, int i) {
  return i == 0 ? q.x : i == 1 ? q.y : i == 2 ? q.z : q.w;
}

// bf16 k (0..7) of a 16-byte vector as float bits
__device__ __forceinline__ uint32_t lane_bits(const uint4& q, int k) {
  const uint32_t p = word(q, k >> 1);
  return (k & 1) ? (p & 0xffff0000u) : (p << 16);
}

// One window row: the three columns' vectors (absent ones are never looked at).
struct Row3 {
  uint4 v[3];
};

__device__ __forceinline__ void load_row(const uint4* __restrict__ x, const PoolGeom& g, int64_t plane,
                                         int ih, int iw0, int vec, Row3& r) {
  const uint4* p = x + ((plane + ih) * g.w + iw0) * g.vecs + vec;
#pragma unroll
  for (int kw = 0; kw < 3; ++kw) {
    const int iw = iw0 + kw;
    r.v[kw] = (iw >= 0 && iw < g.w) ? __ldg(p + kw * g.vecs) : make_uint4(0, 0, 0, 0);
  }
}

// Folds one window row into the running maximum, columns in scan order.
__device__ __forceinline__ void scan_row(const Row3& r, int kh, int iw0, int w, uint32_t (&m)[kVec],
                                         uint32_t (&pos)[kVec]) {
#pragma unroll
  for (int kw = 0; kw < 3; ++kw) {
    const int iw = iw0 + kw;
    if (iw < 0 || iw >= w) continue;
#pragma unroll
    for (int k = 0; k < kVec; ++k) {
      const uint32_t b = lane_bits(r.v[kw], k);
      const float val = __uint_as_float(b);
      if (val > __uint_as_float(m[k]) || isnan(val)) {
        m[k] = b;
        pos[k] = (uint32_t)(kh * 3 + kw);
      }
    }
  }
}

__global__ void __launch_bounds__(kPoolThreads, kPoolBlocksPerSm)
max_pool_fwd_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, uint2* __restrict__ pos_out,
                    const PoolGeom g) {
  // the thread count is below 2^31: the activation has at most 2^31 - 1 elements
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int vec = t % g.vecs;
  int rest = t / g.vecs;
  const int ow = rest % g.ow;
  rest /= g.ow;
  const int run = rest % g.runs;
  const int n = rest / g.runs;
  if (n >= g.n) return;
  const int oh0 = run * kRowRun;
  const int oh1 = min(oh0 + kRowRun, g.oh);
  const int iw0 = 2 * ow - 1;
  const int64_t plane = (int64_t)n * g.h;

  Row3 carry;  // window row 2*oh - 1 of the next window, loaded by the previous one
  for (int oh = oh0; oh < oh1; ++oh) {
    uint32_t m[kVec], pos[kVec];
#pragma unroll
    for (int k = 0; k < kVec; ++k) {
      m[k] = kNegInf;
      // ATen's initial index 0 is the plane's element (0, 0): position 4 of output (0, 0)'s window
      pos[k] = (oh == 0 && ow == 0) ? 4u : kPosNone;
    }
    const int ih0 = 2 * oh - 1;
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int ih = ih0 + kh;
      if (ih < 0 || ih >= g.h) continue;
      Row3 r;
      if (kh == 0 && oh > oh0) r = carry;
      else load_row(x, g, plane, ih, iw0, vec, r);
      scan_row(r, kh, iw0, g.w, m, pos);
      if (kh == 2) carry = r;
    }
    const int64_t o = (((int64_t)n * g.oh + oh) * g.ow + ow) * g.vecs + vec;
    y[o] = make_uint4((m[0] >> 16) | (m[1] & 0xffff0000u), (m[2] >> 16) | (m[3] & 0xffff0000u),
                      (m[4] >> 16) | (m[5] & 0xffff0000u), (m[6] >> 16) | (m[7] & 0xffff0000u));
    pos_out[o] = make_uint2(pos[0] | (pos[1] << 8) | (pos[2] << 16) | (pos[3] << 24),
                            pos[4] | (pos[5] << 8) | (pos[6] << 16) | (pos[7] << 24));
  }
}

// The gradients and positions of one output row at the (at most two) output columns covering an
// input column.
struct OutRow {
  uint4 g[2];
  uint2 p[2];
};

__device__ __forceinline__ void load_out_row(const uint4* __restrict__ gy,
                                             const uint2* __restrict__ pos, const PoolGeom& g,
                                             int64_t oplane, int oh, int pw0, int npw, int vec,
                                             OutRow& r) {
  const int64_t o = ((oplane + oh) * g.ow + pw0) * g.vecs + vec;
  r.g[0] = __ldg(gy + o);
  r.p[0] = __ldg(pos + o);
  if (npw == 2) {
    r.g[1] = __ldg(gy + o + g.vecs);
    r.p[1] = __ldg(pos + o + g.vecs);
  }
}

__device__ __forceinline__ uint32_t pos_byte(const uint2& p, int k) {
  return ((k < 4 ? p.x : p.y) >> (8 * (k & 3))) & 0xffu;
}

// One input element covered by a single window: the gradient's bits where it won, +0 elsewhere.
__device__ __forceinline__ uint4 route_one(const OutRow& r, uint32_t want) {
  uint32_t out[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint32_t gw = word(r.g[0], i);
    const uint32_t lo = pos_byte(r.p[0], 2 * i) == want ? (gw & 0xffffu) : 0u;
    const uint32_t hi = pos_byte(r.p[0], 2 * i + 1) == want ? (gw & 0xffff0000u) : 0u;
    out[i] = lo | hi;
  }
  return make_uint4(out[0], out[1], out[2], out[3]);
}

// Adds the terms of one output row (columns ascending) that recorded this input element.
__device__ __forceinline__ void gather_row(const OutRow& r, int npw, uint32_t want0, float (&acc)[kVec]) {
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    if (j >= npw) break;
    const uint32_t want = want0 - 2u * j;  // the next window starts two columns to the right
#pragma unroll
    for (int k = 0; k < kVec; ++k)
      if (pos_byte(r.p[j], k) == want) acc[k] = __fadd_rn(acc[k], __uint_as_float(lane_bits(r.g[j], k)));
  }
}

__device__ __forceinline__ uint4 round_sum(const float (&acc)[kVec]) {
  uint32_t out[4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
    out[i] = (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(acc[2 * i])) |
             ((uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(acc[2 * i + 1])) << 16);
  return make_uint4(out[0], out[1], out[2], out[3]);
}

// dx of input row ih from the output rows covering it (one or two: rows[0], then rows[1]).
__device__ __forceinline__ uint4 input_grad(const OutRow* rows, int nph, int ph0, int ih, int pw0,
                                            int npw, int iw) {
  // the position of (ih, iw) inside the window of output (oh, pw0) is (ih - 2*oh + 1, iw - 2*pw0 + 1)
  const uint32_t kw0 = (uint32_t)(iw - 2 * pw0 + 1);
  if (nph == 1 && npw == 1) return route_one(rows[0], (uint32_t)(ih - 2 * ph0 + 1) * 3u + kw0);
  float acc[kVec];
#pragma unroll
  for (int k = 0; k < kVec; ++k) acc[k] = 0.0f;
#pragma unroll
  for (int i = 0; i < 2; ++i)
    if (i < nph) gather_row(rows[i], npw, (uint32_t)(ih - 2 * (ph0 + i) + 1) * 3u + kw0, acc);
  return round_sum(acc);
}

__global__ void __launch_bounds__(kPoolThreads, kPoolBlocksPerSm)
max_pool_bwd_kernel(const uint4* __restrict__ gy, const uint2* __restrict__ pos,
                    uint4* __restrict__ dx, const PoolGeom g) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int vec = t % g.vecs;
  int rest = t / g.vecs;
  const int iw = rest % g.w;
  rest /= g.w;
  const int run = rest % g.runs;
  const int n = rest / g.runs;
  if (n >= g.n) return;
  // the output columns covering iw: iw / 2, and iw / 2 + 1 too for an odd iw inside the output
  const int pw0 = iw >> 1;
  const int npw = ((iw & 1) && pw0 + 1 < g.ow) ? 2 : 1;
  const int64_t oplane = (int64_t)n * g.oh;
  const int k0 = run * kRowRun;
  const int k1 = min(k0 + kRowRun, g.oh);

  // input row 2k is covered by output row k alone, input row 2k + 1 by rows k and k + 1 (when
  // k + 1 < OH); row k is loaded once for the input rows 2k - 1, 2k and 2k + 1
  OutRow rows[2];
  load_out_row(gy, pos, g, oplane, k0, pw0, npw, vec, rows[0]);
  for (int k = k0; k < k1; ++k) {
    const int ih = 2 * k;
    const int64_t base = ((int64_t)n * g.h + ih) * g.w + iw;
    dx[base * g.vecs + vec] = input_grad(rows, 1, k, ih, pw0, npw, iw);
    if (ih + 1 >= g.h) break;
    const int nph = k + 1 < g.oh ? 2 : 1;
    if (nph == 2) load_out_row(gy, pos, g, oplane, k + 1, pw0, npw, vec, rows[1]);
    dx[(base + g.w) * g.vecs + vec] = input_grad(rows, nph, k, ih + 1, pw0, npw, iw);
    rows[0] = rows[1];
  }
}

bool misaligned(const void* p, uintptr_t bytes) { return ((uintptr_t)p & (bytes - 1)) != 0; }

int check_pool(const char* who, const void* in, const char* in_name, const void* out,
               const char* out_name, const void* pos, int64_t n, int64_t h, int64_t w, int channels,
               PoolGeom& g) {
  if (!in || !out || !pos) return fail(TOK_ERR_INVALID, "%s: null pointer argument", who);
  if (n <= 0 || h <= 0 || w <= 0 || channels <= 0)
    return fail(TOK_ERR_INVALID, "%s: shape %lld x %lld x %lld x %d must be positive", who,
                (long long)n, (long long)h, (long long)w, channels);
  if (n * h * w * channels > INT32_MAX)
    return fail(TOK_ERR_INVALID, "%s: %lld x %lld x %lld x %d elements exceed 32-bit indexing", who,
                (long long)n, (long long)h, (long long)w, channels);
  if (channels % kVec != 0)
    return fail(TOK_ERR_ALIGN, "%s: channels %d is not a multiple of %d", who, channels, kVec);
  if (misaligned(in, 16)) return fail(TOK_ERR_ALIGN, "%s: %s is not 16-byte aligned", who, in_name);
  if (misaligned(out, 16)) return fail(TOK_ERR_ALIGN, "%s: %s is not 16-byte aligned", who, out_name);
  if (misaligned(pos, 8)) return fail(TOK_ERR_ALIGN, "%s: positions are not 8-byte aligned", who);
  if (!device_ready()) return fail(TOK_ERR_NO_DEVICE, "%s needs a CUDA GPU (no CPU fallback)", who);
  g.n = (int)n;
  g.h = (int)h;
  g.w = (int)w;
  g.oh = (int)((h - 1) / 2 + 1);
  g.ow = (int)((w - 1) / 2 + 1);
  g.vecs = channels / kVec;
  g.runs = (g.oh + kRowRun - 1) / kRowRun;
  return TOK_OK;
}

template <typename Kernel, typename... Args>
int launch_threads(const char* who, Kernel kernel, int64_t threads, void* stream, Args... args) {
  const int64_t blocks = (threads + kPoolThreads - 1) / kPoolThreads;
  kernel<<<(unsigned)blocks, kPoolThreads, 0, (cudaStream_t)stream>>>(args...);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(TOK_ERR_CUDA, "%s launch: %s", who, cudaGetErrorString(e));
  return TOK_OK;
}

}  // namespace
}  // namespace tok

using namespace tok;

extern "C" int tok_max_pool_fwd(const void* x, void* y, void* positions, int64_t n, int64_t h,
                                int64_t w, int channels, void* cuda_stream) {
  const char* who = "tok_max_pool_fwd";
  PoolGeom g{};
  const int rc = check_pool(who, x, "x", y, "y", positions, n, h, w, channels, g);
  if (rc != TOK_OK) return rc;
  const int64_t threads = (int64_t)g.n * g.runs * g.ow * g.vecs;
  return launch_threads(who, max_pool_fwd_kernel, threads, cuda_stream, (const uint4*)x, (uint4*)y,
                        (uint2*)positions, g);
}

extern "C" int tok_max_pool_bwd(const void* gy, const void* positions, void* dx, int64_t n,
                                int64_t h, int64_t w, int channels, void* cuda_stream) {
  const char* who = "tok_max_pool_bwd";
  PoolGeom g{};
  const int rc = check_pool(who, gy, "gy", dx, "dx", positions, n, h, w, channels, g);
  if (rc != TOK_OK) return rc;
  const int64_t threads = (int64_t)g.n * g.runs * g.w * g.vecs;
  return launch_threads(who, max_pool_bwd_kernel, threads, cuda_stream, (const uint4*)gy,
                        (const uint2*)positions, (uint4*)dx, g);
}
