// Batch-norm forward, NHWC bf16 (training): the batch statistics, and the apply fused with ReLU and
// the residual add.
//
// The activation of a channels_last [N, C, H, W] tensor is the row-major matrix [M = N*H*W, C].
// The statistics (mean, biased variance, running-statistics update) reproduce ATen's channels_last
// statistics kernel and batch_norm_update_stats bit for bit (see "batch statistics" below); the apply
// kernels replace the passes that follow it in stock PyTorch:
//
//   mode 0:  y = relu(bf16(T(x)))                                  bn -> relu_
//   mode 1:  y = relu(bf16(f(bf16(T(x))) + f(r)))                  bn -> + identity -> relu_
//   mode 2:  y = relu(bf16(f(bf16(T(x))) + f(bf16(T'(xd)))))       bn, downsample bn -> + -> relu_
//
// f widens bf16 to float.  T is the float expression ATen's batch_norm_transform_input_channels_last
// kernel evaluates, in its order: fma((x - mean) * weight, invstd, bias), with
// invstd = rsqrt(var + eps) as batch_norm_update_stats_and_invert computes it.  The order is pinned
// with __fsub_rn / __fmul_rn / __fmaf_rn so that no contraction can change it, and the roundings to
// bf16 between the steps are the ones the stock composition performs, so the output is bit-identical.
// The ReLU is ATen's clamp_min(v, 0): NaN passes through, anything else is fmaxf(v, 0).
//
// Every thread owns one 16-byte vector column (8 channels) and keeps that column's parameters in
// registers; it walks rows with a grid stride, kRowUnroll rows in flight.  The grid is sized from
// the SM count and the kernel's occupancy.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>

#include "bn_stats_geom.h"
#include "tok_internal.h"

namespace tok {
namespace {

constexpr int kVec = 8;         // bf16 per 16-byte vector
constexpr int kBnThreads = 256;
constexpr int kRowUnroll = 4;
constexpr int kMaxTileVecs = 32;

struct BnSide {
  const uint4* x;
  const float* mean;
  const float* var;
  const __nv_bfloat16* weight;
  const __nv_bfloat16* bias;
  float* invstd;   // written once per channel: the save_invstd the backward needs
  float eps;
};

struct BnArgs {
  BnSide a;         // the main batch norm
  BnSide d;         // mode 2: the downsample batch norm
  const uint4* res; // mode 1: the residual
  uint4* y;
  int64_t rows;
  int vecs;         // C / 8
};

struct Column {
  float mean[kVec], inv[kVec], w[kVec], b[kVec];
};

__device__ __forceinline__ void load_column(const BnSide& s, int v, bool write_inv, Column& c) {
#pragma unroll
  for (int k = 0; k < kVec; ++k) {
    const int ch = v * kVec + k;
    c.mean[k] = s.mean[ch];
    c.inv[k] = rsqrtf(__fadd_rn(s.var[ch], s.eps));
    c.w[k] = __bfloat162float(s.weight[ch]);
    c.b[k] = __bfloat162float(s.bias[ch]);
    if (write_inv) s.invstd[ch] = c.inv[k];
  }
}

__device__ __forceinline__ float widen(uint32_t pair, int hi) {
  return __uint_as_float(hi ? (pair & 0xffff0000u) : (pair << 16));
}

__device__ __forceinline__ uint32_t bf16_bits(float v) {
  return (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(v));
}

// bf16(T(x)) as a float (exactly representable in bf16)
__device__ __forceinline__ float bn_apply(float x, const Column& c, int k) {
  const float t = __fmaf_rn(__fmul_rn(__fsub_rn(x, c.mean[k]), c.w[k]), c.inv[k], c.b[k]);
  return __uint_as_float(bf16_bits(t) << 16);
}

// relu of a bf16 value held as float; returns its bf16 bits
__device__ __forceinline__ uint32_t relu_bits(float v) {
  if (isnan(v)) return __float_as_uint(v) >> 16;
  return __float_as_uint(fmaxf(v, 0.0f)) >> 16;
}

__device__ __forceinline__ uint32_t word(const uint4& q, int i) {
  return i == 0 ? q.x : i == 1 ? q.y : i == 2 ? q.z : q.w;
}

template <int kMode>
__device__ __forceinline__ uint4 transform(const uint4& xa, const uint4& xr, const uint4& xd,
                                           const Column& ca, const Column& cd) {
  uint32_t out[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    uint32_t lohi[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int k = 2 * i + h;
      float v = bn_apply(widen(word(xa, i), h), ca, k);
      if (kMode == 1) v = __uint_as_float(bf16_bits(__fadd_rn(v, widen(word(xr, i), h))) << 16);
      if (kMode == 2) {
        const float u = bn_apply(widen(word(xd, i), h), cd, k);
        v = __uint_as_float(bf16_bits(__fadd_rn(v, u)) << 16);
      }
      lohi[h] = relu_bits(v);
    }
    out[i] = lohi[0] | (lohi[1] << 16);
  }
  return make_uint4(out[0], out[1], out[2], out[3]);
}

template <int kMode>
__global__ void __launch_bounds__(kBnThreads) bn_fused_fwd_kernel(const BnArgs p) {
  const int v = blockIdx.y * blockDim.x + threadIdx.x;
  if (v >= p.vecs) return;
  const bool write_inv = blockIdx.x == 0 && threadIdx.y == 0;
  Column ca, cd;
  load_column(p.a, v, write_inv, ca);
  if (kMode == 2) load_column(p.d, v, write_inv, cd);

  const int64_t stride = (int64_t)gridDim.x * blockDim.y;
  const uint4 zero = make_uint4(0, 0, 0, 0);
  for (int64_t row = (int64_t)blockIdx.x * blockDim.y + threadIdx.y; row < p.rows;
       row += stride * kRowUnroll) {
    uint4 xa[kRowUnroll], xr[kRowUnroll], xd[kRowUnroll];
#pragma unroll
    for (int u = 0; u < kRowUnroll; ++u) {
      const int64_t r = row + u * stride;
      xa[u] = xr[u] = xd[u] = zero;
      if (r < p.rows) {
        const int64_t i = r * p.vecs + v;
        xa[u] = __ldg(p.a.x + i);
        if (kMode == 1) xr[u] = __ldg(p.res + i);
        if (kMode == 2) xd[u] = __ldg(p.d.x + i);
      }
    }
#pragma unroll
    for (int u = 0; u < kRowUnroll; ++u) {
      const int64_t r = row + u * stride;
      if (r < p.rows) p.y[r * p.vecs + v] = transform<kMode>(xa[u], xr[u], xd[u], ca, cd);
    }
  }
}

// ---- batch statistics ---------------------------------------------------------------------------
// The arithmetic of ATen's batch_norm_collect_statistics_channels_last_kernel<Var, BFloat16, float, 4>
// and of the update lambda of batch_norm_update_stats, pinned op by op as the sm_90 code of torch's
// libtorch_cuda.so performs it (cuobjdump -sass):
//   step      d0 = x - mean; mean = fma(d0, inv, mean); d1 = x - mean; m2 = fma(d0 * d1, valid, m2)
//             with inv = 1 / count correctly rounded (valid slot) or x = inv = valid = 0 (a slot past
//             the last row, still executed: it turns an infinite mean into NaN)
//   merge     f = 1 / max(1, n + nb) correctly rounded; d = mean - mean_b;
//             m2 = m2 + fma(((d * d) * nb) * n, f, m2_b); n += nb; and the mean
//             j-merge:   mean = fma(mean_b, nb, mean * n) * f     (chains 1, 2, 3 into chain 0)
//             tree/grid: mean = fma(mean, n, mean_b * nb) * f     (every other merge)
//   finish    var = m2 / n (IEEE division)
//   running   r_mean = bf16(fma(mean, momentum, (1 - momentum) * r_mean))
//             r_var  = bf16(fma(var * bessel, momentum, (1 - momentum) * r_var))
// The geometry is bn_stats_geom.h's.  Logical thread (by, ty) of ATen becomes 4 lanes per 8-channel
// vector here; lane j runs chain j over rows p + (4i + j) * P (p = by * block_y + ty,
// P = block_y * grid_y).
struct StatsArgs {
  const uint4* x;
  int* ws_count;   // grid_y > 1: per logical block partials, merged by the finish kernel
  float* ws_mean;
  float* ws_m2;
  float* mean;
  float* var;
  __nv_bfloat16* running_mean;
  __nv_bfloat16* running_var;
  int rows;
  int channels;
  int vecs;
  int block_y;
  int grid_y;
  int loop_count;
  float momentum;
  float bessel;
};

constexpr int kStatsThreads = 256;  // physical threads per block of the finish kernel
// Physical threads per block of the partial kernel, and chain steps loaded ahead of the one
// computed.  At <= 64 registers two blocks share an SM: a 64-channel site's 128 logical blocks run
// 16 warps on each SM, with 512 * 4 * 16 B = 32 KB of loads in flight.
constexpr int kStatsPartialThreads = 512;
constexpr int kStatsDepth = 4;

// Folds (nb, mean_b, m2_b) into (n, mean, m2); the caller then adds nb to n (one count serves the
// 8 channels of a vector).
template <bool kJMerge>
__device__ __forceinline__ void welford_merge(int n, float& mean, float& m2, int nb, float mean_b,
                                              float m2_b) {
  const float f = __frcp_rn(__int2float_rn(max(1, n + nb)));
  const float fn = __int2float_rn(n), fnb = __int2float_rn(nb);
  const float d = __fsub_rn(mean, mean_b);
  mean = kJMerge ? __fmul_rn(__fmaf_rn(mean_b, fnb, __fmul_rn(mean, fn)), f)
                 : __fmul_rn(__fmaf_rn(mean, fn, __fmul_rn(mean_b, fnb)), f);
  m2 = __fadd_rn(m2, __fmaf_rn(__fmul_rn(__fmul_rn(__fmul_rn(d, d), fnb), fn), f, m2_b));
}

__device__ __forceinline__ void stats_finish(const StatsArgs& a, int c, int n, float mean, float m2) {
  const float var = __fdiv_rn(m2, __int2float_rn(n));
  a.mean[c] = mean;
  a.var[c] = var;
  const float keep = __fsub_rn(1.0f, a.momentum);
  const float rm = __bfloat162float(a.running_mean[c]);
  const float rv = __bfloat162float(a.running_var[c]);
  a.running_mean[c] = __float2bfloat16_rn(__fmaf_rn(mean, a.momentum, __fmul_rn(keep, rm)));
  a.running_var[c] =
      __float2bfloat16_rn(__fmaf_rn(__fmul_rn(var, a.bessel), a.momentum, __fmul_rn(keep, rv)));
}

// blockDim = (4 * tile, block_y): lane j = threadIdx.x % 4 of thread (vx = threadIdx.x / 4, ty) of
// block (bx, by) runs chain j of logical thread (by, ty) on vector bx * tile + vx, the mapping of
// bn_bwd_partial_kernel.
__global__ void __launch_bounds__(kStatsPartialThreads, 2)
    bn_stats_partial_kernel(const StatsArgs a) {
  constexpr int kSlots = kStatsPartialThreads / kStatsChains;
  __shared__ float s_mean[kSlots][kVec];
  __shared__ float s_m2[kSlots][kVec];
  __shared__ int s_n[kSlots];
  const int j = threadIdx.x % kStatsChains, tile = blockDim.x / kStatsChains, ty = threadIdx.y;
  const int vx = threadIdx.x / kStatsChains;
  const int v = blockIdx.x * tile + vx;
  const bool live = v < a.vecs;
  const int64_t stride = (int64_t)a.block_y * a.grid_y;
  const int64_t step = kStatsChains * stride;
  const int64_t p = (int64_t)blockIdx.y * a.block_y + ty + j * stride;

  float mean[kVec], m2[kVec];
  int n = 0;
#pragma unroll
  for (int k = 0; k < kVec; ++k) mean[k] = m2[k] = 0.0f;

  if (live) {
    uint4 buf[kStatsDepth];
#pragma unroll
    for (int s = 0; s < kStatsDepth; ++s) {
      const int64_t r = p + s * step;
      buf[s] = r < a.rows ? __ldg(a.x + r * a.vecs + v) : make_uint4(0, 0, 0, 0);
    }
    for (int i0 = 0; i0 < a.loop_count; i0 += kStatsDepth) {
#pragma unroll
      for (int s = 0; s < kStatsDepth; ++s) {
        // The buffer turns over whether or not step i runs (a load past the last iteration is past
        // the last row, so it reads nothing): a conditional turnover would make the compiler copy
        // the register a load is still filling, and wait for that load.
        const int i = i0 + s;
        const int64_t row = p + (int64_t)i * step;
        const uint4 q = buf[s];
        const int64_t r = row + kStatsDepth * step;
        buf[s] = r < a.rows ? __ldg(a.x + r * a.vecs + v) : make_uint4(0, 0, 0, 0);
        if (i < a.loop_count) {
          // A chain's valid slots are a prefix of its iterations, so a valid slot of iteration i
          // has count i + 1.
          const bool valid = row < a.rows;
          if (valid) ++n;
          const float inv = valid ? __frcp_rn(__int2float_rn(i + 1)) : 0.0f;
          const float vf = valid ? 1.0f : 0.0f;
#pragma unroll
          for (int k = 0; k < kVec; ++k) {
            const float x = widen(word(q, k >> 1), k & 1);
            const float d0 = __fsub_rn(x, mean[k]);
            mean[k] = __fmaf_rn(d0, inv, mean[k]);
            const float d1 = __fsub_rn(x, mean[k]);
            m2[k] = __fmaf_rn(__fmul_rn(d0, d1), vf, m2[k]);
          }
        }
      }
    }
  }

  // chains 1, 2, 3 into chain 0, in order
  const int tid = threadIdx.y * blockDim.x + threadIdx.x;
  const int nthreads = blockDim.x * blockDim.y;
  const int lanes = min(32, nthreads - (tid & ~31));
  const unsigned mask = lanes == 32 ? 0xffffffffu : (1u << lanes) - 1u;
  // (every lane runs the merge on what it reads, so all reads of a value precede its update)
  int nb[kStatsChains];
#pragma unroll
  for (int c = 1; c < kStatsChains; ++c) nb[c] = __shfl_sync(mask, n, c, kStatsChains);
#pragma unroll
  for (int k = 0; k < kVec; ++k) {
    float mean_b[kStatsChains], m2_b[kStatsChains];
#pragma unroll
    for (int c = 1; c < kStatsChains; ++c) {
      mean_b[c] = __shfl_sync(mask, mean[k], c, kStatsChains);
      m2_b[c] = __shfl_sync(mask, m2[k], c, kStatsChains);
    }
    int na = n;
#pragma unroll
    for (int c = 1; c < kStatsChains; ++c) {
      welford_merge<true>(na, mean[k], m2[k], nb[c], mean_b[c], m2_b[c]);
      na += nb[c];
    }
  }
#pragma unroll
  for (int c = 1; c < kStatsChains; ++c) n += nb[c];

  // ATen's welford_merge_block_vertical over ty, lane 0 of each chain group
  const int slot = ty * tile + vx;
  for (int off = a.block_y / 2; off > 0; off >>= 1) {
    if (j == 0 && ty < 2 * off) {
#pragma unroll
      for (int k = 0; k < kVec; ++k) {
        s_mean[slot][k] = mean[k];
        s_m2[slot][k] = m2[k];
      }
      s_n[slot] = n;
    }
    __syncthreads();
    if (j == 0 && ty < off) {
      const int o = slot + off * tile;
      const int nb = s_n[o];
#pragma unroll
      for (int k = 0; k < kVec; ++k)
        welford_merge<false>(n, mean[k], m2[k], nb, s_mean[o][k], s_m2[o][k]);
      n += nb;
    }
    __syncthreads();
  }
  if (j != 0 || ty != 0 || !live) return;
  if (a.grid_y == 1) {
#pragma unroll
    for (int k = 0; k < kVec; ++k) stats_finish(a, v * kVec + k, n, mean[k], m2[k]);
    return;
  }
  const int64_t base = (int64_t)blockIdx.y * a.channels + v * kVec;
#pragma unroll
  for (int k = 0; k < kVec; ++k) {
    a.ws_mean[base + k] = mean[k];
    a.ws_m2[base + k] = m2[k];
  }
  if (v == 0) a.ws_count[blockIdx.y] = n;
}

// ATen's last-block merge: blockDim = (kStatsThreads / block_y, block_y), one channel per column.
// Lane ty folds logical blocks ty, ty + block_y, ... into the zero state, then the vertical tree.
__global__ void __launch_bounds__(kStatsThreads) bn_stats_finish_kernel(const StatsArgs a) {
  __shared__ float s_mean[kStatsThreads], s_m2[kStatsThreads];
  __shared__ int s_n[kStatsThreads];
  const int cols = blockDim.x, ty = threadIdx.y;
  const int c = blockIdx.x * cols + threadIdx.x;
  const bool live = c < a.channels;
  int n = 0;
  float mean = 0.0f, m2 = 0.0f;
  if (live) {
    for (int y = ty; y < a.grid_y; y += a.block_y) {
      const int64_t o = (int64_t)y * a.channels + c;
      const int nb = a.ws_count[y];
      welford_merge<false>(n, mean, m2, nb, a.ws_mean[o], a.ws_m2[o]);
      n += nb;
    }
  }
  const int slot = ty * cols + threadIdx.x;
  for (int off = a.block_y / 2; off > 0; off >>= 1) {
    if (ty < 2 * off) {
      s_mean[slot] = mean;
      s_m2[slot] = m2;
      s_n[slot] = n;
    }
    __syncthreads();
    if (ty < off) {
      const int o = slot + off * cols;
      welford_merge<false>(n, mean, m2, s_n[o], s_mean[o], s_m2[o]);
      n += s_n[o];
    }
    __syncthreads();
  }
  if (ty == 0 && live) stats_finish(a, c, n, mean, m2);
}

// ---- backward ---------------------------------------------------------------------------------
// threshold_backward(gy, y, 0) and native_batch_norm_backward in one reduction and one elementwise
// pass.  The mask is threshold_backward's: dz = (v <= 0) ? +0 : gy, so a NaN v passes gy and ±0 masks.
// Modes 1 and 2 may take y's gradient in two halves (a residual block's output feeds both the next
// block's conv1 and its shortcut): the reduction then forms gy = bf16(f(gy) + f(gy2)) per element
// before the mask, which is what autograd's sum of the two, ATen's CUDAFunctor_add<BFloat16> with
// alpha 1, computes.  Its sm_90 code is one float add of the widened operands (a fma by alpha = 1
// rounds the same way) and one round-to-nearest-even conversion: NaN in either operand gives the
// canonical NaN, inf + -inf the canonical NaN, -0 + -0 = -0, +0 + -0 = +0, and a sum past bf16's
// range rounds to inf.  Every case is symmetric, so which half autograd holds first does not matter.
// The arithmetic is that of ATen's batch_norm_backward_reduce_channels_last_kernel<4, BFloat16, float,
// BFloat16> and batch_norm_backward_elemt_channels_last_kernel, pinned as the sm_90 code of torch's
// libtorch_cuda.so performs it (cuobjdump -sass):
//   reduce    sum_dy = sum_dy + dz; sum_dy_xmu = fma(x - mean, dz, sum_dy_xmu), per chain; a slot
//             past the last row is still executed with dz = x = 0 (an infinite mean makes it NaN)
//   merges    plain float adds: chains 1, 2, 3 into chain 0 in order, then ATen's
//             merge_block_vertical_backward tree, then the grid merge (lane ty adds logical blocks
//             ty, ty + block_y, ... to 0.0, then the tree again)
//   finish    grad_bias = bf16(sum_dy); grad_weight = bf16(sum_dy_xmu * invstd)
//   elemt     dx = bf16(fma(-f1, x - mean, fma(-sum_dy, n, dz)) * f2), with per channel
//             f1 = ((invstd * invstd) * sum_dy_xmu) * n and f2 = weight * invstd, and n = float(1.0 / M)
//             formed in double on the host (ATen passes it as a kernel argument)
// The logical geometry is bn_stats_geom.h's (ATen launches the reduction with the same coop
// configuration).  Physically, the 4 chains of a logical thread run on 4 adjacent lanes, one chain
// per lane on an 8-channel vector; lane 0 then adds lanes 1, 2, 3 in order.  That gives the
// 64-channel sites 4x the threads a chain-per-thread mapping has.
struct BwdSide {
  const uint4* x;
  const float* mean;
  const float* invstd;
  const __nv_bfloat16* weight;
  float* sum_xmu;                  // float[channels]: the reduction's sum_dy_xmu
  float* ws_xmu;                   // grid_y > 1: float[grid_y][channels] partials
  __nv_bfloat16* grad_weight;      // may be null
  __nv_bfloat16* grad_bias;        // may be null
  uint4* dx;                       // may be null
};

struct BwdArgs {
  BwdSide a;                       // the main batch norm
  BwdSide d;                       // mode 2: the downsample batch norm
  const uint4* gy;
  const uint4* gy2;                // modes 1, 2: y's second gradient, summed with gy (may be null)
  const uint4* y;                  // modes 1, 2: the saved output, the mask's v
  uint4* dz;                       // modes 1, 2: the masked gradient, written by the reduction
  const __nv_bfloat16* bias;       // mode 0: for the recomputed v
  float* sum_dy;                   // float[channels]
  float* ws_dy;                    // grid_y > 1: float[grid_y][channels] partials
  float norm;                      // float(1.0 / rows)
  int rows;
  int channels;
  int vecs;
  int block_y;
  int grid_y;
  int loop_count;
};

constexpr int kBwdPartialThreads = 512;  // physical threads per block of the reduction
// chain steps loaded ahead of the one computed (mode 1 loads three streams a step, four with gy2;
// mode 2 four, five with gy2): the most that fit 128 registers without spilling
template <int kMode>
constexpr int kBwdDepth = kMode == 2 ? 2 : kMode == 1 ? 3 : 4;
constexpr int kBwdStreams = 5;           // gy, x, y, xd, gy2

__device__ __forceinline__ float relu_grad(float g, float v) { return v <= 0.0f ? 0.0f : g; }

__device__ __forceinline__ void load_bwd_column(const BwdSide& s, const __nv_bfloat16* bias, int v,
                                                Column& c) {
#pragma unroll
  for (int k = 0; k < kVec; ++k) {
    const int ch = v * kVec + k;
    c.mean[k] = s.mean[ch];
    c.inv[k] = s.invstd[ch];
    c.w[k] = __bfloat162float(s.weight[ch]);
    c.b[k] = bias ? __bfloat162float(bias[ch]) : 0.0f;
  }
}

// q = {gy, x, y, xd, gy2} of row r, zeros past the last row
template <int kMode, bool kTwo>
__device__ __forceinline__ void load_bwd_row(const BwdArgs& a, int v, int64_t r,
                                             uint4 (&q)[kBwdStreams]) {
  const uint4 zero = make_uint4(0, 0, 0, 0);
#pragma unroll
  for (int t = 0; t < kBwdStreams; ++t) q[t] = zero;
  if (r < a.rows) {
    const int64_t i = r * a.vecs + v;
    q[0] = __ldg(a.gy + i);
    q[1] = __ldg(a.a.x + i);
    if (kMode != 0) q[2] = __ldg(a.y + i);
    if (kMode == 2) q[3] = __ldg(a.d.x + i);
    if (kTwo) q[4] = __ldg(a.gy2 + i);
  }
}

template <int kMode>
__device__ __forceinline__ void bwd_finish(const BwdArgs& a, int c, float dy, float xmu,
                                           float xmu_d) {
  a.sum_dy[c] = dy;
  a.a.sum_xmu[c] = xmu;
  if (a.a.grad_bias) a.a.grad_bias[c] = __float2bfloat16_rn(dy);
  if (a.a.grad_weight) a.a.grad_weight[c] = __float2bfloat16_rn(__fmul_rn(xmu, a.a.invstd[c]));
  if (kMode == 2) {
    a.d.sum_xmu[c] = xmu_d;
    if (a.d.grad_bias) a.d.grad_bias[c] = __float2bfloat16_rn(dy);
    if (a.d.grad_weight) a.d.grad_weight[c] = __float2bfloat16_rn(__fmul_rn(xmu_d, a.d.invstd[c]));
  }
}

// blockDim = (4 * tile, block_y): lane j = threadIdx.x % 4 of thread (vx = threadIdx.x / 4, ty) of
// block (bx, by) runs chain j of logical thread (by, ty) on vector bx * tile + vx.  kTwo: gy is the
// sum of gy and gy2.
template <int kMode, bool kTwo>
__global__ void __launch_bounds__(kBwdPartialThreads) bn_bwd_partial_kernel(const BwdArgs a) {
  constexpr int kSlots = kBwdPartialThreads / kStatsChains;
  __shared__ float s_dy[kSlots][kVec];
  __shared__ float s_xmu[kSlots][kVec];
  __shared__ float s_xmu_d[kMode == 2 ? kSlots : 1][kVec];
  const int j = threadIdx.x % kStatsChains, tile = blockDim.x / kStatsChains, ty = threadIdx.y;
  const int vx = threadIdx.x / kStatsChains;
  const int v = blockIdx.x * tile + vx;
  const bool live = v < a.vecs;
  const int64_t stride = (int64_t)a.block_y * a.grid_y;
  const int64_t step = kStatsChains * stride;
  const int64_t p = (int64_t)blockIdx.y * a.block_y + ty + j * stride;

  float dy[kVec], xmu[kVec], xmu_d[kVec];
#pragma unroll
  for (int k = 0; k < kVec; ++k) dy[k] = xmu[k] = xmu_d[k] = 0.0f;

  if (live) {
    Column ca, cd;
    load_bwd_column(a.a, kMode == 0 ? a.bias : nullptr, v, ca);
    if (kMode == 2) load_bwd_column(a.d, nullptr, v, cd);
    uint4 buf[kBwdDepth<kMode>][kBwdStreams];
#pragma unroll
    for (int s = 0; s < kBwdDepth<kMode>; ++s) load_bwd_row<kMode, kTwo>(a, v, p + s * step, buf[s]);
    for (int i0 = 0; i0 < a.loop_count; i0 += kBwdDepth<kMode>) {
#pragma unroll
      for (int s = 0; s < kBwdDepth<kMode>; ++s) {
        // unconditional turnover, as in bn_stats_partial_kernel
        const int64_t row = p + (int64_t)(i0 + s) * step;
        uint4 q[kBwdStreams];
#pragma unroll
        for (int t = 0; t < kBwdStreams; ++t) q[t] = buf[s][t];
        load_bwd_row<kMode, kTwo>(a, v, row + kBwdDepth<kMode> * step, buf[s]);
        if (i0 + s < a.loop_count) {
          uint32_t dz_bits[4];
#pragma unroll
          for (int k = 0; k < kVec; ++k) {
            const int w = k >> 1, h = k & 1;
            const float x = widen(word(q[1], w), h);
            const float v_mask = kMode == 0 ? bn_apply(x, ca, k) : widen(word(q[2], w), h);
            float g = widen(word(q[0], w), h);
            if (kTwo) g = __uint_as_float(bf16_bits(__fadd_rn(g, widen(word(q[4], w), h))) << 16);
            const float dz = relu_grad(g, v_mask);
            dy[k] = __fadd_rn(dy[k], dz);
            xmu[k] = __fmaf_rn(__fsub_rn(x, ca.mean[k]), dz, xmu[k]);
            if (kMode == 2)
              xmu_d[k] = __fmaf_rn(__fsub_rn(widen(word(q[3], w), h), cd.mean[k]), dz, xmu_d[k]);
            const uint32_t b = __float_as_uint(dz) >> 16;
            dz_bits[w] = h ? (dz_bits[w] | (b << 16)) : b;
          }
          if (kMode != 0 && row < a.rows)
            a.dz[row * a.vecs + v] = make_uint4(dz_bits[0], dz_bits[1], dz_bits[2], dz_bits[3]);
        }
      }
    }
  }

  // chains 1, 2, 3 into chain 0, in order
  const int tid = threadIdx.y * blockDim.x + threadIdx.x;
  const int nthreads = blockDim.x * blockDim.y;
  const int lanes = min(32, nthreads - (tid & ~31));
  const unsigned mask = lanes == 32 ? 0xffffffffu : (1u << lanes) - 1u;
#pragma unroll
  for (int k = 0; k < kVec; ++k) {
    float o[kStatsChains], od[kStatsChains], odd[kStatsChains];
#pragma unroll
    for (int c = 1; c < kStatsChains; ++c) {
      o[c] = __shfl_sync(mask, dy[k], c, kStatsChains);
      od[c] = __shfl_sync(mask, xmu[k], c, kStatsChains);
      if (kMode == 2) odd[c] = __shfl_sync(mask, xmu_d[k], c, kStatsChains);
    }
#pragma unroll
    for (int c = 1; c < kStatsChains; ++c) {
      dy[k] = __fadd_rn(dy[k], o[c]);
      xmu[k] = __fadd_rn(xmu[k], od[c]);
      if (kMode == 2) xmu_d[k] = __fadd_rn(xmu_d[k], odd[c]);
    }
  }

  // ATen's merge_block_vertical_backward over ty, lane 0 of each chain group
  const int slot = ty * tile + vx;
  for (int off = a.block_y / 2; off > 0; off >>= 1) {
    if (j == 0 && ty < 2 * off) {
#pragma unroll
      for (int k = 0; k < kVec; ++k) {
        s_dy[slot][k] = dy[k];
        s_xmu[slot][k] = xmu[k];
        if (kMode == 2) s_xmu_d[slot][k] = xmu_d[k];
      }
    }
    __syncthreads();
    if (j == 0 && ty < off) {
      const int o = slot + off * tile;
#pragma unroll
      for (int k = 0; k < kVec; ++k) {
        dy[k] = __fadd_rn(dy[k], s_dy[o][k]);
        xmu[k] = __fadd_rn(xmu[k], s_xmu[o][k]);
        if (kMode == 2) xmu_d[k] = __fadd_rn(xmu_d[k], s_xmu_d[o][k]);
      }
    }
    __syncthreads();
  }
  if (j != 0 || ty != 0 || !live) return;
  if (a.grid_y == 1) {
#pragma unroll
    for (int k = 0; k < kVec; ++k) bwd_finish<kMode>(a, v * kVec + k, dy[k], xmu[k], xmu_d[k]);
    return;
  }
  const int64_t base = (int64_t)blockIdx.y * a.channels + v * kVec;
#pragma unroll
  for (int k = 0; k < kVec; ++k) {
    a.ws_dy[base + k] = dy[k];
    a.a.ws_xmu[base + k] = xmu[k];
    if (kMode == 2) a.d.ws_xmu[base + k] = xmu_d[k];
  }
}

// ATen's last-block merge: blockDim = (kStatsThreads / block_y, block_y), one channel per column.
template <int kMode>
__global__ void __launch_bounds__(kStatsThreads) bn_bwd_finish_kernel(const BwdArgs a) {
  __shared__ float s_dy[kStatsThreads], s_xmu[kStatsThreads];
  __shared__ float s_xmu_d[kMode == 2 ? kStatsThreads : 1];
  const int cols = blockDim.x, ty = threadIdx.y;
  const int c = blockIdx.x * cols + threadIdx.x;
  const bool live = c < a.channels;
  float dy = 0.0f, xmu = 0.0f, xmu_d = 0.0f;
  if (live) {
    for (int y = ty; y < a.grid_y; y += a.block_y) {
      const int64_t o = (int64_t)y * a.channels + c;
      dy = __fadd_rn(dy, a.ws_dy[o]);
      xmu = __fadd_rn(xmu, a.a.ws_xmu[o]);
      if (kMode == 2) xmu_d = __fadd_rn(xmu_d, a.d.ws_xmu[o]);
    }
  }
  const int slot = ty * cols + threadIdx.x;
  for (int off = a.block_y / 2; off > 0; off >>= 1) {
    if (ty < 2 * off) {
      s_dy[slot] = dy;
      s_xmu[slot] = xmu;
      if (kMode == 2) s_xmu_d[slot] = xmu_d;
    }
    __syncthreads();
    if (ty < off) {
      const int o = slot + off * cols;
      dy = __fadd_rn(dy, s_dy[o]);
      xmu = __fadd_rn(xmu, s_xmu[o]);
      if (kMode == 2) xmu_d = __fadd_rn(xmu_d, s_xmu_d[o]);
    }
    __syncthreads();
  }
  if (ty == 0 && live) bwd_finish<kMode>(a, c, dy, xmu, xmu_d);
}

// dx = bf16(fma(-f1, x - mean, fma(-sum_dy, n, dz)) * f2) per side; the forward's physical scheme
struct BwdColumn {
  float mean[kVec], f1[kVec], f2[kVec];
};

__device__ __forceinline__ void load_elemt_column(const BwdSide& s, float norm, int v, BwdColumn& c) {
#pragma unroll
  for (int k = 0; k < kVec; ++k) {
    const int ch = v * kVec + k;
    const float inv = s.invstd[ch];
    c.mean[k] = s.mean[ch];
    c.f1[k] = __fmul_rn(__fmul_rn(__fmul_rn(inv, inv), s.sum_xmu[ch]), norm);
    c.f2[k] = __fmul_rn(__bfloat162float(s.weight[ch]), inv);
  }
}

__device__ __forceinline__ uint32_t elemt_bits(float t, float x, const BwdColumn& c, int k) {
  return bf16_bits(__fmul_rn(__fmaf_rn(-c.f1[k], __fsub_rn(x, c.mean[k]), t), c.f2[k]));
}

template <int kMode>
__global__ void __launch_bounds__(kBnThreads) bn_bwd_elemt_kernel(const BwdArgs p) {
  const int v = blockIdx.y * blockDim.x + threadIdx.x;
  if (v >= p.vecs) return;
  BwdColumn ea, ed;
  Column ca;  // mode 0: the forward's parameters, for the mask
  float sdy[kVec];
  load_elemt_column(p.a, p.norm, v, ea);
  if (kMode == 2) load_elemt_column(p.d, p.norm, v, ed);
  if (kMode == 0) load_bwd_column(p.a, p.bias, v, ca);
#pragma unroll
  for (int k = 0; k < kVec; ++k) sdy[k] = p.sum_dy[v * kVec + k];
  const uint4* g = kMode == 0 ? p.gy : p.dz;

  const int64_t stride = (int64_t)gridDim.x * blockDim.y;
  const uint4 zero = make_uint4(0, 0, 0, 0);
  for (int64_t row = (int64_t)blockIdx.x * blockDim.y + threadIdx.y; row < p.rows;
       row += stride * kRowUnroll) {
    uint4 qg[kRowUnroll], qx[kRowUnroll], qd[kRowUnroll];
#pragma unroll
    for (int u = 0; u < kRowUnroll; ++u) {
      const int64_t r = row + u * stride;
      qg[u] = qx[u] = qd[u] = zero;
      if (r < p.rows) {
        const int64_t i = r * p.vecs + v;
        qg[u] = __ldg(g + i);
        qx[u] = __ldg(p.a.x + i);
        if (kMode == 2) qd[u] = __ldg(p.d.x + i);
      }
    }
#pragma unroll
    for (int u = 0; u < kRowUnroll; ++u) {
      const int64_t r = row + u * stride;
      if (r >= p.rows) continue;
      uint32_t oa[4], od[4];
#pragma unroll
      for (int k = 0; k < kVec; ++k) {
        const int w = k >> 1, h = k & 1;
        const float x = widen(word(qx[u], w), h);
        float dz = widen(word(qg[u], w), h);
        if (kMode == 0) dz = relu_grad(dz, bn_apply(x, ca, k));
        const float t = __fmaf_rn(-sdy[k], p.norm, dz);
        const uint32_t ba = elemt_bits(t, x, ea, k);
        oa[w] = h ? (oa[w] | (ba << 16)) : ba;
        if (kMode == 2) {
          const uint32_t bd = elemt_bits(t, widen(word(qd[u], w), h), ed, k);
          od[w] = h ? (od[w] | (bd << 16)) : bd;
        }
      }
      const int64_t i = r * p.vecs + v;
      if (p.a.dx) p.a.dx[i] = make_uint4(oa[0], oa[1], oa[2], oa[3]);
      if (kMode == 2 && p.d.dx) p.d.dx[i] = make_uint4(od[0], od[1], od[2], od[3]);
    }
  }
}

}  // namespace

// ---- host side --------------------------------------------------------------------------------
int device_ready() {
  static const int ok = [] {
    int n = 0;
    return cudaGetDeviceCount(&n) == cudaSuccess && n > 0 ? 1 : 0;
  }();
  return ok;
}

namespace {

struct DevInfo {
  std::atomic<int> sms{0};
};
constexpr int kMaxDevices = 64;
DevInfo g_dev[kMaxDevices];
std::atomic<int> g_blocks_per_sm[6];  // forward modes 0-2, then the backward's elementwise modes

// One thread per 8-channel vector column, walking rows with a grid stride; the grid is sized from
// the SM count and the kernel's occupancy.  `slot` caches that occupancy.
template <typename Args>
int launch_rows(void (*kernel)(Args), int slot, const Args& a, int64_t rows, int vecs,
                void* stream) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices)
    return fail(TOK_ERR_CUDA, "bn_fused: no current CUDA device");
  int sms = g_dev[dev].sms.load(std::memory_order_relaxed);
  if (sms == 0) {
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 1;
    g_dev[dev].sms.store(sms, std::memory_order_relaxed);
  }
  int per_sm = g_blocks_per_sm[slot].load(std::memory_order_relaxed);
  if (per_sm == 0) {
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kBnThreads, 0);
    if (per_sm <= 0) per_sm = 1;
    g_blocks_per_sm[slot].store(per_sm, std::memory_order_relaxed);
  }
  const int tile = vecs < kMaxTileVecs ? vecs : kMaxTileVecs;
  const dim3 block(tile, kBnThreads / tile);
  const int tiles = (vecs + tile - 1) / tile;
  const int64_t row_blocks = (rows + block.y - 1) / block.y;
  int64_t want = (int64_t)sms * per_sm / tiles;
  if (want < 1) want = 1;
  const dim3 grid((unsigned)(row_blocks < want ? row_blocks : want), tiles);
  kernel<<<grid, block, 0, (cudaStream_t)stream>>>(a);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(TOK_ERR_CUDA, "bn_fused launch: %s", cudaGetErrorString(e));
  return TOK_OK;
}

template <int kMode>
int launch(const BnArgs& a, void* stream) {
  return launch_rows(bn_fused_fwd_kernel<kMode>, kMode, a, a.rows, a.vecs, stream);
}

bool misaligned(const void* p) { return ((uintptr_t)p & 15u) != 0; }

int check_side(const char* who, const void* x, const float* mean, const float* var,
               const void* weight, const void* bias, float* invstd) {
  if (!x || !mean || !var || !weight || !bias || !invstd)
    return fail(TOK_ERR_INVALID, "%s: null pointer argument", who);
  if (misaligned(x)) return fail(TOK_ERR_ALIGN, "%s: activation is not 16-byte aligned", who);
  return TOK_OK;
}

int check_shape(const char* who, const void* y, int64_t rows, int channels) {
  if (!y) return fail(TOK_ERR_INVALID, "%s: null output", who);
  if (rows <= 0 || channels <= 0)
    return fail(TOK_ERR_INVALID, "%s: rows %lld and channels %d must be positive", who,
                (long long)rows, channels);
  if (channels % kVec != 0)
    return fail(TOK_ERR_ALIGN, "%s: channels %d is not a multiple of %d", who, channels, kVec);
  if ((channels / kVec + kMaxTileVecs - 1) / kMaxTileVecs > 65535)
    return fail(TOK_ERR_INVALID, "%s: %d channels are too many", who, channels);
  if (misaligned(y)) return fail(TOK_ERR_ALIGN, "%s: output is not 16-byte aligned", who);
  if (!device_ready()) return fail(TOK_ERR_NO_DEVICE, "%s needs a CUDA GPU (no CPU fallback)", who);
  return TOK_OK;
}

BnSide side(const void* x, const float* mean, const float* var, const void* weight,
            const void* bias, float eps, float* invstd) {
  return BnSide{(const uint4*)x, mean, var, (const __nv_bfloat16*)weight,
                (const __nv_bfloat16*)bias, invstd, eps};
}

int check_stats_shape(const char* who, int64_t rows, int channels) {
  if (rows <= 0 || channels <= 0)
    return fail(TOK_ERR_INVALID, "%s: rows %lld and channels %d must be positive", who,
                (long long)rows, channels);
  if (rows * channels > INT32_MAX)
    return fail(TOK_ERR_INVALID, "%s: %lld x %d elements exceed 32-bit indexing", who,
                (long long)rows, channels);
  if (channels % kVec != 0)
    return fail(TOK_ERR_ALIGN, "%s: channels %d is not a multiple of %d", who, channels, kVec);
  return TOK_OK;
}

int check_act(const char* who, const char* what, const void* p, bool required) {
  if (!p) return required ? fail(TOK_ERR_INVALID, "%s: null %s", who, what) : TOK_OK;
  if (misaligned(p)) return fail(TOK_ERR_ALIGN, "%s: %s is not 16-byte aligned", who, what);
  return TOK_OK;
}

BwdSide bwd_side(const void* x, const float* mean, const float* invstd, const void* weight,
                 void* dx, void* grad_weight, void* grad_bias) {
  BwdSide s{};
  s.x = (const uint4*)x;
  s.mean = mean;
  s.invstd = invstd;
  s.weight = (const __nv_bfloat16*)weight;
  s.grad_weight = (__nv_bfloat16*)grad_weight;
  s.grad_bias = (__nv_bfloat16*)grad_bias;
  s.dx = (uint4*)dx;
  return s;
}

// Checks what every mode shares, lays the workspace out and runs the reduction, its finish and
// (when a dx is asked for) the elementwise pass.  kTwo: y's gradient comes in two halves, gy + gy2.
template <int kMode, bool kTwo>
int bn_bwd(const char* who, BwdArgs& a, int64_t rows, int channels, void* workspace,
           void* cuda_stream) {
  int rc = check_stats_shape(who, rows, channels);
  if (rc == TOK_OK) rc = check_act(who, "gy", a.gy, true);
  if (rc == TOK_OK && kTwo) rc = check_act(who, "gy2", a.gy2, true);
  if (rc == TOK_OK) rc = check_act(who, "x", a.a.x, true);
  if (rc == TOK_OK) rc = check_act(who, "dx", a.a.dx, false);
  if (rc == TOK_OK && kMode != 0) rc = check_act(who, "y", a.y, true);
  if (rc == TOK_OK && kMode != 0) rc = check_act(who, "dz", a.dz, true);
  if (rc == TOK_OK && kMode == 2) rc = check_act(who, "xd", a.d.x, true);
  if (rc == TOK_OK && kMode == 2) rc = check_act(who, "dxd", a.d.dx, false);
  if (rc == TOK_OK) rc = check_act(who, "workspace", workspace, true);
  if (rc != TOK_OK) return rc;
  if (!a.a.mean || !a.a.invstd || !a.a.weight || (kMode == 0 && !a.bias) ||
      (kMode == 2 && (!a.d.mean || !a.d.invstd || !a.d.weight)))
    return fail(TOK_ERR_INVALID, "%s: null pointer argument", who);
  if (!device_ready()) return fail(TOK_ERR_NO_DEVICE, "%s needs a CUDA GPU (no CPU fallback)", who);

  const BnStatsGeom g = bn_stats_geometry((int)rows, channels);
  const int sums = kMode == 2 ? 3 : 2;
  float* f = (float*)workspace;
  a.sum_dy = f;
  a.a.sum_xmu = f + channels;
  if (kMode == 2) a.d.sum_xmu = f + 2 * channels;
  if (g.grid_y > 1) {
    float* part = f + (int64_t)sums * channels;
    const int64_t n = (int64_t)g.grid_y * channels;
    a.ws_dy = part;
    a.a.ws_xmu = part + n;
    if (kMode == 2) a.d.ws_xmu = part + 2 * n;
  }
  a.rows = (int)rows;
  a.channels = channels;
  a.vecs = channels / kVec;
  a.block_y = g.block_y;
  a.grid_y = g.grid_y;
  a.loop_count = g.loop_count;
  a.norm = (float)(1.0 / (double)rows);  // ATen: norm_fct = 1.0 / reduction_size, passed as float

  int tile = kBwdPartialThreads / (kStatsChains * g.block_y);
  if (tile > a.vecs) tile = a.vecs;
  cudaStream_t st = (cudaStream_t)cuda_stream;
  bn_bwd_partial_kernel<kMode, kTwo><<<dim3((a.vecs + tile - 1) / tile, g.grid_y),
                                       dim3(kStatsChains * tile, g.block_y), 0, st>>>(a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(TOK_ERR_CUDA, "bn_bwd_partial launch: %s", cudaGetErrorString(e));
  if (g.grid_y > 1) {
    const int cols = kStatsThreads / g.block_y;
    bn_bwd_finish_kernel<kMode><<<(channels + cols - 1) / cols, dim3(cols, g.block_y), 0, st>>>(a);
    e = cudaGetLastError();
    if (e != cudaSuccess) return fail(TOK_ERR_CUDA, "bn_bwd_finish launch: %s", cudaGetErrorString(e));
  }
  if (!a.a.dx && !(kMode == 2 && a.d.dx)) return TOK_OK;
  return launch_rows(bn_bwd_elemt_kernel<kMode>, 3 + kMode, a, rows, a.vecs, cuda_stream);
}

}  // namespace
}  // namespace tok

using namespace tok;

extern "C" int tok_bn_relu_fwd(const void* x, const float* mean, const float* var,
                               const void* weight, const void* bias, float eps, float* invstd,
                               void* y, int64_t rows, int channels, void* cuda_stream) {
  int rc = check_side("tok_bn_relu_fwd", x, mean, var, weight, bias, invstd);
  if (rc == TOK_OK) rc = check_shape("tok_bn_relu_fwd", y, rows, channels);
  if (rc != TOK_OK) return rc;
  BnArgs a{};
  a.a = side(x, mean, var, weight, bias, eps, invstd);
  a.y = (uint4*)y;
  a.rows = rows;
  a.vecs = channels / kVec;
  return launch<0>(a, cuda_stream);
}

extern "C" int tok_bn_add_relu_fwd(const void* x, const float* mean, const float* var,
                                   const void* weight, const void* bias, float eps, float* invstd,
                                   const void* residual, void* y, int64_t rows, int channels,
                                   void* cuda_stream) {
  int rc = check_side("tok_bn_add_relu_fwd", x, mean, var, weight, bias, invstd);
  if (rc == TOK_OK && !residual) rc = fail(TOK_ERR_INVALID, "tok_bn_add_relu_fwd: null residual");
  if (rc == TOK_OK && misaligned(residual))
    rc = fail(TOK_ERR_ALIGN, "tok_bn_add_relu_fwd: residual is not 16-byte aligned");
  if (rc == TOK_OK) rc = check_shape("tok_bn_add_relu_fwd", y, rows, channels);
  if (rc != TOK_OK) return rc;
  BnArgs a{};
  a.a = side(x, mean, var, weight, bias, eps, invstd);
  a.res = (const uint4*)residual;
  a.y = (uint4*)y;
  a.rows = rows;
  a.vecs = channels / kVec;
  return launch<1>(a, cuda_stream);
}

extern "C" int tok_bn2_add_relu_fwd(const void* x, const float* mean, const float* var,
                                    const void* weight, const void* bias, float eps, float* invstd,
                                    const void* xd, const float* mean_d, const float* var_d,
                                    const void* weight_d, const void* bias_d, float eps_d,
                                    float* invstd_d, void* y, int64_t rows, int channels,
                                    void* cuda_stream) {
  int rc = check_side("tok_bn2_add_relu_fwd", x, mean, var, weight, bias, invstd);
  if (rc == TOK_OK)
    rc = check_side("tok_bn2_add_relu_fwd (downsample)", xd, mean_d, var_d, weight_d, bias_d,
                    invstd_d);
  if (rc == TOK_OK) rc = check_shape("tok_bn2_add_relu_fwd", y, rows, channels);
  if (rc != TOK_OK) return rc;
  BnArgs a{};
  a.a = side(x, mean, var, weight, bias, eps, invstd);
  a.d = side(xd, mean_d, var_d, weight_d, bias_d, eps_d, invstd_d);
  a.y = (uint4*)y;
  a.rows = rows;
  a.vecs = channels / kVec;
  return launch<2>(a, cuda_stream);
}

extern "C" int64_t tok_bn_stats_workspace_bytes(int64_t rows, int channels) {
  const int rc = check_stats_shape("tok_bn_stats_workspace_bytes", rows, channels);
  if (rc != TOK_OK) return rc;
  return bn_stats_workspace(bn_stats_geometry((int)rows, channels), channels);
}

extern "C" int tok_bn_stats_fwd(const void* x, int64_t rows, int channels, double momentum,
                                void* running_mean, void* running_var, void* workspace,
                                float* mean, float* var, void* cuda_stream) {
  const char* who = "tok_bn_stats_fwd";
  if (!x || !running_mean || !running_var || !mean || !var)
    return fail(TOK_ERR_INVALID, "%s: null pointer argument", who);
  int rc = check_stats_shape(who, rows, channels);
  if (rc != TOK_OK) return rc;
  if (misaligned(x)) return fail(TOK_ERR_ALIGN, "%s: activation is not 16-byte aligned", who);
  const BnStatsGeom g = bn_stats_geometry((int)rows, channels);
  const int64_t ws_bytes = bn_stats_workspace(g, channels);
  if (ws_bytes > 0 && !workspace)
    return fail(TOK_ERR_INVALID, "%s: null workspace (%lld bytes needed)", who, (long long)ws_bytes);
  if (ws_bytes > 0 && misaligned(workspace))
    return fail(TOK_ERR_ALIGN, "%s: workspace is not 16-byte aligned", who);
  if (!device_ready()) return fail(TOK_ERR_NO_DEVICE, "%s needs a CUDA GPU (no CPU fallback)", who);

  StatsArgs a{};
  a.x = (const uint4*)x;
  if (ws_bytes > 0) {
    const int64_t counts = ws_bytes - 2 * (int64_t)g.grid_y * channels * 4;
    a.ws_count = (int*)workspace;
    a.ws_mean = (float*)((char*)workspace + counts);
    a.ws_m2 = a.ws_mean + (int64_t)g.grid_y * channels;
  }
  a.mean = mean;
  a.var = var;
  a.running_mean = (__nv_bfloat16*)running_mean;
  a.running_var = (__nv_bfloat16*)running_var;
  a.rows = (int)rows;
  a.channels = channels;
  a.vecs = channels / kVec;
  a.block_y = g.block_y;
  a.grid_y = g.grid_y;
  a.loop_count = g.loop_count;
  // as ATen's batch_norm_update_stats: float(momentum), float(N / (N - 1)) formed in double
  a.momentum = (float)momentum;
  a.bessel = (float)((double)rows / (double)(rows - 1));

  // the partial kernel: block (4 * tile, block_y), one chain of an 8-channel vector per lane
  int tile = kStatsPartialThreads / (kStatsChains * g.block_y);
  if (tile > a.vecs) tile = a.vecs;
  const dim3 block(kStatsChains * tile, g.block_y);
  const dim3 grid((a.vecs + tile - 1) / tile, g.grid_y);
  cudaStream_t st = (cudaStream_t)cuda_stream;
  bn_stats_partial_kernel<<<grid, block, 0, st>>>(a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(TOK_ERR_CUDA, "bn_stats_partial launch: %s", cudaGetErrorString(e));
  if (g.grid_y > 1) {
    const int cols = kStatsThreads / g.block_y;
    bn_stats_finish_kernel<<<(channels + cols - 1) / cols, dim3(cols, g.block_y), 0, st>>>(a);
    e = cudaGetLastError();
    if (e != cudaSuccess)
      return fail(TOK_ERR_CUDA, "bn_stats_finish launch: %s", cudaGetErrorString(e));
  }
  return TOK_OK;
}

extern "C" int64_t tok_bn_bwd_workspace_bytes(int64_t rows, int channels, int mode) {
  const char* who = "tok_bn_bwd_workspace_bytes";
  const int rc = check_stats_shape(who, rows, channels);
  if (rc != TOK_OK) return rc;
  if (mode < 0 || mode > 2) return fail(TOK_ERR_INVALID, "%s: mode %d is not 0, 1 or 2", who, mode);
  return bn_bwd_workspace(bn_stats_geometry((int)rows, channels), channels, mode == 2 ? 3 : 2);
}

extern "C" int tok_bn_relu_bwd(const void* gy, const void* x, const float* mean,
                               const float* invstd, const void* weight, const void* bias, void* dx,
                               void* grad_weight, void* grad_bias, int64_t rows, int channels,
                               void* workspace, void* cuda_stream) {
  BwdArgs a{};
  a.a = bwd_side(x, mean, invstd, weight, dx, grad_weight, grad_bias);
  a.gy = (const uint4*)gy;
  a.bias = (const __nv_bfloat16*)bias;
  return bn_bwd<0, false>("tok_bn_relu_bwd", a, rows, channels, workspace, cuda_stream);
}

namespace {

template <bool kTwo>
int bn_add_relu_bwd(const char* who, const void* gy, const void* gy2, const void* y, const void* x,
                    const float* mean, const float* invstd, const void* weight, void* dz, void* dx,
                    void* grad_weight, void* grad_bias, int64_t rows, int channels,
                    void* workspace, void* cuda_stream) {
  BwdArgs a{};
  a.a = bwd_side(x, mean, invstd, weight, dx, grad_weight, grad_bias);
  a.gy = (const uint4*)gy;
  a.gy2 = (const uint4*)gy2;
  a.y = (const uint4*)y;
  a.dz = (uint4*)dz;
  return bn_bwd<1, kTwo>(who, a, rows, channels, workspace, cuda_stream);
}

template <bool kTwo>
int bn2_add_relu_bwd(const char* who, const void* gy, const void* gy2, const void* y,
                     const void* x, const float* mean, const float* invstd, const void* weight,
                     const void* xd, const float* mean_d, const float* invstd_d,
                     const void* weight_d, void* dz, void* dx, void* grad_weight, void* grad_bias,
                     void* dxd, void* grad_weight_d, void* grad_bias_d, int64_t rows, int channels,
                     void* workspace, void* cuda_stream) {
  BwdArgs a{};
  a.a = bwd_side(x, mean, invstd, weight, dx, grad_weight, grad_bias);
  a.d = bwd_side(xd, mean_d, invstd_d, weight_d, dxd, grad_weight_d, grad_bias_d);
  a.gy = (const uint4*)gy;
  a.gy2 = (const uint4*)gy2;
  a.y = (const uint4*)y;
  a.dz = (uint4*)dz;
  return bn_bwd<2, kTwo>(who, a, rows, channels, workspace, cuda_stream);
}

}  // namespace

extern "C" int tok_bn_add_relu_bwd(const void* gy, const void* y, const void* x, const float* mean,
                                   const float* invstd, const void* weight, void* dz, void* dx,
                                   void* grad_weight, void* grad_bias, int64_t rows, int channels,
                                   void* workspace, void* cuda_stream) {
  return bn_add_relu_bwd<false>("tok_bn_add_relu_bwd", gy, nullptr, y, x, mean, invstd, weight, dz,
                                dx, grad_weight, grad_bias, rows, channels, workspace, cuda_stream);
}

extern "C" int tok_bn_add_relu_bwd2(const void* gy, const void* gy2, const void* y, const void* x,
                                    const float* mean, const float* invstd, const void* weight,
                                    void* dz, void* dx, void* grad_weight, void* grad_bias,
                                    int64_t rows, int channels, void* workspace,
                                    void* cuda_stream) {
  return bn_add_relu_bwd<true>("tok_bn_add_relu_bwd2", gy, gy2, y, x, mean, invstd, weight, dz, dx,
                               grad_weight, grad_bias, rows, channels, workspace, cuda_stream);
}

extern "C" int tok_bn2_add_relu_bwd(const void* gy, const void* y, const void* x, const float* mean,
                                    const float* invstd, const void* weight, const void* xd,
                                    const float* mean_d, const float* invstd_d,
                                    const void* weight_d, void* dz, void* dx, void* grad_weight,
                                    void* grad_bias, void* dxd, void* grad_weight_d,
                                    void* grad_bias_d, int64_t rows, int channels, void* workspace,
                                    void* cuda_stream) {
  return bn2_add_relu_bwd<false>("tok_bn2_add_relu_bwd", gy, nullptr, y, x, mean, invstd, weight,
                                 xd, mean_d, invstd_d, weight_d, dz, dx, grad_weight, grad_bias,
                                 dxd, grad_weight_d, grad_bias_d, rows, channels, workspace,
                                 cuda_stream);
}

extern "C" int tok_bn2_add_relu_bwd2(const void* gy, const void* gy2, const void* y, const void* x,
                                     const float* mean, const float* invstd, const void* weight,
                                     const void* xd, const float* mean_d, const float* invstd_d,
                                     const void* weight_d, void* dz, void* dx, void* grad_weight,
                                     void* grad_bias, void* dxd, void* grad_weight_d,
                                     void* grad_bias_d, int64_t rows, int channels,
                                     void* workspace, void* cuda_stream) {
  return bn2_add_relu_bwd<true>("tok_bn2_add_relu_bwd2", gy, gy2, y, x, mean, invstd, weight, xd,
                                mean_d, invstd_d, weight_d, dz, dx, grad_weight, grad_bias, dxd,
                                grad_weight_d, grad_bias_d, rows, channels, workspace, cuda_stream);
}
