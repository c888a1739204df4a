// Batch-norm forward apply fused with ReLU and the residual add, NHWC bf16 (training).
//
// The activation of a channels_last [N, C, H, W] tensor is the row-major matrix [M = N*H*W, C].
// The statistics (mean, biased variance) come from ATen's own channels_last statistics kernel; these
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
std::atomic<int> g_blocks_per_sm[3];

template <int kMode>
int launch(const BnArgs& a, void* stream) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices)
    return fail(TOK_ERR_CUDA, "bn_fused: no current CUDA device");
  int sms = g_dev[dev].sms.load(std::memory_order_relaxed);
  if (sms == 0) {
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 1;
    g_dev[dev].sms.store(sms, std::memory_order_relaxed);
  }
  int per_sm = g_blocks_per_sm[kMode].load(std::memory_order_relaxed);
  if (per_sm == 0) {
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, bn_fused_fwd_kernel<kMode>,
                                                  kBnThreads, 0);
    if (per_sm <= 0) per_sm = 1;
    g_blocks_per_sm[kMode].store(per_sm, std::memory_order_relaxed);
  }
  const int tile = a.vecs < kMaxTileVecs ? a.vecs : kMaxTileVecs;
  const dim3 block(tile, kBnThreads / tile);
  const int tiles = (a.vecs + tile - 1) / tile;
  const int64_t row_blocks = (a.rows + block.y - 1) / block.y;
  int64_t want = (int64_t)sms * per_sm / tiles;
  if (want < 1) want = 1;
  const dim3 grid((unsigned)(row_blocks < want ? row_blocks : want), tiles);
  bn_fused_fwd_kernel<kMode><<<grid, block, 0, (cudaStream_t)stream>>>(a);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(TOK_ERR_CUDA, "bn_fused launch: %s", cudaGetErrorString(e));
  return TOK_OK;
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
