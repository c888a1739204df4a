// Logical geometry of the batch-norm statistics reduction (bn_fused.cu), CUDA-free so that the host
// compiler alone can build it (tests/test_bn_stats_cpu.py).
//
// The result bits of a Welford reduction depend on how rows are dealt to chains and in which order
// the chains are merged.  bn_fused.cu reproduces ATen's channels_last statistics kernel
// (batch_norm_collect_statistics_channels_last_kernel, launched by flexible_launch_configs with
// coop = true), so the logical shape here is ATen's, restated from ATen/native/cuda/Normalization.cuh
// with MAX_BLOCK_SIZE = 512 (its value on CUDA; the kernel's 6 KiB of static shared memory confirms
// it in the shipped sm_90 code), ELEMENTS_PER_THREAD = 16, OPTIMAL_TILE_W = 32 and MAX_H_BLOCK = 128.
// Only block_y and grid_y shape the arithmetic; block_x just tiles channels, which never interact.
#pragma once
#include <stdint.h>

namespace tok {

struct BnStatsGeom {
  int block_y;     // logical threads per block along the rows (a power of two)
  int grid_y;      // logical blocks along the rows; > 1 means a cross-block merge
  int loop_count;  // iterations of every logical thread, 4 rows each
};

constexpr int kStatsMaxBlock = 512;
constexpr int kStatsElemsPerThread = 16;
constexpr int kStatsTileW = 32;
constexpr int kStatsMaxHBlock = 128;
constexpr int kStatsChains = 4;  // ATen's PARALLEL_LOADS: independent Welford chains per thread

inline int stats_last_pow2(unsigned n) {
  n |= n >> 1;
  n |= n >> 2;
  n |= n >> 4;
  n |= n >> 8;
  n |= n >> 16;
  const int p = (int)(n - (n >> 1));
  return p > 1 ? p : 1;
}

inline int stats_ceil_div(int a, int b) { return (a + b - 1) / b; }

// rows = N*H*W and channels = C, both positive with rows * channels < 2^31.
inline BnStatsGeom bn_stats_geometry(int rows, int channels) {
  int block_x = stats_last_pow2((unsigned)channels);
  if (block_x > kStatsTileW) block_x = kStatsTileW;
  int block_y = stats_last_pow2((unsigned)stats_ceil_div(rows, kStatsElemsPerThread));
  if (block_y > kStatsMaxBlock / block_x) block_y = kStatsMaxBlock / block_x;
  // ATen then widens block_x when block_x * block_y < MAX_BLOCK_SIZE; block_y is final here
  int grid_y = stats_ceil_div(rows, block_y * kStatsElemsPerThread);
  if (grid_y > kStatsMaxHBlock) grid_y = kStatsMaxHBlock;
  if (grid_y < 8) grid_y = 1;
  const int stride = block_y * grid_y;
  return BnStatsGeom{block_y, grid_y, 1 + (rows - 1) / (stride * kStatsChains)};
}

// Bytes of the cross-block workspace: int count[grid_y] (padded to 16 bytes), then float
// mean[grid_y][channels] and m2[grid_y][channels].  0 when grid_y == 1.
inline int64_t bn_stats_workspace(const BnStatsGeom& g, int channels) {
  if (g.grid_y == 1) return 0;
  const int64_t counts = ((int64_t)g.grid_y * 4 + 15) / 16 * 16;
  return counts + 2 * (int64_t)g.grid_y * channels * 4;
}

// The backward reduction (ATen's batch_norm_backward_reduce_channels_last_kernel) is launched with the
// same flexible_launch_configs(coop = true), so it has this geometry too.  Its workspace: `sums`
// float[channels] results (sum_dy, then one sum_dy_xmu per batch norm), then, when grid_y > 1, the
// per logical block partials float[sums][grid_y][channels].
inline int64_t bn_bwd_workspace(const BnStatsGeom& g, int channels, int sums) {
  const int64_t results = (int64_t)sums * channels * 4;
  return g.grid_y == 1 ? results : results * (1 + g.grid_y);
}

}  // namespace tok
