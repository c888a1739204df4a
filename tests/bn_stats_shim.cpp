// C entry point over the batch-norm statistics geometry (csrc/bn_stats_geom.h) for
// tests/test_bn_stats_cpu.py, built with the host compiler alone.
#include "bn_stats_geom.h"

extern "C" {

// out = {block_y, grid_y, loop_count, workspace bytes}
void shim_bn_stats_geometry(int rows, int channels, long long* out) {
  const tok::BnStatsGeom g = tok::bn_stats_geometry(rows, channels);
  out[0] = g.block_y;
  out[1] = g.grid_y;
  out[2] = g.loop_count;
  out[3] = tok::bn_stats_workspace(g, channels);
}

}  // extern "C"
