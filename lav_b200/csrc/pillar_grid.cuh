// The pillar grid's window: which LiDAR points the voxeliser keeps.  pillar.cu's encoders and the painting evaluation
// (paint_eval.cu) share this predicate, so "in window" means the same points in both.
#pragma once
#include "common.cuh"

namespace lavb {

struct Grid {
  float min_x, max_x, min_y, max_y, ppm;
  int nx, ny;
};

// grid_locations, point_pillar.py:70-79: the half-open window test on the raw fp32 coordinates (NaN fails every comparison)
__device__ __forceinline__ bool in_window(const Grid& g, float x, float y) {
  return x >= g.min_x && x < g.max_x && y >= g.min_y && y < g.max_y;
}

}  // namespace lavb
