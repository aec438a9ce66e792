// The actor table of a training batch and the metres -> heat-map pixel mapping of data_pipeline.detections_to_heatmap, shared by
// the detection-target kernel (heatmap.cu) and the evaluation kernel (evaluate.cu), so both place an actor on the same pixel.
#pragma once
#include "common.cuh"

namespace lavb {

struct DetActor { float x, y, ori, bx, by, typ; };   // 24 bytes: ego-frame metres, radians, box extents, class (0 / 1)
static_assert(sizeof(DetActor) == 24, "DetActor layout is part of the ABI (lav_b200.h)");

struct DetGrid { float ppm, cx0, cy0, cy1, inv_r; };

// Centre of an actor in map pixels (column, row): torch computes cx = -x * ppm + cx0 and cy = (-y * ppm + cy0) + cy1 as separate
// fp32 ops; the _rn intrinsics keep nvcc from contracting any of it into an FMA.
__device__ __forceinline__ float2 det_centre(const DetActor& a, const DetGrid& g) {
  return make_float2(__fadd_rn(__fmul_rn(-a.x, g.ppm), g.cx0), __fadd_rn(__fadd_rn(__fmul_rn(-a.y, g.ppm), g.cy0), g.cy1));
}

}  // namespace lavb
