// The painting cameras' projection of a LiDAR point: CoordConverter.forward (team_code_v2/model_inference.py:280-297) in the
// reference's fp32 operation order (k-sequential FMA chains, IEEE division, truncation toward zero, bounds test on the truncated
// integers, later camera wins).  Every kernel that decides which pixel a point hits includes this header, so the painting
// (paint.cu) and its evaluation (paint_eval.cu) make the same visibility decision bit for bit.
#pragma once
#include "common.cuh"

namespace lavb {

struct CamSet {
  float m[4][41];  // K(9) | lidar_to_world(16) | world_to_cam(16)
  int ncam;
};

// row-vector dot in the order a BLAS sgemm with a k-loop produces: ((a0*b0 + a1*b1) + a2*b2) + a3*b3 with FMA
__device__ __forceinline__ float dot4(const float* r, float x, float y, float z, float w) {
  float acc = __fmul_rn(r[0], x);
  acc = __fmaf_rn(r[1], y, acc);
  acc = __fmaf_rn(r[2], z, acc);
  acc = __fmaf_rn(r[3], w, acc);
  return acc;
}
__device__ __forceinline__ float dot3(const float* r, float x, float y, float z) {
  float acc = __fmul_rn(r[0], x);
  acc = __fmaf_rn(r[1], y, acc);
  acc = __fmaf_rn(r[2], z, acc);
  return acc;
}

// float -> int64 the way x86 cvttss2si does for the cases that matter: NaN / inf / |v| >= 2^63 give the
// "indefinite" INT64_MIN (which then fails every >= 0 test in the reference).
__device__ __forceinline__ long long trunc_i64(float v) {
  if (!(fabsf(v) < 9.2233720368547758e18f)) return (long long)0x8000000000000000ull;
  return (long long)v;  // cvt.rzi
}

// The camera that sees (x, y, z): the last of cams.ncam whose truncated projection (u, v) lies inside the W x H image, or -1;
// (hit_u, hit_v) = its pixel.  The one projection every painting kernel uses, so their visibility decisions agree bit for bit.
__device__ __forceinline__ int project_hit(const CamSet& cams, float x, float y, float z, int H, int W, int& hit_u, int& hit_v) {
  int hit_cam = -1;
#pragma unroll 1
  for (int c = 0; c < cams.ncam; ++c) {
    const float* K = cams.m[c];
    const float* L = cams.m[c] + 9;
    const float* Wc = cams.m[c] + 25;
    // world = lidar_to_world @ [x,y,z,1]
    const float w0 = dot4(L + 0, x, y, z, 1.f), w1 = dot4(L + 4, x, y, z, 1.f), w2 = dot4(L + 8, x, y, z, 1.f),
                w3 = dot4(L + 12, x, y, z, 1.f);
    // cam = world_to_cam @ world ; re-axis (cam_y, -cam_z, cam_x)
    const float c0 = dot4(Wc + 0, w0, w1, w2, w3), c1 = dot4(Wc + 4, w0, w1, w2, w3), c2 = dot4(Wc + 8, w0, w1, w2, w3);
    const float a0 = c1, a1 = -c2, a2 = c0;
    // cam_2d = K @ cam
    const float q0 = dot3(K + 0, a0, a1, a2), q1 = dot3(K + 3, a0, a1, a2), q2 = dot3(K + 6, a0, a1, a2);
    const float den = __fadd_rn(1e-5f, q2);
    const long long u = trunc_i64(__fdiv_rn(q0, den));
    const long long v = trunc_i64(__fdiv_rn(q1, den));
    const long long zi = trunc_i64(q2);
    if (zi >= 0 && u >= 0 && u < W && v >= 0 && v < H) {
      hit_cam = c; hit_u = (int)u; hit_v = (int)v;
    }
  }
  return hit_cam;
}

}  // namespace lavb
