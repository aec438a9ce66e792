// Temporal BEV training targets: TemporalLiDARPaintedDataset.load_bev_channels
// (lav/utils/datasets/temporal_lidar_painted_dataset.py:182-198) for every plane of a batch in one launch.
//
// Per plane the reference runs   rotate_image(plane, a1) -> zero-pad 32 -> crop at (dx+32, dy+32) -> rotate_image(., a2) -> > 0
// where rotate_image is cv2.warpAffine(INTER_LINEAR, constant-zero border).  OpenCV evaluates 8-bit bilinear warps in fixed
// point; this kernel restates that arithmetic so the output is bit-identical:
//   X = (rint((A01*y + A02) * 1024) + 16 + rint(A00*x*1024)) >> 5,  sx = X >> 5,  fx = X & 31   (Y likewise from row 1)
//   out = (sum of 4 taps * {(32-fx)(32-fy), fx(32-fy), (32-fx)fy, fx*fy} * 32 + 16384) >> 15,  taps outside the image read 0.
// The fp64 products and sums use explicit _rn intrinsics: a contracted FMA would round differently from the CPU now and then.
// One thread per output pixel evaluates the 4 taps of the second warp, each of which is one pixel of the FIRST warp (rounded to
// uint8, as the reference stores it) built from 4 source taps; all reads hit L1/L2.
#include "common.cuh"

namespace {

struct BevJob {             // 128 bytes, layout documented in lav_b200.h
  long long src;            // source plane index, < 0 = missing frame (plane written as zeros)
  long long dst;            // output plane index
  double m1[6];             // inverse matrix of the first warp  (row-major 2x3)
  double m2[6];             // inverse matrix of the second warp
  int dx, dy;               // crop shift: rows, columns
  int pad[2];
};
static_assert(sizeof(BevJob) == 128, "BevJob layout is part of the ABI (lav_b200.h)");

// OpenCV's fixed-point source coordinate of output pixel (x, y) under inverse matrix m: (X, Y) in 1/32 pixel units.
__device__ __forceinline__ void fixed_coord(const double* m, int x, int y, int& X, int& Y) {
  const double yd = (double)y, xd = (double)x;
  const int x0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[1], yd), m[2]), 1024.0)) + 16;
  const int y0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[4], yd), m[5]), 1024.0)) + 16;
  X = (x0 + __double2int_rn(__dmul_rn(__dmul_rn(m[0], xd), 1024.0))) >> 5;
  Y = (y0 + __double2int_rn(__dmul_rn(__dmul_rn(m[3], xd), 1024.0))) >> 5;
}

__device__ __forceinline__ int tap(const uint8_t* __restrict__ img, int h, int w, int x, int y) {
  return (x >= 0 && x < w && y >= 0 && y < h) ? (int)__ldg(img + (size_t)y * w + x) : 0;
}

// bilinear 8-bit sample of img at the fixed-point coordinate (X, Y), rounded and saturated as cv::warpAffine stores it
__device__ __forceinline__ int sample_u8(const uint8_t* __restrict__ img, int h, int w, int X, int Y) {
  const int sx = X >> 5, fx = X & 31, sy = Y >> 5, fy = Y & 31;
  const int s = tap(img, h, w, sx, sy) * ((32 - fx) * (32 - fy)) + tap(img, h, w, sx + 1, sy) * (fx * (32 - fy)) +
                tap(img, h, w, sx, sy + 1) * ((32 - fx) * fy) + tap(img, h, w, sx + 1, sy + 1) * (fx * fy);
  return min((s * 32 + 16384) >> 15, 255);
}

__global__ void __launch_bounds__(256) bev_targets_kernel(const BevJob* __restrict__ jobs, const uint8_t* __restrict__ src,
                                                          uint8_t* __restrict__ out, int h, int w) {
  const BevJob& j = jobs[blockIdx.z];
  const int x = blockIdx.x * 32 + threadIdx.x, y = blockIdx.y * 8 + threadIdx.y;
  if (x >= w || y >= h) return;
  const size_t plane = (size_t)h * w;
  int v = 0;
  if (j.src >= 0) {
    const uint8_t* img = src + (size_t)j.src * plane;
    int X, Y;
    fixed_coord(j.m2, x, y, X, Y);
    const int sx = X >> 5, fx = X & 31, sy = Y >> 5, fy = Y & 31;
    int s = 0;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int ix = sx + (t & 1), iy = sy + (t >> 1);
      const int wt = (t & 1 ? fx : 32 - fx) * (t >> 1 ? fy : 32 - fy);
      // intermediate pixel (ix, iy) of the cropped image = first-warp pixel (ix + dy, iy + dx); zero padding outside both
      const int cx = ix + j.dy, cy = iy + j.dx;
      if (wt != 0 && ix >= 0 && ix < w && iy >= 0 && iy < h && cx >= 0 && cx < w && cy >= 0 && cy < h) {
        int X1, Y1;
        fixed_coord(j.m1, cx, cy, X1, Y1);
        s += sample_u8(img, h, w, X1, Y1) * wt;
      }
    }
    v = ((min((s * 32 + 16384) >> 15, 255)) > 0) ? 1 : 0;
  }
  out[(size_t)j.dst * plane + (size_t)y * w + x] = (uint8_t)v;
}

}  // namespace

extern "C" int lavb_bev_targets(const void* d_jobs, int n_jobs, const uint8_t* d_src, uint8_t* d_out, int h, int w, void* stream) {
  LAVB_CHECK_ARG(n_jobs >= 0 && n_jobs <= 65535 && h > 0 && w > 0 && h <= 4096 && w <= 4096, "bev_targets: bad arguments");
  if (n_jobs == 0) return 0;
  dim3 grid(lavb::ceil_div(w, 32), lavb::ceil_div(h, 8), n_jobs);
  bev_targets_kernel<<<grid, dim3(32, 8), 0, (cudaStream_t)stream>>>(reinterpret_cast<const BevJob*>(d_jobs), d_src, d_out, h, w);
  LAVB_LAUNCH_OK();
  return 0;
}
