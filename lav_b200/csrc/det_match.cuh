// The matching of decoded detections to the recorded actors, shared by the evaluation kernel (evaluate.cu), the match of the
// detected-forecast rows (det_forecast.cu) and the box scores (det_box_eval.cu): the peak filters, the order detections are
// taken in, the ego window and the greedy nearest-unmatched search, so a detection takes the same actor in all three.
#pragma once
#include "det_grid.cuh"

namespace lavb {

// Squared distance in double with no contraction, so the host's numpy statement gets the same bits.
__device__ __forceinline__ double dist2(double dx, double dy) { return __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)); }

// Distance in pixels from the ego window's centre (cx0, cy0 + cy1), as decode_packed's `dist` (fp64).
__device__ __forceinline__ double window_dist(double x, double y, const DetGrid& g) {
  return sqrt(dist2(x - (double)g.cx0, y - (double)__fadd_rn(g.cy0, g.cy1)));
}

// Whether peak (s, loc, col) is taken before peak (s2, loc2, col2): descending score, then lower flat index, then lower column.
// A NaN score comes after every other score, so the order stays total over any distinct columns.
__device__ __forceinline__ bool ranks_before(float s, long long loc, int col, float s2, long long loc2, int col2) {
  const bool hi = s > s2 || (!isnan(s) && isnan(s2));
  const bool eq = s == s2 || (isnan(s) && isnan(s2));
  return hi || (eq && (loc < loc2 || (loc == loc2 && col < col2)));
}

// Pixel of a packed peak's flat index: numpy's astype(int64) (truncation), then Python's floor % and //.
__device__ __forceinline__ void peak_pixel(float flat, int w, long long& loc, long long& x, long long& y) {
  loc = (long long)flat;
  x = loc % w;
  if (x < 0) x += w;
  y = (loc - x) / w;
}

// The constants of InferModel.decode_packed's filters on a map of ppm pixels per metre: score > float32(min_score) in fp32, the
// class-1 size filter and the ego window 2 < d < 30 m, in pixels.
struct DetFilter {
  float min_score;                   // the reference compares fp32 scores in fp32
  float size_thr;                    // class 1: dropped when both box sides are below it (pixels)
  double win_lo, win_hi;
};

inline DetFilter det_filter(float ppm, double min_score) {
  DetFilter f;
  f.min_score = (float)min_score;
  f.size_thr = (float)(0.1 * (double)ppm);                        // numpy compares the float32 sizes with float32(0.1 * ppm)
  f.win_lo = 2.0;                                                 // decode_packed's `dist <= 2 | dist >= 30 * ppm` (pixels)
  f.win_hi = 30.0 * (double)ppm;
  return f;
}

// Whether a packed peak of class cls with score sc and box sides (bw, bh), at window_dist d, survives decode_packed's filters;
// a NaN score never survives.  f is any struct with DetFilter's four fields (the kernels' argument structs).  A macro rather
// than a function: a function boundary here changes the code nvcc emits for eval_batch_kernel, the expression in place does not.
#define LAVB_PEAK_SURVIVES(sc, bw, bh, d, cls, f) \
  ((sc) > (f).min_score && !((cls) == 1 && (bw) < (f).size_thr && (bh) < (f).size_thr) && (d) > (f).win_lo && (d) < (f).win_hi)

// One warp, every lane calling with the same arguments: the nearest of actors [0, n) with ok(i) whose squared distance from
// (px, py) is at most thr2; equal distances go to the lower row.  -> the row, or -1 with *d2 = +inf, on every lane.
template <typename Ok>
__device__ __forceinline__ int nearest_unmatched(double px, double py, const float* gx, const float* gy, int n, double thr2, Ok ok,
                                                 double* d2) {
  const int lane = threadIdx.x & 31;
  double best = INFINITY;
  int who = 0x7fffffff;
  for (int i = lane; i < n; i += 32) {
    if (!ok(i)) continue;
    const double d = dist2(px - (double)gx[i], py - (double)gy[i]);
    if (d <= thr2 && d < best) { best = d; who = i; }          // lanes visit rows in ascending order: the first equal stays
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int ow = __shfl_xor_sync(0xffffffffu, who, o);
    if (ob < best || (ob == best && ow < who)) { best = ob; who = ow; }
  }
  *d2 = best;
  return who == 0x7fffffff ? -1 : who;
}

}  // namespace lavb
