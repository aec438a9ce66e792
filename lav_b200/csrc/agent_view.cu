// The agent's debug view (lav_agent_fast.py:459-518, lidar_to_bev :567-581) for b agents, bit for bit with the reference's
// numpy and OpenCV 8-bit arithmetic, in four launches plus one memset on the caller's stream:
//   hist    one thread per stacked row: np.histogramdd's bin by exact fp64 comparison with the 321 edges, int atomics;
//   points  one thread per plan point, forecast point and target: a fixed circle stencil, each pixel taking atomicMax of the
//           key (sequence << 32) | rgb, so the last primitive in visualize's loop order wins whatever order threads run in;
//   boxes   one thread per side of a vehicle box: cv2's thickness-2 ThickLine (a 16.16 FillConvexPoly quad and a radius-1 cap)
//           restated in int64, with the same keys;
//   compose one thread per pixel of the (160, 1146) frame: the four canvas pixels it reads are built as the canvas holds them
//           (camera / tele resize, grey + drawing, BEV mean) and the final resize is taken from them.
// Every float operation is a correctly rounded intrinsic, so nothing is contracted.
#include <algorithm>
#include <array>
#include <cstring>
#include <vector>

#include "common.cuh"

namespace {

constexpr int kS = 320;                                   // the LiDAR / BEV image side
constexpr int kCamH = 288, kCamW = 256, kCams = 3;        // the three cameras, side by side 768 wide
constexpr int kTelH = 192, kTelW = 480;
constexpr int kCamOut = 853, kTelOut = 800, kCanvasW = kCamOut + kTelOut + 2 * kS;
constexpr int kOutH = 160, kOutW = 1146;
constexpr int kEgoX = 160, kEgoY = 280;
constexpr int kHistMax = 10;
constexpr int kJet = 256;                                 // colours; rows kJet, kJet + 1, kJet + 2 = under, over, bad
constexpr int kAgentChunk = 256;                          // agents per points launch (their row offsets travel as an argument)
constexpr int kBoxChunk = 96;                             // boxes per boxes launch (their corners travel as an argument)
constexpr int kMaxT = 64, kMaxM = 8;
constexpr int kXYShift = 16;
constexpr long long kXYOne = 1LL << kXYShift;
constexpr unsigned kTargetSeq = 0xFFFFFFFFu;              // the target is drawn last

struct RowChunk { int rows[kAgentChunk + 1]; };
struct BoxChunk { int n; int agent[kBoxChunk]; unsigned seq[kBoxChunk]; int xy[kBoxChunk][8]; };

struct ViewArgs {
  const unsigned char* rgbs; const unsigned char* tels;
  const float* points; long long p; int point_stride;
  const void* bev; int bev_h16, bev_c; long long bev_sb, bev_sc, bev_sy, bev_sx;
  const float2* plan; const float2* cast; const int* cmd;
  const float2* locs; const float* scores; const float* target;
  int t, m;
  int* counts; unsigned long long* keys;                  // (b, 320, 320) each
  unsigned char* out;
};

struct Style { double ppm, thresh; unsigned char jet[(kJet + 3) * 3]; };

__device__ __forceinline__ unsigned long long key_of(unsigned seq, unsigned rgb) { return ((unsigned long long)seq << 32) | rgb; }
__device__ __forceinline__ unsigned rgb_of(int r, int g, int b) { return (unsigned)r | ((unsigned)g << 8) | ((unsigned)b << 16); }

__device__ __forceinline__ void put(unsigned long long* keys, long long x, long long y, unsigned long long key) {
  if (x >= 0 && x < kS && y >= 0 && y < kS) atomicMax(keys + y * kS + x, key);
}

// ---- histogram -------------------------------------------------------------------------------------------------------------
// numpy's linspace(lo, lo + 81, 321): i * (81 / 320) + lo, the last edge exactly lo + 81
__device__ __forceinline__ double edge(int i, double lo) {
  return i == kS ? lo + 81.0 : __dadd_rn(__dmul_rn((double)i, 81.0 / 320.0), lo);
}

// np.histogramdd's bin along one axis: searchsorted(side='right') - 1, the last edge in the last bin; -1 when outside / NaN
__device__ __forceinline__ int hist_bin(float vf, double lo) {
  const double v = (double)vf;
  if (!(v >= lo) || v > lo + 81.0) return -1;
  if (v == lo + 81.0) return kS - 1;
  int g = (int)floor(__ddiv_rn(__dsub_rn(v, lo), 81.0 / 320.0));
  g = g < 0 ? 0 : g > kS - 1 ? kS - 1 : g;
  while (g > 0 && edge(g, lo) > v) --g;
  while (g < kS - 1 && edge(g + 1, lo) <= v) ++g;
  return g;
}

__global__ void __launch_bounds__(256) view_hist_kernel(ViewArgs a) {
  const int b = blockIdx.y;
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < a.p; r += (long long)gridDim.x * blockDim.x) {
    const float* row = a.points + ((long long)b * a.p + r) * a.point_stride;
    const int bx = hist_bin(row[0], -10.0), by = hist_bin(row[1], -40.0);
    if (bx < 0 || by < 0) continue;
    atomicAdd(a.counts + ((long long)b * kS + (kS - 1 - bx)) * kS + by, 1);     // rows flipped
  }
}

// ---- plan, forecast and target circles -----------------------------------------------------------------------------------
// cv2.circle(..., r, color, -1), LINE_8: r = 1 a plus, r = 2 the 13-pixel diamond
__device__ __forceinline__ void stencil(unsigned long long* keys, long long cx, long long cy, int r, unsigned long long key) {
  for (int dy = -r; dy <= r; ++dy) {
    const int w = r - (dy < 0 ? -dy : dy);
    for (int dx = -w; dx <= w; ++dx) put(keys, cx + dx, cy + dy, key);
  }
}

// (ego + loc * ppm).astype(int): fp32 product, fp64 sum, truncation; false for NaN or outside int32
__device__ __forceinline__ bool point_pixel(float2 loc, float ppm, long long& x, long long& y) {
  const double px = __dadd_rn((double)kEgoX, (double)__fmul_rn(loc.x, ppm));
  const double py = __dadd_rn((double)kEgoY, (double)__fmul_rn(loc.y, ppm));
  if (!(px > -2147483649.0 && px < 2147483648.0 && py > -2147483649.0 && py < 2147483648.0)) return false;
  x = (long long)px; y = (long long)py;
  return true;
}

// matplotlib's Colormap.__call__ row for an fp32 score
__device__ __forceinline__ int jet_row(float s) {
  float xa = __fmul_rn(s, (float)kJet);
  if (xa == (float)kJet) xa = (float)(kJet - 1);
  if (isnan(xa)) return kJet + 2;
  if (xa < 0.f) return kJet;
  if (xa >= (float)kJet) return kJet + 1;
  return (int)xa;
}

__global__ void __launch_bounds__(128) view_points_kernel(ViewArgs a, Style st, RowChunk ch, int b0) {
  const int i = blockIdx.y, b = b0 + i;
  const int r0 = ch.rows[i], nrows = ch.rows[i + 1] - r0;
  const int per_row = a.m * a.t;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  const int total = a.t + nrows * per_row + 1;
  if (q >= total) return;
  unsigned long long* keys = a.keys + (long long)b * kS * kS;
  const float ppm = (float)st.ppm;
  long long x, y;
  if (q < a.t) {                                                     // the plan (the ego cast under commands 4 and 5)
    const int c = a.cmd[b];
    const float2 loc = (c == 4 || c == 5 ? a.cast : a.plan)[(long long)b * a.t + q];
    if (point_pixel(loc, ppm, x, y)) stencil(keys, x, y, 1, key_of(1u + q, rgb_of(255, 0, 0)));
  } else if (q < total - 1) {                                        // forecast steps of branches scoring >= cmd_thresh
    const int j = q - a.t, k = j / per_row, br = (j / a.t) % a.m, s = j % a.t;
    const long long row = (long long)r0 + k;
    const float score = a.scores[row * a.m + br];
    if ((double)score < st.thresh) return;
    const unsigned char* c = st.jet + 3 * jet_row(score);
    if (point_pixel(a.locs[(row * a.m + br) * a.t + s], ppm, x, y))
      stencil(keys, x, y, 1, key_of(1u + q, rgb_of(c[0], c[1], c[2])));
  } else {                                                           // the target: clip(ego + tgt * ppm, 0, 255) in fp64
    double tx = __dadd_rn((double)kEgoX, __dmul_rn((double)a.target[2 * b], st.ppm));
    double ty = __dadd_rn((double)kEgoY, __dmul_rn((double)a.target[2 * b + 1], st.ppm));
    if (isnan(tx) || isnan(ty)) return;
    tx = fmin(fmax(tx, 0.0), 255.0); ty = fmin(fmax(ty, 0.0), 255.0);
    stencil(keys, (long long)tx, (long long)ty, 2, key_of(kTargetSeq, rgb_of(0, 255, 0)));
  }
}

// ---- vehicle boxes: cv2.drawContours(..., thickness 2) ---------------------------------------------------------------------
__device__ __forceinline__ long long cdiv(long long a, long long b) { return a / b; }   // C division, as OpenCV's

// OpenCV's clipLine on the int64 rectangle (0, 0, w, h)
__device__ bool clip_line(long long w, long long h, long long& x1, long long& y1, long long& x2, long long& y2) {
  const long long right = w - 1, bottom = h - 1;
  int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
  int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
  if ((c1 & c2) == 0 && (c1 | c2) != 0) {
    long long t;
    if (c1 & 12) {
      t = c1 < 8 ? 0 : bottom;
      x1 += (long long)__ddiv_rn(__dmul_rn((double)(t - y1), (double)(x2 - x1)), (double)(y2 - y1));
      y1 = t;
      c1 = (x1 < 0) + (x1 > right) * 2;
    }
    if (c2 & 12) {
      t = c2 < 8 ? 0 : bottom;
      x2 += (long long)__ddiv_rn(__dmul_rn((double)(t - y2), (double)(x2 - x1)), (double)(y2 - y1));
      y2 = t;
      c2 = (x2 < 0) + (x2 > right) * 2;
    }
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
      if (c1) {
        t = c1 == 1 ? 0 : right;
        y1 += (long long)__ddiv_rn(__dmul_rn((double)(t - x1), (double)(y2 - y1)), (double)(x2 - x1));
        x1 = t; c1 = 0;
      }
      if (c2) {
        t = c2 == 1 ? 0 : right;
        y2 += (long long)__ddiv_rn(__dmul_rn((double)(t - x2), (double)(y2 - y1)), (double)(x2 - x1));
        x2 = t; c2 = 0;
      }
    }
  }
  return (c1 | c2) == 0;
}

// the 16.16 fixed-point line walker FillConvexPoly outlines with (8-connected)
__device__ void line_fixed(unsigned long long* keys, unsigned long long key, long long x1, long long y1, long long x2, long long y2) {
  if (!clip_line((long long)kS << kXYShift, (long long)kS << kXYShift, x1, y1, x2, y2)) return;
  long long dx = x2 - x1, dy = y2 - y1;
  const long long ax = dx < 0 ? -dx : dx, ay = dy < 0 ? -dy : dy;
  long long step, n;
  if (ax > ay) {
    if (dx < 0) { long long s = x1; x1 = x2; x2 = s; s = y1; y1 = y2; y2 = s; dy = -dy; }
    step = cdiv(dy * kXYOne, ax | 1);
    n = (x2 - x1) >> kXYShift;
  } else {
    if (dy < 0) { long long s = x1; x1 = x2; x2 = s; s = y1; y1 = y2; y2 = s; dx = -dx; }
    step = cdiv(dx * kXYOne, ay | 1);
    n = (y2 - y1) >> kXYShift;
  }
  put(keys, (x2 + (kXYOne >> 1)) >> kXYShift, (y2 + (kXYOne >> 1)) >> kXYShift, key);
  x1 += kXYOne >> 1;
  y1 += kXYOne >> 1;
  if (ax > ay) {
    x1 >>= kXYShift;
    for (long long i = 0; i <= n; ++i, ++x1, y1 += step) put(keys, x1, y1 >> kXYShift, key);
  } else {
    y1 >>= kXYShift;
    for (long long i = 0; i <= n; ++i, x1 += step, ++y1) put(keys, x1 >> kXYShift, y1, key);
  }
}

// FillConvexPoly (LINE_8) of a 16.16 fixed-point quad: its outline, then the scanlines between its two edges
__device__ void fill_quad(unsigned long long* keys, unsigned long long key, const long long (&v)[4][2]) {
  constexpr int n = 4;
  const long long delta = kXYOne >> 1;
  int imin = 0;
  long long xmin = v[0][0], xmax = v[0][0], ymin = v[0][1], ymax = v[0][1];
  for (int i = 0; i < n; ++i) {
    if (v[i][1] < ymin) { ymin = v[i][1]; imin = i; }
    ymax = max(ymax, v[i][1]); xmax = max(xmax, v[i][0]); xmin = min(xmin, v[i][0]);
    const int p = (i + n - 1) % n;
    line_fixed(keys, key, v[p][0], v[p][1], v[i][0], v[i][1]);
  }
  xmin = (xmin + delta) >> kXYShift; xmax = (xmax + delta) >> kXYShift;
  ymin = (ymin + delta) >> kXYShift; ymax = (ymax + delta) >> kXYShift;
  if (xmax < 0 || ymin >= kS || xmin >= kS) return;
  ymax = min(ymax, (long long)kS - 1);
  int edges = n;
  int eidx[2] = {imin, imin}, edi[2] = {1, n - 1};
  long long ex[2] = {-kXYOne, -kXYOne}, edx[2] = {0, 0}, eye[2] = {ymin, ymin};
  long long y = ymin;
  for (;;) {
    for (int e = 0; e < 2; ++e) {
      if (y < eye[e]) continue;
      int idx0 = eidx[e], idx = (idx0 + edi[e]) % n;
      while (edges-- > 0) {
        const long long ty = (v[idx][1] + delta) >> kXYShift;
        if (ty > y) {
          const long long xs = v[idx0][0], xe = v[idx][0];
          eye[e] = ty;
          edx[e] = cdiv((xe - xs) * 2 + (ty - y), 2 * (ty - y));
          ex[e] = xs;
          eidx[e] = idx;
          break;
        }
        idx0 = idx;
        idx = (idx + edi[e]) % n;
      }
    }
    if (edges < 0) break;
    if (y >= 0) {
      const int l = ex[0] > ex[1] ? 1 : 0;
      long long x1 = (ex[l] + delta) >> kXYShift, x2 = (ex[1 - l] + delta) >> kXYShift;
      if (x2 >= 0 && x1 < kS) {
        x1 = max(x1, 0LL); x2 = min(x2, (long long)kS - 1);
        for (long long x = x1; x <= x2; ++x) put(keys, x, y, key);
      }
    }
    ex[0] += edx[0]; ex[1] += edx[1];
    if (++y > ymax) break;
  }
}

// one side p0 -> p1 of a box: ThickLine with thickness 2 after clipping to the image grown by 2, the cap at p1
__device__ void thick_segment(unsigned long long* keys, unsigned long long key, long long x1, long long y1, long long x2, long long y2) {
  x1 += 2; y1 += 2; x2 += 2; y2 += 2;
  if (!clip_line(kS + 4, kS + 4, x1, y1, x2, y2)) return;
  x1 -= 2; y1 -= 2; x2 -= 2; y2 -= 2;
  const long long ax = x1 * kXYOne, ay = y1 * kXYOne, bx = x2 * kXYOne, by = y2 * kXYOne;
  const double dx = __dmul_rn((double)(ax - bx), 1.0 / kXYOne), dy = __dmul_rn((double)(by - ay), 1.0 / kXYOne);
  const double rr = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
  if (fabs(rr) > 2.220446049250313e-16) {
    const double r = __ddiv_rn((double)kXYOne, __dsqrt_rn(rr));
    const long long ox = __double2ll_rn(__dmul_rn(dy, r)), oy = __double2ll_rn(__dmul_rn(dx, r));
    const long long q[4][2] = {{ax + ox, ay + oy}, {ax - ox, ay - oy}, {bx - ox, by - oy}, {bx + ox, by + oy}};
    fill_quad(keys, key, q);
  }
  stencil(keys, x2, y2, 1, key);
}

__global__ void __launch_bounds__(128) view_boxes_kernel(ViewArgs a, BoxChunk ch) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= 4 * ch.n) return;
  const int k = q >> 2, j = q & 3, p = (j + 3) & 3;
  unsigned long long* keys = a.keys + (long long)ch.agent[k] * kS * kS;
  thick_segment(keys, key_of(ch.seq[k], rgb_of(255, 0, 0)), ch.xy[k][2 * p], ch.xy[k][2 * p + 1], ch.xy[k][2 * j], ch.xy[k][2 * j + 1]);
}

// ---- compose ----------------------------------------------------------------------------------------------------------------
// cv2.resize INTER_LINEAR's source index and 11-bit coefficients of output position d (src -> dst samples); columns clamp
struct Tap { int s0, s1, c0, c1; };
__device__ __forceinline__ Tap lin_tap(int d, int src, int dst, bool column) {
  const double scale = __ddiv_rn(1.0, __ddiv_rn((double)dst, (double)src));
  float f = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)d, 0.5), scale), 0.5));
  int s = (int)floorf(f);
  f = __fsub_rn(f, (float)s);
  if (column && (s < 0 || s >= src - 1)) { f = 0.f; s = s < 0 ? 0 : src - 1; }
  Tap t;
  t.c0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, f), 2048.f));
  t.c1 = __float2int_rn(__fmul_rn(f, 2048.f));
  t.s0 = min(max(s, 0), src - 1);
  t.s1 = min(max(s + 1, 0), src - 1);
  return t;
}

__device__ __forceinline__ int vpass(int b0, int b1, int s0, int s1) { return (((b0 * (s0 >> 4)) >> 16) + ((b1 * (s1 >> 4)) >> 16) + 2) >> 2; }

struct Px { int v[3]; };

// one pixel of an 8-bit image resized from (sh, sw) to (dh, dw); fetch(y, x, c) reads the source
template <typename F>
__device__ __forceinline__ Px resized(int y, int x, int sh, int sw, int dh, int dw, F fetch) {
  const Tap tx = lin_tap(x, sw, dw, true), ty = lin_tap(y, sh, dh, false);
  Px o;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int s0 = fetch(ty.s0, tx.s0, c) * tx.c0 + fetch(ty.s0, tx.s1, c) * tx.c1;
    const int s1 = fetch(ty.s1, tx.s0, c) * tx.c0 + fetch(ty.s1, tx.s1, c) * tx.c1;
    o.v[c] = vpass(ty.c0, ty.c1, s0, s1);
  }
  return o;
}

__device__ __forceinline__ float bev_logit(const ViewArgs& a, const char* base, long long off) {
  if (a.bev_h16) return lavb::h162float(reinterpret_cast<const lavb::h16*>(base)[off]);
  return reinterpret_cast<const float*>(base)[off];
}

// the (320, 2293) canvas at (y, x): camera strip, tele view, LiDAR view with its drawing, predicted BEV
__device__ Px canvas(const ViewArgs& a, int b, int y, int x) {
  if (x < kCamOut) {
    const unsigned char* cam = a.rgbs + (long long)b * kCams * kCamH * kCamW * 3;
    return resized(y, x, kCamH, kCams * kCamW, kS, kCamOut, [&](int sy, int sx, int c) {
      return (int)cam[(((long long)(sx / kCamW) * kCamH + sy) * kCamW + sx % kCamW) * 3 + c];
    });
  }
  if (x < kCamOut + kTelOut) {
    const unsigned char* tel = a.tels + (long long)b * kTelH * kTelW * 3;
    return resized(y, x - kCamOut, kTelH, kTelW, kS, kTelOut, [&](int sy, int sx, int c) {
      return (int)tel[((long long)sy * kTelW + sx) * 3 + c];
    });
  }
  Px o;
  if (x < kCamOut + kTelOut + kS) {
    const long long i = ((long long)b * kS + y) * kS + (x - kCamOut - kTelOut);
    const unsigned long long key = a.keys[i];
    if (key) {
      o.v[0] = (int)(key & 255); o.v[1] = (int)((key >> 8) & 255); o.v[2] = (int)((key >> 16) & 255);
    } else {
      const int n = min(a.counts[i], kHistMax);
      o.v[0] = o.v[1] = o.v[2] = (int)__dmul_rn(__ddiv_rn((double)n, (double)kHistMax), 255.0);
    }
    return o;
  }
  const int bx = x - kCamOut - kTelOut - kS;
  const char* base = static_cast<const char*>(a.bev);
  const long long off = b * a.bev_sb + y * a.bev_sy + bx * a.bev_sx;
  float s = 0.f;
  for (int c = 0; c < a.bev_c; ++c) {
    const float p = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-bev_logit(a, base, off + c * a.bev_sc))));  // torch.sigmoid's 1 / (1 + exp(-x))
    s = c == 0 ? p : __fadd_rn(s, p);
  }
  const float v = __fmul_rn(255.f, __fdiv_rn(s, (float)a.bev_c));
  o.v[0] = o.v[1] = o.v[2] = isnan(v) ? 0 : (int)v;
  return o;
}

__global__ void __launch_bounds__(256) view_compose_kernel(ViewArgs a) {
  const int b = blockIdx.y;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= kOutH * kOutW) return;
  const int oy = q / kOutW, ox = q % kOutW;
  const Tap tx = lin_tap(ox, kCanvasW, kOutW, true), ty = lin_tap(oy, kS, kOutH, false);
  const Px p00 = canvas(a, b, ty.s0, tx.s0), p01 = canvas(a, b, ty.s0, tx.s1);
  const Px p10 = canvas(a, b, ty.s1, tx.s0), p11 = canvas(a, b, ty.s1, tx.s1);
  unsigned char* o = a.out + ((long long)b * kOutH * kOutW + q) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c)
    o[c] = (unsigned char)vpass(ty.c0, ty.c1, p00.v[c] * tx.c0 + p01.v[c] * tx.c1, p10.v[c] * tx.c0 + p11.v[c] * tx.c1);
}

// visualize's corners of box (x, y, w, h, cos, sin): [x, y] + [+-w, +-h] @ [[-sin, cos], [-cos, -sin]] in fp64, truncated
bool box_corners(const double* bx, int (&xy)[8]) {
  static const int sg[4][2] = {{-1, -1}, {-1, 1}, {1, 1}, {1, -1}};
  const double x = bx[0], y = bx[1], w = bx[2], h = bx[3], c = bx[4], s = bx[5];
  for (int i = 0; i < 4; ++i) {
    const double sw = sg[i][0] * w, sh = sg[i][1] * h;
    volatile double u = sw * -s, v = sh * -c, p = sw * c, r = sh * -s;   // volatile: no contraction, numpy's roundings
    const double cx = x + (u + v), cy = y + (p + r);
    if (!(cx > -2147483649.0 && cx < 2147483648.0 && cy > -2147483649.0 && cy < 2147483648.0)) return false;
    xy[2 * i] = (int)cx; xy[2 * i + 1] = (int)cy;
  }
  return true;
}

}  // namespace

extern "C" size_t lavb_agent_view_scratch_bytes(int b) {
  return b < 0 ? 0 : (size_t)b * kS * kS * (sizeof(unsigned long long) + sizeof(int));
}

extern "C" int lavb_agent_view(const unsigned char* d_rgbs, const unsigned char* d_tels, const float* d_points, int b, long long p,
                               int point_stride, const void* d_bev, int bev_dtype, int bev_c, const long long* h_bev_strides,
                               const float* d_plan, const float* d_cast, const int* d_cmd, int t, const float* d_other_locs,
                               const float* d_other_cmds, int k, int m, const int* h_offsets, const double* h_boxes,
                               int n_boxes, const int* h_box_offsets, const float* d_target, const lavb_view_config* h_config, void* d_scratch,
                               size_t scratch_bytes, unsigned char* d_out, void* stream) {
  LAVB_CHECK_ARG(b >= 0 && b <= 65535 && p >= 0 && point_stride >= 2,
                 "agent_view: b = %d, p = %lld, point_stride = %d (0 <= b <= 65535, p >= 0, stride >= 2)", b, p, point_stride);
  LAVB_CHECK_ARG(t >= 1 && t <= kMaxT && m >= 1 && m <= kMaxM && k >= 0, "agent_view: t = %d (1..%d), m = %d (1..%d), k = %d", t,
                 kMaxT, m, kMaxM, k);
  LAVB_CHECK_ARG(bev_dtype == LAVB_F32 || bev_dtype == LAVB_H16, "agent_view: bev dtype %d is not LAVB_F32 or the 16-bit type",
                 bev_dtype);
  LAVB_CHECK_ARG(bev_c >= 1 && bev_c <= 64, "agent_view: %d BEV channels (1..64)", bev_c);
  LAVB_CHECK_ARG(h_config && h_bev_strides && h_offsets && h_box_offsets, "agent_view: null host pointer");
  const lavb_view_config cfg = *h_config;
  LAVB_CHECK_ARG(cfg.pixels_per_meter > 0.0 && isfinite(cfg.pixels_per_meter) && (double)(float)cfg.pixels_per_meter == cfg.pixels_per_meter,
                 "agent_view: pixels_per_meter %g must be positive and exact in fp32", cfg.pixels_per_meter);
  LAVB_CHECK_ARG(!isnan(cfg.cmd_thresh), "agent_view: cmd_thresh is NaN");
  LAVB_CHECK_ARG(h_offsets[0] >= 0 && h_offsets[b] <= k, "agent_view: row offsets [%d, %d] run outside the %d forecast rows",
                 h_offsets[0], h_offsets[b], k);
  LAVB_CHECK_ARG(n_boxes >= 0 && h_box_offsets[0] >= 0 && h_box_offsets[b] <= n_boxes,
                 "agent_view: box offsets [%d, %d] run outside the %d boxes", h_box_offsets[0], h_box_offsets[b], n_boxes);
  for (int i = 0; i < b; ++i) {
    LAVB_CHECK_ARG(h_offsets[i] <= h_offsets[i + 1], "agent_view: row offsets of agent %d are not monotone (%d -> %d)", i,
                   h_offsets[i], h_offsets[i + 1]);
    LAVB_CHECK_ARG(h_box_offsets[i] <= h_box_offsets[i + 1], "agent_view: box offsets of agent %d are not monotone (%d -> %d)", i,
                   h_box_offsets[i], h_box_offsets[i + 1]);
    LAVB_CHECK_ARG((long long)(h_offsets[i + 1] - h_offsets[i]) * m * t + t + 1 < (1LL << 30),
                   "agent_view: agent %d has too many forecast rows (%d)", i, h_offsets[i + 1] - h_offsets[i]);
  }
  const int nbox = b > 0 ? h_box_offsets[b] - h_box_offsets[0] : 0;
  LAVB_CHECK_ARG(nbox == 0 || h_boxes, "agent_view: missing host box table (%d boxes)", nbox);
  const long long sb = h_bev_strides[0], sc = h_bev_strides[1], sy = h_bev_strides[2], sx = h_bev_strides[3];
  LAVB_CHECK_ARG(sb >= 0 && sc >= 0 && sy >= 0 && sx >= 0, "agent_view: negative BEV strides");
  LAVB_CHECK_ARG(scratch_bytes >= lavb_agent_view_scratch_bytes(b), "agent_view: scratch of %zu bytes, %zu needed", scratch_bytes,
                 lavb_agent_view_scratch_bytes(b));
  if (b == 0) return 0;
  LAVB_CHECK_ARG(d_rgbs && d_tels && (d_points || p == 0) && d_bev && d_plan && d_cast && d_cmd && d_target && d_scratch && d_out &&
                 ((d_other_locs && d_other_cmds) || h_offsets[b] == h_offsets[0]), "agent_view: null device pointer");
  const size_t esz = bev_dtype == LAVB_F32 ? 4 : 2;
  LAVB_CHECK_ARG((uintptr_t)d_points % 4 == 0 && (uintptr_t)d_bev % esz == 0 && (uintptr_t)d_plan % 8 == 0 &&
                 (uintptr_t)d_cast % 8 == 0 && (uintptr_t)d_other_locs % 8 == 0 && (uintptr_t)d_other_cmds % 4 == 0 &&
                 (uintptr_t)d_cmd % 4 == 0 && (uintptr_t)d_target % 4 == 0 && (uintptr_t)d_scratch % 8 == 0,
                 "agent_view: misaligned pointer (plan, cast, other_locs and scratch 8-byte, the other floats 4-byte)");
  // the boxes' corners are computed here, on the host, before anything is written
  std::vector<int> agent_of(nbox);
  std::vector<std::array<int, 8>> corners(nbox);
  std::vector<char> drawn(nbox);
  for (int i = 0; i < b; ++i)
    for (int j = h_box_offsets[i]; j < h_box_offsets[i + 1]; ++j) {
      const int q = j - h_box_offsets[0];
      agent_of[q] = i;
      int xy[8];
      drawn[q] = box_corners(h_boxes + 6LL * j, xy);
      for (int e = 0; e < 8; ++e) corners[q][e] = xy[e];
    }

  ViewArgs a;
  a.rgbs = d_rgbs; a.tels = d_tels; a.points = d_points; a.p = p; a.point_stride = point_stride;
  a.bev = d_bev; a.bev_h16 = bev_dtype != LAVB_F32; a.bev_c = bev_c; a.bev_sb = sb; a.bev_sc = sc; a.bev_sy = sy; a.bev_sx = sx;
  a.plan = reinterpret_cast<const float2*>(d_plan); a.cast = reinterpret_cast<const float2*>(d_cast); a.cmd = d_cmd;
  a.locs = reinterpret_cast<const float2*>(d_other_locs); a.scores = d_other_cmds; a.target = d_target;
  a.t = t; a.m = m;
  a.keys = static_cast<unsigned long long*>(d_scratch);
  a.counts = reinterpret_cast<int*>(a.keys + (size_t)b * kS * kS);
  a.out = d_out;
  Style st;
  st.ppm = cfg.pixels_per_meter; st.thresh = cfg.cmd_thresh;
  memcpy(st.jet, cfg.jet, sizeof(st.jet));
  cudaStream_t s = (cudaStream_t)stream;

  LAVB_CUDA_OK(cudaMemsetAsync(d_scratch, 0, lavb_agent_view_scratch_bytes(b), s));
  if (p > 0) {
    const int gx = (int)std::min<long long>((p + 255) / 256, 1024);
    view_hist_kernel<<<dim3(gx, b), 256, 0, s>>>(a);
    LAVB_LAUNCH_OK();
  }
  for (int b0 = 0; b0 < b; b0 += kAgentChunk) {
    const int nb = std::min(b - b0, kAgentChunk);
    RowChunk ch;
    int most = 0;
    for (int i = 0; i <= nb; ++i) ch.rows[i] = h_offsets[b0 + i];
    for (int i = 0; i < nb; ++i) most = std::max(most, ch.rows[i + 1] - ch.rows[i]);
    const int total = t + most * m * t + 1;
    view_points_kernel<<<dim3((total + 127) / 128, nb), 128, 0, s>>>(a, st, ch, b0);
    LAVB_LAUNCH_OK();
  }
  BoxChunk bc;
  bc.n = 0;
  for (int q = 0; q <= nbox; ++q) {
    if (q < nbox && drawn[q]) {
      const int i = agent_of[q];
      bc.agent[bc.n] = i;
      // after the agent's plan and forecast points, in visualize's order
      bc.seq[bc.n] = 1u + (unsigned)t + (unsigned)((h_offsets[i + 1] - h_offsets[i]) * m * t) + (unsigned)(q - (h_box_offsets[i] - h_box_offsets[0]));
      for (int e = 0; e < 8; ++e) bc.xy[bc.n][e] = corners[q][e];
      ++bc.n;
    }
    if (bc.n == kBoxChunk || (q == nbox && bc.n > 0)) {
      view_boxes_kernel<<<(4 * bc.n + 127) / 128, 128, 0, s>>>(a, bc);
      LAVB_LAUNCH_OK();
      bc.n = 0;
    }
  }
  view_compose_kernel<<<dim3((kOutH * kOutW + 255) / 256, b), 256, 0, s>>>(a);
  LAVB_LAUNCH_OK();
  return 0;
}
