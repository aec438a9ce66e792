// Box scores of the decoded detections, one block per sample: the survivors and ground truth of eval_batch_kernel, each
// survivor's rotated box matched greedily by IoU at three thresholds, and the errors of the 2 m centre match (the IoU, the
// translation, the scale error and the heading error).  Every box operation is fp64 with no contraction, in the order written
// in lavb_det_box_eval's contract (include/lav_b200.h), so a numpy statement gets the same bits up to the fp64 cos / sin /
// atan2, which are not correctly rounded.
#include "det_match.cuh"

namespace {

using lavb::DetActor;
using lavb::DetGrid;

constexpr int kThreads = 128;        // warps 0, 1: the IoU match of class 0, 1; warps 2, 3: their 2 m match
constexpr int kMaxCols = 128;        // 2 classes x at most 64 peaks each
constexpr int kMaxGt = 1024;         // actors of one sample
constexpr int kChunk = 256;          // samples per launch: their actor offsets travel as a kernel argument
constexpr int kNumIou = 3;
constexpr int kMaxPoly = 16;         // vertices kept of a clipped polygon (a convex one never has more than 8)
constexpr int kNumErr = 5;
__constant__ double kIouThr[kNumIou] = {0.3, 0.5, 0.7};

struct Offsets { int a[kChunk + 1]; };

struct BoxArgs {
  const float* packed; const DetActor* actors;
  int w, n_det;
  DetGrid g;
  double win_lo, win_hi;             // LAVB_PEAK_SURVIVES' fields (det_filter)
  float min_score, size_thr;
  double thr2, ppm;                  // the squared 2 m match radius in pixels; pixels per metre
  float* score; int* flags; int* actor; double* err; int* ngt;
};

__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }

struct Box { double x[4], y[4], area, lo_x, hi_x, lo_y, hi_y; bool ok; };

// |shoelace| / 2 of n vertices: s = sum over i ascending of (x_i * y_{i+1} - x_{i+1} * y_i), index n wrapping to 0.
__device__ double poly_area(const double* x, const double* y, int n) {
  double s = 0.0;
  for (int i = 0; i < n; ++i) {
    const int j = i + 1 == n ? 0 : i + 1;
    s = add(s, sub(mul(x[i], y[j]), mul(x[j], y[i])));
  }
  return fabs(s) * 0.5;
}

// visualize's corners of a box centred at (cx, cy) with half extents (hw, hh) and heading (c, s): u = (-(s * hw), c * hw),
// v = (-(c * hh), -(s * hh)), corner k = centre + (a_k * u + b_k * v), (a, b) = (-1, -1), (-1, 1), (1, 1), (1, -1).
__device__ Box make_box(double cx, double cy, double hw, double hh, double c, double s) {
  Box q;
  const double ux = -mul(s, hw), uy = mul(c, hw), vx = -mul(c, hh), vy = -mul(s, hh);
  const double a[4] = {-1.0, -1.0, 1.0, 1.0}, b[4] = {-1.0, 1.0, 1.0, -1.0};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    q.x[k] = add(cx, add(a[k] * ux, b[k] * vx));
    q.y[k] = add(cy, add(a[k] * uy, b[k] * vy));
  }
  q.ok = isfinite(hw) && hw > 0.0 && isfinite(hh) && hh > 0.0 && isfinite(c) && isfinite(s) && isfinite(cx) && isfinite(cy);
  q.area = q.ok ? poly_area(q.x, q.y, 4) : 0.0;
  q.ok = q.ok && q.area > 0.0;
  q.lo_x = fmin(fmin(q.x[0], q.x[1]), fmin(q.x[2], q.x[3])); q.hi_x = fmax(fmax(q.x[0], q.x[1]), fmax(q.x[2], q.x[3]));
  q.lo_y = fmin(fmin(q.y[0], q.y[1]), fmin(q.y[2], q.y[3])); q.hi_y = fmax(fmax(q.y[0], q.y[1]), fmax(q.y[2], q.y[3]));
  return q;
}

// IoU of detection box P and ground-truth box Q: 0 when either is degenerate or their bounding boxes are apart; else P clipped by
// each edge of Q in turn (Sutherland-Hodgman), I = the clipped polygon's area, IoU = I / ((A + B) - I).
__device__ double box_iou(const Box& P, const Box& Q) {
  if (!P.ok || !Q.ok || P.hi_x < Q.lo_x || Q.hi_x < P.lo_x || P.hi_y < Q.lo_y || Q.hi_y < P.lo_y) return 0.0;
  double xa[kMaxPoly], ya[kMaxPoly], xb[kMaxPoly], yb[kMaxPoly];
  int n = 4;
#pragma unroll
  for (int k = 0; k < 4; ++k) { xa[k] = P.x[k]; ya[k] = P.y[k]; }
  double *sx = xa, *sy = ya, *dx = xb, *dy = yb;
  for (int e = 0; e < 4 && n > 0; ++e) {
    const double x0 = Q.x[e], y0 = Q.y[e], ex = sub(Q.x[(e + 1) & 3], x0), ey = sub(Q.y[(e + 1) & 3], y0);
    // side of a point: ex * (py - y0) - ey * (px - x0); <= 0 is inside (the corners run clockwise)
    auto side = [&](double px, double py) { return sub(mul(ex, sub(py, y0)), mul(ey, sub(px, x0))); };
    int m = 0;
    double px = sx[n - 1], py = sy[n - 1], sp = side(px, py);
    for (int i = 0; i < n; ++i) {
      const double qx = sx[i], qy = sy[i], sq = side(qx, qy);
      if ((sq <= 0.0) != (sp <= 0.0) && m < kMaxPoly) {                 // the edge crosses: p + t * (q - p), t = sp / (sp - sq)
        const double t = __ddiv_rn(sp, sub(sp, sq));
        dx[m] = add(px, mul(t, sub(qx, px))); dy[m] = add(py, mul(t, sub(qy, py))); ++m;
      }
      if (sq <= 0.0 && m < kMaxPoly) { dx[m] = qx; dy[m] = qy; ++m; }
      px = qx; py = qy; sp = sq;
    }
    double* t;
    t = sx; sx = dx; dx = t;
    t = sy; sy = dy; dy = t;
    n = m;
  }
  const double inter = n >= 3 ? poly_area(sx, sy, n) : 0.0;
  const double uni = sub(add(P.area, Q.area), inter);
  return uni > 0.0 ? __ddiv_rn(inter, uni) : 0.0;
}

__global__ void __launch_bounds__(kThreads) det_box_eval_kernel(const BoxArgs p, const __grid_constant__ Offsets off, int b0) {
  __shared__ float s_score[kMaxCols];
  __shared__ long long s_loc[kMaxCols];
  __shared__ int s_x[kMaxCols], s_y[kMaxCols], s_keep[kMaxCols], s_flags[kMaxCols], s_who[kNumIou + 1][kMaxCols];
  __shared__ double s_d2[kMaxCols];
  __shared__ int s_order[2][kMaxCols / 2], s_nsurv[2], s_ngt[2];
  __shared__ float s_gx[kMaxGt], s_gy[kMaxGt], s_gbx[kMaxGt], s_gby[kMaxGt];
  __shared__ double s_gc[kMaxGt], s_gs[kMaxGt];
  __shared__ signed char s_gcls[kMaxGt];
  __shared__ unsigned char s_used[kNumIou + 1][kMaxGt];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int bl = blockIdx.x, b = b0 + bl;
  const int ncols = 2 * p.n_det;
  const float* pk0 = p.packed + (long long)b * 7 * ncols;

  // ---- eval_batch_kernel's survivors and ground truth
  if (tid < 2) { s_nsurv[tid] = 0; s_ngt[tid] = 0; }
  __syncthreads();
  if (tid < ncols) {
    const float* pk = pk0 + tid;
    const float sc = pk[0], bw = pk[2 * ncols], bh = pk[3 * ncols];
    long long loc, x, y;
    lavb::peak_pixel(pk[ncols], p.w, loc, x, y);
    const double d = lavb::window_dist((double)x, (double)y, p.g);
    const int cls = tid / p.n_det;
    const bool keep = LAVB_PEAK_SURVIVES(sc, bw, bh, d, cls, p);
    s_score[tid] = sc; s_loc[tid] = loc; s_x[tid] = (int)x; s_y[tid] = (int)y; s_keep[tid] = keep; s_flags[tid] = keep ? 16 : 0;
#pragma unroll
    for (int k = 0; k <= kNumIou; ++k) s_who[k][tid] = -1;
  }
  const int a0 = off.a[bl], n_gt = off.a[bl + 1] - a0;
  for (int i = tid; i < n_gt; i += kThreads) {
    const DetActor A = p.actors[a0 + i];
    const int cls = A.typ == 0.f ? 0 : A.typ == 1.f ? 1 : -1;
    const float2 c = lavb::det_centre(A, p.g);
    const double d = lavb::window_dist((double)c.x, (double)c.y, p.g);
    const bool keep = cls >= 0 && d > p.win_lo && d < p.win_hi;
    double sn, cs;
    sincos((double)A.ori, &sn, &cs);
    s_gx[i] = c.x; s_gy[i] = c.y; s_gbx[i] = A.bx; s_gby[i] = A.by; s_gc[i] = cs; s_gs[i] = sn; s_gcls[i] = keep ? cls : -1;
#pragma unroll
    for (int k = 0; k <= kNumIou; ++k) s_used[k][i] = 0;
    if (keep) atomicAdd(&s_ngt[cls], 1);
  }
  __syncthreads();
  if (tid < ncols && s_keep[tid]) {                               // rank: descending score, then lower flat index, then column
    const int cls = tid / p.n_det, j0 = cls * p.n_det;
    int r = 0;
    for (int i = j0; i < j0 + p.n_det; ++i) r += s_keep[i] && lavb::ranks_before(s_score[i], s_loc[i], i, s_score[tid], s_loc[tid], tid);
    s_order[cls][r] = tid;
    atomicAdd(&s_nsurv[cls], 1);
  }
  __syncthreads();
  const auto det_box = [&](int j) {
    const float* pk = pk0 + j;
    return make_box((double)s_x[j], (double)s_y[j], (double)pk[2 * ncols], (double)pk[3 * ncols], (double)pk[4 * ncols],
                    (double)pk[5 * ncols]);
  };
  const auto gt_box = [&](int i) {                                // half extents bx * ppm, by * ppm: exact in fp64
    return make_box((double)s_gx[i], (double)s_gy[i], mul((double)s_gbx[i], p.ppm), mul((double)s_gby[i], p.ppm), s_gc[i], s_gs[i]);
  };
  const int cls = warp & 1;
  if (warp < 2) {
    // the IoU match of class cls, every threshold in one pass: each survivor in rank order takes, per threshold, the untaken
    // actor of its class with the highest IoU >= the threshold; equal IoUs go to the lower actor row
    for (int r = 0; r < s_nsurv[cls]; ++r) {
      const int j = s_order[cls][r];
      const Box P = det_box(j);
      double best[kNumIou];
      int who[kNumIou];
#pragma unroll
      for (int k = 0; k < kNumIou; ++k) { best[k] = -1.0; who[k] = 0x7fffffff; }
      if (P.ok)
        for (int i = lane; i < n_gt; i += 32) {                    // lanes visit rows in ascending order: the first equal stays
          if (s_gcls[i] != cls || (s_used[0][i] && s_used[1][i] && s_used[2][i])) continue;
          const double iou = box_iou(P, gt_box(i));
#pragma unroll
          for (int k = 0; k < kNumIou; ++k)
            if (!s_used[k][i] && iou >= kIouThr[k] && iou > best[k]) { best[k] = iou; who[k] = i; }
        }
#pragma unroll
      for (int k = 0; k < kNumIou; ++k) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const double ob = __shfl_xor_sync(0xffffffffu, best[k], o);
          const int ow = __shfl_xor_sync(0xffffffffu, who[k], o);
          if (ob > best[k] || (ob == best[k] && ow < who[k])) { best[k] = ob; who[k] = ow; }
        }
      }
      if (lane == 0)
#pragma unroll
        for (int k = 0; k < kNumIou; ++k)
          if (who[k] != 0x7fffffff) { s_used[k][who[k]] = 1; s_who[k][j] = who[k]; atomicOr(&s_flags[j], 1 << k); }
      __syncwarp();
    }
  } else {
    // eval_batch's 2 m match of class cls
    for (int r = 0; r < s_nsurv[cls]; ++r) {
      const int j = s_order[cls][r];
      double d2;
      const int who = lavb::nearest_unmatched((double)s_x[j], (double)s_y[j], s_gx, s_gy, n_gt, p.thr2,
                                              [&](int i) { return s_gcls[i] == cls && !s_used[kNumIou][i]; }, &d2);
      if (who >= 0) {
        if (lane == 0) { s_used[kNumIou][who] = 1; s_who[kNumIou][j] = who; s_d2[j] = d2; atomicOr(&s_flags[j], 1 << kNumIou); }
        __syncwarp();
      }
    }
  }
  __syncthreads();
  if (tid < ncols) {
    const long long o = (long long)b * ncols + tid;
    double e[kNumErr] = {NAN, NAN, NAN, NAN, NAN};
    const int a = s_who[kNumIou][tid];
    if (a >= 0) {
      const float* pk = pk0 + tid;
      const double hw = (double)pk[2 * ncols], hh = (double)pk[3 * ncols];
      const double gw = mul((double)s_gbx[a], p.ppm), gh = mul((double)s_gby[a], p.ppm);
      e[0] = box_iou(det_box(tid), gt_box(a));
      e[1] = __ddiv_rn(sqrt(s_d2[tid]), p.ppm);
      // scale: 1 - the IoU of the two boxes on one centre and heading, from the half extents alone
      const bool ext = isfinite(hw) && hw > 0.0 && isfinite(hh) && hh > 0.0 && isfinite(gw) && gw > 0.0 && isfinite(gh) && gh > 0.0;
      const double i2 = mul(fmin(hw, gw), fmin(hh, gh));
      e[2] = sub(1.0, ext ? __ddiv_rn(i2, sub(add(mul(hw, hh), mul(gw, gh)), i2)) : 0.0);
      // heading: r = fmod(|atan2(sin, cos) - ori|, 2 pi), the error min(r, 2 pi - r)
      const double two_pi = 6.283185307179586;
      const double rr = fmod(fabs(sub(atan2((double)pk[5 * ncols], (double)pk[4 * ncols]), (double)p.actors[a0 + a].ori)), two_pi);
      e[3] = rr <= sub(two_pi, rr) ? rr : sub(two_pi, rr);
      e[4] = __ddiv_rn(lavb::window_dist((double)s_gx[a], (double)s_gy[a], p.g), p.ppm);
    }
    p.score[o] = s_score[tid];
    p.flags[o] = s_flags[tid];
#pragma unroll
    for (int k = 0; k <= kNumIou; ++k) p.actor[o * (kNumIou + 1) + k] = s_who[k][tid];
#pragma unroll
    for (int k = 0; k < kNumErr; ++k) p.err[o * kNumErr + k] = e[k];
  }
  if (tid < 2) p.ngt[b * 2 + tid] = s_ngt[tid];
}

}  // namespace

extern "C" int lavb_det_box_eval(const float* d_packed, int b, int w, int n_det, const void* d_actors, int n_actors,
                                 const int* h_offsets, float ppm, float cx0, float cy0, float cy1, double min_score, float* d_score,
                                 int* d_flags, int* d_actor, double* d_err, int* d_ngt, void* stream) {
  LAVB_CHECK_ARG(b >= 0 && w > 0, "det_box_eval: bad sizes (b %d, w %d)", b, w);
  LAVB_CHECK_ARG(n_det >= 1 && 2 * n_det <= kMaxCols, "det_box_eval: n_det %d outside 1..%d", n_det, kMaxCols / 2);
  LAVB_CHECK_ARG(ppm > 0.f, "det_box_eval: pixels per metre must be positive");
  LAVB_CHECK_ARG(n_actors >= 0 && h_offsets != nullptr, "det_box_eval: bad actor table (%d rows)", n_actors);
  LAVB_CHECK_ARG(h_offsets[0] >= 0 && h_offsets[b] <= n_actors, "det_box_eval: offsets [%d, %d] run outside the %d actor rows",
                 h_offsets[0], h_offsets[b], n_actors);
  for (int i = 0; i < b; ++i)
    LAVB_CHECK_ARG(h_offsets[i] <= h_offsets[i + 1] && h_offsets[i + 1] - h_offsets[i] <= kMaxGt,
                   "det_box_eval: offsets of sample %d are not monotone or hold more than %d actors (%d -> %d)", i, kMaxGt,
                   h_offsets[i], h_offsets[i + 1]);
  if (b == 0) return 0;
  LAVB_CHECK_ARG(d_packed && d_score && d_flags && d_actor && d_err && d_ngt && (d_actors || h_offsets[b] == h_offsets[0]),
                 "det_box_eval: null pointer");
  LAVB_CHECK_ARG((uintptr_t)d_packed % 4 == 0 && (uintptr_t)d_actors % 4 == 0 && (uintptr_t)d_score % 4 == 0 &&
                 (uintptr_t)d_flags % 4 == 0 && (uintptr_t)d_actor % 4 == 0 && (uintptr_t)d_ngt % 4 == 0 && (uintptr_t)d_err % 8 == 0,
                 "det_box_eval: err must be 8-byte aligned, the other arrays 4-byte aligned");
  BoxArgs a;
  a.packed = d_packed; a.actors = reinterpret_cast<const DetActor*>(d_actors);
  a.w = w; a.n_det = n_det;
  a.g = DetGrid{ppm, cx0, cy0, cy1, 0.f};
  const lavb::DetFilter f = lavb::det_filter(ppm, min_score);
  a.min_score = f.min_score; a.win_lo = f.win_lo; a.win_hi = f.win_hi; a.size_thr = f.size_thr;
  const double thr_px = 2.0 * (double)ppm;                        // eval_batch's 2 m threshold
  a.thr2 = thr_px * thr_px;
  a.ppm = (double)ppm;
  a.score = d_score; a.flags = d_flags; a.actor = d_actor; a.err = d_err; a.ngt = d_ngt;
  cudaStream_t st = (cudaStream_t)stream;
  for (int b0 = 0; b0 < b; b0 += kChunk) {
    const int nb = b - b0 < kChunk ? b - b0 : kChunk;
    Offsets off;
    for (int i = 0; i <= nb; ++i) off.a[i] = h_offsets[b0 + i];
    det_box_eval_kernel<<<nb, kThreads, 0, st>>>(a, off, b0);
    LAVB_LAUNCH_OK();
  }
  return 0;
}
