// Scores of one evaluation batch in one launch, one block per sample: the BEV intersection / union counts, the detections matched
// to the recorded actors at four centre-distance thresholds, and the plan's displacement errors.  Everything per pixel and per
// (prediction, actor) pair happens here; the host only sums the counts and ranks the matched flags of a whole recording (AP).
#include "det_match.cuh"

namespace {

using lavb::DetActor;
using lavb::DetGrid;

constexpr int kThreads = 256;
constexpr int kMaxCols = 128;        // 2 classes x at most 64 peaks each
constexpr int kMaxGt = 1024;         // actors of one sample
constexpr int kMaxPlan = 32;
constexpr int kChunk = 256;          // samples per launch: their actor offsets travel as a kernel argument
constexpr int kNumThr = 4;
__constant__ double kThrM[kNumThr] = {0.5, 1.0, 2.0, 4.0};

struct Offsets { int a[kChunk + 1]; };

struct EvalArgs {
  const void* seg; const uint8_t* gt; const float* packed; const DetActor* actors; const float* plan; const float* ego_locs;
  int h, w, gt_planes, n_det, n_plan;
  DetGrid g;
  double win_lo, win_hi;            // the ego window 2 < d < 30 m in pixels
  float min_score;                   // score threshold, float32(min_score): the reference compares fp32 scores in fp32
  float size_thr;                    // class 1: dropped when both box sides are below it (pixels)
  long long* iou; int* ngt; float* score; int* flags; double* plan_err;
};

using lavb::dist2;

template <typename T> __device__ __forceinline__ void load12(const T* p, float (&v)[12]);
template <> __device__ __forceinline__ void load12<float>(const float* p, float (&v)[12]) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float4 f = __ldg(reinterpret_cast<const float4*>(p) + k);
    v[4 * k] = f.x; v[4 * k + 1] = f.y; v[4 * k + 2] = f.z; v[4 * k + 3] = f.w;
  }
}
template <> __device__ __forceinline__ void load12<lavb::h16>(const lavb::h16* p, float (&v)[12]) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const uint2 r = __ldg(reinterpret_cast<const uint2*>(p) + k);
    const float2 a = lavb::unpack_h16(r.x), b = lavb::unpack_h16(r.y);
    v[4 * k] = a.x; v[4 * k + 1] = a.y; v[4 * k + 2] = b.x; v[4 * k + 3] = b.y;
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) eval_batch_kernel(const EvalArgs p, const __grid_constant__ Offsets off, int b0) {
  __shared__ int s_cnt[kThreads / 32][6];
  __shared__ float s_score[kMaxCols];
  __shared__ long long s_loc[kMaxCols];
  __shared__ int s_x[kMaxCols], s_y[kMaxCols], s_keep[kMaxCols], s_flags[kMaxCols];
  __shared__ int s_order[2][kMaxCols / 2], s_nsurv[2], s_ngt[2];
  __shared__ float s_gx[kMaxGt], s_gy[kMaxGt];
  __shared__ signed char s_gcls[kMaxGt];
  __shared__ unsigned char s_used[kNumThr][kMaxGt];
  __shared__ double s_err[kMaxPlan];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int bl = blockIdx.x, b = b0 + bl;
  const long long hw = (long long)p.h * p.w;

  // ---- BEV: per channel, |pred > 0.5 and gt != 0| and |pred > 0.5 or gt != 0|, four pixels per step
  {
    const T* seg = reinterpret_cast<const T*>(p.seg) + (long long)b * hw * 3;
    const uint8_t* gt = p.gt + (long long)b * p.gt_planes * hw;
    int inter[3] = {0, 0, 0}, uni[3] = {0, 0, 0};
#pragma unroll 2
    for (long long q = tid; q < hw / 4; q += kThreads) {
      float v[12];
      load12<T>(seg + q * 12, v);
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const uchar4 t = __ldg(reinterpret_cast<const uchar4*>(gt + c * hw) + q);
        const unsigned char tg[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const bool pr = v[3 * k + c] > 0.5f, gv = tg[k] != 0;
          inter[c] += pr && gv;
          uni[c] += pr || gv;
        }
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        inter[c] += __shfl_xor_sync(0xffffffffu, inter[c], o);
        uni[c] += __shfl_xor_sync(0xffffffffu, uni[c], o);
      }
    if (lane == 0)
#pragma unroll
      for (int c = 0; c < 3; ++c) { s_cnt[warp][2 * c] = inter[c]; s_cnt[warp][2 * c + 1] = uni[c]; }
  }

  // ---- detections: the filters of InferModel.decode_packed on the packed peaks, the same ego window on the actors' centres
  const int ncols = 2 * p.n_det;
  if (tid < 2) { s_nsurv[tid] = 0; s_ngt[tid] = 0; }
  __syncthreads();
  if (tid < ncols) {
    const float* pk = p.packed + (long long)b * 7 * ncols + tid;
    const float sc = pk[0], bw = pk[2 * ncols], bh = pk[3 * ncols];
    long long loc, x, y;
    lavb::peak_pixel(pk[ncols], p.w, loc, x, y);
    const double d = lavb::window_dist((double)x, (double)y, p.g);
    const int cls = tid / p.n_det;
    const bool keep = LAVB_PEAK_SURVIVES(sc, bw, bh, d, cls, p);
    s_score[tid] = sc; s_loc[tid] = loc; s_x[tid] = (int)x; s_y[tid] = (int)y; s_keep[tid] = keep; s_flags[tid] = keep ? 16 : 0;
  }
  const int a0 = off.a[bl], a1 = off.a[bl + 1];
  for (int i = tid; i < a1 - a0; i += kThreads) {
    const DetActor A = p.actors[a0 + i];
    const int cls = A.typ == 0.f ? 0 : A.typ == 1.f ? 1 : -1;    // det_heatmaps ignores any other class
    const float2 c = lavb::det_centre(A, p.g);
    const double d = lavb::window_dist((double)c.x, (double)c.y, p.g);
    const bool keep = cls >= 0 && d > p.win_lo && d < p.win_hi;
    s_gx[i] = c.x; s_gy[i] = c.y; s_gcls[i] = keep ? cls : -1;
#pragma unroll
    for (int k = 0; k < kNumThr; ++k) s_used[k][i] = 0;
    if (keep) atomicAdd(&s_ngt[cls], 1);
  }
  __syncthreads();
  if (tid < ncols && s_keep[tid]) {                               // rank: descending score, then lower flat index, then column
    const int cls = tid / p.n_det, j0 = cls * p.n_det;
    const float sc = s_score[tid];
    const long long loc = s_loc[tid];
    int r = 0;
    for (int i = j0; i < j0 + p.n_det; ++i)
      r += s_keep[i] && lavb::ranks_before(s_score[i], s_loc[i], i, sc, loc, tid);
    s_order[cls][r] = tid;
    atomicAdd(&s_nsurv[cls], 1);
  }
  __syncthreads();
  // greedy matching, one warp per (class, threshold): each prediction in rank order takes the nearest unmatched actor of its
  // class within the threshold; equal distances go to the lower actor row
  {
    const int cls = warp / kNumThr, k = warp % kNumThr;
    const double thr_px = kThrM[k] * (double)p.g.ppm, thr2 = thr_px * thr_px;
    const int n_gt = a1 - a0;
    for (int r = 0; r < s_nsurv[cls]; ++r) {
      const int j = s_order[cls][r];
      const double px = (double)s_x[j], py = (double)s_y[j];
      double d2;
      const int who = lavb::nearest_unmatched(px, py, s_gx, s_gy, n_gt, thr2,
                                              [&](int i) { return s_gcls[i] == cls && !s_used[k][i]; }, &d2);
      if (who >= 0) {
        if (lane == 0) { s_used[k][who] = 1; atomicOr(&s_flags[j], 1 << k); }
        __syncwarp();
      }
    }
  }
  // ---- plan: the displacement of each step against the recorded future (ego_locs[1..T])
  if (warp == 0 && lane < p.n_plan) {
    const float* pl = p.plan + ((long long)b * p.n_plan + lane) * 2;
    const float* gl = p.ego_locs + ((long long)b * (p.n_plan + 1) + lane + 1) * 2;
    s_err[lane] = sqrt(dist2((double)pl[0] - (double)gl[0], (double)pl[1] - (double)gl[1]));
  }
  __syncthreads();
  if (tid < 6) {
    long long s = 0;
    for (int w = 0; w < kThreads / 32; ++w) s += s_cnt[w][tid];
    p.iou[(long long)b * 6 + tid] = s;
  }
  if (tid < 2) p.ngt[b * 2 + tid] = s_ngt[tid];
  if (tid < ncols) {
    p.score[(long long)b * ncols + tid] = s_score[tid];
    p.flags[(long long)b * ncols + tid] = s_flags[tid];
  }
  if (tid == 0) {
    double s = 0.0;
    for (int t = 0; t < p.n_plan; ++t) s += s_err[t];
    p.plan_err[b * 2] = s / p.n_plan;
    p.plan_err[b * 2 + 1] = s_err[p.n_plan - 1];
  }
}

}  // namespace

extern "C" int lavb_eval_batch(const void* d_seg, int seg_dtype, const uint8_t* d_gt, int gt_planes, int b, int h, int w,
                               const float* d_packed, int n_det, const void* d_actors, int n_actors, const int* h_offsets,
                               float ppm, float cx0, float cy0, float cy1, double min_score, const float* d_plan,
                               const float* d_ego_locs, int n_plan, long long* d_iou, int* d_ngt, float* d_score, int* d_flags,
                               double* d_plan_err, void* stream) {
  LAVB_CHECK_ARG(seg_dtype == LAVB_F32 || seg_dtype == LAVB_H16, "eval_batch: seg dtype %d is neither fp32 nor the 16-bit type",
                 seg_dtype);
  LAVB_CHECK_ARG(b >= 0 && h > 0 && w > 0 && (long long)h * w % 4 == 0 && (long long)h * w <= 0x7fffffffLL,
                 "eval_batch: bad sizes (b %d, %d x %d; h * w must be a multiple of 4)", b, h, w);
  LAVB_CHECK_ARG(gt_planes >= 3, "eval_batch: the GT map needs at least 3 planes, got %d", gt_planes);
  LAVB_CHECK_ARG(n_det >= 1 && 2 * n_det <= kMaxCols, "eval_batch: n_det %d outside 1..%d", n_det, kMaxCols / 2);
  LAVB_CHECK_ARG(n_plan >= 1 && n_plan <= kMaxPlan, "eval_batch: n_plan %d outside 1..%d", n_plan, kMaxPlan);
  LAVB_CHECK_ARG(ppm > 0.f, "eval_batch: pixels per metre must be positive");
  LAVB_CHECK_ARG(n_actors >= 0 && h_offsets != nullptr, "eval_batch: bad actor table (%d rows)", n_actors);
  LAVB_CHECK_ARG(h_offsets[0] >= 0 && h_offsets[b] <= n_actors, "eval_batch: offsets [%d, %d] run outside the %d actor rows",
                 h_offsets[0], h_offsets[b], n_actors);
  for (int i = 0; i < b; ++i)
    LAVB_CHECK_ARG(h_offsets[i] <= h_offsets[i + 1] && h_offsets[i + 1] - h_offsets[i] <= kMaxGt,
                   "eval_batch: offsets of sample %d are not monotone or hold more than %d actors (%d -> %d)", i, kMaxGt,
                   h_offsets[i], h_offsets[i + 1]);
  if (b == 0) return 0;
  LAVB_CHECK_ARG(d_seg && d_gt && d_packed && d_plan && d_ego_locs && d_iou && d_ngt && d_score && d_flags && d_plan_err &&
                 (d_actors || h_offsets[b] == h_offsets[0]), "eval_batch: null pointer");
  const size_t seg_align = seg_dtype == LAVB_F32 ? 16 : 8;
  LAVB_CHECK_ARG((uintptr_t)d_seg % seg_align == 0 && (uintptr_t)d_gt % 4 == 0 && (uintptr_t)d_actors % 4 == 0,
                 "eval_batch: seg must be %zu-byte and the GT map 4-byte aligned", seg_align);
  EvalArgs a;
  a.seg = d_seg; a.gt = d_gt; a.packed = d_packed; a.actors = reinterpret_cast<const DetActor*>(d_actors);
  a.plan = d_plan; a.ego_locs = d_ego_locs;
  a.h = h; a.w = w; a.gt_planes = gt_planes; a.n_det = n_det; a.n_plan = n_plan;
  a.g = DetGrid{ppm, cx0, cy0, cy1, 0.f};
  const lavb::DetFilter f = lavb::det_filter(ppm, min_score);
  a.min_score = f.min_score; a.win_lo = f.win_lo; a.win_hi = f.win_hi; a.size_thr = f.size_thr;
  a.iou = d_iou; a.ngt = d_ngt; a.score = d_score; a.flags = d_flags; a.plan_err = d_plan_err;
  cudaStream_t st = (cudaStream_t)stream;
  for (int b0 = 0; b0 < b; b0 += kChunk) {
    const int nb = b - b0 < kChunk ? b - b0 : kChunk;
    Offsets off;
    for (int i = 0; i <= nb; ++i) off.a[i] = h_offsets[b0 + i];
    if (seg_dtype == LAVB_F32)
      eval_batch_kernel<float><<<nb, kThreads, 0, st>>>(a, off, b0);
    else
      eval_batch_kernel<lavb::h16><<<nb, kThreads, 0, st>>>(a, off, b0);
    LAVB_LAUNCH_OK();
  }
  return 0;
}
