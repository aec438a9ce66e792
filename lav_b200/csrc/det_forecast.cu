// The match of the vehicles the agent forecasts (its class-1 detections that UniPlanner.infer_batch crops) to the recorded
// actors, one block per sample: the sample's actors into shared memory, its rows ranked, the greedy match in one warp with
// det_match.cuh's search (the one eval_batch_kernel runs), then each matched row's recorded future gathered in parallel as the
// target forecast_eval_kernel scores the row's forecast against.
#include "det_match.cuh"

namespace {

using lavb::DetActor;
using lavb::DetGrid;

constexpr int kThreads = 128;
constexpr int kMaxDet = 64;          // class-1 columns of the packed peaks
constexpr int kMaxGt = 1024;         // actors of one sample
constexpr int kMaxSteps = 32;
constexpr int kChunk = 128;          // samples per launch: their tables travel as a kernel argument (2.5 KB)

// per sample of a chunk: actor rows [act[i], act[i+1]), forecast rows [row[i], row[i+1]), the recorded tracks (labels) of its
// first nobj[i] actor rows, and the packed class-1 columns of its rows as bits (column n_det + c -> bit c)
struct Chunk {
  int act[kChunk + 1], row[kChunk + 1], nobj[kChunk];
  unsigned long long cols[kChunk];
};

struct MatchArgs {
  const float* packed; const DetActor* actors; const float* locs; const float* ego_locs;
  int w, n_det, max_objs, t;
  DetGrid g;
  double win_lo, win_hi, thr2, ppm;  // the ego window 2 < d < 30 m and the squared match radius, in pixels
  int* actor; int* flag; double* dist; float2* target; int* ngt;
};

__global__ void __launch_bounds__(kThreads) det_forecast_match_kernel(const MatchArgs p, const __grid_constant__ Chunk c, int b0) {
  __shared__ float s_gx[kMaxGt], s_gy[kMaxGt];
  __shared__ unsigned char s_veh[kMaxGt];                           // a vehicle in the window, not yet taken
  __shared__ float s_score[kMaxDet];
  __shared__ long long s_loc[kMaxDet];
  __shared__ int s_x[kMaxDet], s_y[kMaxDet], s_col[kMaxDet], s_order[kMaxDet], s_who[kMaxDet];
  __shared__ double s_d2[kMaxDet];
  __shared__ int s_cnt[2];
  const int tid = threadIdx.x, bl = blockIdx.x, b = b0 + bl;
  const int a0 = c.act[bl], n_gt = c.act[bl + 1] - a0, r0 = c.row[bl], n_rows = c.row[bl + 1] - r0, n_obj = c.nobj[bl];
  const unsigned long long cols = c.cols[bl];
  if (tid < 2) s_cnt[tid] = 0;
  __syncthreads();
  for (int i = tid; i < n_gt; i += kThreads) {                      // eval_batch's vehicle class and window
    const DetActor A = p.actors[a0 + i];
    const float2 q = lavb::det_centre(A, p.g);
    const double d = lavb::window_dist((double)q.x, (double)q.y, p.g);
    const bool veh = A.typ == 1.f && d > p.win_lo && d < p.win_hi;
    s_gx[i] = q.x; s_gy[i] = q.y; s_veh[i] = veh;
    if (veh) atomicAdd(&s_cnt[i < n_obj ? 0 : 1], 1);
  }
  if (tid < p.n_det && (cols >> tid & 1ull)) {                      // row r = the r-th set bit
    const int r = __popcll(cols & ((1ull << tid) - 1ull)), col = p.n_det + tid;
    const float* pk = p.packed + (long long)b * 7 * 2 * p.n_det + col;
    long long loc, x, y;
    lavb::peak_pixel(pk[2 * p.n_det], p.w, loc, x, y);
    s_score[r] = pk[0]; s_loc[r] = loc; s_x[r] = (int)x; s_y[r] = (int)y; s_col[r] = col;
  }
  __syncthreads();
  if (tid < n_rows) {                                               // rank: descending score, then lower flat index, then column
    int r = 0;
    for (int i = 0; i < n_rows; ++i) r += lavb::ranks_before(s_score[i], s_loc[i], s_col[i], s_score[tid], s_loc[tid], s_col[tid]);
    s_order[r] = tid;
  }
  __syncthreads();
  if (tid < 32) {                                                   // greedy: each row in rank order takes the nearest free vehicle
    for (int k = 0; k < n_rows; ++k) {
      const int j = s_order[k];
      double d2;
      const int who = lavb::nearest_unmatched((double)s_x[j], (double)s_y[j], s_gx, s_gy, n_gt, p.thr2,
                                              [&](int i) { return s_veh[i] != 0; }, &d2);
      if (tid == 0) {
        s_who[j] = who; s_d2[j] = d2;
        if (who >= 0) s_veh[who] = 0;
      }
      __syncwarp();
    }
  }
  __syncthreads();
  for (int j = tid; j < n_rows; j += kThreads) {
    const int who = s_who[j];
    p.actor[r0 + j] = who;
    p.flag[r0 + j] = (who >= 0) | ((who >= 0 && who < n_obj) << 1);
    p.dist[r0 + j] = who >= 0 ? __ddiv_rn(sqrt(s_d2[j]), p.ppm) : (double)NAN;
  }
  // target of a row matched to a tracked actor a: locs[b, a, 1 + s] - ego_locs[b, 0], the frame of other_cast_locs; NaN otherwise
  const float* ego = p.ego_locs + (long long)b * (p.t + 1) * 2;
  for (int e = tid; e < n_rows * p.t; e += kThreads) {
    const int j = e / p.t, s = e - j * p.t, who = s_who[j];
    float2 v = make_float2(NAN, NAN);
    if (who >= 0 && who < n_obj) {
      const float* l = p.locs + (((long long)b * p.max_objs + who) * (p.t + 1) + 1 + s) * 2;
      v = make_float2(__fsub_rn(__ldg(l), __ldg(ego)), __fsub_rn(__ldg(l + 1), __ldg(ego + 1)));
    }
    p.target[(long long)(r0 + j) * p.t + s] = v;
  }
  if (tid < 2) p.ngt[b * 2 + tid] = s_cnt[tid];
}

}  // namespace

extern "C" int lavb_det_forecast_match(const float* d_packed, int b, int w, int n_det, const void* d_actors, int n_actors,
                                       const int* h_actor_offsets, const int* h_row_offsets, const int* h_cols,
                                       const int* h_num_objs, const float* d_locs, const float* d_ego_locs, int max_objs, int t,
                                       float ppm, float cx0, float cy0, float cy1, double match_m, int* d_actor, int* d_flag,
                                       double* d_dist, float* d_target, int* d_ngt, void* stream) {
  LAVB_CHECK_ARG(b >= 0 && w > 0, "det_forecast_match: bad sizes (b %d, w %d)", b, w);
  LAVB_CHECK_ARG(n_det >= 1 && n_det <= kMaxDet, "det_forecast_match: n_det %d outside 1..%d", n_det, kMaxDet);
  LAVB_CHECK_ARG(t >= 1 && t <= kMaxSteps, "det_forecast_match: %d steps outside 1..%d", t, kMaxSteps);
  LAVB_CHECK_ARG(max_objs >= 0, "det_forecast_match: negative label slot count %d", max_objs);
  LAVB_CHECK_ARG(ppm > 0.f, "det_forecast_match: pixels per metre must be positive");
  LAVB_CHECK_ARG(match_m > 0.0 && match_m < 1e6, "det_forecast_match: match radius %g m outside (0, 1e6)", match_m);
  LAVB_CHECK_ARG(n_actors >= 0 && h_actor_offsets && h_row_offsets && h_num_objs && (h_cols || h_row_offsets[b] == 0),
                 "det_forecast_match: missing host table (%d actor rows)", n_actors);
  LAVB_CHECK_ARG(h_actor_offsets[0] >= 0 && h_actor_offsets[b] <= n_actors,
                 "det_forecast_match: actor offsets [%d, %d] run outside the %d actor rows", h_actor_offsets[0], h_actor_offsets[b],
                 n_actors);
  LAVB_CHECK_ARG(h_row_offsets[0] == 0, "det_forecast_match: row offsets must start at 0, got %d", h_row_offsets[0]);
  for (int i = 0; i < b; ++i) {
    const int a0 = h_actor_offsets[i], a1 = h_actor_offsets[i + 1], r0 = h_row_offsets[i], r1 = h_row_offsets[i + 1];
    LAVB_CHECK_ARG(a0 <= a1 && a1 - a0 <= kMaxGt, "det_forecast_match: actor offsets of sample %d are not monotone or hold more "
                   "than %d actors (%d -> %d)", i, kMaxGt, a0, a1);
    LAVB_CHECK_ARG(r0 <= r1 && r1 - r0 <= n_det, "det_forecast_match: row offsets of sample %d are not monotone or hold more than "
                   "n_det = %d rows (%d -> %d)", i, n_det, r0, r1);
    LAVB_CHECK_ARG(h_num_objs[i] >= 0 && h_num_objs[i] <= max_objs, "det_forecast_match: sample %d has %d tracks, outside 0..%d",
                   i, h_num_objs[i], max_objs);
    for (int r = r0; r < r1; ++r)
      LAVB_CHECK_ARG(h_cols[r] >= n_det && h_cols[r] < 2 * n_det && (r == r0 || h_cols[r] > h_cols[r - 1]),
                     "det_forecast_match: row %d of sample %d has column %d: rows take ascending class-1 columns %d..%d", r, i,
                     h_cols[r], n_det, 2 * n_det - 1);
  }
  if (b == 0) return 0;
  const int k = h_row_offsets[b];
  LAVB_CHECK_ARG(d_packed && d_locs && d_ego_locs && d_ngt && (d_actors || h_actor_offsets[b] == h_actor_offsets[0]) &&
                 (k == 0 || (d_actor && d_flag && d_dist && d_target)), "det_forecast_match: null pointer");
  LAVB_CHECK_ARG((uintptr_t)d_packed % 4 == 0 && (uintptr_t)d_actors % 4 == 0 && (uintptr_t)d_locs % 4 == 0 &&
                 (uintptr_t)d_ego_locs % 4 == 0 && (uintptr_t)d_actor % 4 == 0 && (uintptr_t)d_flag % 4 == 0 &&
                 (uintptr_t)d_ngt % 4 == 0 && (uintptr_t)d_dist % 8 == 0 && (uintptr_t)d_target % 8 == 0,
                 "det_forecast_match: dist and target must be 8-byte aligned, the other arrays 4-byte aligned");
  MatchArgs a;
  a.packed = d_packed; a.actors = reinterpret_cast<const DetActor*>(d_actors); a.locs = d_locs; a.ego_locs = d_ego_locs;
  a.w = w; a.n_det = n_det; a.max_objs = max_objs; a.t = t;
  a.g = DetGrid{ppm, cx0, cy0, cy1, 0.f};
  a.win_lo = 2.0;                                                 // decode_packed's `dist <= 2 | dist >= 30 * ppm` (pixels)
  a.win_hi = 30.0 * (double)ppm;
  const double thr_px = match_m * (double)ppm;
  a.thr2 = thr_px * thr_px;
  a.ppm = (double)ppm;
  a.actor = d_actor; a.flag = d_flag; a.dist = d_dist; a.target = reinterpret_cast<float2*>(d_target); a.ngt = d_ngt;
  cudaStream_t st = (cudaStream_t)stream;
  for (int b0 = 0; b0 < b; b0 += kChunk) {
    const int nb = b - b0 < kChunk ? b - b0 : kChunk;
    Chunk ch;
    for (int i = 0; i <= nb; ++i) { ch.act[i] = h_actor_offsets[b0 + i]; ch.row[i] = h_row_offsets[b0 + i]; }
    for (int i = 0; i < nb; ++i) {
      ch.nobj[i] = h_num_objs[b0 + i];
      ch.cols[i] = 0;
      for (int r = h_row_offsets[b0 + i]; r < h_row_offsets[b0 + i + 1]; ++r) ch.cols[i] |= 1ull << (h_cols[r] - n_det);
    }
    det_forecast_match_kernel<<<nb, kThreads, 0, st>>>(a, ch, b0);
    LAVB_LAUNCH_OK();
  }
  return 0;
}
