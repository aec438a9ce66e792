// Scores of the planners' motion forecasts in one launch, one warp per forecast row and one lane per command branch: each lane
// walks its branch's steps in order (fp64 Euclidean errors, no contraction, summed in ascending step), then every lane of the
// warp takes the same selections over the branches in ascending order.  The host only averages the per-row errors over a
// recording.
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kRowsPerBlock = kThreads / 32;
constexpr int kMaxBranches = 32;
constexpr int kMaxSteps = 32;
constexpr unsigned kFull = 0xffffffffu;

__device__ __forceinline__ double dist(float ax, float ay, float bx, float by) {
  const double dx = (double)ax - (double)bx, dy = (double)ay - (double)by;
  return sqrt(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
}

// `v` replaces `best` when it is lower, or when `best` is NaN and `v` is not: NaN never wins, the first of equals stays.
__device__ __forceinline__ bool lower(double v, double best) { return v < best || (isnan(best) && !isnan(v)); }

__global__ void __launch_bounds__(kThreads) forecast_eval_kernel(const float2* __restrict__ cast, const float* __restrict__ score,
                                                                 const float2* __restrict__ target, const int* __restrict__ cmd,
                                                                 int k, int c, int t, double* __restrict__ err,
                                                                 int* __restrict__ branch) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * kRowsPerBlock + (threadIdx.x >> 5);
  if (row >= k) return;                                           // the whole warp leaves together
  double ade = NAN, fde = NAN;
  float sc = NAN;
  if (lane < c) {
    const float2* cp = cast + (row * c + lane) * t;
    const float2* tp = target + row * t;
    double sum = 0.0, e = 0.0;
    for (int i = 0; i < t; ++i) {
      const float2 a = __ldg(cp + i), b = __ldg(tp + i);
      e = dist(a.x, a.y, b.x, b.y);
      sum = __dadd_rn(sum, e);
    }
    ade = __ddiv_rn(sum, (double)t);
    fde = e;
    sc = __ldg(score + row * c + lane);
  }
  double min_ade = 0.0, min_fde = 0.0;
  float best_score = 0.f;
  int arg_ade = 0, top = 0;
  for (int j = 0; j < c; ++j) {
    const double a = __shfl_sync(kFull, ade, j), f = __shfl_sync(kFull, fde, j);
    const float s = __shfl_sync(kFull, sc, j);
    if (j == 0 || lower(a, min_ade)) { min_ade = a; arg_ade = j; }
    if (j == 0 || lower(f, min_fde)) min_fde = f;
    if (j == 0 || s > best_score || (isnan(best_score) && !isnan(s))) { best_score = s; top = j; }
  }
  const int cm = __ldg(cmd + row);
  const bool has_cmd = cm >= 0 && cm < c;
  const double top_ade = __shfl_sync(kFull, ade, top), top_fde = __shfl_sync(kFull, fde, top);
  const double cmd_ade = __shfl_sync(kFull, ade, has_cmd ? cm : 0), cmd_fde = __shfl_sync(kFull, fde, has_cmd ? cm : 0);
  if (lane < 6) {
    const double v = lane == 0 ? min_ade : lane == 1 ? min_fde : lane == 2 ? top_ade : lane == 3 ? top_fde
                   : !has_cmd ? (double)NAN : lane == 4 ? cmd_ade : cmd_fde;
    err[row * 6 + lane] = v;
  } else if (lane < 8) {
    branch[row * 2 + lane - 6] = lane == 6 ? arg_ade : top;
  }
}

}  // namespace

extern "C" int lavb_forecast_eval(const float* d_cast, const float* d_score, const float* d_target, const int* d_cmd, int k, int c,
                                  int t, double* d_err, int* d_branch, void* stream) {
  LAVB_CHECK_ARG(k >= 0, "forecast_eval: negative row count %d", k);
  LAVB_CHECK_ARG(c >= 1 && c <= kMaxBranches, "forecast_eval: %d branches outside 1..%d", c, kMaxBranches);
  LAVB_CHECK_ARG(t >= 1 && t <= kMaxSteps, "forecast_eval: %d steps outside 1..%d", t, kMaxSteps);
  if (k == 0) return 0;
  LAVB_CHECK_ARG(d_cast && d_score && d_target && d_cmd && d_err && d_branch, "forecast_eval: null pointer");
  LAVB_CHECK_ARG((uintptr_t)d_cast % 8 == 0 && (uintptr_t)d_target % 8 == 0 && (uintptr_t)d_err % 8 == 0 &&
                 (uintptr_t)d_score % 4 == 0 && (uintptr_t)d_cmd % 4 == 0 && (uintptr_t)d_branch % 4 == 0,
                 "forecast_eval: cast, target and err must be 8-byte aligned, score, cmd and branch 4-byte aligned");
  const int blocks = (int)(((long long)k + kRowsPerBlock - 1) / kRowsPerBlock);
  forecast_eval_kernel<<<blocks, kThreads, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float2*>(d_cast), d_score,
                                                                      reinterpret_cast<const float2*>(d_target), d_cmd, k, c, t,
                                                                      d_err, d_branch);
  LAVB_LAUNCH_OK();
  return 0;
}
