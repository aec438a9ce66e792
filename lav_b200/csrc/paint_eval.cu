// Confusion counts of the point painting against the recorded semantic cameras: for every LiDAR point of a batch of sweeps, the
// hit camera and pixel through project_hit.cuh (the projection every painting kernel runs), the recorded class there, and the
// class the painting gives it -- online from the decoder's 16-channel map through deconv_logits.cuh (the logits
// paint_deconv_kernel and seg_confusion_kernel compute), and / or stored, decoded from a recording's lidar_sem row.  Integer
// counters (shared per block, then one global atomic per non-zero bin) keep the counts independent of the schedule.
#include "deconv_logits.cuh"
#include "pillar_grid.cuh"
#include "project_hit.cuh"

namespace {

using lavb::CamSet;
using lavb::DeconvW;

constexpr int kThreads = 256;
constexpr int kMaxCls = 8;
constexpr int kRanges = 4;                 // horizontal distance [0, 10), [10, 20), [20, 40), [40, inf) m
constexpr int kCounters = 8;               // points, nan, roof, in_window, not_visible, not_visible_in_window, invalid, stored_invalid
enum { kPoints, kNan, kRoof, kInWindow, kNotVisible, kNotVisibleInWindow, kInvalid, kStoredInvalid };

struct TagTable { unsigned char cls[256]; };

struct Layout {
  int conf0, agree0, ints;                 // first confusion bin, first agreement bin (or -1), row length
  __host__ __device__ Layout(int ncam, int c, bool online, bool stored) {
    const int per_src = ncam * kRanges * 2 * c * c;
    conf0 = kCounters;
    agree0 = online && stored ? conf0 + 2 * per_src : -1;
    ints = conf0 + ((int)online + (int)stored) * per_src + (online && stored ? ncam * c * c : 0);
  }
};

// LAVAgent.preprocess's roof box (lav_agent.py:448-457) as data_pipeline.roof_keep and roof_filter_kernel test it, in fp32
__device__ __forceinline__ bool roof_point(float x, float y, float z) {
  return x > -2.4f && x < 0.f && y > -0.8f && y < 0.8f && z > -1.5f && z < -1.f;
}

// the class a lidar_sem row s_k = p_k (1 - p_0), k = 1 .. NC-1, encodes, decoded in fp64 without contraction: q = sqrt(sum s_k),
// p_0 = 1 - q, p_k = s_k / q, the first index of the largest of (p_0, p_1, ...); a row summing to 0 is class 0; -1 when a NaN
// enters (a NaN entry, a negative sum, an infinite entry)
template <int NC>
__device__ __forceinline__ int stored_class(const float* row) {
  double s[kMaxCls - 1];
  bool nan = false;
#pragma unroll
  for (int k = 0; k < NC - 1; ++k) { s[k] = (double)__ldg(row + k); nan |= isnan(s[k]); }
  if (nan) return -1;
  double sum = s[0];
#pragma unroll
  for (int k = 1; k < NC - 1; ++k) sum = __dadd_rn(sum, s[k]);
  if (sum == 0.0) return 0;
  const double q = __dsqrt_rn(sum);
  double top = __dsub_rn(1.0, q);
  if (isnan(top)) return -1;
  int best = 0;
#pragma unroll
  for (int k = 0; k < NC - 1; ++k) {
    const double p = __ddiv_rn(s[k], q);
    if (isnan(p)) return -1;
    if (p > top) { top = p; best = k + 1; }                  // strict: ties go to the lower class
  }
  return best;
}

template <typename TF, int NC>
__global__ void __launch_bounds__(kThreads) paint_confusion_kernel(
    const float* __restrict__ pts, int n, const int* __restrict__ meta, const TF* __restrict__ feat,
    const DeconvW* __restrict__ dw, const uint8_t* __restrict__ tags, const __grid_constant__ TagTable lut,
    const float* __restrict__ stored, const __grid_constant__ CamSet cams, int H, int W, const lavb::Grid grid,
    int* __restrict__ out) {
  extern __shared__ int s_cnt[];
  __shared__ DeconvW sw;
  __shared__ unsigned char s_lut[256];
  const int f = blockIdx.y, ncam = cams.ncam;
  const bool online = feat != nullptr;
  const Layout L(ncam, NC, online, stored != nullptr);
  if (online)
    for (int i = threadIdx.x; i < (int)(sizeof(DeconvW) / 4); i += kThreads)
      reinterpret_cast<float*>(&sw)[i] = __ldg(reinterpret_cast<const float*>(dw) + i);
  s_lut[threadIdx.x] = lut.cls[threadIdx.x];               // a shared copy: per-lane tags would serialise on the constant bank
  for (int b = threadIdx.x; b < L.ints; b += kThreads) s_cnt[b] = 0;
  __syncthreads();

  int rows = n, stored_on = stored != nullptr;
  if (meta) {
    rows = min(max(__ldg(meta + 2 * f), 0), n);
    stored_on &= __ldg(meta + 2 * f + 1) != 0;
  }
  const int i = blockIdx.x * kThreads + threadIdx.x;
  // the bins this point adds one to (-1: none): points | nan, roof or in_window | not_visible | not_visible_in_window |
  // online class or invalid | stored class or stored_invalid | agreement
  int bin[7] = {-1, -1, -1, -1, -1, -1, -1};
  if (i < rows) {
    bin[0] = kPoints;
    const float4 p = __ldg(reinterpret_cast<const float4*>(pts) + ((long long)f * n + i));
    if (isnan(p.x) || isnan(p.y) || isnan(p.z)) {
      bin[1] = kNan;
    } else {
      const bool roof = roof_point(p.x, p.y, p.z);
      const bool win = !roof && lavb::in_window(grid, p.x, p.y);
      if (roof) bin[1] = kRoof; else if (win) bin[1] = kInWindow;
      int u = 0, v = 0;
      const int cam = lavb::project_hit(cams, p.x, p.y, p.z, H, W, u, v);
      if (cam < 0) {
        bin[2] = kNotVisible;
        if (win) bin[3] = kNotVisibleInWindow;
      } else {
        const long long img = (long long)f * ncam + cam;
        const int gt = s_lut[__ldg(tags + (img * H + v) * W + u)];
        const float r = __fsqrt_rn(__fadd_rn(__fmul_rn(p.x, p.x), __fmul_rn(p.y, p.y)));
        const int rb = r < 10.f ? 0 : r < 20.f ? 1 : r < 40.f ? 2 : 3;
        const int cell = ((cam * kRanges + rb) * 2 + (int)win) * NC * NC + gt * NC;     // + pred
        const int per_src = ncam * kRanges * 2 * NC * NC;
        int pred_on = -1, pred_st = -1;
        if (online) {
          float fv[16];
          lavb::load_feat16<TF>(feat + ((img * (H >> 1) + (v >> 1)) * (W >> 1) + (u >> 1)) * 16, fv);
          float pr[8];
          lavb::deconv_logits<NC>(sw, fv, v & 1, u & 1, pr);
          bool nan = isnan(pr[0]);
          int best = 0;
          float top = pr[0];
#pragma unroll
          for (int k = 1; k < NC; ++k) {
            nan |= isnan(pr[k]);
            if (pr[k] > top) { top = pr[k]; best = k; }    // strict: ties go to the lower class
          }
          pred_on = nan ? -1 : best;
          bin[4] = nan ? kInvalid : L.conf0 + cell + best;
        }
        if (stored_on) {
          pred_st = stored_class<NC>(stored + ((long long)f * n + i) * (NC - 1));
          bin[5] = pred_st < 0 ? kStoredInvalid : L.conf0 + (int)online * per_src + cell + pred_st;
        }
        if (L.agree0 >= 0 && pred_on >= 0 && pred_st >= 0) bin[6] = L.agree0 + (cam * NC + pred_on) * NC + pred_st;
      }
    }
  }
  // warp-aggregated shared increments: the lanes holding the same bin add their count once
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < 7; ++j) {
    const unsigned peers = __match_any_sync(0xffffffffu, bin[j]);
    if (bin[j] >= 0 && lane == __ffs(peers) - 1) atomicAdd(&s_cnt[bin[j]], __popc(peers));
  }
  __syncthreads();
  int* o = out + (long long)f * L.ints;
  for (int b = threadIdx.x; b < L.ints; b += kThreads) {
    const int c = s_cnt[b];
    if (c) atomicAdd(o + b, c);
  }
}

template <typename TF>
void launch(int c_cls, dim3 grid, size_t smem, cudaStream_t st, const float* pts, int n, const int* meta, const void* feat,
            const DeconvW* dw, const uint8_t* tags, const TagTable& lut, const float* stored, const CamSet& cams, int h, int w,
            const lavb::Grid& g, int* out) {
  const TF* f = static_cast<const TF*>(feat);
  switch (c_cls) {
#define CASE(N) case N: paint_confusion_kernel<TF, N><<<grid, kThreads, smem, st>>>(pts, n, meta, f, dw, tags, lut, stored, cams, \
                                                                                    h, w, g, out); break;
    CASE(2) CASE(3) CASE(4) CASE(5) CASE(6) CASE(7) CASE(8)
#undef CASE
  }
}

}  // namespace

extern "C" int lavb_paint_confusion_ints(int ncam, int c_cls, int online, int stored) {
  if (ncam < 1 || ncam > 4 || c_cls < 2 || c_cls > kMaxCls || !(online || stored)) return -1;
  return Layout(ncam, c_cls, online != 0, stored != 0).ints;
}

extern "C" int lavb_paint_confusion(const float* d_pts, int frames, int n, const int* d_meta, const void* d_feat, int feat_dtype,
                                    const float* d_deconv, const uint8_t* d_tags, const uint8_t* h_lut, const float* d_stored,
                                    const float* h_cams, int ncam, int c_cls, int h, int w, float min_x, float max_x, float min_y,
                                    float max_y, int* d_out, void* stream) {
  LAVB_CHECK_ARG(c_cls >= 2 && c_cls <= kMaxCls, "paint_confusion: %d classes outside 2..%d", c_cls, kMaxCls);
  LAVB_CHECK_ARG(ncam >= 1 && ncam <= 4, "paint_confusion: %d cameras outside 1..4", ncam);
  LAVB_CHECK_ARG(frames >= 0 && frames <= 65535 && n >= 0, "paint_confusion: %d frames outside 0..65535 or %d points < 0", frames,
                 n);
  LAVB_CHECK_ARG(h >= 2 && w >= 2 && h % 2 == 0 && w % 2 == 0 && (long long)h * w <= 0x7fffffffLL,
                 "paint_confusion: the image size %d x %d must be even (the feature map is h/2 x w/2)", h, w);
  LAVB_CHECK_ARG(d_feat != nullptr || d_stored != nullptr, "paint_confusion: neither features nor stored rows to score");
  LAVB_CHECK_ARG(d_feat == nullptr || feat_dtype == LAVB_F32 || feat_dtype == LAVB_H16,
                 "paint_confusion: feature dtype %d is neither fp32 nor the 16-bit type", feat_dtype);
  LAVB_CHECK_ARG(min_x < max_x && min_y < max_y, "paint_confusion: empty pillar grid window");
  LAVB_CHECK_ARG(h_lut != nullptr && h_cams != nullptr, "paint_confusion: null tag table or cameras");
  for (int t = 0; t < 256; ++t)
    LAVB_CHECK_ARG(h_lut[t] < c_cls, "paint_confusion: tag %d maps to class %d, outside 0..%d", t, h_lut[t], c_cls - 1);
  if (frames == 0) return 0;
  LAVB_CHECK_ARG(d_out != nullptr && (n == 0 || (d_pts != nullptr && d_tags != nullptr)), "paint_confusion: null pointer");
  LAVB_CHECK_ARG(d_feat == nullptr || d_deconv != nullptr, "paint_confusion: features without the output layer's table");
  const size_t feat_align = feat_dtype == LAVB_F32 ? 16 : 8;
  LAVB_CHECK_ARG((uintptr_t)d_pts % 16 == 0 && (uintptr_t)d_feat % feat_align == 0 && (uintptr_t)d_deconv % 4 == 0 &&
                 (uintptr_t)d_stored % 4 == 0 && (uintptr_t)d_meta % 4 == 0 && (uintptr_t)d_out % 4 == 0,
                 "paint_confusion: points must be 16-byte, features %zu-byte and the other buffers 4-byte aligned",
                 d_feat ? feat_align : (size_t)1);
  const Layout L(ncam, c_cls, d_feat != nullptr, d_stored != nullptr);
  TagTable lut;
  memcpy(lut.cls, h_lut, 256);
  CamSet cs;
  memcpy(cs.m, h_cams, sizeof(float) * 41 * ncam);
  cs.ncam = ncam;
  const lavb::Grid g{min_x, max_x, min_y, max_y, 0.f, 0, 0};
  cudaStream_t st = (cudaStream_t)stream;
  LAVB_CUDA_OK(cudaMemsetAsync(d_out, 0, sizeof(int) * (size_t)frames * L.ints, st));
  if (n == 0) return 0;
  const dim3 grid(lavb::ceil_div(n, kThreads), frames);
  const size_t smem = sizeof(int) * L.ints;              // <= 4360 ints (C = 8, 4 cameras, both sources): no opt-in needed
  const DeconvW* dw = reinterpret_cast<const DeconvW*>(d_deconv);
  if (d_feat == nullptr || feat_dtype == LAVB_F32)
    launch<float>(c_cls, grid, smem, st, d_pts, n, d_meta, d_feat, dw, d_tags, lut, d_stored, cs, h, w, g, d_out);
  else
    launch<lavb::h16>(c_cls, grid, smem, st, d_pts, n, d_meta, d_feat, dw, d_tags, lut, d_stored, cs, h, w, g, d_out);
  LAVB_LAUNCH_OK();
  return 0;
}
