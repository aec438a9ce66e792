// Confusion counts of ERFNet's class map against the recorded CARLA tags, straight from the decoder's 16-channel map: the last
// layer (deconv_logits.cuh, the arithmetic of the painting gather), the argmax and the counting in one launch, so the (h x w x C)
// logit maps are never written.  One thread per feature pixel evaluates its 2 x 2 output pixels from one load of the 16 features;
// integer counters (shared per block, then global atomics) keep the counts independent of the schedule.
#include "deconv_logits.cuh"

namespace {

using lavb::DeconvW;

constexpr int kThreads = 256;
constexpr int kMaxCls = 8;

struct TagTable { unsigned char cls[256]; };

template <typename TF, int NC>
__global__ void __launch_bounds__(kThreads) seg_confusion_kernel(const TF* __restrict__ feat, const DeconvW* __restrict__ dw,
                                                                 const uint8_t* __restrict__ labels,
                                                                 const __grid_constant__ TagTable lut, int h, int w,
                                                                 int* __restrict__ out) {
  constexpr int kBins = NC * NC + 1;               // confusion[gt][pred], then invalid
  __shared__ DeconvW sw;
  __shared__ unsigned char s_lut[256];
  __shared__ int s_cnt[kBins];
  for (int i = threadIdx.x; i < (int)(sizeof(DeconvW) / 4); i += kThreads)
    reinterpret_cast<float*>(&sw)[i] = __ldg(reinterpret_cast<const float*>(dw) + i);
  s_lut[threadIdx.x] = lut.cls[threadIdx.x];       // a shared copy: per-lane tags would serialise on the constant bank
  if (threadIdx.x < kBins) s_cnt[threadIdx.x] = 0;
  __syncthreads();

  const int img = blockIdx.y, hh = h >> 1, wh = w >> 1;
  const long long q = (long long)blockIdx.x * kThreads + threadIdx.x;
  const bool live = q < (long long)hh * wh;
  int bin[4] = {-1, -1, -1, -1};
  if (live) {
    const int fy = (int)(q / wh), fx = (int)(q - (long long)fy * wh);
    float fv[16];
    lavb::load_feat16<TF>(feat + ((long long)img * hh * wh + q) * 16, fv);
    const uint8_t* lab = labels + (long long)img * h * w + (long long)(2 * fy) * w + 2 * fx;
#pragma unroll
    for (int pv = 0; pv < 2; ++pv) {
      const uchar2 t = *reinterpret_cast<const uchar2*>(lab + (long long)pv * w);
#pragma unroll
      for (int pu = 0; pu < 2; ++pu) {
        float pr[8];
        lavb::deconv_logits<NC>(sw, fv, pv, pu, pr);
        bool nan = isnan(pr[0]);
        int best = 0;
        float top = pr[0];
#pragma unroll
        for (int k = 1; k < NC; ++k) {
          nan |= isnan(pr[k]);
          if (pr[k] > top) { top = pr[k]; best = k; }   // strict: ties go to the lower class
        }
        const int gt = s_lut[pu ? t.y : t.x];
        bin[2 * pv + pu] = nan ? NC * NC : gt * NC + best;
      }
    }
  }
  // warp-aggregated shared increments: the lanes holding the same bin add their count once
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const unsigned peers = __match_any_sync(0xffffffffu, bin[j]);
    if (bin[j] >= 0 && lane == __ffs(peers) - 1) atomicAdd(&s_cnt[bin[j]], __popc(peers));
  }
  __syncthreads();
  if (threadIdx.x < kBins) {
    const int c = s_cnt[threadIdx.x];
    if (c) atomicAdd(out + (long long)img * kBins + threadIdx.x, c);
  }
}

template <typename TF>
void launch(int c_cls, dim3 grid, cudaStream_t st, const void* feat, const DeconvW* dw, const uint8_t* labels, const TagTable& lut,
            int h, int w, int* out) {
  const TF* f = static_cast<const TF*>(feat);
  switch (c_cls) {
#define CASE(N) case N: seg_confusion_kernel<TF, N><<<grid, kThreads, 0, st>>>(f, dw, labels, lut, h, w, out); break;
    CASE(2) CASE(3) CASE(4) CASE(5) CASE(6) CASE(7) CASE(8)
#undef CASE
  }
}

}  // namespace

extern "C" int lavb_seg_confusion(const void* d_feat, int feat_dtype, const float* d_deconv, const uint8_t* d_labels,
                                  const uint8_t* h_lut, int n, int c_cls, int h, int w, int* d_out, void* stream) {
  LAVB_CHECK_ARG(feat_dtype == LAVB_F32 || feat_dtype == LAVB_H16, "seg_confusion: feature dtype %d is neither fp32 nor the "
                 "16-bit type", feat_dtype);
  LAVB_CHECK_ARG(c_cls >= 2 && c_cls <= kMaxCls, "seg_confusion: %d classes outside 2..%d", c_cls, kMaxCls);
  LAVB_CHECK_ARG(n >= 0 && n <= 65535, "seg_confusion: %d images outside 0..65535", n);
  LAVB_CHECK_ARG(h >= 2 && w >= 2 && h % 2 == 0 && w % 2 == 0 && (long long)h * w <= 0x7fffffffLL,
                 "seg_confusion: the image size %d x %d must be even (the feature map is h/2 x w/2)", h, w);
  LAVB_CHECK_ARG(h_lut != nullptr, "seg_confusion: null tag table");
  for (int t = 0; t < 256; ++t)
    LAVB_CHECK_ARG(h_lut[t] < c_cls, "seg_confusion: tag %d maps to class %d, outside 0..%d", t, h_lut[t], c_cls - 1);
  if (n == 0) return 0;
  LAVB_CHECK_ARG(d_feat && d_deconv && d_labels && d_out, "seg_confusion: null pointer");
  const size_t feat_align = feat_dtype == LAVB_F32 ? 16 : 8;
  LAVB_CHECK_ARG((uintptr_t)d_feat % feat_align == 0 && (uintptr_t)d_labels % 2 == 0 && (uintptr_t)d_deconv % 4 == 0 &&
                 (uintptr_t)d_out % 4 == 0, "seg_confusion: features must be %zu-byte and labels 2-byte aligned", feat_align);
  TagTable lut;
  memcpy(lut.cls, h_lut, 256);
  cudaStream_t st = (cudaStream_t)stream;
  LAVB_CUDA_OK(cudaMemsetAsync(d_out, 0, sizeof(int) * (size_t)n * (c_cls * c_cls + 1), st));
  const dim3 grid(lavb::ceil_div((long long)(h / 2) * (w / 2), kThreads), n);
  const DeconvW* dw = reinterpret_cast<const DeconvW*>(d_deconv);
  if (feat_dtype == LAVB_F32) launch<float>(c_cls, grid, st, d_feat, dw, d_labels, lut, h, w, d_out);
  else launch<lavb::h16>(c_cls, grid, st, d_feat, dw, d_labels, lut, h, w, d_out);
  LAVB_LAUNCH_OK();
  return 0;
}
