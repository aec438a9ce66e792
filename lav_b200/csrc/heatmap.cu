// Detection targets of a training batch in one launch: the heat, size and orientation maps of LiDARDataset.detections_to_heatmap
// (lidar_dataset.py:92-127) for every sample, restating data_pipeline.detections_to_heatmap (the same computation in torch ops)
// operation for operation so that the maps are bit-identical to it.
#include "det_grid.cuh"

namespace {

using lavb::DetActor;
using lavb::DetGrid;

// torch's arg-max over a reduced dimension (GreaterOrNan in ATen's SharedReduceOps.h): a NaN beats everything, the larger value
// wins, and a tie keeps the lower index.  Actors are visited in index order, so "take" means strictly better.
__device__ __forceinline__ bool better(float best, float v) { return !isnan(best) && (isnan(v) || v > best); }

// gx * gy of one actor at pixel (px, py): the centre as lavb::det_centre, then torch's (p - c) / radius as (p - c) * (1 / radius),
// ** 2 as d * d, then exp of the negation, then the product of the two separable factors.  The _rn intrinsics keep nvcc from
// contracting any of it into an FMA.
__device__ __forceinline__ float gauss(const DetActor& a, const DetGrid& g, float px, float py) {
  const float2 c = lavb::det_centre(a, g);
  const float cx = c.x, cy = c.y;
  const float dx = __fmul_rn(__fsub_rn(px, cx), g.inv_r), dy = __fmul_rn(__fsub_rn(py, cy), g.inv_r);
  return __fmul_rn(expf(-__fmul_rn(dx, dx)), expf(-__fmul_rn(dy, dy)));
}

// One thread per output pixel of one sample (blockIdx.y); it walks the sample's actors once and keeps the best of each class.
__global__ void __launch_bounds__(256) det_heatmaps_kernel(const DetActor* __restrict__ actors, const int* __restrict__ offsets,
                                                           int h, int w, const DetGrid g, float* __restrict__ heat,
                                                           float* __restrict__ size, float* __restrict__ orim) {
  const int pix = blockIdx.x * 256 + threadIdx.x;
  if (pix >= h * w) return;
  const int b = blockIdx.y;
  const float px = (float)(pix % w), py = (float)(pix / w);
  const int a0 = __ldg(offsets + b), a1 = __ldg(offsets + b + 1);
  float g0 = 0.f, g1 = 0.f;
  int who0 = -1, who1 = -1;
  for (int a = a0; a < a1; ++a) {
    const DetActor A = actors[a];
    if (A.typ == 0.f) {
      const float v = gauss(A, g, px, py);
      if (who0 < 0 || better(g0, v)) { g0 = v; who0 = a; }
    } else if (A.typ == 1.f) {
      const float v = gauss(A, g, px, py);
      if (who1 < 0 || better(g1, v)) { g1 = v; who1 = a; }
    }
  }
  // class 0: mask = g0 > max(zeros) = g0 > 0.  class 1: mask = g1 > max over classes of the heat so far, which is g0 (>= 0, or
  // NaN, which torch's max propagates and which fails every >) when class 0 had actors, else 0.  A class without actors leaves
  // its planes untouched; class 1 overwrites class 0's size and orientation where its mask holds.
  int sel = -1;
  if (who0 >= 0 && g0 > 0.f) sel = who0;
  if (who1 >= 0 && g1 > (who0 >= 0 ? g0 : 0.f)) sel = who1;
  float s0 = 0.f, s1 = 0.f, o0 = 0.f, o1 = 0.f;
  if (sel >= 0) {
    const DetActor A = actors[sel];
    s0 = __fmul_rn(A.bx, g.ppm);
    s1 = __fmul_rn(A.by, g.ppm);
    o0 = cosf(A.ori);
    o1 = sinf(A.ori);
  }
  const size_t plane = (size_t)h * w, base = (size_t)b * 2 * plane + pix;
  heat[base] = who0 >= 0 ? g0 : 0.f;
  heat[base + plane] = who1 >= 0 ? g1 : 0.f;
  size[base] = s0;
  size[base + plane] = s1;
  orim[base] = o0;
  orim[base + plane] = o1;
}

}  // namespace

extern "C" int lavb_det_heatmaps(const void* d_actors, const int* d_offsets, int b, int h, int w, float ppm, float cx0, float cy0,
                                 float cy1, float inv_radius, float* d_heat, float* d_size, float* d_ori, void* stream) {
  LAVB_CHECK_ARG(b >= 0 && b <= 65535 && h > 0 && w > 0 && (long long)h * w <= 0x7fffffffLL,
                 "det_heatmaps: bad sizes (b %d, %d x %d)", b, h, w);
  LAVB_CHECK_ARG(b == 0 || (d_offsets != nullptr && d_heat != nullptr && d_size != nullptr && d_ori != nullptr),
                 "det_heatmaps: null offsets or output");
  if (b == 0) return 0;
  const DetGrid g{ppm, cx0, cy0, cy1, inv_radius};
  det_heatmaps_kernel<<<dim3(lavb::ceil_div((long long)h * w, 256), b), 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const DetActor*>(d_actors), d_offsets, h, w, g, d_heat, d_size, d_ori);
  LAVB_LAUNCH_OK();
  return 0;
}
