// Rotated bilinear window gather: F.affine_grid(theta, align_corners=True) + F.grid_sample(bilinear, zeros,
// align_corners=True) of UniPlanner.crop_feature (team_code_v2/models/uniplanner.py:303-340) as one kernel on the
// channels-last feature map.  Crop k reads frame frame_idx[k] directly (the reference's `features.expand(N,...)`
// view, without materialising it for batched frames).
#include "common.cuh"

namespace lavb {

// 16 B of channels per thread (4 fp32 / 8 h16): C*sizeof(T)/16 threads per output pixel, four 16 B loads + one 16 B store
// each — one warp per pixel left a third of the lanes idle at C = 384 and issued twice as many (8 B) loads.
template <typename T> struct Vec16;
template <> struct Vec16<float> {
  static constexpr int N = 4;
  static __device__ __forceinline__ void load(const float* p, float (&v)[4]) {
    const float4 r = __ldg(reinterpret_cast<const float4*>(p)); v[0] = r.x; v[1] = r.y; v[2] = r.z; v[3] = r.w;
  }
  static __device__ __forceinline__ void store(float* p, const float (&v)[4]) { *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]); }
};
template <> struct Vec16<h16> {
  static constexpr int N = 8;
  static __device__ __forceinline__ void load(const h16* p, float (&v)[8]) {
    const uint4 r = __ldg(reinterpret_cast<const uint4*>(p));
    const uint32_t u[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = h1622float2(*reinterpret_cast<const h162*>(&u[e]));
      v[2 * e] = f.x; v[2 * e + 1] = f.y;
    }
  }
  static __device__ __forceinline__ void store(h16* p, const float (&v)[8]) {
    uint32_t u[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const h162 h = floats2h162(v[2 * e], v[2 * e + 1]);
      u[e] = *reinterpret_cast<const uint32_t*>(&h);
    }
    *reinterpret_cast<uint4*>(p) = make_uint4(u[0], u[1], u[2], u[3]);
  }
};

// sample position (feature-map pixels) of crop pixel (i, j): F.affine_grid(align_corners=True) then grid_sample's un-normalisation.
// torch.linspace(-1, 1, S): start + step*idx for the first half, end - step*(S-1-idx) for the second
__device__ __forceinline__ void crop_sample_pos(int i, int j, int S, const float* __restrict__ th, int H, int W, float& ix, float& iy) {
  const float step = 2.f / (float)(S - 1);
  const float xb = (i < S / 2) ? (-1.f + step * (float)i) : (1.f - step * (float)(S - 1 - i));
  const float yb = (j < S / 2) ? (-1.f + step * (float)j) : (1.f - step * (float)(S - 1 - j));
  const float gx = fmaf(th[0], xb, fmaf(th[1], yb, th[2]));
  const float gy = fmaf(th[3], xb, fmaf(th[4], yb, th[5]));
  ix = (gx + 1.f) * 0.5f * (float)(W - 1);
  iy = (gy + 1.f) * 0.5f * (float)(H - 1);
}

// the four bilinear taps of sample position (ix, iy) on an H x W map, shared by both forward kernels so that they agree on
// every position.  x0 = floor(ix) through the saturating conversion (a position past +-2^31 or infinite gives INT_MAX / INT_MIN)
// and the on-map tests never form x0 + 1, so no int overflows.  A NaN coordinate reads pixel (0, 0) with its NaN weights, so
// every channel of the sample is NaN, whatever the other coordinate; a tap off the map is skipped (zero padding).
struct CropTaps {
  int x0, y0;
  float w00, w01, w10, w11;
  bool v00, v01, v10, v11;
};

__device__ __forceinline__ CropTaps crop_taps(float ix, float iy, int H, int W) {
  CropTaps t;
  const bool nan = isnan(ix) || isnan(iy);
  t.x0 = nan ? 0 : __float2int_rd(ix);
  t.y0 = nan ? 0 : __float2int_rd(iy);
  const float ax = ix - floorf(ix), ay = iy - floorf(iy);
  t.w00 = (1.f - ax) * (1.f - ay); t.w01 = ax * (1.f - ay); t.w10 = (1.f - ax) * ay; t.w11 = ax * ay;
  const bool vx0 = t.x0 >= 0 && t.x0 < W, vx1 = t.x0 >= -1 && t.x0 < W - 1;
  const bool vy0 = t.y0 >= 0 && t.y0 < H, vy1 = t.y0 >= -1 && t.y0 < H - 1;
  t.v00 = vx0 && vy0; t.v01 = vx1 && vy0; t.v10 = vx0 && vy1; t.v11 = vx1 && vy1;
  return t;
}

// block = one 8x8 patch of output pixels x one 64 B channel slice (4 threads of 16 B per pixel): neighbouring output
// pixels sample overlapping 2x2 input neighbourhoods, so a compact patch lets L1 serve the ~4x re-reads that a row-major
// pixel order sent to L2.  grid = (patches per crop, channel slices, crops).
template <typename T>
__global__ void __launch_bounds__(256) crop_kernel(const T* __restrict__ feat, int B, int H, int W, int C,
                                                   const int* __restrict__ frame_idx, const float* __restrict__ theta,
                                                   int K, int S, T* __restrict__ out) {
  constexpr int VEC = Vec16<T>::N;
  const int pw = (S + 7) >> 3;
  const int pj = blockIdx.x / pw, pi = blockIdx.x - pj * pw;
  const int k = blockIdx.z;
  const int j = pj * 8 + (threadIdx.x >> 5), i = pi * 8 + ((threadIdx.x >> 2) & 7);
  const int c = (blockIdx.y * 4 + (threadIdx.x & 3)) * VEC;
  if (i >= S || j >= S || c >= C) return;
  const long long pix = ((long long)k * S + j) * S + i;
  float th[6];
#pragma unroll
  for (int e = 0; e < 6; ++e) th[e] = __ldg(theta + k * 6 + e);
  float ix, iy;
  crop_sample_pos(i, j, S, th, H, W, ix, iy);
  const CropTaps tp = crop_taps(ix, iy, H, W);
  int b = __ldg(frame_idx + k);
  b = b < 0 ? 0 : (b >= B ? B - 1 : b);
  const T* p00 = feat + (long long)b * H * W * C + ((long long)tp.y0 * W + tp.x0) * C + c;
  float acc[VEC];
#pragma unroll
  for (int e = 0; e < VEC; ++e) acc[e] = 0.f;
  auto add = [&](const T* p, float wgt, bool ok) {
    if (!ok) return;
    float v[VEC];
    Vec16<T>::load(p, v);
#pragma unroll
    for (int e = 0; e < VEC; ++e) acc[e] = fmaf(wgt, v[e], acc[e]);
  };
  add(p00, tp.w00, tp.v00); add(p00 + C, tp.w01, tp.v01);
  add(p00 + (long long)W * C, tp.w10, tp.v10); add(p00 + (long long)W * C + C, tp.w11, tp.v11);
  Vec16<T>::store(out + pix * C + c, acc);
}

// ---------------------------------------------------------------------------------------------------------------------
// The same crop read straight from a uint8 PLANAR map (b, c, h, w) — the ground-truth BEV of the dataset and of bev_targets —
// into an fp32 NCHW crop (k, c, S, S), the layout F.grid_sample returns and the 9-channel embedder's conv1 consumes.  It replaces
// `bev.float()` + the per-crop gather + affine_grid + grid_sample of BEVPlanner's training forward.  HBM-write-bound (4 B per
// output element, the u8 taps are re-read from L1 / L2), so a thread owns one output pixel and walks the channels: its sample
// position and weights are computed once, and a warp stores 32 consecutive floats of one output row (128 B) per channel.
// block = 32 x 8 output pixels (rows overlap in L1); grid = (patches per crop, crops).  Per channel, the four taps accumulate
// in crop_kernel's order with its fmaf chain, so the result is bit-identical to crop_kernel<float> on the float copy of the map.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) crop_u8_kernel(const uint8_t* __restrict__ map, int B, int C, int H, int W,
                                                      const int* __restrict__ frame_idx, const float* __restrict__ theta,
                                                      int S, float* __restrict__ out) {
  const int pw = (S + 31) >> 5;
  const int pj = blockIdx.x / pw, pi = blockIdx.x - pj * pw;
  const int k = blockIdx.y;
  const int i = pi * 32 + (threadIdx.x & 31), j = pj * 8 + (threadIdx.x >> 5);
  if (i >= S || j >= S) return;
  float th[6];
#pragma unroll
  for (int e = 0; e < 6; ++e) th[e] = __ldg(theta + k * 6 + e);
  float ix, iy;
  crop_sample_pos(i, j, S, th, H, W, ix, iy);
  const CropTaps tp = crop_taps(ix, iy, H, W);
  int b = __ldg(frame_idx + k);
  b = b < 0 ? 0 : (b >= B ? B - 1 : b);
  const long long plane = (long long)H * W;
  // offset of tap 00 inside a plane; a tap is read only when it lies on the map
  const long long o00 = (long long)tp.y0 * W + tp.x0;
  const uint8_t* src = map + (long long)b * C * plane;
  float* dst = out + (long long)k * C * S * S + (long long)j * S + i;
  for (int c = 0; c < C; ++c, src += plane, dst += (long long)S * S) {
    float acc = 0.f;
    if (tp.v00) acc = fmaf(tp.w00, (float)__ldg(src + o00), acc);
    if (tp.v01) acc = fmaf(tp.w01, (float)__ldg(src + o00 + 1), acc);
    if (tp.v10) acc = fmaf(tp.w10, (float)__ldg(src + o00 + W), acc);
    if (tp.v11) acc = fmaf(tp.w11, (float)__ldg(src + o00 + W + 1), acc);
    *dst = acc;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Backward of the crop with respect to the feature map, as a GATHER (no atomics, every feature pixel written exactly once,
// zeros included, fixed summation order): cudnn's bilinear_sampler_bw scatters 4 atomics per crop pixel and channel.
//   gfeat[b, y, x, :] = sum over crops k of frame b, crop pixels (i, j) whose 2x2 footprint contains (x, y):  w * gout[k, j, i, :]
// The sample position is affine in (i, j); its inverse gives the (at most ~4x4) candidate crop pixels of a feature pixel, and
// each candidate's weight is then recomputed with the forward's own arithmetic, so forward and backward agree exactly on
// which corner a sample touches.  A crop whose sample position has no usable inverse (a map one pixel wide or high, a
// rank-deficient theta) takes every crop pixel as a candidate: correct, and slow only for inputs the planners never build.
// block = 8x8 feature pixels of one frame, one warp per patch row; the crops of the frame whose footprint meets the patch
// are listed once per block (in k order) in shared memory.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kBwdList = 32;                       // crops per pass of the shared-memory list
struct BwdCrop { float th[6]; float inv[4]; float c0, c1, pad; int k; };

__global__ void __launch_bounds__(256) crop_bwd_kernel(const float* __restrict__ gout, int B, int H, int W, int C,
                                                       const int* __restrict__ frame_idx, const float* __restrict__ theta,
                                                       int K, int S, float* __restrict__ gfeat) {
  __shared__ BwdCrop list[kBwdList];
  __shared__ int n_list, k_next;
  const int pw = (W + 7) >> 3;
  const int py = blockIdx.x / pw, px = blockIdx.x - py * pw;
  const int b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int y = py * 8 + warp;
  const int groups = C >> 2;                       // float4 groups per pixel
  const float sx = 0.5f * (float)(W - 1), sy = 0.5f * (float)(H - 1), step = 2.f / (float)(S - 1);
  for (int g0 = 0; g0 < groups; g0 += 96) {        // 3 float4 per lane per pass over the channels
    if (threadIdx.x == 0) k_next = 0;
    __syncthreads();
    for (int pass = 0;; ++pass) {
      // ---- warp 0 lists the next crops of frame b that can touch this patch, in k order
      if (warp == 0) {
        int n = 0, k0 = k_next;
        while (k0 < K && n < kBwdList) {
          const int k = k0 + lane;
          bool hit = false;
          float th[6];
          if (k < K) {
            int fb = __ldg(frame_idx + k);
            fb = fb < 0 ? 0 : (fb >= B ? B - 1 : fb);
            if (fb == b) {
#pragma unroll
              for (int e = 0; e < 6; ++e) th[e] = __ldg(theta + k * 6 + e);
              // footprint bounding box from the four corner samples (+1 pixel for the 2x2 support)
              float x0 = 1e30f, x1 = -1e30f, y0 = 1e30f, y1 = -1e30f;
#pragma unroll
              for (int cnr = 0; cnr < 4; ++cnr) {
                float ix, iy;
                crop_sample_pos((cnr & 1) ? S - 1 : 0, (cnr & 2) ? S - 1 : 0, S, th, H, W, ix, iy);
                x0 = fminf(x0, ix); x1 = fmaxf(x1, ix); y0 = fminf(y0, iy); y1 = fmaxf(y1, iy);
              }
              hit = x1 + 1.f >= (float)(px * 8) && x0 - 1.f <= (float)(px * 8 + 7) && y1 + 1.f >= (float)(py * 8) && y0 - 1.f <= (float)(py * 8 + 7);
            }
          }
          const unsigned m = __ballot_sync(0xffffffffu, hit);
          const int pos = n + __popc(m & ((1u << lane) - 1u));
          if (hit && pos < kBwdList) {
            BwdCrop& c = list[pos];
#pragma unroll
            for (int e = 0; e < 6; ++e) c.th[e] = th[e];
            const float a00 = sx * th[0] * step, a01 = sx * th[1] * step, a10 = sy * th[3] * step, a11 = sy * th[4] * step;
            const float det = a00 * a11 - a01 * a10, r = det != 0.f ? 1.f / det : 0.f;
            c.inv[0] = a11 * r; c.inv[1] = -a01 * r; c.inv[2] = -a10 * r; c.inv[3] = a00 * r;
            c.c0 = sx * (th[2] + 1.f - th[0] - th[1]); c.c1 = sy * (th[5] + 1.f - th[3] - th[4]);
            c.k = k;
            c.pad = 1e-3f;                         // margin of the candidate window around the inverse image
            // det 0 (sx or sy is 0 on a one-pixel map), lost to cancellation (rank-1 theta) or not finite: no inverse, so
            // the window is centred on crop pixel 0 with a margin of S, i.e. the whole crop
            const bool finite = isfinite(c.inv[0]) && isfinite(c.inv[1]) && isfinite(c.inv[2]) && isfinite(c.inv[3]);
            if (!(fabsf(det) > 1e-5f * (fabsf(a00 * a11) + fabsf(a01 * a10))) || !finite) {
              c.inv[0] = c.inv[1] = c.inv[2] = c.inv[3] = 0.f;
              c.c0 = c.c1 = 0.f;
              c.pad = (float)S;
            }
          }
          const int total = n + __popc(m);
          if (total > kBwdList) {                  // list full inside this chunk: resume at the first crop that did not fit
            unsigned mm = m; int fit = kBwdList - n;
            while (fit-- > 0) mm &= mm - 1;        // drop the crops that fitted
            k0 = k0 + __ffs(mm) - 1; n = kBwdList;
          } else { n = total; k0 += 32; }
        }
        if (lane == 0) { n_list = n; k_next = k0; }
      }
      __syncthreads();
      const int n = n_list;
      const bool more = k_next < K;
      if (y < H) {
        for (int q = 0; q < 8; ++q) {
          const int x = px * 8 + q;
          if (x >= W) break;
          float4* op = reinterpret_cast<float4*>(gfeat + (((long long)b * H + y) * W + x) * C) + g0;
          float4 acc[3];
#pragma unroll
          for (int t = 0; t < 3; ++t)              // a later pass (> kBwdList crops on this patch) continues the running sum
            acc[t] = (pass > 0 && g0 + lane + 32 * t < groups) ? op[lane + 32 * t] : make_float4(0.f, 0.f, 0.f, 0.f);
          for (int ci = 0; ci < n; ++ci) {
            const BwdCrop& c = list[ci];
            const float dx = (float)x - c.c0, dy = (float)y - c.c1;
            const float is = c.inv[0] * dx + c.inv[1] * dy, js = c.inv[2] * dx + c.inv[3] * dy;
            const float ri = fabsf(c.inv[0]) + fabsf(c.inv[1]) + c.pad, rj = fabsf(c.inv[2]) + fabsf(c.inv[3]) + c.pad;
            const int i_lo = max(0, (int)ceilf(is - ri)), i_hi = min(S - 1, (int)floorf(is + ri));
            const int j_lo = max(0, (int)ceilf(js - rj)), j_hi = min(S - 1, (int)floorf(js + rj));
            const int ni = i_hi - i_lo + 1, nj = j_hi - j_lo + 1;
            if (ni <= 0 || nj <= 0) continue;
            const int ncand = ni * nj;
            for (int cb = 0; cb < ncand; cb += 32) {
              const int cnd = cb + lane;
              float wgt = 0.f; int ii = 0, jj = 0;
              if (cnd < ncand) {
                jj = j_lo + cnd / ni; ii = i_lo + cnd - (cnd / ni) * ni;
                float ix, iy;
                crop_sample_pos(ii, jj, S, c.th, H, W, ix, iy);
                const float fx = floorf(ix), fy = floorf(iy);
                const int x0 = (int)fx, y0 = (int)fy;
                const float ax = ix - fx, ay = iy - fy;
                const float wx = x0 == x ? 1.f - ax : (x0 + 1 == x ? ax : 0.f);
                const float wy = y0 == y ? 1.f - ay : (y0 + 1 == y ? ay : 0.f);
                wgt = wx * wy;
              }
              unsigned m = __ballot_sync(0xffffffffu, wgt != 0.f);
              while (m) {
                const int src = __ffs(m) - 1; m &= m - 1;
                const float w_ = __shfl_sync(0xffffffffu, wgt, src);
                const int i_ = __shfl_sync(0xffffffffu, ii, src), j_ = __shfl_sync(0xffffffffu, jj, src);
                const float4* gp = reinterpret_cast<const float4*>(gout + (((long long)c.k * S + j_) * S + i_) * C) + g0;
#pragma unroll
                for (int t = 0; t < 3; ++t) {
                  const int g = lane + 32 * t;
                  if (g0 + g < groups) {
                    const float4 v = __ldg(gp + g);
                    acc[t].x = fmaf(w_, v.x, acc[t].x); acc[t].y = fmaf(w_, v.y, acc[t].y);
                    acc[t].z = fmaf(w_, v.z, acc[t].z); acc[t].w = fmaf(w_, v.w, acc[t].w);
                  }
                }
              }
            }
          }
#pragma unroll
          for (int t = 0; t < 3; ++t)
            if (g0 + lane + 32 * t < groups) op[lane + 32 * t] = acc[t];
        }
      }
      __syncthreads();
      if (!more) break;
    }
  }
}

}  // namespace lavb

using namespace lavb;

extern "C" int lavb_crop_bilinear(const void* d_feat, int dtype, int b, int h, int w, int c, const int* d_frame_idx,
                                  const float* d_theta, int k, int crop, void* d_out, void* stream) {
  LAVB_CHECK_ARG(dtype == LAVB_F32 || dtype == LAVB_H16, "crop_bilinear: bad dtype %d", dtype);
  const int vec = dtype == LAVB_F32 ? 4 : 8;       // channels per 16-byte vector
  LAVB_CHECK_ARG(c >= vec && c % vec == 0, "crop_bilinear: channels must be a positive multiple of %d (got %d)", vec, c);
  LAVB_CHECK_ARG(crop >= 2 && crop <= 65535 && b >= 1 && h >= 1 && w >= 1, "crop_bilinear: bad crop size / map (%d; %d x %d x %d)", crop,
                 b, h, w);
  LAVB_CHECK_ARG(k >= 0, "crop_bilinear: negative crop count");
  if (k == 0) return 0;
  LAVB_CHECK_ARG(k <= 65535, "crop_bilinear: at most 65535 crops per call");
  LAVB_CHECK_ARG((uintptr_t)d_feat % 16 == 0 && (uintptr_t)d_out % 16 == 0, "crop_bilinear: feat and out must be 16-byte aligned");
  const int pw = (crop + 7) / 8;
  const dim3 blocks(pw * pw, ceil_div(c, 4 * vec), k);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == LAVB_F32)
    crop_kernel<float><<<blocks, 256, 0, st>>>((const float*)d_feat, b, h, w, c, d_frame_idx, d_theta, k, crop, (float*)d_out);
  else
    crop_kernel<h16><<<blocks, 256, 0, st>>>((const h16*)d_feat, b, h, w, c, d_frame_idx, d_theta, k, crop,
                                                           (h16*)d_out);
  LAVB_LAUNCH_OK();
  return 0;
}

// uint8 planar (b, c, h, w) map -> fp32 NCHW crops (k, c, crop, crop); frame indices are clamped to [0, b-1] as in
// lavb_crop_bilinear.  Every output element is written (zeros where the sample falls off the map).
extern "C" int lavb_crop_bilinear_u8(const uint8_t* d_map, int b, int c, int h, int w, const int* d_frame_idx, const float* d_theta,
                                     int k, int crop, float* d_out, void* stream) {
  LAVB_CHECK_ARG(c >= 1, "crop_bilinear_u8: need at least one channel (got %d)", c);
  LAVB_CHECK_ARG(crop >= 2 && crop <= 65535, "crop_bilinear_u8: crop size must be in [2, 65535] (got %d)", crop);
  LAVB_CHECK_ARG(b >= 1 && h >= 1 && w >= 1, "crop_bilinear_u8: empty map (%d x %d x %d)", b, h, w);
  LAVB_CHECK_ARG(k >= 0, "crop_bilinear_u8: negative crop count");
  if (k == 0) return 0;
  LAVB_CHECK_ARG(k <= 65535, "crop_bilinear_u8: at most 65535 crops per call");
  LAVB_CHECK_ARG(d_map && d_frame_idx && d_theta && d_out, "crop_bilinear_u8: null pointer");
  LAVB_CHECK_ARG(is_aligned(d_frame_idx, 4) && is_aligned(d_theta, 4) && is_aligned(d_out, 4),
                 "crop_bilinear_u8: frame_idx, theta and out must be 4-byte aligned");
  const size_t out_bytes = (size_t)k * c * crop * crop * sizeof(float);
  LAVB_CHECK_ARG(!ranges_overlap(d_out, out_bytes, d_map, (size_t)b * c * h * w) &&
                     !ranges_overlap(d_out, out_bytes, d_frame_idx, (size_t)k * sizeof(int)) &&
                     !ranges_overlap(d_out, out_bytes, d_theta, (size_t)k * 6 * sizeof(float)),
                 "crop_bilinear_u8: out overlaps map, frame_idx or theta");
  const dim3 blocks(((crop + 31) / 32) * ((crop + 7) / 8), k);
  crop_u8_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(d_map, b, c, h, w, d_frame_idx, d_theta, crop, d_out);
  LAVB_LAUNCH_OK();
  return 0;
}

// d(loss)/d(feat) of lavb_crop_bilinear for fp32 NHWC tensors: d_gout (k, crop, crop, c) -> d_gfeat (b, h, w, c), every element
// written (zeros where no crop samples, every frame when k = 0).  Replaces cudnn_grid_sampler_backward + the index_put of
// `features[frame]` in the training forward of UniPlanner (lav/models/uniplanner.py:56-151).
extern "C" int lavb_crop_bilinear_bwd(const float* d_gout, int b, int h, int w, int c, const int* d_frame_idx, const float* d_theta,
                                      int k, int crop, float* d_gfeat, void* stream) {
  LAVB_CHECK_ARG(c >= 4 && c % 4 == 0, "crop_bilinear_bwd: channels must be a positive multiple of 4 (got %d)", c);
  LAVB_CHECK_ARG(crop >= 2 && b >= 1 && b <= 65535 && h >= 1 && w >= 1, "crop_bilinear_bwd: bad crop size / map (%d; %d x %d x %d)",
                 crop, b, h, w);
  LAVB_CHECK_ARG(k >= 0, "crop_bilinear_bwd: negative crop count");
  LAVB_CHECK_ARG((uintptr_t)d_gout % 16 == 0 && (uintptr_t)d_gfeat % 16 == 0, "crop_bilinear_bwd: gout and gfeat must be 16-byte aligned");
  const dim3 blocks(((w + 7) / 8) * ((h + 7) / 8), b);
  crop_bwd_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(d_gout, b, h, w, c, d_frame_idx, d_theta, k, crop, d_gfeat);
  LAVB_LAUNCH_OK();
  return 0;
}
