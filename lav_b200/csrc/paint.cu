// Point painting, sweep stacking and small ingest kernels (HBM-bound, one thread per point / element).
//
// paint: restates CoordConverter.forward + InferModel.point_painting
// (team_code_v2/model_inference.py:75-93,280-297) as ONE kernel: 3 camera projections in the
// reference's fp32 operation order (k-sequential FMA chains, IEEE division, truncation toward
// zero, bounds test on the truncated integers, later camera wins: project_hit.cuh), then one gather.
#include "common.cuh"
#include "deconv_logits.cuh"
#include "project_hit.cuh"

namespace lavb {

template <int MODE>
__global__ void __launch_bounds__(256) paint_kernel(const float* __restrict__ pts, int n, int pt_stride,
                                                    const float* __restrict__ sem, int c_in, int H, int W,
                                                    long long s_cam, long long s_c, long long s_y, long long s_x,
                                                    const __grid_constant__ CamSet cams, float* __restrict__ out,
                                                    int out_stride, int out_col0, int copy_cols,
                                                    long long pts_frame_stride, long long sem_frame_stride,
                                                    long long out_frame_stride, int vec_in, int vec_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  // blockIdx.y = frame of a batch of independent agents (each with its own sweep and semantic maps)
  pts += blockIdx.y * pts_frame_stride;
  sem += blockIdx.y * sem_frame_stride;
  out += blockIdx.y * out_frame_stride;
  const float* p = pts + (size_t)i * pt_stride;
  float x, y, z;
  float4 p4;
  if (vec_in) {
    p4 = __ldg(reinterpret_cast<const float4*>(p));
    x = p4.x; y = p4.y; z = p4.z;
  } else {
    x = __ldg(p); y = __ldg(p + 1); z = __ldg(p + 2);
  }
  int hit_u = 0, hit_v = 0;
  const int hit_cam = project_hit(cams, x, y, z, H, W, hit_u, hit_v);
  float* o = out + (size_t)i * out_stride;
  if (vec_out) {
    *reinterpret_cast<float4*>(o) = p4;
  } else {
    for (int k = 0; k < copy_cols; ++k) o[k] = __ldg(p + k);
  }
  const int c_out = (MODE == 0) ? c_in : c_in - 1;
  o += out_col0;
  if (hit_cam < 0) {
    for (int k = 0; k < c_out; ++k) o[k] = 0.f;
    return;
  }
  const float* s = sem + hit_cam * s_cam + hit_v * s_y + hit_u * s_x;
  if (MODE == 0) {
    for (int k = 0; k < c_out; ++k) o[k] = __ldg(s + k * s_c);
  } else {
    float pr[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) pr[k] = (k < c_in) ? __ldg(s + k * s_c) : 0.f;
    if (MODE == 2) {  // softmax over c_in logits (torch.softmax: exp(x-max)/sum)
      float mx = pr[0];
#pragma unroll
      for (int k = 1; k < 8; ++k) if (k < c_in) mx = fmaxf(mx, pr[k]);
      float sum = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) if (k < c_in) { pr[k] = expf(pr[k] - mx); sum += pr[k]; }
#pragma unroll
      for (int k = 0; k < 8; ++k) if (k < c_in) pr[k] = __fdiv_rn(pr[k], sum);
    }
    const float bg = __fsub_rn(1.f, pr[0]);  // pred_sem[:,1:] * (1 - pred_sem[:,:1]), model_inference.py:45
#pragma unroll
    for (int k = 1; k < 8; ++k) if (k < c_in) o[k - 1] = __fmul_rn(pr[k], bg);
  }
}

struct StackParams { float R[9]; float dx, dy; };

// [x y z] @ R (row vector times the row-major 3x3 R, k-sequential _rn FMAs), then x += dx, y += dy: lav_agent_fast.py:555-563.
// The adds are real fp32 adds even when dx = dy = 0 (-0 + 0 = +0), as in the reference's rotate-then-translate.
__device__ __forceinline__ void move_point(const float* R, float dx, float dy, float x, float y, float z, float& nx, float& ny,
                                           float& nz) {
  nx = __fadd_rn(__fmaf_rn(z, R[6], __fmaf_rn(y, R[3], __fmul_rn(x, R[0]))), dx);
  ny = __fadd_rn(__fmaf_rn(z, R[7], __fmaf_rn(y, R[4], __fmul_rn(x, R[1]))), dy);
  nz = __fmaf_rn(z, R[8], __fmaf_rn(y, R[5], __fmul_rn(x, R[2])));
}

__global__ void __launch_bounds__(256) stack_kernel(const float* __restrict__ src, int n, int src_cols,
                                                    const __grid_constant__ StackParams P, int time_idx, int n_time,
                                                    int roof_filter, float* __restrict__ dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* s = src + (size_t)i * src_cols;
  const int dcols = src_cols + n_time;
  float* d = dst + (size_t)i * dcols;
  const float x = __ldg(s), y = __ldg(s + 1), z = __ldg(s + 2);
  float nx, ny, nz;
  move_point(P.R, P.dx, P.dy, x, y, z, nx, ny, nz);
  if (roof_filter) {  // LAVAgent.preprocess, lav_agent.py:450 — on the sensor-frame coordinates
    if (x > -2.4f && x < 0.f && y > -0.8f && y < 0.8f && z > -1.5f && z < -1.f) nx = __int_as_float(0x7fc00000);
  }
  d[0] = nx; d[1] = ny; d[2] = nz;
  for (int k = 3; k < src_cols; ++k) d[k] = __ldg(s + k);
  for (int k = 0; k < n_time; ++k) d[src_cols + k] = (k == time_idx) ? 1.f : 0.f;
}

template <typename TOut>
__global__ void __launch_bounds__(256) rgb_norm_kernel(const void* __restrict__ rgb, int src_u8_nhwc, int n, int h, int w,
                                                       TOut* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // pixel index
  const long long npix = (long long)n * h * w;
  if (i >= npix) return;
  float r, g, b;
  if (src_u8_nhwc) {
    const unsigned char* p = reinterpret_cast<const unsigned char*>(rgb) + i * 3;
    r = p[0]; g = p[1]; b = p[2];
  } else {
    const long long hw = (long long)h * w;
    const long long img = i / hw, pix = i - img * hw;
    const float* p = reinterpret_cast<const float*>(rgb) + img * 3 * hw + pix;
    r = __ldg(p); g = __ldg(p + hw); b = __ldg(p + 2 * hw);
  }
  // (x/255. - .5)*2 , rgb.py:41 — same three fp32 roundings
  float4 v;
  v.x = __fmul_rn(__fsub_rn(__fdiv_rn(r, 255.f), .5f), 2.f);
  v.y = __fmul_rn(__fsub_rn(__fdiv_rn(g, 255.f), .5f), 2.f);
  v.z = __fmul_rn(__fsub_rn(__fdiv_rn(b, 255.f), .5f), 2.f);
  v.w = 0.f;
  store4<TOut>(out + i * 4, v);
}

template <typename TS, typename TD>
__global__ void __launch_bounds__(256) convert_kernel(const TS* __restrict__ s, TD* __restrict__ d, long long count, int vec) {
  long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  const long long end = i + 4 < count ? i + 4 : count;
  if (vec && end == i + 4) {
    store4<TD>(d + i, load4<TS>(s + i));
  } else {
    for (; i < end; ++i) d[i] = from_f32<TD>(to_f32<TS>(s[i]));
  }
}

}  // namespace lavb

using namespace lavb;

// The float4 paths of the painting kernels, decided here from the pointers and strides: a point row is loaded as one float4
// when every frame's rows are 4 floats and 16-byte aligned; its 4 copied columns are stored as one float4 when, in addition,
// every output row is 16-byte aligned and the painted channels start past them.  Any other layout takes the per-element path.
static void paint_vec(const float* d_pts, int pt_stride, long long pts_fs, const float* d_out, int out_stride, long long out_fs,
                      int out_col0, int copy_cols, int frames, int& vec_in, int& vec_out) {
  vec_in = pt_stride == 4 && is_aligned(d_pts, 16) && (frames <= 1 || pts_fs % 4 == 0);
  vec_out = vec_in && copy_cols == 4 && out_col0 >= 4 && out_stride % 4 == 0 && is_aligned(d_out, 16) &&
            (frames <= 1 || out_fs % 4 == 0);
}

static int paint_impl(const float* d_pts, int n, int pt_stride, const float* d_sem, int ncam, int c_in, int h, int w,
                      long long s_cam, long long s_c, long long s_y, long long s_x, const float* h_cams, int mode,
                      float* d_out, int out_stride, int out_col0, int copy_cols, int frames, long long pts_fs, long long sem_fs,
                      long long out_fs, void* stream) {
  LAVB_CHECK_ARG(n >= 0 && pt_stride >= 3, "paint: bad n/pt_stride");
  LAVB_CHECK_ARG(ncam >= 1 && ncam <= 4, "paint: ncam must be 1..4 (got %d)", ncam);
  LAVB_CHECK_ARG(mode >= 0 && mode <= 2, "paint: mode must be 0..2");
  LAVB_CHECK_ARG(c_in >= (mode ? 2 : 1) && c_in <= 8, "paint: c_in out of range (got %d)", c_in);
  const int c_out = mode ? c_in - 1 : c_in;
  LAVB_CHECK_ARG(copy_cols >= 0 && copy_cols <= pt_stride && out_col0 >= copy_cols && out_col0 + c_out <= out_stride,
                 "paint: output row layout inconsistent");
  if (n == 0 || frames == 0) return 0;
  LAVB_CHECK_ARG(d_pts && d_sem && d_out && h_cams, "paint: null pointer");
  LAVB_CHECK_ARG(is_aligned(d_pts, 4) && is_aligned(d_sem, 4) && is_aligned(d_out, 4), "paint: d_pts, d_sem and d_out must be 4-byte aligned");
  CamSet cs;
  memcpy(cs.m, h_cams, sizeof(float) * 41 * ncam);
  cs.ncam = ncam;
  int vec_in, vec_out;
  paint_vec(d_pts, pt_stride, pts_fs, d_out, out_stride, out_fs, out_col0, copy_cols, frames, vec_in, vec_out);
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 blocks(ceil_div(n, 256), frames);
#define LAUNCH(M) paint_kernel<M><<<blocks, 256, 0, st>>>(d_pts, n, pt_stride, d_sem, c_in, h, w, s_cam, s_c, s_y, s_x, cs, \
                                                           d_out, out_stride, out_col0, copy_cols, pts_fs, sem_fs, out_fs, vec_in, vec_out)
  if (mode == 0) LAUNCH(0); else if (mode == 1) LAUNCH(1); else LAUNCH(2);
#undef LAUNCH
  LAVB_LAUNCH_OK();
  return 0;
}

extern "C" int lavb_paint(const float* d_pts, int n, int pt_stride, const float* d_sem, int ncam, int c_in, int h, int w,
                          long long s_cam, long long s_c, long long s_y, long long s_x, const float* h_cams, int mode,
                          float* d_out, int out_stride, int out_col0, int copy_cols, void* stream) {
  return paint_impl(d_pts, n, pt_stride, d_sem, ncam, c_in, h, w, s_cam, s_c, s_y, s_x, h_cams, mode, d_out, out_stride, out_col0,
                    copy_cols, 1, 0, 0, 0, stream);
}

extern "C" int lavb_paint_batched(const float* d_pts, int frames, int n, int pt_stride, long long pts_frame_stride,
                                  const float* d_sem, int ncam, int c_in, int h, int w, long long s_frame, long long s_cam,
                                  long long s_c, long long s_y, long long s_x, const float* h_cams, int mode, float* d_out,
                                  int out_stride, long long out_frame_stride, int out_col0, int copy_cols, void* stream) {
  LAVB_CHECK_ARG(frames >= 0 && frames <= 65535, "paint_batched: frames out of range");
  return paint_impl(d_pts, n, pt_stride, d_sem, ncam, c_in, h, w, s_cam, s_c, s_y, s_x, h_cams, mode, d_out, out_stride, out_col0,
                    copy_cols, frames, pts_frame_stride, s_frame, out_frame_stride, stream);
}

// ---- painting straight from the ERFNet decoder's last feature map ------------------------------------------------------------
// The frame path consumes the segmentation logits ONLY through the point-painting gather (<= 120 k samples of 221 k pixels per
// frame).  So the last ERFNet layer — output_conv = ConvTranspose2d(16, C, 2, stride 2) (lav/models/erfnet.py:122-124,132) — is
// evaluated inside the gather, for the hit pixel only: logits[k](v,u) = bias[k] + sum_c feat[v/2, u/2, c] * W[c][k][v%2][u%2],
// followed by softmax and the background suppression of model_inference.py:45.  The (H x W x C) fp32 logit maps (141 MB per 32
// frames) are never written, and the four launches of the transposed conv disappear.  The logits are deconv_logits.cuh's.

template <typename TF>
__global__ void __launch_bounds__(256) paint_deconv_kernel(const float* __restrict__ pts, int n, int pt_stride,
                                                           const TF* __restrict__ feat, int c_cls, int H, int W,
                                                           const __grid_constant__ CamSet cams, const DeconvW* __restrict__ dw,
                                                           float* __restrict__ out, int out_stride, int out_col0, int copy_cols,
                                                           long long pts_frame_stride, long long out_frame_stride, int vec_in,
                                                           int vec_out) {
  __shared__ DeconvW sw;
  for (int i = threadIdx.x; i < (int)(sizeof(DeconvW) / 4); i += blockDim.x) reinterpret_cast<float*>(&sw)[i] = __ldg(reinterpret_cast<const float*>(dw) + i);
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  pts += blockIdx.y * pts_frame_stride;
  out += blockIdx.y * out_frame_stride;
  const float* p = pts + (size_t)i * pt_stride;
  float x, y, z;
  float4 p4;
  if (vec_in) { p4 = __ldg(reinterpret_cast<const float4*>(p)); x = p4.x; y = p4.y; z = p4.z; }
  else { x = __ldg(p); y = __ldg(p + 1); z = __ldg(p + 2); }
  int hit_u = 0, hit_v = 0;
  const int hit_cam = project_hit(cams, x, y, z, H, W, hit_u, hit_v);
  float* o = out + (size_t)i * out_stride;
  if (vec_out) *reinterpret_cast<float4*>(o) = p4;
  else for (int k = 0; k < copy_cols; ++k) o[k] = __ldg(p + k);
  o += out_col0;
  if (hit_cam < 0) {
    for (int k = 0; k < c_cls - 1; ++k) o[k] = 0.f;
    return;
  }
  const int hh = H >> 1, wh = W >> 1;
  const TF* f = feat + ((((long long)blockIdx.y * cams.ncam + hit_cam) * hh + (hit_v >> 1)) * wh + (hit_u >> 1)) * 16;
  float fv[16];
  load_feat16<TF>(f, fv);
  float pr[8];
  deconv_logits<8>(sw, fv, hit_v & 1, hit_u & 1, pr);
  softmax_suppress(pr, c_cls, o);
}

extern "C" int lavb_paint_deconv_batched(const float* d_pts, int frames, int n, int pt_stride, long long pts_frame_stride,
                                         const void* d_feat, int feat_dtype, int ncam, int c_cls, int h, int w,
                                         const float* d_deconv, const float* h_cams, float* d_out, int out_stride,
                                         long long out_frame_stride, int out_col0, int copy_cols, void* stream) {
  LAVB_CHECK_ARG(frames >= 0 && frames <= 65535 && n >= 0 && pt_stride >= 3, "paint_deconv: bad sizes");
  LAVB_CHECK_ARG(ncam >= 1 && ncam <= 4 && c_cls >= 2 && c_cls <= 8, "paint_deconv: ncam 1..4, classes 2..8");
  LAVB_CHECK_ARG(h % 2 == 0 && w % 2 == 0, "paint_deconv: image size must be even (the feature map is h/2 x w/2)");
  LAVB_CHECK_ARG(copy_cols >= 0 && copy_cols <= pt_stride && out_col0 >= copy_cols && out_col0 + c_cls - 1 <= out_stride,
                 "paint_deconv: output row layout inconsistent");
  LAVB_CHECK_ARG(feat_dtype == LAVB_F32 || feat_dtype == LAVB_H16, "paint_deconv: feature dtype must be fp32 or h16");
  if (n == 0 || frames == 0) return 0;
  LAVB_CHECK_ARG(d_pts && d_feat && d_deconv && h_cams && d_out, "paint_deconv: null pointer");
  LAVB_CHECK_ARG(is_aligned(d_pts, 4) && is_aligned(d_deconv, 4) && is_aligned(d_out, 4) &&
                     is_aligned(d_feat, feat_dtype == LAVB_F32 ? 16 : 8),
                 "paint_deconv: d_feat must be 16-byte (fp32) / 8-byte (h16) aligned, d_pts, d_deconv and d_out 4-byte aligned");
  CamSet cs;
  memcpy(cs.m, h_cams, sizeof(float) * 41 * ncam);
  cs.ncam = ncam;
  int vec_in, vec_out;
  paint_vec(d_pts, pt_stride, pts_frame_stride, d_out, out_stride, out_frame_stride, out_col0, copy_cols, frames, vec_in, vec_out);
  const dim3 blocks(ceil_div(n, 256), frames);
  cudaStream_t st = (cudaStream_t)stream;
  const DeconvW* dw = reinterpret_cast<const DeconvW*>(d_deconv);
  if (feat_dtype == LAVB_F32)
    paint_deconv_kernel<float><<<blocks, 256, 0, st>>>(d_pts, n, pt_stride, (const float*)d_feat, c_cls, h, w, cs, dw, d_out, out_stride,
                                                       out_col0, copy_cols, pts_frame_stride, out_frame_stride, vec_in, vec_out);
  else
    paint_deconv_kernel<h16><<<blocks, 256, 0, st>>>(d_pts, n, pt_stride, (const h16*)d_feat, c_cls, h, w, cs, dw, d_out, out_stride,
                                                     out_col0, copy_cols, pts_frame_stride, out_frame_stride, vec_in, vec_out);
  LAVB_LAUNCH_OK();
  return 0;
}

// ---- table-driven sweep stacking: every (frame, sweep) job of a batch in one launch; the job table lives in DEVICE
// memory so a captured CUDA graph replays with new poses / ring-buffer slots after a small H2D table update.
struct StackJob {            // 72 bytes
  const float* src; float* dst; int n; int time_idx; float R[9]; float dx, dy; int pad;
};
static_assert(sizeof(StackJob) == 72, "StackJob layout is part of the ABI (lav_b200.h)");

// Rows are 8 floats in, 8 + n_time (= 11) floats out: a thread-per-row store pattern scatters every store instruction over 32
// rows (44-byte stride, 11x the sector transactions).  The block therefore builds its 256 output rows in shared memory and copies
// them out as one contiguous, fully coalesced run.
constexpr int kStackMaxCols = 16;
__global__ void __launch_bounds__(256) stack_jobs_kernel(const StackJob* __restrict__ jobs, int src_cols, int n_time,
                                                         int roof_filter) {
  __shared__ float rows[256 * kStackMaxCols];
  const StackJob j = jobs[blockIdx.y];
  // the table is rewritten between graph replays without the host seeing it, so the vector path is chosen here, per job (one
  // branch, uniform across the block)
  const bool src16 = (reinterpret_cast<uintptr_t>(j.src) & 15) == 0;
  const int dcols = src_cols + n_time;
  for (int i0 = blockIdx.x * 256; i0 < j.n; i0 += gridDim.x * 256) {
    const int i = i0 + threadIdx.x;
    if (i < j.n) {
      const float* s = j.src + (size_t)i * src_cols;
      float* d = rows + threadIdx.x * dcols;
      float x, y, z;
      if (src_cols == 8 && src16) {   // fused sweeps: two 16-byte loads per row
        const float4 a = __ldg(reinterpret_cast<const float4*>(s)), b = __ldg(reinterpret_cast<const float4*>(s) + 1);
        x = a.x; y = a.y; z = a.z;
        d[3] = a.w; d[4] = b.x; d[5] = b.y; d[6] = b.z; d[7] = b.w;
      } else {
        x = __ldg(s); y = __ldg(s + 1); z = __ldg(s + 2);
        for (int k = 3; k < src_cols; ++k) d[k] = __ldg(s + k);
      }
      float nx, ny, nz;
      move_point(j.R, j.dx, j.dy, x, y, z, nx, ny, nz);
      if (roof_filter && x > -2.4f && x < 0.f && y > -0.8f && y < 0.8f && z > -1.5f && z < -1.f) nx = __int_as_float(0x7fc00000);
      d[0] = nx; d[1] = ny; d[2] = nz;
      for (int k = 0; k < n_time; ++k) d[src_cols + k] = (k == j.time_idx) ? 1.f : 0.f;
    }
    __syncthreads();
    const int nrow = min(256, j.n - i0);
    float* out = j.dst + (size_t)i0 * dcols;
    for (int e = threadIdx.x; e < nrow * dcols; e += 256) out[e] = rows[e];
    __syncthreads();
  }
}

extern "C" int lavb_stack_jobs(const void* d_jobs, int n_jobs, int max_n, int src_cols, int n_time, int roof_filter, void* stream) {
  LAVB_CHECK_ARG(n_jobs >= 0 && n_jobs <= 65535 && max_n >= 0 && src_cols >= 3 && n_time >= 0,
                 "stack_jobs: bad arguments (n_jobs %d, max_n %d, src_cols %d, n_time %d)", n_jobs, max_n, src_cols, n_time);
  LAVB_CHECK_ARG(src_cols + n_time <= kStackMaxCols, "stack_jobs: rows wider than %d floats", kStackMaxCols);
  if (n_jobs == 0 || max_n == 0) return 0;
  LAVB_CHECK_ARG(d_jobs != nullptr && is_aligned(d_jobs, 8), "stack_jobs: d_jobs null or not 8-byte aligned");
  dim3 grid(min(ceil_div(max_n, 256), 64), n_jobs);
  stack_jobs_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const StackJob*>(d_jobs), src_cols, n_time, roof_filter);
  LAVB_LAUNCH_OK();
  return 0;
}

// ---- the LiDAR rows of a whole training batch in one launch: GpuLidarStacker (data_pipeline.py) for every sample at once.
// The host has already applied the roof filter, the shuffle, the truncation and the zero padding to row INDICES (rows[r] = raw
// row of output row r, or -1); this kernel gathers and restates the stacker's per-row arithmetic: stack_sweep with R_aug and a
// zero shift, paint (mode 0) on a ones map, the in-place multiply of the painted columns by that 0/1, stack_sweep with R_mv.
struct LidarSweep {          // 88 bytes
  float R_aug[9]; float R_mv[9]; float dx, dy; int time_idx; int row0;
};
static_assert(sizeof(LidarSweep) == 88, "LidarSweep layout is part of the ABI (lav_b200.h)");

__global__ void __launch_bounds__(256) lidar_batch_kernel(const float* __restrict__ raw, long long n_raw, int src_cols,
                                                          const int* __restrict__ rows, long long n_rows,
                                                          const LidarSweep* __restrict__ sweeps, int n_sweeps,
                                                          const __grid_constant__ CamSet cams, int H, int W, int n_time,
                                                          float* __restrict__ out) {
  __shared__ float tile[256 * kStackMaxCols];
  const int dcols = src_cols + n_time;
  const long long r0 = (long long)blockIdx.x * 256, r = r0 + threadIdx.x;
  if (r < n_rows) {
    float* d = tile + threadIdx.x * dcols;
    const int src = __ldg(rows + r);
    int s = -1;
    if (src >= 0 && src < n_raw) {   // the sweep holding raw row src: the last one with row0 <= src
      int lo = 0, hi = n_sweeps;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(&sweeps[mid].row0) <= src) lo = mid + 1; else hi = mid;
      }
      s = lo - 1;
    }
    if (s < 0) {
      for (int k = 0; k < dcols; ++k) d[k] = 0.f;
    } else {
      const LidarSweep& sw = sweeps[s];
      const float* p = raw + (size_t)src * src_cols;
      float ax, ay, az;
      move_point(sw.R_aug, 0.f, 0.f, __ldg(p), __ldg(p + 1), __ldg(p + 2), ax, ay, az);
      int u = 0, v = 0;
      const float vis = project_hit(cams, ax, ay, az, H, W, u, v) >= 0 ? 1.f : 0.f;
      move_point(sw.R_mv, sw.dx, sw.dy, ax, ay, az, d[0], d[1], d[2]);
      d[3] = __ldg(p + 3);
      for (int k = 4; k < src_cols; ++k) d[k] = __fmul_rn(__ldg(p + k), vis);   // NaN * 0 stays NaN, -x * 0 = -0, as in torch
      for (int k = 0; k < n_time; ++k) d[src_cols + k] = (k == sw.time_idx) ? 1.f : 0.f;
    }
  }
  __syncthreads();
  const int nrow = (int)min(256LL, n_rows - r0);
  float* o = out + r0 * dcols;
  for (int e = threadIdx.x; e < nrow * dcols; e += 256) o[e] = tile[e];
}

extern "C" int lavb_lidar_batch(const float* d_raw, long long n_raw, int c, const int* d_rows, long long n_rows,
                                const void* d_sweeps, int n_sweeps, const float* h_cams, int ncam, int h, int w, int n_time,
                                float* d_out, void* stream) {
  LAVB_CHECK_ARG(n_raw >= 0 && n_raw <= 0x7fffffffLL && n_rows >= 0 && n_sweeps >= 0 && c >= 0 && n_time >= 0,
                 "lidar_batch: bad sizes (n_raw %lld, n_rows %lld, n_sweeps %d, c %d, n_time %d)", n_raw, n_rows, n_sweeps, c,
                 n_time);
  LAVB_CHECK_ARG(4 + c + n_time <= kStackMaxCols, "lidar_batch: rows wider than %d floats", kStackMaxCols);
  LAVB_CHECK_ARG(h_cams != nullptr && ncam >= 1 && ncam <= 4 && h > 0 && w > 0, "lidar_batch: bad cameras (ncam %d, %d x %d)",
                 ncam, h, w);
  LAVB_CHECK_ARG(n_rows == 0 || (d_rows != nullptr && d_out != nullptr), "lidar_batch: null row table or output");
  LAVB_CHECK_ARG(n_raw == 0 || (d_raw != nullptr && d_sweeps != nullptr && n_sweeps > 0), "lidar_batch: null raw rows or sweeps");
  LAVB_CHECK_ARG((n_rows + 255) / 256 <= 0x7fffffffLL, "lidar_batch: n_rows %lld needs 2^31 or more blocks", n_rows);
  LAVB_CHECK_ARG(is_aligned(d_raw, 4) && is_aligned(d_rows, 4) && is_aligned(d_sweeps, 4) && is_aligned(d_out, 4),
                 "lidar_batch: d_raw, d_rows, d_sweeps and d_out must be 4-byte aligned");
  if (n_rows == 0) return 0;
  CamSet cs;
  memcpy(cs.m, h_cams, sizeof(float) * 41 * ncam);
  cs.ncam = ncam;
  lidar_batch_kernel<<<(unsigned)((n_rows + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      d_raw, n_raw, 4 + c, d_rows, n_rows, reinterpret_cast<const LidarSweep*>(d_sweeps), n_sweeps, cs, h, w, n_time, d_out);
  LAVB_LAUNCH_OK();
  return 0;
}

// ---- the same batch painted online: lidar_batch_kernel with the painted columns computed from the ERFNet decoder's features
// instead of read from raw.  Per row: project_hit of the raw, unrotated point; at a hit, the 16 features of the sweep's frame slot
// and camera at (v/2, u/2), deconv_logits and softmax_suppress, exactly paint_deconv_kernel's chain; then lidar_batch_kernel's
// rotation, re-mask, move and one-hot.  Bit-identical to lavb_paint_deconv_batched on each sweep followed by lavb_lidar_batch on
// the painted rows, without the painted intermediate: a row reads 16 B of raw point and, when a camera sees it, 32 B (h16) or
// 64 B (fp32) of features.
template <typename TF>
__global__ void __launch_bounds__(256) lidar_batch_paint_kernel(const float* __restrict__ raw, long long n_raw,
                                                                const int* __restrict__ rows, long long n_rows,
                                                                const LidarSweep* __restrict__ sweeps,
                                                                const int* __restrict__ slots, int n_sweeps,
                                                                const TF* __restrict__ feat, int n_frames, int c_cls,
                                                                const DeconvW* __restrict__ dw, const __grid_constant__ CamSet cams,
                                                                int H, int W, int n_time, float* __restrict__ out) {
  __shared__ float tile[256 * kStackMaxCols];
  __shared__ DeconvW sdw;
  for (int i = threadIdx.x; i < (int)(sizeof(DeconvW) / 4); i += blockDim.x) reinterpret_cast<float*>(&sdw)[i] = __ldg(reinterpret_cast<const float*>(dw) + i);
  __syncthreads();
  const int npaint = c_cls - 1, dcols = 4 + npaint + n_time;
  const long long r0 = (long long)blockIdx.x * 256, r = r0 + threadIdx.x;
  if (r < n_rows) {
    float* d = tile + threadIdx.x * dcols;
    const int src = __ldg(rows + r);
    int s = -1;
    if (src >= 0 && src < n_raw) {
      int lo = 0, hi = n_sweeps;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(&sweeps[mid].row0) <= src) lo = mid + 1; else hi = mid;
      }
      s = lo - 1;
    }
    if (s < 0) {
      for (int k = 0; k < dcols; ++k) d[k] = 0.f;
    } else {
      const LidarSweep& sw = sweeps[s];
      const float4 p = __ldg(reinterpret_cast<const float4*>(raw) + src);
      float* pc = d + 4;
      const int f = __ldg(slots + s);
      int u = 0, v = 0;
      const int cam = project_hit(cams, p.x, p.y, p.z, H, W, u, v);
      if (f < 0 || f >= n_frames) {          // a frame slot outside the feature buffer: NaN, never an unseen point's zeros
        for (int k = 0; k < npaint; ++k) pc[k] = __int_as_float(0x7fc00000);
      } else if (cam < 0) {
        for (int k = 0; k < npaint; ++k) pc[k] = 0.f;
      } else {
        const TF* fp = feat + ((((long long)f * cams.ncam + cam) * (H >> 1) + (v >> 1)) * (W >> 1) + (u >> 1)) * 16;
        float fv[16];
        load_feat16<TF>(fp, fv);
        float pr[8];
        deconv_logits<8>(sdw, fv, v & 1, u & 1, pr);
        softmax_suppress(pr, c_cls, pc);
      }
      float ax, ay, az;
      move_point(sw.R_aug, 0.f, 0.f, p.x, p.y, p.z, ax, ay, az);
      const float vis = project_hit(cams, ax, ay, az, H, W, u, v) >= 0 ? 1.f : 0.f;
      move_point(sw.R_mv, sw.dx, sw.dy, ax, ay, az, d[0], d[1], d[2]);
      d[3] = p.w;
      for (int k = 0; k < npaint; ++k) pc[k] = __fmul_rn(pc[k], vis);
      for (int k = 0; k < n_time; ++k) d[4 + npaint + k] = (k == sw.time_idx) ? 1.f : 0.f;
    }
  }
  __syncthreads();
  const int nrow = (int)min(256LL, n_rows - r0);
  float* o = out + r0 * dcols;
  for (int e = threadIdx.x; e < nrow * dcols; e += 256) o[e] = tile[e];
}

extern "C" int lavb_lidar_batch_paint(const float* d_raw, long long n_raw, const int* d_rows, long long n_rows, const void* d_sweeps,
                                      const int* d_slots, int n_sweeps, const void* d_feat, int feat_dtype, int n_frames, int c_cls,
                                      const float* d_deconv, const float* h_cams, int ncam, int h, int w, int n_time, float* d_out,
                                      void* stream) {
  LAVB_CHECK_ARG(n_raw >= 0 && n_raw <= 0x7fffffffLL && n_rows >= 0 && n_sweeps >= 0 && n_frames >= 0 && n_time >= 0,
                 "lidar_batch_paint: bad sizes (n_raw %lld, n_rows %lld, n_sweeps %d, n_frames %d, n_time %d)", n_raw, n_rows,
                 n_sweeps, n_frames, n_time);
  LAVB_CHECK_ARG(c_cls >= 2 && c_cls <= 8, "lidar_batch_paint: c_cls must be 2..8 (got %d)", c_cls);
  LAVB_CHECK_ARG(3 + c_cls + n_time <= kStackMaxCols, "lidar_batch_paint: rows wider than %d floats", kStackMaxCols);
  LAVB_CHECK_ARG(h_cams != nullptr && ncam >= 1 && ncam <= 4 && h > 0 && w > 0 && h % 2 == 0 && w % 2 == 0,
                 "lidar_batch_paint: bad cameras (ncam %d, %d x %d; the image size must be even)", ncam, h, w);
  LAVB_CHECK_ARG(feat_dtype == LAVB_F32 || feat_dtype == LAVB_H16, "lidar_batch_paint: feature dtype must be fp32 or h16");
  LAVB_CHECK_ARG(n_rows == 0 || (d_rows != nullptr && d_out != nullptr && d_deconv != nullptr),
                 "lidar_batch_paint: null row table, output or deconv table");
  LAVB_CHECK_ARG(n_raw == 0 || (d_raw != nullptr && d_sweeps != nullptr && d_slots != nullptr && n_sweeps > 0),
                 "lidar_batch_paint: null raw rows, sweeps or frame slots");
  LAVB_CHECK_ARG(n_raw == 0 || n_frames == 0 || d_feat != nullptr, "lidar_batch_paint: null features");
  LAVB_CHECK_ARG((n_rows + 255) / 256 <= 0x7fffffffLL, "lidar_batch_paint: n_rows %lld needs 2^31 or more blocks", n_rows);
  LAVB_CHECK_ARG(is_aligned(d_raw, 16) && is_aligned(d_feat, feat_dtype == LAVB_F32 ? 16 : 8) && is_aligned(d_rows, 4) &&
                     is_aligned(d_sweeps, 4) && is_aligned(d_slots, 4) && is_aligned(d_deconv, 4) && is_aligned(d_out, 4),
                 "lidar_batch_paint: d_raw must be 16-byte aligned, d_feat 16-byte (fp32) / 8-byte (h16), the others 4-byte");
  if (n_rows == 0) return 0;
  CamSet cs;
  memcpy(cs.m, h_cams, sizeof(float) * 41 * ncam);
  cs.ncam = ncam;
  const unsigned blocks = (unsigned)((n_rows + 255) / 256);
  cudaStream_t st = (cudaStream_t)stream;
  const LidarSweep* sw = reinterpret_cast<const LidarSweep*>(d_sweeps);
  const DeconvW* dw = reinterpret_cast<const DeconvW*>(d_deconv);
  if (feat_dtype == LAVB_F32)
    lidar_batch_paint_kernel<float><<<blocks, 256, 0, st>>>(d_raw, n_raw, d_rows, n_rows, sw, d_slots, n_sweeps, (const float*)d_feat,
                                                            n_frames, c_cls, dw, cs, h, w, n_time, d_out);
  else
    lidar_batch_paint_kernel<h16><<<blocks, 256, 0, st>>>(d_raw, n_raw, d_rows, n_rows, sw, d_slots, n_sweeps, (const h16*)d_feat,
                                                          n_frames, c_cls, dw, cs, h, w, n_time, d_out);
  LAVB_LAUNCH_OK();
  return 0;
}

// Ego-roof filter as the reference applies it: an ORDER-PRESERVING drop (np.delete) of the points inside the roof box, on the
// raw sensor sweep before painting (LAVAgent.preprocess, team_code_v2/lav_agent.py:448-457, call sites :236 and
// lav_agent_fast.py:247).  One block per sweep walks it in chunks of 1024 rows: ballot + block scan give every kept row its
// output slot, so the order is the input order.  Rows past the kept count are filled with NaN (the fixed-shape pipeline's padding,
// which every downstream kernel drops).
__global__ void __launch_bounds__(1024) roof_filter_kernel(const float* __restrict__ src, int n, int cols, long long src_frame_stride,
                                                           float* __restrict__ dst, long long dst_frame_stride,
                                                           int* __restrict__ counts, int pad_nan) {
  __shared__ int warp_cnt[32];
  __shared__ int base_s;
  const float* s0 = src + (long long)blockIdx.x * src_frame_stride;
  float* d0 = dst + (long long)blockIdx.x * dst_frame_stride;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) base_s = 0;
  __syncthreads();
  for (int c0 = 0; c0 < n; c0 += 1024) {
    const int i = c0 + threadIdx.x;
    bool keep = false;
    if (i < n) {
      const float x = __ldg(s0 + (size_t)i * cols), y = __ldg(s0 + (size_t)i * cols + 1), z = __ldg(s0 + (size_t)i * cols + 2);
      keep = !(x > -2.4f && x < 0.f && y > -0.8f && y < 0.8f && z > -1.5f && z < -1.f);
    }
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) warp_cnt[warp] = __popc(m);
    __syncthreads();
    const int base = base_s;
    int woff = 0, total = 0;
    for (int w = 0; w < 32; ++w) { const int c = warp_cnt[w]; if (w < warp) woff += c; total += c; }
    if (keep) {
      const int row = base + woff + __popc(m & ((1u << lane) - 1u));
      for (int k = 0; k < cols; ++k) d0[(size_t)row * cols + k] = __ldg(s0 + (size_t)i * cols + k);
    }
    __syncthreads();
    if (threadIdx.x == 0) base_s = base + total;
    __syncthreads();
  }
  const int kept = base_s;
  if (threadIdx.x == 0 && counts) counts[blockIdx.x] = kept;
  if (pad_nan) {
    const float nanv = __int_as_float(0x7fc00000);
    for (long long e = (long long)kept * cols + threadIdx.x; e < (long long)n * cols; e += 1024) d0[e] = nanv;
  }
}

extern "C" int lavb_roof_filter(const float* d_src, int frames, int n, int cols, long long src_frame_stride, float* d_dst,
                                long long dst_frame_stride, int* d_counts, int pad_nan, void* stream) {
  LAVB_CHECK_ARG(frames >= 0 && n >= 0 && cols >= 3 && src_frame_stride >= 0, "roof_filter: bad arguments");
  if (frames == 0) return 0;
  const long long frame = (long long)n * cols;
  LAVB_CHECK_ARG(frames == 1 || dst_frame_stride >= frame, "roof_filter: output frames overlap (dst_frame_stride %lld < n * cols %lld)",
                 dst_frame_stride, frame);
  LAVB_CHECK_ARG(d_src && d_dst, "roof_filter: null pointer");
  LAVB_CHECK_ARG(is_aligned(d_src, 4) && is_aligned(d_dst, 4) && is_aligned(d_counts, 4), "roof_filter: pointers must be 4-byte aligned");
  LAVB_CHECK_ARG(!ranges_overlap(d_src, 4 * (size_t)((frames - 1) * src_frame_stride + frame), d_dst,
                                 4 * (size_t)((frames - 1) * (frames > 1 ? dst_frame_stride : 0) + frame)),
                 "roof_filter: d_dst overlaps d_src (in-place compaction is not supported)");
  roof_filter_kernel<<<frames, 1024, 0, (cudaStream_t)stream>>>(d_src, n, cols, src_frame_stride, d_dst, dst_frame_stride, d_counts,
                                                                  pad_nan);
  LAVB_LAUNCH_OK();
  return 0;
}

extern "C" int lavb_stack_sweep(const float* d_src, int n, int src_cols, const float* h_R, float dx, float dy, int time_idx,
                                int n_time, int roof_filter, float* d_dst, void* stream) {
  LAVB_CHECK_ARG(n >= 0 && src_cols >= 3 && n_time >= 0 && time_idx >= 0 && (n_time == 0 || time_idx < n_time),
                 "stack_sweep: bad arguments");
  if (n == 0) return 0;
  LAVB_CHECK_ARG(d_src && d_dst && h_R, "stack_sweep: null pointer");
  LAVB_CHECK_ARG(is_aligned(d_src, 4) && is_aligned(d_dst, 4), "stack_sweep: d_src and d_dst must be 4-byte aligned");
  LAVB_CHECK_ARG(!ranges_overlap(d_src, 4 * (size_t)n * src_cols, d_dst, 4 * (size_t)n * (src_cols + n_time)),
                 "stack_sweep: d_dst overlaps d_src");
  StackParams P;
  memcpy(P.R, h_R, sizeof(float) * 9);
  P.dx = dx; P.dy = dy;
  stack_kernel<<<ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(d_src, n, src_cols, P, time_idx, n_time, roof_filter, d_dst);
  LAVB_LAUNCH_OK();
  return 0;
}

extern "C" int lavb_rgb_normalize(const void* d_rgb, int src_is_u8_nhwc, int n, int h, int w, void* d_out, int out_dtype,
                                  void* stream) {
  LAVB_CHECK_ARG(n >= 0 && h >= 0 && w >= 0, "rgb_normalize: n, h, w must be >= 0");
  LAVB_CHECK_ARG(out_dtype == LAVB_F32 || out_dtype == LAVB_H16, "rgb_normalize: bad dtype");
  const long long npix = (long long)n * h * w;
  if (npix == 0) return 0;
  // one 4-channel pixel is stored at a time; the float source is read per element
  LAVB_CHECK_ARG(d_rgb != nullptr && d_out != nullptr && (src_is_u8_nhwc || reinterpret_cast<uintptr_t>(d_rgb) % 4 == 0) &&
                     reinterpret_cast<uintptr_t>(d_out) % (out_dtype == LAVB_F32 ? 16 : 8) == 0,
                 "rgb_normalize: null pointer, or d_out not 4-element aligned (16 B fp32, 8 B 16-bit)");
  const int blocks = ceil_div(npix, 256);
  if (out_dtype == LAVB_F32)
    rgb_norm_kernel<float><<<blocks, 256, 0, (cudaStream_t)stream>>>(d_rgb, src_is_u8_nhwc, n, h, w, (float*)d_out);
  else if (out_dtype == LAVB_H16)
    rgb_norm_kernel<h16><<<blocks, 256, 0, (cudaStream_t)stream>>>(d_rgb, src_is_u8_nhwc, n, h, w, (h16*)d_out);
  LAVB_LAUNCH_OK();
  return 0;
}

extern "C" int lavb_convert(const void* d_src, int src_dtype, void* d_dst, int dst_dtype, long long count, void* stream) {
  LAVB_CHECK_ARG((src_dtype == LAVB_F32 && dst_dtype == LAVB_H16) || (src_dtype == LAVB_H16 && dst_dtype == LAVB_F32),
                 "convert: unsupported dtype pair");
  LAVB_CHECK_ARG(count >= 0, "convert: negative count");
  if (count == 0) return 0;
  const uintptr_t ss = src_dtype == LAVB_F32 ? 4 : 2, ds = dst_dtype == LAVB_F32 ? 4 : 2;
  const uintptr_t src = reinterpret_cast<uintptr_t>(d_src), dst = reinterpret_cast<uintptr_t>(d_dst);
  LAVB_CHECK_ARG(d_src != nullptr && d_dst != nullptr && src % ss == 0 && dst % ds == 0,
                 "convert: null pointer, or a pointer not aligned to its element size");
  // 4 elements per thread: vector loads / stores when both pointers are 4-element aligned, element by element otherwise
  const int vec = src % (4 * ss) == 0 && dst % (4 * ds) == 0;
  const int blocks = ceil_div(ceil_div(count, 4), 256);
  cudaStream_t st = (cudaStream_t)stream;
  if (src_dtype == LAVB_F32)
    convert_kernel<float, h16><<<blocks, 256, 0, st>>>((const float*)d_src, (h16*)d_dst, count, vec);
  else
    convert_kernel<h16, float><<<blocks, 256, 0, st>>>((const h16*)d_src, (float*)d_dst, count, vec);
  LAVB_LAUNCH_OK();
  return 0;
}
