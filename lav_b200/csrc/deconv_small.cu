// Grouped ConvTranspose2d(k=3, s=2, p=1, output_padding=1) with a handful of output channels — the second layer
// of LAV's four detection/segmentation heads (lav/models/lidar.py:155: ConvTranspose2d(64 -> {2,2,2,3})).
// All heads read one NHWC hidden tensor (group g = channels [g*cin_g, (g+1)*cin_g)); one thread owns one input
// pixel of one group and produces its 2x2 output block (all 9 kernel taps are used exactly once per block), so the
// hidden tensor is read once and the tiny outputs are written coalesced.  HBM-bound by construction.
#include "common.cuh"

namespace lavb {

constexpr int kMaxGroups = 8;

struct DeconvArgs {
  const void* in; int n, h, w, in_cstride, cin_g, groups;
  const float* wgt;    // [g][cin_g][9][4] fp32 (tap = ky*3+kx, 4 = padded cout)
  const float* bias;   // [g][4]
  float* out[kMaxGroups]; int n_out[kMaxGroups]; int sigmoid[kMaxGroups];
};

constexpr int kTH = 8, kTW = 16;          // input-pixel tile of one block (one thread per pixel)
constexpr int kPitch = 68;                // floats per staged pixel (64 channels + 4 pad): conflict-free LDS.128 across lanes

// Block = one 8x16 input tile of one group.  The (8+1)x(16+1) pixel halo x cin_g channels is staged in shared memory
// with coalesced 16 B loads (a pixel's group slice is contiguous), then every thread reads its 2x2 neighbourhood from
// shared memory — global memory sees each hidden value once (+halo), the taps' weights are broadcast LDS.128.
template <typename T>
__global__ void __launch_bounds__(kTH * kTW) deconv3x3s2_small_kernel(const __grid_constant__ DeconvArgs a) {
  extern __shared__ __align__(16) float smem[];
  float* ws = smem;                                   // [cin_g][9][4]
  float* xs = smem + a.cin_g * 36;                    // [(kTH+1)*(kTW+1)][kPitch]
  const int g = blockIdx.y;
  const int tiles_x = (a.w + kTW - 1) / kTW, tiles_y = (a.h + kTH - 1) / kTH;
  const int img = blockIdx.x / (tiles_x * tiles_y), tr = blockIdx.x - img * tiles_x * tiles_y;
  const int y0 = (tr / tiles_x) * kTH, x0 = (tr % tiles_x) * kTW;
  for (int i = threadIdx.x; i < a.cin_g * 36; i += blockDim.x) ws[i] = __ldg(a.wgt + (size_t)g * a.cin_g * 36 + i);
  const T* in = reinterpret_cast<const T*>(a.in);
  const int vec_per_px = a.cin_g / 4;
  for (int i = threadIdx.x; i < (kTH + 1) * (kTW + 1) * vec_per_px; i += blockDim.x) {
    const int px = i / vec_per_px, v = i - px * vec_per_px;
    const int yy = y0 + px / (kTW + 1), xx = x0 + px % (kTW + 1);
    float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
    if (yy < a.h && xx < a.w) val = load4<T>(in + (((long long)img * a.h + yy) * a.w + xx) * a.in_cstride + g * a.cin_g + v * 4);
    *reinterpret_cast<float4*>(xs + px * kPitch + v * 4) = val;
  }
  __syncthreads();
  const int ty = threadIdx.x / kTW, tx = threadIdx.x % kTW;
  const int iy = y0 + ty, ix = x0 + tx;
  if (iy >= a.h || ix >= a.w) return;
  const float* p00 = xs + (ty * (kTW + 1) + tx) * kPitch;
  const float* p01 = p00 + kPitch;
  const float* p10 = p00 + (kTW + 1) * kPitch;
  const float* p11 = p10 + kPitch;
  float acc[4][4];   // [position 00,01,10,11][cout]
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int o = 0; o < 4; ++o) acc[q][o] = 0.f;
  for (int c = 0; c < a.cin_g; c += 4) {
    const float4 x00 = *reinterpret_cast<const float4*>(p00 + c), x01 = *reinterpret_cast<const float4*>(p01 + c);
    const float4 x10 = *reinterpret_cast<const float4*>(p10 + c), x11 = *reinterpret_cast<const float4*>(p11 + c);
    const float v00[4] = {x00.x, x00.y, x00.z, x00.w}, v01[4] = {x01.x, x01.y, x01.z, x01.w};
    const float v10[4] = {x10.x, x10.y, x10.z, x10.w}, v11[4] = {x11.x, x11.y, x11.z, x11.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float4* wc = reinterpret_cast<const float4*>(ws + (size_t)(c + e) * 36);   // wc[tap] = 4 couts
      auto fma4 = [&](float (&dst)[4], float x, const float4 w) {
        dst[0] = fmaf(x, w.x, dst[0]); dst[1] = fmaf(x, w.y, dst[1]); dst[2] = fmaf(x, w.z, dst[2]); dst[3] = fmaf(x, w.w, dst[3]);
      };
      // out(2iy,2ix) = P00 w11 ; out(2iy,2ix+1) = P01 w10 + P00 w12 ; out(2iy+1,2ix) = P10 w01 + P00 w21 ;
      // out(2iy+1,2ix+1) = P11 w00 + P10 w02 + P01 w20 + P00 w22      (w[ky][kx], tap = 3*ky+kx)
      fma4(acc[0], v00[e], wc[4]);
      fma4(acc[1], v01[e], wc[3]); fma4(acc[1], v00[e], wc[5]);
      fma4(acc[2], v10[e], wc[1]); fma4(acc[2], v00[e], wc[7]);
      fma4(acc[3], v11[e], wc[0]); fma4(acc[3], v10[e], wc[2]); fma4(acc[3], v01[e], wc[6]); fma4(acc[3], v00[e], wc[8]);
    }
  }
  const int no = a.n_out[g];
  float* out = a.out[g];
  const int H2 = 2 * a.h, W2 = 2 * a.w;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int oy = 2 * iy + (q >> 1), ox = 2 * ix + (q & 1);
    float* o = out + (((long long)img * H2 + oy) * W2 + ox) * no;
    for (int k = 0; k < no; ++k) {
      float v = acc[q][k] + __ldg(a.bias + g * 4 + k);
      if (a.sigmoid[g]) v = 1.f / (1.f + expf(-v));
      o[k] = v;
    }
  }
}

}  // namespace lavb

using namespace lavb;

extern "C" int lavb_deconv3x3s2_small(const void* d_in, int dtype, int n, int h, int w, int in_cstride, int groups, int cin_g,
                                      const float* d_w, const float* d_bias, const int* h_n_out, const int* h_sigmoid,
                                      float* const* h_out_ptrs, void* stream) {
  LAVB_CHECK_ARG(groups >= 1 && groups <= kMaxGroups, "deconv_small: 1..8 groups");
  LAVB_CHECK_ARG(dtype == LAVB_F32 || dtype == LAVB_H16, "deconv_small: bad dtype");
  LAVB_CHECK_ARG(cin_g >= 8 && cin_g % 8 == 0 && groups * cin_g <= in_cstride && in_cstride % 8 == 0,
                 "deconv_small: channels must be positive multiples of 8");
  LAVB_CHECK_ARG(cin_g <= 64, "deconv_small: at most 64 input channels per group (got %d)", cin_g);
  LAVB_CHECK_ARG(n >= 0 && h >= 0 && w >= 0, "deconv_small: n, h, w must be >= 0");
  LAVB_CHECK_ARG(h_n_out != nullptr && h_sigmoid != nullptr && h_out_ptrs != nullptr, "deconv_small: null host array");
  // the input is staged 4 channels at a time; weights, bias and outputs are accessed per element
  LAVB_CHECK_ARG((long long)n * h * w == 0 ||
                     (d_in != nullptr && d_w != nullptr && d_bias != nullptr &&
                      reinterpret_cast<uintptr_t>(d_in) % (dtype == LAVB_F32 ? 16 : 8) == 0 &&
                      reinterpret_cast<uintptr_t>(d_w) % 4 == 0 && reinterpret_cast<uintptr_t>(d_bias) % 4 == 0),
                 "deconv_small: d_in must be 4-element aligned (16 B fp32, 8 B 16-bit), d_w and d_bias non-null and 4-byte aligned");
  DeconvArgs a;
  a.in = d_in; a.n = n; a.h = h; a.w = w; a.in_cstride = in_cstride; a.cin_g = cin_g; a.groups = groups; a.wgt = d_w; a.bias = d_bias;
  for (int g = 0; g < groups; ++g) {
    LAVB_CHECK_ARG(h_n_out[g] >= 1 && h_n_out[g] <= 4, "deconv_small: 1..4 output channels per group");
    LAVB_CHECK_ARG((long long)n * h * w == 0 || (h_out_ptrs[g] != nullptr && reinterpret_cast<uintptr_t>(h_out_ptrs[g]) % 4 == 0),
                   "deconv_small: output %d null or not 4-byte aligned", g);
    a.out[g] = h_out_ptrs[g]; a.n_out[g] = h_n_out[g]; a.sigmoid[g] = h_sigmoid[g];
  }
  if ((long long)n * h * w == 0) return 0;
  dim3 grid(n * ceil_div(h, kTH) * ceil_div(w, kTW), groups);
  const size_t smem = ((size_t)cin_g * 36 + (size_t)(kTH + 1) * (kTW + 1) * kPitch) * sizeof(float);
  cudaStream_t st = (cudaStream_t)stream;
  LAVB_CUDA_OK(ensure_dyn_smem((const void*)deconv3x3s2_small_kernel<float>, 64 * 1024));
  LAVB_CUDA_OK(ensure_dyn_smem((const void*)deconv3x3s2_small_kernel<h16>, 64 * 1024));
  if (dtype == LAVB_F32) deconv3x3s2_small_kernel<float><<<grid, kTH * kTW, smem, st>>>(a);
  else deconv3x3s2_small_kernel<h16><<<grid, kTH * kTW, smem, st>>>(a);
  LAVB_LAUNCH_OK();
  return 0;
}
