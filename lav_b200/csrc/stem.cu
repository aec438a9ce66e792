// 7x7 stride-2 stem convolution of the brake predictor's ResNet-18 on raw uint8 camera frames
// (lav/models/resnet.py:178,235-238 conv1+bn1+relu; team_code_v2/models/rgb.py:66-70 normalisation) and the 3x3/s2 max-pool
// behind it, as an implicit GEMM on the tensor cores: M = output pixels, N = 64, K = 7 rows x 22 (21 = 7 px x 3 channels of one
// window row + 1 zero slot) = 154, padded to 160.  The stem is 48 % of the brake model's GPU time in cuDNN (3 input
// channels); here:
//   * a block owns kStemRows output rows x 128 output columns of one image and stages the 2*rows+5 input rows it needs ONCE
//     in shared memory, already normalised ((u8 - 255 mean_c) / (255 std_c)) and rounded to h16, zero outside the image
//     (zero padding acts on the NORMALISED image, as in the reference); input is read with aligned 4-byte loads;
//   * with that K order one window row is 21 CONSECUTIVE staged elements, so an A-fragment register is a single 4-byte
//     shared-memory load (no im2col buffer, no per-element index arithmetic);
//   * B = BatchNorm-folded weights [64][160] h16 staged once per block; fp32 accumulate (mma.sync m16n8k16);
//   * epilogue bias + ReLU -> h16, transposed through shared memory so every pixel's 128 B leave as full lines.
// The "wide" image of the brake model is three cameras side by side (lav_agent_fast.py:257): `ncam`/`cam_w` index the
// (B, ncam, H, cam_w, 3) camera tensor directly.
#include <climits>
#include <cmath>

#include "common.cuh"

namespace lavb {

constexpr int kStemK = 160, kStemPitch = 168;   // h16 per weight row in smem (pitch chosen bank-conflict free)
constexpr int kStemRows = 8;                     // output rows per block
constexpr int kStemInRows = 2 * kStemRows + 5;   // input rows staged per block
constexpr int kStemQW = 792;                     // staged elements per input row: 6*127 + 22 = 784 used, padded
constexpr int kStemOutPitch = 72;                // h16 per pixel in the per-warp output staging tile
constexpr int kStemSmem = (64 * kStemPitch + kStemInRows * kStemQW + 4 * 32 * kStemOutPitch) * 2;

struct StemArgs {
  const unsigned char* img; int batch, ncam, h, cam_w;     // logical image: h x (ncam*cam_w) x 3
  const h16* w; const float* bias;               // w [64][160], k = ky*22 + kx*3 + c
  float na[3], nb[3];                                       // normalised = u8 * na[c] + nb[c]
  h16* out; int ho, wo;                           // NHWC (batch, ho, wo, 64)
};

__device__ __forceinline__ void mma_h16(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32." LAVB_H16_PTX "." LAVB_H16_PTX ".f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__global__ void __launch_bounds__(128) stem7x7_u8_kernel(const __grid_constant__ StemArgs a) {
  extern __shared__ __align__(16) uint8_t stem_sm[];
  h16* ws = reinterpret_cast<h16*>(stem_sm);              // [64][kStemPitch]
  h16* S = ws + 64 * kStemPitch;                                    // [kStemInRows][kStemQW]
  h16* Ot = S + kStemInRows * kStemQW;                              // [4 warps][32 px][kStemOutPitch]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, gq = lane >> 2, tq = lane & 3;
  const int groups = (a.ho + kStemRows - 1) / kStemRows;
  const int b = blockIdx.x / groups, oy0 = (blockIdx.x - b * groups) * kStemRows;
  const int ox0 = blockIdx.y * 128;
  for (int i = tid; i < 64 * kStemK / 2; i += 128) {                          // weights: 4 B per copy
    const int n = i / (kStemK / 2), k2 = i - n * (kStemK / 2);
    reinterpret_cast<uint32_t*>(ws + n * kStemPitch)[k2] = __ldg(reinterpret_cast<const uint32_t*>(a.w) + i);
  }
  // ---- stage the input rows: element q of a row <-> logical byte (6*ox0 - 9) + q of that image row (byte = ix*3 + c)
  {
    const int base = 6 * ox0 - 9;                           // odd, may be negative
    const int w_first = (base - 3) >> 2;                    // floor((base - 3) / 4): first aligned word touching q >= 0... (q = -3..0)
    const int nwords = (kStemQW + 3 + 3) / 4 + 1;
    const int row_bytes = a.ncam * a.cam_w * 3, cam_bytes = a.cam_w * 3;
    const unsigned char* imgb = a.img + (long long)b * a.ncam * a.h * cam_bytes;
    for (int i = tid; i < kStemInRows * nwords; i += 128) {
      const int r = i / nwords, w = w_first + (i - r * nwords);
      const int iy = 2 * oy0 - 3 + r, byte0 = 4 * w;
      uint32_t word = 0;
      const bool ok = iy >= 0 && iy < a.h && byte0 >= 0 && byte0 < row_bytes;
      if (ok) {
        const int cam = (byte0 >= cam_bytes) + (byte0 >= 2 * cam_bytes) + (byte0 >= 3 * cam_bytes);
        word = __ldg(reinterpret_cast<const uint32_t*>(imgb + ((long long)cam * a.h + iy) * cam_bytes + (byte0 - cam * cam_bytes)));
      }
      int c = byte0 >= 0 ? byte0 % 3 : (3 - ((-byte0) % 3)) % 3;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int q = byte0 + j - base;
        if (q >= 0 && q < kStemQW) {
          const float u = (float)((word >> (8 * j)) & 0xffu);
          const float nrm = c == 0 ? fmaf(u, a.na[0], a.nb[0]) : (c == 1 ? fmaf(u, a.na[1], a.nb[1]) : fmaf(u, a.na[2], a.nb[2]));
          S[r * kStemQW + q] = float2h16(ok ? nrm : 0.f);
        }
        c = c == 2 ? 0 : c + 1;
      }
    }
  }
  __syncthreads();
  // per-lane element offsets of its A-fragment registers: k = 16kk + 2tq + 8h -> (ky, k') ; ky clamped for the K padding
  int offs[kStemK / 16][2];
#pragma unroll
  for (int kk = 0; kk < kStemK / 16; ++kk)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int k = kk * 16 + 2 * tq + 8 * h;
      const int ky = min(k / 22, 6);
      offs[kk][h] = ky * kStemQW + (k - ky * 22);
    }
  const int pxw = warp * 32;                                // the warp's first pixel inside the block's 128 columns
  if (ox0 + pxw >= a.wo) return;
  h16* ot = Ot + warp * 32 * kStemOutPitch;
  float bias2[8][2];
#pragma unroll
  for (int nn = 0; nn < 8; ++nn) { bias2[nn][0] = __ldg(a.bias + nn * 8 + 2 * tq); bias2[nn][1] = __ldg(a.bias + nn * 8 + 2 * tq + 1); }
#pragma unroll 1
  for (int rr = 0; rr < kStemRows; ++rr) {
    const int oy = oy0 + rr;
    if (oy >= a.ho) break;
    float acc[2][8][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nn = 0; nn < 8; ++nn) acc[mt][nn][0] = acc[mt][nn][1] = acc[mt][nn][2] = acc[mt][nn][3] = 0.f;
    const h16* srow = S + 2 * rr * kStemQW + 6 * (pxw + gq);
#pragma unroll
    for (int kk = 0; kk < kStemK / 16; ++kk) {
      uint32_t af[4][2];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int h = 0; h < 2; ++h) af[r][h] = *reinterpret_cast<const uint32_t*>(srow + 48 * r + offs[kk][h]);   // pixel gq + 8r
#pragma unroll
      for (int nn = 0; nn < 8; ++nn) {
        const h16* wp = ws + (nn * 8 + gq) * kStemPitch + kk * 16 + 2 * tq;
        const uint32_t b0 = *reinterpret_cast<const uint32_t*>(wp), b1 = *reinterpret_cast<const uint32_t*>(wp + 8);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) mma_h16(acc[mt][nn], af[mt * 2][0], af[mt * 2 + 1][0], af[mt * 2][1], af[mt * 2 + 1][1], b0, b1);
      }
    }
    // bias + ReLU -> h16 into the warp's staging tile (C fragment: rows gq | gq+8 of each m-tile, cols 8nn + 2tq, +1)
    __syncwarp();
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int nn = 0; nn < 8; ++nn) {
        const float x0 = fmaxf(acc[r >> 1][nn][(r & 1) * 2] + bias2[nn][0], 0.f), x1 = fmaxf(acc[r >> 1][nn][(r & 1) * 2 + 1] + bias2[nn][1], 0.f);
        store2<h16>(ot + ((r >> 1) * 16 + (r & 1) * 8 + gq) * kStemOutPitch + nn * 8 + 2 * tq, x0, x1);
      }
    __syncwarp();
    h16* orow = a.out + (((long long)b * a.ho + oy) * a.wo + ox0 + pxw) * 64;
    const int npx = min(32, a.wo - ox0 - pxw);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int id = i * 32 + lane, px = id >> 3, ch = id & 7;
      if (px < npx) *reinterpret_cast<uint4*>(orow + px * 64 + ch * 8) = *reinterpret_cast<const uint4*>(ot + px * kStemOutPitch + ch * 8);
    }
  }
}

// 3x3 stride-2 pad-1 max-pool on NHWC h16 (lav/models/resnet.py:181,238): one thread = one output pixel x 8 channels.
// __hmax2_nan: a NaN in the window gives the canonical NaN, as MaxPool2d propagates NaN (__hmax2 would drop it).
__global__ void __launch_bounds__(256) maxpool3x3s2_kernel(const h16* __restrict__ in, int n, int h, int w, int c8,
                                                           h16* __restrict__ out, int ho, int wo) {
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)n * ho * wo * c8;
  if (gid >= total) return;
  const int ch = (int)(gid % c8);
  long long p = gid / c8;
  const int ox = (int)(p % wo); p /= wo;
  const int oy = (int)(p % ho);
  const int b = (int)(p / ho);
  const uint4* src = reinterpret_cast<const uint4*>(in) + (long long)b * h * w * c8 + ch;
  h162 m[4];
  bool first = true;
#pragma unroll
  for (int dy = -1; dy <= 1; ++dy) {
    const int iy = 2 * oy + dy;
    if (iy < 0 || iy >= h) continue;
#pragma unroll
    for (int dx = -1; dx <= 1; ++dx) {
      const int ix = 2 * ox + dx;
      if (ix < 0 || ix >= w) continue;
      const uint4 v = __ldg(src + ((long long)iy * w + ix) * c8);
      const h162* pv = reinterpret_cast<const h162*>(&v);
      if (first) { m[0] = pv[0]; m[1] = pv[1]; m[2] = pv[2]; m[3] = pv[3]; first = false; }
      else { m[0] = __hmax2_nan(m[0], pv[0]); m[1] = __hmax2_nan(m[1], pv[1]); m[2] = __hmax2_nan(m[2], pv[2]); m[3] = __hmax2_nan(m[3], pv[3]); }
    }
  }
  uint4 o;
  o.x = *reinterpret_cast<uint32_t*>(&m[0]); o.y = *reinterpret_cast<uint32_t*>(&m[1]);
  o.z = *reinterpret_cast<uint32_t*>(&m[2]); o.w = *reinterpret_cast<uint32_t*>(&m[3]);
  reinterpret_cast<uint4*>(out)[gid] = o;
}

}  // namespace lavb

using namespace lavb;

extern "C" int lavb_stem7x7s2_u8(const void* d_img, int batch, int ncam, int h, int cam_w, const void* d_w, const float* d_bias,
                                 const float* h_mean, const float* h_std, void* d_out, void* stream) {
  LAVB_CHECK_ARG(batch >= 0 && ncam >= 1 && ncam <= 4 && h >= 7 && cam_w >= 8, "stem7x7s2_u8: bad shape");
  LAVB_CHECK_ARG(cam_w % 4 == 0, "stem7x7s2_u8: camera width must be a multiple of 4 (got %d)", cam_w);
  LAVB_CHECK_ARG(cam_w <= INT_MAX / 12, "stem7x7s2_u8: camera width %d is too large", cam_w);
  const int ho = (h + 6 - 7) / 2 + 1, wo = (ncam * cam_w + 6 - 7) / 2 + 1;
  LAVB_CHECK_ARG((long long)batch * ceil_div(ho, kStemRows) <= INT_MAX && ceil_div(wo, 128) <= 65535,
                 "stem7x7s2_u8: %d images of %d x %d need more blocks than a grid holds", batch, h, ncam * cam_w);
  if (batch == 0) return 0;
  LAVB_CHECK_ARG(d_img && d_w && d_bias && d_out && h_mean && h_std, "stem7x7s2_u8: null pointer");
  LAVB_CHECK_ARG(is_aligned(d_img, 4) && is_aligned(d_w, 4) && is_aligned(d_bias, 4) && is_aligned(d_out, 16),
                 "stem7x7s2_u8: d_img, d_w and d_bias must be 4-byte and d_out 16-byte aligned");
  const size_t out_bytes = (size_t)batch * ho * wo * 64 * sizeof(h16);
  LAVB_CHECK_ARG(!ranges_overlap(d_img, (size_t)batch * ncam * h * cam_w * 3, d_out, out_bytes), "stem7x7s2_u8: d_out overlaps d_img");
  LAVB_CHECK_ARG(!ranges_overlap(d_w, 64 * 160 * sizeof(h16), d_out, out_bytes) && !ranges_overlap(d_bias, 64 * sizeof(float), d_out, out_bytes),
                 "stem7x7s2_u8: d_out overlaps d_w or d_bias (every block reads them at its start)");
  StemArgs a;
  for (int c = 0; c < 3; ++c) {
    a.na[c] = 1.f / (255.f * h_std[c]); a.nb[c] = -h_mean[c] / h_std[c];
    LAVB_CHECK_ARG(std::isfinite(a.na[c]) && std::isfinite(a.nb[c]) && h_std[c] != 0.f,
                   "stem7x7s2_u8: mean[%d] = %g and std[%d] = %g give a non-finite normalisation", c, h_mean[c], c, h_std[c]);
  }
  LAVB_CUDA_OK(ensure_dyn_smem((const void*)stem7x7_u8_kernel, kStemSmem));
  a.img = reinterpret_cast<const unsigned char*>(d_img); a.batch = batch; a.ncam = ncam; a.h = h; a.cam_w = cam_w;
  a.w = reinterpret_cast<const h16*>(d_w); a.bias = d_bias;
  a.out = reinterpret_cast<h16*>(d_out);
  a.ho = ho; a.wo = wo;
  dim3 grid(batch * ceil_div(a.ho, kStemRows), ceil_div(a.wo, 128));
  stem7x7_u8_kernel<<<grid, 128, kStemSmem, (cudaStream_t)stream>>>(a);
  LAVB_LAUNCH_OK();
  return 0;
}

extern "C" int lavb_maxpool3x3s2_nhwc(const void* d_in, int n, int h, int w, int c, void* d_out, void* stream) {
  LAVB_CHECK_ARG(n >= 0 && h >= 1 && w >= 1 && c >= 8 && c % 8 == 0, "maxpool3x3s2_nhwc: bad shape (channels must be a multiple of 8)");
  const int ho = (h - 1) / 2 + 1, wo = (w - 1) / 2 + 1;
  const long long total = (long long)n * ho * wo * (c / 8);
  LAVB_CHECK_ARG((total + 255) / 256 <= INT_MAX, "maxpool3x3s2_nhwc: %lld output vectors need more than 2^31 - 1 blocks", total);
  if (n == 0) return 0;
  LAVB_CHECK_ARG(d_in && d_out, "maxpool3x3s2_nhwc: null pointer");
  LAVB_CHECK_ARG(is_aligned(d_in, 16) && is_aligned(d_out, 16), "maxpool3x3s2_nhwc: d_in and d_out must be 16-byte aligned");
  LAVB_CHECK_ARG(!ranges_overlap(d_in, (size_t)n * h * w * c * sizeof(h16), d_out, (size_t)total * 8 * sizeof(h16)),
                 "maxpool3x3s2_nhwc: d_out overlaps d_in");
  maxpool3x3s2_kernel<<<ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const h16*>(d_in), n, h, w, c / 8,
                                                                              reinterpret_cast<h16*>(d_out), ho, wo);
  LAVB_LAUNCH_OK();
  return 0;
}
