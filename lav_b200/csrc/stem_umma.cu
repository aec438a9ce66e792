// wgmma / TMA implicit-GEMM 7x7 stride-2 pad-3 convolution to 64 channels + bias + ReLU (h16 in and out, fp32 accumulate in
// registers): the stem of the planner's crop embedder (resnet18(num_channels=384).conv1 + bn1 + relu, BatchNorm folded).
//
// GEMM view with the operands swapped against conv_umma.cu: M = the 64 output channels, N = output pixels, K = 49 taps x cin.
// One m64n128k16 reads 2 KB of weights and 4 KB of pixels from shared memory for 64 x 128 x 16 MACs, where pixels-in-M with
// N = 64 would re-read the pixel slice once per 32 output channels.
//
// A CTA tile is 16 x 16 output pixels of one image.  K-block (64-channel chunk kc outer, tap t = 7 ky + kx inner):
//   weights: one 2-D TMA box {64 ch, 64 cout} of the [49 * 64][cin] packed weights (8 KB, L2-resident)
//   pixels : one 4-D TMA box {64 ch, 32 px, 32 rows, 1 image} with element strides {1, 2, 2, 1} starting at input
//            (2 ox0 - 3 + kx, 2 oy0 - 3 + ky): 256 rows of 128 B = the 16 x 16 strided input pixels of the tap, landing in
//            the K-major SWIZZLE_128B layout wgmma reads.  TMA's out-of-bounds zero fill is the convolution's padding.
// Warp roles (288 threads, 1 CTA per SM, persistent over tiles):
//   warps 0-3, 4-7: two consumer warpgroups, output rows 0-7 / 8-15 of the tile (N = 128 each, 64 fp32 accumulators per
//                   thread); one K-block of MMAs in flight; epilogue bias + ReLU -> h16, transposed through shared memory
//                   (the accumulator holds D[cout][pixel], NHWC wants the 64 channels of a pixel contiguous) -> 16 B stores
//   warp 8         : TMA producer (one lane), ring of kStages {weights 8 KB, pixels 32 KB}
#include "sm90.cuh"

namespace lavb {
namespace stem7 {

using namespace sm90;

constexpr int kTile = 16;                         // output pixels per tile side
constexpr int kCout = 64, kBlockK = 64, kTaps = 49;
constexpr int kWBytes = kCout * kBlockK * 2;      // 8 KB
constexpr int kPBytes = kTile * kTile * kBlockK * 2;   // 32 KB
constexpr int kStageBytes = kWBytes + kPBytes;
constexpr int kStages = 5;
constexpr int kThreads = 288;
constexpr int kEpiPitch = kCout * 2 + 16;         // bytes per pixel row of the epilogue transpose (+16: 4-bank skew per row)
constexpr int kEpiPx = 64;                        // pixels per epilogue pass of one warpgroup
constexpr int kEpiBytes = kEpiPx * kEpiPitch;
constexpr int kSmemBytes = 1024 /*align*/ + kStages * kStageBytes + 2 * kEpiBytes + 16 * kStages + kCout * 4;

struct StemArgs {
  int ho, wo, kchunks, tiles_x, tiles_per_img, num_tiles;
  h16* out; const float* bias;
};

__global__ void __launch_bounds__(kThreads, 1) conv7x7s2_umma_kernel(const __grid_constant__ CUtensorMap tmap_x,
                                                                    const __grid_constant__ CUtensorMap tmap_w,
                                                                    const __grid_constant__ StemArgs p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;   // SWIZZLE_128B operands need 1024 B alignment
  uint8_t* gen = smem_raw + (base - smem_u32(smem_raw));
  const uint32_t epi = base + kStages * kStageBytes;
  const uint32_t ctrl = epi + 2 * kEpiBytes;
  const uint32_t full_bar = ctrl, empty_bar = ctrl + 8 * kStages;
  float* ep_bias = reinterpret_cast<float*>(gen + (ctrl - base) + 16 * kStages);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_x)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_w)) : "memory");
    // empty: one arrival per consumer warp once its MMAs have read the slot
    for (int s = 0; s < kStages; ++s) { mbar_init(full_bar + 8 * s, 1); mbar_init(empty_bar + 8 * s, 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int c = threadIdx.x; c < kCout; c += blockDim.x) ep_bias[c] = __ldg(p.bias + c);
  __syncthreads();
  const int nkb = kTaps * p.kchunks;

  if (warp == 8) {
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const int img = tile / p.tiles_per_img, r = tile - img * p.tiles_per_img;
        const int y0 = (r / p.tiles_x) * 2 * kTile - 3, x0 = (r % p.tiles_x) * 2 * kTile - 3;
        // chunk-major: the live input window of a tile is 38 x 38 pixels x 64 channels (185 KB), about 24 MB over all SMs,
        // so it stays in L2 across the 49 taps.  Tap-major would cycle 38 x 38 x cin (1.1 MB at cin = 384) per tile per tap,
        // more than L2 holds over 132 SMs.
        for (int kc = 0; kc < p.kchunks; ++kc) {
          for (int t = 0; t < kTaps; ++t) {
            const int ky = t / 7, kx = t - 7 * ky;
            mbar_wait(empty_bar + 8 * stage, phase ^ 1);
            const uint32_t sw = base + stage * kStageBytes;
            mbar_expect_tx(full_bar + 8 * stage, kStageBytes);
            tma_load_2d(sw, &tmap_w, full_bar + 8 * stage, kc * kBlockK, t * kCout);
            tma_load_4d(sw + kWBytes, &tmap_x, full_bar + 8 * stage, kc * kBlockK, x0 + kx, y0 + ky, img);
            if (++stage == kStages) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
    return;
  }

  const int wg = warp >> 2;                        // output rows [8 wg, 8 wg + 8) of the tile = pixel rows [128 wg, 128 wg + 128)
  const int wtid = threadIdx.x & 127;
  uint8_t* ep = gen + (epi - base) + wg * kEpiBytes;
  // accumulator rows (output channels) of this thread: co and co + 8
  const int co = 16 * (warp & 3) + (lane >> 2);
  int stage = 0; uint32_t phase = 0;
  float acc[64];
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    int prev_stage = -1;
    for (int kb = 0; kb < nkb; ++kb) {
      mbar_wait(full_bar + 8 * stage, phase);
      const uint32_t sw = base + stage * kStageBytes;
      const uint64_t a_desc = desc_sw128(sw), b_desc = desc_sw128(sw + kWBytes + wg * (kPBytes / 2));
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBlockK / 16; ++k)      // +32 B per K16 step inside the 128 B swizzle atom
        wgmma<128>(acc, a_desc + (uint64_t)(2 * k), b_desc + (uint64_t)(2 * k), (kb | k) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();                             // the previous K-block's MMAs are done: its slot may be refilled
      if (prev_stage >= 0 && lane == 0) mbar_arrive(empty_bar + 8 * prev_stage);
      prev_stage = stage;
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    acc_fence(acc);
    if (prev_stage >= 0 && lane == 0) mbar_arrive(empty_bar + 8 * prev_stage);

    // ---- epilogue: relu(acc + bias) -> h16 -> [pixel][cout] in shared memory -> 16 B NHWC stores, 64 pixels per pass.
    // acc[4 i + 2 h + e] = D[co + 8 h][8 i + 2 (lane % 4) + e]
    const int img = tile / p.tiles_per_img, r = tile - img * p.tiles_per_img;
    const int oy0 = (r / p.tiles_x) * kTile + 8 * wg, ox0 = (r % p.tiles_x) * kTile;
    const float b0 = ep_bias[co], b1 = ep_bias[co + 8];
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      bar_sync(1 + wg, 128);                       // the previous pass's reads of `ep` are done
#pragma unroll
      for (int i = 8 * half; i < 8 * half + 8; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int px = 8 * i + 2 * (lane & 3) + e - kEpiPx * half;
          uint8_t* row = ep + px * kEpiPitch;
          *reinterpret_cast<h16*>(row + 2 * co) = float2h16(fmaxf(acc[4 * i + e] + b0, 0.f));
          *reinterpret_cast<h16*>(row + 2 * (co + 8)) = float2h16(fmaxf(acc[4 * i + 2 + e] + b1, 0.f));
        }
      bar_sync(1 + wg, 128);
#pragma unroll
      for (int j = 0; j < kEpiPx * kCout * 2 / 16 / 128; ++j) {   // 4 x 16 B per thread
        const int q = wtid + 128 * j, px = q >> 3, piece = q & 7;
        const int n = kEpiPx * half + px, oy = oy0 + n / kTile, ox = ox0 + n % kTile;
        if (oy < p.ho && ox < p.wo)
          *reinterpret_cast<uint4*>(p.out + (((long long)img * p.ho + oy) * p.wo + ox) * kCout + 8 * piece) =
              *reinterpret_cast<const uint4*>(ep + px * kEpiPitch + 16 * piece);
      }
    }
  }
}

}  // namespace stem7
}  // namespace lavb

using namespace lavb;
using namespace lavb::stem7;

extern "C" int lavb_conv7x7s2_umma(const void* d_in, int n, int h, int w, int cin, const void* d_w, const float* d_bias,
                                   void* d_out, void* stream) {
  LAVB_CHECK_ARG(d_in && d_w && d_bias && d_out, "conv7x7s2_umma: null operand");
  LAVB_CHECK_ARG(n >= 0 && h >= 7 && w >= 7, "conv7x7s2_umma: bad shape n=%d h=%d w=%d (h, w >= 7)", n, h, w);
  LAVB_CHECK_ARG(cin > 0 && cin % 64 == 0, "conv7x7s2_umma: cin must be a multiple of 64 (got %d)", cin);
  if (n == 0) return 0;
  auto encode = get_encode();
  LAVB_CHECK_ARG(encode != nullptr, "conv7x7s2_umma: cuTensorMapEncodeTiled not available from the driver");
  CUtensorMap tmap_x, tmap_w;
  {
    cuuint64_t dims[4] = {(cuuint64_t)cin, (cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)n};
    cuuint64_t strides[3] = {(cuuint64_t)cin * 2, (cuuint64_t)w * cin * 2, (cuuint64_t)h * w * cin * 2};
    cuuint32_t box[4] = {(cuuint32_t)kBlockK, 2 * kTile, 2 * kTile, 1};
    cuuint32_t estr[4] = {1, 2, 2, 1};
    CUresult r = encode(&tmap_x, LAVB_TMAP_H16, 4, const_cast<void*>(d_in), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    LAVB_CHECK_ARG(r == CUDA_SUCCESS, "conv7x7s2_umma: cuTensorMapEncodeTiled(x) failed with %d", (int)r);
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)cin, (cuuint64_t)kTaps * kCout};
    cuuint64_t strides[1] = {(cuuint64_t)cin * 2};
    cuuint32_t box[2] = {(cuuint32_t)kBlockK, (cuuint32_t)kCout};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = encode(&tmap_w, LAVB_TMAP_H16, 2, const_cast<void*>(d_w), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    LAVB_CHECK_ARG(r == CUDA_SUCCESS, "conv7x7s2_umma: cuTensorMapEncodeTiled(w) failed with %d", (int)r);
  }
  StemArgs a;
  memset(&a, 0, sizeof(a));
  a.ho = (h - 1) / 2 + 1; a.wo = (w - 1) / 2 + 1; a.kchunks = cin / kBlockK;
  a.tiles_x = ceil_div(a.wo, kTile);
  a.tiles_per_img = a.tiles_x * ceil_div(a.ho, kTile);
  a.num_tiles = n * a.tiles_per_img;
  a.out = reinterpret_cast<h16*>(d_out); a.bias = d_bias;
  // once per device, never during a later stream capture (callers warm up first)
  LAVB_CUDA_OK(ensure_dyn_smem((const void*)conv7x7s2_umma_kernel, kSmemBytes));
  conv7x7s2_umma_kernel<<<min(a.num_tiles, kNumSMs), kThreads, kSmemBytes, (cudaStream_t)stream>>>(tmap_x, tmap_w, a);
  LAVB_LAUNCH_OK();
  return 0;
}
