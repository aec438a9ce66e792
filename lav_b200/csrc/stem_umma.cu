// wgmma / TMA implicit-GEMM 7x7 stride-2 pad-3 convolution to 64 channels + bias + ReLU (h16 in and out, fp32 accumulate in
// registers): the stem of the planner's crop embedder (resnet18(num_channels=384).conv1 + bn1 + relu, BatchNorm folded).
//
// GEMM view with the operands swapped against conv_umma.cu: M = the 64 output channels, N = output pixels, K = 49 taps x cin.
// One m64n128k16 reads 2 KB of weights and 4 KB of pixels from shared memory for 64 x 128 x 16 MACs, where pixels-in-M with
// N = 64 would re-read the pixel slice once per 32 output channels.
//
// A CTA tile is 16 x 16 output pixels of one image, held COLUMN-major in shared memory (GEMM column n = 16 x + y): the pixel
// tensor map lists H before W, so a TMA box lands as whole output columns of 16 pixels x 128 B = 2 KB each.  Taps of one kernel
// row ky with the same kx parity then read the same box shifted by whole columns, (kx >> 1) x 2 KB, a whole number of 1024 B
// swizzle atoms, so the plain SWIZZLE_128B descriptor holds.  K walk (chunk kc outer, kernel row ky, tap kx inner: the same
// MMA sequence per accumulator as one box per tap, so the sums are bit-identical to it):
//   pixels : per (kc, ky) two 4-D TMA boxes {64 ch, 32 rows, 38 columns, 1 image} with element strides {1, 2, 2, 1} starting
//            at input (x, y) = (2 ox0 - 3 + parity, 2 oy0 - 3 + ky): 19 strided columns x 16 strided rows (38 KB) each, the
//            even-kx box serving kx = 0, 2, 4, 6 and the odd one kx = 1, 3, 5 (its 19th column is over-fetch).  TMA's
//            out-of-bounds zero fill is the convolution's padding.  Against one 32 KB box per tap this moves 14 x 38 KB
//            instead of 49 x 32 KB per chunk.
//   weights: per tap one 2-D TMA box {64 ch, 64 cout} of the [49 * 64][cin] packed weights (8 KB, L2-resident)
// Warp roles (288 threads, 1 CTA per SM, persistent over tiles):
//   warps 0-3, 4-7: two consumer warpgroups, output columns 0-7 / 8-15 of the tile (N = 128 each, 64 fp32 accumulators per
//                   thread); one K-block of MMAs in flight; epilogue bias + ReLU -> h16, transposed through shared memory
//                   (the accumulator holds D[cout][pixel], NHWC wants the 64 channels of a pixel contiguous) -> 16 B stores
//   warp 8         : TMA producer (one lane): a pixel ring of kPStages slots of one kernel row's two boxes (76 KB) and a
//                    weight ring of kWStages x 8 KB (one slot per tap), each with its own full / empty barriers; a pixel slot
//                    is released once the MMAs of its row's last tap have completed
#include "sm90.cuh"

namespace lavb {
namespace stem7 {

using namespace sm90;

constexpr int kTile = 16;                         // output pixels per tile side
constexpr int kCout = 64, kBlockK = 64, kTaps = 49;
constexpr int kWBytes = kCout * kBlockK * 2;      // 8 KB
constexpr int kColBytes = kTile * kBlockK * 2;    // one output column of the tile (16 strided input pixels): 2 KB
constexpr int kBoxBytes = (kTile + 3) * kColBytes;   // 19 columns: the 4 even-kx taps span 3 strided columns (38 KB)
constexpr int kPBytes = 2 * kBoxBytes;            // pixel slot: the even-kx and the odd-kx box of one kernel row
constexpr int kPStages = 2, kWStages = 6;
constexpr int kThreads = 288;
constexpr int kEpiPitch = kCout * 2 + 16;         // bytes per pixel row of the epilogue transpose (+16: 4-bank skew per row)
constexpr int kEpiPx = 64;                        // pixels per epilogue pass of one warpgroup
constexpr int kEpiBytes = kEpiPx * kEpiPitch;
constexpr int kSmemBytes = 1024 /*align*/ + kPStages * kPBytes + kWStages * kWBytes + 2 * kEpiBytes + 16 * (kPStages + kWStages) +
                           kCout * 4;

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
  const uint32_t wring = base + kPStages * kPBytes;
  const uint32_t epi = wring + kWStages * kWBytes;
  const uint32_t ctrl = epi + 2 * kEpiBytes;
  const uint32_t p_full = ctrl, p_empty = ctrl + 8 * kPStages, w_full = ctrl + 16 * kPStages, w_empty = w_full + 8 * kWStages;
  float* ep_bias = reinterpret_cast<float*>(gen + (ctrl - base) + 16 * (kPStages + kWStages));

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_x)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_w)) : "memory");
    // empty: one arrival per consumer warp once its MMAs have read the slot
    for (int s = 0; s < kPStages; ++s) { mbar_init(p_full + 8 * s, 1); mbar_init(p_empty + 8 * s, 8); }
    for (int s = 0; s < kWStages; ++s) { mbar_init(w_full + 8 * s, 1); mbar_init(w_empty + 8 * s, 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int c = threadIdx.x; c < kCout; c += blockDim.x) ep_bias[c] = __ldg(p.bias + c);
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      int ps = 0, ws = 0; uint32_t pph = 0, wph = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const int img = tile / p.tiles_per_img, r = tile - img * p.tiles_per_img;
        const int y0 = (r / p.tiles_x) * 2 * kTile - 3, x0 = (r % p.tiles_x) * 2 * kTile - 3;
        // chunk-major: the live input window of a tile is 38 x 38 pixels x 64 channels (185 KB), about 24 MB over all SMs,
        // so it stays in L2 across the 49 taps.  Tap-major would cycle 38 x 38 x cin (1.1 MB at cin = 384) per tile per tap,
        // more than L2 holds over 132 SMs.
        for (int kc = 0; kc < p.kchunks; ++kc) {
          for (int ky = 0; ky < 7; ++ky) {
            mbar_wait(p_empty + 8 * ps, pph ^ 1);
            const uint32_t sp = base + ps * kPBytes;
            mbar_expect_tx(p_full + 8 * ps, kPBytes);
            tma_load_4d(sp, &tmap_x, p_full + 8 * ps, kc * kBlockK, y0 + ky, x0, img);                  // kx = 0, 2, 4, 6
            tma_load_4d(sp + kBoxBytes, &tmap_x, p_full + 8 * ps, kc * kBlockK, y0 + ky, x0 + 1, img);  // kx = 1, 3, 5
            if (++ps == kPStages) { ps = 0; pph ^= 1; }
            for (int kx = 0; kx < 7; ++kx) {
              mbar_wait(w_empty + 8 * ws, wph ^ 1);
              mbar_expect_tx(w_full + 8 * ws, kWBytes);
              tma_load_2d(wring + ws * kWBytes, &tmap_w, w_full + 8 * ws, kc * kBlockK, (7 * ky + kx) * kCout);
              if (++ws == kWStages) { ws = 0; wph ^= 1; }
            }
          }
        }
      }
    }
    return;
  }

  const int wg = warp >> 2;                        // output columns [8 wg, 8 wg + 8) of the tile = GEMM columns [128 wg, 128 wg + 128)
  const int wtid = threadIdx.x & 127;
  uint8_t* ep = gen + (epi - base) + wg * kEpiBytes;
  // accumulator rows (output channels) of this thread: co and co + 8
  const int co = 16 * (warp & 3) + (lane >> 2);
  int ps = 0, ws = 0; uint32_t pph = 0, wph = 0;
  float acc[64];
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    // After the wgmma_wait<1> of a K-block other than the tile's first, the previous K-block's MMAs are done: its weight
    // slot (ws - 1) is free, and so is the previous kernel row's pixel slot (ps - 1) when this K-block is a row's first tap.
    for (int kc = 0; kc < p.kchunks; ++kc) {
      for (int ky = 0; ky < 7; ++ky) {
        mbar_wait(p_full + 8 * ps, pph);
        const uint32_t sp = base + ps * kPBytes + wg * (8 * kColBytes);
        for (int kx = 0; kx < 7; ++kx) {
          mbar_wait(w_full + 8 * ws, wph);
          const uint64_t a_desc = desc_sw128(wring + ws * kWBytes);
          const uint64_t b_desc = desc_sw128(sp + (kx & 1) * kBoxBytes + (kx >> 1) * kColBytes);
          const bool first = (kc | ky | kx) == 0;
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < kBlockK / 16; ++k)  // +32 B per K16 step inside the 128 B swizzle atom
            wgmma<128>(acc, a_desc + (uint64_t)(2 * k), b_desc + (uint64_t)(2 * k), (!first || k) ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<1>();
          if (lane == 0 && !first) {
            mbar_arrive(w_empty + 8 * (ws ? ws - 1 : kWStages - 1));
            if (kx == 0) mbar_arrive(p_empty + 8 * (ps ? ps - 1 : kPStages - 1));
          }
          if (++ws == kWStages) { ws = 0; wph ^= 1; }
        }
        if (++ps == kPStages) { ps = 0; pph ^= 1; }
      }
    }
    wgmma_wait<0>();
    acc_fence(acc);
    if (lane == 0) {                               // the tile's last K-block: its weight slot and its row's pixel slot
      mbar_arrive(w_empty + 8 * (ws ? ws - 1 : kWStages - 1));
      mbar_arrive(p_empty + 8 * (ps ? ps - 1 : kPStages - 1));
    }

    // ---- epilogue: relu(acc + bias) -> h16 -> [pixel][cout] in shared memory -> 16 B NHWC stores, 64 pixels per pass.
    // acc[4 i + 2 h + e] = D[co + 8 h][8 i + 2 (lane % 4) + e]
    const int img = tile / p.tiles_per_img, r = tile - img * p.tiles_per_img;
    const int oy0 = (r / p.tiles_x) * kTile, ox0 = (r % p.tiles_x) * kTile + 8 * wg;
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
        const int n = kEpiPx * half + px, oy = oy0 + n % kTile, ox = ox0 + n / kTile;   // GEMM column n = 16 x + y
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
    // NHWC memory listed as {C, H, W, N}: the box lands column-major (rows of one output column contiguous)
    cuuint64_t dims[4] = {(cuuint64_t)cin, (cuuint64_t)h, (cuuint64_t)w, (cuuint64_t)n};
    cuuint64_t strides[3] = {(cuuint64_t)w * cin * 2, (cuuint64_t)cin * 2, (cuuint64_t)h * w * cin * 2};
    cuuint32_t box[4] = {(cuuint32_t)kBlockK, 2 * kTile, 2 * (kTile + 3), 1};
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
