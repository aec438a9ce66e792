// wgmma / TMA implicit-GEMM convolution with the output channels in M (h16 in and out, fp32 accumulate in registers), in two
// forms: the 7x7 / stride-2 / pad-3 stem of the planner's crop embedder (resnet18(num_channels=384).conv1 + bn1 + relu,
// BatchNorm folded), and the 3x3 / pad-1 / stride-1 or -2 convolutions of the BEV stack (backbone conv1 / conv2, the fused
// 384->256 heads conv).
//
// GEMM view with the operands swapped against conv_umma.cu: M = output channels, N = output pixels, K = taps x cin.
// One m64n128k16 reads 2 KB of weights and 4 KB of pixels from shared memory for 64 x 128 x 16 MACs, where pixels-in-M with
// N = 64 would re-read the pixel slice once per 32 output channels.
//
// A CTA tile is 16 x 16 output pixels of one image, held COLUMN-major in shared memory (GEMM column n = 16 x + y): the pixel
// tensor map lists H before W, so a TMA box lands as whole output columns of 16 pixels x 128 B = 2 KB each.  Taps of one kernel
// row ky read the same box shifted by whole columns, a whole number of 1024 B swizzle atoms, so the plain SWIZZLE_128B
// descriptor holds:
//   stride 1: per (chunk, ky) one 4-D TMA box {64 ch, 16 rows, 16 + KS - 1 columns, 1 image} at input (x, y) =
//             (ox0 - KS/2, oy0 - KS/2 + ky); tap kx reads it from column kx on (3x3: 18 columns, 36 KB);
//   stride 2: per (chunk, ky) two boxes with element strides {1, 2, 2, 1}, at x = 2 ox0 - KS/2 + parity: 16 + (KS - 1)/2 strided
//             columns each (3x3: 17, 34 KB; the stem: 19, 38 KB), the even box serving kx = 0, 2, .. and the odd one kx = 1, 3, ..;
//             tap kx reads box kx % 2 from column kx / 2 on.
// TMA's out-of-bounds zero fill is the convolution's padding.
//   weights: per (tap, chunk) one 2-D TMA box {64 ch, CO cout} of the [taps * cout][cin] packed weights (CO x 128 B, L2-resident)
// K order (every accumulator sees the same MMA sequence as with one box per tap, so the sums do not depend on the boxes):
//   SC = 1: chunk kc outer, kernel row ky, tap kx inner (the stem, cin = 64, and cin = 384: chunk-major keeps a tile's input
//           window in L2 across the taps; tap-major would cycle (16 S + KS)^2 x cin pixels per tile per tap);
//   SC = 2: kernel row ky, tap kx, chunk kc inner (cin = 128, both chunks of a kernel row in one pixel slot): the tap-outer,
//           chunk-inner order of conv_umma_kernel, whose outputs this kernel then reproduces bit for bit.
// Output channels per CTA:
//   CO = 64 : both warpgroups m64 over the same 64 channels, output columns 0-7 / 8-15 of the tile (N = 128 each, 64 fp32
//             accumulators per thread);
//   CO = 128: warpgroup g owns channels 64 g .. 64 g + 63 over the whole tile (N = 256, 128 accumulators per thread);
//   more channels run as CTA columns of CO channels each (the 256-channel heads conv: two), adjacent in the tile order so
//   that both columns of a tile read its input window from L2 at about the same time.
// Warp roles (288 threads, 1 CTA per SM, persistent over tiles):
//   warps 0-7: two consumer warpgroups; one K-block of MMAs in flight; epilogue [max](acc [+ b], 0) * s + t -> h16 (conv_umma's
//              fp32 operations and saturating conversion), transposed through shared memory (the accumulator holds
//              D[cout][pixel], NHWC wants the channels of a pixel contiguous) -> 16 B stores
//   warp 8   : TMA producer (one lane): a pixel ring of kPStages slots of one kernel row's boxes (SC chunks) and a weight ring of
//              kWStages x CO x 128 B (one slot per tap and chunk), each with its own full / empty barriers; a pixel slot is
//              released once the MMAs of its row's last tap have completed
#include "sm90.cuh"

namespace lavb {
namespace cmajor {

using namespace sm90;

constexpr int kTile = 16;                         // output pixels per tile side
constexpr int kBlockK = 64;
constexpr int kColBytes = kTile * kBlockK * 2;    // one output column of the tile (16 input pixels): 2 KB
constexpr int kThreads = 288;
constexpr int kEpiPitch = 64 * 2 + 16;            // bytes per pixel row of the epilogue transpose (+16: 4-bank skew per row)
constexpr int kEpiPx = 64;                        // pixels per epilogue pass of one warpgroup
constexpr int kEpiBytes = kEpiPx * kEpiPitch;
constexpr int kMaxCout = 256;
constexpr int kSmemCap = 227 * 1024;

template <int KS, int S, int CO, int SC>
struct Cfg {
  static constexpr int kCols = S == 1 ? kTile + KS - 1 : kTile + (KS - 1) / 2;   // input columns per box
  static constexpr int kBoxBytes = kCols * kColBytes;
  static constexpr int kPBytes = SC * S * kBoxBytes;   // pixel slot: the S parity boxes of SC chunks of one kernel row
  static constexpr int kWBytes = CO * kBlockK * 2;
  static constexpr int kN = CO == 64 ? 8 * kTile : 16 * kTile;   // GEMM columns (pixels) per warpgroup
  static constexpr int kCtrl = 16 * 32 + 3 * kMaxCout * 4;       // barriers (<= 32 slots), bias / scale / shift
  static constexpr int kFixed = 1024 /*align*/ + 2 * kEpiBytes + kCtrl;
  static constexpr int kPStages = kPBytes <= 40 * 1024 ? 3 : 2;
  static constexpr int kWFit = (kSmemCap - kFixed - kPStages * kPBytes) / kWBytes;
  static constexpr int kWStages = kWFit < 12 ? kWFit : 12;
  static constexpr int kSmem = kFixed + kPStages * kPBytes + kWStages * kWBytes;
  static_assert(kWStages >= 3 && kPStages + kWStages <= 32 && kSmem <= kSmemCap, "shared-memory plan");
};

struct Args {
  int ho, wo, cout, kchunks, tiles_x, tiles_per_img, ncol, num_tiles;
  int pre_bias;           // bias added before the ReLU (else folded into the shift)
  int pre_relu;           // max(a [+ b], 0) before the affine (fmaxf: a NaN becomes 0); without it a NaN stays NaN
  float shift0;           // the shift where none is given
  h16* out;
  const float* bias; const float* scale; const float* shift;
};

template <int KS, int S, int CO, int SC>
__global__ void __launch_bounds__(kThreads, 1) conv_cmajor_kernel(const __grid_constant__ CUtensorMap tmap_x,
                                                                  const __grid_constant__ CUtensorMap tmap_w,
                                                                  const __grid_constant__ Args p) {
  using C = Cfg<KS, S, CO, SC>;
  constexpr int kPStages = C::kPStages, kWStages = C::kWStages, kPBytes = C::kPBytes, kWBytes = C::kWBytes;
  constexpr int kBoxBytes = C::kBoxBytes, kN = C::kN;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;   // SWIZZLE_128B operands need 1024 B alignment
  uint8_t* gen = smem_raw + (base - smem_u32(smem_raw));
  const uint32_t wring = base + kPStages * kPBytes;
  const uint32_t epi = wring + kWStages * kWBytes;
  const uint32_t ctrl = epi + 2 * kEpiBytes;
  const uint32_t p_full = ctrl, p_empty = ctrl + 8 * kPStages, w_full = ctrl + 16 * kPStages, w_empty = w_full + 8 * kWStages;
  float* ep_b = reinterpret_cast<float*>(gen + (ctrl - base) + 16 * 32);
  float* ep_s = ep_b + kMaxCout;
  float* ep_t = ep_s + kMaxCout;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_x)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_w)) : "memory");
    // empty: one arrival per consumer warp once its MMAs have read the slot
    for (int s = 0; s < kPStages; ++s) { mbar_init(p_full + 8 * s, 1); mbar_init(p_empty + 8 * s, 8); }
    for (int s = 0; s < kWStages; ++s) { mbar_init(w_full + 8 * s, 1); mbar_init(w_empty + 8 * s, 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int c = threadIdx.x; c < p.cout; c += blockDim.x) {
    // epi(a) = max(a + b, 0) * s + t with the pre-ReLU.  Without it the bias folds into the shift: (a + b) s + t = a s + (b s + t)
    const float b = p.bias ? __ldg(p.bias + c) : 0.f;
    const float sc = p.scale ? __ldg(p.scale + c) : 1.f;
    const float sh = p.shift ? __ldg(p.shift + c) : p.shift0;
    ep_b[c] = b;
    ep_s[c] = sc;
    ep_t[c] = p.pre_bias ? sh : fmaf(b, sc, sh);
  }
  __syncthreads();
  const int nkg = p.kchunks / SC;

  if (warp == 8) {
    if (lane == 0) {
      int ps = 0, ws = 0; uint32_t pph = 0, wph = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const int col = tile % p.ncol, sp = tile / p.ncol;
        const int img = sp / p.tiles_per_img, r = sp - img * p.tiles_per_img;
        const int y0 = (r / p.tiles_x) * S * kTile - KS / 2, x0 = (r % p.tiles_x) * S * kTile - KS / 2;
        for (int kg = 0; kg < nkg; ++kg) {
          for (int ky = 0; ky < KS; ++ky) {
            mbar_wait(p_empty + 8 * ps, pph ^ 1);
            const uint32_t sp_at = base + ps * kPBytes;
            mbar_expect_tx(p_full + 8 * ps, kPBytes);
            for (int c = 0; c < SC; ++c)
              for (int par = 0; par < S; ++par)
                tma_load_4d(sp_at + (c * S + par) * kBoxBytes, &tmap_x, p_full + 8 * ps, (kg * SC + c) * kBlockK, y0 + ky,
                            x0 + par, img);
            if (++ps == kPStages) { ps = 0; pph ^= 1; }
            for (int kx = 0; kx < KS; ++kx) {
              for (int c = 0; c < SC; ++c) {
                mbar_wait(w_empty + 8 * ws, wph ^ 1);
                mbar_expect_tx(w_full + 8 * ws, kWBytes);
                tma_load_2d(wring + ws * kWBytes, &tmap_w, w_full + 8 * ws, (kg * SC + c) * kBlockK,
                            (KS * ky + kx) * p.cout + col * CO);
                if (++ws == kWStages) { ws = 0; wph ^= 1; }
              }
            }
          }
        }
      }
    }
    return;
  }

  const int wg = warp >> 2;
  const int wtid = threadIdx.x & 127;
  uint8_t* ep = gen + (epi - base) + wg * kEpiBytes;
  // CO = 64: GEMM columns [128 wg, 128 wg + 128) = output columns [8 wg, 8 wg + 8); CO = 128: weight rows [64 wg, 64 wg + 64)
  const uint32_t a_off = CO == 128 ? wg * (64 * kBlockK * 2) : 0;
  const uint32_t b_off = CO == 64 ? wg * (8 * kColBytes) : 0;
  // accumulator rows (output channels of this warpgroup's 64) of this thread: co and co + 8
  const int co = 16 * (warp & 3) + (lane >> 2);
  int ps = 0, ws = 0; uint32_t pph = 0, wph = 0;
  float acc[kN / 2];
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    // After the wgmma_wait<1> of a K-block other than the tile's first, the previous K-block's MMAs are done: its weight
    // slot (ws - 1) is free, and so is the previous kernel row's pixel slot (ps - 1) when this K-block is a row's first.
    for (int kg = 0; kg < nkg; ++kg) {
      for (int ky = 0; ky < KS; ++ky) {
        mbar_wait(p_full + 8 * ps, pph);
        const uint32_t sp_at = base + ps * kPBytes + b_off;
        for (int kx = 0; kx < KS; ++kx) {
#pragma unroll
          for (int c = 0; c < SC; ++c) {
            mbar_wait(w_full + 8 * ws, wph);
            const uint64_t a_desc = desc_sw128(wring + ws * kWBytes + a_off);
            const uint64_t b_desc = desc_sw128(sp_at + (c * S + kx % S) * kBoxBytes + (kx / S) * kColBytes);
            const bool first = (kg | ky | kx | c) == 0;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < kBlockK / 16; ++k)  // +32 B per K16 step inside the 128 B swizzle atom
              wgmma<kN>(acc, a_desc + (uint64_t)(2 * k), b_desc + (uint64_t)(2 * k), (!first || k) ? 1u : 0u);
            wgmma_commit();
            wgmma_wait<1>();
            if (lane == 0 && !first) {
              mbar_arrive(w_empty + 8 * (ws ? ws - 1 : kWStages - 1));
              if (kx == 0 && c == 0) mbar_arrive(p_empty + 8 * (ps ? ps - 1 : kPStages - 1));
            }
            if (++ws == kWStages) { ws = 0; wph ^= 1; }
          }
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

    // ---- epilogue: [max](acc [+ b], 0) * s + t -> h16 -> [pixel][64 cout] in shared memory -> 16 B NHWC stores, 64 pixels
    // per pass.  acc[4 i + 2 h + e] = D[co + 8 h][8 i + 2 (lane % 4) + e]
    const int col = tile % p.ncol, sp = tile / p.ncol;
    const int img = sp / p.tiles_per_img, r = sp - img * p.tiles_per_img;
    const int oy0 = (r / p.tiles_x) * kTile, ox0 = (r % p.tiles_x) * kTile + (CO == 64 ? 8 * wg : 0);
    const int ch0 = col * CO + (CO == 128 ? 64 * wg : 0);   // this warpgroup's first output channel
    const float b0 = ep_b[ch0 + co], b1 = ep_b[ch0 + co + 8];
    const float s0 = ep_s[ch0 + co], s1 = ep_s[ch0 + co + 8];
    const float t0 = ep_t[ch0 + co], t1 = ep_t[ch0 + co + 8];
#pragma unroll
    for (int pass = 0; pass < kN / kEpiPx; ++pass) {
      bar_sync(1 + wg, 128);                       // the previous pass's reads of `ep` are done
#pragma unroll
      for (int i = 8 * pass; i < 8 * pass + 8; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int px = 8 * i + 2 * (lane & 3) + e - kEpiPx * pass;
          uint8_t* row = ep + px * kEpiPitch;
          float x0 = acc[4 * i + e], x1 = acc[4 * i + 2 + e];
          if (p.pre_bias) { x0 += b0; x1 += b1; }
          if (p.pre_relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }   // only when set: fmaxf(NaN, -inf) would be -inf
          x0 = fmaf(x0, s0, t0);
          x1 = fmaf(x1, s1, t1);
          *reinterpret_cast<h16*>(row + 2 * co) = float2h16(x0);
          *reinterpret_cast<h16*>(row + 2 * (co + 8)) = float2h16(x1);
        }
      bar_sync(1 + wg, 128);
#pragma unroll
      for (int j = 0; j < kEpiPx * 64 * 2 / 16 / 128; ++j) {   // 4 x 16 B per thread
        const int q = wtid + 128 * j, px = q >> 3, piece = q & 7;
        const int n = kEpiPx * pass + px, oy = oy0 + n % kTile, ox = ox0 + n / kTile;   // GEMM column n = 16 x + y
        if (oy < p.ho && ox < p.wo)
          *reinterpret_cast<uint4*>(p.out + (((long long)img * p.ho + oy) * p.wo + ox) * p.cout + ch0 + 8 * piece) =
              *reinterpret_cast<const uint4*>(ep + px * kEpiPitch + 16 * piece);
      }
    }
  }
}

// Tensor maps of the NHWC input (listed {C, H, W, N}, so a box lands column-major) and of the [taps * cout][cin] weights.
static int encode_maps(const char* who, const void* d_in, int n, int h, int w, int cin, int ks, int s, const void* d_w, int cout,
                       int co, CUtensorMap* tmap_x, CUtensorMap* tmap_w) {
  auto encode = get_encode();
  LAVB_CHECK_ARG(encode != nullptr, "%s: cuTensorMapEncodeTiled not available from the driver", who);
  {
    const int cols = s == 1 ? kTile + ks - 1 : kTile + (ks - 1) / 2;
    cuuint64_t dims[4] = {(cuuint64_t)cin, (cuuint64_t)h, (cuuint64_t)w, (cuuint64_t)n};
    cuuint64_t strides[3] = {(cuuint64_t)w * cin * 2, (cuuint64_t)cin * 2, (cuuint64_t)h * w * cin * 2};
    cuuint32_t box[4] = {(cuuint32_t)kBlockK, (cuuint32_t)(s * kTile), (cuuint32_t)(s * cols), 1};
    cuuint32_t estr[4] = {1, (cuuint32_t)s, (cuuint32_t)s, 1};
    CUresult r = encode(tmap_x, LAVB_TMAP_H16, 4, const_cast<void*>(d_in), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    LAVB_CHECK_ARG(r == CUDA_SUCCESS, "%s: cuTensorMapEncodeTiled(x) failed with %d", who, (int)r);
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)cin, (cuuint64_t)ks * ks * cout};
    cuuint64_t strides[1] = {(cuuint64_t)cin * 2};
    cuuint32_t box[2] = {(cuuint32_t)kBlockK, (cuuint32_t)co};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = encode(tmap_w, LAVB_TMAP_H16, 2, const_cast<void*>(d_w), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    LAVB_CHECK_ARG(r == CUDA_SUCCESS, "%s: cuTensorMapEncodeTiled(w) failed with %d", who, (int)r);
  }
  return 0;
}

template <int KS, int S, int CO, int SC>
static int launch(const CUtensorMap& tmap_x, const CUtensorMap& tmap_w, const Args& a, void* stream) {
  constexpr int smem = Cfg<KS, S, CO, SC>::kSmem;
  // once per (variant, device), never during a later stream capture (callers warm up first)
  LAVB_CUDA_OK(ensure_dyn_smem((const void*)conv_cmajor_kernel<KS, S, CO, SC>, smem));
  conv_cmajor_kernel<KS, S, CO, SC><<<min(a.num_tiles, kNumSMs), kThreads, smem, (cudaStream_t)stream>>>(tmap_x, tmap_w, a);
  LAVB_LAUNCH_OK();
  return 0;
}

// The checks both entries make once their sizes are valid: alignment (TMA reads d_in / d_w, the epilogue stores d_out in 16 B
// vectors and reads bias / scale / shift as floats), d_out apart from every operand (each CTA reads them while others store),
// and the tile count, an int in the kernel.
static int check_operands(const char* who, const void* d_in, int n, int h, int w, int cin, int taps, const void* d_w, int cout,
                          const float* bias, const float* scale, const float* shift, const void* d_out, int ho, int wo, int co) {
  const auto al = [](const void* q, int a) { return reinterpret_cast<uintptr_t>(q) % a == 0; };
  LAVB_CHECK_ARG(al(d_in, 16) && al(d_w, 16) && al(d_out, 16), "%s: d_in, d_w and d_out must be 16 B aligned", who);
  LAVB_CHECK_ARG(al(bias, 4) && al(scale, 4) && al(shift, 4), "%s: bias, scale and shift must be 4 B aligned", who);
  LAVB_CHECK_ARG((long long)n * ceil_div(ho, kTile) * ceil_div(wo, kTile) * (cout / co) < (1LL << 31), "%s: more than 2^31 tiles", who);
  const long long out_bytes = (long long)n * ho * wo * cout * 2;
  const auto overlap = [&](const void* q, long long bytes) {
    const char *o = static_cast<const char*>(d_out), *c = static_cast<const char*>(q);
    return q && o < c + bytes && c < o + out_bytes;
  };
  LAVB_CHECK_ARG(!overlap(d_in, (long long)n * h * w * cin * 2) && !overlap(d_w, (long long)taps * cout * cin * 2) &&
                 !overlap(bias, 4LL * cout) && !overlap(scale, 4LL * cout) && !overlap(shift, 4LL * cout),
                 "%s: d_out must not overlap d_in, d_w, bias, scale or shift", who);
  return 0;
}

static void tiles(Args& a, int n, int ho, int wo, int cout, int co) {
  a.ho = ho; a.wo = wo; a.cout = cout; a.ncol = cout / co;
  a.tiles_x = ceil_div(wo, kTile);
  a.tiles_per_img = a.tiles_x * ceil_div(ho, kTile);
  a.num_tiles = n * a.tiles_per_img * a.ncol;
}

}  // namespace cmajor
}  // namespace lavb

using namespace lavb;
using namespace lavb::cmajor;

extern "C" int lavb_conv7x7s2_umma(const void* d_in, int n, int h, int w, int cin, const void* d_w, const float* d_bias,
                                   void* d_out, void* stream) {
  LAVB_CHECK_ARG(d_in && d_w && d_bias && d_out, "conv7x7s2_umma: null operand");
  LAVB_CHECK_ARG(n >= 0 && h >= 7 && w >= 7, "conv7x7s2_umma: bad shape n=%d h=%d w=%d (h, w >= 7)", n, h, w);
  LAVB_CHECK_ARG(cin > 0 && cin % 64 == 0, "conv7x7s2_umma: cin must be a multiple of 64 (got %d)", cin);
  if (n == 0) return 0;
  if (int e = check_operands("conv7x7s2_umma", d_in, n, h, w, cin, 49, d_w, 64, d_bias, nullptr, nullptr, d_out, (h - 1) / 2 + 1,
                             (w - 1) / 2 + 1, 64)) return e;
  CUtensorMap tmap_x, tmap_w;
  if (int e = encode_maps("conv7x7s2_umma", d_in, n, h, w, cin, 7, 2, d_w, 64, 64, &tmap_x, &tmap_w)) return e;
  Args a;
  memset(&a, 0, sizeof(a));
  tiles(a, n, (h - 1) / 2 + 1, (w - 1) / 2 + 1, 64, 64);
  a.kchunks = cin / kBlockK;
  // relu(acc + b) as max(acc + b, 0) * 1 + (-0): adding -0 leaves every value, a -0 from fmaxf included, as it is
  a.pre_bias = 1; a.pre_relu = 1; a.shift0 = -0.f;
  a.out = reinterpret_cast<h16*>(d_out); a.bias = d_bias;
  return launch<7, 2, 64, 1>(tmap_x, tmap_w, a, stream);
}

extern "C" int lavb_conv3x3_umma(const void* d_in, int n, int h, int w, int cin, int stride, const void* d_w, int cout,
                                 const float* d_bias, const float* d_scale, const float* d_shift, int pre_relu, void* d_out,
                                 void* stream) {
  LAVB_CHECK_ARG(d_in && d_w && d_out, "conv3x3_umma: null operand");
  LAVB_CHECK_ARG(n >= 0 && h >= 1 && w >= 1, "conv3x3_umma: bad shape n=%d h=%d w=%d", n, h, w);
  LAVB_CHECK_ARG(stride == 1 || stride == 2, "conv3x3_umma: stride must be 1 or 2 (got %d)", stride);
  LAVB_CHECK_ARG(cin == 64 || cin == 128 || cin == 384, "conv3x3_umma: cin must be 64, 128 or 384 (got %d)", cin);
  LAVB_CHECK_ARG(cout == 64 || cout == 128 || cout == 256, "conv3x3_umma: cout must be 64, 128 or 256 (got %d)", cout);
  LAVB_CHECK_ARG((d_scale == nullptr) == (d_shift == nullptr), "conv3x3_umma: scale and shift come together");
  if (n == 0) return 0;
  const int co = cout == 64 ? 64 : 128;
  if (int e = check_operands("conv3x3_umma", d_in, n, h, w, cin, 9, d_w, cout, d_bias, d_scale, d_shift, d_out, (h - 1) / stride + 1,
                             (w - 1) / stride + 1, co)) return e;
  CUtensorMap tmap_x, tmap_w;
  if (int e = encode_maps("conv3x3_umma", d_in, n, h, w, cin, 3, stride, d_w, cout, co, &tmap_x, &tmap_w)) return e;
  Args a;
  memset(&a, 0, sizeof(a));
  tiles(a, n, (h - 1) / stride + 1, (w - 1) / stride + 1, cout, co);
  a.kchunks = cin / kBlockK;
  a.pre_bias = pre_relu && d_bias != nullptr;
  a.pre_relu = pre_relu != 0;
  a.shift0 = 0.f;
  a.out = reinterpret_cast<h16*>(d_out); a.bias = d_bias; a.scale = d_scale; a.shift = d_shift;
  // cin = 128 at stride 1: both chunks of a kernel row per pixel slot (tap-major K, as conv_umma_kernel); otherwise chunk-major
  // (at stride 2 a two-chunk slot would be 136 KB, and no two of them fit)
  const int variant = (stride == 2) * 4 + (co == 128) * 2 + (stride == 1 && cin == 128);
  switch (variant) {
    case 0: return launch<3, 1, 64, 1>(tmap_x, tmap_w, a, stream);
    case 1: return launch<3, 1, 64, 2>(tmap_x, tmap_w, a, stream);
    case 2: return launch<3, 1, 128, 1>(tmap_x, tmap_w, a, stream);
    case 3: return launch<3, 1, 128, 2>(tmap_x, tmap_w, a, stream);
    case 4: return launch<3, 2, 64, 1>(tmap_x, tmap_w, a, stream);
    default: return launch<3, 2, 128, 1>(tmap_x, tmap_w, a, stream);
  }
}
