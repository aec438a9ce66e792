// Fused ERFNet pair kernel (lav_b200.erfnet.FUSE_PAIRS, on by default):
// one kernel for a (3x1 -> 1x3) convolution pair of ERFNet's non_bottleneck_1d (lav/models/erfnet.py:37-63):
//     mid = relu(conv3x1(x) + b1)                      (vertical taps, dilation d)
//     out = [relu]( (conv1x3(mid) + b2) * s + t [+ res] )   (horizontal taps, dilation d; BN affine; residual)
// Un-fused, each of the two layers is HBM-bound;
// fused, `mid` never leaves the SM.  A tile is 128 pixels made of FULL-WIDTH image rows (W = 64 -> 2 rows, W = 32 -> 4 rows),
// so the horizontal conv needs no halo: its zero padding is the image border.
//   stage 1: wgmma over 3 vertical taps (A = 4-D TMA boxes shifted by the tap, B = W1 blocks) into register accumulators
//   epilogue 1: acc1 + bias1 -> h16 -> relu -> shared memory, written three times in the SWIZZLE_128B K-major operand layout:
//               shifted by +d, 0, -d pixels inside each image row (rows that fall off the image border stay zero), i.e. the
//               three A operands of the horizontal taps
//   stage 2: wgmma over the 3 horizontal taps (A = those copies, B = W2 blocks through the same TMA ring)
//   epilogue 2: acc2 + shift2 -> h16 (+ residual, saturating) -> ReLU = max(a, 0) with NaN -> 0, written in place over the residual tile in a
//               ring slot and stored to NHWC by one TMA store per 64 channels.  The BatchNorm scale is folded into W2 by the caller.
// Warp roles: warps 0-3 and 4-7 are two consumer warpgroups (tile pixels 0-63 / 64-127), warp 8 is the TMA producer; persistent
// over tiles.  Ring order per tile: stage-1 fills (A + W1), stage-2 fills (W2 only), then the tile's output slot, which the
// producer fills with the residual tile (rows past the image zero-filled) ahead of stage 2, so epilogue 2 reads it from shared
// memory; the slot is released once the TMA store has read it, and the store clips rows past the image.  With C = 64 two
// CTAs share an SM, so one CTA's epilogues overlap the other's MMAs.
#include <stdlib.h>
#include "sm90.cuh"

namespace lavb {
namespace pair {

constexpr int kBlockM = 128, kBlockK = 64;
constexpr int kABytes = kBlockM * kBlockK * 2;  // 16 KB: one K-block of an A operand
constexpr int kMaxStages = 8;
constexpr int kPairThreads = 288;

struct PairArgs {
  int n, h, w, c, kchunks, dil, tile_w, tile_h, tiles_per_img, num_tiles, stages, post_relu;
  const h16* res;                          // only tested for null: the residual tile arrives by TMA
  const float* bias1; const float* shift2;
  long long* trace; int trace_tiles;      // profiling aid (lavb_conv_pair_set_trace): per-CTA, per-tile clock64 stamps, or null
};
// stamps of tile iteration i of this CTA, taken by thread 0: [0] acc1 ready, [1] mid written, [2] acc2 ready, [3] tile stored
#define PAIR_STAMP(slot, i)                                                                                         \
  do {                                                                                                              \
    if (p.trace && threadIdx.x == 0 && (i) < p.trace_tiles)                                                         \
      p.trace[((long long)blockIdx.x * p.trace_tiles + (i)) * 8 + (slot)] = clock64();                              \
  } while (0)

using namespace sm90;

// ReLU as fmaxf(a, 0): __hmax2 returns the operand that is not NaN, so a NaN comes out as 0
__device__ __forceinline__ h162 relu2(h162 v) { return __hmax2(v, floats2h162(0.f, 0.f)); }
__device__ __forceinline__ uint32_t relu2(uint32_t x) {
  const h162 v = relu2(*reinterpret_cast<const h162*>(&x));
  return *reinterpret_cast<const uint32_t*>(&v);
}
// residual add in packed 16-bit arithmetic.  A packed add rounds a sum past the finite range to inf, so the sum is clamped to
// the largest finite value (+-65504; +-bf16's maximum in the bf16 build) afterwards: the same saturating store as every
// cvt.rn.satfinite in the library (in-range sums are unchanged).  The clamp keeps a NaN (the _nan forms), and the ReLU then
// turns it into 0, so the residual paths follow the same NaN rule as the residual-free ones.
__device__ __forceinline__ uint32_t add2(uint32_t x, uint32_t r, bool relu) {
  const h162 a = *reinterpret_cast<const h162*>(&x), b = *reinterpret_cast<const h162*>(&r);
#ifndef LAVB_H16_BF16
  const uint32_t hi = 0x7BFF7BFFu, lo = 0xFBFFFBFFu;           // +65504 / -65504 in both halves
#else
  const uint32_t hi = 0x7F7F7F7Fu, lo = 0xFF7FFF7Fu;           // +-bf16's largest finite value in both halves
#endif
  h162 v = __hmin2_nan(__hadd2(a, b), *reinterpret_cast<const h162*>(&hi));
  v = relu ? relu2(v) : __hmax2_nan(v, *reinterpret_cast<const h162*>(&lo));
  return *reinterpret_cast<const uint32_t*>(&v);
}

template <int kC>
__global__ void __launch_bounds__(kPairThreads, kC == 64 ? 2 : 1) conv_pair_umma_kernel(const __grid_constant__ CUtensorMap tmap_a,
                                                                                       const __grid_constant__ CUtensorMap tmap_w1,
                                                                                       const __grid_constant__ CUtensorMap tmap_w2,
                                                                                       const __grid_constant__ CUtensorMap tmap_r,
                                                                                       const __grid_constant__ CUtensorMap tmap_o,
                                                                                       const __grid_constant__ PairArgs p) {
  constexpr int kNC = kC / 64;                                      // 64-column MMA chunks
  constexpr int kChunks = kC / kBlockK;                             // K-blocks per tap
  constexpr int kWBytes = kC * kBlockK * 2;                         // one weight K-block: c rows x 128 B
  constexpr int kSlotBytes = kABytes + kWBytes;
  constexpr int kNkb = 3 * kChunks;                                 // K-blocks per stage
  constexpr int kBpf = kSlotBytes / kWBytes;                        // W2 K-blocks per ring slot in stage 2
  constexpr int kOutBytes = kChunks * kABytes;                      // one tile of the residual / output: 128 px x c x 2 B
  static_assert(kNkb % kBpf == 0, "stage 2 fills whole ring slots");
  static_assert(kOutBytes <= kSlotBytes, "the residual / output tile fits one ring slot");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;     // SWIZZLE_128B operands need 1024 B alignment
  uint8_t* gen = smem_raw + (base - smem_u32(smem_raw));
  const uint32_t mid = base + p.stages * kSlotBytes;                // [3 taps][kchunks] x 16 KB, K-major SW128
  constexpr int kMidBytes = 3 * kChunks * kABytes;
  const uint32_t ctrl = mid + kMidBytes;
  const uint32_t full_bar = ctrl, empty_bar = ctrl + 8 * kMaxStages;
  float* ep_b1 = reinterpret_cast<float*>(gen + (ctrl - base) + 16 * kMaxStages);   // bias of conv A
  float* ep_t2 = ep_b1 + 128;                                                       // shift of conv B (BatchNorm folded by the caller)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_a)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_w1)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_w2)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_r)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_o)) : "memory");
    for (int s = 0; s < p.stages; ++s) { mbar_init(full_bar + 8 * s, 1); mbar_init(empty_bar + 8 * s, 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int c = threadIdx.x; c < kC; c += blockDim.x) {
    ep_b1[c] = __ldg(p.bias1 + c);
    ep_t2[c] = p.shift2 ? __ldg(p.shift2 + c) : 0.f;
  }
  // the shifted copies keep zero rows where a tap falls off the image border: clear `mid` once, data rows are rewritten per tile
  for (int i = threadIdx.x; i < kMidBytes / 16; i += blockDim.x)
    *reinterpret_cast<uint4*>(gen + (mid - base) + 16 * i) = make_uint4(0u, 0u, 0u, 0u);
  proxy_fence_async();
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      int slot = 0; uint32_t phase = 0;
      // ring order = consumption order, per tile: stage 1 (A + W1 per K-block); stage 2, which needs only weights: a ring slot
      // (A part + W part) takes kBpf whole W2 K-blocks, so the stage is 1 fill (c = 64) or 3 fills (c = 128); then the tile's
      // output slot, filled with the residual tile (or, without a residual, just marked full), where epilogue 2 stages the output
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const int img = tile / p.tiles_per_img, y0 = (tile - img * p.tiles_per_img) * p.tile_h;
        for (int t = 0; t < 3; ++t)
          for (int kc = 0; kc < kChunks; ++kc) {
            mbar_wait(empty_bar + 8 * slot, phase ^ 1);
            const uint32_t sa = base + slot * kSlotBytes;
            mbar_expect_tx(full_bar + 8 * slot, kSlotBytes);
            tma_load_4d(sa, &tmap_a, full_bar + 8 * slot, kc * kBlockK, 0, y0 + (t - 1) * p.dil, img);
            tma_load_2d(sa + kABytes, &tmap_w1, full_bar + 8 * slot, kc * kBlockK, t * kC);
            if (++slot == p.stages) { slot = 0; phase ^= 1; }
          }
        for (int kb0 = 0; kb0 < kNkb; kb0 += kBpf) {
          mbar_wait(empty_bar + 8 * slot, phase ^ 1);
          const uint32_t sa = base + slot * kSlotBytes;
          mbar_expect_tx(full_bar + 8 * slot, kBpf * kWBytes);
          for (int b = 0; b < kBpf; ++b) {
            const int kb = kb0 + b, t = kb / kChunks, kc = kb - t * kChunks;
            tma_load_2d(sa + b * kWBytes, &tmap_w2, full_bar + 8 * slot, kc * kBlockK, t * kC);
          }
          if (++slot == p.stages) { slot = 0; phase ^= 1; }
        }
        mbar_wait(empty_bar + 8 * slot, phase ^ 1);
        if (p.res) {                                 // rows past the image are zero-filled (and never stored)
          mbar_expect_tx(full_bar + 8 * slot, kOutBytes);
          for (int kc = 0; kc < kChunks; ++kc)
            tma_load_4d(base + slot * kSlotBytes + kc * kABytes, &tmap_r, full_bar + 8 * slot, kc * kBlockK, 0, y0, img);
        } else {
          mbar_arrive(full_bar + 8 * slot);
        }
        if (++slot == p.stages) { slot = 0; phase ^= 1; }
      }
    }
    return;
  }

  const int wg = warp >> 2;                          // tile pixels [64 wg, 64 wg + 64)
  const int d = p.dil;
  const bool relu_out = p.post_relu != 0;
  uint8_t* midp = gen + (mid - base);
  int slot = 0; uint32_t phase = 0;
  int i = 0;
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, ++i) {
    const int img = tile / p.tiles_per_img, y0 = (tile - img * p.tiles_per_img) * p.tile_h;
    // ---- stage 1: acc1 = conv3x1(x)
    float acc[kC / 2];                               // 64-column chunk cc: acc[32cc .. 32cc+31]
    int prev = -1;
    for (int kb = 0; kb < kNkb; ++kb) {
      mbar_wait(full_bar + 8 * slot, phase);
      const uint32_t sa = base + slot * kSlotBytes;
      const uint64_t a_desc = sm90::desc_sw128(sa + wg * (kABytes / 2)), b_desc = sm90::desc_sw128(sa + kABytes);
      sm90::wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBlockK / 16; ++k)         // one MMA over all kC columns per K16 step
        sm90::wgmma<kC>(acc, a_desc + (uint64_t)(2 * k), b_desc + (uint64_t)(2 * k), (kb | k) ? 1u : 0u);
      sm90::wgmma_commit();
      sm90::wgmma_wait<1>();
      if (prev >= 0 && lane == 0) mbar_arrive(empty_bar + 8 * prev);
      prev = slot;
      if (++slot == p.stages) { slot = 0; phase ^= 1; }
    }
    sm90::wgmma_wait<0>();
    sm90::acc_fence(acc);
    if (lane == 0) mbar_arrive(empty_bar + 8 * prev);
    PAIR_STAMP(0, i);
    // ---- epilogue 1: acc1 + bias1 -> h16 -> relu -> three shifted K-major copies in shared memory.  Both warpgroups' stage-2 MMAs
    // of the previous tile have completed (each waited for its own before its epilogue 2) once all 256 threads pass here.
    sm90::bar_sync(1, 256);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = 64 * wg + 16 * (warp & 3) + (lane >> 2) + 8 * h;   // tile row = pixel
      const int px = m % p.tile_w;
      // destination rows of this pixel's data in the three shifted copies (tap t reads x + (t-1) d): row m - (t-1) d
      const bool ok0 = px + d < p.tile_w, ok2 = px - d >= 0;
      const int r0 = m + d, r2 = m - d;
#pragma unroll
      for (int cc = 0; cc < kNC; ++cc)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int col = 64 * cc + 8 * j + 2 * (lane & 3);
          const float2 b = *reinterpret_cast<const float2*>(ep_b1 + col);
          const uint32_t v = relu2(pack_h16(acc[32 * cc + 4 * j + 2 * h] + b.x, acc[32 * cc + 4 * j + 2 * h + 1] + b.y));
          uint8_t* blk = midp + cc * kABytes + (col & 7) * 2;              // K-block cc (64 channels), piece j, this pair
          if (ok0) *reinterpret_cast<uint32_t*>(blk + 0 * kChunks * kABytes + r0 * 128 + ((j ^ (r0 & 7)) << 4)) = v;
          *reinterpret_cast<uint32_t*>(blk + 1 * kChunks * kABytes + m * 128 + ((j ^ (m & 7)) << 4)) = v;
          if (ok2) *reinterpret_cast<uint32_t*>(blk + 2 * kChunks * kABytes + r2 * 128 + ((j ^ (r2 & 7)) << 4)) = v;
        }
    }
    proxy_fence_async();                             // generic-proxy stores -> visible to the tensor core's async-proxy reads
    sm90::bar_sync(1, 256);
    PAIR_STAMP(1, i);
    // ---- stage 2: acc2 = conv1x3(mid)
    prev = -1;
    for (int kb0 = 0; kb0 < kNkb; kb0 += kBpf) {
      mbar_wait(full_bar + 8 * slot, phase);
      const uint32_t sa = base + slot * kSlotBytes;
      sm90::wgmma_fence();
#pragma unroll
      for (int b = 0; b < kBpf; ++b) {
        const uint64_t a_desc = sm90::desc_sw128(mid + (kb0 + b) * kABytes + wg * (kABytes / 2)), b_desc = sm90::desc_sw128(sa + b * kWBytes);   // kb = t*kchunks + kc
#pragma unroll
        for (int k = 0; k < kBlockK / 16; ++k)
          sm90::wgmma<kC>(acc, a_desc + (uint64_t)(2 * k), b_desc + (uint64_t)(2 * k), (kb0 | b | k) ? 1u : 0u);
      }
      sm90::wgmma_commit();
      sm90::wgmma_wait<1>();
      if (prev >= 0 && lane == 0) mbar_arrive(empty_bar + 8 * prev);
      prev = slot;
      if (++slot == p.stages) { slot = 0; phase ^= 1; }
    }
    sm90::wgmma_wait<0>();
    sm90::acc_fence(acc);
    if (lane == 0) mbar_arrive(empty_bar + 8 * prev);
    PAIR_STAMP(2, i);
    const int out_slot = slot; const uint32_t out_phase = phase;
    if (++slot == p.stages) { slot = 0; phase ^= 1; }
    // ---- epilogue 2: acc2 + shift2 -> h16 (+ residual) -> ReLU, staged in the output slot in the input's layout, one TMA store
    mbar_wait(full_bar + 8 * out_slot, out_phase);
    uint8_t* outp = gen + out_slot * kSlotBytes;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = 64 * wg + 16 * (warp & 3) + (lane >> 2) + 8 * h;
#pragma unroll
      for (int cc = 0; cc < kNC; ++cc)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int col = 64 * cc + 8 * j + 2 * (lane & 3);
          const float2 t = *reinterpret_cast<const float2*>(ep_t2 + col);
          uint32_t* o = reinterpret_cast<uint32_t*>(outp + cc * kABytes + m * 128 + ((j ^ (m & 7)) << 4) + (col & 7) * 2);
          uint32_t v = pack_h16(acc[32 * cc + 4 * j + 2 * h] + t.x, acc[32 * cc + 4 * j + 2 * h + 1] + t.y);
          if (p.res) v = add2(v, *o, relu_out);
          else if (relu_out) v = relu2(v);
          *o = v;
        }
    }
    proxy_fence_async();                             // the TMA store reads what these threads wrote
    sm90::bar_sync(1, 256);
    if (threadIdx.x == 0) {                          // rows past the image are clipped by the tensor map
      for (int kc = 0; kc < kChunks; ++kc) tma_store_4d(&tmap_o, base + out_slot * kSlotBytes + kc * kABytes, kc * kBlockK, 0, y0, img);
      bulk_commit();
      bulk_wait_read<0>();
      mbar_arrive(empty_bar + 8 * out_slot, 8);      // the slot is free once the store has read it
    }
    PAIR_STAMP(3, i);
  }
  if (threadIdx.x == 0) bulk_wait<0>();              // the last stores have landed before the CTA retires
}

}  // namespace pair
}  // namespace lavb

using namespace lavb;
using namespace lavb::pair;

static long long* g_pair_trace = nullptr;
static int g_pair_trace_tiles = 0;
extern "C" int lavb_conv_pair_set_trace(void* d_buf, int tiles_per_cta) {
  g_pair_trace = reinterpret_cast<long long*>(d_buf);
  g_pair_trace_tiles = d_buf ? tiles_per_cta : 0;
  return 0;
}

extern "C" int lavb_conv_pair_umma(const lavb_conv_pair_desc* d, void* stream) {
  LAVB_CHECK_ARG(d != nullptr, "conv_pair_umma: null descriptor");
  LAVB_CHECK_ARG(d->c == 64 || d->c == 128, "conv_pair_umma: channels must be 64 or 128 (got %d)", d->c);
  LAVB_CHECK_ARG(d->w == 32 || d->w == 64 || d->w == 128, "conv_pair_umma: image width must be 32, 64 or 128 (a tile is made of full rows)");
  LAVB_CHECK_ARG(d->dil >= 1 && d->dil < d->w, "conv_pair_umma: dilation must be in [1, width)");
  LAVB_CHECK_ARG(d->n >= 0 && d->h >= 1, "conv_pair_umma: bad shape");
  LAVB_CHECK_ARG(d->w1 && d->w2 && d->bias1 && d->in && d->out, "conv_pair_umma: null operand");
  LAVB_CHECK_ARG((long long)d->n * ceil_div(d->h, kBlockM / d->w) < (1LL << 31), "conv_pair_umma: more than 2^31 tiles");
  LAVB_CHECK_ARG(reinterpret_cast<uintptr_t>(d->bias1) % 4 == 0 && reinterpret_cast<uintptr_t>(d->shift2) % 4 == 0,
                 "conv_pair_umma: bias1 and shift2 must be 4 B aligned");
  {  // the residual tile is prefetched while earlier tiles are stored: `out` must not overlap `in` or `res`
    const size_t bytes = (size_t)d->n * d->h * d->w * d->c * 2;
    const auto overlap = [&](const void* x) {
      const char *o = static_cast<const char*>(d->out), *q = static_cast<const char*>(x);
      return x && o < q + bytes && q < o + bytes;
    };
    LAVB_CHECK_ARG(!overlap(d->in) && !overlap(d->res), "conv_pair_umma: out must not overlap in or res");
  }
  if (d->n == 0) return 0;
  auto encode = get_encode();
  LAVB_CHECK_ARG(encode != nullptr, "conv_pair_umma: cuTensorMapEncodeTiled not available from the driver");
  PairArgs a;
  memset(&a, 0, sizeof(a));
  a.n = d->n; a.h = d->h; a.w = d->w; a.c = d->c; a.kchunks = d->c / kBlockK; a.dil = d->dil;
  a.tile_w = d->w; a.tile_h = kBlockM / d->w;
  a.tiles_per_img = ceil_div(d->h, a.tile_h);
  a.num_tiles = d->n * a.tiles_per_img;
  a.post_relu = d->post_relu;
  a.res = reinterpret_cast<const h16*>(d->res);
  a.bias1 = d->bias1; a.shift2 = d->shift2;
  a.trace = g_pair_trace; a.trace_tiles = g_pair_trace_tiles;
  const int slot_bytes = kABytes + d->c * kBlockK * 2;
  const int mid_bytes = 3 * a.kchunks * kABytes;
  const int ctrl_bytes = 1024 /*align*/ + 16 * kMaxStages + 2 * 128 * (int)sizeof(float);
  // C = 64: TWO co-resident CTAs per SM (~113 KB of shared memory each)
  const bool two = d->c == 64;
  const int smem_cap = two ? 113 * 1024 : 227 * 1024;
  a.stages = min(kMaxStages, (smem_cap - mid_bytes - ctrl_bytes) / slot_bytes);
  const int smem = a.stages * slot_bytes + mid_bytes + ctrl_bytes;
  CUtensorMap tmap_a, tmap_w1, tmap_w2, tmap_r, tmap_o;
  // input, residual and output: one geometry, boxes of 64 channels x one tile of full rows
  const auto encode_act = [&](CUtensorMap* m, const void* ptr) {
    cuuint64_t dims[4] = {(cuuint64_t)d->c, (cuuint64_t)d->w, (cuuint64_t)d->h, (cuuint64_t)d->n};
    cuuint64_t strides[3] = {(cuuint64_t)d->c * 2, (cuuint64_t)d->w * d->c * 2, (cuuint64_t)d->h * d->w * d->c * 2};
    cuuint32_t box[4] = {(cuuint32_t)kBlockK, (cuuint32_t)a.tile_w, (cuuint32_t)a.tile_h, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    return encode(m, LAVB_TMAP_H16, 4, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  };
  CUresult r = encode_act(&tmap_a, d->in);
  LAVB_CHECK_ARG(r == CUDA_SUCCESS, "conv_pair_umma: cuTensorMapEncodeTiled(in) failed with %d", (int)r);
  r = encode_act(&tmap_r, d->res ? d->res : d->in);           // without a residual the map is never read
  LAVB_CHECK_ARG(r == CUDA_SUCCESS, "conv_pair_umma: cuTensorMapEncodeTiled(res) failed with %d", (int)r);
  r = encode_act(&tmap_o, d->out);
  LAVB_CHECK_ARG(r == CUDA_SUCCESS, "conv_pair_umma: cuTensorMapEncodeTiled(out) failed with %d", (int)r);
  for (int which = 0; which < 2; ++which) {
    cuuint64_t dims[2] = {(cuuint64_t)d->c, (cuuint64_t)3 * d->c};
    cuuint64_t strides[1] = {(cuuint64_t)d->c * 2};
    cuuint32_t box[2] = {(cuuint32_t)kBlockK, (cuuint32_t)d->c};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = encode(which ? &tmap_w2 : &tmap_w1, LAVB_TMAP_H16, 2, const_cast<void*>(which ? d->w2 : d->w1), dims,
                        strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    LAVB_CHECK_ARG(r == CUDA_SUCCESS, "conv_pair_umma: cuTensorMapEncodeTiled(W%d) failed with %d", which + 1, (int)r);
  }
  if (two) {
    LAVB_CUDA_OK(ensure_dyn_smem((const void*)conv_pair_umma_kernel<64>, smem_cap));
    conv_pair_umma_kernel<64><<<min(a.num_tiles, 2 * kNumSMs), kPairThreads, smem, (cudaStream_t)stream>>>(tmap_a, tmap_w1, tmap_w2, tmap_r, tmap_o, a);
  } else {
    LAVB_CUDA_OK(ensure_dyn_smem((const void*)conv_pair_umma_kernel<128>, smem_cap));
    conv_pair_umma_kernel<128><<<min(a.num_tiles, kNumSMs), kPairThreads, smem, (cudaStream_t)stream>>>(tmap_a, tmap_w1, tmap_w2, tmap_r, tmap_o, a);
  }
  LAVB_LAUNCH_OK();
  return 0;
}
