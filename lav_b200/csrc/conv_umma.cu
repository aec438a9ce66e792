// wgmma / TMA implicit-GEMM tap-list convolution (h16 in, fp32 accumulate in registers).
//
// GEMM view of one CTA tile: M = 128 output-grid pixels (an 8 x 16 spatial patch), N = cout (<= 256, padded to 32),
// K = ntaps * cin walked in blocks of 64 channels.  No im2col buffer exists anywhere: for tap (dy,dx) the
// A operand of a K-block is ONE 4-D TMA box {64 ch, 16 px, 8 rows, 1 image} of the NHWC activation tensor whose
// start coordinate is shifted by the tap offset (out-of-bounds rows/columns are zero-filled by TMA, which IS the
// conv padding); with SWIZZLE_128B the box lands in shared memory exactly in the K-major layout wgmma reads
// (128 rows x 128 B).  Strided convs use the tensor map's element strides; a transposed conv is issued per output
// phase with its own tap list (same host packing as conv_taps.cu).
//
// Warp roles (288 threads, persistent over tiles):
//   warps 0-3, 4-7: two consumer warpgroups, one per 64-pixel half of the tile (tile rows 0-3 / 4-7).  Each issues ONE
//                   m64 x N x k16 wgmma per K16 step over its half of the A block and the whole B block (N = cout_mma, so
//                   the A fragment is read from shared memory once per step, not once per 32 columns), keeps one K-block
//                   of MMAs in flight, and runs the epilogue (bias / BN affine / ReLU / residual / sigmoid) from its registers.
//   warp 8         : TMA producer (one lane) — smem ring of `stages` {A 16 KB, B cout*128 B}
// Layers with cout <= 128 run two CTAs per SM so that one CTA's epilogue overlaps the other's MMAs.
#include "sm90.cuh"

namespace lavb {

constexpr int kTileH = 8, kTileW = 16, kBlockM = 128, kBlockK = 64;
constexpr int kABytes = kBlockM * kBlockK * 2;  // 16 KB
constexpr int kMaxStages = 8;
constexpr int kMaxTaps = 16;
constexpr int kConvThreads = 288;

struct ConvArgs {
  int n, hog, wog, tiles_x, tiles_y, num_tiles;
  int hout, wout, cin, cout, kchunks, ntaps, stages;
  int in_sy, in_sx, out_sy, out_sx, out_oy, out_ox;
  int out_cstride, out_coff, out_is_f32, res_cstride, res_coff;
  int pre_bias, pre_relu, post_relu, sigmoid, d2s_nout, cout_store;
  int dy[kMaxTaps], dx[kMaxTaps];
  void* out; const h16* res;
  const float* bias; const float* scale; const float* shift;
};

using namespace sm90;

// kNC = cout_mma / 32 (the MMA width in 32-column chunks)
template <int kNC>
__global__ void __launch_bounds__(kConvThreads, kNC <= 4 ? 2 : 1) conv_umma_kernel(const __grid_constant__ CUtensorMap tmap_a,
                                                                                 const __grid_constant__ CUtensorMap tmap_b,
                                                                                 const __grid_constant__ ConvArgs p) {
  constexpr int kN = 32 * kNC;
  constexpr int kBBytes = kN * kBlockK * 2;
  constexpr int kStageBytes = kABytes + kBBytes;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;   // SWIZZLE_128B operands need 1024 B alignment
  uint8_t* gen = smem_raw + (base - smem_u32(smem_raw));
  const uint32_t ctrl = base + p.stages * kStageBytes;
  const uint32_t full_bar = ctrl, empty_bar = ctrl + 8 * kMaxStages;
  float* ep_bias = reinterpret_cast<float*>(gen + (ctrl - base) + 16 * kMaxStages);   // only read when pre_bias
  float* ep_st = ep_bias + 256;                                                       // interleaved (scale, shift) per channel

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_a)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap_b)) : "memory");
    // empty: one arrival per consumer warp once its MMAs have read the slot
    for (int s = 0; s < p.stages; ++s) { mbar_init(full_bar + 8 * s, 1); mbar_init(empty_bar + 8 * s, 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int c = threadIdx.x; c < kN; c += blockDim.x) {
    // epi(a) = max(a + b, 0) * s + t with the pre-ReLU.  Without it the bias folds into the shift: (a + b) s + t = a s + (b s + t)
    const bool real = c < p.cout_store;      // columns past cout_store are MMA padding (never stored)
    const float b = (p.bias && real) ? __ldg(p.bias + c) : 0.f;
    const float sc = (p.scale && real) ? __ldg(p.scale + c) : 1.f;
    const float sh = (p.shift && real) ? __ldg(p.shift + c) : 0.f;
    ep_bias[c] = b;
    ep_st[2 * c] = sc;
    ep_st[2 * c + 1] = p.pre_bias ? sh : fmaf(b, sc, sh);
  }
  __syncthreads();
  const int nkb = p.ntaps * p.kchunks;
  const int tiles_per_img = p.tiles_x * p.tiles_y;

  if (warp == 8) {
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const int img = tile / tiles_per_img, r = tile - img * tiles_per_img;
        const int y0 = (r / p.tiles_x) * kTileH * p.in_sy, x0 = (r % p.tiles_x) * kTileW * p.in_sx;
        for (int t = 0; t < p.ntaps; ++t) {
          for (int kc = 0; kc < p.kchunks; ++kc) {
            mbar_wait(empty_bar + 8 * stage, phase ^ 1);
            const uint32_t sa = base + stage * kStageBytes;
            mbar_expect_tx(full_bar + 8 * stage, kStageBytes);
            tma_load_4d(sa, &tmap_a, full_bar + 8 * stage, kc * kBlockK, x0 + p.dx[t], y0 + p.dy[t], img);
            tma_load_2d(sa + kABytes, &tmap_b, full_bar + 8 * stage, kc * kBlockK, t * kN);
            if (++stage == p.stages) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
    return;
  }

  const int wg = warp >> 2;                        // tile rows [64 wg, 64 wg + 64)
  int stage = 0; uint32_t phase = 0;
  float acc[16 * kNC];                             // 32-column chunk c: acc[16c .. 16c+15]
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    int prev_stage = -1;
    for (int kb = 0; kb < nkb; ++kb) {
      mbar_wait(full_bar + 8 * stage, phase);
      const uint32_t sa = base + stage * kStageBytes;
      const uint64_t a_desc = sm90::desc_sw128(sa + wg * (kABytes / 2)), b_desc = sm90::desc_sw128(sa + kABytes);
      sm90::wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBlockK / 16; ++k)       // +32 B per K16 step inside the 128 B swizzle atom; one MMA over all kN columns
        sm90::wgmma<kN>(acc, a_desc + (uint64_t)(2 * k), b_desc + (uint64_t)(2 * k), (kb | k) ? 1u : 0u);
      sm90::wgmma_commit();
      sm90::wgmma_wait<1>();                             // the previous K-block's MMAs are done: its slot may be refilled
      if (prev_stage >= 0 && lane == 0) mbar_arrive(empty_bar + 8 * prev_stage);
      prev_stage = stage;
      if (++stage == p.stages) { stage = 0; phase ^= 1; }
    }
    sm90::wgmma_wait<0>();
    sm90::acc_fence(acc);
    if (prev_stage >= 0 && lane == 0) mbar_arrive(empty_bar + 8 * prev_stage);

    // ---- epilogue: this thread holds rows m and m + 8 of the tile, columns 8 j + c0 (+1) of every 8-column group j.
    // Every per-column offset below is the compile-time 8 j on top of a per-thread base, so no column index is kept live
    // in registers across tiles next to the 16 kNC accumulators.
    const int c0 = 2 * (lane & 3), store_lim = p.cout_store - c0;
    const int img = tile / tiles_per_img, r = tile - img * tiles_per_img;
    // tile row m = 64 wg + 16 (warp & 3) + (lane >> 2) + 8 h is grid pixel (row 4 wg + (warp & 3), column (lane >> 2) + 8 h)
    const int gy = (r / p.tiles_x) * kTileH + 4 * wg + (warp & 3), oy = gy * p.out_sy + p.out_oy;
    if (!(gy < p.hog && oy < p.hout)) continue;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int gx = (r % p.tiles_x) * kTileW + (lane >> 2) + 8 * h, ox = gx * p.out_sx + p.out_ox;
      if (!(gx < p.wog && ox < p.wout)) continue;
      const long long pix = ((long long)img * p.hout + oy) * p.wout + ox;
      uint8_t* out_at = reinterpret_cast<uint8_t*>(p.out) + (pix * p.out_cstride + p.out_coff + c0) * (p.out_is_f32 ? 4 : 2);
      const h16* res_at = p.res ? p.res + pix * p.res_cstride + p.res_coff + c0 : nullptr;
      const float* bias_at = ep_bias + c0;
      const float* st_at = ep_st + 2 * c0;
#pragma unroll
      for (int j = 0; j < 4 * kNC; ++j) {
        const int g = 8 * j;                         // column = g + c0
        float x0 = acc[4 * j + 2 * h], x1 = acc[4 * j + 2 * h + 1];
        if (p.pre_bias) { x0 += bias_at[g]; x1 += bias_at[g + 1]; }
        const float4 st = *reinterpret_cast<const float4*>(st_at + 2 * g);   // (s0, t0, s1, t1)
        // each max only when its flag is set, as in conv_taps.cu: fmaxf(NaN, -inf) would turn a NaN into -inf
        if (p.pre_relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
        x0 = fmaf(x0, st.x, st.y);
        x1 = fmaf(x1, st.z, st.w);
        if (res_at) {
          const float2 rv = unpack_h16(__ldg(reinterpret_cast<const uint32_t*>(res_at + g)));
          x0 += rv.x; x1 += rv.y;
        }
        if (p.post_relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
        if (p.sigmoid) { x0 = 1.f / (1.f + expf(-x0)); x1 = 1.f / (1.f + expf(-x1)); }
        if (kNC == 1 && p.d2s_nout) {   // depth-to-space (cout 32 only): column q = pos*nout + k -> pixel (oy + pos/2, ox + pos%2), channel k
          float* ob = reinterpret_cast<float*>(p.out);
          const int no = p.d2s_nout;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int q = g + c0 + e;
            if (q < 4 * no) {
              const int pos = q / no, k = q - pos * no;
              // each of the four pixels is clipped to hout x wout on its own (oy < hout, ox < wout hold already)
              if (oy + (pos >> 1) < p.hout && ox + (pos & 1) < p.wout)
                ob[(pix + (long long)(pos >> 1) * p.wout + (pos & 1)) * no + k] = e ? x1 : x0;
            }
          }
        } else if (g < store_lim) {                  // g + c0 < cout_store
          if (p.out_is_f32)
            *reinterpret_cast<float2*>(out_at + 4 * g) = make_float2(x0, x1);
          else
            *reinterpret_cast<uint32_t*>(out_at + 2 * g) = pack_h16(x0, x1);
        }
      }
    }
  }
}

}  // namespace lavb

using namespace lavb;

extern "C" int lavb_conv_umma(const lavb_conv_desc* d, void* stream) {
  LAVB_CHECK_ARG(d != nullptr, "conv_umma: null descriptor");
  LAVB_CHECK_ARG(d->in_dtype == LAVB_H16, "conv_umma: input must be h16");
  LAVB_CHECK_ARG(d->out_dtype == LAVB_H16 || d->out_dtype == LAVB_F32, "conv_umma: bad output dtype");
  LAVB_CHECK_ARG(d->ntaps >= 1 && d->ntaps <= kMaxTaps, "conv_umma: ntaps must be 1..16");
  LAVB_CHECK_ARG(d->cin % 64 == 0 && d->cin > 0, "conv_umma: cin must be a multiple of 64 (got %d)", d->cin);
  LAVB_CHECK_ARG(d->cout % 8 == 0 && d->cout >= 8 && d->cout <= 256, "conv_umma: cout must be 8..256, multiple of 8 (got %d)", d->cout);
  const int cout_mma = (d->cout + 31) / 32 * 32;      // MMA width; d->w holds cout_mma rows per tap (zero rows past cout)
  LAVB_CHECK_ARG(d->res == nullptr || cout_mma == d->cout, "conv_umma: residual needs cout %% 32 == 0");
  LAVB_CHECK_ARG(d->in_cstride % 8 == 0 && d->in_coff % 8 == 0 && d->in_coff >= 0 && d->in_coff + d->cin <= d->in_cstride,
                 "conv_umma: input slice misaligned or out of range");
  LAVB_CHECK_ARG(d->out_cstride % 8 == 0 && d->out_coff % 8 == 0 && d->out_coff >= 0 && d->out_coff + d->cout <= d->out_cstride,
                 "conv_umma: output slice misaligned or out of range");
  LAVB_CHECK_ARG(d->res == nullptr || (d->res_dtype == LAVB_H16 && d->res_cstride % 8 == 0 && d->res_coff % 8 == 0 && d->res_coff >= 0 &&
                                       d->res_coff + d->cout <= d->res_cstride),
                 "conv_umma: residual must be h16, its slice 16 B aligned and inside res_cstride");
  LAVB_CHECK_ARG((d->scale == nullptr) == (d->shift == nullptr), "conv_umma: scale and shift come together");
  LAVB_CHECK_ARG(d->n >= 1 && d->hog >= 1 && d->wog >= 1, "conv_umma: empty problem");
  LAVB_CHECK_ARG(d->hin >= 1 && d->win >= 1 && d->hout >= 1 && d->wout >= 1, "conv_umma: map sizes must be >= 1");
  LAVB_CHECK_ARG(d->in_sy >= 1 && d->in_sy <= 8 && d->in_sx >= 1 && d->in_sx <= 8, "conv_umma: bad input stride");
  LAVB_CHECK_ARG(d->out_sy >= 1 && d->out_sx >= 1 && d->out_oy >= 0 && d->out_ox >= 0, "conv_umma: bad output stride or offset");
  // the output lattice's coordinates and the tile count are ints in the kernel
  LAVB_CHECK_ARG((long long)(d->hog - 1) * d->out_sy + d->out_oy < (1LL << 31) && (long long)(d->wog - 1) * d->out_sx + d->out_ox < (1LL << 31),
                 "conv_umma: output lattice past 2^31");
  LAVB_CHECK_ARG((long long)d->n * ceil_div(d->hog, kTileH) * ceil_div(d->wog, kTileW) < (1LL << 31), "conv_umma: more than 2^31 tiles");
  LAVB_CHECK_ARG(d->in != nullptr && d->out != nullptr && d->w != nullptr, "conv_umma: null in / out / w");
  // TMA reads in and w; the epilogue stores up to 8 B (fp32 pairs) and reads 4 B residual pairs and 4 B bias / scale / shift
  const auto al = [](const void* q, int a) { return reinterpret_cast<uintptr_t>(q) % a == 0; };
  LAVB_CHECK_ARG(al(d->in, 16) && al(d->out, 16) && al(d->w, 16) && al(d->res, 16), "conv_umma: in, out, w and res must be 16 B aligned");
  LAVB_CHECK_ARG(al(d->bias, 4) && al(d->scale, 4) && al(d->shift, 4), "conv_umma: bias, scale and shift must be 4 B aligned");
  {  // every tile reads in and w while others store: out must not overlap them.  out may be res itself, element for element
     // (each thread reads a residual pair before it stores the same output pair); any other overlap with res is refused
    const long long px = (long long)d->n * d->hout * d->wout;
    const long long out_bytes = px * (d->d2s_nout ? 4LL * d->d2s_nout : (long long)d->out_cstride * (d->out_dtype == LAVB_F32 ? 4 : 2));
    const auto overlap = [&](const void* q, long long bytes) {
      const char *o = static_cast<const char*>(d->out), *c = static_cast<const char*>(q);
      return q && o < c + bytes && c < o + out_bytes;
    };
    LAVB_CHECK_ARG(!overlap(d->in, (long long)d->n * d->hin * d->win * d->in_cstride * 2) &&
                   !overlap(d->w, (long long)d->ntaps * ((d->cout + 31) / 32 * 32) * d->cin * 2),
                   "conv_umma: out must not overlap in or w");
    const bool same = d->res == d->out && d->out_dtype == LAVB_H16 && d->res_cstride == d->out_cstride && d->res_coff == d->out_coff;
    LAVB_CHECK_ARG(same || !overlap(d->res, px * d->res_cstride * 2), "conv_umma: out may only overlap res element for element");
  }
  auto encode = get_encode();
  LAVB_CHECK_ARG(encode != nullptr, "conv_umma: cuTensorMapEncodeTiled not available from the driver");

  CUtensorMap tmap_a, tmap_b;
  {
    const h16* in = reinterpret_cast<const h16*>(d->in) + d->in_coff;
    cuuint64_t dims[4] = {(cuuint64_t)d->cin, (cuuint64_t)d->win, (cuuint64_t)d->hin, (cuuint64_t)d->n};
    cuuint64_t strides[3] = {(cuuint64_t)d->in_cstride * 2, (cuuint64_t)d->win * d->in_cstride * 2,
                             (cuuint64_t)d->hin * d->win * d->in_cstride * 2};
    cuuint32_t box[4] = {(cuuint32_t)kBlockK, (cuuint32_t)(kTileW * d->in_sx), (cuuint32_t)(kTileH * d->in_sy), 1};
    cuuint32_t estr[4] = {1, (cuuint32_t)d->in_sx, (cuuint32_t)d->in_sy, 1};
    CUresult r = encode(&tmap_a, LAVB_TMAP_H16, 4, const_cast<h16*>(in), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    LAVB_CHECK_ARG(r == CUDA_SUCCESS, "conv_umma: cuTensorMapEncodeTiled(A) failed with %d", (int)r);
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)d->cin, (cuuint64_t)d->ntaps * cout_mma};
    cuuint64_t strides[1] = {(cuuint64_t)d->cin * 2};
    cuuint32_t box[2] = {(cuuint32_t)kBlockK, (cuuint32_t)cout_mma};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = encode(&tmap_b, LAVB_TMAP_H16, 2, const_cast<float*>(d->w), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    LAVB_CHECK_ARG(r == CUDA_SUCCESS, "conv_umma: cuTensorMapEncodeTiled(B) failed with %d", (int)r);
  }
  ConvArgs a;
  memset(&a, 0, sizeof(a));
  a.n = d->n; a.hog = d->hog; a.wog = d->wog;
  a.tiles_x = ceil_div(d->wog, kTileW); a.tiles_y = ceil_div(d->hog, kTileH);
  a.num_tiles = a.n * a.tiles_x * a.tiles_y;
  a.hout = d->hout; a.wout = d->wout; a.cin = d->cin; a.cout = cout_mma; a.cout_store = d->cout; a.kchunks = d->cin / kBlockK;
  a.ntaps = d->ntaps;
  const int nc = cout_mma / 32;
  const bool two_per_sm = nc <= 4;                    // narrow layers: 2 CTAs / SM, each with half the shared memory
  const int stage_bytes = kABytes + cout_mma * kBlockK * 2;
  const int ctrl_bytes = 1024 /*align*/ + 16 * kMaxStages + 3 * 256 * (int)sizeof(float);
  const int smem_cap = two_per_sm ? 113 * 1024 : 227 * 1024;
  a.stages = min(kMaxStages, (smem_cap - ctrl_bytes) / stage_bytes);
  a.in_sy = d->in_sy; a.in_sx = d->in_sx; a.out_sy = d->out_sy; a.out_sx = d->out_sx; a.out_oy = d->out_oy; a.out_ox = d->out_ox;
  a.out_cstride = d->out_cstride; a.out_coff = d->out_coff; a.out_is_f32 = d->out_dtype == LAVB_F32;
  a.res_cstride = d->res_cstride; a.res_coff = d->res_coff;
  a.pre_bias = d->pre_relu && d->bias != nullptr;
  a.pre_relu = d->pre_relu; a.post_relu = d->post_relu; a.sigmoid = d->sigmoid; a.d2s_nout = d->d2s_nout;
  if (d->d2s_nout) {
    LAVB_CHECK_ARG(d->cout == 32 && d->d2s_nout >= 1 && 4 * d->d2s_nout <= 32 && d->out_dtype == LAVB_F32 && d->out_sy == 2 &&
                   d->out_sx == 2 && d->res == nullptr, "conv_umma: depth-to-space epilogue needs cout=32, fp32 out, out_s=2, no residual");
  }
  for (int t = 0; t < d->ntaps; ++t) { a.dy[t] = d->dy[t]; a.dx[t] = d->dx[t]; }
  a.out = d->out; a.res = reinterpret_cast<const h16*>(d->res);
  a.bias = d->bias; a.scale = d->scale; a.shift = d->shift;
  if (a.num_tiles == 0) return 0;
  const int smem = a.stages * stage_bytes + ctrl_bytes;
  const int grid = min(a.num_tiles, two_per_sm ? 2 * kNumSMs : kNumSMs);
#define LAVB_CONV_LAUNCH(NC)                                                                                              \
  case NC: {                                                                                                              \
    /* once per (variant, device), never during a later stream capture (callers warm up first) */                         \
    LAVB_CUDA_OK(ensure_dyn_smem((const void*)conv_umma_kernel<NC>, smem_cap));                                          \
    conv_umma_kernel<NC><<<grid, kConvThreads, smem, (cudaStream_t)stream>>>(tmap_a, tmap_b, a);                          \
    break;                                                                                                                \
  }
  switch (nc) {
    LAVB_CONV_LAUNCH(1) LAVB_CONV_LAUNCH(2) LAVB_CONV_LAUNCH(3) LAVB_CONV_LAUNCH(4)
    LAVB_CONV_LAUNCH(5) LAVB_CONV_LAUNCH(6) LAVB_CONV_LAUNCH(7) LAVB_CONV_LAUNCH(8)
  }
#undef LAVB_CONV_LAUNCH
  LAVB_LAUNCH_OK();
  return 0;
}
