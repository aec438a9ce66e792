// Fused non_bottleneck_1d block for the 16-channel ERFNet decoder stage (lav/models/erfnet.py:37-63, Decoder layers 4-5):
//     t1 = relu(conv3x1_1(x) + b)         t2 = relu(bn1(conv1x3_1(t1) + b))
//     t3 = relu(conv3x1_2(t2) + b)        y  = relu(bn2(conv1x3_2(t3) + b) + x)          (dilation 1, Dropout2d inactive in eval)
// in ONE kernel: a CTA owns 8 output rows of one image at full width, stages the 12 input rows it needs (+-2 halo rows for the two
// vertical convs) in shared memory and runs the four convolutions there, ping-ponging between two row buffers.  Each conv tap is
// one K16 step of mma.sync m16n8k16 (16 input channels = one k-step, 16 output channels = two n-tiles); A fragments come from
// shared memory by ldmatrix.x4 (16 consecutive pixels of a row x 16 channels), the 4 x 3 x 2 weight fragments live in
// registers.  Layer by layer this stage moved every activation through HBM eight times (8 launches of conv_c16_mma, ~56 us each
// at 96 images); fused, the block reads its input once (+ halo re-reads that hit L2) and writes its output once.
//
// Shared-memory row layout: (W + 2) pixels of 32 B (one zero guard pixel on each side = the horizontal zero padding); the two
// 16-byte halves of a pixel are swapped when bit 2 of the pixel index is set, which makes both the ldmatrix row reads and the
// fragment-layout epilogue stores bank-conflict free.
#include <climits>

#include "common.cuh"

namespace lavb {

constexpr int kNbRowsOut = 8, kNbHalo = 2, kNbRows = kNbRowsOut + 2 * kNbHalo;      // 12 staged rows per tile
constexpr int kNbThreads = 256;

struct Nb16Args {
  const h16* in; h16* out;
  int n, h, w;
  const float* w4;        // [4 convs][3 taps][16 cin][16 cout] fp32
  const float* st;        // [4 convs][16 cout][2] = (scale, shift) with the conv bias folded in: epi(a) = relu(a * s + t)
};

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32." LAVB_H16_PTX "." LAVB_H16_PTX ".f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// byte offset of (pixel index incl. guard, 16-byte half) inside a buffer
__device__ __forceinline__ uint32_t px_off(int pix, int half) { return (uint32_t)pix * 32u + (uint32_t)((half ^ ((pix >> 2) & 1)) << 4); }

// One convolution stage over tile rows [row_lo, row_hi): kVert = 3x1 (taps along rows) else 1x3 (taps along columns).
// kRes: add the residual found in `dst` at the output position and write in place (dst holds x there).
template <bool kVert, bool kRes>
__device__ __forceinline__ void nb16_stage(uint32_t src, uint32_t dst, int pitch, int w, int row_lo, int row_hi, int g_row0, int h,
                                           const uint32_t (&bf)[3][2][2], const float (&st)[2][2][2], int warp, int lane) {
  const int tpr = w >> 4;                       // m16 tiles per row
  const int gq = lane >> 2, tq = lane & 3;
  const int mi = lane & 7, mj = lane >> 3;      // ldmatrix: this lane addresses row mi of matrix mj
  for (int mt = warp; mt < (row_hi - row_lo) * tpr; mt += kNbThreads / 32) {
    const int r = row_lo + mt / tpr, c0 = (mt % tpr) << 4;
    float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
#pragma unroll
    for (int tap = 0; tap < 3; ++tap) {
      const int rr = kVert ? r + tap - 1 : r, cc = kVert ? c0 : c0 + tap - 1;
      const int pix = rr * pitch + cc + mi + ((mj & 1) << 3) + 1;
      uint32_t a[4];
      ldsm_x4(src + px_off(pix, mj >> 1), a);
      mma16816(acc[0], a, bf[tap][0][0], bf[tap][0][1]);
      mma16816(acc[1], a, bf[tap][1][0], bf[tap][1][1]);
    }
    const bool inside = (unsigned)(g_row0 + r) < (unsigned)h;     // rows outside the image are the next conv's zero padding
#pragma unroll
    for (int hrow = 0; hrow < 2; ++hrow) {                        // accumulator rows gq (c[0], c[1]) and gq + 8 (c[2], c[3])
      const int pix = r * pitch + c0 + gq + 8 * hrow + 1;
#pragma unroll
      for (int nn = 0; nn < 2; ++nn) {
        const uint32_t addr = dst + px_off(pix, nn) + (uint32_t)tq * 4u;
        float v0 = fmaf(acc[nn][2 * hrow], st[nn][0][0], st[nn][0][1]), v1 = fmaf(acc[nn][2 * hrow + 1], st[nn][1][0], st[nn][1][1]);
        if (kRes) {
          uint32_t xr;
          asm volatile("ld.shared.b32 %0, [%1];" : "=r"(xr) : "r"(addr));
          const float2 xf = unpack_h16(xr);
          v0 += xf.x; v1 += xf.y;
        }
        const uint32_t o = inside ? pack_h16(fmaxf(v0, 0.f), fmaxf(v1, 0.f)) : 0u;
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(o) : "memory");
      }
    }
  }
}

__global__ void __launch_bounds__(kNbThreads, 2) erf_nb16_kernel(const __grid_constant__ Nb16Args p) {
  extern __shared__ __align__(128) uint8_t nb_sm[];
  const int pitch = p.w + 2;
  const uint32_t buf_bytes = (uint32_t)kNbRows * pitch * 32u;
  const uint32_t A = (uint32_t)__cvta_generic_to_shared(nb_sm), B = A + buf_bytes;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, gq = lane >> 2, tq = lane & 3;
  const int tiles_y = (p.h + kNbRowsOut - 1) / kNbRowsOut;
  const int img = blockIdx.x / tiles_y, ty = blockIdx.x - img * tiles_y;
  const int g_row0 = ty * kNbRowsOut - kNbHalo;             // global row of tile row 0

  // weight fragments (B operand, "col" layout): b0 = W[k = 2tq, 2tq+1][n = gq], b1 = W[k = 2tq+8, +9][n = gq] per n-tile
  uint32_t bf[4][3][2][2];
  float st[4][2][2][2];                                     // [conv][n-tile][col 2tq / 2tq+1][scale, shift]
#pragma unroll
  for (int cv = 0; cv < 4; ++cv) {
#pragma unroll
    for (int tap = 0; tap < 3; ++tap)
#pragma unroll
      for (int nn = 0; nn < 2; ++nn) {
        const float* wp = p.w4 + ((cv * 3 + tap) * 16) * 16 + nn * 8 + gq;          // [cin][cout]
        bf[cv][tap][nn][0] = pack_h16(__ldg(wp + (2 * tq) * 16), __ldg(wp + (2 * tq + 1) * 16));
        bf[cv][tap][nn][1] = pack_h16(__ldg(wp + (2 * tq + 8) * 16), __ldg(wp + (2 * tq + 9) * 16));
      }
#pragma unroll
    for (int nn = 0; nn < 2; ++nn)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float2 v = __ldg(reinterpret_cast<const float2*>(p.st) + cv * 16 + nn * 8 + 2 * tq + e);
        st[cv][nn][e][0] = v.x; st[cv][nn][e][1] = v.y;
      }
  }
  // zero both buffers' guard pixels (the stages never write them)
  for (int i = tid; i < 2 * kNbRows * 2 * 2; i += kNbThreads) {
    const int buf = i / (kNbRows * 4), rem = i % (kNbRows * 4), r = rem >> 2, side = (rem >> 1) & 1, half = rem & 1;
    const int pix = r * pitch + (side ? p.w + 1 : 0);
    asm volatile("st.shared.v4.b32 [%0], {%1, %1, %1, %1};" ::"r"((buf ? B : A) + px_off(pix, half)), "r"(0u) : "memory");
  }
  // stage 0: x rows [g_row0, g_row0 + 12) -> A (zeros outside the image)
  const h16* src_img = p.in + (size_t)img * p.h * p.w * 16;
  const int chunks_per_row = p.w * 2;
  for (int i = tid; i < kNbRows * chunks_per_row; i += kNbThreads) {
    const int r = i / chunks_per_row, c = i - r * chunks_per_row, px = c >> 1, half = c & 1;
    const int gr = g_row0 + r;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if ((unsigned)gr < (unsigned)p.h) v = __ldg(reinterpret_cast<const uint4*>(src_img + ((size_t)gr * p.w + px) * 16) + half);
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(A + px_off(r * pitch + px + 1, half)), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
  }
  __syncthreads();
  nb16_stage<true, false>(A, B, pitch, p.w, 1, kNbRows - 1, g_row0, p.h, bf[0], st[0], warp, lane);       // t1: rows 1..10
  __syncthreads();
  nb16_stage<false, false>(B, A, pitch, p.w, 1, kNbRows - 1, g_row0, p.h, bf[1], st[1], warp, lane);      // t2: rows 1..10
  __syncthreads();
  nb16_stage<true, false>(A, B, pitch, p.w, 2, kNbRows - 2, g_row0, p.h, bf[2], st[2], warp, lane);       // t3: rows 2..9
  __syncthreads();
  // the residual: x rows 2..9 back into A (L2 hits), then the last conv adds it in place
  for (int i = tid; i < kNbRowsOut * chunks_per_row; i += kNbThreads) {
    const int r = kNbHalo + i / chunks_per_row, c = i % chunks_per_row, px = c >> 1, half = c & 1;
    const int gr = g_row0 + r;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if ((unsigned)gr < (unsigned)p.h) v = __ldg(reinterpret_cast<const uint4*>(src_img + ((size_t)gr * p.w + px) * 16) + half);
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(A + px_off(r * pitch + px + 1, half)), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
  }
  __syncthreads();
  nb16_stage<false, true>(B, A, pitch, p.w, 2, kNbRows - 2, g_row0, p.h, bf[3], st[3], warp, lane);       // y: rows 2..9, in place over x
  __syncthreads();
  h16* dst_img = p.out + (size_t)img * p.h * p.w * 16;
  for (int i = tid; i < kNbRowsOut * chunks_per_row; i += kNbThreads) {
    const int r = kNbHalo + i / chunks_per_row, c = i % chunks_per_row, px = c >> 1, half = c & 1;
    const int gr = g_row0 + r;
    if ((unsigned)gr >= (unsigned)p.h) continue;
    uint4 v;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(A + px_off(r * pitch + px + 1, half)));
    *(reinterpret_cast<uint4*>(dst_img + ((size_t)gr * p.w + px) * 16) + half) = v;
  }
}


// ---------------------------------------------------------------------------------------------------------------------------------
// Fused ERFNet entry: RGBSegmentationModel.normalize + Encoder.initial_block = DownsamplerBlock(3, 16) (lav/models/rgb.py:41-45,
// erfnet.py:12-23,67): out = relu(bn(cat[conv3x3_s2_p1(x) (13 ch), maxpool2x2(x) (3 ch)])) with x = (rgb / 255 - .5) * 2, straight
// from the uint8 camera frames.  One thread = one output pixel; a block stages the 17 x 65 input pixels of its 8 x 32 output
// patch in shared memory as normalised floats (zero outside the image = the conv's zero padding in the normalised domain), the
// 27 x 13 weights and the folded BN constants come from the constant bank (kernel parameters), each thread leaves with one
// 32-byte h16 pixel.  Replaces three launches (rgb_norm, conv_small, pool2) that moved the image through HBM three times.
// ---------------------------------------------------------------------------------------------------------------------------------
struct StemW { float w[27][16]; float s[16]; float t[16]; };      // w[(ky*3+kx)*3+c][co] (co >= 13 zero); epi: relu(acc*s + t)

constexpr int kSt_OH = 8, kSt_OW = 32, kSt_IH = 2 * kSt_OH + 1, kSt_IW = 2 * kSt_OW + 1, kSt_Pitch = kSt_IW * 3 + 2;

template <typename TOut>
__global__ void __launch_bounds__(kSt_OH * kSt_OW) erf_stem_kernel(const unsigned char* __restrict__ img, int n, int h, int w,
                                                                     const __grid_constant__ StemW k, TOut* __restrict__ out) {
  __shared__ float tile[kSt_IH][kSt_Pitch];
  __shared__ float lut[256];                              // (v / 255 - .5) * 2 for the 256 byte values, in the reference's op order
  lut[threadIdx.x] = (__fdiv_rn((float)threadIdx.x, 255.f) - 0.5f) * 2.f;      // rgb.py:41 (blockDim.x == 256)
  const int ho = h >> 1, wo = w >> 1;
  const int tiles_x = (wo + kSt_OW - 1) / kSt_OW, tiles_y = (ho + kSt_OH - 1) / kSt_OH;
  const int b = blockIdx.x / (tiles_x * tiles_y), tr = blockIdx.x % (tiles_x * tiles_y);
  const int oy0 = (tr / tiles_x) * kSt_OH, ox0 = (tr % tiles_x) * kSt_OW;
  const unsigned char* src = img + (size_t)b * h * w * 3;
  const int iy0 = 2 * oy0 - 1, ix0 = 2 * ox0 - 1;
  __syncthreads();
  if (threadIdx.x < kSt_IW * 3) {                         // thread = one byte column of the staged rows (195 of the 256 threads)
    const int q = threadIdx.x, ix = ix0 + q / 3;
    const bool col_ok = (unsigned)ix < (unsigned)w;
    const unsigned char* colp = src + (size_t)ix * 3 + q % 3;
#pragma unroll
    for (int r = 0; r < kSt_IH; ++r) {
      const int iy = iy0 + r;
      tile[r][q] = (col_ok && (unsigned)iy < (unsigned)h) ? lut[__ldg(colp + (size_t)iy * w * 3)] : 0.f;
    }
  }
  __syncthreads();
  const int ly = threadIdx.x / kSt_OW, lx = threadIdx.x % kSt_OW;
  const int oy = oy0 + ly, ox = ox0 + lx;
  if (oy >= ho || ox >= wo) return;
  float acc[13];
#pragma unroll
  for (int c = 0; c < 13; ++c) acc[c] = 0.f;
#pragma unroll
  for (int ky = 0; ky < 3; ++ky)
#pragma unroll
    for (int kx = 0; kx < 3; ++kx)
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float v = tile[2 * ly + ky][(2 * lx + kx) * 3 + c];
#pragma unroll
        for (int co = 0; co < 13; ++co) acc[co] = fmaf(v, k.w[(ky * 3 + kx) * 3 + c][co], acc[co]);
      }
  float o[16];
#pragma unroll
  for (int c = 0; c < 13; ++c) o[c] = fmaxf(fmaf(acc[c], k.s[c], k.t[c]), 0.f);
#pragma unroll
  for (int c = 0; c < 3; ++c) {      // 2x2 max-pool of the normalised image: input pixels (2oy, 2ox)..(+1,+1) = tile rows 2ly+1.., cols 2lx+1..
    const float m = fmaxf(fmaxf(tile[2 * ly + 1][(2 * lx + 1) * 3 + c], tile[2 * ly + 1][(2 * lx + 2) * 3 + c]),
                          fmaxf(tile[2 * ly + 2][(2 * lx + 1) * 3 + c], tile[2 * ly + 2][(2 * lx + 2) * 3 + c]));
    o[13 + c] = fmaxf(fmaf(m, k.s[13 + c], k.t[13 + c]), 0.f);
  }
  TOut* dst = out + (((size_t)b * ho + oy) * wo + ox) * 16;
#pragma unroll
  for (int q = 0; q < 4; ++q) store4<TOut>(dst + 4 * q, make_float4(o[4 * q], o[4 * q + 1], o[4 * q + 2], o[4 * q + 3]));
}


// ---------------------------------------------------------------------------------------------------------------------------------
// Fused DownsamplerBlock(16, 64) (Encoder.layers[0], lav/models/erfnet.py:12-23,71): out = relu(bn(cat[conv3x3 s2 p1 (16 -> 48),
// maxpool2x2 (16 ch)])) on the h16 16-channel map.  A CTA produces 4 output rows x (up to) 64 output columns: it stages the 9 input
// rows it needs in shared memory split into EVEN and ODD pixel columns (tap kx = 0 reads O[x-1], kx = 1 reads E[x], kx = 2 reads
// O[x]: every tap is a stride-1 run of 16 pixels = one ldmatrix.x4), runs the 9 taps x 6 n-tiles on mma.sync with the weight
// fragments fetched from shared memory once per tap for both of a warp's m-tiles, max-pools the same staged pixels, and leaves the
// 128-byte output pixels through a shared-memory staging tile as full-line stores.  Replaces conv_c16_mma<9> (147 us at 96
// images, A fragments straight from global memory) + pool2 (33 us).
// ---------------------------------------------------------------------------------------------------------------------------------
constexpr int kDnRows = 4, kDnCols = 64, kDnInRows = 2 * kDnRows + 1, kDnPlane = kDnCols + 1;    // per row: E[0..63] | O[-1..63]
constexpr int kDnRowPix = kDnCols + kDnPlane;                                                     // 129 pixels of 32 B per staged row
constexpr int kDnThreads = 256;

struct Dn16Args {
  const h16* in; h16* out;
  int n, h, w;              // input size; output (h/2, w/2, 64)
  const float* w9;          // [9 taps (ky*3+kx)][16 cin][48 cout] fp32
  const float* st;          // [64][2] (scale, shift): relu(a*s + t), conv bias folded into the first 48 shifts
};

__global__ void __launch_bounds__(kDnThreads, 2) erf_down16_kernel(const __grid_constant__ Dn16Args p) {
  extern __shared__ __align__(128) uint8_t dn_sm[];
  const uint32_t IN = (uint32_t)__cvta_generic_to_shared(dn_sm);                    // [9 rows][129 px][32 B]
  const uint32_t WS = IN + kDnInRows * kDnRowPix * 32;                              // weights h16 [9][48 n][16 k] (B fragments: k pairs)
  const uint32_t OUT = WS + 9 * 48 * 16 * 2;                                        // [256 px][128 B] output staging
  float* stf = reinterpret_cast<float*>(dn_sm + (OUT - IN) + kDnRows * kDnCols * 128);   // [64][2]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, gq = lane >> 2, tq = lane & 3;
  const int ho = p.h >> 1, wo = p.w >> 1;
  const int tiles_y = (ho + kDnRows - 1) / kDnRows;
  const int img = blockIdx.x / tiles_y, oy0 = (blockIdx.x - img * tiles_y) * kDnRows;
  // weights -> shared memory as h16 [tap][n][k]; affine constants
  for (int e = tid; e < 9 * 48 * 16; e += kDnThreads) {
    const int tap = e / (48 * 16), r = e - tap * 48 * 16, n = r >> 4, k = r & 15;
    reinterpret_cast<h16*>(dn_sm + (WS - IN))[e] = float2h16(__ldg(p.w9 + (tap * 16 + k) * 48 + n));
  }
  for (int e = tid; e < 128; e += kDnThreads) stf[e] = __ldg(p.st + e);
  // stage the input rows 2*oy0-1 .. 2*oy0+7: pixel 2x -> E[x], pixel 2x+1 -> O[x] (O[-1] = the left zero padding)
  const h16* src = p.in + (size_t)img * p.h * p.w * 16;
  for (int e = tid; e < kDnInRows * (2 * kDnCols + 1) * 2; e += kDnThreads) {
    const int r = e / ((2 * kDnCols + 1) * 2), q = e - r * ((2 * kDnCols + 1) * 2), px = (q >> 1) - 1, half = q & 1;   // px = -1 .. 127
    const int iy = 2 * oy0 - 1 + r;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if ((unsigned)iy < (unsigned)p.h && (unsigned)px < (unsigned)p.w) v = __ldg(reinterpret_cast<const uint4*>(src + ((size_t)iy * p.w + px) * 16) + half);
    const int slot = (px & 1) ? kDnCols + ((px + 1) >> 1) : (px >> 1);              // odd px -> O plane index (px+1)/2 (O[-1] at 0); even -> E[px/2]
    const int pix = r * kDnRowPix + (px < 0 ? kDnCols : slot);
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(IN + px_off(pix, half)), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
  }
  __syncthreads();
  const int mi = lane & 7, mj = lane >> 3;
  const int n_mt = kDnRows * (kDnCols / 16);                                        // 16 m-tiles, 2 per warp
  float acc[2][6][4];
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int nn = 0; nn < 6; ++nn)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[m][nn][e] = 0.f;
#pragma unroll 1
  for (int tap = 0; tap < 9; ++tap) {
    const int ky = tap / 3, kx = tap - 3 * ky;
    uint32_t b[6][2];
#pragma unroll
    for (int nn = 0; nn < 6; ++nn) {
      const uint32_t wa = WS + (uint32_t)(((tap * 48 + nn * 8 + gq) * 16 + 2 * tq) * 2);
      asm volatile("ld.shared.b32 %0, [%1];" : "=r"(b[nn][0]) : "r"(wa));
      asm volatile("ld.shared.b32 %0, [%1];" : "=r"(b[nn][1]) : "r"(wa + 16));
    }
#pragma unroll
    for (int m = 0; m < 2; ++m) {
      const int mt = warp * 2 + m, ly = mt / (kDnCols / 16), x0 = (mt % (kDnCols / 16)) * 16;
      // input row 2*ly + ky of the staged 9; plane / first pixel by kx: O[x0-1..] (plane slots x0.., since O[-1] sits at slot 0), E[x0..], O[x0..]
      const int base = (2 * ly + ky) * kDnRowPix + (kx == 1 ? x0 : kDnCols + x0 + (kx == 2 ? 1 : 0));
      const int pix = base + mi + ((mj & 1) << 3);
      uint32_t a[4];
      ldsm_x4(IN + px_off(pix, mj >> 1), a);
#pragma unroll
      for (int nn = 0; nn < 6; ++nn) mma16816(acc[m][nn], a, b[nn][0], b[nn][1]);
    }
  }
  // conv epilogue -> staging tile (pixel = 128 B; 16-byte pieces rotated by the pixel index so fragment stores spread over the banks)
#pragma unroll
  for (int m = 0; m < 2; ++m) {
    const int mt = warp * 2 + m, ly = mt / (kDnCols / 16), x0 = (mt % (kDnCols / 16)) * 16;
#pragma unroll
    for (int hrow = 0; hrow < 2; ++hrow) {
      const int opix = ly * kDnCols + x0 + gq + 8 * hrow;
#pragma unroll
      for (int nn = 0; nn < 6; ++nn) {
        const int c = nn * 8 + 2 * tq;
        const float v0 = fmaxf(fmaf(acc[m][nn][2 * hrow], stf[2 * c], stf[2 * c + 1]), 0.f);
        const float v1 = fmaxf(fmaf(acc[m][nn][2 * hrow + 1], stf[2 * c + 2], stf[2 * c + 3]), 0.f);
        const uint32_t addr = OUT + (uint32_t)opix * 128u + (uint32_t)(((nn ^ (opix & 7)) << 4) + tq * 4);
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(pack_h16(v0, v1)) : "memory");
      }
    }
  }
  // pool branch: thread = (output pixel, 8-channel half): max over the 2x2 input pixels -> affine -> ReLU -> channels 48 + 8*half..
  for (int e = tid; e < kDnRows * kDnCols * 2; e += kDnThreads) {
    const int opix = e >> 1, half = e & 1, ly = opix / kDnCols, lx = opix - ly * kDnCols;
    float m8[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) m8[k] = -INFINITY;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        const int pix = (2 * ly + 1 + dy) * kDnRowPix + (dx ? kDnCols + lx + 1 : lx);          // E[lx] / O[lx] of input rows 2oy, 2oy+1
        uint4 v;
        asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(IN + px_off(pix, half)));
        const uint32_t w4[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) { const float2 f = unpack_h16(w4[k]); m8[2 * k] = fmaxf(m8[2 * k], f.x); m8[2 * k + 1] = fmaxf(m8[2 * k + 1], f.y); }
      }
    uint32_t o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = 48 + 8 * half + 2 * k;
      o[k] = pack_h16(fmaxf(fmaf(m8[2 * k], stf[2 * c], stf[2 * c + 1]), 0.f), fmaxf(fmaf(m8[2 * k + 1], stf[2 * c + 2], stf[2 * c + 3]), 0.f));
    }
    const uint32_t addr = OUT + (uint32_t)opix * 128u + (uint32_t)((((6 + half) ^ (opix & 7)) << 4));
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(o[0]), "r"(o[1]), "r"(o[2]), "r"(o[3]) : "memory");
  }
  __syncthreads();
  h16* dst = p.out + (size_t)img * ho * wo * 64;
  for (int e = tid; e < kDnRows * kDnCols * 8; e += kDnThreads) {
    const int opix = e >> 3, j = e & 7, ly = opix / kDnCols, lx = opix - ly * kDnCols;
    const int oy = oy0 + ly;
    if (oy >= ho || lx >= wo) continue;
    uint4 v;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(OUT + (uint32_t)opix * 128u + (uint32_t)((j ^ (opix & 7)) << 4)));
    *(reinterpret_cast<uint4*>(dst + ((size_t)oy * wo + lx) * 64) + j) = v;
  }
}

}  // namespace lavb

using namespace lavb;

extern "C" int lavb_erf_nb16(const void* d_in, void* d_out, int n, int h, int w, const float* d_w4, const float* d_st, void* stream) {
  LAVB_CHECK_ARG(n >= 0 && h >= 1 && w >= 16 && w % 16 == 0 && w <= 256, "erf_nb16: width must be a multiple of 16, <= 256 (got %d)", w);
  const int tiles_y = (h + kNbRowsOut - 1) / kNbRowsOut;
  LAVB_CHECK_ARG((long long)n * tiles_y <= INT_MAX, "erf_nb16: %d images of %d rows need more than 2^31 - 1 blocks", n, h);
  if (n == 0) return 0;
  LAVB_CHECK_ARG(d_in && d_out && d_w4 && d_st, "erf_nb16: null pointer");
  LAVB_CHECK_ARG(is_aligned(d_in, 16) && is_aligned(d_out, 16) && is_aligned(d_w4, 4) && is_aligned(d_st, 8),
                 "erf_nb16: d_in and d_out must be 16-byte, d_w4 4-byte and d_st 8-byte aligned");
  const size_t bytes = (size_t)n * h * w * 16 * sizeof(h16);
  LAVB_CHECK_ARG(!ranges_overlap(d_in, bytes, d_out, bytes), "erf_nb16: d_out overlaps d_in (halo rows of neighbouring tiles are re-read)");
  LAVB_CHECK_ARG(!ranges_overlap(d_w4, 4 * 3 * 16 * 16 * sizeof(float), d_out, bytes) && !ranges_overlap(d_st, 4 * 16 * 2 * sizeof(float), d_out, bytes),
                 "erf_nb16: d_out overlaps d_w4 or d_st (every block reads them at its start)");
  Nb16Args a;
  a.in = reinterpret_cast<const h16*>(d_in); a.out = reinterpret_cast<h16*>(d_out);
  a.n = n; a.h = h; a.w = w; a.w4 = d_w4; a.st = d_st;
  const int smem = 2 * kNbRows * (w + 2) * 32;
  LAVB_CUDA_OK(ensure_dyn_smem((const void*)erf_nb16_kernel, smem));
  erf_nb16_kernel<<<n * tiles_y, kNbThreads, smem, (cudaStream_t)stream>>>(a);
  LAVB_LAUNCH_OK();
  return 0;
}

extern "C" int lavb_erf_stem(const void* d_rgb_u8, int n, int h, int w, const float* h_w27x16, const float* h_scale16,
                             const float* h_shift16, void* d_out, int out_dtype, void* stream) {
  LAVB_CHECK_ARG(n >= 0 && h >= 2 && w >= 2 && h % 2 == 0 && w % 2 == 0, "erf_stem: image size must be even");
  LAVB_CHECK_ARG(out_dtype == LAVB_F32 || out_dtype == LAVB_H16, "erf_stem: output dtype must be fp32 or h16");
  const long long blocks = (long long)n * ceil_div(h / 2, kSt_OH) * ceil_div(w / 2, kSt_OW);
  LAVB_CHECK_ARG(blocks <= INT_MAX, "erf_stem: %d images of %d x %d need more than 2^31 - 1 blocks", n, h, w);
  if (n == 0) return 0;
  LAVB_CHECK_ARG(d_rgb_u8 && d_out && h_w27x16 && h_scale16 && h_shift16, "erf_stem: null pointer");
  const size_t esize = out_dtype == LAVB_F32 ? sizeof(float) : sizeof(h16);
  LAVB_CHECK_ARG(is_aligned(d_out, 4 * esize), "erf_stem: d_out must be %d-byte aligned", (int)(4 * esize));
  LAVB_CHECK_ARG(!ranges_overlap(d_rgb_u8, (size_t)n * h * w * 3, d_out, (size_t)n * (h / 2) * (w / 2) * 16 * esize),
                 "erf_stem: d_out overlaps d_rgb_u8");
  StemW k;
  memcpy(k.w, h_w27x16, sizeof(k.w));
  memcpy(k.s, h_scale16, sizeof(k.s));
  memcpy(k.t, h_shift16, sizeof(k.t));
  const unsigned char* img = reinterpret_cast<const unsigned char*>(d_rgb_u8);
  if (out_dtype == LAVB_F32) erf_stem_kernel<float><<<(int)blocks, kSt_OH * kSt_OW, 0, (cudaStream_t)stream>>>(img, n, h, w, k, (float*)d_out);
  else erf_stem_kernel<h16><<<(int)blocks, kSt_OH * kSt_OW, 0, (cudaStream_t)stream>>>(img, n, h, w, k, (h16*)d_out);
  LAVB_LAUNCH_OK();
  return 0;
}

extern "C" int lavb_erf_down16(const void* d_in, void* d_out, int n, int h, int w, const float* d_w9, const float* d_st, void* stream) {
  LAVB_CHECK_ARG(n >= 0 && h >= 2 && w >= 2 && h % 2 == 0 && w % 2 == 0 && w <= 2 * kDnCols, "erf_down16: even input size, width <= %d (got %d x %d)", 2 * kDnCols, h, w);
  const int tiles_y = ceil_div(h / 2, kDnRows);
  LAVB_CHECK_ARG((long long)n * tiles_y <= INT_MAX, "erf_down16: %d images of %d rows need more than 2^31 - 1 blocks", n, h);
  if (n == 0) return 0;
  LAVB_CHECK_ARG(d_in && d_out && d_w9 && d_st, "erf_down16: null pointer");
  LAVB_CHECK_ARG(is_aligned(d_in, 16) && is_aligned(d_out, 16) && is_aligned(d_w9, 4) && is_aligned(d_st, 4),
                 "erf_down16: d_in and d_out must be 16-byte, d_w9 and d_st 4-byte aligned");
  const size_t out_bytes = (size_t)n * (h / 2) * (w / 2) * 64 * sizeof(h16);
  LAVB_CHECK_ARG(!ranges_overlap(d_in, (size_t)n * h * w * 16 * sizeof(h16), d_out, out_bytes), "erf_down16: d_out overlaps d_in");
  LAVB_CHECK_ARG(!ranges_overlap(d_w9, 9 * 16 * 48 * sizeof(float), d_out, out_bytes) && !ranges_overlap(d_st, 64 * 2 * sizeof(float), d_out, out_bytes),
                 "erf_down16: d_out overlaps d_w9 or d_st (every block reads them at its start)");
  Dn16Args a;
  a.in = reinterpret_cast<const h16*>(d_in); a.out = reinterpret_cast<h16*>(d_out);
  a.n = n; a.h = h; a.w = w; a.w9 = d_w9; a.st = d_st;
  const int smem = kDnInRows * kDnRowPix * 32 + 9 * 48 * 16 * 2 + kDnRows * kDnCols * 128 + 128 * 4;
  LAVB_CUDA_OK(ensure_dyn_smem((const void*)erf_down16_kernel, smem));
  erf_down16_kernel<<<n * tiles_y, kDnThreads, smem, (cudaStream_t)stream>>>(a);
  LAVB_LAUNCH_OK();
  return 0;
}
