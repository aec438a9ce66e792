// Generic "tap-list" convolution on the CUDA cores (fp32 accumulate), NHWC.
//
// One kernel covers every Conv2d / ConvTranspose2d shape of ERFNet, the BEV backbone and the heads
// (lav/models/erfnet.py, lav/models/lidar.py): the host expresses a layer as a list of taps
// (dy,dx,weight block) over an output grid; strided convs set in_s = stride, transposed convs are
// issued once per output phase with out_s = stride.  The GEMM view is M = n*hog*wog pixels,
// N = cout, K = ntaps*cin; tiles BM x BN x 16 with a register-prefetched, double-buffered smem
// pipeline and a fused epilogue (bias, ReLU, BN affine, residual, ReLU, sigmoid).
// This is the exact-fp32 workhorse (parity path and all HBM-bound layers); the tensor-core
// layers of the h16 path live in conv_umma.cu.
#include <algorithm>
#include <type_traits>
#include "common.cuh"

namespace lavb {

struct ConvArgs {
  const void* in; void* out; const void* res;
  const float* w; const float* bias; const float* scale; const float* shift;
  int n, hin, win, cin, in_cstride, in_coff;
  int hout, wout, cout, cout_pad, out_cstride, out_coff;
  int hog, wog, in_sy, in_sx, out_sy, out_sx, out_oy, out_ox;
  int res_cstride, res_coff;
  int ntaps;
  int dy[16], dx[16];
  int pre_relu, post_relu, sigmoid;
  int rows_pb;   // conv_c16_mma_kernel: output-grid rows each block walks (amortises its weight/epilogue preamble)
};

constexpr int BK = 16;

template <typename TIn, typename TOut, int BM, int BN, int TM, int NH>
__global__ void __launch_bounds__((BM / TM) * (BN / (4 * NH))) conv_taps_kernel(const __grid_constant__ ConvArgs a) {
  constexpr int TXN = BN / (4 * NH);       // threads along channels
  constexpr int NT = (BM / TM) * TXN;      // threads per block
  constexpr int PPT = BM / NT;             // pixels each thread stages per k-step
  constexpr int BV4 = BK * BN / 4;         // float4 in one B stage
  constexpr int BV = (BV4 + NT - 1) / NT;  // float4 of B each thread stages per k-step
  static_assert(BM % NT == 0, "tile/threads mismatch");
  __shared__ __align__(16) float As[2][BK][BM];
  __shared__ __align__(16) float Bs[2][BK][BN];

  const int tid = threadIdx.x;
  const int tx = tid % TXN, ty = tid / TXN;
  const long long M = (long long)a.n * a.hog * a.wog;
  const long long m0 = (long long)blockIdx.x * BM;
  const int co0 = blockIdx.y * BN;

  // pixels this thread stages
  int pn[PPT], py[PPT], px[PPT];
  bool pv[PPT];
#pragma unroll
  for (int i = 0; i < PPT; ++i) {
    const long long m = m0 + tid + i * NT;
    pv[i] = m < M;
    const long long mm = pv[i] ? m : 0;
    const int hw = a.hog * a.wog;
    pn[i] = (int)(mm / hw);
    const int r = (int)(mm - (long long)pn[i] * hw);
    py[i] = (r / a.wog) * a.in_sy;
    px[i] = (r % a.wog) * a.in_sx;
  }
  const TIn* in = reinterpret_cast<const TIn*>(a.in);
  const int kchunks = (a.cin + BK - 1) / BK;
  const int nk = a.ntaps * kchunks;

  float4 ra[PPT][4];
  float4 rb[BV];

  auto load_stage = [&](int kit) {
    const int t = kit / kchunks, ci0 = (kit - t * kchunks) * BK;
#pragma unroll
    for (int i = 0; i < PPT; ++i) {
      const int iy = py[i] + a.dy[t], ix = px[i] + a.dx[t];
      const bool ok = pv[i] && iy >= 0 && iy < a.hin && ix >= 0 && ix < a.win;
      const TIn* p = in + (((long long)pn[i] * a.hin + iy) * a.win + ix) * a.in_cstride + a.in_coff + ci0;
#pragma unroll
      for (int q = 0; q < 4; ++q)
        ra[i][q] = (ok && ci0 + q * 4 < a.cin) ? load4<TIn>(p + q * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int v = 0; v < BV; ++v) {
      const int idx = tid + v * NT;            // float4 index inside the BK x BN tile
      const int kk = idx / (BN / 4), c4 = idx % (BN / 4);
      const int ci = ci0 + kk;
      rb[v] = (idx < BV4 && ci < a.cin) ? __ldg(reinterpret_cast<const float4*>(a.w + ((long long)t * a.cin + ci) * a.cout_pad + co0) + c4)
                           : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto store_stage = [&](int buf) {
#pragma unroll
    for (int i = 0; i < PPT; ++i) {
      const int m = tid + i * NT;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        As[buf][q * 4 + 0][m] = ra[i][q].x; As[buf][q * 4 + 1][m] = ra[i][q].y;
        As[buf][q * 4 + 2][m] = ra[i][q].z; As[buf][q * 4 + 3][m] = ra[i][q].w;
      }
    }
#pragma unroll
    for (int v = 0; v < BV; ++v) {
      const int idx = tid + v * NT;
      const int kk = idx / (BN / 4), c4 = idx % (BN / 4);
      if (idx < BV4) *reinterpret_cast<float4*>(&Bs[buf][kk][c4 * 4]) = rb[v];
    }
  };

  float acc[TM][4 * NH];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < 4 * NH; ++j) acc[i][j] = 0.f;

  load_stage(0);
  store_stage(0);
  __syncthreads();
  for (int kit = 0; kit < nk; ++kit) {
    const int buf = kit & 1;
    if (kit + 1 < nk) load_stage(kit + 1);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float av[TM], bv[4 * NH];
#pragma unroll
      for (int i = 0; i < TM; i += 4) {
        const float4 t4 = *reinterpret_cast<const float4*>(&As[buf][k][ty * TM + i]);
        av[i] = t4.x; av[i + 1] = t4.y; av[i + 2] = t4.z; av[i + 3] = t4.w;
      }
#pragma unroll
      for (int h = 0; h < NH; ++h) {
        const float4 t4 = *reinterpret_cast<const float4*>(&Bs[buf][k][h * (BN / NH) + tx * 4]);
        bv[h * 4] = t4.x; bv[h * 4 + 1] = t4.y; bv[h * 4 + 2] = t4.z; bv[h * 4 + 3] = t4.w;
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < 4 * NH; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (kit + 1 < nk) store_stage(buf ^ 1);
    __syncthreads();
  }

  // ---- epilogue
  TOut* out = reinterpret_cast<TOut*>(a.out);
  const TOut* res = reinterpret_cast<const TOut*>(a.res);
  const bool vec_ok = (a.cout % 4 == 0) && (a.out_coff % 4 == 0) && (a.out_cstride % 4 == 0) &&
                      (res == nullptr || (a.res_coff % 4 == 0 && a.res_cstride % 4 == 0));
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const long long m = m0 + ty * TM + i;
    if (m >= M) continue;
    const int hw = a.hog * a.wog;
    const int nn = (int)(m / hw);
    const int r = (int)(m - (long long)nn * hw);
    const int oy = (r / a.wog) * a.out_sy + a.out_oy, ox = (r % a.wog) * a.out_sx + a.out_ox;
    if (oy >= a.hout || ox >= a.wout) continue;
    const long long pix = ((long long)nn * a.hout + oy) * a.wout + ox;
#pragma unroll
    for (int h = 0; h < NH; ++h) {
      const int co = co0 + h * (BN / NH) + tx * 4;
      if (co >= a.cout) continue;
      float v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = co + j;
        float x = acc[i][h * 4 + j];
        if (c < a.cout) {
          if (a.bias) x += __ldg(a.bias + c);
          if (a.pre_relu) x = fmaxf(x, 0.f);
          if (a.scale) x = fmaf(x, __ldg(a.scale + c), __ldg(a.shift + c));
        }
        v[j] = x;
      }
      if (vec_ok) {
        if (res) {
          const float4 rr = load4<TOut>(res + pix * a.res_cstride + a.res_coff + co);
          v[0] += rr.x; v[1] += rr.y; v[2] += rr.z; v[3] += rr.w;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (a.post_relu) v[j] = fmaxf(v[j], 0.f);
          if (a.sigmoid) v[j] = 1.f / (1.f + expf(-v[j]));
        }
        store4<TOut>(out + pix * a.out_cstride + a.out_coff + co, make_float4(v[0], v[1], v[2], v[3]));
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int c = co + j;
          if (c >= a.cout) continue;
          float x = v[j];
          if (res) x += to_f32<TOut>(res[pix * a.res_cstride + a.res_coff + c]);
          if (a.post_relu) x = fmaxf(x, 0.f);
          if (a.sigmoid) x = 1.f / (1.f + expf(-x));
          out[pix * a.out_cstride + a.out_coff + c] = from_f32<TOut>(x);
        }
      }
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(256) pool2_vec4_kernel(const T* __restrict__ in, int n, int hin, int win, int c, int in_cstride,
                                                         int in_coff, const float* __restrict__ scale,
                                                         const float* __restrict__ shift, T* __restrict__ out, int out_cstride,
                                                         int out_coff) {
  const int ho = hin / 2, wo = win / 2, c4 = c / 4;
  const long long total = (long long)n * ho * wo * c4;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int ch = (int)(i % c4) * 4;
  long long p = i / c4;
  const int ox = (int)(p % wo); p /= wo;
  const int oy = (int)(p % ho);
  const int nn = (int)(p / ho);
  const T* s = in + (((long long)nn * hin + oy * 2) * win + ox * 2) * in_cstride + in_coff + ch;
  const float4 a = load4<T>(s), b = load4<T>(s + in_cstride), cc = load4<T>(s + (long long)win * in_cstride),
               d = load4<T>(s + (long long)(win + 1) * in_cstride);
  const float4 sc = __ldg(reinterpret_cast<const float4*>(scale + ch)), sh = __ldg(reinterpret_cast<const float4*>(shift + ch));
  float4 y;
  y.x = fmaxf(fmaf(fmaxf(fmaxf(a.x, b.x), fmaxf(cc.x, d.x)), sc.x, sh.x), 0.f);
  y.y = fmaxf(fmaf(fmaxf(fmaxf(a.y, b.y), fmaxf(cc.y, d.y)), sc.y, sh.y), 0.f);
  y.z = fmaxf(fmaf(fmaxf(fmaxf(a.z, b.z), fmaxf(cc.z, d.z)), sc.z, sh.z), 0.f);
  y.w = fmaxf(fmaf(fmaxf(fmaxf(a.w, b.w), fmaxf(cc.w, d.w)), sc.w, sh.w), 0.f);
  store4<T>(out + (((long long)nn * ho + oy) * wo + ox) * out_cstride + out_coff + ch, y);
}

template <typename T>
__global__ void __launch_bounds__(256) pool2_kernel(const T* __restrict__ in, int n, int hin, int win, int c, int in_cstride,
                                                    int in_coff, const float* __restrict__ scale,
                                                    const float* __restrict__ shift, T* __restrict__ out, int out_cstride,
                                                    int out_coff) {
  const int ho = hin / 2, wo = win / 2;
  const long long total = (long long)n * ho * wo * c;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int ch = (int)(i % c);
  long long p = i / c;
  const int ox = (int)(p % wo); p /= wo;
  const int oy = (int)(p % ho);
  const int nn = (int)(p / ho);
  const T* s = in + (((long long)nn * hin + oy * 2) * win + ox * 2) * in_cstride + in_coff + ch;
  const float v = fmaxf(fmaxf(to_f32<T>(s[0]), to_f32<T>(s[in_cstride])),
                        fmaxf(to_f32<T>(s[(long long)win * in_cstride]), to_f32<T>(s[(long long)(win + 1) * in_cstride])));
  const float y = fmaxf(fmaf(v, __ldg(scale + ch), __ldg(shift + ch)), 0.f);
  out[(((long long)nn * ho + oy) * wo + ox) * out_cstride + out_coff + ch] = from_f32<T>(y);
}

// ---- small-channel direct convolution (cin <= 16): one thread per output-grid pixel, 16 output channels per pass.
// The GEMM tiling above wastes its K loop on these layers (ERFNet's 3->13 / 16->48 entry convs, the 16-channel decoder
// blocks and the 16->5 output ConvT, erfnet.py:67-71,116-124); they are pure HBM streams: coalesced 32-64 B per
// thread in, same out, weights broadcast from shared memory.
template <typename TIn, typename TOut, int CIN>
__global__ void __launch_bounds__(256) conv_small_kernel(const __grid_constant__ ConvArgs a) {
  extern __shared__ __align__(16) float wsm[];   // [ntaps][CIN][16] for the current cout chunk
  const int co0 = blockIdx.y * 16;
  for (int i = threadIdx.x; i < a.ntaps * CIN * 16; i += blockDim.x) {
    const int t = i / (CIN * 16), r = i - t * CIN * 16, ci = r / 16, co = r % 16;
    wsm[i] = (ci < a.cin) ? __ldg(a.w + ((long long)t * a.cin + ci) * a.cout_pad + co0 + co) : 0.f;
  }
  __syncthreads();
  const long long M = (long long)a.n * a.hog * a.wog;
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  const int hw = a.hog * a.wog;
  const int nn = (int)(m / hw);
  const int r = (int)(m - (long long)nn * hw);
  const int gy = r / a.wog, gx = r % a.wog;
  const TIn* in = reinterpret_cast<const TIn*>(a.in);
  float acc[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) acc[j] = 0.f;
  for (int t = 0; t < a.ntaps; ++t) {
    const int iy = gy * a.in_sy + a.dy[t], ix = gx * a.in_sx + a.dx[t];
    if (iy < 0 || iy >= a.hin || ix < 0 || ix >= a.win) continue;
    const TIn* p = in + (((long long)nn * a.hin + iy) * a.win + ix) * a.in_cstride + a.in_coff;
    float xv[CIN];
#pragma unroll
    for (int c = 0; c < CIN; c += 4) {
      const float4 v = (c < a.cin) ? load4<TIn>(p + c) : make_float4(0.f, 0.f, 0.f, 0.f);
      xv[c] = v.x; xv[c + 1] = v.y; xv[c + 2] = v.z; xv[c + 3] = v.w;
    }
    const float4* wt = reinterpret_cast<const float4*>(wsm + (size_t)t * CIN * 16);
#pragma unroll
    for (int c = 0; c < CIN; ++c) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 w = wt[c * 4 + q];
        acc[q * 4] = fmaf(xv[c], w.x, acc[q * 4]); acc[q * 4 + 1] = fmaf(xv[c], w.y, acc[q * 4 + 1]);
        acc[q * 4 + 2] = fmaf(xv[c], w.z, acc[q * 4 + 2]); acc[q * 4 + 3] = fmaf(xv[c], w.w, acc[q * 4 + 3]);
      }
    }
  }
  const int oy = gy * a.out_sy + a.out_oy, ox = gx * a.out_sx + a.out_ox;
  if (oy >= a.hout || ox >= a.wout) return;
  const long long pix = ((long long)nn * a.hout + oy) * a.wout + ox;
  TOut* out = reinterpret_cast<TOut*>(a.out) + pix * a.out_cstride + a.out_coff;
  const TOut* res = a.res ? reinterpret_cast<const TOut*>(a.res) + pix * a.res_cstride + a.res_coff : nullptr;
  const bool vec_ok = (a.cout % 4 == 0) && (a.out_coff % 4 == 0) && (a.out_cstride % 4 == 0) &&
                      (res == nullptr || (a.res_coff % 4 == 0 && a.res_cstride % 4 == 0));
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int co = co0 + q * 4;
    if (co >= a.cout) break;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = co + j;
      float x = acc[q * 4 + j];
      if (c < a.cout) {
        if (a.bias) x += __ldg(a.bias + c);
        if (a.pre_relu) x = fmaxf(x, 0.f);
        if (a.scale) x = fmaf(x, __ldg(a.scale + c), __ldg(a.shift + c));
        if (res && !vec_ok) x += to_f32<TOut>(res[c]);
      }
      v[j] = x;
    }
    if (vec_ok) {
      if (res) { const float4 rr = load4<TOut>(res + co); v[0] += rr.x; v[1] += rr.y; v[2] += rr.z; v[3] += rr.w; }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (a.post_relu) v[j] = fmaxf(v[j], 0.f);
        if (a.sigmoid) v[j] = 1.f / (1.f + expf(-v[j]));
      }
      store4<TOut>(out + co, make_float4(v[0], v[1], v[2], v[3]));
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (co + j >= a.cout) continue;
        float x = v[j];
        if (a.post_relu) x = fmaxf(x, 0.f);
        if (a.sigmoid) x = 1.f / (1.f + expf(-x));
        out[co + j] = from_f32<TOut>(x);
      }
    }
  }
}

// ---- 16-input-channel layers on the tensor cores (h16 path): one tap = one K16 step of mma.sync m16n8k16.
// ERFNet's 16-channel decoder blocks, the 16->48 downsampler conv and the 16->5 output ConvT (erfnet.py:71,121-124) are
// FFMA-bound in conv_small_kernel (768 FMA per pixel); here a warp owns 32 output pixels, the A fragment of a tap is
// loaded straight from global memory (a pixel's 16 channels are 32 contiguous bytes = exactly one fragment row), the
// weights of a 16-wide output chunk live in registers as B fragments, and the epilogue is the usual fused one.
__device__ __forceinline__ void mma_16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32." LAVB_H16_PTX "." LAVB_H16_PTX ".f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

template <typename TOut, int NTAPS>
__global__ void __launch_bounds__(128) conv_c16_mma_kernel(const __grid_constant__ ConvArgs a) {
  // grid: x = (image, group of rows_pb output-grid rows), y = 128-pixel segment of a row, z = 16-column chunk -> no per-pixel
  // div/mod; the weight fragments and epilogue constants are built once and reused for every row of the group
  const int lane = threadIdx.x & 31, gq = lane >> 2, tq = lane & 3;
  const int co0 = blockIdx.z * 16;
  const int groups = (a.hog + a.rows_pb - 1) / a.rows_pb;
  const int img = blockIdx.x / groups, gy_begin = (blockIdx.x - img * groups) * a.rows_pb;
  const int gy_end = min(gy_begin + a.rows_pb, a.hog);
  const int gx0 = blockIdx.y * 128 + (threadIdx.x >> 5) * 32;
  if (gx0 >= a.wog) return;
  // B fragments of this 16-column chunk: b0 = W[tap][k = 2tq, 2tq+1][n = 8nn + gq], b1 = same with k + 8
  uint32_t bf[NTAPS][2][2];
#pragma unroll
  for (int t = 0; t < NTAPS; ++t)
#pragma unroll
    for (int nn = 0; nn < 2; ++nn)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float* wp = a.w + ((long long)t * 16 + (2 * tq + 8 * h)) * a.cout_pad + co0 + nn * 8 + gq;
        const h162 b2 = floats2h162(t < a.ntaps ? __ldg(wp) : 0.f, t < a.ntaps ? __ldg(wp + a.cout_pad) : 0.f);
        bf[t][nn][h] = *reinterpret_cast<const uint32_t*>(&b2);
      }
  float e_bias[2][2], e_scale[2][2], e_shift[2][2];
#pragma unroll
  for (int nn = 0; nn < 2; ++nn)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int c = co0 + nn * 8 + 2 * tq + e;
      const bool in_range = c < a.cout;
      e_bias[nn][e] = (a.bias && in_range) ? __ldg(a.bias + c) : 0.f;
      e_scale[nn][e] = (a.scale && in_range) ? __ldg(a.scale + c) : 1.f;
      e_shift[nn][e] = (a.shift && in_range) ? __ldg(a.shift + c) : 0.f;
    }
  const bool pair_ok = (a.out_coff % 2 == 0) && (a.out_cstride % 2 == 0) && (a.res == nullptr || (a.res_coff % 2 == 0 && a.res_cstride % 2 == 0));
  const h16* in = reinterpret_cast<const h16*>(a.in) + (long long)img * a.hin * a.win * a.in_cstride + a.in_coff + 2 * tq;
  // the 4 pixels this lane touches: rows gq, gq+8 of both m-tiles
  int gx[4]; bool pv[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) { gx[r] = gx0 + (r >> 1) * 16 + (r & 1) * 8 + gq; pv[r] = gx[r] < a.wog; }
#pragma unroll 1
  for (int gy = gy_begin; gy < gy_end; ++gy) {
  float acc[2][2][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nn = 0; nn < 2; ++nn) acc[mt][nn][0] = acc[mt][nn][1] = acc[mt][nn][2] = acc[mt][nn][3] = 0.f;
#pragma unroll
  for (int t = 0; t < NTAPS; ++t) {
    if (t < a.ntaps) {
      const int iy = gy * a.in_sy + a.dy[t];
      const bool row_ok = iy >= 0 && iy < a.hin;
      const h16* rowp = in + (long long)iy * a.win * a.in_cstride;
      uint32_t af[4][2];
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int ix = gx[r] * a.in_sx + a.dx[t];
        const bool ok = row_ok && pv[r] && ix >= 0 && ix < a.win;
        const uint32_t* p = reinterpret_cast<const uint32_t*>(rowp + (long long)ix * a.in_cstride);
        af[r][0] = ok ? __ldg(p) : 0u;        // channels 2tq, 2tq+1
        af[r][1] = ok ? __ldg(p + 4) : 0u;    // channels 2tq+8, 2tq+9
      }
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nn = 0; nn < 2; ++nn)
          mma_16816(acc[mt][nn], af[mt * 2][0], af[mt * 2 + 1][0], af[mt * 2][1], af[mt * 2 + 1][1], bf[t][nn][0], bf[t][nn][1]);
    }
  }
  // epilogue: C fragment = (row gq | gq+8, cols 8nn + 2tq, +1); the lane's 4 columns' parameters sit in registers
  const int oy = gy * a.out_sy + a.out_oy;
  if (oy >= a.hout) continue;
  TOut* orow = reinterpret_cast<TOut*>(a.out) + ((long long)img * a.hout + oy) * a.wout * a.out_cstride + a.out_coff;
  const TOut* rrow = a.res ? reinterpret_cast<const TOut*>(a.res) + ((long long)img * a.hout + oy) * a.wout * a.res_cstride + a.res_coff : nullptr;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int ox = gx[r] * a.out_sx + a.out_ox;
    if (!pv[r] || ox >= a.wout) continue;
    TOut* op = orow + (long long)ox * a.out_cstride;
    const TOut* rp = rrow ? rrow + (long long)ox * a.res_cstride : nullptr;
#pragma unroll
    for (int nn = 0; nn < 2; ++nn) {
      const int c = co0 + nn * 8 + 2 * tq;
      if (c >= a.cout) continue;
      float x0 = acc[r >> 1][nn][(r & 1) * 2] + e_bias[nn][0], x1 = acc[r >> 1][nn][(r & 1) * 2 + 1] + e_bias[nn][1];
      // each step only when its flag / pointer is set, as in the other bodies: fmaxf(NaN, -inf) would turn a NaN into -inf
      if (a.pre_relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
      if (a.scale) { x0 = fmaf(x0, e_scale[nn][0], e_shift[nn][0]); x1 = fmaf(x1, e_scale[nn][1], e_shift[nn][1]); }
      const bool pair = pair_ok && (c + 1 < a.cout);
      if (rp) {
        if (pair) { const float2 rr = load2<TOut>(rp + c); x0 += rr.x; x1 += rr.y; }
        else { x0 += to_f32<TOut>(rp[c]); if (c + 1 < a.cout) x1 += to_f32<TOut>(rp[c + 1]); }
      }
      if (a.post_relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
      if (a.sigmoid) { x0 = 1.f / (1.f + expf(-x0)); x1 = 1.f / (1.f + expf(-x1)); }
      if (pair) store2<TOut>(op + c, x0, x1);
      else { op[c] = from_f32<TOut>(x0); if (c + 1 < a.cout) op[c + 1] = from_f32<TOut>(x1); }
    }
  }
  }   // row loop
}

template <typename TIn, typename TOut>
static int launch_conv(ConvArgs& a, cudaStream_t st) {
  const long long M = (long long)a.n * a.hog * a.wog;
  if constexpr (std::is_same<TIn, h16>::value) {
    if (a.cin == 16 && a.ntaps <= 9 && a.in_coff % 2 == 0 && a.in_cstride % 2 == 0) {   // tensor-core path for 16-channel layers
      // rows per block: as many as keeps >= ~16 blocks per SM in flight, at most 8
      const long long row_blocks = (long long)a.n * a.hog * ceil_div(a.wog, 128) * (a.cout_pad / 16);
      a.rows_pb = (int)std::max<long long>(1, std::min<long long>(8, row_blocks / (kNumSMs * 16)));
      dim3 grid(a.n * ceil_div(a.hog, a.rows_pb), ceil_div(a.wog, 128), a.cout_pad / 16);
      if (a.ntaps <= 3) conv_c16_mma_kernel<TOut, 3><<<grid, 128, 0, st>>>(a);
      else if (a.ntaps <= 4) conv_c16_mma_kernel<TOut, 4><<<grid, 128, 0, st>>>(a);
      else conv_c16_mma_kernel<TOut, 9><<<grid, 128, 0, st>>>(a);
      LAVB_LAUNCH_OK();
      return 0;
    }
  }
  if (a.cin <= 16) {
    dim3 grid(ceil_div(M, 256), a.cout_pad / 16);
    const size_t smem = (size_t)a.ntaps * 16 * 16 * sizeof(float);
    if (a.cin <= 4) conv_small_kernel<TIn, TOut, 4><<<grid, 256, (size_t)a.ntaps * 4 * 16 * sizeof(float), st>>>(a);
    else conv_small_kernel<TIn, TOut, 16><<<grid, 256, smem, st>>>(a);
    LAVB_LAUNCH_OK();
    return 0;
  }
  if (a.cout_pad % 64 == 0) {
    dim3 grid(ceil_div(M, 128), a.cout_pad / 64);
    conv_taps_kernel<TIn, TOut, 128, 64, 8, 2><<<grid, 128, 0, st>>>(a);
  } else {
    dim3 grid(ceil_div(M, 256), a.cout_pad / 16);
    conv_taps_kernel<TIn, TOut, 256, 16, 8, 1><<<grid, 128, 0, st>>>(a);
  }
  LAVB_LAUNCH_OK();
  return 0;
}

}  // namespace lavb

using namespace lavb;

extern "C" int lavb_conv_taps(const lavb_conv_desc* d, void* stream) {
  LAVB_CHECK_ARG(d != nullptr, "conv_taps: null descriptor");
  LAVB_CHECK_ARG(d->ntaps >= 1 && d->ntaps <= 16, "conv_taps: ntaps must be 1..16 (got %d)", d->ntaps);
  LAVB_CHECK_ARG(d->cin % 4 == 0 && d->in_coff % 4 == 0 && d->in_cstride % 4 == 0,
                 "conv_taps: cin/in_coff/in_cstride must be multiples of 4 (got %d/%d/%d)", d->cin, d->in_coff, d->in_cstride);
  LAVB_CHECK_ARG(d->cin >= 4, "conv_taps: cin must be >= 4 (got %d)", d->cin);
  LAVB_CHECK_ARG(d->in_coff >= 0 && d->out_coff >= 0 && d->in_coff + d->cin <= d->in_cstride && d->out_coff + d->cout <= d->out_cstride,
                 "conv_taps: channel slice out of range");
  LAVB_CHECK_ARG(d->res == nullptr || (d->res_coff >= 0 && d->res_coff + d->cout <= d->res_cstride),
                 "conv_taps: residual channel slice out of range");
  LAVB_CHECK_ARG((d->scale == nullptr) == (d->shift == nullptr), "conv_taps: scale and shift come together");
  LAVB_CHECK_ARG(d->n > 0 && d->hog > 0 && d->wog > 0 && d->cout > 0, "conv_taps: empty problem");
  LAVB_CHECK_ARG(d->hin >= 1 && d->win >= 1 && d->hout >= 1 && d->wout >= 1, "conv_taps: map sizes must be >= 1");
  LAVB_CHECK_ARG(d->in_sy >= 1 && d->in_sx >= 1 && d->out_sy >= 1 && d->out_sx >= 1 && d->out_oy >= 0 && d->out_ox >= 0,
                 "conv_taps: strides must be >= 1 and output offsets >= 0");
  LAVB_CHECK_ARG(d->in != nullptr && d->out != nullptr && d->w != nullptr, "conv_taps: null in / out / w");
  // the bodies move 4 channels at a time (float4 / 4 x h16) from these base pointers; bias / scale / shift are read per element
  const uintptr_t in_al = d->in_dtype == LAVB_F32 ? 16 : 8, out_al = d->out_dtype == LAVB_F32 ? 16 : 8;
  LAVB_CHECK_ARG(reinterpret_cast<uintptr_t>(d->in) % in_al == 0 && reinterpret_cast<uintptr_t>(d->out) % out_al == 0 &&
                     reinterpret_cast<uintptr_t>(d->res) % out_al == 0 && reinterpret_cast<uintptr_t>(d->w) % 16 == 0 &&
                     reinterpret_cast<uintptr_t>(d->bias) % 4 == 0 && reinterpret_cast<uintptr_t>(d->scale) % 4 == 0 &&
                     reinterpret_cast<uintptr_t>(d->shift) % 4 == 0,
                 "conv_taps: in / out / res must be 4-element aligned (16 B fp32, 8 B 16-bit), w 16-byte aligned");
  ConvArgs a;
  a.in = d->in; a.out = d->out; a.res = d->res; a.w = d->w; a.bias = d->bias; a.scale = d->scale; a.shift = d->shift;
  a.n = d->n; a.hin = d->hin; a.win = d->win; a.cin = d->cin; a.in_cstride = d->in_cstride; a.in_coff = d->in_coff;
  a.hout = d->hout; a.wout = d->wout; a.cout = d->cout; a.cout_pad = (d->cout + 15) / 16 * 16;
  a.out_cstride = d->out_cstride; a.out_coff = d->out_coff;
  a.hog = d->hog; a.wog = d->wog; a.in_sy = d->in_sy; a.in_sx = d->in_sx; a.out_sy = d->out_sy; a.out_sx = d->out_sx;
  a.out_oy = d->out_oy; a.out_ox = d->out_ox; a.res_cstride = d->res_cstride; a.res_coff = d->res_coff;
  a.ntaps = d->ntaps;
  for (int t = 0; t < 16; ++t) { a.dy[t] = d->dy[t]; a.dx[t] = d->dx[t]; }
  a.pre_relu = d->pre_relu; a.post_relu = d->post_relu; a.sigmoid = d->sigmoid;
  LAVB_CHECK_ARG(d->res == nullptr || d->res_dtype == d->out_dtype, "conv_taps: residual dtype must equal output dtype");
  cudaStream_t st = (cudaStream_t)stream;
  if (d->in_dtype == LAVB_F32 && d->out_dtype == LAVB_F32) return launch_conv<float, float>(a, st);
  if (d->in_dtype == LAVB_H16 && d->out_dtype == LAVB_H16) return launch_conv<h16, h16>(a, st);
  if (d->in_dtype == LAVB_F32 && d->out_dtype == LAVB_H16) return launch_conv<float, h16>(a, st);
  if (d->in_dtype == LAVB_H16 && d->out_dtype == LAVB_F32) return launch_conv<h16, float>(a, st);
  LAVB_CHECK_ARG(false, "conv_taps: unsupported dtype combination");
}

extern "C" int lavb_pool2_affine_relu(const void* d_in, int dtype, int n, int hin, int win, int c, int in_cstride, int in_coff,
                                      const float* d_scale, const float* d_shift, void* d_out, int out_cstride, int out_coff,
                                      void* stream) {
  LAVB_CHECK_ARG(dtype == LAVB_F32 || dtype == LAVB_H16, "pool2: bad dtype");
  LAVB_CHECK_ARG(n >= 0 && hin >= 0 && win >= 0 && c >= 1, "pool2: n, hin, win must be >= 0 and c >= 1");
  LAVB_CHECK_ARG(hin % 2 == 0 && win % 2 == 0, "pool2: odd input size");
  LAVB_CHECK_ARG(in_coff >= 0 && in_coff + c <= in_cstride && out_coff >= 0 && out_coff + c <= out_cstride,
                 "pool2: channel slice out of range");
  const long long total = (long long)n * (hin / 2) * (win / 2) * c;
  if (total == 0) return 0;
  const uintptr_t esz = dtype == LAVB_F32 ? 4 : 2;
  LAVB_CHECK_ARG(d_in != nullptr && d_out != nullptr && d_scale != nullptr && d_shift != nullptr, "pool2: null pointer");
  LAVB_CHECK_ARG(reinterpret_cast<uintptr_t>(d_in) % esz == 0 && reinterpret_cast<uintptr_t>(d_out) % esz == 0 &&
                     reinterpret_cast<uintptr_t>(d_scale) % 4 == 0 && reinterpret_cast<uintptr_t>(d_shift) % 4 == 0,
                 "pool2: pointers must be aligned to their element size");
  cudaStream_t st = (cudaStream_t)stream;
  // the vector body moves 4 channels at a time: it needs 4-element aligned maps and 16-byte aligned scale / shift
  const bool vec = c % 4 == 0 && in_cstride % 4 == 0 && in_coff % 4 == 0 && out_cstride % 4 == 0 && out_coff % 4 == 0 &&
                   reinterpret_cast<uintptr_t>(d_in) % (4 * esz) == 0 && reinterpret_cast<uintptr_t>(d_out) % (4 * esz) == 0 &&
                   (reinterpret_cast<uintptr_t>(d_scale) % 16 == 0) && (reinterpret_cast<uintptr_t>(d_shift) % 16 == 0);
  if (vec && dtype == LAVB_F32) {
    pool2_vec4_kernel<float><<<ceil_div(total / 4, 256), 256, 0, st>>>((const float*)d_in, n, hin, win, c, in_cstride, in_coff, d_scale,
                                                                        d_shift, (float*)d_out, out_cstride, out_coff);
  } else if (vec && dtype == LAVB_H16) {
    pool2_vec4_kernel<h16><<<ceil_div(total / 4, 256), 256, 0, st>>>((const h16*)d_in, n, hin, win, c, in_cstride,
                                                                                in_coff, d_scale, d_shift, (h16*)d_out,
                                                                                out_cstride, out_coff);
  } else if (dtype == LAVB_F32)
    pool2_kernel<float><<<ceil_div(total, 256), 256, 0, st>>>((const float*)d_in, n, hin, win, c, in_cstride, in_coff, d_scale,
                                                               d_shift, (float*)d_out, out_cstride, out_coff);
  else
    pool2_kernel<h16><<<ceil_div(total, 256), 256, 0, st>>>((const h16*)d_in, n, hin, win, c, in_cstride,
                                                                       in_coff, d_scale, d_shift, (h16*)d_out,
                                                                       out_cstride, out_coff);
  LAVB_LAUNCH_OK();
  return 0;
}
