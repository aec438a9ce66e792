// ERFNet's last layer, Decoder.output_conv = ConvTranspose2d(16, C, 2, stride 2) (lav/models/erfnet.py:122-124,132), at one output
// pixel: the one arithmetic every kernel that reads the decoder's 16-channel map uses, so their logits agree bit for bit.
#pragma once
#include "common.cuh"

namespace lavb {

struct DeconvW { float w[2][2][16][8]; float bias[8]; };      // [v%2][u%2][c_in][k]  (k < c_cls <= 8), ops.pack_deconv2x2

// the 16 features of one half-resolution pixel (16-byte aligned for fp32, 8-byte for h16) -> fv
template <typename TF>
__device__ __forceinline__ void load_feat16(const TF* f, float (&fv)[16]) {
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float4 t = load4<TF>(f + 4 * q);
    fv[4 * q] = t.x; fv[4 * q + 1] = t.y; fv[4 * q + 2] = t.z; fv[4 * q + 3] = t.w;
  }
}

// logits[k](v, u) = bias[k], then fmaf(feat[c], W[c][k][v%2][u%2], .) over c = 0..15 in order, for k < NK (pr[k >= NK] untouched)
template <int NK>
__device__ __forceinline__ void deconv_logits(const DeconvW& dw, const float (&fv)[16], int pv, int pu, float (&pr)[8]) {
  const float (*wk)[8] = dw.w[pv][pu];
#pragma unroll
  for (int k = 0; k < NK; ++k) {
    float acc = dw.bias[k];
#pragma unroll
    for (int c = 0; c < 16; ++c) acc = fmaf(fv[c], wk[c][k], acc);
    pr[k] = acc;
  }
}

}  // namespace lavb
