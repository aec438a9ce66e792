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

// torch.softmax over the c_cls logits pr[0 .. c_cls) (expf(x - max) / sum: fmaxf max, so a NaN logit is skipped by the max; sum
// in class order; IEEE division), then the background suppression of forward_paint (model_inference.py:45): o[k - 1] = p_k *
// (1 - p_0) for k = 1 .. c_cls - 1.  The one tail every kernel that paints from the logits uses, so their columns agree bit for bit.
__device__ __forceinline__ void softmax_suppress(float (&pr)[8], int c_cls, float* o) {
  float mx = pr[0];
#pragma unroll
  for (int k = 1; k < 8; ++k) if (k < c_cls) mx = fmaxf(mx, pr[k]);
  float sum = 0.f;
#pragma unroll
  for (int k = 0; k < 8; ++k) if (k < c_cls) { pr[k] = expf(pr[k] - mx); sum += pr[k]; }
#pragma unroll
  for (int k = 0; k < 8; ++k) if (k < c_cls) pr[k] = __fdiv_rn(pr[k], sum);
  const float bg = __fsub_rn(1.f, pr[0]);
#pragma unroll
  for (int k = 1; k < 8; ++k) if (k < c_cls) o[k - 1] = __fmul_rn(pr[k], bg);
}

}  // namespace lavb
