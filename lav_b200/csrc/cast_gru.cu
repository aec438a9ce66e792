// Motion-forecast ("cast") heads of UniPlanner / BEVPlanner in one launch (team_code_v2/models/uniplanner.py:286-301,
// lav/models/bev_planner_v2.py:226-236): for each of the 6 command branches
//     out, _ = nn.GRU(512, 64, batch_first=True)(embd repeated T times);  locs = cumsum(nn.Linear(64, 2)(out), dim=1)
// The reference (and cuDNN under it) runs 6 GRUs x T steps of tiny GEMM + cell kernels plus 6 Linear + 6 cumsum launches per call
// — ~100 dependent launches, 0.29 ms per tick whatever the batch.  Here a block owns 16 sequences of one branch for the whole
// roll-out, in fp32 FFMA (the matrices are tiny: W_hh is 48 KB):
//   phase 1  gi[16][192] = embd . W_ih^T + b_ih            (the input is the same at every step, so this is done once)
//   per step gh = h . W_hh^T + b_hh  ->  PyTorch gate math (r, z, n; n = tanh(gi_n + r * gh_n); h' = (1 - z) n + z h)
//            -> loc += W_mlp h' + b_mlp  ->  out[n][branch][t][:]
// thread = gate column (192 threads): it reads the TRANSPOSED weight matrices (the host packs them once) so that consecutive
// threads read consecutive floats, and the hidden state from shared memory as a broadcast.
#include "common.cuh"

namespace lavb {

constexpr int kCgIn = 512, kCgH = 64, kCgCols = 192, kCgSeq = 16;

struct __align__(16) CastSmem {
  float whh[kCgH][kCgCols];        // W_hh^T
  float gi[kCgSeq][kCgCols];
  float gh[kCgSeq][kCgCols];
  float h[kCgSeq][kCgH];
  float x[kCgSeq][kCgIn];          // the block's embeddings
  float wm[2][kCgH];
};

__device__ __forceinline__ float cg_sigmoid(float v) { return 1.f / (1.f + expf(-v)); }

__global__ void __launch_bounds__(kCgCols) cast_gru_kernel(const float* __restrict__ embd, int n, const float* __restrict__ wih_t,
                                                           const float* __restrict__ whh_t, const float* __restrict__ bih,
                                                           const float* __restrict__ bhh, const float* __restrict__ wmlp,
                                                           const float* __restrict__ bmlp, int ncmd, int steps, float* __restrict__ out) {
  extern __shared__ __align__(16) uint8_t cg_raw[];
  CastSmem& sm = *reinterpret_cast<CastSmem*>(cg_raw);
  const int cmd = blockIdx.y, s0 = blockIdx.x * kCgSeq, c = threadIdx.x;
  const float* wi = wih_t + (long long)cmd * kCgIn * kCgCols;      // [512][192]
  const float* wh = whh_t + (long long)cmd * kCgH * kCgCols;       // [64][192]
  for (int i = c; i < kCgH * kCgCols; i += kCgCols) (&sm.whh[0][0])[i] = __ldg(wh + i);
  for (int i = c; i < kCgSeq * kCgIn; i += kCgCols) {
    const int s = i / kCgIn, k = i - s * kCgIn;
    sm.x[s][k] = (s0 + s < n) ? __ldg(embd + (long long)(s0 + s) * kCgIn + k) : 0.f;
  }
  for (int i = c; i < 2 * kCgH; i += kCgCols) (&sm.wm[0][0])[i] = __ldg(wmlp + cmd * 2 * kCgH + i);
  for (int i = c; i < kCgSeq * kCgH; i += kCgCols) (&sm.h[0][0])[i] = 0.f;       // nn.GRU's default initial state
  __syncthreads();
  // ---- phase 1: input projection of column c for the 16 sequences
  {
    float acc[kCgSeq];
    const float b = __ldg(bih + cmd * kCgCols + c);
#pragma unroll
    for (int s = 0; s < kCgSeq; ++s) acc[s] = b;
    for (int k = 0; k < kCgIn; k += 4) {            // 4 k per pass: the embeddings come as broadcast LDS.128
      const float w0 = __ldg(wi + k * kCgCols + c), w1 = __ldg(wi + (k + 1) * kCgCols + c), w2 = __ldg(wi + (k + 2) * kCgCols + c),
                  w3 = __ldg(wi + (k + 3) * kCgCols + c);
#pragma unroll
      for (int s = 0; s < kCgSeq; ++s) {
        const float4 x4 = *reinterpret_cast<const float4*>(&sm.x[s][k]);
        acc[s] = fmaf(x4.w, w3, fmaf(x4.z, w2, fmaf(x4.y, w1, fmaf(x4.x, w0, acc[s]))));
      }
    }
#pragma unroll
    for (int s = 0; s < kCgSeq; ++s) sm.gi[s][c] = acc[s];
  }
  const float bh = __ldg(bhh + cmd * kCgCols + c);
  // threads 0..31 carry the running waypoint of (sequence c >> 1, coordinate c & 1)
  float loc = 0.f;
  const float bm = c < 2 * kCgSeq ? __ldg(bmlp + cmd * 2 + (c & 1)) : 0.f;
  for (int t = 0; t < steps; ++t) {
    __syncthreads();                                 // h (and, the first time, gi) complete
    {
      float acc[kCgSeq];
#pragma unroll
      for (int s = 0; s < kCgSeq; ++s) acc[s] = bh;
#pragma unroll 4
      for (int j = 0; j < kCgH; j += 4) {
        const float w0 = sm.whh[j][c], w1 = sm.whh[j + 1][c], w2 = sm.whh[j + 2][c], w3 = sm.whh[j + 3][c];
#pragma unroll
        for (int s = 0; s < kCgSeq; ++s) {
          const float4 h4 = *reinterpret_cast<const float4*>(&sm.h[s][j]);
          acc[s] = fmaf(h4.w, w3, fmaf(h4.z, w2, fmaf(h4.y, w1, fmaf(h4.x, w0, acc[s]))));
        }
      }
#pragma unroll
      for (int s = 0; s < kCgSeq; ++s) sm.gh[s][c] = acc[s];
    }
    __syncthreads();
    for (int i = c; i < kCgSeq * kCgH; i += kCgCols) {
      const int s = i >> 6, j = i & 63;
      const float r = cg_sigmoid(sm.gi[s][j] + sm.gh[s][j]);
      const float z = cg_sigmoid(sm.gi[s][kCgH + j] + sm.gh[s][kCgH + j]);
      const float nn_ = tanhf(fmaf(r, sm.gh[s][2 * kCgH + j], sm.gi[s][2 * kCgH + j]));
      sm.h[s][j] = fmaf(z, sm.h[s][j] - nn_, nn_);                 // (1 - z) n + z h
    }
    __syncthreads();
    if (c < 2 * kCgSeq) {
      const int s = c >> 1, o = c & 1;
      float v = bm;
#pragma unroll 8
      for (int j = 0; j < kCgH; ++j) v = fmaf(sm.wm[o][j], sm.h[s][j], v);
      loc += v;                                                     // torch.cumsum over the steps
      if (s0 + s < n) out[(((long long)(s0 + s) * ncmd + cmd) * steps + t) * 2 + o] = loc;
    }
  }
}

}  // namespace lavb

using namespace lavb;

extern "C" int lavb_cast_gru(const float* d_embd, int n, const float* d_wih_t, const float* d_whh_t, const float* d_bih,
                             const float* d_bhh, const float* d_wmlp, const float* d_bmlp, int ncmd, int steps, float* d_out,
                             void* stream) {
  LAVB_CHECK_ARG(n >= 0 && ncmd >= 1 && ncmd <= 65535 && steps >= 1, "cast_gru: bad shape (n %d, ncmd %d, steps %d)", n, ncmd, steps);
  if (n == 0) return 0;
  const float* ins[7] = {d_embd, d_wih_t, d_whh_t, d_bih, d_bhh, d_wmlp, d_bmlp};
  const size_t in_floats[7] = {(size_t)n * kCgIn, (size_t)ncmd * kCgIn * kCgCols, (size_t)ncmd * kCgH * kCgCols, (size_t)ncmd * kCgCols,
                               (size_t)ncmd * kCgCols, (size_t)ncmd * 2 * kCgH, (size_t)ncmd * 2};
  LAVB_CHECK_ARG(d_out != nullptr, "cast_gru: null pointer (out)");
  LAVB_CHECK_ARG(is_aligned(d_out, 4), "cast_gru: out must be 4-byte aligned");
  const size_t out_bytes = (size_t)n * ncmd * steps * 2 * sizeof(float);
  for (int a = 0; a < 7; ++a) {
    LAVB_CHECK_ARG(ins[a] != nullptr, "cast_gru: null pointer (input %d)", a);
    LAVB_CHECK_ARG(is_aligned(ins[a], 4), "cast_gru: input %d must be 4-byte aligned", a);
    LAVB_CHECK_ARG(!ranges_overlap(d_out, out_bytes, ins[a], in_floats[a] * sizeof(float)), "cast_gru: out overlaps input %d", a);
  }
  LAVB_CUDA_OK(ensure_dyn_smem((const void*)cast_gru_kernel, (int)sizeof(CastSmem)));
  const dim3 grid(ceil_div(n, kCgSeq), ncmd);
  cast_gru_kernel<<<grid, kCgCols, sizeof(CastSmem), (cudaStream_t)stream>>>(d_embd, n, d_wih_t, d_whh_t, d_bih, d_bhh, d_wmlp, d_bmlp, ncmd,
                                                                              steps, d_out);
  LAVB_LAUNCH_OK();
  return 0;
}
