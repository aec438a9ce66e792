// Detection decode, device part (extract_peak of team_code_v2/model_inference.py:189-202 + the map reads of
// det_inference :100-112): sigmoid -> 7x7 max-pool NMS -> top-k -> gather size / orientation at the peaks.
// The reference builds the full NMS map and runs a 102400-wide top-k per class; only local maxima above the score
// threshold can survive the host filter (`s > min_score`), so here every pixel above the threshold checks its own 7x7
// window (rare), survivors are appended to a short candidate list, and one block per (frame, class) selects the
// max_det best.  Output layout = InferModel.pack_peaks: [B][7][ncls*max_det] = score | flat index | w | h | cos | sin | W.
//
// A pixel is a candidate when it is not suppressed (nothing in its 7x7 window is larger, the window maximum propagating
// NaN as max_pool2d does) and its score is > min_score in fp32, or is NaN (torch.topk ranks NaN first, so a NaN takes a
// slot of the reference's top-k).  Candidates rank NaN first, then by descending score, ties to the lower flat index.
#include <climits>

#include "common.cuh"

namespace lavb {

constexpr int kCandCap = 8192;   // candidates listed per (frame, class); past it the select block rescans the map instead

__device__ __forceinline__ float sigmoidf_ref(float x) { return 1.f / (1.f + expf(-x)); }   // torch.sigmoid, fp32
__device__ __forceinline__ float fmax_nan(float a, float b) {                               // NaN wins, as in max_pool2d
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
// candidate (as, al) ranks ahead of (bs, bl): NaN first (among NaNs the lower flat index), then descending score, then
// the lower flat index
__device__ __forceinline__ bool ahead(float as, int al, float bs, int bl) {
  const bool an = isnan(as), bn = isnan(bs);
  if (an || bn) return an && (!bn || al < bl);
  return as > bs || (as == bs && al < bl);
}
__device__ __forceinline__ bool passes(float s, float min_score) { return s > min_score || isnan(s); }

// Tile kernel: a 32x32 pixel tile (+3 halo) of one class is turned into sigmoid values in shared memory, the 7x7
// window maximum is built separably (7-wide row max, then 7-high column max) and a pixel is a peak when nothing in its
// window is larger — exactly max_pool2d(heat, 7, 1, 3) followed by `max_cls > heat` (ties of saturated values all count).
constexpr int kPT = 32, kPH = 3, kPW = kPT + 2 * kPH;      // 38

__global__ void __launch_bounds__(256) peak_candidates_kernel(const float* __restrict__ center, int B, int H, int W, int ncls,
                                                              float min_score, int* __restrict__ counts,
                                                              float2* __restrict__ cand) {
  __shared__ float sv[kPW][kPW + 1];      // sigmoid values, -inf outside the map (max_pool2d pads with -inf)
  __shared__ float rm[kPW][kPT + 1];      // row-wise 7-max for the 32 centre columns
  const int tiles_x = (W + kPT - 1) / kPT, tiles_y = (H + kPT - 1) / kPT;
  int t = blockIdx.x;
  const int c = t % ncls; t /= ncls;
  const int tx = t % tiles_x; t /= tiles_x;
  const int ty = t % tiles_y; const int b = t / tiles_y;
  const int x0 = tx * kPT - kPH, y0 = ty * kPT - kPH;
  for (int i = threadIdx.x; i < kPW * kPW; i += blockDim.x) {
    const int ly = i / kPW, lx = i - ly * kPW, y = y0 + ly, x = x0 + lx;
    sv[ly][lx] = (y >= 0 && y < H && x >= 0 && x < W) ? sigmoidf_ref(__ldg(center + (((long long)b * H + y) * W + x) * ncls + c)) : -INFINITY;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kPW * kPT; i += blockDim.x) {
    const int ly = i / kPT, lx = i - ly * kPT;
    float m = sv[ly][lx];
#pragma unroll
    for (int d = 1; d < 7; ++d) m = fmax_nan(m, sv[ly][lx + d]);
    rm[ly][lx] = m;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kPT * kPT; i += blockDim.x) {
    const int ly = i / kPT, lx = i - ly * kPT, y = y0 + kPH + ly, x = x0 + kPH + lx;
    if (y >= H || x >= W) continue;
    const float s = sv[ly + kPH][lx + kPH];
    if (!passes(s, min_score)) continue;
    float m = rm[ly][lx];
#pragma unroll
    for (int d = 1; d < 7; ++d) m = fmax_nan(m, rm[ly + d][lx]);
    if (m > s) continue;                                     // something in the 7x7 window is larger: not a peak
    const int slot = atomicAdd(&counts[b * ncls + c], 1);
    if (slot < kCandCap) cand[(long long)(b * ncls + c) * kCandCap + slot] = make_float2(s, __int_as_float(y * W + x));
  }
}

constexpr int kSel = 256;         // threads of the select block

// The select block's path past the candidate cap: one pass over the (frame, class) plane in chunks of kSel pixels, each pixel
// tested as peak_candidates_kernel tests it, keeping the max_det first candidates in ts / tl (ranked).  A pixel is tested
// only when it would enter the list, so a saturated plateau costs one sigmoid per pixel.  -> the number of candidates kept.
// Out of line: the common path never takes it.
__device__ __forceinline__ int rescan_plane(const float* __restrict__ plane, int H, int W, int ncls, float min_score, int max_det,
                                         float* ts, int* tl, float* cs, int* cl) {
  const int tid = threadIdx.x, hw = H * W;
  int cnt = 0;
  for (int base = 0; base < hw; base += kSel) {
    const int p = base + tid;
    float s = -INFINITY; int l = INT_MAX;                      // ranks after every candidate
    if (p < hw) {
      const float v = sigmoidf_ref(__ldg(plane + (long long)p * ncls));
      if (passes(v, min_score) && (cnt < max_det || ahead(v, p, ts[max_det - 1], tl[max_det - 1]))) {
        bool peak = true;
        if (!isnan(v)) {
          const int y = p / W, x = p - y * W;
          float m = -INFINITY;
          for (int yy = max(y - kPH, 0); yy <= min(y + kPH, H - 1); ++yy)
            for (int xx = max(x - kPH, 0); xx <= min(x + kPH, W - 1); ++xx)
              m = fmax_nan(m, sigmoidf_ref(__ldg(plane + ((long long)yy * W + xx) * ncls)));
          peak = !(m > v);
        }
        if (peak) { s = v; l = p; }
      }
    }
    const int nc = __syncthreads_count(l != INT_MAX);
    if (nc == 0) continue;
    // merge: every entry's new rank = entries of the list and of this chunk ahead of it
    cs[tid] = s; cl[tid] = l;
    const float ls = tid < cnt ? ts[tid] : 0.f;
    const int ll = tid < cnt ? tl[tid] : 0;
    __syncthreads();
    int r = 0, rl = tid;
    if (l != INT_MAX) {
      for (int j = 0; j < cnt; ++j) r += ahead(ts[j], tl[j], s, l);
      for (int j = 0; j < kSel; ++j) r += ahead(cs[j], cl[j], s, l);
    }
    if (tid < cnt)
      for (int j = 0; j < kSel; ++j) rl += ahead(cs[j], cl[j], ls, ll);
    __syncthreads();
    if (l != INT_MAX && r < max_det) { ts[r] = s; tl[r] = l; }
    if (tid < cnt && rl < max_det) { ts[rl] = ls; tl[rl] = ll; }
    cnt = min(max_det, cnt + nc);
    __syncthreads();
  }
  return cnt;
}

// one block per (frame, class) selects the max_det first candidates.  Common path: max_det rounds over the list
// peak_candidates_kernel built, each taking the best entry ranked after the previous round's pick.  When more than kCandCap
// candidates were found the list holds an arbitrary subset of them, so the plane is scanned again (rescan_plane).  Either
// way the pick depends on the map alone.
__global__ void __launch_bounds__(kSel) peak_select_kernel(const float* __restrict__ center, const float* __restrict__ box,
                                                           const float* __restrict__ ori, int H, int W, int ncls, float min_score,
                                                           int max_det, const int* __restrict__ counts,
                                                           const float2* __restrict__ cand, float* __restrict__ packed) {
  __shared__ float ts[64]; __shared__ int tl[64];          // the picks, ranked
  __shared__ float cs[kSel]; __shared__ int cl[kSel];
  const int bc = blockIdx.x, b = bc / ncls, c = bc % ncls, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n = counts[bc];
  int found = 0;
  if (n > kCandCap) {
    found = rescan_plane(center + (long long)b * H * W * ncls + c, H, W, ncls, min_score, max_det, ts, tl, cs, cl);
  } else {
    const float2* list = cand + (long long)bc * kCandCap;
    float prev = NAN; int prev_loc = -1;                   // ranks ahead of every candidate
    for (; found < max_det; ++found) {
      float best = -INFINITY; int best_loc = INT_MAX;        // ranks after every candidate (scores are >= 0 or NaN)
      for (int j = tid; j < n; j += kSel) {
        const float2 e = list[j];
        const float s = e.x;
        const int loc = __float_as_int(e.y);
        if (ahead(prev, prev_loc, s, loc) && ahead(s, loc, best, best_loc)) { best = s; best_loc = loc; }   // not taken yet
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int ol = __shfl_xor_sync(0xffffffffu, best_loc, o);
        if (ahead(ob, ol, best, best_loc)) { best = ob; best_loc = ol; }
      }
      if (lane == 0) { cs[warp] = best; cl[warp] = best_loc; }
      __syncthreads();
      for (int w = 0; w < kSel / 32; ++w)
        if (ahead(cs[w], cl[w], best, best_loc)) { best = cs[w]; best_loc = cl[w]; }
      __syncthreads();
      if (best_loc == INT_MAX) break;                        // fewer than max_det candidates
      if (tid == 0) { ts[found] = best; tl[found] = best_loc; }
      prev = best; prev_loc = best_loc;
    }
    __syncthreads();
  }
  const int cols = ncls * max_det;
  float* out = packed + (long long)b * 7 * cols + c * max_det;
  for (int k = tid; k < max_det; k += kSel) {
    if (k < found) {
      const long long px = ((long long)b * H * W + tl[k]) * 2;
      out[0 * cols + k] = ts[k]; out[1 * cols + k] = (float)tl[k];
      out[2 * cols + k] = __ldg(box + px); out[3 * cols + k] = __ldg(box + px + 1);
      out[4 * cols + k] = __ldg(ori + px); out[5 * cols + k] = __ldg(ori + px + 1);
    } else {                                                 // padding past the last candidate
      out[0 * cols + k] = -1e5f;
      out[1 * cols + k] = out[2 * cols + k] = out[3 * cols + k] = out[4 * cols + k] = out[5 * cols + k] = 0.f;
    }
    out[6 * cols + k] = (float)W;
  }
}

}  // namespace lavb

using namespace lavb;

extern "C" size_t lavb_det_peaks_workspace_bytes(int batch, int ncls) {
  return (size_t)batch * ncls * (sizeof(int) + kCandCap * sizeof(float2)) + 256;
}

extern "C" int lavb_det_peaks(const float* d_center, const float* d_box, const float* d_ori, int batch, int h, int w, int ncls,
                              float min_score, int max_det, float* d_packed, void* d_workspace, void* stream) {
  LAVB_CHECK_ARG(ncls >= 1 && ncls <= 8 && max_det >= 1 && max_det <= 64, "det_peaks: bad ncls %d / max_det %d", ncls, max_det);
  LAVB_CHECK_ARG(batch >= 0 && h >= 1 && w >= 1 && (long long)h * w <= (1LL << 24),
                 "det_peaks: bad sizes (batch %d, %d x %d; h * w must be 1..2^24, the flat index is stored as a float)", batch, h, w);
  const long long tiles = (long long)batch * ceil_div(h, kPT) * ceil_div(w, kPT) * ncls;
  LAVB_CHECK_ARG(tiles <= INT_MAX, "det_peaks: batch %d of %d x %d maps is too large for one launch", batch, h, w);
  if (batch == 0) return 0;
  LAVB_CHECK_ARG(d_center && d_box && d_ori && d_packed && d_workspace, "det_peaks: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  int* counts = reinterpret_cast<int*>(d_workspace);
  float2* cand = reinterpret_cast<float2*>(reinterpret_cast<char*>(d_workspace) + ((size_t)batch * ncls * sizeof(int) + 255) / 256 * 256);
  LAVB_CUDA_OK(cudaMemsetAsync(counts, 0, (size_t)batch * ncls * sizeof(int), st));
  peak_candidates_kernel<<<(int)tiles, 256, 0, st>>>(d_center, batch, h, w, ncls, min_score, counts, cand);
  LAVB_LAUNCH_OK();
  peak_select_kernel<<<batch * ncls, kSel, 0, st>>>(d_center, d_box, d_ori, h, w, ncls, min_score, max_det, counts, cand, d_packed);
  LAVB_LAUNCH_OK();
  return 0;
}
