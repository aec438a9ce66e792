// PointPillars dynamic voxeliser + pillar encoder (lav/models/point_pillar.py:55-116) without sort/unique:
// a pillar is addressed directly by (b, xi, yi); pass 1 accumulates the per-pillar centroid sums, pass 2
// decorates each point, runs the 2-layer point MLP and max-pools into the NHWC canvas.
#include <math.h>
#include <stdlib.h>
#include "common.cuh"
#include "pillar_grid.cuh"

namespace lavb {

constexpr int kMaxBatch = 128;

struct Clouds {
  long long start[kMaxBatch];  // first row of cloud b in the point buffer
  int cum[kMaxBatch + 1];      // exclusive prefix of cloud sizes
  int batch;
};

__device__ __forceinline__ int find_cloud(const Clouds& c, int i) {
  int lo = 0, hi = c.batch - 1;
  while (lo < hi) {
    int mid = (lo + hi + 1) >> 1;
    if (c.cum[mid] <= i) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// grid_locations, point_pillar.py:70-79: half-open window test on the raw fp32 coordinates (in_window), then
// trunc((v - min) * ppm) in fp32.  Returns false for dropped points (NaN fails every comparison).
__device__ __forceinline__ bool locate(const Grid& g, float x, float y, int& xi, int& yi) {
  if (!in_window(g, x, y)) return false;
  xi = (int)__fmul_rn(__fsub_rn(x, g.min_x), g.ppm);
  yi = (int)__fmul_rn(__fsub_rn(y, g.min_y), g.ppm);
  return true;
}

// pillar key space: xi in [0,nx], yi in [0,ny]  (index == n can occur by rounding, SURVEY App. C.5)
__device__ __forceinline__ long long pillar_key(const Grid& g, int b, int xi, int yi) {
  return ((long long)b * (g.nx + 1) + xi) * (g.ny + 1) + yi;
}
// scatter_points, point_pillar.py:87-90: row = clamp(ny-1-xi), col = clamp(yi)
__device__ __forceinline__ long long canvas_cell(const Grid& g, int b, int xi, int yi) {
  int row = g.ny - 1 - xi; row = row < 0 ? 0 : (row > g.ny - 1 ? g.ny - 1 : row);
  int col = yi < 0 ? 0 : (yi > g.nx - 1 ? g.nx - 1 : yi);
  return ((long long)b * g.ny + row) * g.nx + col;
}

__global__ void __launch_bounds__(256) pillar_stats_kernel(const float* __restrict__ pts, int pt_stride,
                                                           const __grid_constant__ Clouds clouds,
                                                           const __grid_constant__ Grid g, float4* __restrict__ stats) {
  const int total = clouds.cum[clouds.batch];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int b = find_cloud(clouds, i);
    const float* p = pts + (clouds.start[b] + (i - clouds.cum[b])) * pt_stride;
    const float x = __ldg(p), y = __ldg(p + 1), z = __ldg(p + 2);
    int xi, yi;
    if (!locate(g, x, y, xi, yi)) continue;
    atomicAdd(&stats[pillar_key(g, b, xi, yi)], make_float4(x, y, z, 1.f));  // red.global.add.v4.f32 (sm_90+)
  }
}

// decorate, point_pillar.py:55-68: [pt(D) | xyz - centroid | x - (yi/ppm + min_x) | y - (xi/ppm + min_y)]
// (the cell-origin terms use the OTHER axis' index and no +0.5 — replicated on purpose).
template <int D>
__device__ __forceinline__ void decorate(const Grid& g, const float* __restrict__ p, int xi, int yi, float4 st,
                                         float* f) {
#pragma unroll
  for (int k = 0; k < D; ++k) f[k] = __ldg(p + k);
  f[D + 0] = __fsub_rn(f[0], __fdiv_rn(st.x, st.w));
  f[D + 1] = __fsub_rn(f[1], __fdiv_rn(st.y, st.w));
  f[D + 2] = __fsub_rn(f[2], __fdiv_rn(st.z, st.w));
  f[D + 3] = __fsub_rn(f[0], __fadd_rn(__fdiv_rn((float)yi, g.ppm), g.min_x));
  f[D + 4] = __fsub_rn(f[1], __fadd_rn(__fdiv_rn((float)xi, g.ppm), g.min_y));
}

// One thread per point; both weight matrices live in shared memory k-major so that a thread reads the
// weights of 4 consecutive output channels with one broadcast LDS.128.
template <int D, int H1, int H2>
__global__ void __launch_bounds__(128) pillar_encode_kernel(const float* __restrict__ pts, int pt_stride,
                                                            const __grid_constant__ Clouds clouds,
                                                            const __grid_constant__ Grid g,
                                                            const float4* __restrict__ stats,
                                                            const float* __restrict__ w1, const float* __restrict__ s1,
                                                            const float* __restrict__ t1, const float* __restrict__ w2,
                                                            const float* __restrict__ s2, const float* __restrict__ t2,
                                                            float* __restrict__ canvas) {
  constexpr int F = D + 5;
  __shared__ __align__(16) float w1s[F][H1];
  __shared__ __align__(16) float w2s[H1][H2];
  __shared__ float s1s[H1], t1s[H1], s2s[H2], t2s[H2];
  for (int i = threadIdx.x; i < F * H1; i += blockDim.x) w1s[i % F][i / F] = __ldg(w1 + i);   // w1 is [H1][F]
  for (int i = threadIdx.x; i < H1 * H2; i += blockDim.x) w2s[i % H1][i / H1] = __ldg(w2 + i); // w2 is [H2][H1]
  for (int i = threadIdx.x; i < H1; i += blockDim.x) { s1s[i] = __ldg(s1 + i); t1s[i] = __ldg(t1 + i); }
  for (int i = threadIdx.x; i < H2; i += blockDim.x) { s2s[i] = __ldg(s2 + i); t2s[i] = __ldg(t2 + i); }
  __syncthreads();
  const int total = clouds.cum[clouds.batch];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int b = find_cloud(clouds, i);
    const float* p = pts + (clouds.start[b] + (i - clouds.cum[b])) * pt_stride;
    int xi, yi;
    if (!locate(g, __ldg(p), __ldg(p + 1), xi, yi)) continue;
    const float4 st = __ldg(&stats[pillar_key(g, b, xi, yi)]);
    float f[F];
    decorate<D>(g, p, xi, yi, st, f);
    float h[H1];
#pragma unroll
    for (int j = 0; j < H1; ++j) h[j] = 0.f;
#pragma unroll
    for (int k = 0; k < F; ++k) {
#pragma unroll
      for (int j = 0; j < H1; j += 4) {
        const float4 w = *reinterpret_cast<const float4*>(&w1s[k][j]);
        h[j] = fmaf(f[k], w.x, h[j]); h[j + 1] = fmaf(f[k], w.y, h[j + 1]);
        h[j + 2] = fmaf(f[k], w.z, h[j + 2]); h[j + 3] = fmaf(f[k], w.w, h[j + 3]);
      }
    }
#pragma unroll
    for (int j = 0; j < H1; ++j) { const float v = fmaf(h[j], s1s[j], t1s[j]); h[j] = v > 0.f ? v : 0.f; }
    float* cell = canvas + canvas_cell(g, b, xi, yi) * H2;
#pragma unroll 1
    for (int j0 = 0; j0 < H2; j0 += 16) {
      float o[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) o[j] = 0.f;
#pragma unroll
      for (int k = 0; k < H1; ++k) {
#pragma unroll
        for (int j = 0; j < 16; j += 4) {
          const float4 w = *reinterpret_cast<const float4*>(&w2s[k][j0 + j]);
          o[j] = fmaf(h[k], w.x, o[j]); o[j + 1] = fmaf(h[k], w.y, o[j + 1]);
          o[j + 2] = fmaf(h[k], w.z, o[j + 2]); o[j + 3] = fmaf(h[k], w.w, o[j + 3]);
        }
      }
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float v = fmaf(o[j], s2s[j0 + j], t2s[j0 + j]);
        // post-ReLU values are >= +0, so float max == signed-int max on the bit pattern and the zero-filled
        // canvas is both the identity of the max and the value of empty cells.
        if (v > 0.f) atomicMax(reinterpret_cast<int*>(cell + j0 + j), __float_as_int(v));
      }
    }
  }
}

// ---------------------------------------------------------------- training-mode pieces
// order-preserving compaction of the in-window points: per-block counts -> single-block scan -> write
constexpr int kCompactBlock = 1024;

__global__ void __launch_bounds__(kCompactBlock) keep_count_kernel(const float* __restrict__ pts, int pt_stride,
                                                                   const __grid_constant__ Clouds clouds,
                                                                   const __grid_constant__ Grid g, int* __restrict__ block_count) {
  const int total = clouds.cum[clouds.batch];
  const int i = blockIdx.x * kCompactBlock + threadIdx.x;
  int keep = 0;
  if (i < total) {
    const int b = find_cloud(clouds, i);
    const float* p = pts + (clouds.start[b] + (i - clouds.cum[b])) * pt_stride;
    int xi, yi;
    keep = locate(g, __ldg(p), __ldg(p + 1), xi, yi) ? 1 : 0;
  }
  const int c = __syncthreads_count(keep);
  if (threadIdx.x == 0) block_count[blockIdx.x] = c;
}

__global__ void __launch_bounds__(1024) scan_blocks_kernel(int* __restrict__ block_count, int nblocks, int* __restrict__ total_out) {
  __shared__ int warp_sum[32];
  __shared__ int carry_s;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  for (int base = 0; base < nblocks; base += 1024) {
    const int i = base + threadIdx.x;
    const int v = i < nblocks ? block_count[i] : 0;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int y = __shfl_up_sync(0xffffffffu, x, o); if ((threadIdx.x & 31) >= o) x += y; }
    if ((threadIdx.x & 31) == 31) warp_sum[threadIdx.x >> 5] = x;
    __syncthreads();
    if (threadIdx.x < 32) {
      int w = warp_sum[threadIdx.x];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { int y = __shfl_up_sync(0xffffffffu, w, o); if (threadIdx.x >= o) w += y; }
      warp_sum[threadIdx.x] = w;
    }
    __syncthreads();
    const int warp_off = (threadIdx.x >> 5) ? warp_sum[(threadIdx.x >> 5) - 1] : 0;
    const int carry = carry_s;
    if (i < nblocks) block_count[i] = carry + warp_off + x - v;  // exclusive
    __syncthreads();
    if (threadIdx.x == 1023) carry_s = carry + warp_off + x;
    __syncthreads();
  }
  if (threadIdx.x == 0) *total_out = carry_s;
}

template <int D>
__global__ void __launch_bounds__(kCompactBlock) decorate_write_kernel(const float* __restrict__ pts, int pt_stride,
                                                                       const __grid_constant__ Clouds clouds,
                                                                       const __grid_constant__ Grid g,
                                                                       const float4* __restrict__ stats,
                                                                       const int* __restrict__ block_off,
                                                                       float* __restrict__ feat, int* __restrict__ cell) {
  constexpr int F = D + 5;
  __shared__ int warp_cnt[32];
  const int total = clouds.cum[clouds.batch];
  const int i = blockIdx.x * kCompactBlock + threadIdx.x;
  int keep = 0, xi = 0, yi = 0, b = 0;
  const float* p = nullptr;
  if (i < total) {
    b = find_cloud(clouds, i);
    p = pts + (clouds.start[b] + (i - clouds.cum[b])) * pt_stride;
    keep = locate(g, __ldg(p), __ldg(p + 1), xi, yi) ? 1 : 0;
  }
  const unsigned m = __ballot_sync(0xffffffffu, keep);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) warp_cnt[warp] = __popc(m);
  __syncthreads();
  if (warp == 0) {
    int w = warp_cnt[lane], x = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    warp_cnt[lane] = x - w;
  }
  __syncthreads();
  if (!keep) return;
  const int row = block_off[blockIdx.x] + warp_cnt[warp] + __popc(m & ((1u << lane) - 1u));
  float f[F];
  decorate<D>(g, p, xi, yi, __ldg(&stats[pillar_key(g, b, xi, yi)]), f);
#pragma unroll
  for (int k = 0; k < F; ++k) feat[(size_t)row * F + k] = f[k];
  cell[row] = (int)canvas_cell(g, b, xi, yi);
}

__global__ void __launch_bounds__(256) scatter_max_kernel(const float* __restrict__ h, const int* __restrict__ cell,
                                                          long long mc, int c, float* __restrict__ canvas) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= mc) return;
  const int row = (int)(i / c), ch = (int)(i - (long long)row * c);
  const float v = __ldg(h + i);
  if (v > 0.f) atomicMax(reinterpret_cast<int*>(canvas + (long long)__ldg(cell + row) * c + ch), __float_as_int(v));
}
__global__ void __launch_bounds__(256) scatter_arg_kernel(const float* __restrict__ h, const int* __restrict__ cell,
                                                          long long mc, int c, const float* __restrict__ canvas,
                                                          int* __restrict__ argmax) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= mc) return;
  const int row = (int)(i / c), ch = (int)(i - (long long)row * c);
  const long long o = (long long)__ldg(cell + row) * c + ch;
  const float v = __ldg(h + i);
  const float top = canvas[o];
  if (v == top || (!(v > 0.f) && top == 0.f)) atomicMin(argmax + o, row);  // ties -> smallest row (deterministic)
}
__global__ void __launch_bounds__(256) scatter_bwd_kernel(const float* __restrict__ gcanvas, const int* __restrict__ argmax,
                                                          const int* __restrict__ cell, long long mc, int c,
                                                          float* __restrict__ gh) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= mc) return;
  const int row = (int)(i / c), ch = (int)(i - (long long)row * c);
  const long long o = (long long)__ldg(cell + row) * c + ch;
  gh[i] = (__ldg(argmax + o) == row) ? __ldg(gcanvas + o) : 0.f;
}

static int fill_clouds(Clouds& c, const long long* start, const int* count, int batch) {
  if (batch < 1 || batch > kMaxBatch) { set_error("pillar: batch must be 1..%d (got %d)", kMaxBatch, batch); return 1; }
  c.batch = batch;
  long long cum = 0;
  for (int b = 0; b < batch; ++b) {
    if (count[b] < 0 || start[b] < 0) { set_error("pillar: negative cloud start/count"); return 1; }
    c.start[b] = start[b];
    c.cum[b] = (int)cum;
    cum += count[b];
    if (cum > 0x7fffffffLL) { set_error("pillar: more than 2^31 points"); return 1; }
  }
  c.cum[batch] = (int)cum;
  return 0;
}

static size_t stats_bytes(int batch, int nx, int ny) { return (size_t)batch * (nx + 1) * (ny + 1) * sizeof(float4); }

static bool aligned(const void* p, size_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

// The grid must hold every point the window keeps: pillar_key addresses xi in [0, nx] and yi in [0, ny].  The largest index is
// reached by the largest fp32 coordinate below max, computed in the kernel's fp32 arithmetic (trunc(v) <= n  <=>  v < n + 1).
static int check_grid(const char* who, float min_x, float max_x, float min_y, float max_y, float ppm, int nx, int ny) {
  LAVB_CHECK_ARG(isfinite(ppm) && ppm > 0.f, "%s: ppm must be finite and > 0 (got %g)", who, ppm);
  LAVB_CHECK_ARG(isfinite(min_x) && isfinite(max_x) && isfinite(min_y) && isfinite(max_y) && min_x < max_x && min_y < max_y,
                 "%s: the window must be finite with min < max (got x [%g, %g), y [%g, %g))", who, min_x, max_x, min_y, max_y);
  LAVB_CHECK_ARG(nx >= 1 && ny >= 1, "%s: nx, ny must be >= 1 (got %d, %d)", who, nx, ny);
  const float top_x = (nextafterf(max_x, -INFINITY) - min_x) * ppm, top_y = (nextafterf(max_y, -INFINITY) - min_y) * ppm;
  LAVB_CHECK_ARG((double)top_x < (double)nx + 1.0 && (double)top_y < (double)ny + 1.0,
                 "%s: the window reaches index (%.0f, %.0f), beyond the grid's (%d, %d)", who, floor(top_x), floor(top_y), nx, ny);
  return 0;
}

// pointer checks shared by both encoders: point rows are read as floats, the workspace holds float4 centroid sums
static int check_encoder_ptrs(const char* who, const float* pts, int total, const float* w1, const float* s1, const float* t1,
                              const float* w2, const float* s2, const float* t2, const void* canvas, size_t canvas_align,
                              const void* ws) {
  LAVB_CHECK_ARG(total == 0 || (pts != nullptr && aligned(pts, 4)), "%s: d_pts must be non-null and 4-byte aligned", who);
  LAVB_CHECK_ARG(w1 && s1 && t1 && w2 && s2 && t2 && canvas && ws, "%s: null weight, canvas or workspace pointer", who);
  LAVB_CHECK_ARG(aligned(w1, 4) && aligned(s1, 4) && aligned(t1, 4) && aligned(w2, 8) && aligned(s2, 4) && aligned(t2, 4),
                 "%s: w2 must be 8-byte aligned, w1 / s1 / t1 / s2 / t2 4-byte aligned", who);
  LAVB_CHECK_ARG(aligned(canvas, canvas_align) && aligned(ws, 16), "%s: the canvas must be %zu-byte and the workspace 16-byte "
                 "aligned", who, canvas_align);
  return 0;
}

// =====================================================================================================================
// Sorted (atomic-free canvas) pillar encoder for the tensor-core pipeline.
//   K1 count   : per point -> centroid sums (one vector RED) + per-canvas-cell point count
//   K2 offsets : exclusive scan of the counts (block sums -> single-block scan -> per-cell offsets); the same pass
//                zero-fills the canvas rows of EMPTY cells (so every canvas byte is written exactly once overall)
//                and records for every 128-slot window the first segment head at/after it (tile_start)
//   K3 fill    : counting-sort scatter of point indices into cell order
//   K4 encode  : block i owns the whole pillars whose first point lies in slots [128 i, 128 (i+1)); per 128-row chunk:
//                decorate + layer 1 (fp32 FFMA) -> h16 hidden tile in swizzled smem -> layer 2 on the tensor cores
//                (mma.sync m16n8k16 h16, fp32 accumulate; the 64x64 weight fragments live in registers) ->
//                BN affine + ReLU -> fp32 tile in smem -> 64 channel-threads walk the rows and emit one canvas row per
//                pillar (running max), as fp32 or as h16.
// The first layer stays fp32 because its inputs are raw metric coordinates (h16 would quantise x to 0.25 m).
// =====================================================================================================================
constexpr int kCellsPerBlock = 1024;
constexpr int kRows = 128;            // slots per encode chunk
constexpr int kOsPitch = 68;          // fp32 output tile pitch (floats): conflict-free fragment stores

__global__ void __launch_bounds__(256) pillar_count_kernel(const float* __restrict__ pts, int pt_stride,
                                                           const __grid_constant__ Clouds clouds,
                                                           const __grid_constant__ Grid g, float4* __restrict__ stats,
                                                           int* __restrict__ count) {
  const int total = clouds.cum[clouds.batch];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int b = find_cloud(clouds, i);
    const float* p = pts + (clouds.start[b] + (i - clouds.cum[b])) * pt_stride;
    const float x = __ldg(p), y = __ldg(p + 1), z = __ldg(p + 2);
    int xi, yi;
    if (!locate(g, x, y, xi, yi)) continue;
    atomicAdd(&stats[pillar_key(g, b, xi, yi)], make_float4(x, y, z, 1.f));
    atomicAdd(&count[canvas_cell(g, b, xi, yi)], 1);
  }
}

__global__ void __launch_bounds__(kCellsPerBlock) cell_block_sum_kernel(const int* __restrict__ count, long long ncells,
                                                                        int* __restrict__ block_sum) {
  const long long c = (long long)blockIdx.x * kCellsPerBlock + threadIdx.x;
  int v = c < ncells ? count[c] : 0;
  __shared__ int ws[32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    int w = ws[threadIdx.x];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) w += __shfl_xor_sync(0xffffffffu, w, o);
    if (threadIdx.x == 0) block_sum[blockIdx.x] = w;
  }
}

// per-cell exclusive offsets + zero-fill of empty canvas rows + tile_start table
__global__ void __launch_bounds__(kCellsPerBlock) cell_offsets_kernel(const int* __restrict__ count, long long ncells,
                                                                      const int* __restrict__ block_off,
                                                                      int* __restrict__ offsets, int* __restrict__ tile_start,
                                                                      const int* __restrict__ total_kept,
                                                                      uint4* __restrict__ canvas16, int row_vec16) {
  __shared__ int ws[32];
  const long long c = (long long)blockIdx.x * kCellsPerBlock + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int cnt = c < ncells ? count[c] : 0;
  int x = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
  if (lane == 31) ws[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int w = ws[lane], s = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += y; }
    ws[lane] = s - w;
  }
  __syncthreads();
  const int off = block_off[blockIdx.x] + ws[warp] + x - cnt;
  if (c < ncells) offsets[c] = off;
  if (c == ncells - 1) { offsets[ncells] = off + cnt; }
  if (cnt > 0) {   // window boundaries 128*i inside [off, off+cnt): first head at/after the boundary
    for (int i = (off + kRows - 1) / kRows; i * kRows < off + cnt; ++i) tile_start[i] = (i * kRows == off) ? off : off + cnt;
  }
  if (c == 0) { const int tk = *total_kept; tile_start[(tk + kRows - 1) / kRows] = tk; }
  // zero-fill: the warp's 32 cells are one contiguous canvas span; lanes sweep it 16 B at a time, skipping occupied rows
  const unsigned occ = __ballot_sync(0xffffffffu, cnt > 0 || c >= ncells);
  const long long c0 = c - lane;
  const int per_iter = 32 / row_vec16 > 0 ? 32 / row_vec16 : 1;      // rows covered per sweep step (row_vec16 = 16 B pieces / row)
  for (int r0 = 0; r0 < 32; r0 += per_iter) {
    if (row_vec16 <= 32) {
      const int r = r0 + lane / row_vec16, v = lane % row_vec16;
      if (r < 32 && !((occ >> r) & 1u)) canvas16[(c0 + r) * row_vec16 + v] = make_uint4(0u, 0u, 0u, 0u);
    } else {
      if (!((occ >> r0) & 1u))
        for (int v = lane; v < row_vec16; v += 32) canvas16[(c0 + r0) * row_vec16 + v] = make_uint4(0u, 0u, 0u, 0u);
    }
  }
}

__global__ void __launch_bounds__(256) pillar_fill_kernel(const float* __restrict__ pts, int pt_stride,
                                                          const __grid_constant__ Clouds clouds, const __grid_constant__ Grid g,
                                                          const int* __restrict__ offsets, int* __restrict__ cursor,
                                                          int* __restrict__ order, int* __restrict__ ocell) {
  const int total = clouds.cum[clouds.batch];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int b = find_cloud(clouds, i);
    const float* p = pts + (clouds.start[b] + (i - clouds.cum[b])) * pt_stride;
    int xi, yi;
    if (!locate(g, __ldg(p), __ldg(p + 1), xi, yi)) continue;
    const int cell = (int)canvas_cell(g, b, xi, yi);
    const int slot = __ldg(offsets + cell) + atomicAdd(cursor + cell, 1);
    order[slot] = i;
    ocell[slot] = cell;
  }
}

__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma_h16_16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32." LAVB_H16_PTX "." LAVB_H16_PTX ".f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

constexpr int kFsPitch = 20;          // fp32 decorated-feature tile pitch (floats)
constexpr int kW1Pitch = 24;          // h16 layer-1 weight row pitch: conflict-free B-fragment loads

struct EncSmem {                      // shared-memory plan of pillar_encode_sorted_kernel (bytes from the base)
  static constexpr int fs = 0;                                             // [128][kFsPitch] fp32
  static constexpr int os = fs + kRows * kFsPitch * 4;                     // [128][kOsPitch] fp32
  static constexpr int w1h = os + kRows * kOsPitch * 4;                    // [64][kW1Pitch] h16 (hi)
  static constexpr int w1l = w1h + 64 * kW1Pitch * 2;                      // (lo)
  static constexpr int aff = w1l + 64 * kW1Pitch * 2;                      // s1 | t1 | s2 | t2
  static constexpr int cells = aff + 4 * 64 * 4;                           // [128] int
  static constexpr int pmax = cells + kRows * 4;                           // [2 parity][first|last][4 quarters][64] fp32
  static constexpr int pcell = pmax + 2 * 2 * 4 * 64 * 4;                  // [2 parity][4 quarters][first, last, n, pad] int
  static constexpr int total = pcell + 2 * 4 * 4 * 4;
};

template <int kOutMode>      // 0: fp32 [64]; 2: h16 [64]
__device__ __forceinline__ void emit_pair(void* canvas, int cell, int c, float m0, float m1) {     // channels c, c+1 (c even)
  if (kOutMode == 2) {
    *reinterpret_cast<uint32_t*>(reinterpret_cast<h16*>(canvas) + (long long)cell * 64 + c) = pack_h16(m0, m1);
  } else {
    *reinterpret_cast<float2*>(reinterpret_cast<float*>(canvas) + (long long)cell * 64 + c) = make_float2(m0, m1);
  }
}
template <int kOutMode>
__device__ __forceinline__ void emit_one(void* canvas, int cell, int c, float m) {
  if (kOutMode == 2) {
    reinterpret_cast<h16*>(canvas)[(long long)cell * 64 + c] = float2h16(m);
  } else {
    reinterpret_cast<float*>(canvas)[(long long)cell * 64 + c] = m;
  }
}
// fp32 pair -> h16 hi pair + h16 residual pair (error-free split to ~2^-16 relative)
__device__ __forceinline__ void split_pair(float2 f, uint32_t& hi, uint32_t& lo) {
  const h162 h = floats2h162(f.x, f.y);
  const float2 hf = h1622float2(h);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = pack_h16(f.x - hf.x, f.y - hf.y);
}

// Pillar encoder over the cell-sorted point order (both MLP layers on the tensor cores, no canvas atomics).
// A block walks "windows" of ~128 sorted rows that begin and end on pillar boundaries (tile_start), 128 rows per batch,
// warp w owning rows [32w, 32w+32) of the batch end to end — one __syncthreads per batch:
//   (1) gather + decorate: one thread per row -> 16 fp32 features in shared memory;
//   (2) layer 1 (16 -> 64) as mma.sync m16n8k16 with the features AND weights split into h16 hi + lo (3 MMAs per tile:
//       hi*hi + lo*hi + hi*lo, fp32 accumulate ~ fp32 accuracy); BN affine + ReLU on the accumulator fragments, which are
//       then re-packed IN REGISTERS as the h16 A fragments of layer 2 (64 -> 64; C-fragment layout == A-fragment layout);
//       BN affine + ReLU -> fp32 tile in shared memory;
//   (3) segmented max: each warp walks its own 32 rows, one lane per channel pair; runs that start and end inside the
//       quarter go straight to the canvas, the first / last run's partial maxima to a small table;
//   (4) after the barrier, 64 threads stitch the quarter tables with the run carried from the previous batch.
// Every canvas row of an occupied cell is written exactly once; empty cells were zero-filled by cell_offsets_kernel.
template <int D, int kOutMode>
__global__ void __launch_bounds__(kRows, 3) pillar_encode_sorted_kernel(
    const float* __restrict__ pts, int pt_stride, const __grid_constant__ Clouds clouds, const __grid_constant__ Grid g,
    const float4* __restrict__ stats, const int* __restrict__ order, const int* __restrict__ ocell,
    const int* __restrict__ tile_start, const int* __restrict__ total_kept, const float* __restrict__ w1,
    const float* __restrict__ s1, const float* __restrict__ t1, const float* __restrict__ w2, const float* __restrict__ s2,
    const float* __restrict__ t2, void* __restrict__ canvas) {
  constexpr int F = D + 5, H = 64;
  static_assert(F == 16, "layer 1 is one k16 MMA step");
  extern __shared__ __align__(128) uint8_t sm[];
  float* fs = reinterpret_cast<float*>(sm + EncSmem::fs);
  float* Os = reinterpret_cast<float*>(sm + EncSmem::os);
  h16* w1h = reinterpret_cast<h16*>(sm + EncSmem::w1h);
  h16* w1l = reinterpret_cast<h16*>(sm + EncSmem::w1l);
  float* aff = reinterpret_cast<float*>(sm + EncSmem::aff);
  int* cells = reinterpret_cast<int*>(sm + EncSmem::cells);
  float* pmax = reinterpret_cast<float*>(sm + EncSmem::pmax);
  int* pcell = reinterpret_cast<int*>(sm + EncSmem::pcell);

  const int nt = (*total_kept + kRows - 1) / kRows;
  if ((int)blockIdx.x >= nt) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, gq = lane >> 2, tq = lane & 3;
  for (int i = tid; i < H * F; i += kRows) {                                      // w1 is [64 n][16 k]
    const float v = __ldg(w1 + i);
    const h16 hi = float2h16(v);
    w1h[(i / F) * kW1Pitch + i % F] = hi;
    w1l[(i / F) * kW1Pitch + i % F] = float2h16(v - h162float(hi));
  }
  for (int i = tid; i < H; i += kRows) { aff[i] = __ldg(s1 + i); aff[H + i] = __ldg(t1 + i); aff[2 * H + i] = __ldg(s2 + i); aff[3 * H + i] = __ldg(t2 + i); }
  // layer-2 weight fragments (B operand, "col" layout = rows of w2 [64 n][64 k]): b0 (k = 16kk + 2tq.., n = 8nn + gq), b1 (k + 8)
  uint32_t bfrag[4][8][2];
#pragma unroll
  for (int kk = 0; kk < 4; ++kk)
#pragma unroll
    for (int nn = 0; nn < 8; ++nn) {
      const float* wp = w2 + (nn * 8 + gq) * H + kk * 16 + tq * 2;
      const float2 lo = __ldg(reinterpret_cast<const float2*>(wp)), hi = __ldg(reinterpret_cast<const float2*>(wp + 8));
      bfrag[kk][nn][0] = pack_h16(lo.x, lo.y);
      bfrag[kk][nn][1] = pack_h16(hi.x, hi.y);
    }
  __syncthreads();
  int it = 0;               // batch counter: parity of the quarter tables
  // persistent: the block walks windows blockIdx.x, +gridDim.x, ...
  for (int win = blockIdx.x; win < nt; win += gridDim.x) {
    const int row_begin = tile_start[win], row_end = tile_start[win + 1];
    if (row_begin >= row_end) continue;
    float run_max = 0.f;      // stitch state of channel `tid` (threads 0..63)
    int run_cell = -1;
    for (int base = row_begin; base < row_end; base += kRows, ++it) {
      const int rows = min(kRows, row_end - base);
      // ---- (1) gather + decorate (one thread per row; the row belongs to this thread's own warp)
      {
        float f[F];
#pragma unroll
        for (int k = 0; k < F; ++k) f[k] = 0.f;
        int cell = -1;
        if (tid < rows) {
          const int i = __ldg(order + base + tid);
          cell = __ldg(ocell + base + tid);
          const int b = find_cloud(clouds, i);
          const float* p = pts + (clouds.start[b] + (i - clouds.cum[b])) * pt_stride;
          int xi, yi;
          locate(g, __ldg(p), __ldg(p + 1), xi, yi);
          decorate<D>(g, p, xi, yi, __ldg(&stats[pillar_key(g, b, xi, yi)]), f);
        }
        cells[tid] = cell;
#pragma unroll
        for (int k = 0; k < F; k += 4) *reinterpret_cast<float4*>(&fs[tid * kFsPitch + k]) = make_float4(f[k], f[k + 1], f[k + 2], f[k + 3]);
      }
      __syncwarp();
      // ---- (2) both MLP layers on the tensor cores: warp w -> rows [32w, 32w+32) as two m16 tiles
#pragma unroll 1
      for (int mt = 0; mt < 2; ++mt) {
        const int row0 = warp * 32 + mt * 16;
        uint32_t ah[4], al[4];
        split_pair(*reinterpret_cast<const float2*>(&fs[(row0 + gq) * kFsPitch + 2 * tq]), ah[0], al[0]);
        split_pair(*reinterpret_cast<const float2*>(&fs[(row0 + gq + 8) * kFsPitch + 2 * tq]), ah[1], al[1]);
        split_pair(*reinterpret_cast<const float2*>(&fs[(row0 + gq) * kFsPitch + 2 * tq + 8]), ah[2], al[2]);
        split_pair(*reinterpret_cast<const float2*>(&fs[(row0 + gq + 8) * kFsPitch + 2 * tq + 8]), ah[3], al[3]);
        uint32_t a2[4][4];        // layer-2 A fragments (h16 h), one k16 step per pair of layer-1 n-tiles
#pragma unroll
        for (int nn = 0; nn < 8; ++nn) {
          const h16* wh = w1h + (nn * 8 + gq) * kW1Pitch + 2 * tq;
          const h16* wl = w1l + (nn * 8 + gq) * kW1Pitch + 2 * tq;
          const uint32_t bh0 = *reinterpret_cast<const uint32_t*>(wh), bh1 = *reinterpret_cast<const uint32_t*>(wh + 8);
          const uint32_t bl0 = *reinterpret_cast<const uint32_t*>(wl), bl1 = *reinterpret_cast<const uint32_t*>(wl + 8);
          float acc[4] = {0.f, 0.f, 0.f, 0.f};
          mma_h16_16816(acc, al[0], al[1], al[2], al[3], bh0, bh1);       // small terms first
          mma_h16_16816(acc, ah[0], ah[1], ah[2], ah[3], bl0, bl1);
          mma_h16_16816(acc, ah[0], ah[1], ah[2], ah[3], bh0, bh1);
          const int col = nn * 8 + 2 * tq;
          const float2 sc = *reinterpret_cast<const float2*>(&aff[col]), sh = *reinterpret_cast<const float2*>(&aff[H + col]);
          const float sc0 = sc.x, sc1 = sc.y, sh0 = sh.x, sh1 = sh.y;
          a2[nn >> 1][(nn & 1) * 2] = pack_h16(fmaxf(fmaf(acc[0], sc0, sh0), 0.f), fmaxf(fmaf(acc[1], sc1, sh1), 0.f));       // row gq
          a2[nn >> 1][(nn & 1) * 2 + 1] = pack_h16(fmaxf(fmaf(acc[2], sc0, sh0), 0.f), fmaxf(fmaf(acc[3], sc1, sh1), 0.f));   // row gq + 8
        }
#pragma unroll
        for (int nn = 0; nn < 8; ++nn) {
          float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) mma_h16_16816(acc, a2[kk][0], a2[kk][1], a2[kk][2], a2[kk][3], bfrag[kk][nn][0], bfrag[kk][nn][1]);
          const int col = nn * 8 + 2 * tq;
          const float2 sc = *reinterpret_cast<const float2*>(&aff[2 * H + col]), sh = *reinterpret_cast<const float2*>(&aff[3 * H + col]);
          const float sc0 = sc.x, sc1 = sc.y, sh0 = sh.x, sh1 = sh.y;
          *reinterpret_cast<float2*>(&Os[(row0 + gq) * kOsPitch + col]) = make_float2(fmaxf(fmaf(acc[0], sc0, sh0), 0.f), fmaxf(fmaf(acc[1], sc1, sh1), 0.f));
          *reinterpret_cast<float2*>(&Os[(row0 + gq + 8) * kOsPitch + col]) = make_float2(fmaxf(fmaf(acc[2], sc0, sh0), 0.f), fmaxf(fmaf(acc[3], sc1, sh1), 0.f));
        }
      }
      __syncwarp();
      // ---- (3) quarter walk: lane = channel pair (2 lane, 2 lane + 1) over the warp's own rows
      float* pm = pmax + (it & 1) * (2 * 4 * 64);
      int* pc = pcell + (it & 1) * 16 + warp * 4;
      {
        const int n = max(0, min(32, rows - warp * 32));
        if (n > 0) {
          const int* cq = cells + warp * 32;
          const float* oq = Os + warp * 32 * kOsPitch + 2 * lane;
          const int fc = cq[0];
          int cur = fc;
          float m0 = 0.f, m1 = 0.f;
          bool first = true;
          for (int r = 0; r < n; ++r) {
            const int c = cq[r];
            if (c != cur) {
              if (first) { *reinterpret_cast<float2*>(pm + warp * 64 + 2 * lane) = make_float2(m0, m1); first = false; }
              else emit_pair<kOutMode>(canvas, cur, 2 * lane, m0, m1);
              cur = c; m0 = 0.f; m1 = 0.f;
            }
            const float2 v = *reinterpret_cast<const float2*>(oq + r * kOsPitch);
            m0 = fmaxf(m0, v.x); m1 = fmaxf(m1, v.y);
          }
          *reinterpret_cast<float2*>(pm + (first ? 0 : 4 * 64) + warp * 64 + 2 * lane) = make_float2(m0, m1);
          if (lane == 0) { pc[0] = fc; pc[1] = cur; }
        }
        if (lane == 0) pc[2] = n;
      }
      __syncthreads();
      // ---- (4) stitch the four quarters with the carried run (thread = channel)
      if (tid < H) {
        const int* pcb = pcell + (it & 1) * 16;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          if (pcb[q * 4 + 2] == 0) continue;
          const int fc = pcb[q * 4], lc = pcb[q * 4 + 1];
          const float fm = pm[q * 64 + tid];
          if (fc != run_cell) {
            if (run_cell >= 0) emit_one<kOutMode>(canvas, run_cell, tid, run_max);
            run_cell = fc; run_max = fm;
          } else {
            run_max = fmaxf(run_max, fm);
          }
          if (lc != fc) {
            emit_one<kOutMode>(canvas, run_cell, tid, run_max);
            run_cell = lc; run_max = pm[4 * 64 + q * 64 + tid];
          }
        }
      }
    }
    if (tid < H && run_cell >= 0) emit_one<kOutMode>(canvas, run_cell, tid, run_max);
  }   // window loop
}

struct SortedWs {
  float4* stats; int* count; int* offsets; int* cursor; int* block_sum; int* total; int* tile_start; int* order; int* ocell;
  size_t bytes;
};
static SortedWs carve_sorted(void* base, int batch, int nx, int ny, long long total_pts) {
  SortedWs w;
  const long long ncells = (long long)batch * nx * ny;
  const long long nblk = (ncells + kCellsPerBlock - 1) / kCellsPerBlock;
  char* p = reinterpret_cast<char*>(base);
  auto take = [&](size_t n) { char* r = p; p += (n + 255) / 256 * 256; return r; };
  w.stats = reinterpret_cast<float4*>(take(stats_bytes(batch, nx, ny)));
  w.count = reinterpret_cast<int*>(take(ncells * 4));
  w.cursor = reinterpret_cast<int*>(take(ncells * 4));
  w.offsets = reinterpret_cast<int*>(take((ncells + 1) * 4));
  w.block_sum = reinterpret_cast<int*>(take((nblk + 1) * 4));
  w.total = reinterpret_cast<int*>(take(256));
  w.tile_start = reinterpret_cast<int*>(take((total_pts / kRows + 2) * 4));
  w.order = reinterpret_cast<int*>(take((size_t)total_pts * 4));
  w.ocell = reinterpret_cast<int*>(take((size_t)total_pts * 4));
  w.bytes = (size_t)(p - reinterpret_cast<char*>(base));
  return w;
}

}  // namespace lavb

using namespace lavb;

extern "C" size_t lavb_pillar_workspace_bytes(int batch, int nx, int ny) {
  // centroid sums + compaction scratch (block counts for up to 2^31 points / 1024) + total
  return stats_bytes(batch, nx, ny) + ((size_t)(1 << 21) + 16) * sizeof(int);
}

extern "C" int lavb_pillar_forward(const float* d_pts, int pt_stride, int d, const long long* h_cloud_start,
                                   const int* h_cloud_count, int batch, float min_x, float max_x, float min_y, float max_y,
                                   float ppm, int nx, int ny, const float* d_w1, const float* d_s1, const float* d_t1, int h1,
                                   const float* d_w2, const float* d_s2, const float* d_t2, int h2, void* d_canvas,
                                   int canvas_dtype, void* d_workspace, void* stream) {
  Clouds clouds;
  if (fill_clouds(clouds, h_cloud_start, h_cloud_count, batch)) return 1;
  LAVB_CHECK_ARG(d == 11 && h1 == 64 && h2 == 64, "pillar_forward: only the v2 configuration (D=11, features [64,64]) is built (got D=%d [%d,%d])", d, h1, h2);
  LAVB_CHECK_ARG(canvas_dtype == LAVB_F32, "pillar_forward: canvas must be fp32");
  LAVB_CHECK_ARG(pt_stride >= d, "pillar_forward: pt_stride < d");
  if (check_grid("pillar_forward", min_x, max_x, min_y, max_y, ppm, nx, ny)) return 1;
  if (check_encoder_ptrs("pillar_forward", d_pts, clouds.cum[batch], d_w1, d_s1, d_t1, d_w2, d_s2, d_t2, d_canvas, 4, d_workspace))
    return 1;
  cudaStream_t st = (cudaStream_t)stream;
  Grid g{min_x, max_x, min_y, max_y, ppm, nx, ny};
  float4* stats = reinterpret_cast<float4*>(d_workspace);
  LAVB_CUDA_OK(cudaMemsetAsync(stats, 0, stats_bytes(batch, nx, ny), st));
  LAVB_CUDA_OK(cudaMemsetAsync(d_canvas, 0, (size_t)batch * nx * ny * h2 * sizeof(float), st));
  const int total = clouds.cum[batch];
  if (total == 0) return 0;
  const int blocks1 = min(ceil_div(total, 256), kNumSMs * 8);
  pillar_stats_kernel<<<blocks1, 256, 0, st>>>(d_pts, pt_stride, clouds, g, stats);
  LAVB_LAUNCH_OK();
  const int blocks2 = min(ceil_div(total, 128), kNumSMs * 4);
  pillar_encode_kernel<11, 64, 64><<<blocks2, 128, 0, st>>>(d_pts, pt_stride, clouds, g, stats, d_w1, d_s1, d_t1, d_w2, d_s2,
                                                              d_t2, reinterpret_cast<float*>(d_canvas));
  LAVB_LAUNCH_OK();
  return 0;
}

extern "C" int lavb_pillar_decorate(const float* d_pts, int pt_stride, int d, const long long* h_cloud_start,
                                    const int* h_cloud_count, int batch, float min_x, float max_x, float min_y, float max_y,
                                    float ppm, int nx, int ny, float* d_feat, int* d_cell, int* h_m, void* d_workspace,
                                    void* stream) {
  Clouds clouds;
  if (fill_clouds(clouds, h_cloud_start, h_cloud_count, batch)) return 1;
  LAVB_CHECK_ARG(d == 11, "pillar_decorate: only D=11 is built (got %d)", d);
  LAVB_CHECK_ARG(pt_stride >= d, "pillar_decorate: pt_stride < d");
  if (check_grid("pillar_decorate", min_x, max_x, min_y, max_y, ppm, nx, ny)) return 1;
  cudaStream_t st = (cudaStream_t)stream;
  Grid g{min_x, max_x, min_y, max_y, ppm, nx, ny};
  float4* stats = reinterpret_cast<float4*>(d_workspace);
  int* scratch = reinterpret_cast<int*>(reinterpret_cast<char*>(d_workspace) + stats_bytes(batch, nx, ny));
  const int total = clouds.cum[batch];
  *h_m = 0;
  if (total == 0) return 0;
  const int nblk = ceil_div(total, kCompactBlock);
  LAVB_CHECK_ARG(nblk <= (1 << 21), "pillar_decorate: too many points");
  int* d_total = scratch + (1 << 21);
  LAVB_CUDA_OK(cudaMemsetAsync(stats, 0, stats_bytes(batch, nx, ny), st));
  pillar_stats_kernel<<<min(ceil_div(total, 256), kNumSMs * 8), 256, 0, st>>>(d_pts, pt_stride, clouds, g, stats);
  LAVB_LAUNCH_OK();
  keep_count_kernel<<<nblk, kCompactBlock, 0, st>>>(d_pts, pt_stride, clouds, g, scratch);
  LAVB_LAUNCH_OK();
  scan_blocks_kernel<<<1, 1024, 0, st>>>(scratch, nblk, d_total);
  LAVB_LAUNCH_OK();
  if (d_feat != nullptr) {
    decorate_write_kernel<11><<<nblk, kCompactBlock, 0, st>>>(d_pts, pt_stride, clouds, g, stats, scratch, d_feat, d_cell);
    LAVB_LAUNCH_OK();
  }
  LAVB_CUDA_OK(cudaMemcpyAsync(h_m, d_total, sizeof(int), cudaMemcpyDeviceToHost, st));
  LAVB_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

extern "C" int lavb_pillar_scatter_max(const float* d_h, const int* d_cell, int m, int c, long long n_cells, float* d_canvas,
                                       int* d_argmax, void* stream) {
  LAVB_CHECK_ARG(m >= 0 && c >= 1 && n_cells >= 0, "pillar_scatter_max: bad shape (m=%d, c=%d, n_cells=%lld)", m, c, n_cells);
  cudaStream_t st = (cudaStream_t)stream;
  LAVB_CUDA_OK(cudaMemsetAsync(d_canvas, 0, (size_t)n_cells * c * sizeof(float), st));
  if (d_argmax) LAVB_CUDA_OK(cudaMemsetAsync(d_argmax, 0x7f, (size_t)n_cells * c * sizeof(int), st));
  const long long mc = (long long)m * c;
  if (mc == 0) return 0;
  scatter_max_kernel<<<ceil_div(mc, 256), 256, 0, st>>>(d_h, d_cell, mc, c, d_canvas);
  LAVB_LAUNCH_OK();
  if (d_argmax) {
    scatter_arg_kernel<<<ceil_div(mc, 256), 256, 0, st>>>(d_h, d_cell, mc, c, d_canvas, d_argmax);
    LAVB_LAUNCH_OK();
  }
  return 0;
}

extern "C" int lavb_pillar_scatter_max_bwd(const float* d_gcanvas, const int* d_argmax, const int* d_cell, int m, int c,
                                                 float* d_gh, void* stream) {
  LAVB_CHECK_ARG(m >= 0 && c >= 1, "pillar_scatter_max_bwd: bad shape (m=%d, c=%d)", m, c);
  const long long mc = (long long)m * c;
  if (mc == 0) return 0;
  scatter_bwd_kernel<<<ceil_div(mc, 256), 256, 0, (cudaStream_t)stream>>>(d_gcanvas, d_argmax, d_cell, mc, c, d_gh);
  LAVB_LAUNCH_OK();
  return 0;
}

extern "C" size_t lavb_pillar_sorted_workspace_bytes(int batch, int nx, int ny, long long total_points) {
  return carve_sorted(nullptr, batch, nx, ny, total_points).bytes;
}

extern "C" int lavb_pillar_forward_sorted(const float* d_pts, int pt_stride, int d, const long long* h_cloud_start,
                                          const int* h_cloud_count, int batch, float min_x, float max_x, float min_y,
                                          float max_y, float ppm, int nx, int ny, const float* d_w1, const float* d_s1,
                                          const float* d_t1, int h1, const float* d_w2, const float* d_s2, const float* d_t2,
                                          int h2, void* d_canvas, int out_mode, void* d_workspace, void* stream) {
  Clouds clouds;
  if (fill_clouds(clouds, h_cloud_start, h_cloud_count, batch)) return 1;
  LAVB_CHECK_ARG(d == 11 && h1 == 64 && h2 == 64, "pillar_forward_sorted: only the v2 configuration (D=11, features [64,64]) is built");
  LAVB_CHECK_ARG(out_mode == 0 || out_mode == 2, "pillar_forward_sorted: out_mode must be 0 (fp32) or 2 (h16) (got %d)", out_mode);
  LAVB_CHECK_ARG(pt_stride >= d, "pillar_forward_sorted: pt_stride < d");
  if (check_grid("pillar_forward_sorted", min_x, max_x, min_y, max_y, ppm, nx, ny)) return 1;
  if (check_encoder_ptrs("pillar_forward_sorted", d_pts, clouds.cum[batch], d_w1, d_s1, d_t1, d_w2, d_s2, d_t2, d_canvas, 16,
                         d_workspace))
    return 1;
  cudaStream_t st = (cudaStream_t)stream;
  Grid g{min_x, max_x, min_y, max_y, ppm, nx, ny};
  const int total = clouds.cum[batch];
  const long long ncells = (long long)batch * nx * ny;
  LAVB_CHECK_ARG(ncells < (1LL << 31), "pillar_forward_sorted: too many cells");
  const SortedWs w = carve_sorted(d_workspace, batch, nx, ny, total);
  const int row_bytes = h2 * (out_mode == 2 ? 2 : 4);        // fp32: 64*4; h16: 64*2
  LAVB_CUDA_OK(cudaMemsetAsync(w.stats, 0, stats_bytes(batch, nx, ny), st));
  LAVB_CUDA_OK(cudaMemsetAsync(w.count, 0, (size_t)ncells * 8 + 512, st));       // count + cursor (adjacent, 256 B padded)
  LAVB_CUDA_OK(cudaMemsetAsync(w.tile_start, 0, ((size_t)total / kRows + 2) * 4, st));
  if (total > 0) {
    pillar_count_kernel<<<min(ceil_div(total, 256), kNumSMs * 8), 256, 0, st>>>(d_pts, pt_stride, clouds, g, w.stats, w.count);
    LAVB_LAUNCH_OK();
  }
  const int nblk = ceil_div(ncells, kCellsPerBlock);
  cell_block_sum_kernel<<<nblk, kCellsPerBlock, 0, st>>>(w.count, ncells, w.block_sum);
  LAVB_LAUNCH_OK();
  scan_blocks_kernel<<<1, 1024, 0, st>>>(w.block_sum, nblk, w.total);
  LAVB_LAUNCH_OK();
  cell_offsets_kernel<<<nblk, kCellsPerBlock, 0, st>>>(w.count, ncells, w.block_sum, w.offsets, w.tile_start, w.total,
                                                       reinterpret_cast<uint4*>(d_canvas), row_bytes / 16);
  LAVB_LAUNCH_OK();
  if (total == 0) return 0;
  pillar_fill_kernel<<<min(ceil_div(total, 256), kNumSMs * 8), 256, 0, st>>>(d_pts, pt_stride, clouds, g, w.offsets, w.cursor,
                                                                             w.order, w.ocell);
  LAVB_LAUNCH_OK();
  const size_t smem = EncSmem::total;
  LAVB_CUDA_OK(ensure_dyn_smem((const void*)pillar_encode_sorted_kernel<11, 0>, 72 * 1024));
  LAVB_CUDA_OK(ensure_dyn_smem((const void*)pillar_encode_sorted_kernel<11, 2>, 72 * 1024));
  const int ntiles = min(ceil_div(total, kRows), kNumSMs * 3);     // persistent: 3 resident blocks per SM
#define LAVB_SORTED_LAUNCH(M)                                                                                                        \
  pillar_encode_sorted_kernel<11, M><<<ntiles, kRows, smem, st>>>(d_pts, pt_stride, clouds, g, w.stats, w.order, w.ocell, w.tile_start, \
                                                                  w.total, d_w1, d_s1, d_t1, d_w2, d_s2, d_t2, d_canvas)
  if (out_mode == 0) LAVB_SORTED_LAUNCH(0); else LAVB_SORTED_LAUNCH(2);
#undef LAVB_SORTED_LAUNCH
  LAVB_LAUNCH_OK();
  return 0;
}
