// Collision and road-departure checks of planned ego trajectories against the recorded traffic and the road plane, one block per
// sample: the ego boxes of the sample's n trajectories x T steps are built in shared memory (one thread per trajectory walks
// its headings in step order), then the threads stride over the (step, map corner) pairs and over the sample's (actor, step)
// records, each record tested against the ego boxes of its step by a separating-axis test in fp64 with no contraction.  The
// first colliding step and its actor row are reduced per trajectory and class with a 64-bit shared-memory minimum.
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kMaxTraj = 8;
constexpr int kMaxSteps = 32;
constexpr int kChunk = 512;          // samples per launch: their actor offsets travel as a kernel argument (2 KB)
constexpr int kOut = 8;              // int32 results per (sample, trajectory)
constexpr unsigned long long kNone = ~0ull;

// one (actor, step) record of the host table (lav_b200.h): label-frame centre, fp64 cos / sin of the relative yaw, box half
// extents, class and presence
struct SafetyActor { double x, y, c, s, e1, e2; int typ, present; };
static_assert(sizeof(SafetyActor) == 56, "SafetyActor layout is part of the ABI (lav_b200.h)");

struct Chunk { int act[kChunk + 1]; };

struct SafetyArgs {
  const float2* traj; const SafetyActor* actors; const double* ego_ext; const unsigned char* map;
  long long map_stride;
  int n, t, h, w;
  double ppm, cx0, cy0, cy1;
  int* out;
};

// a rectangle: centre, unit heading u1 = (hx, hy) (u2 = (-hy, hx)), half extents along u1 and u2
struct Box { double x, y, hx, hy, e1, e2; };

__device__ __forceinline__ double dot(double ax, double ay, double bx, double by) {
  return __dadd_rn(__dmul_rn(ax, bx), __dmul_rn(ay, by));
}

// r(n) = e1 |u1 . n| + e2 |u2 . n|
__device__ __forceinline__ double reach(const Box& b, double nx, double ny) {
  return __dadd_rn(__dmul_rn(b.e1, fabs(dot(b.hx, b.hy, nx, ny))), __dmul_rn(b.e2, fabs(dot(-b.hy, b.hx, nx, ny))));
}

__device__ __forceinline__ bool separated(const Box& a, const Box& b, double dx, double dy, double nx, double ny) {
  return fabs(dot(dx, dy, nx, ny)) >= __dadd_rn(reach(a, nx, ny), reach(b, nx, ny));
}

// the separating-axis test over both boxes' headings and their perpendiculars; touching boxes are separated
__device__ __forceinline__ bool overlap(const Box& a, const Box& b) {
  const double dx = __dsub_rn(b.x, a.x), dy = __dsub_rn(b.y, a.y);
  return !(separated(a, b, dx, dy, a.hx, a.hy) || separated(a, b, dx, dy, -a.hy, a.hx) ||
           separated(a, b, dx, dy, b.hx, b.hy) || separated(a, b, dx, dy, -b.hy, b.hx));
}

__global__ void __launch_bounds__(kThreads) plan_safety_kernel(const SafetyArgs p, const __grid_constant__ Chunk c, int b0) {
  __shared__ double s_x[kMaxTraj * kMaxSteps], s_y[kMaxTraj * kMaxSteps], s_hx[kMaxTraj * kMaxSteps], s_hy[kMaxTraj * kMaxSteps];
  __shared__ unsigned char s_ok[kMaxTraj * kMaxSteps];
  __shared__ unsigned long long s_key[kMaxTraj][2];             // per class: (first step << 32) | actor row
  __shared__ int s_road[kMaxTraj], s_off_map[kMaxTraj], s_invalid[kMaxTraj];
  const int tid = threadIdx.x, bl = blockIdx.x, b = b0 + bl, n = p.n, t = p.t;
  const int a0 = c.act[bl], n_act = c.act[bl + 1] - a0;
  const double e1 = __ldg(p.ego_ext + 2 * b), e2 = __ldg(p.ego_ext + 2 * b + 1);
  if (tid < n) {                                                // the ego boxes: heading of the step, carried below 0.1 m
    const float2* tr = p.traj + ((long long)b * n + tid) * t;
    double px = 0.0, py = 0.0, hx = 0.0, hy = -1.0;
    for (int s = 0; s < t; ++s) {
      const float2 q = __ldg(tr + s);
      const double x = q.x, y = q.y, dx = __dsub_rn(x, px), dy = __dsub_rn(y, py);
      const double len = __dsqrt_rn(dot(dx, dy, dx, dy));
      if (!(len < 0.1)) { hx = __ddiv_rn(dx, len); hy = __ddiv_rn(dy, len); }
      const int i = tid * t + s;
      s_x[i] = x; s_y[i] = y; s_hx[i] = hx; s_hy[i] = hy;
      s_ok[i] = isfinite(x) && isfinite(y) && isfinite(hx) && isfinite(hy);
      px = x; py = y;
    }
    s_key[tid][0] = s_key[tid][1] = kNone;
    s_road[tid] = 0x7fffffff; s_off_map[tid] = 0; s_invalid[tid] = 0;
  }
  __syncthreads();
  const unsigned char* map = p.map + (long long)b * p.map_stride;
  for (int e = tid; e < n * t; e += kThreads) {                // the four corners of each box on the road plane
    const int j = e / t, s = e - j * t;
    if (!s_ok[e]) { atomicAdd(&s_invalid[j], 1); continue; }
    const double ax = __dmul_rn(e1, s_hx[e]), ay = __dmul_rn(e1, s_hy[e]), bx = __dmul_rn(e2, -s_hy[e]), by = __dmul_rn(e2, s_hx[e]);
    bool off_map = false, off_road = false;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const double ux = (k & 2) ? __dsub_rn(s_x[e], ax) : __dadd_rn(s_x[e], ax), uy = (k & 2) ? __dsub_rn(s_y[e], ay) : __dadd_rn(s_y[e], ay);
      const double cx = (k & 1) ? __dsub_rn(ux, bx) : __dadd_rn(ux, bx), cy = (k & 1) ? __dsub_rn(uy, by) : __dadd_rn(uy, by);
      const double col = floor(__dadd_rn(__dmul_rn(cx, p.ppm), p.cx0));
      const double row = floor(__dadd_rn(__dadd_rn(__dmul_rn(cy, p.ppm), p.cy0), p.cy1));
      if (!(col >= 0.0 && col < (double)p.w && row >= 0.0 && row < (double)p.h)) { off_map = true; continue; }
      if (map[(long long)row * p.w + (long long)col] == 0) off_road = true;
    }
    if (off_map) atomicAdd(&s_off_map[j], 1);
    if (off_road) atomicMin(&s_road[j], s + 1);
  }
  const SafetyActor* act = p.actors + (long long)a0 * t;
  for (long long r = tid; r < (long long)n_act * t; r += kThreads) {   // every present (actor, step) against that step's boxes
    const SafetyActor A = act[r];
    if (!A.present || (A.typ != 0 && A.typ != 1)) continue;
    const int a = (int)(r / t), s = (int)(r - (long long)a * t), cls = A.typ == 1 ? 0 : 1;
    const Box other{A.x, A.y, A.s, -A.c, A.e1, A.e2};             // heading (sin psi, -cos psi) in the label frame
    for (int j = 0; j < n; ++j) {
      const int i = j * t + s;
      if (!s_ok[i]) continue;
      const Box ego{s_x[i], s_y[i], s_hx[i], s_hy[i], e1, e2};
      if (overlap(ego, other)) atomicMin(&s_key[j][cls], ((unsigned long long)(s + 1) << 32) | (unsigned)a);
    }
  }
  __syncthreads();
  if (tid < n) {
    int* o = p.out + ((long long)b * n + tid) * kOut;
    const unsigned long long kv = s_key[tid][0], kp = s_key[tid][1];
    const int vs = kv == kNone ? -1 : (int)(kv >> 32), ps = kp == kNone ? -1 : (int)(kp >> 32);
    o[0] = vs; o[1] = kv == kNone ? -1 : (int)(kv & 0xffffffffu);
    o[2] = ps; o[3] = kp == kNone ? -1 : (int)(kp & 0xffffffffu);
    o[4] = s_road[tid] == 0x7fffffff ? -1 : s_road[tid];
    o[5] = s_off_map[tid]; o[6] = s_invalid[tid];
    o[7] = vs < 0 ? ps : ps < 0 ? vs : min(vs, ps);
  }
}

}  // namespace

extern "C" int lavb_plan_safety(const float* d_traj, int b, int n, int t, const void* d_actors, int n_actors,
                                const int* h_offsets, const double* d_ego_ext, const uint8_t* d_map, long long map_stride, int h,
                                int w, float ppm, float cx0, float cy0, float cy1, int* d_out, void* stream) {
  LAVB_CHECK_ARG(b >= 0 && h > 0 && w > 0, "plan_safety: bad sizes (b %d, map %d x %d)", b, h, w);
  LAVB_CHECK_ARG(n >= 1 && n <= kMaxTraj, "plan_safety: %d trajectories per sample outside 1..%d", n, kMaxTraj);
  LAVB_CHECK_ARG(t >= 1 && t <= kMaxSteps, "plan_safety: %d steps outside 1..%d", t, kMaxSteps);
  LAVB_CHECK_ARG(map_stride >= (long long)h * w, "plan_safety: map stride %lld below the %d x %d plane", map_stride, h, w);
  LAVB_CHECK_ARG(ppm > 0.f && isfinite(ppm) && isfinite(cx0) && isfinite(cy0) && isfinite(cy1),
                 "plan_safety: the grid (ppm %g, cx0 %g, cy0 %g, cy1 %g) must be finite with ppm > 0", ppm, cx0, cy0, cy1);
  LAVB_CHECK_ARG(n_actors >= 0 && h_offsets, "plan_safety: missing host offsets (%d actor rows)", n_actors);
  LAVB_CHECK_ARG(h_offsets[0] >= 0 && h_offsets[b] <= n_actors, "plan_safety: actor offsets [%d, %d] run outside the %d actor rows",
                 h_offsets[0], h_offsets[b], n_actors);
  for (int i = 0; i < b; ++i)
    LAVB_CHECK_ARG(h_offsets[i] <= h_offsets[i + 1], "plan_safety: actor offsets of sample %d are not monotone (%d -> %d)", i,
                   h_offsets[i], h_offsets[i + 1]);
  if (b == 0) return 0;
  LAVB_CHECK_ARG(d_traj && d_ego_ext && d_map && d_out && (d_actors || h_offsets[b] == h_offsets[0]), "plan_safety: null pointer");
  LAVB_CHECK_ARG((uintptr_t)d_traj % 8 == 0 && (uintptr_t)d_actors % 8 == 0 && (uintptr_t)d_ego_ext % 8 == 0 &&
                 (uintptr_t)d_out % 4 == 0, "plan_safety: traj, actors and ego_ext must be 8-byte aligned, out 4-byte aligned");
  SafetyArgs a;
  a.traj = reinterpret_cast<const float2*>(d_traj); a.actors = reinterpret_cast<const SafetyActor*>(d_actors);
  a.ego_ext = d_ego_ext; a.map = d_map; a.map_stride = map_stride;
  a.n = n; a.t = t; a.h = h; a.w = w;
  a.ppm = (double)ppm; a.cx0 = (double)cx0; a.cy0 = (double)cy0; a.cy1 = (double)cy1;
  a.out = d_out;
  cudaStream_t st = (cudaStream_t)stream;
  for (int b0 = 0; b0 < b; b0 += kChunk) {
    const int nb = b - b0 < kChunk ? b - b0 : kChunk;
    Chunk ch;
    for (int i = 0; i <= nb; ++i) ch.act[i] = h_offsets[b0 + i];
    plan_safety_kernel<<<nb, kThreads, 0, st>>>(a, ch, b0);
    LAVB_LAUNCH_OK();
  }
  return 0;
}
