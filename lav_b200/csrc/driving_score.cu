// The terms of a PDM-style driving score of planned ego trajectories against the recorded (non-reactive) traffic and the road
// plane, one warp per (sample, trajectory) and one block per sample.  Lane 0 walks the ego's steps in order (centres, carried
// headings, velocities) and the expert polyline (its arc length and the projection of the trajectory's last point); then the
// lanes take one step each for the road corners and the comfort terms, and stride over the sample's actor rows for the
// collisions and the time-to-collision projections, each row walked in step order so that "new at step t" needs no second
// pass.  The first (step, actor row) of each kind is reduced over the warp with a 64-bit minimum.  Geometry is fp64 with no
// contraction, in plan_safety.cu's order.
#include "common.cuh"

namespace {

constexpr int kMaxTraj = 8;
constexpr int kMaxSteps = 32;       // one lane per step 1..T
constexpr int kMaxK = 64;           // time-to-collision projections per step
constexpr int kChunk = 512;         // samples per launch: their actor offsets travel as a kernel argument (2 KB)
constexpr int kOut = 16;            // int32 results per (sample, trajectory)
constexpr unsigned long long kNone = ~0ull;
constexpr unsigned kAll = 0xffffffffu;
constexpr double kPi = 3.141592653589793, kTwoPi = 6.283185307179586;
constexpr double kStopped = 0.05;   // m/s: below this the ego is stopped

// the comfort bounds (nuPlan's): longitudinal acceleration, its jerk, yaw rate, yaw acceleration, lateral acceleration
constexpr double kAccMin = -4.05, kAccMax = 2.40, kJerk = 4.13, kYawRate = 0.95, kYawAcc = 1.93, kLatAcc = 4.89;

// one (actor, step) record of the host table (lav_b200.h), plan_safety's layout
struct Actor { double x, y, c, s, e1, e2; int typ, present; };
static_assert(sizeof(Actor) == 56, "the actor record layout is part of the ABI (lav_b200.h)");

struct Chunk { int act[kChunk + 1]; };

struct ScoreArgs {
  const float2* traj; const float2* expert; const Actor* actors; const double* ego_ext; const unsigned char* map;
  long long map_stride;
  int n, t, h, w, k;
  double ppm, cx0, cy0, cy1, dt;
  double* ep; int* out;
};

struct Box { double x, y, hx, hy, e1, e2; };

__device__ __forceinline__ double dot(double ax, double ay, double bx, double by) {
  return __dadd_rn(__dmul_rn(ax, bx), __dmul_rn(ay, by));
}

__device__ __forceinline__ double reach(const Box& b, double nx, double ny) {
  return __dadd_rn(__dmul_rn(b.e1, fabs(dot(b.hx, b.hy, nx, ny))), __dmul_rn(b.e2, fabs(dot(-b.hy, b.hx, nx, ny))));
}

__device__ __forceinline__ bool separated(const Box& a, const Box& b, double dx, double dy, double nx, double ny) {
  return fabs(dot(dx, dy, nx, ny)) >= __dadd_rn(reach(a, nx, ny), reach(b, nx, ny));
}

// plan_safety.cu's separating-axis test; touching boxes are separated
__device__ __forceinline__ bool overlap(const Box& a, const Box& b) {
  const double dx = __dsub_rn(b.x, a.x), dy = __dsub_rn(b.y, a.y);
  return !(separated(a, b, dx, dy, a.hx, a.hy) || separated(a, b, dx, dy, -a.hy, a.hx) ||
           separated(a, b, dx, dy, b.hx, b.hy) || separated(a, b, dx, dy, -b.hy, b.hx));
}

// the actor's centre behind the ego's rear face: (q - p) . h < -e1
__device__ __forceinline__ bool behind(const Box& ego, double qx, double qy) {
  return dot(__dsub_rn(qx, ego.x), __dsub_rn(qy, ego.y), ego.hx, ego.hy) < -ego.e1;
}

__device__ __forceinline__ unsigned long long warp_min(unsigned long long v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = min(v, __shfl_xor_sync(kAll, v, o));
  return v;
}

__device__ __forceinline__ double wrap(double d) {       // to (-pi, pi] from (-2 pi, 2 pi]
  return d > kPi ? __dsub_rn(d, kTwoPi) : d <= -kPi ? __dadd_rn(d, kTwoPi) : d;
}

__global__ void __launch_bounds__(kMaxTraj * 32) driving_score_kernel(const ScoreArgs p, const __grid_constant__ Chunk c, int b0) {
  // per warp, steps 0..T: centre, heading, velocity, speed, yaw
  __shared__ double s_x[kMaxTraj][kMaxSteps + 1], s_y[kMaxTraj][kMaxSteps + 1], s_hx[kMaxTraj][kMaxSteps + 1],
      s_hy[kMaxTraj][kMaxSteps + 1], s_vx[kMaxTraj][kMaxSteps + 1], s_vy[kMaxTraj][kMaxSteps + 1],
      s_sp[kMaxTraj][kMaxSteps + 1], s_psi[kMaxTraj][kMaxSteps + 1];
  const int j = threadIdx.x >> 5, lane = threadIdx.x & 31, bl = blockIdx.x, b = b0 + bl, t = p.t;
  const int a0 = c.act[bl], n_act = c.act[bl + 1] - a0;
  const double e1 = __ldg(p.ego_ext + 2 * b), e2 = __ldg(p.ego_ext + 2 * b + 1), dt = p.dt;
  double* sx = s_x[j]; double* sy = s_y[j]; double* shx = s_hx[j]; double* shy = s_hy[j];
  double* svx = s_vx[j]; double* svy = s_vy[j]; double* ssp = s_sp[j]; double* spsi = s_psi[j];
  double L = 0.0;
  if (lane == 0) {                                   // the ego's steps: plan_safety's headings, velocities at dt
    const float2* tr = p.traj + ((long long)b * p.n + j) * t;
    double px = 0.0, py = 0.0, hx = 0.0, hy = -1.0;
    sx[0] = 0.0; sy[0] = 0.0; shx[0] = 0.0; shy[0] = -1.0; svx[0] = 0.0; svy[0] = 0.0; ssp[0] = 0.0;
    for (int s = 1; s <= t; ++s) {
      const float2 q = __ldg(tr + s - 1);
      const double x = q.x, y = q.y, dx = __dsub_rn(x, px), dy = __dsub_rn(y, py);
      const double len = __dsqrt_rn(dot(dx, dy, dx, dy));
      if (!(len < 0.1)) { hx = __ddiv_rn(dx, len); hy = __ddiv_rn(dy, len); }
      const double vx = __ddiv_rn(dx, dt), vy = __ddiv_rn(dy, dt);
      sx[s] = x; sy[s] = y; shx[s] = hx; shy[s] = hy; svx[s] = vx; svy[s] = vy;
      ssp[s] = __dsqrt_rn(dot(vx, vy, vx, vy));
      px = x; py = y;
    }
  }
  __syncwarp();
  const int s = lane + 1;                            // this lane's step
  const bool has = s <= t;
  const bool ok = !has || (isfinite(sx[s]) && isfinite(sy[s]) && isfinite(shx[s]) && isfinite(shy[s]));
  const unsigned bad = __ballot_sync(kAll, !ok);
  const bool valid = bad == 0u;

  // road: plan_safety's corner rule at every valid step
  bool off_road = false;
  if (has && ok) {
    const unsigned char* map = p.map + (long long)b * p.map_stride;
    const double ax = __dmul_rn(e1, shx[s]), ay = __dmul_rn(e1, shy[s]), bx = __dmul_rn(e2, -shy[s]), by = __dmul_rn(e2, shx[s]);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const double ux = (k & 2) ? __dsub_rn(sx[s], ax) : __dadd_rn(sx[s], ax), uy = (k & 2) ? __dsub_rn(sy[s], ay) : __dadd_rn(sy[s], ay);
      const double cx = (k & 1) ? __dsub_rn(ux, bx) : __dadd_rn(ux, bx), cy = (k & 1) ? __dsub_rn(uy, by) : __dadd_rn(uy, by);
      const double col = floor(__dadd_rn(__dmul_rn(cx, p.ppm), p.cx0));
      const double row = floor(__dadd_rn(__dadd_rn(__dmul_rn(cy, p.ppm), p.cy0), p.cy1));
      if (!(col >= 0.0 && col < (double)p.w && row >= 0.0 && row < (double)p.h)) continue;
      if (map[(long long)row * p.w + (long long)col] == 0) off_road = true;
    }
  }
  const unsigned road = __ballot_sync(kAll, off_road);

  // comfort: finite differences at dt of the speed and of the yaw of the heading
  if (has) spsi[s] = atan2(shy[s], shx[s]);
  __syncwarp();
  unsigned fail[5] = {0u, 0u, 0u, 0u, 0u};
  {
    bool f_acc = false, f_jerk = false, f_rate = false, f_yacc = false, f_lat = false;
    if (valid && has && s >= 2) {
      const double acc = __ddiv_rn(__dsub_rn(ssp[s], ssp[s - 1]), dt);
      const double rate = __ddiv_rn(wrap(__dsub_rn(spsi[s], spsi[s - 1])), dt);
      const double lat = __dmul_rn(ssp[s], rate);
      f_acc = acc < kAccMin || acc > kAccMax;
      f_rate = fabs(rate) > kYawRate;
      f_lat = fabs(lat) > kLatAcc;
      if (s >= 3) {
        const double acc0 = __ddiv_rn(__dsub_rn(ssp[s - 1], ssp[s - 2]), dt);
        const double rate0 = __ddiv_rn(wrap(__dsub_rn(spsi[s - 1], spsi[s - 2])), dt);
        f_jerk = fabs(__ddiv_rn(__dsub_rn(acc, acc0), dt)) > kJerk;
        f_yacc = fabs(__ddiv_rn(__dsub_rn(rate, rate0), dt)) > kYawAcc;
      }
    }
    fail[0] = __ballot_sync(kAll, f_acc); fail[1] = __ballot_sync(kAll, f_jerk); fail[2] = __ballot_sync(kAll, f_rate);
    fail[3] = __ballot_sync(kAll, f_yacc); fail[4] = __ballot_sync(kAll, f_lat);
  }

  // progress: the expert's arc length L and the arc-length position of the last point, closest point, first segment on ties
  double prog = __longlong_as_double(0x7ff8000000000000ll);
  if (lane == 0) {
    const float2* ex = p.expert + (long long)b * t;
    const double Px = sx[t], Py = sy[t];
    double qx = 0.0, qy = 0.0, best = __longlong_as_double(0x7ff0000000000000ll);
    for (int k = 1; k <= t; ++k) {
      const float2 q = __ldg(ex + k - 1);
      const double nx = q.x, ny = q.y, dx = __dsub_rn(nx, qx), dy = __dsub_rn(ny, qy);
      const double dd = dot(dx, dy, dx, dy), len = __dsqrt_rn(dd);
      if (valid) {
        double u = dd > 0.0 ? __ddiv_rn(dot(__dsub_rn(Px, qx), __dsub_rn(Py, qy), dx, dy), dd) : 0.0;
        u = u < 0.0 ? 0.0 : u > 1.0 ? 1.0 : u;
        const double rx = __dsub_rn(Px, __dadd_rn(qx, __dmul_rn(u, dx))), ry = __dsub_rn(Py, __dadd_rn(qy, __dmul_rn(u, dy)));
        const double d2 = dot(rx, ry, rx, ry);
        if (d2 < best) { best = d2; prog = __dadd_rn(L, __dmul_rn(u, len)); }
      }
      L = __dadd_rn(L, len);
      qx = nx; qy = ny;
    }
  }

  // collisions and time to collision against every actor row, each walked in step order
  unsigned long long k_fault = kNone, k_exempt = kNone, k_ttc = kNone;
  if (valid) {
    const int t1 = t + 1;
    const Box origin{0.0, 0.0, 0.0, -1.0, e1, e2};
    for (int a = lane; a < n_act; a += 32) {
      const Actor* R = p.actors + (long long)(a0 + a) * t1;
      Actor P = R[0];
      bool live = P.present && (P.typ == 0 || P.typ == 1);
      bool was = live && overlap(origin, Box{P.x, P.y, P.s, -P.c, P.e1, P.e2});
      for (int st = 1; st <= t; ++st) {
        const Actor A = R[st];
        live = A.present && (A.typ == 0 || A.typ == 1);
        const unsigned long long key = ((unsigned long long)st << 32) | (unsigned)a;
        const Box ego{sx[st], sy[st], shx[st], shy[st], e1, e2}, other{A.x, A.y, A.s, -A.c, A.e1, A.e2};
        const bool now = live && overlap(ego, other);
        if (now && !was) {
          if (ssp[st] < kStopped || behind(ego, A.x, A.y)) k_exempt = min(k_exempt, key);
          else k_fault = min(k_fault, key);
        }
        if (live && !now && !(ssp[st] < kStopped) && key < k_ttc) {
          const bool moving = P.present && A.present;
          const double ux = moving ? __ddiv_rn(__dsub_rn(A.x, P.x), dt) : 0.0, uy = moving ? __ddiv_rn(__dsub_rn(A.y, P.y), dt) : 0.0;
          for (int k = 1; k <= p.k; ++k) {
            const double tau = __dmul_rn((double)k, dt);
            const Box e{__dadd_rn(ego.x, __dmul_rn(tau, svx[st])), __dadd_rn(ego.y, __dmul_rn(tau, svy[st])), ego.hx, ego.hy, e1, e2};
            const double qx = __dadd_rn(A.x, __dmul_rn(tau, ux)), qy = __dadd_rn(A.y, __dmul_rn(tau, uy));
            if (overlap(e, Box{qx, qy, A.s, -A.c, A.e1, A.e2})) {     // the projected collision, judged where it begins
              if (!behind(e, qx, qy)) k_ttc = key;
              break;
            }
          }
        }
        was = now;
        P = A;
      }
    }
  }
  k_fault = warp_min(k_fault); k_exempt = warp_min(k_exempt); k_ttc = warp_min(k_ttc);

  if (lane == 0) {
    const long long o_i = (long long)b * p.n + j;
    int* o = p.out + o_i * kOut;
    const Actor* base = p.actors + (long long)a0 * (t + 1);
    auto put = [&](int* f, unsigned long long key, bool typ) {
      const int st = key == kNone ? -1 : (int)(key >> 32), row = key == kNone ? -1 : (int)(key & 0xffffffffu);
      f[0] = st; f[1] = row;
      if (typ) f[2] = key == kNone ? -1 : base[(long long)row * (t + 1) + st].typ;
    };
    put(o + 0, k_fault, true); put(o + 3, k_exempt, true); put(o + 6, k_ttc, false);
    o[8] = road ? __ffs(road) : -1;
    int mask = 0;
    for (int q = 0; q < 5; ++q) {
      mask |= fail[q] ? 1 << q : 0;
      o[10 + q] = fail[q] ? __ffs(fail[q]) : -1;
    }
    o[9] = mask;
    o[15] = bad ? __ffs(bad) : -1;
    p.ep[2 * o_i] = prog; p.ep[2 * o_i + 1] = L;
  }
}

}  // namespace

extern "C" int lavb_driving_score(const float* d_traj, const float* d_expert, int b, int n, int t, const void* d_actors, int n_actors,
                                  const int* h_offsets, const double* d_ego_ext, const uint8_t* d_map, long long map_stride, int h,
                                  int w, float ppm, float cx0, float cy0, float cy1, double dt, double* d_ep, int* d_out,
                                  void* stream) {
  LAVB_CHECK_ARG(b >= 0 && h > 0 && w > 0, "driving_score: bad sizes (b %d, map %d x %d)", b, h, w);
  LAVB_CHECK_ARG(n >= 1 && n <= kMaxTraj, "driving_score: %d trajectories per sample outside 1..%d", n, kMaxTraj);
  LAVB_CHECK_ARG(t >= 1 && t <= kMaxSteps, "driving_score: %d steps outside 1..%d", t, kMaxSteps);
  LAVB_CHECK_ARG(map_stride >= (long long)h * w, "driving_score: map stride %lld below the %d x %d plane", map_stride, h, w);
  LAVB_CHECK_ARG(ppm > 0.f && isfinite(ppm) && isfinite(cx0) && isfinite(cy0) && isfinite(cy1),
                 "driving_score: the grid (ppm %g, cx0 %g, cy0 %g, cy1 %g) must be finite with ppm > 0", ppm, cx0, cy0, cy1);
  LAVB_CHECK_ARG(dt > 0.0 && isfinite(dt), "driving_score: step period %g s must be finite and > 0", dt);
  const double kf = floor(1.0 / dt + 1e-9);
  LAVB_CHECK_ARG(kf <= kMaxK, "driving_score: step period %g s gives %g projections per second, over %d", dt, kf, kMaxK);
  LAVB_CHECK_ARG(n_actors >= 0 && h_offsets, "driving_score: missing host offsets (%d actor rows)", n_actors);
  LAVB_CHECK_ARG(h_offsets[0] >= 0 && h_offsets[b] <= n_actors, "driving_score: actor offsets [%d, %d] run outside the %d actor rows",
                 h_offsets[0], h_offsets[b], n_actors);
  for (int i = 0; i < b; ++i)
    LAVB_CHECK_ARG(h_offsets[i] <= h_offsets[i + 1], "driving_score: actor offsets of sample %d are not monotone (%d -> %d)", i,
                   h_offsets[i], h_offsets[i + 1]);
  if (b == 0) return 0;
  LAVB_CHECK_ARG(d_traj && d_expert && d_ego_ext && d_map && d_ep && d_out && (d_actors || h_offsets[b] == h_offsets[0]),
                 "driving_score: null pointer");
  LAVB_CHECK_ARG((uintptr_t)d_traj % 8 == 0 && (uintptr_t)d_expert % 8 == 0 && (uintptr_t)d_actors % 8 == 0 &&
                 (uintptr_t)d_ego_ext % 8 == 0 && (uintptr_t)d_ep % 8 == 0 && (uintptr_t)d_out % 4 == 0,
                 "driving_score: traj, expert, actors, ego_ext and ep must be 8-byte aligned, out 4-byte aligned");
  ScoreArgs a;
  a.traj = reinterpret_cast<const float2*>(d_traj); a.expert = reinterpret_cast<const float2*>(d_expert);
  a.actors = reinterpret_cast<const Actor*>(d_actors); a.ego_ext = d_ego_ext; a.map = d_map; a.map_stride = map_stride;
  a.n = n; a.t = t; a.h = h; a.w = w; a.k = (int)kf;
  a.ppm = (double)ppm; a.cx0 = (double)cx0; a.cy0 = (double)cy0; a.cy1 = (double)cy1; a.dt = dt;
  a.ep = d_ep; a.out = d_out;
  cudaStream_t st = (cudaStream_t)stream;
  for (int b0 = 0; b0 < b; b0 += kChunk) {
    const int nb = b - b0 < kChunk ? b - b0 : kChunk;
    Chunk ch;
    for (int i = 0; i <= nb; ++i) ch.act[i] = h_offsets[b0 + i];
    driving_score_kernel<<<nb, 32 * n, 0, st>>>(a, ch, b0);
    LAVB_LAUNCH_OK();
  }
  return 0;
}
