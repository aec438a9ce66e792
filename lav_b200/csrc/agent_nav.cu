// The agent's localisation and route following (lav_agent_fast.py:215-226, 280-308, 338) for b agents, one thread per agent:
//  * lavb_agent_nav_front: the compass NaN rule, EKF.init on an agent's first frame, the pose, Waypointer.tick, RoutePlanner.run_step,
//    the command mapping, the lane-change rule and the target point in the ego frame;
//  * lavb_agent_nav_update: EKF.step after the controls (ekf.py:45-91);
//  * lavb_stack_job_poses: the pose fields of the sweep stack's job table (StaticFramePipeline._fill_jobs) from a device pose ring.
// The route scans of waypointer.py / planner.py are O(1): only node current_idx + 1 can satisfy i - current_idx == 1.  Every
// arithmetic operation is a correctly rounded fp64 intrinsic in numpy's order, so nothing is contracted; only cos, sin, tan and
// atan differ from the host's libm (by an ulp or two).
#include "common.cuh"

namespace {

constexpr int kThreads = 128;
constexpr double kPi = 3.141592653589793;                  // math.pi
constexpr double kHalfPi = kPi / 2;                         // math.pi / 2 == np.pi / 2
constexpr double kEarth = 6371e3;                           // EKF / Waypointer / RoutePlanner .EARTH_RADIUS
constexpr double kDeg = kPi / 180;                          // (math.pi / 180)
// EKF(1, 1.477531, 1.393600) with its defaults (lav_agent_fast.py:137, ekf.py:8-31)
constexpr double kLr = 1.393600;
constexpr double kL = 1.477531 + 1.393600;
constexpr double kMaxSteer = 70 * kPi / 180.;
constexpr double kDt = 1. / 20;
constexpr double kQ = 1e-7;
constexpr double kXyNoise = kEarth * 0.000005 * kPi / 180.;
constexpr double kCompassNoise = 1e-7 * kPi / 180.;
constexpr double kRxy = kXyNoise * kXyNoise;                // xy_noise**2 (equal to the product for this value)
constexpr double kRc = kCompassNoise * kCompassNoise;
// Waypointer defaults and the agent's settings (waypointer.py:11-20, lav_agent_fast.py:282-284), RoutePlanner defaults
constexpr double kThreshBefore = 4.5, kThreshAfter = 3.0;
constexpr double kCurrThreshold = 20, kNextThreshold = 75;
constexpr int kLaneFollow = 4, kChangeLaneLeft = 5, kChangeLaneRight = 6;   // RoadOption values
constexpr int kLaneChangeTicks = 300;                       // {4: 300, 5: 300}

__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }

// np.linalg.norm([dx, dy]) = sqrt(dx * dx + dy * dy)
__device__ __forceinline__ double norm2(double dx, double dy) { return __dsqrt_rn(dadd(dmul(dx, dx), dmul(dy, dy))); }

// latlon_to_xy (ekf.py:94-99, waypointer.py:98-103, planner.py:53-58): x = R * lat * (pi / 180), y = R * lon * (pi / 180) * scale
__device__ __forceinline__ double lat_x(double lat) { return dmul(dmul(kEarth, lat), kDeg); }
__device__ __forceinline__ double lon_y(double lon, double scale) { return dmul(dmul(dmul(kEarth, lon), kDeg), scale); }

// (start, count) of agent i's route in the node table, or false when the entry is not a route
__device__ __forceinline__ bool route_of(const int* route, int i, int n_nodes, int& start, int& count) {
  start = __ldg(route + 2 * i);
  count = __ldg(route + 2 * i + 1);
  return start >= 0 && count >= 1 && count <= n_nodes - start;
}

__global__ void __launch_bounds__(kThreads) nav_front_kernel(int b, const double2* __restrict__ nodes,
                                                               const int* __restrict__ node_cmd, int n_nodes,
                                                               const int* __restrict__ route, const double2* __restrict__ gnss,
                                                               const double* __restrict__ compass, lavb_nav_state* __restrict__ state,
                                                               int* __restrict__ cmds, float2* __restrict__ nxps,
                                                               double* __restrict__ poses, int* __restrict__ flags) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= b) return;
  const double nan = __longlong_as_double(0x7ff8000000000000LL);
  int start, n;
  if (!route_of(route, i, n_nodes, start, n)) {
    cmds[i] = 3; nxps[i] = make_float2(__double2float_rn(nan), __double2float_rn(nan));
    poses[3 * i] = nan; poses[3 * i + 1] = nan; poses[3 * i + 2] = nan;
    flags[i] = LAVB_NAV_NO_ROUTE;
    return;
  }
  lavb_nav_state s = state[i];
  const double2 g = __ldg(gnss + i);
  const double raw = __ldg(compass + i);
  const double cmp = isnan(raw) ? 0.0 : raw;                                               // :219-220
  if (s.frames == 0) {                                                                     // :222-224, ekf.init
    s.ekf_x[0] = lat_x(g.x);
    s.ekf_x[1] = lon_y(g.y, s.ekf_scale);
    s.ekf_x[2] = dsub(cmp, kHalfPi);
    s.ekf_p[0] = s.ekf_p[1] = s.ekf_p[2] = 0.0;
  }
  if (s.frames < 0x40000000) ++s.frames;
  poses[3 * i] = s.ekf_x[0]; poses[3 * i + 1] = s.ekf_x[1]; poses[3 * i + 2] = s.ekf_x[2];    // :226
  if (s.frames <= 1) {                                                                     // :235-237, the early return
    cmds[i] = 3; nxps[i] = make_float2(0.f, 0.f);
    flags[i] = LAVB_NAV_FIRST_FRAME;
    state[i] = s;
    return;
  }
  const double cx = lat_x(g.x), cy = lon_y(g.y, s.route_scale);
  const double2* nd = nodes + start;
  const int* nc = node_cmd + start;
  if (s.frames == 2) {                                                                     // :280-286, the planners' constructors
    s.wp_x = cx; s.wp_y = cy; s.wp_cmd = kLaneFollow; s.wp_idx = -1;
    const double2 n0 = __ldg(nd);
    s.rp_x = n0.x; s.rp_y = n0.y; s.rp_idx = 0;
  }
  // Waypointer.tick (waypointer.py:50-96): the loop can only take node current_idx + 1; after it, i is that node when it was
  // taken and len - 1 otherwise, and the lane-change look-ahead starts from that i
  int last = n - 1;
  const int j = s.wp_idx + 1;
  if (j < n) {
    const double2 w = __ldg(nd + j);
    const int wc = __ldg(nc + j);
    const double thr = (s.wp_cmd == kLaneFollow && wc != kLaneFollow) ? kThreshBefore : kThreshAfter;
    if (norm2(dsub(cx, w.x), dsub(cy, w.y)) < thr) {
      s.wp_x = w.x; s.wp_y = w.y; s.wp_cmd = wc; s.wp_idx = j;
      last = j;
    }
  }
  {
    int cmd = s.wp_cmd;
    for (int look = 0; last + 1 < n && look < 3; ++look) {                                 // :78-93
      if (cmd != kLaneFollow) break;
      const int wc = __ldg(nc + last + 1);
      if (wc == kChangeLaneLeft || wc == kChangeLaneRight) {
        const double2 w = __ldg(nd + last + 1);
        s.wp_x = w.x; s.wp_y = w.y; s.wp_cmd = wc; s.wp_idx = last + 1;
        break;
      }
      cmd = wc;
      ++last;
    }
  }
  // RoutePlanner.run_step (planner.py:34-50)
  {
    const double curr = norm2(dsub(s.rp_x, cx), dsub(s.rp_y, cy));
    const int k = s.rp_idx + 1;
    if (k < n) {
      const double2 w = __ldg(nd + k);
      if (norm2(dsub(w.x, cx), dsub(w.y, cy)) < kNextThreshold && curr < kCurrThreshold) {
        s.rp_x = w.x; s.rp_y = w.y; s.rp_idx = k;
      }
    }
  }
  const double wx = dsub(s.rp_x, cx), wy = dsub(s.rp_y, cy);
  int cv = s.wp_cmd - 1;                                                                   // :291-292
  if (cv < 0) cv = 3;
  if (cv == 4 || cv == 5) {                                                                // :294-302
    if (s.lane_changed >= 0 && cv != s.lane_changed) s.lane_counter = 0;
    if (s.lane_counter < 0x40000000) ++s.lane_counter;
    s.lane_changed = s.lane_counter > kLaneChangeTicks ? cv : -1;
  } else {
    s.lane_counter = 0;
    s.lane_changed = -1;
  }
  int fl = 0;
  if (cv == s.lane_changed) { cv = 3; fl |= LAVB_NAV_LANE_HELD; }                          // :304-305
  // _rotate(wx, wy, -imu[-1] + pi/2) with the raw compass (:308, :520-526), then nxps = [-wx, -wy] in fp32 (:314)
  const double th = dadd(-raw, kHalfPi);
  double sn, cs;
  sincos(th, &sn, &cs);
  const double rx = dadd(dmul(cs, wx), dmul(-sn, wy)), ry = dadd(dmul(sn, wx), dmul(cs, wy));
  cmds[i] = cv;
  nxps[i] = make_float2(__double2float_rn(-rx), __double2float_rn(-ry));
  flags[i] = fl;
  state[i] = s;
}

// EKF.step(spd, steer, lat, lon, compass - pi/2) (ekf.py:45-91) with F = H = I and diagonal Q, R and P: the covariance stays
// diagonal and the gain K = P (P + R)^-1 is diagonal; every product numpy forms with a zero of K is kept, so a non-finite
// innovation spreads to all three states as it does in K_kp @ y_kp
__global__ void __launch_bounds__(kThreads) nav_update_kernel(int b, const float* __restrict__ control,
                                                                const double* __restrict__ speed, const double2* __restrict__ gnss,
                                                                const double* __restrict__ compass, lavb_nav_state* __restrict__ state) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= b) return;
  lavb_nav_state s = state[i];
  if (s.frames < 2) return;                                                                // the first frame has no EKF step
  const double spd = __ldg(speed + i), steer = (double)__ldg(control + 3LL * i);
  const double2 g = __ldg(gnss + i);
  const double raw = __ldg(compass + i);
  const double z[3] = {lat_x(g.x), lon_y(g.y, s.ekf_scale), dsub(isnan(raw) ? 0.0 : raw, kHalfPi)};
  // kbm_step (ekf.py:74-91), tan(theta_k) as written
  const double xk = s.ekf_x[0], yk = s.ekf_x[1], tk = s.ekf_x[2];
  const double beta = atan(__ddiv_rn(dmul(kLr, tan(dmul(steer, kMaxSteer))), kL));
  const double xp[3] = {dadd(xk, dmul(dmul(spd, cos(dadd(tk, beta))), kDt)),
                        dadd(yk, dmul(dmul(spd, sin(dadd(tk, beta))), kDt)),
                        dadd(tk, dmul(__ddiv_rn(dmul(dmul(spd, tan(tk)), cos(beta)), kL), kDt))};
  double y[3], k[3], pp[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    pp[a] = dadd(s.ekf_p[a], kQ);                                                          // F P F^T + Q
    k[a] = dmul(pp[a], __drcp_rn(dadd(pp[a], a < 2 ? kRxy : kRc)));                        // P H^T inv(H P H^T + R)
    y[a] = dsub(z[a], xp[a]);
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    double c = a == 0 ? dmul(k[0], y[0]) : dmul(0.0, y[0]);                                // (K @ y)[a], in index order
    c = dadd(c, a == 1 ? dmul(k[1], y[1]) : dmul(0.0, y[1]));
    c = dadd(c, a == 2 ? dmul(k[2], y[2]) : dmul(0.0, y[2]));
    s.ekf_x[a] = dadd(xp[a], c);
    s.ekf_p[a] = dmul(dsub(1.0, k[a]), pp[a]);                                             // (I - K H) P
  }
  state[i] = s;
}

// the pose fields of StaticFramePipeline._fill_jobs: the agent's pose goes to ring slot tick % keep, then job (agent, t) reads
// slot (tick - t * gap) mod keep against slot tick % keep
__global__ void __launch_bounds__(kThreads) stack_job_poses_kernel(unsigned char* __restrict__ jobs, int b, int t, int gap, int keep,
                                                                     long long tick, double* __restrict__ ring,
                                                                     const double* __restrict__ poses) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= b) return;
  double* rp = ring + (long long)i * keep * 3;
  const int s0 = (int)(tick % keep);
  if (poses) {
    rp[3 * s0] = poses[3 * i]; rp[3 * s0 + 1] = poses[3 * i + 1]; rp[3 * s0 + 2] = poses[3 * i + 2];
  }
  const double x0 = rp[3 * s0], y0 = rp[3 * s0 + 1], o0 = rp[3 * s0 + 2];
  double si0, c0;
  sincos(o0, &si0, &c0);
  for (int k = 0; k < t; ++k) {
    const long long tk = tick - (long long)k * gap;
    const int sl = (int)(((tk % keep) + keep) % keep);
    const double d = dsub(rp[3 * sl + 2], o0);
    const double dlx = dsub(rp[3 * sl], x0), dly = dsub(rp[3 * sl + 1], y0);
    double sd, cd;
    sincos(d, &sd, &cd);
    float* f = reinterpret_cast<float*>(jobs + ((long long)i * t + k) * LAVB_STACK_JOB_BYTES + 24);    // R[9], dx, dy
    f[0] = __double2float_rn(cd); f[1] = __double2float_rn(sd); f[2] = 0.f;
    f[3] = __double2float_rn(-sd); f[4] = __double2float_rn(cd); f[5] = 0.f;
    f[6] = 0.f; f[7] = 0.f; f[8] = 1.f;
    f[9] = __double2float_rn(dadd(dmul(dlx, c0), dmul(dly, si0)));
    f[10] = __double2float_rn(dadd(dmul(-dlx, si0), dmul(dly, c0)));
  }
}

bool aligned(const void* p, int a) { return (uintptr_t)p % a == 0; }

}  // namespace

extern "C" size_t lavb_agent_nav_state_bytes(void) { return sizeof(lavb_nav_state); }

extern "C" int lavb_agent_nav_front(int b, const double* d_nodes, const int* d_node_cmd, int n_nodes, const int* d_route,
                                    const double* d_gnss, const double* d_compass, void* d_state, int* d_cmds, float* d_nxps,
                                    double* d_poses, int* d_flags, void* stream) {
  LAVB_CHECK_ARG(b >= 0 && n_nodes >= 0, "agent_nav_front: bad sizes (b %d, n_nodes %d)", b, n_nodes);
  if (b == 0) return 0;
  LAVB_CHECK_ARG(d_route && d_gnss && d_compass && d_state && d_cmds && d_nxps && d_poses && d_flags &&
                 ((d_nodes && d_node_cmd) || n_nodes == 0), "agent_nav_front: null pointer");
  LAVB_CHECK_ARG(aligned(d_nodes, 16) && aligned(d_gnss, 16) && aligned(d_state, 8) && aligned(d_compass, 8) &&
                 aligned(d_poses, 8) && aligned(d_nxps, 8) && aligned(d_node_cmd, 4) && aligned(d_route, 4) &&
                 aligned(d_cmds, 4) && aligned(d_flags, 4),
                 "agent_nav_front: nodes and gnss must be 16-byte aligned, state, compass, poses and nxps 8-byte, the rest 4-byte");
  nav_front_kernel<<<lavb::ceil_div(b, kThreads), kThreads, 0, (cudaStream_t)stream>>>(
      b, reinterpret_cast<const double2*>(d_nodes), d_node_cmd, n_nodes, d_route, reinterpret_cast<const double2*>(d_gnss),
      d_compass, static_cast<lavb_nav_state*>(d_state), d_cmds, reinterpret_cast<float2*>(d_nxps), d_poses, d_flags);
  LAVB_LAUNCH_OK();
  return 0;
}

extern "C" int lavb_agent_nav_update(int b, const float* d_control, const double* d_speed, const double* d_gnss,
                                     const double* d_compass, void* d_state, void* stream) {
  LAVB_CHECK_ARG(b >= 0, "agent_nav_update: bad size (b %d)", b);
  if (b == 0) return 0;
  LAVB_CHECK_ARG(d_control && d_speed && d_gnss && d_compass && d_state, "agent_nav_update: null pointer");
  LAVB_CHECK_ARG(aligned(d_gnss, 16) && aligned(d_state, 8) && aligned(d_speed, 8) && aligned(d_compass, 8) && aligned(d_control, 4),
                 "agent_nav_update: gnss must be 16-byte aligned, state, speed and compass 8-byte, control 4-byte");
  nav_update_kernel<<<lavb::ceil_div(b, kThreads), kThreads, 0, (cudaStream_t)stream>>>(
      b, d_control, d_speed, reinterpret_cast<const double2*>(d_gnss), d_compass, static_cast<lavb_nav_state*>(d_state));
  LAVB_LAUNCH_OK();
  return 0;
}

extern "C" int lavb_stack_job_poses(void* d_jobs, int b, int t, int gap, int keep, long long tick, double* d_ring_pose,
                                    const double* d_poses, void* stream) {
  LAVB_CHECK_ARG(b >= 0 && t >= 1 && gap >= 1 && keep >= 1 && tick >= 0, "stack_job_poses: bad sizes (b %d, t %d, gap %d, keep %d, "
                 "tick %lld)", b, t, gap, keep, tick);
  if (b == 0) return 0;
  LAVB_CHECK_ARG(d_jobs && d_ring_pose, "stack_job_poses: null pointer");
  LAVB_CHECK_ARG(aligned(d_jobs, 8) && aligned(d_ring_pose, 8) && aligned(d_poses, 8),
                 "stack_job_poses: jobs, ring and poses must be 8-byte aligned");
  stack_job_poses_kernel<<<lavb::ceil_div(b, kThreads), kThreads, 0, (cudaStream_t)stream>>>(
      static_cast<unsigned char*>(d_jobs), b, t, gap, keep, tick, d_ring_pose, d_poses);
  LAVB_LAUNCH_OK();
  return 0;
}
