// The agent's decision tail (lav_agent_fast.py:228-231, 325-352) for b agents, one warp per agent: the lanes stride over the
// agent's (forecast row, branch) pairs for plan_collide (fp32 norms and means in numpy's pairwise order, fp64 comparisons,
// NaN = no collision) and combine their verdicts with a vote; lane 0 then steps the two PID windows of pid_control (twice, as
// run_step calls it twice), applies the brake rules and writes the controls, the flags and the agent's state.  Every operation
// is a correctly rounded intrinsic, so nothing is contracted.  The per-agent offsets and commands travel as a kernel argument.
#include "common.cuh"

namespace {

constexpr int kWarps = 4;                // agents per block
constexpr int kMaxSteps = 32;
constexpr int kMaxWindow = 64;
constexpr int kChunk = 512;              // agents per launch: their row offsets and commands travel as a kernel argument (2.5 KB)
constexpr int kHeader = 16;              // stop counter, creep counter, turn head, speed head
constexpr double kPi = 3.141592653589793;

struct Chunk { int rows[kChunk + 1]; signed char cmd[kChunk]; };

struct CtlArgs {
  const float2* plan; const float2* cast; const float2* locs; const float* scores; const float* pred_bra; const float* speed;
  unsigned char* state; long long state_bytes;
  float* control; int* flags;
  const int* cmd;                        // the device commands of lavb_agent_control_dcmd; null when they travel in the Chunk
  int t, c;
};

__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }

// numpy's add.reduce of term(0) .. term(n-1), n <= 128, in its order: below 8 terms a running sum from 0, otherwise 8 running
// sums over strides of 8 combined as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the last n % 8 terms in order
template <typename T, typename F>
__device__ __forceinline__ T pairwise_sum(int n, F term) {
  if (n < 8) {
    T r = T(0);
    for (int i = 0; i < n; ++i) r = add(r, term(i));
    return r;
  }
  T r[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) r[j] = term(j);
  const int m = n - n % 8;
  for (int i = 8; i < m; i += 8) {
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = add(r[j], term(i + j));
  }
  T res = add(add(add(r[0], r[1]), add(r[2], r[3])), add(add(r[4], r[5]), add(r[6], r[7])));
  for (int i = m; i < n; ++i) res = add(res, term(i));
  return res;
}

__device__ __forceinline__ float norm2(float dx, float dy) { return __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy))); }

// np.clip of an fp64 value: min(max(x, lo), hi) with a > b ? a : b; NaN passes through
__device__ __forceinline__ double clip(double x, double lo, double hi) {
  if (isnan(x)) return x;
  const double y = x > lo ? x : lo;
  return y < hi ? y : hi;
}

// PIDController.step (pid.py:14-26) twice with the error e on the window win[n] whose oldest value sits at head; returns the
// second step's kp * e + ki * mean + kd * (w[-1] - w[-2])
__device__ __forceinline__ double pid_twice(double* win, int n, int& head, double e, double kp, double ki, double kd) {
  head = (int)((unsigned)head % (unsigned)n);
  win[head] = e; head = head + 1 == n ? 0 : head + 1;
  win[head] = e; head = head + 1 == n ? 0 : head + 1;
  double integral = 0.0, derivative = 0.0;
  if (n >= 2) {
    const int h = head;
    integral = __ddiv_rn(pairwise_sum<double>(n, [&](int j) { return win[(h + j) % n]; }), (double)n);
    derivative = __dsub_rn(win[(h + n - 1) % n], win[(h + n - 2) % n]);
  }
  return __dadd_rn(__dadd_rn(__dmul_rn(kp, e), __dmul_rn(ki, integral)), __dmul_rn(kd, derivative));
}

__global__ void __launch_bounds__(kWarps * 32) agent_control_kernel(const CtlArgs p, const lavb_control_config cfg,
                                                                     const __grid_constant__ Chunk ch, int b0, int nb) {
  const int lane = threadIdx.x & 31, w = blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (w >= nb) return;                                            // whole warps leave together
  const int i = b0 + w, t = p.t, c = p.c, cmd = p.cmd ? __ldg(p.cmd + i) : ch.cmd[w];
  if (cmd < 0 || cmd >= c) {                                      // only a device command can get here
    if (lane == 0) {
      const float nan = __int_as_float(0x7fc00000);
      p.control[3LL * i] = nan; p.control[3LL * i + 1] = nan; p.control[3LL * i + 2] = nan;
      p.flags[i] = LAVB_CTL_BAD_CMD;
    }
    return;
  }
  const float2* plan = ((cmd == 4 || cmd == 5) ? p.cast : p.plan) + (long long)i * t;   // :325-326
  const float2 q = lane < t ? __ldg(plan + lane) : make_float2(0.f, 0.f);
  const bool valid = !__any_sync(0xffffffffu, isnan(q.x) || isnan(q.y));                 // :328
  const double ppm = cfg.pixels_per_meter, far_y = __dmul_rn(0.5, ppm);
  const float fp = __double2float_rn(ppm);
  // the aim point's fp32 atan2 (:413-414), correctly rounded from fp64; taken first, while little else is live across the call
  const float2 aim = __ldg(plan + cfg.aim_point[cmd]);
  const float a32 = __double2float_rn(atan2((double)-__fmul_rn(aim.y, fp), (double)__fmul_rn(aim.x, fp)));

  // plan_collide (:385-401): every (row, branch) pair of the agent, one per lane
  const int r0 = ch.rows[w], pairs = (ch.rows[w + 1] - r0) * c;
  bool hit = false;
  for (int e = lane; e < pairs; e += 32) {
    const long long r = r0 + e / c;
    const int br = e % c;
    const float2* row = p.locs + r * c * t;
    if ((double)__ldg(&row->y) > far_y) continue;                                       // :388-390
    if ((double)__ldg(p.scores + r * c + br) < cfg.cmd_thresh) continue;              // :392-393
    const float2* tr = row + br * t;
    const float spd = __fdiv_rn(pairwise_sum<float>(t - 1, [&](int s) {             // :395
      const float2 a = __ldg(tr + s), b = __ldg(tr + s + 1);
      return norm2(__fsub_rn(b.x, a.x), __fsub_rn(b.y, a.y));
    }), (float)(t - 1));
    const double thresh = (double)spd < cfg.brake_speed ? 1.0 : 2.5;                   // :396
    bool nan = false;
    float dist = __int_as_float(0x7f800000);
    for (int s = 0; s < t; ++s) {                                                       // :397, NaN propagates through min
      const float2 a = __ldg(tr + s), b = __ldg(plan + s);
      const float d = norm2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y));
      if (isnan(d)) nan = true;
      else if (d < dist) dist = d;
    }
    hit |= !nan && (double)dist < thresh;                                               // :398
  }
  hit = __any_sync(0xffffffffu, hit);
  if (lane != 0) return;

  unsigned char* st = p.state + (long long)i * p.state_bytes;
  int* hdr = reinterpret_cast<int*>(st);
  double* turn = reinterpret_cast<double*>(st + kHeader);
  double* speed_win = turn + cfg.turn_n;
  const double spd = (double)__ldg(p.speed + i);
  int stop = spd < 0.1 ? hdr[0] + 1 : 0, creep = hdr[1], turn_head = hdr[2], speed_head = hdr[3];   // :228-231
  double steer = 0.0, throttle = 0.0, brake = 0.0;
  int flags = valid ? 0 : LAVB_CTL_PLAN_INVALID;
  if (valid) {                                                                          // pid_control (:404-426), twice
    const float desired = __fdiv_rn(pairwise_sum<float>(t - 1, [&](int s) {          // :406-411
      const float2 a = __ldg(plan + s), b = __ldg(plan + s + 1);
      return norm2(__fsub_rn(__fmul_rn(b.x, fp), __fmul_rn(a.x, fp)), __fsub_rn(-__fmul_rn(b.y, fp), -__fmul_rn(a.y, fp)));
    }), (float)(t - 1));
    const double angle = __ddiv_rn(__dmul_rn(__dsub_rn(kPi / 2, (double)a32), 180.0 / kPi), 90.0);   // :414
    steer = clip(pid_twice(turn, cfg.turn_n, turn_head, angle, cfg.turn_kp, cfg.turn_ki, cfg.turn_kd), -1.0, 1.0);
    const bool pid_brake = (double)desired < __dmul_rn(cfg.brake_speed, ppm);           // :420
    const double delta = clip(__dsub_rn(__dmul_rn((double)desired, cfg.speed_ratio[cmd]), spd), 0.0, cfg.clip_delta);
    throttle = clip(pid_twice(speed_win, cfg.speed_n, speed_head, delta, cfg.speed_kp, cfg.speed_ki, cfg.speed_kd), 0.0,
                    cfg.max_throttle);
    if (pid_brake) { throttle = 0.0; brake = 1.0; flags |= LAVB_CTL_PID_BRAKE; }        // :424-426
  }
  const bool bm = (double)__ldg(p.pred_bra + i) > 0.1;                                 // :340-343
  if (bm) flags |= LAVB_CTL_BRAKE_MODEL;
  if (hit) flags |= LAVB_CTL_COLLIDE;
  if (bm || hit) { throttle = 0.0; brake = 1.0; }
  if (__dmul_rn(spd, 3.6) > cfg.max_speed) { throttle = 0.0; flags |= LAVB_CTL_SPEED_CAP; }   // :344-345
  if (stop >= 600) creep = 20;                                                          // :347-348
  if (creep > 0) {                                                                      // :350-352
    throttle = throttle > 0.4 ? throttle : 0.4;
    brake = 0.0;
    --creep;
    flags |= LAVB_CTL_CREEP;
  }
  hdr[0] = stop; hdr[1] = creep; hdr[2] = turn_head; hdr[3] = speed_head;
  float* o = p.control + 3LL * i;
  o[0] = __double2float_rn(steer); o[1] = __double2float_rn(throttle); o[2] = __double2float_rn(brake);
  p.flags[i] = flags;
}

}  // namespace

extern "C" size_t lavb_agent_control_state_bytes(int turn_n, int speed_n) {
  if (turn_n < 1 || turn_n > kMaxWindow || speed_n < 1 || speed_n > kMaxWindow) return 0;
  return (size_t)kHeader + sizeof(double) * (size_t)(turn_n + speed_n);
}

static int agent_control(const float* d_plan, const float* d_cast, int b, int t, int c, const float* d_other_locs,
                         const float* d_other_cmds, int k, const int* h_offsets, const float* d_pred_bra, const float* d_speed,
                         const int* h_cmd, const int* d_cmd, const lavb_control_config* h_config, void* d_state, float* d_control,
                         int* d_flags, void* stream) {
  LAVB_CHECK_ARG(b >= 0 && k >= 0, "agent_control: bad sizes (b %d, k %d)", b, k);
  LAVB_CHECK_ARG(t >= 2 && t <= kMaxSteps, "agent_control: %d steps outside 2..%d", t, kMaxSteps);
  LAVB_CHECK_ARG(c >= 1 && c <= LAVB_CTL_MAX_CMDS, "agent_control: %d branches outside 1..%d", c, LAVB_CTL_MAX_CMDS);
  LAVB_CHECK_ARG(h_config, "agent_control: missing config");
  const lavb_control_config cfg = *h_config;
  LAVB_CHECK_ARG(lavb_agent_control_state_bytes(cfg.turn_n, cfg.speed_n) > 0, "agent_control: windows %d, %d outside 1..%d",
                 cfg.turn_n, cfg.speed_n, kMaxWindow);
  for (int j = 0; j < c; ++j)
    LAVB_CHECK_ARG(cfg.aim_point[j] >= 0 && cfg.aim_point[j] < t, "agent_control: aim_point[%d] = %d outside 0..%d", j,
                   cfg.aim_point[j], t - 1);
  LAVB_CHECK_ARG(cfg.pixels_per_meter > 0.0 && isfinite(cfg.pixels_per_meter), "agent_control: pixels_per_meter %g", cfg.pixels_per_meter);
  LAVB_CHECK_ARG(h_offsets, "agent_control: missing host offsets (%d forecast rows)", k);
  LAVB_CHECK_ARG(h_offsets[0] >= 0 && h_offsets[b] <= k, "agent_control: row offsets [%d, %d] run outside the %d forecast rows",
                 h_offsets[0], h_offsets[b], k);
  for (int i = 0; i < b; ++i)
    LAVB_CHECK_ARG(h_offsets[i] <= h_offsets[i + 1], "agent_control: row offsets of agent %d are not monotone (%d -> %d)", i,
                   h_offsets[i], h_offsets[i + 1]);
  if (!d_cmd) {
    LAVB_CHECK_ARG(h_cmd || b == 0, "agent_control: missing host commands");
    for (int i = 0; i < b; ++i)
      LAVB_CHECK_ARG(h_cmd[i] >= 0 && h_cmd[i] < c, "agent_control: command %d of agent %d outside 0..%d", h_cmd[i], i, c - 1);
  }
  if (b == 0) return 0;
  LAVB_CHECK_ARG((uintptr_t)d_cmd % 4 == 0, "agent_control: device commands must be 4-byte aligned");
  LAVB_CHECK_ARG(d_plan && d_cast && d_pred_bra && d_speed && d_state && d_control && d_flags &&
                 ((d_other_locs && d_other_cmds) || h_offsets[b] == h_offsets[0]), "agent_control: null pointer");
  LAVB_CHECK_ARG((uintptr_t)d_plan % 8 == 0 && (uintptr_t)d_cast % 8 == 0 && (uintptr_t)d_other_locs % 8 == 0 &&
                 (uintptr_t)d_state % 8 == 0 && (uintptr_t)d_other_cmds % 4 == 0 && (uintptr_t)d_pred_bra % 4 == 0 &&
                 (uintptr_t)d_speed % 4 == 0 && (uintptr_t)d_control % 4 == 0 && (uintptr_t)d_flags % 4 == 0,
                 "agent_control: plan, cast, other_locs and state must be 8-byte aligned, the rest 4-byte aligned");
  CtlArgs a;
  a.plan = reinterpret_cast<const float2*>(d_plan); a.cast = reinterpret_cast<const float2*>(d_cast);
  a.locs = reinterpret_cast<const float2*>(d_other_locs); a.scores = d_other_cmds;
  a.pred_bra = d_pred_bra; a.speed = d_speed;
  a.state = static_cast<unsigned char*>(d_state); a.state_bytes = (long long)lavb_agent_control_state_bytes(cfg.turn_n, cfg.speed_n);
  a.control = d_control; a.flags = d_flags;
  a.t = t; a.c = c;
  a.cmd = d_cmd;
  cudaStream_t st = (cudaStream_t)stream;
  for (int b0 = 0; b0 < b; b0 += kChunk) {
    const int nb = b - b0 < kChunk ? b - b0 : kChunk;
    Chunk ch;
    for (int i = 0; i <= nb; ++i) ch.rows[i] = h_offsets[b0 + i];
    for (int i = 0; i < nb && !d_cmd; ++i) ch.cmd[i] = (signed char)h_cmd[b0 + i];
    agent_control_kernel<<<(nb + kWarps - 1) / kWarps, kWarps * 32, 0, st>>>(a, cfg, ch, b0, nb);
    LAVB_LAUNCH_OK();
  }
  return 0;
}

extern "C" int lavb_agent_control(const float* d_plan, const float* d_cast, int b, int t, int c, const float* d_other_locs,
                                  const float* d_other_cmds, int k, const int* h_offsets, const float* d_pred_bra,
                                  const float* d_speed, const int* h_cmd, const lavb_control_config* h_config, void* d_state,
                                  float* d_control, int* d_flags, void* stream) {
  return agent_control(d_plan, d_cast, b, t, c, d_other_locs, d_other_cmds, k, h_offsets, d_pred_bra, d_speed, h_cmd, nullptr,
                       h_config, d_state, d_control, d_flags, stream);
}

extern "C" int lavb_agent_control_dcmd(const float* d_plan, const float* d_cast, int b, int t, int c, const float* d_other_locs,
                                       const float* d_other_cmds, int k, const int* h_offsets, const float* d_pred_bra,
                                       const float* d_speed, const int* d_cmd, const lavb_control_config* h_config, void* d_state,
                                       float* d_control, int* d_flags, void* stream) {
  LAVB_CHECK_ARG(d_cmd || b == 0, "agent_control: missing device commands");
  return agent_control(d_plan, d_cast, b, t, c, d_other_locs, d_other_cmds, k, h_offsets, d_pred_bra, d_speed, nullptr, d_cmd,
                       h_config, d_state, d_control, d_flags, stream);
}
