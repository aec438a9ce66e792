"""ORACLE — test infrastructure, never the product path.

A numpy restatement of the agent's decision tail for B agents: what lav_agent_fast.py:run_step does with the planner's outputs
once they are on the host (team_code_v2/lav_agent_fast.py:228-231 and 325-352), i.e. the stop counter, the 4/5 plan swap,
pid_control (:404-426, called twice) with its two team_code_v2/pid.py PIDControllers, plan_collide (:385-401) and the brake
rules.  It is the contract lavb_agent_control (include/lav_b200.h) is tested against, and the host baseline of
scripts/control_measure.py.  oracle/pin_control.py checks it against the reference's own methods and writes
tests/golden/agent_control.npz.

Precision follows the reference's environment (Python 3.7, numpy 1.x promotion rules):
  * the trajectories stay fp32: the scaled waypoints, every norm, the means (numpy's pairwise summation order, pairwise_sum
    below) and the minimums; np.min / np.mean propagate NaN;
  * np.arctan2 of two fp32 scalars is fp32 (taken correctly rounded here, from the fp64 atan2);
  * a numpy fp32 scalar combined with a Python float is fp64: the angle, the speed error, the PID arithmetic and every threshold
    comparison.  (numpy 2 keeps the angle and the speed error fp32, so the reference run under numpy 2 differs from this
    statement in the last bits of steer and throttle.)
Vectorised over agents, forecast rows and branches; the order of every rounding is the reference's.
"""
import numpy as np

# flag bits of one agent's tick (LAVB_CTL_* in include/lav_b200.h)
CTL_PLAN_INVALID, CTL_PID_BRAKE, CTL_BRAKE_MODEL, CTL_COLLIDE, CTL_SPEED_CAP, CTL_CREEP = 1, 2, 4, 8, 16, 32
# the keys of the agent's YAML config the tail reads (team_code_v2/config.yaml, CONTROLLER section + cmd_thresh, pixels_per_meter)
CONTROL_KEYS = ("aim_point", "speed_ratio", "turn_KP", "turn_KI", "turn_KD", "turn_n", "speed_KP", "speed_KI", "speed_KD",
                "speed_n", "brake_speed", "clip_delta", "max_throttle", "max_speed", "cmd_thresh", "pixels_per_meter")
STOP_TICKS, CREEP_TICKS, CREEP_THROTTLE = 600, 20, 0.4      # lav_agent_fast.py:347-351
BRAKE_MODEL_THRESH = 0.1                                      # :340
STOPPED_SPEED = 0.1                                           # :228
DIST_STATIC, DIST_MOVING = 1.0, 2.5                           # plan_collide's default thresholds, :385


def config_of(config):
    """the CONTROL_KEYS of the agent's loaded YAML dict; a missing key is an error."""
    missing = [k for k in CONTROL_KEYS if k not in config]
    if missing:
        raise KeyError(f"agent config lacks {missing}")
    return {k: config[k] for k in CONTROL_KEYS}


def pairwise_sum(x):
    """numpy's add.reduce over the last axis of x (<= 128 terms) in x's dtype and order: below 8 terms a running sum from 0,
    otherwise 8 running sums over strides of 8 combined as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the remaining n % 8 terms
    in order (pairwise_sum of numpy's umath loops)."""
    n = x.shape[-1]
    assert n <= 128, n
    if n < 8:
        res = np.zeros(x.shape[:-1], x.dtype)
        for i in range(n):
            res = res + x[..., i]
        return res
    m = n - n % 8
    r = x[..., 0:8].copy()
    for i in range(8, m, 8):
        r = r + x[..., i:i + 8]
    res = ((r[..., 0] + r[..., 1]) + (r[..., 2] + r[..., 3])) + ((r[..., 4] + r[..., 5]) + (r[..., 6] + r[..., 7]))
    for i in range(m, n):
        res = res + x[..., i]
    return res


def norm2(d):
    """np.linalg.norm(d, axis=-1) of fp32 (..., 2): sqrt(x*x + y*y), each operation rounded to fp32."""
    return np.sqrt(d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1])


def mean_f32(x):
    """ndarray.mean over the last axis of fp32 x: the pairwise fp32 sum divided by the count in fp32."""
    return pairwise_sum(x) / np.float32(x.shape[-1])


def clip(x, lo, hi):
    """np.clip of fp64 values: min(max(x, lo), hi) with a > b ? a : b, a NaN x passes through."""
    y = np.where(x > lo, x, lo)
    y = np.where(y < hi, y, hi)
    return np.where(np.isnan(x), x, y)


def atan2_f32(y, x):
    """np.arctan2 of two fp32 scalars, correctly rounded to fp32."""
    return np.arctan2(y.astype(np.float64), x.astype(np.float64)).astype(np.float32)


def collide(plan, locs, cmds, agent, B, ppm, cmd_thresh, brake_speed):
    """plan_collide (lav_agent_fast.py:385-401) of every agent at once.  plan (B,T,2) fp32 = the plan the agent drives; locs
    (K,C,T,2) / cmds (K,C) fp32 = every agent's forecast rows, row k owned by agent[k].  -> (B,) bool."""
    hit = np.zeros(B, dtype=bool)
    if locs.shape[0] == 0:
        return hit
    far = locs[:, 0, 0, 1].astype(np.float64) > 0.5 * ppm                              # :388-390, the row's first point
    live = ~far[:, None] & ~(cmds.astype(np.float64) < cmd_thresh)                    # :392-393
    spd = mean_f32(norm2(locs[:, :, 1:] - locs[:, :, :-1]))                          # :395
    thresh = np.where(spd.astype(np.float64) < brake_speed, DIST_STATIC, DIST_MOVING)  # :396
    dist = norm2(locs - plan[agent][:, None]).min(-1)                                 # :397, NaN propagates
    np.logical_or.at(hit, agent, (live & (dist.astype(np.float64) < thresh)).any(1))  # :398-399
    return hit


class ControlTail:
    """The decision tail of B agents with its per-agent state: a turn and a speed PID window (oldest value first, starting as n
    zeros), the stop counter and the creep counter."""

    def __init__(self, batch, config):
        self.cfg = config_of(config)
        self.B = batch
        self.turn = np.zeros((batch, int(self.cfg["turn_n"])))
        self.speed = np.zeros((batch, int(self.cfg["speed_n"])))
        self.stop = np.zeros(batch, dtype=np.int64)
        self.force = np.zeros(batch, dtype=np.int64)

    def reset(self, agents=None):
        """a new route for ``agents`` (all when None): their windows and counters back to zero."""
        idx = slice(None) if agents is None else np.asarray(agents, dtype=np.int64)
        self.turn[idx] = 0.0
        self.speed[idx] = 0.0
        self.stop[idx] = 0
        self.force[idx] = 0

    @staticmethod
    def _pid(win, err, kp, ki, kd):
        """PIDController.step (pid.py:14-26) twice with the same error on the rows of ``win`` (updated in place); returns the
        second step's output."""
        n = win.shape[1]
        win[:] = np.concatenate([win, err[:, None], err[:, None]], axis=1)[:, -n:]
        if n >= 2:
            integral = pairwise_sum(win) / float(n)
            derivative = win[:, -1] - win[:, -2]
        else:
            integral = derivative = np.zeros(len(err))
        return kp * err + ki * integral + kd * derivative

    def step(self, plan, cast, other_locs, other_cmds, pred_bra, speed, cmd):
        """One tick.  plan / cast (B,T,2) fp32 = ego plan and ego cast under the command; other_locs: B arrays (k_b,C,T,2) fp32
        and other_cmds: B arrays (k_b,C) fp32 = each agent's forecast rows and their command scores; pred_bra, speed (B,) fp32
        (speed in m/s); cmd (B,) ints.  -> dict(control (B,3) fp64 = steer, throttle, brake; flags (B,) int32;
        desired_speed (B,) fp32)."""
        c = self.cfg
        B = self.B
        plan, cast = np.asarray(plan, np.float32), np.asarray(cast, np.float32)
        cmd = np.asarray(cmd, dtype=np.int64)
        spd = np.asarray(speed, dtype=np.float32).astype(np.float64)
        ppm = c["pixels_per_meter"]
        self.stop = np.where(spd < STOPPED_SPEED, self.stop + 1, 0)                      # :228-231
        p = np.where(((cmd == 4) | (cmd == 5))[:, None, None], cast, plan)               # :325-326
        valid = ~np.isnan(p).reshape(B, -1).any(1)                                       # :328, :333

        # pid_control (:404-426), stepped only where the plan is valid
        w = p * np.float32(ppm)                                                          # :406
        w[..., 1] = -w[..., 1]                                                           # :407
        desired = mean_f32(norm2(w[:, 1:] - w[:, :-1]))                                  # :411
        aim = w[np.arange(B), np.asarray(c["aim_point"])[cmd]]                           # :413
        angle = np.degrees(np.pi / 2 - atan2_f32(aim[:, 1], aim[:, 0]).astype(np.float64)) / 90   # :414
        ds = desired.astype(np.float64)
        delta = clip(ds * np.asarray(c["speed_ratio"], dtype=np.float64)[cmd] - spd, 0.0, c["clip_delta"])   # :421
        v = np.flatnonzero(valid)
        steer, throttle, brake = np.zeros(B), np.zeros(B), np.zeros(B)
        pid_brake = np.zeros(B, dtype=bool)
        if v.size:
            tw, sw = self.turn[v], self.speed[v]
            st = clip(self._pid(tw, angle[v], c["turn_KP"], c["turn_KI"], c["turn_KD"]), -1.0, 1.0)             # :415-416
            th = clip(self._pid(sw, delta[v], c["speed_KP"], c["speed_KI"], c["speed_KD"]), 0.0, c["max_throttle"])  # :422-423
            br = ds[v] < c["brake_speed"] * ppm                                                                  # :420
            self.turn[v], self.speed[v] = tw, sw
            steer[v], throttle[v], brake[v], pid_brake[v] = st, np.where(br, 0.0, th), br.astype(np.float64), br  # :424-426

        # plan_collide against every agent's forecast rows (evaluated for all agents, :342)
        counts = [len(o) for o in other_locs]
        T, C = p.shape[1], len(c["aim_point"])
        locs = np.concatenate([np.asarray(o, np.float32).reshape(-1, C, T, 2) for o in other_locs]) if B else np.zeros((0, C, T, 2), np.float32)
        cmds = np.concatenate([np.asarray(o, np.float32).reshape(-1, C) for o in other_cmds]) if B else np.zeros((0, C), np.float32)
        agent = np.repeat(np.arange(B), counts)
        hit = collide(p, locs, cmds, agent, B, ppm, c["cmd_thresh"], c["brake_speed"])

        # the brake rules (:340-352)
        bm = np.asarray(pred_bra, dtype=np.float32).reshape(B).astype(np.float64) > BRAKE_MODEL_THRESH
        stop = bm | hit
        throttle = np.where(stop, 0.0, throttle)
        brake = np.where(stop, 1.0, brake)
        cap = spd * 3.6 > c["max_speed"]
        throttle = np.where(cap, 0.0, throttle)
        self.force = np.where(self.stop >= STOP_TICKS, CREEP_TICKS, self.force)
        creep = self.force > 0
        throttle = np.where(creep, np.where(throttle > CREEP_THROTTLE, throttle, CREEP_THROTTLE), throttle)
        brake = np.where(creep, 0.0, brake)
        self.force = np.where(creep, self.force - 1, self.force)

        flags = ((~valid) * CTL_PLAN_INVALID | pid_brake * CTL_PID_BRAKE | bm * CTL_BRAKE_MODEL | hit * CTL_COLLIDE |
                 cap * CTL_SPEED_CAP | creep * CTL_CREEP).astype(np.int32)
        return dict(control=np.stack([steer, throttle, brake], axis=1), flags=flags, desired_speed=desired)


def control_sequence(seed, batch, ticks, T=20, C=6, max_rows=15, nan_plan=0.02, nan_step=0.03, stopped=(), halts=()):
    """A seeded tick sequence of decision-tail inputs (np.random.RandomState, stable across numpy versions), yielded per tick as
    dict(plan, cast, other_locs, other_cmds, pred_bra, speed, cmd).  Agent 0 never sees a forecast row, agent 1 always sees
    ``max_rows``; the others 0..max_rows.  Agents in ``stopped`` stand still throughout, agents in ``halts`` stand still for the
    first 620 ticks and then move.  Plans step 0..1.1 m per step (some below the PID brake speed), forecasts start around the
    plan (some far, some behind), scores and brake predictions straddle their thresholds; a fraction of plans and of forecast
    branches carries a NaN step."""
    rs = np.random.RandomState(seed)
    base_speed = rs.uniform(0.0, 12.0, batch)
    for tick in range(ticks):
        cmd = rs.randint(0, C, batch)
        step = rs.uniform(0.0, 1.1, (batch, 1, 1)) * rs.uniform(0.6, 1.0, (batch, T, 1))
        head = rs.normal(0.0, 0.25, (batch, 1, 1)) + rs.normal(0.0, 0.05, (batch, T, 1))
        plan = np.cumsum(np.concatenate([np.sin(head), -np.cos(head)], -1) * step, axis=1).astype(np.float32)
        cast = (plan * rs.uniform(0.5, 1.5, (batch, 1, 1)) + rs.normal(0.0, 0.1, (batch, T, 2))).astype(np.float32)
        for arr in (plan, cast):
            bad = np.flatnonzero(rs.rand(batch) < nan_plan)
            arr[bad, rs.randint(0, T, len(bad)), rs.randint(0, 2, len(bad))] = np.nan
        other_locs, other_cmds = [], []
        for b in range(batch):
            k = 0 if b == 0 else max_rows if b == 1 else rs.randint(0, max_rows + 1)
            start = plan[b, rs.randint(0, T, k)] + rs.normal(0.0, 6.0, (k, 2)) * rs.uniform(0.2, 2.0, (k, 1))
            start[rs.rand(k) < 0.15, 1] = 2.0 + rs.choice([-0.5, 0.0, 0.5])
            v = rs.uniform(0.0, 0.5, (k, C, 1, 1)) * rs.choice([0.0, 1.0], (k, C, 1, 1), p=[0.3, 0.7])
            dirs = rs.normal(0.0, 1.0, (k, C, 1, 2))
            dirs /= np.maximum(np.linalg.norm(dirs, axis=-1, keepdims=True), 1e-6)
            traj = start[:, None, None] + np.cumsum(np.concatenate([np.zeros((k, C, 1, 2)), np.repeat(dirs * v, T - 1, 2)], 2), 2)
            traj = (traj + rs.normal(0.0, 0.02, traj.shape)).astype(np.float32)
            bad = rs.rand(k, C) < nan_step
            traj[bad, rs.randint(0, T, int(bad.sum()))] = np.nan
            score = rs.uniform(0.0, 0.5, (k, C)).astype(np.float32)
            score[rs.rand(k, C) < 0.05] = np.float32(0.2)
            other_locs.append(traj)
            other_cmds.append(score)
        pred_bra = rs.uniform(0.0, 0.12, batch).astype(np.float32)
        pred_bra[rs.rand(batch) < 0.03] = np.float32(0.1)
        speed = np.clip(base_speed + rs.normal(0.0, 1.5, batch), 0.0, None).astype(np.float32)
        speed[list(stopped)] = rs.uniform(0.0, 0.09, len(stopped))
        if tick < 620:
            speed[list(halts)] = 0.0
        yield dict(plan=plan, cast=cast, other_locs=other_locs, other_cmds=other_cmds, pred_bra=pred_bra, speed=speed, cmd=cmd)
