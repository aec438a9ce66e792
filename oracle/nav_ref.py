"""ORACLE — test infrastructure, never the product path.

A numpy restatement of the agent's localisation and route following for B agents: the head of LAVAgent.run_step
(team_code_v2/lav_agent_fast.py:215-226, 280-308, 314) with EKF.init, Waypointer.tick (pop_lane_change=True, pop_turning=False,
default thresholds) and RoutePlanner.run_step, and the EKF.step after the controls (:338).  It is the contract
lavb_agent_nav_front / lavb_agent_nav_update (include/lav_b200.h) are tested against.  oracle/pin_nav.py checks it against the
reference's own classes and writes tests/golden/agent_nav.npz.

The route scans are restated in O(1): only node current_idx + 1 can satisfy ``i - current_idx == 1``, and after Waypointer.tick's
loop ``i`` is that node when it was taken and len - 1 otherwise, which is where the lane-change look-ahead starts.  Every value
is fp64 in the reference's order of operations; np.linalg.norm of a pair is sqrt(dx*dx + dy*dy).  EKF.step is stated in closed
form: F = H = I with diagonal Q, R and a zero start keep P diagonal, the gain is P * (1 / (P + R)) per axis, and the products numpy
forms with K's zeros are kept, so a non-finite innovation reaches every state as it does in ``K_kp @ y_kp``.
"""
import math

import numpy as np

NAV_FIRST_FRAME, NAV_NO_ROUTE, NAV_LANE_HELD = 1, 2, 4          # LAVB_NAV_* of include/lav_b200.h
EARTH_RADIUS = 6371e3
LANEFOLLOW, CHANGELANELEFT, CHANGELANERIGHT = 4, 5, 6             # RoadOption values
THRESH_BEFORE, THRESH_AFTER = 4.5, 3.0                            # Waypointer defaults (waypointer.py:14-16)
CURR_THRESHOLD, NEXT_THRESHOLD = 20, 75                           # RoutePlanner defaults (planner.py:11)
LANE_CHANGE_TICKS = 300                                           # lav_agent_fast.py:299
# EKF(1, 1.477531, 1.393600) (lav_agent_fast.py:137) with its defaults (ekf.py:8-31)
EKF_COS0, LF, LR = 1, 1.477531, 1.393600
L = LF + LR
MAX_STEER = 70 * math.pi / 180.
DT = 1. / 20
Q = 1e-7
XY_NOISE = EARTH_RADIUS * 0.000005 * math.pi / 180.
COMPASS_NOISE = 1e-7 * math.pi / 180.
R_DIAG = np.array([XY_NOISE ** 2, XY_NOISE ** 2, COMPASS_NOISE ** 2])
assert XY_NOISE ** 2 == XY_NOISE * XY_NOISE and COMPASS_NOISE ** 2 == COMPASS_NOISE * COMPASS_NOISE   # the kernel squares by a product


def road_option_value(cmd):
    """the integer value of a RoadOption (or of an int already holding one)."""
    return int(getattr(cmd, "value", cmd))


def route_table(route):
    """(scale, xy (n, 2) fp64, cmd (n,) int32) of one _global_plan [(gnss dict, RoadOption or int)], as the Waypointer and the
    RoutePlanner convert it (waypointer.py:30-42, planner.py:16-27): cos_0 = the route latitudes in radians summed in order over
    the count, scale = math.cos(cos_0)."""
    if len(route) == 0:
        raise ValueError("a route needs at least one node")
    cos_0 = 0.
    for gnss, _ in route:
        cos_0 += gnss['lat'] * (math.pi / 180)
    cos_0 = cos_0 / (len(route))
    scale = math.cos(cos_0)
    xy = np.array([(EARTH_RADIUS * g['lat'] * (math.pi / 180), EARTH_RADIUS * g['lon'] * (math.pi / 180) * scale)
                   for g, _ in route], dtype=np.float64)
    cmd = np.array([road_option_value(c) for _, c in route], dtype=np.int32)
    return scale, xy, cmd


def waypointer_tick(xy, rc, idx, cp, cp_cmd, cx, cy):
    """Waypointer.tick (waypointer.py:50-96, pop_lane_change=True, pop_turning=False) in O(1) on a route (xy, rc) from the state
    (current_idx, checkpoint (x, y), checkpoint RoadOption value) at the position (cx, cy) -> the new state."""
    n = len(xy)
    i = n - 1
    j = idx + 1
    if j < n:
        thr = THRESH_BEFORE if cp_cmd == LANEFOLLOW and rc[j] != LANEFOLLOW else THRESH_AFTER
        dx, dy = cx - xy[j, 0], cy - xy[j, 1]
        if np.sqrt(dx * dx + dy * dy) < thr:
            idx, cp, cp_cmd = j, (xy[j, 0], xy[j, 1]), int(rc[j])
            i = j
    look, cmd = 0, cp_cmd
    while i + 1 < n and look < 3:
        if cmd != LANEFOLLOW:
            break
        if rc[i + 1] in (CHANGELANELEFT, CHANGELANERIGHT):
            idx, cp, cp_cmd = i + 1, (xy[i + 1, 0], xy[i + 1, 1]), int(rc[i + 1])
            break
        cmd = rc[i + 1]
        i += 1
        look += 1
    return idx, cp, cp_cmd


class AgentNavRef:
    """Navigation state of ``batch`` agents; agents without a route yield NAV_NO_ROUTE."""

    def __init__(self, batch):
        B = self.B = int(batch)
        self.routes = [None] * B                          # (xy, cmd) per agent
        self.scale = np.zeros(B)
        self.frames = np.zeros(B, np.int64)
        self.x = np.zeros((B, 3))
        self.p = np.zeros((B, 3))
        self.wp = np.zeros((B, 2)); self.wp_cmd = np.zeros(B, np.int64); self.wp_idx = np.zeros(B, np.int64)
        self.rp = np.zeros((B, 2)); self.rp_idx = np.zeros(B, np.int64)
        self.lane_counter = np.zeros(B, np.int64); self.lane_changed = np.full(B, -1, np.int64)
        self.theta_pred = np.zeros(B)                     # kbm_step's heading of the last update (its size sets theta's conditioning)

    def set_routes(self, agents, routes):
        for a, r in zip(agents, routes):
            scale, xy, cmd = route_table(r)
            self.routes[a] = (xy, cmd)
            self.scale[a] = scale
            self.frames[a] = 0
            self.x[a] = 0; self.p[a] = 0
            self.wp[a] = 0; self.wp_cmd[a] = 0; self.wp_idx[a] = 0
            self.rp[a] = 0; self.rp_idx[a] = 0
            self.lane_counter[a] = 0; self.lane_changed[a] = -1

    @staticmethod
    def ekf_xy(lat, lon):
        return EARTH_RADIUS * lat * (math.pi / 180), EARTH_RADIUS * lon * (math.pi / 180) * math.cos(EKF_COS0)

    def front(self, gnss, compass):
        """gnss (B, >=2) fp64 lat, lon; compass (B,) fp64 raw imu[-1].  -> dict(cmds (B,) int32, nxps (B, 2) fp32, poses (B, 3)
        fp64, flags (B,) int32)."""
        B = self.B
        gnss, raw = np.asarray(gnss, np.float64), np.asarray(compass, np.float64)
        cmds = np.full(B, 3, np.int32)
        nxps = np.zeros((B, 2), np.float32)
        poses = np.full((B, 3), np.nan)
        flags = np.zeros(B, np.int32)
        for b in range(B):
            if self.routes[b] is None:
                nxps[b] = np.nan
                flags[b] = NAV_NO_ROUTE
                continue
            xy, rc = self.routes[b]
            n = len(xy)
            lat, lon = gnss[b, 0], gnss[b, 1]
            cmp = 0. if np.isnan(raw[b]) else raw[b]                                       # :219-220
            if self.frames[b] == 0:                                                        # :222-224
                self.x[b, 0], self.x[b, 1] = self.ekf_xy(lat, lon)
                self.x[b, 2] = cmp - math.pi / 2
                self.p[b] = 0
            self.frames[b] = min(self.frames[b] + 1, 1 << 30)
            poses[b] = self.x[b]                                                           # :226
            if self.frames[b] <= 1:                                                        # :235-237
                flags[b] = NAV_FIRST_FRAME
                continue
            cx = EARTH_RADIUS * lat * (math.pi / 180)
            cy = EARTH_RADIUS * lon * (math.pi / 180) * self.scale[b]
            if self.frames[b] == 2:                                                        # :280-286
                self.wp[b] = cx, cy; self.wp_cmd[b] = LANEFOLLOW; self.wp_idx[b] = -1
                self.rp[b] = xy[0]; self.rp_idx[b] = 0
            idx, cp, cp_cmd = waypointer_tick(xy, rc, int(self.wp_idx[b]), tuple(self.wp[b]), int(self.wp_cmd[b]), cx, cy)
            self.wp_idx[b], self.wp[b], self.wp_cmd[b] = idx, cp, cp_cmd
            # RoutePlanner.run_step
            dx, dy = self.rp[b, 0] - cx, self.rp[b, 1] - cy
            curr = np.sqrt(dx * dx + dy * dy)
            k = self.rp_idx[b] + 1
            if k < n:
                dx, dy = xy[k, 0] - cx, xy[k, 1] - cy
                if np.sqrt(dx * dx + dy * dy) < NEXT_THRESHOLD and curr < CURR_THRESHOLD:
                    self.rp[b] = xy[k]; self.rp_idx[b] = k
            wx, wy = self.rp[b, 0] - cx, self.rp[b, 1] - cy
            cv = int(self.wp_cmd[b]) - 1                                                   # :291-292
            cv = 3 if cv < 0 else cv
            if cv in (4, 5):                                                               # :294-302
                if self.lane_changed[b] >= 0 and cv != self.lane_changed[b]:
                    self.lane_counter[b] = 0
                self.lane_counter[b] = min(self.lane_counter[b] + 1, 1 << 30)
                self.lane_changed[b] = cv if self.lane_counter[b] > LANE_CHANGE_TICKS else -1
            else:
                self.lane_counter[b] = 0
                self.lane_changed[b] = -1
            if cv == self.lane_changed[b]:                                                 # :304-305
                cv = 3
                flags[b] = NAV_LANE_HELD
            th = -raw[b] + np.pi / 2                                                       # :308, _rotate
            c, s = np.cos(th), np.sin(th)
            rx, ry = c * wx + (-s) * wy, s * wx + c * wy
            cmds[b] = cv
            nxps[b] = np.float32(-rx), np.float32(-ry)                                     # :314
        return dict(cmds=cmds, nxps=nxps, poses=poses, flags=flags)

    def update(self, steer, speeds, gnss, compass):
        """EKF.step(spd, steer, lat, lon, compass - pi/2) (:338, ekf.py:45-91) of the agents past their first frame."""
        gnss, raw = np.asarray(gnss, np.float64), np.asarray(compass, np.float64)
        steer, speeds = np.asarray(steer, np.float64), np.asarray(speeds, np.float64)
        for b in np.flatnonzero(self.frames >= 2):
            spd, st = speeds[b], steer[b]
            cmp = 0. if np.isnan(raw[b]) else raw[b]
            z = np.array([*self.ekf_xy(gnss[b, 0], gnss[b, 1]), cmp - math.pi / 2])
            xk, yk, tk = self.x[b]
            beta = np.arctan(LR * np.tan(st * MAX_STEER) / L)                              # kbm_step
            xp = np.array([xk + spd * math.cos(tk + beta) * DT, yk + spd * math.sin(tk + beta) * DT,
                           tk + spd * np.tan(tk) * np.cos(beta) / L * DT])
            pp = self.p[b] + Q
            k = pp * (1.0 / (pp + R_DIAG))
            y = z - xp
            corr = np.array([(k[0] * y[0] + 0.0 * y[1]) + 0.0 * y[2], (0.0 * y[0] + k[1] * y[1]) + 0.0 * y[2],
                             (0.0 * y[0] + 0.0 * y[1]) + k[2] * y[2]])
            self.x[b] = xp + corr
            self.theta_pred[b] = xp[2]
            self.p[b] = (1.0 - k) * pp


# ---------------------------------------------------------------------------------------------------------------- the sequence
M_PER_DEG = EARTH_RADIUS * math.pi / 180
ALL_OPTIONS = (-1, 1, 2, 3, 4, 5, 6)


def _to_gnss(xy, lat0):
    """metres -> (lat, lon) degrees near latitude lat0 (the inverse of latlon_to_xy up to the route's own scale)."""
    return np.stack([lat0 + xy[..., 0] / M_PER_DEG, xy[..., 1] / (M_PER_DEG * math.cos(math.radians(lat0)))], -1)


def _polyline(rs, n, spacing, turn=0.15):
    """n nodes from the origin, ``spacing`` metres apart, heading drifting by up to ``turn`` rad per node."""
    head = np.cumsum(np.concatenate([[rs.uniform(0, 2 * np.pi)], rs.uniform(-turn, turn, max(n - 1, 0))]))
    steps = spacing * np.stack([np.cos(head), np.sin(head)], -1)
    return np.concatenate([np.zeros((1, 2)), np.cumsum(steps[:-1], 0)])[:n], head


def _along(nodes, s):
    """points at arc lengths s along the polyline (extended straight past its last node), and their headings."""
    if len(nodes) == 1:
        nodes = np.concatenate([nodes, nodes + [[1.0, 0.0]]])
    seg = np.diff(nodes, axis=0)
    ln = np.linalg.norm(seg, axis=1)
    cum = np.concatenate([[0], np.cumsum(ln)])
    k = np.clip(np.searchsorted(cum, s, side="right") - 1, 0, len(seg) - 1)
    u = (s - cum[k]) / ln[k]
    return nodes[k] + u[:, None] * seg[k], np.arctan2(seg[k, 1], seg[k, 0])


def nav_sequence(seed, ticks=1100):
    """The pinned 8-agent sequence: dict(routes = {tick: [(agent, route)]} (routes as _global_plan lists with int RoadOption
    values), gnss (ticks, 8, 3), compass (ticks, 8), speed (ticks, 8) fp64, steer (ticks, 8) fp32-representable fp64).
      0: a 1-node route, re-set at tick 500 to a 3-node route         4: a 4 held 150 ticks, then a 5 held past the window
      1: a 2-node route driven past its end                           5: compass within 1e-3 of pi for 300 ticks; a stop
      2: 450 nodes, every RoadOption, lane changes in the look-ahead  6: 400 nodes, re-set at tick 550 to 300 new nodes
      3: a 4 held past 300 ticks, then a 5                            7: 60 m off its route: never advances
    Every agent has NaN compass ticks, zero-speed stretches and a fp32 steer random walk."""
    rs = np.random.RandomState(seed)
    B = 8
    gnss = np.zeros((ticks, B, 3))
    compass = np.zeros((ticks, B))
    speed = np.zeros((ticks, B))
    steer = np.zeros((ticks, B))
    routes = {0: []}
    for b in range(B):
        lat0 = 0.0004 * b - 0.001
        v = np.full(ticks, 0.3)                                  # metres per tick along the route
        lateral = np.zeros(ticks)
        plans = []                                               # (first tick, nodes (n, 2) m, cmds)
        if b == 0:
            plans = [(0, np.array([[4.0, 0.0]]), [4]), (500, None, [2, -1, 4])]
        elif b == 1:
            plans = [(0, np.array([[0.0, 0.0], [8.0, 0.0]]), [4, 3])]
        elif b == 2:
            cm = rs.choice(ALL_OPTIONS, 450, p=[0.04, 0.06, 0.06, 0.06, 0.64, 0.07, 0.07])
            cm[:7] = [-1, 1, 2, 3, 4, 5, 6]
            plans = [(0, _polyline(rs, 450, 3.0)[0], list(cm))]
            v = rs.uniform(0.2, 0.45, ticks)
        elif b in (3, 4):
            nodes = np.stack([np.arange(40) * 4.0, np.zeros(40)], -1)
            cm = [4] * 40
            cm[10], cm[14] = 5, 6
            plans = [(0, nodes, cm)]
            if b == 3:      # reach node 10 (40 m) and stay 420 ticks, then on to node 14
                v[:] = 0.4; v[105:525] = 0.0
            else:           # creep: ~150 ticks on the 5 (cmd 4), then the 6 (cmd 5) for the rest of the window and beyond
                v[:] = 0.4; v[96:] = 0.027
        elif b == 5:
            plans = [(0, _polyline(rs, 200, 5.0, turn=0.05)[0], list(rs.choice([3, 4, 4, 4, 1, 2], 200)))]
            v[600:700] = 0.0
        elif b == 6:
            plans = [(0, _polyline(rs, 400, 4.0)[0], list(rs.choice(ALL_OPTIONS, 400))),
                     (550, _polyline(rs, 300, 4.0)[0], list(rs.choice(ALL_OPTIONS, 300)))]
        else:
            plans = [(0, _polyline(rs, 100, 5.0)[0], [4] * 100)]
            lateral[:] = 60.0
        v[rs.rand(ticks) < 0.05] = 0.0                           # zero-speed ticks
        for k, (t0, nodes, cm) in enumerate(plans):
            t1 = plans[k + 1][0] if k + 1 < len(plans) else ticks
            if nodes is None:                                    # continue from where the previous plan left the agent
                nodes = pos[-1] + np.stack([np.arange(len(cm)) * 6.0 + 3.0, np.zeros(len(cm))], -1)
            else:
                nodes = nodes + (pos[-1] if t0 > 0 else 0)
            s = np.cumsum(v[t0:t1]) - v[t0]
            if b == 1:
                s = s - 3.0                                      # start 3 m before the first node
            p, head = _along(nodes, s)
            normal = np.stack([-np.sin(head), np.cos(head)], -1)
            pos = p + lateral[t0:t1, None] * normal + rs.normal(0, 0.25, (t1 - t0, 2))
            gnss[t0:t1, b, :2] = _to_gnss(pos, lat0)
            gnss[t0:t1, b, 2] = rs.uniform(0, 2, t1 - t0)
            compass[t0:t1, b] = np.mod(head + np.pi / 2 + rs.normal(0, 0.02, t1 - t0), 2 * np.pi)
            speed[t0:t1, b] = v[t0:t1] * 20.0
            g = _to_gnss(nodes, lat0)
            routes.setdefault(t0, []).append((b, [({"lat": float(la), "lon": float(lo), "z": 0.0}, int(c))
                                                  for (la, lo), c in zip(g, cm)]))
        steer[:, b] = np.clip(np.cumsum(rs.normal(0, 0.05, ticks)), -1, 1).astype(np.float32)
    compass[100:400, 5] = np.pi + rs.uniform(-1e-3, 1e-3, 300)
    compass[rs.rand(ticks, B) < 0.03] = np.nan
    speed[speed == 0] = 0.0
    return dict(routes=routes, gnss=gnss, compass=compass, speed=speed, steer=steer)


def nav_drive(B, lengths, ticks, seed, reset_at=500):
    """B agents on routes of ``lengths[b % len(lengths)]`` nodes 4 m apart with every RoadOption: gnss (ticks, B, 3), compass
    (ticks, B) raw with NaN ticks and stretches near pi, speed (ticks, B) with stops, steer (ticks, B) fp32; every fifth agent
    60 m off its route, every seventh re-set to a new route at ``reset_at``.  -> (routes {tick: [(agent, route)]}, inputs)"""
    rs = np.random.RandomState(seed)
    gnss, compass = np.zeros((ticks, B, 3)), np.zeros((ticks, B))
    speed = np.zeros((ticks, B))
    steer = np.clip(np.cumsum(rs.normal(0, 0.05, (ticks, B)), 0), -1, 1).astype(np.float32).astype(np.float64)
    routes = {}
    for b in range(B):
        n = lengths[b % len(lengths)]
        lat0 = rs.uniform(-0.002, 0.002)
        v = rs.uniform(0.15, 0.5) * np.ones(ticks)
        v[rs.rand(ticks) < 0.05] = 0.0
        starts = [0] + ([reset_at] if b % 7 == 3 and reset_at < ticks else [])
        pos0 = np.zeros(2)
        for k, t0 in enumerate(starts):
            t1 = starts[k + 1] if k + 1 < len(starts) else ticks
            nodes = _polyline(rs, n, 4.0, turn=0.1)[0] + pos0
            cm = rs.choice(ALL_OPTIONS, n, p=[0.05, 0.07, 0.07, 0.07, 0.6, 0.07, 0.07])
            s = np.cumsum(v[t0:t1]) - v[t0]
            p, head = _along(nodes, s)
            off = 60.0 if b % 5 == 4 else 0.0
            pos = p + off * np.stack([-np.sin(head), np.cos(head)], -1) + rs.normal(0, 0.25, (t1 - t0, 2))
            gnss[t0:t1, b, :2] = _to_gnss(pos, lat0)
            compass[t0:t1, b] = np.mod(head + np.pi / 2 + rs.normal(0, 0.02, t1 - t0), 2 * np.pi)
            speed[t0:t1, b] = v[t0:t1] * 20.0
            g = _to_gnss(nodes, lat0)
            routes.setdefault(t0, []).append((b, [({"lat": float(a), "lon": float(o)}, int(c)) for (a, o), c in zip(g, cm)]))
            pos0 = pos[-1]
        if b % 4 == 1 and ticks > 200:
            t0 = rs.randint(0, ticks - 200)
            compass[t0:t0 + 200, b] = np.pi + rs.uniform(-1e-3, 1e-3, 200)
    compass[rs.rand(ticks, B) < 0.03] = np.nan
    return routes, dict(gnss=gnss, compass=compass, speed=speed, steer=steer)
