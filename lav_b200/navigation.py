"""The agent's localisation and route following on the GPU: the head of LAVAgent.run_step (team_code_v2/lav_agent_fast.py:215-226,
280-308, 314) — the compass NaN rule, EKF.init, the pose, Waypointer.tick, RoutePlanner.run_step, the command mapping, the
lane-change rule and the target point in the ego frame — and its EKF step after the controls (:338), for B agents in one
launch each, with every agent's EKF, Waypointer, RoutePlanner and lane-change state resident on the device.

    nav = AgentNavigator(B, device)
    nav.set_routes(range(B), plans)                  # each agent's _global_plan: [(gnss dict, RoadOption or int)]
    res = nav.front(gnss, compass)                   # cmds (B,) int32, nxps (B, 2) fp32, poses (B, 3) fp64, flags (B,) int32
    ...                                              # planner (StaticFramePipeline(navigator=nav)), AgentController.step
    nav.update(control, speeds)                      # EKF.step with the controller's steer; the gnss and compass of front()

The route scans are O(1) per agent: only node current_idx + 1 can be taken (include/lav_b200.h, lavb_agent_nav_front).  A route's
node positions and scale are computed once, on the host, by set_routes with the reference's own float operations.
Flags per agent (res["flags"]) are the FLAG_* bits below.
"""
import math

import numpy as np
import torch

from . import capi, ops

# LAVB_NAV_* of include/lav_b200.h
FLAG_FIRST_FRAME, FLAG_NO_ROUTE, FLAG_LANE_HELD = 1, 2, 4
EARTH_RADIUS = 6371e3
ROAD_OPTIONS = (-1, 1, 2, 3, 4, 5, 6)               # the values of CARLA's RoadOption


def route_table(route):
    """(scale, xy (n, 2) fp64, cmd (n,) int32) of one _global_plan, as Waypointer and RoutePlanner convert it
    (waypointer.py:30-42, planner.py:16-27): cos_0 = the route latitudes in radians summed in order over the count,
    scale = math.cos(cos_0), x = R * lat * (pi / 180), y = R * lon * (pi / 180) * scale."""
    if len(route) == 0:
        raise capi.LavbError("set_routes: a route needs at least one node")
    cos_0 = 0.
    for gnss, _ in route:
        cos_0 += gnss['lat'] * (math.pi / 180)
    cos_0 = cos_0 / (len(route))
    scale = math.cos(cos_0)
    xy = np.array([(EARTH_RADIUS * g['lat'] * (math.pi / 180), EARTH_RADIUS * g['lon'] * (math.pi / 180) * scale)
                   for g, _ in route], dtype=np.float64)
    cmd = np.array([int(getattr(c, "value", c)) for _, c in route], dtype=np.int32)
    bad = sorted(set(cmd.tolist()) - set(ROAD_OPTIONS))
    if bad:
        raise capi.LavbError(f"set_routes: {bad} are not RoadOption values")
    return scale, xy, cmd


class AgentNavigator:
    """Navigation state and per-tick front / EKF step of ``batch`` agents on ``device``.  Until set_routes gives an agent a route,
    front() flags it FLAG_NO_ROUTE and computes nothing for it."""

    def __init__(self, batch, device=torch.device("cuda"), pop_turning=False):
        if pop_turning:
            raise capi.LavbError("AgentNavigator: the agent runs the Waypointer with pop_turning=False; pop_turning=True is not "
                                 "supported")
        self.B = int(batch)
        self.device = torch.device(device)
        self.record = ops.agent_nav_state_bytes()
        self.state = torch.zeros((self.B * self.record,), dtype=torch.uint8, device=self.device)
        self._routes = [None] * self.B                   # (xy, cmd) per agent, the host copy the node table is packed from
        self.nodes = torch.zeros((0, 2), dtype=torch.float64, device=self.device)
        self.node_cmd = torch.zeros((0,), dtype=torch.int32, device=self.device)
        self.route = torch.full((self.B, 2), -1, dtype=torch.int32, device=self.device)
        self.gnss = torch.zeros((self.B, 2), dtype=torch.float64, device=self.device)
        self.compass = torch.zeros((self.B,), dtype=torch.float64, device=self.device)
        self.speed = torch.zeros((self.B,), dtype=torch.float64, device=self.device)
        # set_routes, front and update all read and write the state, the route table and the staged inputs, and each may run on
        # another stream (a pipeline's begin() runs front on the pipeline's stream): each waits for the event of the one before
        self._last = None
        self.out = dict(cmds=torch.zeros((self.B,), dtype=torch.int32, device=self.device),
                        nxps=torch.zeros((self.B, 2), dtype=torch.float32, device=self.device),
                        poses=torch.zeros((self.B, 3), dtype=torch.float64, device=self.device),
                        flags=torch.zeros((self.B,), dtype=torch.int32, device=self.device))

    def set_routes(self, agents, routes):
        """give ``agents`` their routes (each a _global_plan: [(gnss dict with 'lat' / 'lon', RoadOption or its int value)]) and
        reset their EKF, Waypointer, RoutePlanner and lane-change state; no other agent's state changes."""
        agents = [int(a) for a in agents]
        routes = list(routes)
        if len(agents) != len(routes):
            raise capi.LavbError(f"set_routes: {len(agents)} agents for {len(routes)} routes")
        if any(a < 0 or a >= self.B for a in agents) or len(set(agents)) != len(agents):
            raise IndexError(f"set_routes: agents {agents} must be distinct, in 0..{self.B - 1}")
        tables = [route_table(r) for r in routes]        # every route is checked before anything changes
        rec = np.zeros(len(agents), dtype=ops.NAV_STATE_DTYPE)
        rec["route_scale"] = [t[0] for t in tables]
        rec["ekf_scale"] = math.cos(1)                   # EKF(1, ...) (lav_agent_fast.py:137): latlon_to_xy's math.cos(self.cos0)
        rec["lane_changed"] = -1
        for a, (_, xy, cmd) in zip(agents, tables):
            self._routes[a] = (xy, cmd)
        have = [b for b in range(self.B) if self._routes[b] is not None]
        counts = np.array([len(self._routes[b][0]) for b in have], dtype=np.int64)
        starts = np.concatenate([[0], np.cumsum(counts)[:-1]]) if len(have) else np.zeros(0, np.int64)
        if counts.sum() >= 2 ** 31:
            raise capi.LavbError(f"set_routes: {int(counts.sum())} route nodes in all, more than an int32 index")
        route = np.full((self.B, 2), -1, dtype=np.int32)
        route[have, 0], route[have, 1] = starts, counts
        self._wait_last()
        if self.device.type == "cuda":               # the old tables stay allocated until the fronts that read them are done
            cur = torch.cuda.current_stream(self.device)
            self.nodes.record_stream(cur)
            self.node_cmd.record_stream(cur)
        self.nodes = torch.from_numpy(np.concatenate([np.zeros((0, 2))] + [self._routes[b][0] for b in have])).to(self.device)
        self.node_cmd = torch.from_numpy(np.concatenate([np.zeros(0, np.int32)] + [self._routes[b][1] for b in have])).to(self.device)
        self.route.copy_(torch.from_numpy(route))
        rows = self.state.view(self.B, self.record)
        idx = torch.tensor(agents, dtype=torch.int64, device=self.device)
        rows[idx] = torch.from_numpy(rec.view(np.uint8).reshape(len(agents), self.record)).to(self.device)
        self._mark()

    def _wait_last(self):
        """order the current stream after the navigator's last set_routes / front / update, on whichever stream it ran"""
        if self._last is not None:
            torch.cuda.current_stream(self.device).wait_event(self._last)

    def _mark(self):
        if self.device.type == "cuda":
            self._last = torch.cuda.Event()
            self._last.record(torch.cuda.current_stream(self.device))

    def _inputs(self, gnss, compass):
        """stage this tick's gnss ((B, >=2) lat, lon) and raw compass ((B,)) into the navigator's fp64 device buffers"""
        g = torch.as_tensor(gnss, dtype=torch.float64)
        if g.dim() != 2 or g.shape[0] != self.B or g.shape[1] < 2:
            raise capi.LavbError(f"AgentNavigator: gnss must be ({self.B}, >=2), got {tuple(g.shape)}")
        c = torch.as_tensor(compass, dtype=torch.float64).reshape(-1)
        if c.shape[0] != self.B:
            raise capi.LavbError(f"AgentNavigator: compass must be ({self.B},), got {tuple(c.shape)}")
        self.gnss.copy_(g[:, :2], non_blocking=True)
        self.compass.copy_(c, non_blocking=True)

    def front(self, gnss, compass, out=None):
        """One tick's front: gnss (B, >=2) lat, lon (the GPS sensor's values); compass (B,) imu[-1], raw (NaN allowed); host arrays
        or device tensors.  -> dict(cmds, nxps, poses, flags), device tensors on the current stream (the navigator's own buffers,
        or ``out``'s tensors where given: cmds (B,) int32, nxps (B, 2) fp32, poses (B, 3) fp64, flags (B,) int32)."""
        self._wait_last()
        self._inputs(gnss, compass)
        res = dict(self.out, **(out or {}))
        ops.agent_nav_front(self.nodes, self.node_cmd, self.route, self.gnss, self.compass, self.state, res["cmds"], res["nxps"],
                            res["poses"], res["flags"])
        self._mark()
        return res

    def update(self, control, speeds):
        """EKF.step of every agent past its first frame, after the controls: control (B, 3) fp32 device tensor (AgentController's
        output; steer in column 0); speeds (B,) m/s; the gnss and compass of the last front()."""
        s = torch.as_tensor(speeds, dtype=torch.float64).reshape(-1)
        if s.shape[0] != self.B:
            raise capi.LavbError(f"AgentNavigator.update: speeds must be ({self.B},), got {tuple(s.shape)}")
        self._wait_last()
        self.speed.copy_(s, non_blocking=True)
        ops.agent_nav_update(control.contiguous(), self.speed, self.gnss, self.compass, self.state)
        self._mark()

    def state_views(self):
        """a host copy of the state (synchronises): the lavb_nav_state fields per agent (ops.NAV_STATE_DTYPE)."""
        self._wait_last()
        return self.state.cpu().numpy().view(ops.NAV_STATE_DTYPE).copy()
