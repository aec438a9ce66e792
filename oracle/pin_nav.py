"""Pin the agent's localisation and route following (oracle/nav_ref.py) against the REFERENCE and write tests/golden/agent_nav.npz.
Every other golden is left untouched.

Runs only where the reference sources are readable.  It imports the unmodified team_code_v2/ekf.py, waypointer.py and planner.py
(RoadOption from oracle/refshim) and lav_agent_fast._rotate, and drives them per agent through run_step's head and EKF step in
the reference's own order, restated below with line citations: the seeded 8-agent sequence of oracle.nav_ref.nav_sequence over
1100 ticks, whose routes are set and re-set as _global_plan lists of (gnss dict, RoadOption).  It checks AgentNavRef against it
(integer state, commands and flags exactly; the EKF state, poses and targets within the tolerance it measures and states) and
stores the seed and the reference's outputs and state per tick (the inputs are regenerated from the seed).

    python oracle/pin_nav.py
"""
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("LAV_REFERENCE", "/root/reference")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "refshim"))
sys.path.insert(0, os.path.join(REF, "team_code_v2"))

from oracle.nav_ref import (NAV_FIRST_FRAME, NAV_LANE_HELD, AgentNavRef, nav_sequence)  # noqa: E402

SEED, B, TICKS = 1207, 8, 1100
GOLD = os.path.join(ROOT, "tests", "golden", "agent_nav.npz")
TOL = 1e-12          # relative, per value (the trig functions of numpy and math against each other)


class RefAgent:
    """what LAVAgent holds for the head of run_step (lav_agent_fast.py:76-77, 137-138, 155-158), for one route"""

    def __init__(self, plan):
        from agents.navigation.local_planner import RoadOption
        from ekf import EKF
        self.plan = [(g, RoadOption(c)) for g, c in plan]
        self.ekf = EKF(1, 1.477531, 1.393600)                                             # :137
        self.ekf_initialized = False
        self.num_frames = 0
        self.waypointer = self.planner = None
        self.lane_change_counter, self.lane_changed = 0, None

    def head(self, gps, imu_compass):
        from lav_agent_fast import _rotate
        from planner import RoutePlanner
        from waypointer import Waypointer
        import torch
        self.num_frames += 1                                                              # :207
        compass = imu_compass                                                             # :215
        if np.isnan(compass):                                                             # :219-220
            compass = 0.
        self.compass = compass
        if not self.ekf_initialized:                                                      # :222-224
            self.ekf.init(*gps[:2], compass - math.pi / 2)
            self.ekf_initialized = True
        pose = np.array([*self.ekf.x[:2], self.ekf.x[2]])                                 # :226
        if self.num_frames <= 1:                                                          # :235-237
            return 3, np.zeros(2, np.float32), pose, NAV_FIRST_FRAME
        if self.waypointer is None:                                                       # :280-286
            self.waypointer = Waypointer(self.plan, gps, pop_lane_change=True)
            self.planner = RoutePlanner(self.plan)
        _, _, cmd = self.waypointer.tick(gps)                                             # :288-289
        wx, wy = self.planner.run_step(gps)
        cmd_value = cmd.value - 1                                                         # :291-305
        cmd_value = 3 if cmd_value < 0 else cmd_value
        if cmd_value in [4, 5]:
            if self.lane_changed is not None and cmd_value != self.lane_changed:
                self.lane_change_counter = 0
            self.lane_change_counter += 1
            self.lane_changed = cmd_value if self.lane_change_counter > {4: 300, 5: 300}.get(cmd_value) else None
        else:
            self.lane_change_counter = 0
            self.lane_changed = None
        flag = 0
        if cmd_value == self.lane_changed:
            cmd_value = 3
            flag = NAV_LANE_HELD
        wx, wy = _rotate(wx, wy, -imu_compass + np.pi / 2)                                # :308
        nxps = torch.tensor([-wx, -wy]).float().numpy()                                   # :314
        return cmd_value, nxps, pose, flag

    def step(self, spd, steer, gps):
        if self.num_frames > 1:                                                           # :338, past the early return
            self.ekf.step(spd, steer, *gps[:2], self.compass - math.pi / 2)


def main():
    x = nav_sequence(SEED, TICKS)
    ref = [None] * B
    mine = AgentNavRef(B)
    cmds = np.zeros((TICKS, B), np.int32)
    nxps = np.zeros((TICKS, B, 2), np.float32)
    poses = np.zeros((TICKS, B, 3))
    flags = np.zeros((TICKS, B), np.int32)
    ekf_x = np.zeros((TICKS, B, 3))
    ekf_p = np.zeros((TICKS, B, 3))
    ints = np.zeros((TICKS, B, 4), np.int64)            # Waypointer / RoutePlanner current_idx, lane counter, lane_changed
    worst = dict(poses=0.0, nxps=0.0, ekf_x=0.0, ekf_p=0.0)
    rel = lambda a, b: float(np.nanmax(np.abs(a - b) / np.maximum(np.abs(b), 1.0))) if np.isfinite(b).any() else 0.0
    lookahead = 0
    for t in range(TICKS):
        if t in x["routes"]:
            agents = [a for a, _ in x["routes"][t]]
            plans = [r for _, r in x["routes"][t]]
            for a, r in zip(agents, plans):
                ref[a] = RefAgent(r)
            mine.set_routes(agents, plans)
        got = mine.front(x["gnss"][t], x["compass"][t])
        for b in range(B):
            before = (ref[b].waypointer.current_idx if ref[b].waypointer else None)
            c, n, p, f = ref[b].head(x["gnss"][t, b], x["compass"][t, b])
            cmds[t, b], nxps[t, b], poses[t, b], flags[t, b] = c, n, p, f
            wp, rp = ref[b].waypointer, ref[b].planner
            ints[t, b] = (wp.current_idx if wp else 0, rp.current_idx if rp else 0, ref[b].lane_change_counter,
                          -1 if ref[b].lane_changed is None else ref[b].lane_changed)
            if wp is not None and before is not None and wp.current_idx > before + 1:
                lookahead += 1
        assert np.array_equal(got["cmds"], cmds[t]), (t, got["cmds"], cmds[t])
        assert np.array_equal(got["flags"], flags[t]), (t, got["flags"], flags[t])
        live = flags[t] != NAV_FIRST_FRAME
        assert np.array_equal(mine.wp_idx[live], ints[t, live, 0]) and np.array_equal(mine.rp_idx[live], ints[t, live, 1]), t
        assert np.array_equal(mine.lane_counter, ints[t, :, 2]) and np.array_equal(mine.lane_changed, ints[t, :, 3]), t
        assert np.array_equal(np.isnan(got["nxps"]), np.isnan(nxps[t])), t
        worst["poses"] = max(worst["poses"], rel(got["poses"], poses[t]))
        worst["nxps"] = max(worst["nxps"], rel(got["nxps"].astype(np.float64), nxps[t].astype(np.float64)))
        control = np.zeros((B, 3), np.float32)
        control[:, 0] = x["steer"][t]
        mine.update(control[:, 0], x["speed"][t], x["gnss"][t], x["compass"][t])
        for b in range(B):
            ref[b].step(x["speed"][t, b], float(control[b, 0]), x["gnss"][t, b])
            ekf_x[t, b], ekf_p[t, b] = ref[b].ekf.x, np.diag(ref[b].ekf.P)
            assert not np.any(ref[b].ekf.P - np.diag(np.diag(ref[b].ekf.P))), (t, b)      # P stays diagonal
        worst["ekf_x"] = max(worst["ekf_x"], rel(mine.x, ekf_x[t]))
        worst["ekf_p"] = max(worst["ekf_p"], rel(mine.p, ekf_p[t]))
    # the O(1) Waypointer.tick against the reference's full loop, on every route of the sequence, from random states at
    # positions around the next node
    from agents.navigation.local_planner import RoadOption
    from waypointer import Waypointer
    from oracle.nav_ref import route_table, waypointer_tick
    rs = np.random.RandomState(SEED)
    checked = 0
    for t, lst in x["routes"].items():
        for _, r in lst:
            _, xy, rc = route_table(r)
            plan = [(g, RoadOption(c)) for g, c in r]
            for _ in range(300):
                idx = int(rs.randint(-1, len(xy)))
                cp_cmd = int(rs.choice([4, 3, 5, 6, -1]))
                g = r[min(idx + 1, len(r) - 1)][0]
                gps = np.array([g["lat"] + rs.normal(0, 3e-5), g["lon"] + rs.normal(0, 3e-5), 0.0])
                wp = Waypointer(plan, gps, pop_lane_change=True)
                cp = tuple(xy[max(idx, 0)])
                wp.current_idx, wp.checkpoint = idx, (cp[0], cp[1], RoadOption(cp_cmd))
                _, _, cmd = wp.tick(gps)
                cx, cy = wp.latlon_to_xy(gps[0], gps[1])
                got = waypointer_tick(xy, rc, idx, cp, cp_cmd, cx, cy)
                assert (got[0], got[1], got[2]) == (wp.current_idx, tuple(wp.checkpoint[:2]), cmd.value), (got, wp.current_idx)
                checked += 1
    counts = dict(first_frames=int((flags == NAV_FIRST_FRAME).sum()), lane_held=int((flags == NAV_LANE_HELD).sum()),
                  lookahead_jumps=lookahead, nan_compass=int(np.isnan(x["compass"]).sum()),
                  cmd_values=sorted(set(int(v) for v in np.unique(cmds))),
                  waypointer_max_idx=[int(ints[:, b, 0].max()) for b in range(B)],
                  planner_max_idx=[int(ints[:, b, 1].max()) for b in range(B)],
                  max_lane_counter=[int(ints[:, b, 2].max()) for b in range(B)])
    print("events:", counts)
    print(f"AgentNavRef against the reference over {TICKS} ticks x {B} agents: commands, flags, indices and lane state equal; "
          f"max relative diff {', '.join(f'{k} {v:.2e}' for k, v in worst.items())} (numpy {np.__version__}); "
          f"O(1) Waypointer.tick equals the reference's full loop on {checked} states")
    assert max(worst.values()) <= TOL, worst
    assert counts["lane_held"] > 0 and lookahead > 0 and counts["first_frames"] == 10
    assert ints[1:, 7, 0].max() == -1 and ints[:, 7, 1].max() == 0                       # the agent off its route never advances
    np.savez_compressed(GOLD, seed=SEED, batch=B, ticks=TICKS, tolerance=TOL, numpy_version=np.__version__, cmds=cmds,
                        nxps=nxps, poses=poses, flags=flags, ekf_x=ekf_x, ekf_p=ekf_p, ints=ints)
    print(f"wrote {GOLD} ({os.path.getsize(GOLD) / 1e3:.0f} kB)")


if __name__ == "__main__":
    main()
