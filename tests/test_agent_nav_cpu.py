"""CPU: the numpy statement of the agent's localisation and route following (oracle/nav_ref.py) against the reference's outputs
pinned in tests/golden/agent_nav.npz (oracle/pin_nav.py), its O(1) route scans against the reference's full loops, the host side
of AgentNavigator.set_routes, and the C ABI of the new entry points."""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch

from lav_b200 import capi, control, navigation, ops
from oracle import nav_ref as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "agent_nav.npz"))


def _rel(a, b):
    fin = np.isfinite(b)
    assert np.array_equal(fin, np.isfinite(a))
    return float((np.abs(a[fin] - b[fin]) / np.maximum(np.abs(b[fin]), 1.0)).max()) if fin.any() else 0.0


def test_statement_equals_the_pinned_reference():
    seed, B, T, tol = int(GOLD["seed"]), int(GOLD["batch"]), int(GOLD["ticks"]), float(GOLD["tolerance"])
    assert B == 8 and T >= 1000
    x = N.nav_sequence(seed, T)
    nav = N.AgentNavRef(B)
    worst = 0.0
    for t in range(T):
        if t in x["routes"]:
            nav.set_routes([a for a, _ in x["routes"][t]], [r for _, r in x["routes"][t]])
        got = nav.front(x["gnss"][t], x["compass"][t])
        assert np.array_equal(got["cmds"], GOLD["cmds"][t]) and np.array_equal(got["flags"], GOLD["flags"][t]), t
        live = GOLD["flags"][t] != N.NAV_FIRST_FRAME
        ints = GOLD["ints"][t]
        assert np.array_equal(nav.wp_idx[live], ints[live, 0]) and np.array_equal(nav.rp_idx[live], ints[live, 1]), t
        assert np.array_equal(nav.lane_counter, ints[:, 2]) and np.array_equal(nav.lane_changed, ints[:, 3]), t
        worst = max(worst, _rel(got["poses"], GOLD["poses"][t]), _rel(got["nxps"].astype(np.float64), GOLD["nxps"][t].astype(np.float64)))
        nav.update(x["steer"][t], x["speed"][t], x["gnss"][t], x["compass"][t])
        worst = max(worst, _rel(nav.x, GOLD["ekf_x"][t]), _rel(nav.p, GOLD["ekf_p"][t]))
    assert worst <= tol, worst


def test_sequence_covers_the_cases():
    x = N.nav_sequence(int(GOLD["seed"]), int(GOLD["ticks"]))
    lens = sorted({len(r) for lst in x["routes"].values() for _, r in lst})
    assert lens[0] == 1 and 2 in lens and max(lens) >= 300
    assert {c for lst in x["routes"].values() for _, r in lst for _, c in r} == set(N.ALL_OPTIONS)
    assert len([t for t in x["routes"] if t > 0]) >= 1                                  # a route re-set mid-run
    assert np.isnan(x["compass"]).any() and (x["speed"] == 0).any()
    near_pi = np.abs(np.nan_to_num(x["compass"], nan=0.0) - np.pi) < 1e-3
    assert near_pi.sum() > 100
    flags, ints = GOLD["flags"], GOLD["ints"]
    assert (flags == N.NAV_LANE_HELD).any()                                              # a 4 / 5 held past 300 ticks
    assert ints[:, 4, 2].max() > 300 and (ints[:, 4, 3] == 5).any()                      # 4 -> 5 inside the window, no reset
    assert ints[1:, 7, 0].max() == -1 and ints[:, 7, 1].max() == 0                       # never advances
    assert ints[:, 1, 0].max() == 1 and ints[:, 1, 1].max() == 1                         # the end of a 2-node route


def _full_waypointer(xy, rc, idx, cp, cp_cmd, cx, cy):
    """Waypointer.tick as written (waypointer.py:55-96, pop_turning False): the loop over every node, then the look-ahead"""
    i = None
    for i in range(len(xy)):
        wx, wy, cmd = xy[i, 0], xy[i, 1], rc[i]
        dx, dy = cx - wx, cy - wy
        distance = np.sqrt(dx * dx + dy * dy)
        threshold = N.THRESH_BEFORE if cp_cmd == N.LANEFOLLOW and cmd != N.LANEFOLLOW else N.THRESH_AFTER
        if distance < threshold and i - idx == 1:
            cp, cp_cmd, idx = (wx, wy), int(cmd), idx + 1
            break
    look, cmd = 0, cp_cmd
    while i + 1 < len(xy) and look < 3:
        wcmd = rc[i + 1]
        if cmd != N.LANEFOLLOW:
            break
        if wcmd in (N.CHANGELANELEFT, N.CHANGELANERIGHT):
            cp, cp_cmd, idx = (xy[i + 1, 0], xy[i + 1, 1]), int(wcmd), i + 1
            break
        cmd = wcmd
        i += 1
        look += 1
    return idx, cp, cp_cmd


def test_o1_scan_equals_the_full_loop_on_the_sequence_routes():
    x = N.nav_sequence(int(GOLD["seed"]), int(GOLD["ticks"]))
    rs = np.random.RandomState(3)
    n = 0
    for lst in x["routes"].values():
        for _, r in lst:
            _, xy, rc = N.route_table(r)
            for _ in range(400):
                idx = int(rs.randint(-1, len(xy)))
                cp_cmd = int(rs.choice([4, 3, 5, 6, -1]))
                cp = tuple(xy[max(idx, 0)])
                c = xy[min(idx + 1, len(xy) - 1)] + rs.normal(0, 3.0, 2)
                assert N.waypointer_tick(xy, rc, idx, cp, cp_cmd, c[0], c[1]) == _full_waypointer(xy, rc, idx, cp, cp_cmd, c[0], c[1])
                n += 1
    assert n >= 4000


def test_route_table_is_the_planners_conversion():
    x = N.nav_sequence(int(GOLD["seed"]), int(GOLD["ticks"]))
    for _, r in x["routes"][0]:
        s1, xy1, c1 = navigation.route_table(r)
        s2, xy2, c2 = N.route_table(r)
        assert s1 == s2 and np.array_equal(xy1, xy2) and np.array_equal(c1, c2)
        lat = sum(g["lat"] * (math.pi / 180) for g, _ in r) / len(r)
        assert s1 == math.cos(lat)
    with pytest.raises(capi.LavbError):
        navigation.route_table([])
    with pytest.raises(capi.LavbError):
        navigation.route_table([({"lat": 0.0, "lon": 0.0}, 7)])


def test_set_routes_touches_only_its_agents():
    nav = navigation.AgentNavigator(5, device="cpu")
    x = N.nav_sequence(int(GOLD["seed"]), int(GOLD["ticks"]))
    routes = [r for _, r in x["routes"][0]]
    nav.set_routes(range(5), routes[:5])
    nav.state.view(5, -1)[:, :48] = torch.arange(48, dtype=torch.uint8)                  # stand-in for driven EKF state
    before = nav.state.clone().view(5, -1)
    nav.set_routes([1, 3], [routes[6], routes[0]])
    after = nav.state.view(5, -1)
    for b in (0, 2, 4):
        assert torch.equal(after[b], before[b])
    v = nav.state_views()
    assert (v["frames"][[1, 3]] == 0).all() and (v["lane_changed"][[1, 3]] == -1).all() and (v["ekf_x"][[1, 3]] == 0).all()
    assert v["route_scale"][1] == navigation.route_table(routes[6])[0] and v["ekf_scale"][3] == math.cos(1)
    route = nav.route.numpy()
    for b, r in zip(range(5), [routes[0], routes[6], routes[2], routes[0], routes[4]]):
        s, c = route[b]
        np.testing.assert_array_equal(nav.nodes.numpy()[s:s + c], navigation.route_table(r)[1])
    with pytest.raises(IndexError):
        nav.set_routes([5], [routes[0]])
    with pytest.raises(capi.LavbError):
        nav.set_routes([0], [[]])
    assert torch.equal(nav.state.view(5, -1)[0], before[0])
    with pytest.raises(capi.LavbError):
        navigation.AgentNavigator(2, device="cpu", pop_turning=True)


def test_abi_of_the_navigation_entry_points():
    hdr = open(os.path.join(ROOT, "include", "lav_b200.h")).read()
    handle = ctypes.CDLL(capi.LIB_PATH)
    for sym in ("lavb_agent_nav_state_bytes", "lavb_agent_nav_front", "lavb_agent_nav_update", "lavb_stack_job_poses",
                "lavb_agent_control_dcmd"):
        assert re.search(rf"\b{sym}\s*\(", hdr) and hasattr(handle, sym) and sym in capi.exported_symbols(), sym
    assert ops.agent_nav_state_bytes() == ops.NAV_STATE_DTYPE.itemsize == 128
    body = re.search(r"typedef struct lavb_nav_state \{(.*?)\} lavb_nav_state;", hdr, re.S).group(1)
    fields = []
    for ty, names in re.findall(r"^\s*(double|int)\s+([^;]+);", body, re.M):
        for nm in names.split(","):
            m = re.match(r"\s*(\w+)(?:\[(\d+)\])?", nm)
            fields.append((m.group(1), ty, int(m.group(2) or 1)))
    want = [(nm, "double" if ops.NAV_STATE_DTYPE[nm].base == np.float64 else "int",
             int(np.prod(ops.NAV_STATE_DTYPE[nm].shape) or 1)) for nm in ops.NAV_STATE_DTYPE.names]
    assert fields == want
    flags = dict(re.findall(r"#define (LAVB_NAV_\w+) (\d+)", hdr))
    assert {k: int(v) for k, v in flags.items()} == {"LAVB_NAV_FIRST_FRAME": navigation.FLAG_FIRST_FRAME,
                                                     "LAVB_NAV_NO_ROUTE": navigation.FLAG_NO_ROUTE,
                                                     "LAVB_NAV_LANE_HELD": navigation.FLAG_LANE_HELD}
    assert (navigation.FLAG_FIRST_FRAME, navigation.FLAG_NO_ROUTE, navigation.FLAG_LANE_HELD) == (
        N.NAV_FIRST_FRAME, N.NAV_NO_ROUTE, N.NAV_LANE_HELD)
    assert int(re.search(r"#define LAVB_CTL_BAD_CMD (\d+)", hdr).group(1)) == control.FLAG_BAD_CMD
    assert int(re.search(r"#define LAVB_STACK_JOB_BYTES (\d+)", hdr).group(1)) == ops.STACK_JOB_DTYPE.itemsize
    assert ops.STACK_JOB_DTYPE.fields["R"][1] == 24 and ops.STACK_JOB_DTYPE.fields["dx"][1] == 60
    assert ops.STACK_JOB_DTYPE.fields["dy"][1] == 64


def test_entry_points_reject_malformed_calls_before_writing():
    lib = capi.lib()
    V = ctypes.c_void_p
    # sizes and null pointers are checked on the host, before any launch (no device is touched)
    assert lib.lavb_agent_nav_front(-1, None, None, 0, None, None, None, None, None, None, None, None, None) != 0
    assert lib.lavb_agent_nav_front(2, None, None, -1, None, None, None, None, None, None, None, None, None) != 0
    assert lib.lavb_agent_nav_front(2, None, None, 0, V(64), V(64), V(64), V(64), V(64), V(64), None, V(64), None) != 0
    assert lib.lavb_agent_nav_front(2, V(64), V(64), 4, V(64), V(72), V(64), V(64), V(64), V(64), V(64), V(64), None) != 0
    assert lib.lavb_agent_nav_front(0, None, None, 0, None, None, None, None, None, None, None, None, None) == 0
    assert lib.lavb_agent_nav_update(-1, None, None, None, None, None, None) != 0
    assert lib.lavb_agent_nav_update(3, V(64), V(64), None, V(64), V(64), None) != 0
    assert lib.lavb_agent_nav_update(3, V(64), V(64), V(72), V(64), V(64), None) != 0
    assert lib.lavb_stack_job_poses(V(64), 2, 0, 5, 11, 0, V(64), None, None) != 0
    assert lib.lavb_stack_job_poses(V(64), 2, 3, 5, 11, -1, V(64), None, None) != 0
    assert lib.lavb_stack_job_poses(None, 2, 3, 5, 11, 0, V(64), None, None) != 0
    assert lib.lavb_stack_job_poses(V(64), 2, 3, 5, 11, 0, V(64), V(68), None) != 0
    assert b"stack_job_poses" in lib.lavb_last_error()
