"""CPU: the numpy fp64 statement of ops.driving_score (at-fault and exempt collisions, time to collision, the road, progress,
comfort) and of the host reduction DrivingScores, checked on hand-built cases with known answers; datasets.driving_score_table
against a direct loop over the keys of a recording written here."""
import math

import numpy as np
import pytest
import torch

from lav_b200 import ops
from lav_b200.ops import PLAN_SAFETY_ACTOR_DTYPE as DTYPE
from tests import test_plan_safety_cpu as P

EGO = P.EGO                                                   # (2.25, 1.0) half extents
DT = 0.25
FIELDS = {k: i for i, k in enumerate(ops.DRIVING_SCORE_FIELDS)}
# (low, high) of each comfort term, in ops.DRIVING_SCORE_COMFORT order; a symmetric bound is stated on |quantity|
BOUNDS = ((-4.05, 2.40), (None, 4.13), (None, 0.95), (None, 1.93), (None, 4.89))
NEAR = 1e-9                                                   # relative margin around a bound that device atan2 may cross


# ---------------------------------------------------------------------------------------------------- the numpy statement
def _wrap(d):
    return d - 2 * math.pi if d > math.pi else d + 2 * math.pi if d <= -math.pi else d


def _behind(ex, ey, hx, hy, e1, qx, qy):
    return (qx - ex) * hx + (qy - ey) * hy < -e1


def _fails(q, term):
    lo, hi = BOUNDS[term]
    fail = (q < lo or q > hi) if lo is not None else abs(q) > hi
    near = any(abs(abs(q) - abs(b)) <= NEAR * abs(b) for b in (lo, hi) if b is not None)
    return fail, near


def driving_score_ref(traj, expert, actors, offsets, ego_ext, road, dt=DT, grid=P.GRID):
    """every output of ops.driving_score: traj (B, n, T, 2) fp32, expert (B, T, 2) fp32, actors = PLAN_SAFETY_ACTOR_DTYPE records
    (rows x (T + 1), flat), offsets (B+1,), ego_ext (B, 2) fp64, road (B, H, W) uint8.  -> (res (B, n, 16) int32, ep (B, n, 2)
    fp64, near (B, n, 5) bool: a comfort term whose quantity came within NEAR of its bound at some step)."""
    traj, expert = np.asarray(traj, np.float32), np.asarray(expert, np.float32)
    B, n, T, _ = traj.shape
    actors = np.asarray(actors, DTYPE).reshape(-1, T + 1)
    K = int(math.floor(1.0 / dt + 1e-9))
    res = np.full((B, n, 16), -1, np.int32)
    ep = np.full((B, n, 2), np.nan)
    near = np.zeros((B, n, 5), bool)
    road_first = P.plan_safety_ref(traj, np.zeros(0, DTYPE), np.zeros(B + 1, np.int32), ego_ext, road, grid)[..., 4]
    res[..., FIELDS["off_road_step"]] = road_first
    for b in range(B):
        e1, e2 = float(ego_ext[b][0]), float(ego_ext[b][1])
        a = actors[offsets[b]:offsets[b + 1]]                                     # (A, T + 1)
        live = (a["present"] != 0) & ((a["typ"] == 0) | (a["typ"] == 1))
        box = lambda s: (a["x"][:, s], a["y"][:, s], a["sin"][:, s], -a["cos"][:, s], a["e1"][:, s], a["e2"][:, s])
        ex = [float(v) for v in expert[b].reshape(-1)]
        for j in range(n):
            x1, y1, hx1, hy1, ok = P.ego_boxes(traj[b, j][None])
            x, y = [0.0] + x1[0].tolist(), [0.0] + y1[0].tolist()
            hx, hy = [0.0] + hx1[0].tolist(), [-1.0] + hy1[0].tolist()
            with np.errstate(invalid="ignore"):
                vx = [0.0] + [(x[s] - x[s - 1]) / dt for s in range(1, T + 1)]
                vy = [0.0] + [(y[s] - y[s - 1]) / dt for s in range(1, T + 1)]
                sp = [0.0] + [math.sqrt(vx[s] * vx[s] + vy[s] * vy[s]) if np.isfinite(vx[s] * vx[s] + vy[s] * vy[s]) else np.nan
                              for s in range(1, T + 1)]
            bad = np.nonzero(~ok[0])[0]
            o = res[b, j]
            o[FIELDS["invalid_step"]] = bad[0] + 1 if len(bad) else -1
            o[FIELDS["comfort_mask"]] = 0
            valid = not len(bad)
            # progress along the expert
            L, qx, qy, best, prog = 0.0, 0.0, 0.0, math.inf, math.nan
            Px, Py = x[T], y[T]
            for k in range(1, T + 1):
                nx, ny = ex[2 * k - 2], ex[2 * k - 1]
                dx, dy = nx - qx, ny - qy
                dd = dx * dx + dy * dy
                length = math.sqrt(dd) if dd == dd and dd != math.inf else dd
                if valid:
                    u = ((Px - qx) * dx + (Py - qy) * dy) / dd if dd > 0.0 else 0.0
                    u = 0.0 if u < 0.0 else 1.0 if u > 1.0 else u
                    rx, ry = Px - (qx + u * dx), Py - (qy + u * dy)
                    d2 = rx * rx + ry * ry
                    if d2 < best:
                        best, prog = d2, L + u * length
                L = L + length
                qx, qy = nx, ny
            ep[b, j] = (prog, L)
            if not valid:
                continue
            # comfort
            psi = [None] + [math.atan2(hy[s], hx[s]) for s in range(1, T + 1)]
            mask = 0
            acc = {s: (sp[s] - sp[s - 1]) / dt for s in range(2, T + 1)}
            rate = {s: _wrap(psi[s] - psi[s - 1]) / dt for s in range(2, T + 1)}
            for s in range(2, T + 1):
                qs = [(0, acc[s]), (2, rate[s]), (4, sp[s] * rate[s])]
                if s >= 3:
                    qs += [(1, (acc[s] - acc[s - 1]) / dt), (3, (rate[s] - rate[s - 1]) / dt)]
                for term, q in qs:
                    fail, close = _fails(q, term)
                    near[b, j, term] |= close
                    if fail and not mask & (1 << term):
                        mask |= 1 << term
                        o[10 + term] = s
            o[FIELDS["comfort_mask"]] = mask
            # collisions and time to collision
            if not len(a):
                continue
            first = {}
            with np.errstate(invalid="ignore"):
                was = live[:, 0] & P.overlap((0.0, 0.0, 0.0, -1.0, e1, e2), box(0))
                for s in range(1, T + 1):
                    ego = (x[s], y[s], hx[s], hy[s], e1, e2)
                    now = live[:, s] & P.overlap(ego, box(s))
                    new = now & ~was
                    exempt = new & ((sp[s] < 0.05) | _behind(x[s], y[s], hx[s], hy[s], e1, a["x"][:, s], a["y"][:, s]))
                    moving = (a["present"][:, s - 1] != 0) & (a["present"][:, s] != 0)
                    ux = np.where(moving, (a["x"][:, s] - a["x"][:, s - 1]) / dt, 0.0)
                    uy = np.where(moving, (a["y"][:, s] - a["y"][:, s - 1]) / dt, 0.0)
                    ttc, seen = np.zeros(len(a), bool), np.zeros(len(a), bool)
                    if not sp[s] < 0.05:
                        for k in range(1, K + 1):                               # judged at the first projected overlap
                            tau = k * dt
                            ex_, ey_ = x[s] + tau * vx[s], y[s] + tau * vy[s]
                            qx_, qy_ = a["x"][:, s] + tau * ux, a["y"][:, s] + tau * uy
                            hit = P.overlap((ex_, ey_, hx[s], hy[s], e1, e2), (qx_, qy_, a["sin"][:, s], -a["cos"][:, s], a["e1"][:, s],
                                                                                a["e2"][:, s]))
                            ttc |= hit & ~seen & ~_behind(ex_, ey_, hx[s], hy[s], e1, qx_, qy_)
                            seen |= hit
                        ttc &= live[:, s] & ~now
                    for name, m in (("fault", new & ~exempt), ("exempt", exempt), ("ttc", ttc)):
                        if name not in first and m.any():
                            first[name] = (s, int(np.nonzero(m)[0][0]))
                    was = now
            for name, (s, row) in first.items():
                o[FIELDS[f"{name}_step"]], o[FIELDS[f"{name}_row"]] = s, row
                if name != "ttc":
                    o[FIELDS[f"{name}_class"]] = a["typ"][row, s]
    return res, ep, near


def views(res, ep):
    """driving_score_views of statement outputs."""
    v = {k: res[..., i] for k, i in FIELDS.items()}
    v["progress"], v["length"] = ep[..., 0], ep[..., 1]
    return v


# ---------------------------------------------------------------------------------------------------- hand-built cases
def track(xy, psi=0.0, e=EGO, typ=1, present=None):
    """one actor row of T + 1 records at the points ``xy`` (T + 1, 2) with relative yaw psi."""
    xy = np.asarray(xy, np.float64)
    r = np.zeros(len(xy), DTYPE)
    for s, (px, py) in enumerate(xy):
        if present is None or present[s]:
            r[s] = (px, py, math.cos(psi), math.sin(psi), e[0], e[1], typ, 1)
    return r


def line(T, x0, y0, vx=0.0, vy=0.0):
    """T + 1 points from (x0, y0) moving (vx, vy) metres per step."""
    return [(x0 + vx * s, y0 + vy * s) for s in range(T + 1)]


def plan(points):
    return np.array([points], np.float32)


def run_case(traj, rows, road=None, expert=None, fn=None):
    """the record, ep and near of one sample's trajectories (n, T, 2) against actor rows; the expert defaults to trajectory 0."""
    T = traj.shape[1]
    actors, offsets = P.pack([rows], T + 1)
    expert = traj[0] if expert is None else np.asarray(expert, np.float32)
    road = P.road_plane() if road is None else road
    res, ep, near = (fn or driving_score_ref)(traj[None], expert[None], actors, offsets, np.array([EGO]), road[None])
    return res[0], ep[0], near[0]


def terms(traj, rows, **kw):
    from lav_b200.evaluate import driving_terms
    res, ep, _ = run_case(traj, rows, **kw)
    t = driving_terms(views(res, ep))
    return res[0], {k: v[0] for k, v in t.items()}


def straight(T, step=1.0):
    return plan([(0.0, -step * (t + 1)) for t in range(T)])


def test_moving_ego_runs_into_a_stopped_car():
    T = 6
    res, t = terms(straight(T), [track(line(T, 0.0, -8.0))])
    assert (res[FIELDS["fault_step"]], res[FIELDS["fault_row"]], res[FIELDS["fault_class"]]) == (4, 0, 1)
    assert res[FIELDS["exempt_step"]] == -1 and res[FIELDS["ttc_step"]] == 1 and not t["nc"] and t["pdms"] == 0.0


def test_a_faster_car_from_behind_is_exempt():
    T = 5
    res, t = terms(straight(T), [track(line(T, 0.0, 8.0, vy=-2.0))])
    assert res[FIELDS["fault_step"]] == -1 and (res[FIELDS["exempt_step"]], res[FIELDS["exempt_class"]]) == (4, 1)
    assert res[FIELDS["ttc_step"]] == -1 and t["nc"] and t["ttc"] and t["pdms"] == 1.0


def test_a_stopped_ego_that_is_hit_keeps_nc():
    T = 4
    res, t = terms(plan([(0.0, 0.0)] * T), [track(line(T, 8.0, 0.0, vx=-2.0), psi=math.pi / 2)])
    assert res[FIELDS["exempt_step"]] == 3 and res[FIELDS["fault_step"]] == -1 and res[FIELDS["ttc_step"]] == -1
    assert t["nc"] and t["ep"] == 1.0 and t["comfort"] and t["pdms"] == 1.0


@pytest.mark.parametrize("after,ttc", [(2, 1), (8, -1)])
def test_a_car_crossing_ahead(after, ttc):
    """a car crossing the path ``after`` steps past the horizon (0.5 s and 2 s): a TTC violation only within 1 s."""
    T, cross = 2, 2 + after
    car = track(line(T, -4.0 * cross, -float(cross), vx=4.0), psi=math.pi / 2)
    res, t = terms(straight(T), [car])
    assert res[FIELDS["fault_step"]] == -1 and res[FIELDS["exempt_step"]] == -1 and t["nc"]
    assert res[FIELDS["ttc_step"]] == ttc and bool(t["ttc"]) == (ttc < 0)


def test_progress_along_the_expert():
    T = 4
    res, ep, _ = run_case(straight(T, 1.25), [], expert=straight(T, 2.5)[0])
    assert ep[0].tolist() == [5.0, 10.0]
    _, t = terms(straight(T, 1.25), [], expert=straight(T, 2.5)[0])
    assert t["ep"] == 0.5 and t["pdms"] == (5 + 5 * 0.5 + 2) / 12
    _, t = terms(straight(T, 0.5), [], expert=straight(T, 1.0)[0])          # an expert of 4 m
    assert t["ep"] == 1.0


def test_hard_braking_fails_only_the_acceleration():
    pts, y = [], 0.0
    for d in (2.5, 2.1875, 1.875, 1.5625):                                   # 10, 8.75, 7.5, 6.25 m/s: -5 m/s^2
        y -= d
        pts.append((0.0, y))
    res, t = terms(plan(pts), [])
    assert res[FIELDS["comfort_mask"]] == 1 and res[FIELDS["lon_acceleration_step"]] == 2 and not t["comfort"]
    assert [res[FIELDS[f"{c}_step"]] for c in ops.DRIVING_SCORE_COMFORT[1:]] == [-1] * 4
    assert t["comfort_fail"].tolist() == [True, False, False, False, False]


def test_a_two_step_zig_zag_fails_only_the_yaw_rate():
    res, t = terms(plan([(0.1, -0.2), (0.0, -0.4)]), [])
    assert res[FIELDS["comfort_mask"]] == 4 and res[FIELDS["yaw_rate_step"]] == 2
    assert t["comfort_fail"].tolist() == [False, False, True, False, False] and t["pdms"] == 10 / 12


def test_an_off_road_corner_gives_dac_0():
    road = P.road_plane()
    road[:, 164] = 0
    res, t = terms(plan([(0.0, -1.0)] * 3), [], road=road)
    assert res[FIELDS["off_road_step"]] == 1 and not t["dac"] and t["pdms"] == 0.0


def test_a_nan_step_makes_the_trajectory_invalid():
    traj = straight(4)
    traj[0, 1] = np.nan
    res, ep, _ = run_case(traj, [track(line(4, 0.0, -8.0))], expert=straight(4)[0])
    assert res[0, FIELDS["invalid_step"]] == 2 and np.isnan(ep[0, 0]) and ep[0, 1] == 4.0
    assert res[0, :FIELDS["off_road_step"]].tolist() == [-1] * 8 and res[0, FIELDS["comfort_mask"]] == 0
    from lav_b200.evaluate import driving_terms
    t = driving_terms(views(res, ep))
    assert t["invalid"][0] and t["pdms"][0] == 0.0


def test_an_overlap_present_at_step_0_is_not_new():
    T = 4
    res, t = terms(straight(T), [track(line(T, 0.0, -3.0))])
    assert res[FIELDS["fault_step"]] == -1 and res[FIELDS["exempt_step"]] == -1 and res[FIELDS["ttc_step"]] == -1 and t["nc"]
    absent = track(line(T, 0.0, -3.0), present=[False] + [True] * T)          # the same car unseen at step 0 is new at step 1
    res, t = terms(straight(T), [absent])
    assert res[FIELDS["fault_step"]] == 1 and not t["nc"]


def test_classes_other_than_vehicles_and_pedestrians_are_ignored():
    T = 6
    res, _ = terms(straight(T), [track(line(T, 0.0, -8.0), typ=2), track(line(T, 0.0, -8.0), typ=0, e=(0.3, 0.3))])
    assert (res[FIELDS["fault_step"]], res[FIELDS["fault_row"]], res[FIELDS["fault_class"]]) == (6, 1, 0)


def test_statement_is_per_sample():
    """a batch of samples equals the samples one by one, with the second trajectory its own."""
    T, rs = 5, np.random.RandomState(3)
    cases = []
    for i in range(6):
        traj = np.cumsum(rs.uniform(-1.5, 0.3, (2, T, 2)), 1).astype(np.float32)
        rows = [track(line(T, *rs.uniform(-6, 2, 2), *rs.uniform(-2, 2, 2)), psi=rs.uniform(-3, 3)) for _ in range(i)]
        cases.append((traj, rows))
    actors, offsets = P.pack([c[1] for c in cases], T + 1)
    traj = np.stack([c[0] for c in cases])
    got, ep, _ = driving_score_ref(traj, traj[:, 1], actors, offsets, np.array([EGO] * 6), np.stack([P.road_plane()] * 6))
    for i, (tr, rows) in enumerate(cases):
        r1, e1, _ = run_case(tr, rows, expert=tr[1])
        assert np.array_equal(got[i], r1) and np.array_equal(ep[i], e1, equal_nan=True)


# ---------------------------------------------------------------------------------------------------- host reduction
def buffer(res, ep):
    """a host result buffer of driving_score_views from (B, n, 16) records and (B, n, 2) progress / length."""
    b, n = res.shape[:2]
    buf = torch.zeros(b * n * (16 + 64), dtype=torch.uint8)
    v = ops._views(buf, ops._driving_parts(b, n))
    v["res"].copy_(torch.from_numpy(np.ascontiguousarray(res, np.int32)))
    v["ep"].copy_(torch.from_numpy(np.ascontiguousarray(ep, np.float64)))
    return buf


def test_driving_scores_reduction():
    from lav_b200.evaluate import DrivingScores
    none = [-1] * 9 + [0] + [-1] * 6
    fault = list(none)
    fault[0:3] = [3, 0, 1]
    exempt = list(none)
    exempt[3:6] = [2, 1, 0]
    ttc = list(none)
    ttc[6:8] = [1, 2]
    comfort = list(none)
    comfort[9], comfort[12] = 4, 2                                        # yaw rate from step 2
    bad = list(none)
    bad[15] = 3
    off = list(none)
    off[8] = 5
    res = np.array([[fault, none], [exempt, ttc], [comfort, none], [bad, off]], np.int32)
    ep = np.array([[[5.0, 10.0], [10.0, 10.0]], [[2.0, 4.0], [9.0, 10.0]], [[12.0, 10.0], [-1.0, 10.0]],
                   [[np.nan, 10.0], [10.0, 10.0]]])
    s = DrivingScores()
    s.add(buffer(res[:3], ep[:3]), [0, 1, 0])
    other = DrivingScores()
    other.add(buffer(res[3:], ep[3:]), [1])
    s.extend(other)
    got = s.summary()
    p, e = got["plan"], got["expert"]
    assert got["step_seconds"] == 0.25 and p["samples"] == 4 and p["invalid"] == 1
    # plan: 0 at fault; 1 exempt, EP 1 (4 m expert); 2 comfort fails, EP 1 (clamped); 3 invalid
    assert p["pdms"] == pytest.approx((0 + 1 + 10 / 12 + 0) / 4, abs=1e-15)
    assert p["nc"] == 2 / 3 and p["dac"] == 1.0 and p["ttc"] == 1.0 and p["comfort"] == 2 / 3 and p["ep"] == pytest.approx(2.5 / 3)
    assert p["at_fault_collisions"] == 1 and p["exempt_collisions"] == 1
    assert p["comfort_failure_rate"] == dict(lon_acceleration=0.0, lon_jerk=0.0, yaw_rate=1 / 3, yaw_acceleration=0.0,
                                             lat_acceleration=0.0)
    # expert: 0 all pass; 1 TTC fails with EP 0.9; 2 EP 0 (clamped); 3 off road
    assert e["pdms"] == pytest.approx((1 + (5 * 0 + 5 * 0.9 + 2) / 12 + 7 / 12 + 0) / 4, abs=1e-15)
    assert e["dac"] == 0.75 and e["ttc"] == 0.75 and e["invalid"] == 0
    assert p["per_cmd"]["0"]["samples"] == 2 and p["per_cmd"]["1"]["invalid"] == 1 and p["per_cmd"]["1"]["nc"] == 1.0
    empty = DrivingScores().summary()
    assert empty["plan"]["samples"] == 0 and empty["plan"]["pdms"] is None and empty["plan"]["per_cmd"] == {}


def test_format_and_headline():
    from lav_b200 import evaluate as E
    from lav_b200.evaluate import DrivingScores, format_driving_score
    s = DrivingScores()
    s.add(buffer(np.array([[[-1] * 9 + [0] + [-1] * 6] * 2], np.int32), np.array([[[10.0, 10.0]] * 2])), [2])
    summary = s.summary()
    lines = format_driving_score(summary)
    assert lines[0].startswith("driving score, plan (dt 0.25 s): 1 samples, PDMS 1.0000") and len(lines) == 6
    assert ("PDMS", 1.0) in E.headline(dict(bev_iou=[None] * 3, det=dict(pedestrian=dict(ap=dict(mean=None)), vehicle=dict(ap=dict(mean=None))),
                                            plan=dict(ade=None, fde=None), driving_score=summary))


def test_parse_args_driving_score():
    from lav_b200 import evaluate as E
    from lav_b200 import evaluate_bev as EB
    a = E.parse_args(["--data-dir", "d", "--lidar-weights", "l", "--uniplanner-weights", "u"])
    assert not a.driving_score and a.step_seconds == 0.25
    a = EB.parse_args(["--data-dir", "d", "--bev-weights", "b", "--driving-score", "--step-seconds", "0.1"])
    assert a.driving_score and a.step_seconds == 0.1


# ---------------------------------------------------------------------------------------------------- host table
def direct_table(env, index, T):
    """the table by a direct loop over the keys: per actor of frame index but the ego, per step 0..T, look its id up."""
    get = lambda tag, i, dt=np.float32: np.frombuffer(env.get(f"{tag}_{i:05d}"), dt)
    ids0 = get("id", index, np.int32)
    ego = int(ids0[0])
    e = int(np.nonzero(ids0 == ego)[0][0])
    ox, oy = (float(v) for v in get("loc", index).reshape(-1, 2)[e])
    yaw = float(np.deg2rad(get("ori", index)[e]))
    out = []
    for i in sorted(set(ids0.tolist()) - {ego}):
        row = []
        for t in range(T + 1):
            ids = get("id", index + t, np.int32)
            hit = np.nonzero(ids == i)[0]
            if not len(hit):
                row.append(None)
                continue
            k = int(hit[0])
            lx, ly = (float(v) for v in get("loc", index + t).reshape(-1, 2)[k])
            dx, dy = lx - ox, ly - oy
            psi = float(np.deg2rad(get("ori", index + t)[k])) - yaw
            row.append(dict(x=-(dx * math.sin(yaw) - dy * math.cos(yaw)), y=-(dx * math.cos(yaw) + dy * math.sin(yaw)),
                            cos=math.cos(psi), sin=math.sin(psi), bbox=get("bbox", index + t).reshape(-1, 2)[k].tolist(),
                            typ=int(get("type", index + t, np.uint8)[k])))
        out.append(row)
    return out, get("bbox", index).reshape(-1, 2)[e].tolist()


def test_driving_score_table_equals_a_direct_loop(tmp_path):
    from lav_b200.datasets import driving_score_table, plan_safety_table, stage_plan_safety
    env = P.write_recording(str(tmp_path / "traj"))
    T = 4
    for index in (0, 2, 3):
        got = driving_score_table(env, index, T)
        want, ego_bbox = direct_table(env, index, T)
        assert got["ego_bbox"].tolist() == ego_bbox and len(got["locs"]) == len(want) and got["locs"].shape[1] == T + 1
        for a, row in enumerate(want):
            for t, w in enumerate(row):
                assert bool(got["present"][a, t]) == (w is not None)
                if w is None:
                    assert got["locs"][a, t].tolist() == [0.0, 0.0] and got["typ"][a, t] == 0
                    continue
                assert np.allclose(got["locs"][a, t], [w["x"], w["y"]], rtol=0, atol=1e-9)
                assert abs(got["cos"][a, t] - w["cos"]) < 1e-12 and abs(got["sin"][a, t] - w["sin"]) < 1e-12
                assert got["bbox"][a, t].tolist() == w["bbox"] and got["typ"][a, t] == w["typ"]
        ps = plan_safety_table(env, index, T)                       # steps 1..T are the plan-safety table's
        assert all(np.array_equal(got[k][:, 1:], ps[k]) for k in ("locs", "cos", "sin", "bbox", "typ", "present"))
    st = stage_plan_safety([driving_score_table(env, i, T) for i in (0, 3)], False)
    rec = st["actors"].numpy().view(DTYPE).reshape(-1, T + 1)
    first = driving_score_table(env, 0, T)
    assert st["offsets"].tolist() == [0, 3, 7] and np.array_equal(rec["x"][:3], first["locs"][..., 0])


def test_prepare_builds_the_driving_table_only_when_asked(tmp_path):
    import lav_b200.datasets as D
    from lav_b200.capi import LavbError
    env = P.write_recording(str(tmp_path / "traj"))
    tracks = D._read_tracks(env, 1, 4)
    with pytest.raises(LavbError):
        D._driving_score_of(tracks, True, True)
    assert D._driving_score_of(tracks, False, True) is None
    got = D._driving_score_of(tracks, True, False)
    assert np.array_equal(got["locs"], D.driving_score_table(env, 1, 4)["locs"])
    with pytest.raises(LavbError):
        D.TemporalBatchLoader(None, 4, ordered=False, driving_score=True)
