"""CPU: the numpy statement of ops.plan_safety (the ego boxes, the separating-axis collision test, the road-corner test) and of the
host reduction PlanSafetyScores, checked on hand-built cases with known answers; datasets.plan_safety_table against a direct loop
over the keys of a recording written here."""
import math

import numpy as np
import pytest

from lav_b200.ops import PLAN_SAFETY_ACTOR_DTYPE as DTYPE

GRID = dict(ppm=4.0, cx0=160.0, cy0=320.0, cy1=-40.0)       # ops.det_grid() at the v2 grid: (160 + 4x, 280 + 4y)
EGO = (2.25, 1.0)                                             # half length, half width: exact in binary


# ---------------------------------------------------------------------------------------------------- the numpy statement
def ego_boxes(traj):
    """traj (n, T, 2) fp32 -> x, y, hx, hy (n, T) fp64 and ok (n, T): the ego box centres, unit headings and validity."""
    traj = np.asarray(traj, np.float32)
    n, T = traj.shape[:2]
    x, y = traj[..., 0].astype(np.float64), traj[..., 1].astype(np.float64)
    hx, hy = np.zeros((n, T)), np.zeros((n, T))
    px, py, cx, cy = np.zeros(n), np.zeros(n), np.zeros(n), -np.ones(n)
    with np.errstate(invalid="ignore", divide="ignore"):
        for t in range(T):
            dx, dy = x[:, t] - px, y[:, t] - py
            length = np.sqrt(dx * dx + dy * dy)
            move = ~(length < 0.1)
            cx, cy = np.where(move, dx / length, cx), np.where(move, dy / length, cy)
            hx[:, t], hy[:, t] = cx, cy
            px, py = x[:, t], y[:, t]
    ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(hx) & np.isfinite(hy)
    return x, y, hx, hy, ok


def _reach(e1, e2, hx, hy, nx, ny):
    return e1 * np.abs(hx * nx + hy * ny) + e2 * np.abs(-hy * nx + hx * ny)


def overlap(a, b):
    """separating-axis test of boxes a, b = (x, y, hx, hy, e1, e2) (broadcasting arrays); touching boxes are separated."""
    dx, dy = b[0] - a[0], b[1] - a[1]
    sep = np.zeros(np.broadcast(dx, b[2]).shape, bool)
    for nx, ny in ((a[2], a[3]), (-a[3], a[2]), (b[2], b[3]), (-b[3], b[2])):
        sep |= np.abs(dx * nx + dy * ny) >= _reach(a[4], a[5], a[2], a[3], nx, ny) + _reach(b[4], b[5], b[2], b[3], nx, ny)
    return ~sep


def corners(x, y, hx, hy, e1, e2):
    """the four corners (4, ...) of boxes, in the kernel's order and roundings."""
    ax, ay, bx, by = e1 * hx, e1 * hy, e2 * -hy, e2 * hx
    out = []
    for k in range(4):
        ux, uy = (x - ax, y - ay) if k & 2 else (x + ax, y + ay)
        out.append((ux - bx, uy - by) if k & 1 else (ux + bx, uy + by))
    return np.array([c[0] for c in out]), np.array([c[1] for c in out])


def plan_safety_ref(traj, actors, offsets, ego_ext, road, grid=GRID):
    """every output of ops.plan_safety: traj (B, n, T, 2) fp32; actors = PLAN_SAFETY_ACTOR_DTYPE records (rows x T, flat);
    offsets (B+1,) actor rows; ego_ext (B, 2) fp64; road (B, H, W) uint8 = plane 0 of the bev.  -> (B, n, 8) int32."""
    traj = np.asarray(traj, np.float32)
    B, n, T, _ = traj.shape
    actors = np.asarray(actors, DTYPE).reshape(-1, T)
    H, W = road.shape[1:]
    ppm, cx0, cy0, cy1 = (float(np.float32(grid[k])) for k in ("ppm", "cx0", "cy0", "cy1"))
    out = np.full((B, n, 8), -1, np.int32)
    for b in range(B):
        e1, e2 = float(ego_ext[b][0]), float(ego_ext[b][1])
        x, y, hx, hy, ok = ego_boxes(traj[b])
        cx, cy = corners(x, y, hx, hy, e1, e2)                                  # (4, n, T)
        col, row = np.floor(cx * ppm + cx0), np.floor((cy * ppm + cy0) + cy1)
        with np.errstate(invalid="ignore"):
            in_map = (col >= 0) & (col < W) & (row >= 0) & (row < H)
        pix = road[b][np.where(in_map, row, 0).astype(np.int64), np.where(in_map, col, 0).astype(np.int64)]
        off_road = (in_map & (pix == 0)).any(0) & ok
        off_map = (~in_map).any(0) & ok
        out[b, :, 4] = [t + 1 if t < T else -1 for t in np.where(off_road.any(1), off_road.argmax(1), T)]
        out[b, :, 5], out[b, :, 6] = off_map.sum(1), (~ok).sum(1)
        a = actors[offsets[b]:offsets[b + 1]]                                   # (A, T)
        live = (a["present"] != 0) & ((a["typ"] == 0) | (a["typ"] == 1))
        other = (a["x"], a["y"], a["sin"], -a["cos"], a["e1"], a["e2"])
        for j in range(n):
            ego = (x[j], y[j], hx[j], hy[j], e1, e2)
            with np.errstate(invalid="ignore"):
                hit = overlap(ego, other) & live & ok[j]                        # (A, T)
            for cls, col_s in ((1, 0), (0, 2)):
                h = hit & (a["typ"] == cls)
                if h.any():
                    t = int(np.nonzero(h.any(0))[0][0])
                    out[b, j, col_s], out[b, j, col_s + 1] = t + 1, int(np.nonzero(h[:, t])[0][0])
            v, p = out[b, j, 0], out[b, j, 2]
            out[b, j, 7] = p if v < 0 else v if p < 0 else min(v, p)
    return out


# ---------------------------------------------------------------------------------------------------- hand-built cases
def actor(T, steps, x, y, psi=0.0, e=(1.0, 1.0), typ=1):
    """one actor row (T,) present at ``steps`` (1..T) at (x, y) with relative yaw psi."""
    r = np.zeros(T, DTYPE)
    for t in steps:
        r[t - 1] = (x, y, math.cos(psi), math.sin(psi), e[0], e[1], typ, 1)
    return r


def pack(samples, T):
    """a list of per-sample lists of actor rows -> (flat records, offsets)."""
    rows = [np.stack(s) if s else np.zeros((0, T), DTYPE) for s in samples]
    offsets = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
    return np.concatenate(rows + [np.zeros((0, T), DTYPE)]).reshape(-1), offsets


def straight(T, step=1.0, n=1):
    """n copies of a plan driving straight ahead (negative y), ``step`` metres per step."""
    return np.array([[[0.0, -step * (t + 1)] for t in range(T)]] * n, np.float32)


def road_plane(fill=1):
    return np.full((320, 320), fill, np.uint8)


def case_table():
    """(name, traj (n, T, 2), actor rows, road (320, 320), expected (n, 8)) of the hand-built cases; ego extents EGO."""
    T, cases = 4, []
    below = float(np.nextafter(np.float32(2.0), np.float32(0)))
    # two boxes sharing an edge at x = 1 (the ego spans x in [-1, 1] at step 1), then one fp32 ulp closer
    cases.append(("shared edge", straight(T), [actor(T, [1], 2.0, -1.0)], road_plane(), [[-1, -1, -1, -1, -1, 0, 0, -1]]))
    cases.append(("one ulp closer", straight(T), [actor(T, [1], below, -1.0)], road_plane(), [[1, 0, -1, -1, -1, 0, 0, 1]]))
    # a 45-degree square (corner reach sqrt(1/2)) whose corner enters the ego's right edge by 0.01 m, and one 0.01 m short
    reach = math.sqrt(0.5)
    cases.append(("45 deg corner in", straight(T), [actor(T, [2], 1.0 + reach - 0.01, -2.0, math.pi / 4, (0.5, 0.5))], road_plane(),
                  [[2, 0, -1, -1, -1, 0, 0, 2]]))
    cases.append(("45 deg corner out", straight(T), [actor(T, [2], 1.0 + reach + 0.01, -2.0, math.pi / 4, (0.5, 0.5))],
                  road_plane(), [[-1, -1, -1, -1, -1, 0, 0, -1]]))
    # a stationary step keeps the heading (0, -1): a box beside it collides only if the ego turned towards (1, 0)
    still = np.array([[[0.0, -1.0], [0.05, -1.0], [0.05, -1.0], [0.05, -1.0]]], np.float32)
    cases.append(("stationary", still, [actor(T, [2, 3, 4], 1.65, -1.0, 0.0, (0.5, 0.5))], road_plane(),
                  [[-1, -1, -1, -1, -1, 0, 0, -1]]))
    # corners exactly on pixel edges: at step 1 the corners are at columns 156 / 164 and rows 267 / 285 exactly
    for name, zero, hit in (("edge col 163", (slice(None), 163), -1), ("edge col 164", (slice(None), 164), 1),
                            ("edge row 284", (284, slice(None)), -1), ("edge row 285", (285, slice(None)), 1),
                            ("edge col 155", (slice(None), 155), -1), ("edge col 156", (slice(None), 156), 1)):
        road = road_plane()
        road[zero] = 0
        plan = np.array([[[0.0, -1.0], [0.0, -1.0], [0.0, -1.0], [0.0, -1.0]]], np.float32)
        cases.append((name, plan, [], road, [[-1, -1, -1, -1, hit, 0, 0, -1]]))
    # a plan leaving the map: steps 3 and 4 lie past row 0
    cases.append(("off map", straight(T, 25.0), [], road_plane(), [[-1, -1, -1, -1, -1, 2, 0, -1]]))
    # half off the map (corners past row 319) with an in-map corner on a 0 pixel: off-road and off-map
    back = np.array([[[0.0, 9.0], [0.0, 9.0], [0.0, 9.0], [0.0, 9.0]]], np.float32)
    road = road_plane()
    road[307] = 0
    cases.append(("half off map", back, [], road, [[-1, -1, -1, -1, 1, 4, 0, -1]]))
    # a NaN point: its step and the next (whose heading needs it) are invalid, never a collision; an actor at both
    nan = straight(T)
    nan[0, 1] = np.nan
    cases.append(("nan point", nan, [actor(T, [2, 3], 0.0, -2.5)], road_plane(0), [[-1, -1, -1, -1, 1, 0, 2, -1]]))
    # an actor absent at a step: overlapping geometry at step 1 without presence, present from step 3
    absent = actor(T, [3], 0.0, -3.0)
    absent[0] = (0.0, -1.0, 1.0, 0.0, 1.0, 1.0, 1, 0)
    cases.append(("absent", straight(T), [absent], road_plane(), [[3, 0, -1, -1, -1, 0, 0, 3]]))
    # pedestrians apart from vehicles, class 2 ignored, the lowest row of the first step
    rows = [actor(T, [1], 0.0, -1.0, typ=2), actor(T, [3], 0.0, -3.0), actor(T, [2], 0.5, -2.0, typ=0, e=(0.3, 0.3)),
            actor(T, [3], 0.0, -3.5), actor(T, [2], -0.5, -2.0, typ=0, e=(0.3, 0.3))]
    cases.append(("classes", straight(T), rows, road_plane(), [[3, 1, 2, 2, -1, 0, 0, 2]]))
    # two trajectories: the second shifted 6 m sideways hits a car the first passes
    two = np.concatenate([straight(T), straight(T) + np.float32([6.0, 0.0])])
    cases.append(("two trajectories", two, [actor(T, [4], 6.0, -4.0)], road_plane(), [[-1, -1, -1, -1, -1, 0, 0, -1],
                                                                                   [4, 0, -1, -1, -1, 0, 0, 4]]))
    return cases


def run_case(traj, rows, road, fn=plan_safety_ref):
    T = traj.shape[1]
    actors, offsets = pack([rows], T)
    return fn(traj[None], actors, offsets, np.array([EGO]), road[None])[0]


@pytest.mark.parametrize("case", case_table(), ids=lambda c: c[0])
def test_statement_known_answers(case):
    name, traj, rows, road, want = case
    assert run_case(traj, rows, road).tolist() == want, name


def test_heading_carries_over_a_stationary_step():
    x, y, hx, hy, ok = ego_boxes(np.array([[[0.0, -1.0], [0.05, -1.0], [0.05, -1.0], [3.0, -1.0]]], np.float32))
    assert hx[0].tolist() == [0.0, 0.0, 0.0, 1.0] and hy[0].tolist() == [-1.0, -1.0, -1.0, 0.0] and ok.all()
    x, y, hx, hy, ok = ego_boxes(np.zeros((1, 3, 2), np.float32))             # a standing ego faces forward
    assert (hx == 0).all() and (hy == -1).all()


def test_actor_heading_convention():
    """an actor at relative yaw psi heads along (sin psi, -cos psi): a long thin car crossing the path collides, the same car
    along the path beside it does not."""
    T = 2
    car = lambda psi: actor(T, [1], 3.2, -1.0, psi, (2.4, 0.5))
    assert run_case(straight(T), [car(0.0)], road_plane())[0, 0] == -1
    assert run_case(straight(T), [car(math.pi / 2)], road_plane())[0, 0] == 1
    assert run_case(straight(T), [car(-math.pi / 2)], road_plane())[0, 0] == 1


def test_statement_is_per_sample():
    """a batch of the cases equals the cases one by one."""
    cases = [c for c in case_table() if c[1].shape[0] == 1]
    traj = np.stack([c[1] for c in cases])
    actors, offsets = pack([c[2] for c in cases], 4)
    got = plan_safety_ref(traj, actors, offsets, np.array([EGO] * len(cases)), np.stack([c[3] for c in cases]))
    assert got[:, 0].tolist() == [c[4][0] for c in cases]


# ---------------------------------------------------------------------------------------------------- host reduction
def test_plan_safety_scores_reduction():
    from lav_b200.evaluate import PlanSafetyScores
    s = PlanSafetyScores()
    none = [-1, -1, -1, -1, -1, 0, 0, -1]
    r1 = np.array([[[2, 0, -1, -1, -1, 1, 0, 2], none], [[-1, -1, 1, 4, 3, 0, 2, 1], none]], np.int32)
    r2 = np.array([[none, [4, 1, 3, 0, 2, 0, 0, 3]]], np.int32)
    s.add(r1, [0, 1])
    s.add(r2, [0])
    got = s.summary(4)
    p, e = got["plan"], got["expert"]
    assert p["samples"] == 3 and p["collision_rate"] == 2 / 3 and p["vehicle_collision_rate"] == 1 / 3
    assert p["pedestrian_collision_rate"] == 1 / 3 and p["off_road_rate"] == 1 / 3
    assert p["collision_rate_by_step"] == [1 / 3, 2 / 3, 2 / 3, 2 / 3]
    assert p["off_map_steps"] == 1 and p["invalid_steps"] == 2
    assert e["collision_rate"] == 1 / 3 and e["collision_rate_by_step"] == [0.0, 0.0, 1 / 3, 1 / 3] and e["off_road_rate"] == 1 / 3
    assert p["per_cmd"]["0"]["samples"] == 2 and p["per_cmd"]["0"]["collision_rate"] == 0.5
    assert p["per_cmd"]["1"]["pedestrian_collision_rate"] == 1.0 and set(p["per_cmd"]) == {"0", "1"}
    empty = PlanSafetyScores().summary(3)
    assert empty["plan"]["samples"] == 0 and empty["plan"]["collision_rate"] is None
    assert empty["expert"]["collision_rate_by_step"] == [None] * 3 and empty["plan"]["per_cmd"] == {}


# ---------------------------------------------------------------------------------------------------- host table
def write_recording(path, n_frames=8):
    """a recording of one trajectory: the ego (id 7) turning, a car that leaves after frame 4, a pedestrian, a class-2 actor and
    an actor that appears at frame 3; ids out of order in the frames."""
    from lav_b200.data_paint import DirEnv
    env = DirEnv(path)
    env.put("len", str(n_frames).encode())
    env.put("town", b"Town01")
    for f in range(n_frames):
        ids, locs, oris, boxes, typs = [7], [[10.0 + f, 5.0 + 0.3 * f]], [30.0 + 4 * f], [[2.4, 1.1]], [1]
        for i, (dx, dy, o, box, typ, first, last) in {40: (8.0, 1.0, -70.0, (2.0, 0.9), 1, 0, 4), 12: (-3.0, 6.0, 200.0, (0.3, 0.3), 0, 0, 99),
                                                     25: (2.0, -9.0, 5.0, (1.0, 1.0), 2, 0, 99), 3: (1.0, 1.0, 0.0, (2.0, 1.0), 1, 3, 99)}.items():
            if first <= f <= last:
                ids.append(i)
                locs.append([10.0 + dx + 0.5 * f, 5.0 + dy - 0.2 * f])
                oris.append(o + f)
                boxes.append(box)
                typs.append(typ)
        env.put(f"id_{f:05d}", np.array(ids, np.int32).tobytes())
        env.put(f"loc_{f:05d}", np.array(locs, np.float32).tobytes())
        env.put(f"ori_{f:05d}", np.array(oris, np.float32).tobytes())
        env.put(f"bbox_{f:05d}", np.array(boxes, np.float32).tobytes())
        env.put(f"type_{f:05d}", np.array(typs, np.uint8).tobytes())
    return env


def direct_table(env, index, T):
    """the table by a direct loop over the keys: per actor of frame index but the ego, per step, look its id up."""
    get = lambda tag, i, dt=np.float32: np.frombuffer(env.get(f"{tag}_{i:05d}"), dt)
    ids0 = get("id", index, np.int32)
    ego = int(ids0[0])
    e = int(np.nonzero(ids0 == ego)[0][0])
    ox, oy = (float(v) for v in get("loc", index).reshape(-1, 2)[e])
    yaw = float(np.deg2rad(get("ori", index)[e]))
    out = []
    for i in sorted(set(ids0.tolist()) - {ego}):
        row = []
        for t in range(1, T + 1):
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
        out.append((i, row))
    return out, get("bbox", index).reshape(-1, 2)[e].tolist()


def test_plan_safety_table_equals_a_direct_loop(tmp_path):
    from lav_b200.datasets import actor_tracks, plan_safety_table, stage_plan_safety
    env = write_recording(str(tmp_path / "traj"))
    T = 4
    for index in (0, 2, 3):
        got = plan_safety_table(env, index, T)
        want, ego_bbox = direct_table(env, index, T)
        assert got["ego_bbox"].tolist() == ego_bbox and len(got["locs"]) == len(want)       # the ego is not an actor
        for a, (_, row) in enumerate(want):
            for t, w in enumerate(row):
                assert bool(got["present"][a, t]) == (w is not None)
                if w is None:
                    assert got["locs"][a, t].tolist() == [0.0, 0.0] and got["typ"][a, t] == 0
                    continue
                assert np.allclose(got["locs"][a, t], [w["x"], w["y"]], rtol=0, atol=1e-9)
                assert abs(got["cos"][a, t] - w["cos"]) < 1e-12 and abs(got["sin"][a, t] - w["sin"]) < 1e-12
                assert got["bbox"][a, t].tolist() == w["bbox"] and got["typ"][a, t] == w["typ"]
        # the positions are actor_tracks' ego frame, negated as the labels are (actors seen in every frame)
        ego_locs, locs, oris, bbox, typs = actor_tracks(env, index, T, 1e9, 1e9)
        full = got["present"].all(1)
        others = [r for r in range(len(locs)) if not np.allclose(locs[r], ego_locs, rtol=0, atol=1e-9)]
        assert len(others) == len(locs) - 1 and np.allclose(-locs[others][:, 1:], got["locs"][full], rtol=0, atol=1e-9)
    st = stage_plan_safety([plan_safety_table(env, i, T) for i in (0, 3)], False)
    rec = st["actors"].numpy().view(DTYPE).reshape(-1, T)
    assert st["offsets"].tolist() == [0, 3, 7] and st["ego_ext"].dtype.is_floating_point and st["ego_ext"].shape == (2, 2)
    first = plan_safety_table(env, 0, T)
    assert np.array_equal(rec["x"][:3], first["locs"][..., 0]) and np.array_equal(rec["sin"][:3], first["sin"])
    assert np.array_equal(rec["present"][:3] != 0, first["present"]) and np.array_equal(rec["e2"][:3], first["bbox"][..., 1])


def test_prepare_builds_the_table_only_when_asked(tmp_path, monkeypatch):
    """actor_tracks' outputs and the prepared labels do not change; the table appears only with plan_safety and refuses
    augmented samples."""
    import lav_b200.datasets as D
    env = write_recording(str(tmp_path / "traj"))
    tracks = D._read_tracks(env, 1, 4)
    assert all(np.array_equal(a, b) for a, b in zip(D._label_tracks(tracks, 15, 25), D.actor_tracks(env, 1, 4, 15, 25)))
    from lav_b200.capi import LavbError
    with pytest.raises(LavbError):
        D._plan_safety_of(tracks, True, True)
    assert D._plan_safety_of(tracks, False, True) is None
