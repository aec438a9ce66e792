"""CPU: the fp64 statement of lavb_det_box_eval (box corners, Sutherland-Hodgman clipping, shoelace areas, the IoU and 2 m
matches and the per-match errors) on cases with known answers and against a fine raster estimate, and lav_b200.evaluate's
DetBoxScores reduction and its merge."""
import math

import numpy as np
import torch

from tests import test_evaluate_cpu as E

THRESHOLDS = (0.3, 0.5, 0.7)
TWO_PI = 6.283185307179586
MAX_POLY = 16
CORNERS = ((-1.0, -1.0), (-1.0, 1.0), (1.0, 1.0), (1.0, -1.0))


# ---------------------------------------------------------------------------------------------------- the fp64 statement
# Python floats are IEEE doubles and Python never contracts a multiply-add, so each line is the kernel's operation order.
def poly_area(x, y):
    s = 0.0
    for i in range(len(x)):
        j = 0 if i + 1 == len(x) else i + 1
        s = s + (x[i] * y[j] - x[j] * y[i])
    return abs(s) * 0.5


def make_box(cx, cy, hw, hh, c, s):
    """the corners, area and bounding box of a box centred at (cx, cy), half extents (hw, hh), heading (c, s); ok = not
    degenerate."""
    cx, cy, hw, hh, c, s = (float(v) for v in (cx, cy, hw, hh, c, s))
    ux, uy, vx, vy = -(s * hw), c * hw, -(c * hh), -(s * hh)
    x = [cx + (a * ux + b * vx) for a, b in CORNERS]
    y = [cy + (a * uy + b * vy) for a, b in CORNERS]
    ok = all(map(math.isfinite, (hw, hh, c, s, cx, cy))) and hw > 0 and hh > 0
    area = poly_area(x, y) if ok else 0.0
    return dict(x=x, y=y, area=area, ok=ok and area > 0)


def clip(P, Q):
    """P's corners clipped by each edge of Q in turn -> the polygon's (x, y) lists."""
    sx, sy = list(P["x"]), list(P["y"])
    for e in range(4):
        if not sx:
            break
        x0, y0 = Q["x"][e], Q["y"][e]
        ex, ey = Q["x"][(e + 1) & 3] - x0, Q["y"][(e + 1) & 3] - y0
        side = lambda px, py: ex * (py - y0) - ey * (px - x0)
        dx, dy = [], []
        px, py = sx[-1], sy[-1]
        sp = side(px, py)
        for qx, qy in zip(sx, sy):
            sq = side(qx, qy)
            if (sq <= 0.0) != (sp <= 0.0) and len(dx) < MAX_POLY:
                t = sp / (sp - sq)
                dx.append(px + t * (qx - px))
                dy.append(py + t * (qy - py))
            if sq <= 0.0 and len(dx) < MAX_POLY:
                dx.append(qx)
                dy.append(qy)
            px, py, sp = qx, qy, sq
        sx, sy = dx, dy
    return sx, sy


def box_iou(P, Q):
    if not (P["ok"] and Q["ok"]):
        return 0.0
    if max(P["x"]) < min(Q["x"]) or max(Q["x"]) < min(P["x"]) or max(P["y"]) < min(Q["y"]) or max(Q["y"]) < min(P["y"]):
        return 0.0
    x, y = clip(P, Q)
    inter = poly_area(x, y) if len(x) >= 3 else 0.0
    uni = (P["area"] + Q["area"]) - inter
    return inter / uni if uni > 0.0 else 0.0


def scale_error(hw, hh, gw, gh):
    hw, hh, gw, gh = (float(v) for v in (hw, hh, gw, gh))
    ext = all(math.isfinite(v) and v > 0 for v in (hw, hh, gw, gh))
    i2 = min(hw, gw) * min(hh, gh)
    return 1.0 - (i2 / ((hw * hh + gw * gh) - i2) if ext else 0.0)


def heading_error(c, s, ori):
    r = math.fmod(abs(math.atan2(float(s), float(c)) - float(ori)), TWO_PI)
    return r if r <= TWO_PI - r else TWO_PI - r


def det_box_ref(packed, actors, offsets, w=320, min_score=0.2, grid=E.GRID, near=1e-12):
    """every output of ops.det_box_eval, as det_box_views names them, and ``near``: the count of (survivor, candidate actor)
    IoUs within ``near`` of a threshold, where the kernel's fp64 cos / sin may decide a match differently."""
    packed = np.asarray(packed, np.float32)
    B, _, cols = packed.shape
    n_det = cols // 2
    ppm = float(grid["ppm"])
    keep, x, y, loc = E.survivors(packed, w, min_score, grid)
    actors = np.asarray(actors, np.float32).reshape(-1, 6)
    cx, cy = E.centres(actors, grid)
    d = E.window_dist(cx, cy, grid)
    typ = actors[:, 5]
    gcls = np.where(typ == 0, 0, np.where(typ == 1, 1, -1))
    gkeep = (gcls >= 0) & (d > 2) & (d < 30 * ppm)
    flags = np.where(keep, 16, 0).astype(np.int32)
    actor = np.full((B, cols, 4), -1, np.int32)
    err = np.full((B, cols, 5), np.nan)
    ngt = np.zeros((B, 2), np.int32)
    thr2 = (2.0 * ppm) * (2.0 * ppm)
    n_near = 0
    for b in range(B):
        a0, a1 = int(offsets[b]), int(offsets[b + 1])
        gt_box = {r: make_box(cx[r], cy[r], float(actors[r, 3]) * ppm, float(actors[r, 4]) * ppm, math.cos(float(actors[r, 2])),
                              math.sin(float(actors[r, 2]))) for r in range(a0, a1)}
        det_box = lambda j: make_box(float(x[b, j]), float(y[b, j]), *packed[b, 2:6, j])
        for c in range(2):
            g = [r for r in range(a0, a1) if gkeep[r] and gcls[r] == c]
            ngt[b, c] = len(g)
            cand = [j for j in range(c * n_det, (c + 1) * n_det) if keep[b, j]]
            cand.sort(key=lambda j: (-packed[b, 0, j], loc[b, j], j))
            used = [set() for _ in range(4)]
            for j in cand:
                P = det_box(j)
                ious = {r: box_iou(P, gt_box[r]) for r in g}
                n_near += sum(abs(v - t) <= near for v in ious.values() for t in THRESHOLDS)
                for k, t in enumerate(THRESHOLDS):
                    best = None
                    for r in g:                                    # ascending rows: a strict > keeps the lower row on a tie
                        if r not in used[k] and ious[r] >= t and (best is None or ious[r] > best[0]):
                            best = (ious[r], r)
                    if best is not None:
                        used[k].add(best[1])
                        actor[b, j, k] = best[1] - a0
                        flags[b, j] |= 1 << k
                best = None
                for r in g:                                        # eval_batch's 2 m search
                    if r in used[3]:
                        continue
                    dx, dy = float(x[b, j]) - float(cx[r]), float(y[b, j]) - float(cy[r])
                    d2 = dx * dx + dy * dy
                    if d2 <= thr2 and (best is None or d2 < best[0]):
                        best = (d2, r)
                if best is not None:
                    d2, r = best
                    used[3].add(r)
                    actor[b, j, 3] = r - a0
                    flags[b, j] |= 8
                    err[b, j] = (ious[r], math.sqrt(d2) / ppm,
                                 scale_error(packed[b, 2, j], packed[b, 3, j], float(actors[r, 3]) * ppm, float(actors[r, 4]) * ppm),
                                 heading_error(packed[b, 4, j], packed[b, 5, j], actors[r, 2]), float(d[r]) / ppm)
    return dict(score=packed[:, 0].copy(), flags=flags, actor=actor, err=err, ngt=ngt, near=n_near)


def reduce_ref(batches):
    """the host reduction of a recording [(score (B, cols), flags, err (B, cols, 5), ngt (B, 2))] per class, written out."""
    out = {}
    for c, name in enumerate(("pedestrian", "vehicle")):
        s, f, e, n_gt = [], [], [], 0
        for score, flags, err, ngt in batches:
            n = score.shape[1] // 2
            for b in range(score.shape[0]):
                for j in range(c * n, (c + 1) * n):
                    if flags[b, j] & 16:
                        s.append(score[b, j])
                        f.append(int(flags[b, j]))
                        e.append(err[b, j])
            n_gt += int(ngt[:, c].sum())
        e = np.array(e).reshape(-1, 5)
        f = np.array(f, np.int64)
        m = e[(f & 8) != 0]

        def errors(m):
            mean = lambda a: float(np.mean(a)) if len(a) else None
            h = [v for v in m[:, 3] if math.isfinite(v)]
            return dict(matched=len(m), mean_iou=mean(m[:, 0]), translation_m=mean(m[:, 1]), scale=mean(m[:, 2]), heading_rad=mean(h),
                        flipped_rate=mean([v > math.pi / 2 for v in h]))
        d = dict(n_gt=n_gt, n_det=len(s), ap_iou={f"{t:g}": E.average_precision(s, (f >> k) & 1, n_gt) for k, t in enumerate(THRESHOLDS)},
                 recall=len(m) / n_gt if n_gt else None, **errors(m))
        d["by_range"] = {f"{lo}-{hi}": errors(m[(m[:, 4] >= lo) & (m[:, 4] < hi)]) for lo, hi in ((0, 10), (10, 20), (20, 30))}
        out[name] = d
    return out


def close_dicts(a, b, tol=1e-12):
    """equal nests, floats within tol."""
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(close_dicts(a[k], b[k], tol) for k in a)
    if isinstance(a, float) and isinstance(b, float):
        return abs(a - b) <= tol * max(1.0, abs(b))
    return a == b


# ---------------------------------------------------------------------------------------------------- known answers
def test_identical_disjoint_touching_and_nested_boxes():
    A = make_box(100, 50, 3, 2, math.cos(0.4), math.sin(0.4))
    assert box_iou(A, A) == 1.0
    assert box_iou(A, make_box(140, 50, 3, 2, 1, 0)) == 0.0                           # apart
    sq = lambda x, y, h: make_box(x, y, h, h, 1.0, 0.0)
    assert box_iou(sq(0, 0, 1), sq(2, 0, 1)) == 0.0                                  # sharing an edge
    assert box_iou(sq(0, 0, 1), sq(2, 2, 1)) == 0.0                                  # sharing a corner
    assert box_iou(sq(0, 0, 1), sq(1, 0, 1)) == 2 / 6                                # half overlap
    inner, outer = make_box(10, 10, 1, 1, 1, 0), make_box(10.5, 10, 3, 2, 1, 0)
    assert abs(box_iou(inner, outer) - 4 / 24) < 1e-15 and abs(box_iou(outer, inner) - 4 / 24) < 1e-15
    t = 0.3                                                                           # also nested when both are turned
    assert abs(box_iou(make_box(0, 0, 1, 0.5, math.cos(t), math.sin(t)), make_box(0, 0, 3, 2, math.cos(t), math.sin(t))) - 2 / 24) < 1e-14


def test_square_over_itself_turned_45_degrees_is_the_octagon():
    a = 2.0                                                                           # side; the octagon is 2 a^2 (sqrt 2 - 1)
    octagon = 2 * a * a * (math.sqrt(2) - 1)
    got = box_iou(make_box(5, 7, 1, 1, 1, 0), make_box(5, 7, 1, 1, math.cos(math.pi / 4), math.sin(math.pi / 4)))
    assert abs(got - octagon / (2 * a * a - octagon)) < 1e-14


def test_box_turned_by_pi_has_iou_one_and_heading_error_pi():
    ori = 0.7
    c, s = math.cos(ori + math.pi), math.sin(ori + math.pi)
    P, Q = make_box(60, 80, 4, 2, c, s), make_box(60, 80, 4, 2, math.cos(ori), math.sin(ori))
    assert abs(box_iou(P, Q) - 1) < 1e-12
    assert abs(heading_error(c, s, ori) - math.pi) < 1e-12
    assert heading_error(math.cos(ori), math.sin(ori), ori) < 1e-15
    assert abs(heading_error(1, 0, 2 * math.pi + 0.25) - 0.25) < 1e-12 and abs(heading_error(1, 0, -3.0) - 3.0) < 1e-12
    assert math.isnan(heading_error(float("nan"), 0, 0.1))
    assert scale_error(4, 2, 4, 2) == 0.0 and abs(scale_error(2, 2, 4, 2) - 0.5) < 1e-15 and scale_error(0, 2, 4, 2) == 1.0


def test_degenerate_boxes_give_zero():
    Q = make_box(10, 10, 2, 2, 1, 0)
    for bad in (make_box(10, 10, 0, 2, 1, 0), make_box(10, 10, float("nan"), 2, 1, 0), make_box(10, 10, 2, float("inf"), 1, 0),
                make_box(10, 10, 2, 2, float("nan"), 0), make_box(10, 10, 2, 2, 0, float("inf")), make_box(10, 10, 2, 2, 0.0, 0.0),
                make_box(10, 10, -1, 2, 1, 0)):
        assert not bad["ok"] and box_iou(bad, Q) == 0.0 and box_iou(Q, bad) == 0.0
    assert box_iou(make_box(10, 10, 2, 2, 1e-3, 0), Q) > 0                            # a short heading vector only scales the box


def raster_iou(P, Q, n=600):
    """the IoU of two boxes estimated on an n x n grid of points over their joint bounding box."""
    xs, ys = P["x"] + Q["x"], P["y"] + Q["y"]
    gx, gy = np.meshgrid(np.linspace(min(xs), max(xs), n), np.linspace(min(ys), max(ys), n))

    def inside(B):
        m = np.ones_like(gx, bool)
        for e in range(4):
            x0, y0 = B["x"][e], B["y"][e]
            ex, ey = B["x"][(e + 1) & 3] - x0, B["y"][(e + 1) & 3] - y0
            m &= ex * (gy - y0) - ey * (gx - x0) <= 0
        return m
    a, b = inside(P), inside(Q)
    return (a & b).sum() / max((a | b).sum(), 1)


def test_random_pairs_against_a_raster_estimate():
    rs = np.random.RandomState(0)
    worst, overlapping = 0.0, 0
    for _ in range(60):
        P = make_box(*rs.uniform(0, 6, 2), *rs.uniform(0.5, 4, 2), *(lambda t: (math.cos(t), math.sin(t)))(rs.uniform(-4, 4)))
        Q = make_box(*rs.uniform(0, 6, 2), *rs.uniform(0.5, 4, 2), *(lambda t: (math.cos(t), math.sin(t)))(rs.uniform(-4, 4)))
        got, want = box_iou(P, Q), raster_iou(P, Q)
        assert abs(box_iou(Q, P) - got) < 1e-12                                       # either box clipped by the other
        worst = max(worst, abs(got - want))
        overlapping += got > 0.1
    assert worst < 0.01 and overlapping > 20, (worst, overlapping)


def test_statement_matches_on_a_hand_built_sample():
    """one vehicle seen exactly, one seen turned around and shifted one pixel, one missed; a pedestrian decoy."""
    acts = [E.actor(100, 200), E.actor(120, 200), E.actor(140, 200), E.actor(100, 230, typ=0)]
    for a in acts:
        a[2], a[3], a[4] = 0.5, 2.0, 1.0
    c, s = math.cos(0.5), math.sin(0.5)
    pk = E.packed_of([(1, 0.9, 100, 200, 8, 4), (1, 0.8, 121, 200, 8, 4), (0, 0.5, 130, 240, 1, 1)])
    pk[0, 4:6, 15] = np.float32(c), np.float32(s)
    pk[0, 4:6, 16] = np.float32(-c), np.float32(-s)
    pk[0, 4:6, 0] = 1, 0
    r = det_box_ref(pk, acts, [0, 4])
    assert r["ngt"].tolist() == [[1, 3]] and r["near"] == 0
    assert r["flags"][0, 15] == 16 | 8 | 7 and r["actor"][0, 15].tolist() == [0, 0, 0, 0]
    e = r["err"][0, 15]
    assert abs(e[0] - 1) < 1e-6 and e[1] == 0 and e[2] == 0 and e[3] < 1e-6 and abs(e[4] - math.hypot(60, 80) / 4) < 1e-12
    assert r["flags"][0, 16] & 8 and r["actor"][0, 16, 3] == 1
    e = r["err"][0, 16]
    assert abs(e[1] - 0.25) < 1e-15 and e[2] == 0 and abs(e[3] - math.pi) < 1e-6 and 0.5 < e[0] < 1
    assert r["flags"][0, 0] == 16 and np.isnan(r["err"][0, 0]).all()                  # the decoy: a false positive
    assert r["flags"][0, 1] == 0                                                       # padding does not survive


# ---------------------------------------------------------------------------------------------------- the host reduction
def random_batches(n, seed):
    rs = np.random.RandomState(seed)
    out = []
    for _ in range(n):
        B, cols = rs.randint(1, 5), 30
        flags = ((rs.rand(B, cols) < 0.7) * 16 + rs.randint(0, 16, (B, cols))).astype(np.int32)
        err = np.stack([rs.rand(B, cols), rs.rand(B, cols) * 2, rs.rand(B, cols), rs.rand(B, cols) * math.pi, rs.rand(B, cols) * 30], -1)
        err[rs.rand(B, cols) < 0.1, 3] = np.nan
        out.append((np.round(rs.rand(B, cols), 1).astype(np.float32), flags, err, rs.randint(0, 6, (B, 2)).astype(np.int32)))
    return out


def accumulate(batches):
    from lav_b200.evaluate import DetBoxScores
    acc = DetBoxScores()
    for score, flags, err, ngt in batches:
        B = len(score)
        acc.add(dict(score=torch.from_numpy(score), flags=torch.from_numpy(flags), err=torch.from_numpy(err),
                     actor=torch.zeros((B, 30, 4), dtype=torch.int32), ngt=torch.from_numpy(ngt)))
    return acc


def test_det_box_scores_reduce_as_the_statement_and_merge_in_order():
    import pickle
    batches = random_batches(9, 0)
    one = accumulate(batches).summary()
    assert close_dicts(one, reduce_ref(batches))
    v = one["vehicle"]
    assert v["matched"] > 0 and sum(b["matched"] for b in v["by_range"].values()) == v["matched"]
    for cut in (0, 4, 9):
        a, b = accumulate(batches[:cut]), pickle.loads(pickle.dumps(accumulate(batches[cut:])))
        a.extend(b)
        assert a.summary() == one
    empty = accumulate([]).summary()["pedestrian"]
    assert empty["recall"] is None and empty["mean_iou"] is None and empty["ap_iou"]["0.5"] is None


def test_printout_and_headline_columns():
    from lav_b200 import evaluate as EV
    r = dict(samples=3, precision="f16", bev_iou=[None] * 3, det={}, plan=dict(ade=None, fde=None, per_cmd={}),
             det_boxes=accumulate(random_batches(3, 1)).summary())
    text = EV.format_result(r)
    assert "det boxes, vehicle" in text and "10-20 m:" in text
    cols = dict(EV.headline(dict(r, det=dict(pedestrian=dict(ap=dict(mean=None)), vehicle=dict(ap=dict(mean=None))))))
    assert cols["veh AP@IoU.5"] == r["det_boxes"]["vehicle"]["ap_iou"]["0.5"]
    assert cols["veh heading"] == r["det_boxes"]["vehicle"]["heading_rad"]
