"""CPU: the numpy statement of the forecasts on detected vehicles (the row table of decode_packed + det_to_locs, the greedy match to
the recorded actors with its target gather, the host reduction) on hand-built cases with known answers, and the evaluator's row
table and DetectedForecastScores against it.  The per-row errors are tests/test_forecast_eval_cpu.py's statement."""
import math

import numpy as np
import torch

from lav_b200.model_inference import score_kept
from tests import test_evaluate_cpu as E
from tests import test_forecast_eval_cpu as F

GRID = E.GRID
CENTRE = (160.0, 280.0)                 # UniPlanner.crop_centre(320, 320) at the default offsets (0, 0.75)
MATCH_M = 2.0


# ---------------------------------------------------------------------------------------------------- the numpy statement
def row_table_ref(packed, ppm=4, centre=CENTRE, min_score=0.2):
    """the rows infer_batch forecasts, peak by peak: class-1 columns passing decode_packed's filters and det_to_locs' centre test,
    in frame, then column order.  -> frame (K,), col (K,), locs (K, 2) fp32 in det_to_locs' metres."""
    packed = np.asarray(packed, np.float32)
    B, _, cols = packed.shape
    n_det, W = cols // 2, int(packed[0, 6, 0])
    frame, col, locs = [], [], []
    for b in range(B):
        for j in range(n_det, cols):
            loc = int(packed[b, 1, j].astype(np.int64))
            x, y = loc % W, loc // W
            d = math.sqrt((x - 160) ** 2 + (y - 280) ** 2)
            small = np.float32(max(packed[b, 2, j], packed[b, 3, j])) < np.float32(0.1 * ppm)
            if not score_kept(packed[b, 0, j], min_score) or small or d <= 2 or d >= 30 * ppm:
                continue
            if math.sqrt((x - centre[0]) ** 2 + (y - centre[1]) ** 2) <= 4:
                continue
            frame.append(b)
            col.append(j)
            locs.append([(x - centre[0]) / ppm, (y - centre[1]) / ppm])
    return np.array(frame, np.int64), np.array(col, np.int64), np.array(locs, np.float32).reshape(-1, 2)


def match_ref(packed, actors, offsets, row_offsets, cols, num_objs, locs, ego_locs, match_m=MATCH_M, w=320, grid=GRID):
    """every output of ops.det_forecast_match, as det_match_views names them (without err / branch)."""
    packed = np.asarray(packed, np.float32)
    actors = np.asarray(actors, np.float32).reshape(-1, 6)
    locs, ego_locs = np.asarray(locs, np.float32), np.asarray(ego_locs, np.float32)
    B, k, T = packed.shape[0], int(row_offsets[-1]), locs.shape[2] - 1
    ppm = float(np.float32(grid["ppm"]))
    cx, cy = E.centres(actors, grid)
    d = E.window_dist(cx, cy, grid)
    vehicle = (actors[:, 5] == 1) & (d > 2) & (d < 30 * ppm)
    thr2 = (match_m * ppm) ** 2
    out = dict(actor=np.full(k, -1, np.int32), flag=np.zeros(k, np.int32), dist=np.full(k, np.nan),
               target=np.full((k, T, 2), np.nan, np.float32), ngt=np.zeros((B, 2), np.int32))
    for b in range(B):
        a0, a1 = offsets[b], offsets[b + 1]
        cand = [i for i in range(a1 - a0) if vehicle[a0 + i]]
        out["ngt"][b] = sum(i < num_objs[b] for i in cand), sum(i >= num_objs[b] for i in cand)
        rows = list(range(row_offsets[b], row_offsets[b + 1]))
        loc = {r: int(packed[b, 1, cols[r]].astype(np.int64)) for r in rows}
        rows.sort(key=lambda r: (-float(packed[b, 0, cols[r]]), loc[r], cols[r]))
        taken = set()
        for r in rows:
            x, y = loc[r] % w, loc[r] // w
            best = None
            for i in cand:                                                  # ascending rows: a strict < keeps the lower row on a tie
                if i in taken:
                    continue
                dx, dy = float(x) - float(cx[a0 + i]), float(y) - float(cy[a0 + i])
                d2 = dx * dx + dy * dy
                if d2 <= thr2 and (best is None or d2 < best[0]):
                    best = (d2, i)
            if best is None:
                continue
            d2, i = best
            taken.add(i)
            tracked = i < num_objs[b]
            out["actor"][r], out["flag"][r], out["dist"][r] = i, 1 | (2 * tracked), math.sqrt(d2) / ppm
            if tracked:
                out["target"][r] = locs[b, i, 1:] - ego_locs[b, 0]
    return out


def reduce_ref(batches, match_m=MATCH_M):
    """the host reduction over a recording of [(scores (K,), flag (K,), err (K, >= 4), ngt (B, 2))] -> DetectedForecastScores'
    summary."""
    s = np.concatenate([np.asarray(b[0], np.float32) for b in batches] or [np.zeros(0, np.float32)])
    f = np.concatenate([np.asarray(b[1]) for b in batches] or [np.zeros(0, np.int32)])
    e = np.concatenate([np.asarray(b[2])[:, :4] for b in batches] or [np.zeros((0, 4))])
    gt = int(sum(int(np.asarray(b[3])[:, 0].sum()) for b in batches))
    tracked = [bool(v & 2) for v in f]
    untracked = [bool(v & 1) and not v & 2 for v in f]
    m = e[np.array(tracked, bool)].reshape(-1, 4)
    mean = lambda a: float(np.mean(a)) if len(a) else None
    keep = [i for i in range(len(f)) if not untracked[i]]
    tp = [tracked[i] and e[i, 1] <= F.MISS_M for i in keep]
    return dict(rows=len(f), matched=int(sum(tracked)), matched_untracked=int(sum(untracked)), gt=gt,
                recall=sum(tracked) / gt if gt else None, min_ade=mean(m[:, 0]), min_fde=mean(m[:, 1]), top_ade=mean(m[:, 2]),
                top_fde=mean(m[:, 3]), miss_rate=mean(m[:, 1] > F.MISS_M), ap=E.average_precision(s[keep], tp, gt), match_m=match_m)


# ---------------------------------------------------------------------------------------------------- the row table
def agent_rows(packed, ppm=4):
    """what the agent forecasts: InferModel.decode_packed, then UniPlanner.det_to_locs per frame."""
    from lav_b200.heads import UniPlanner
    from lav_b200.model_inference import InferModel

    class Planner:
        offset_x, offset_y, pixels_per_meter = torch.tensor(0.0), torch.tensor(0.75), ppm
        crop_centre, det_to_locs = UniPlanner.crop_centre, UniPlanner.det_to_locs

    class Model:
        pixels_per_meter = ppm
    dets = InferModel.decode_packed(Model(), torch.from_numpy(np.asarray(packed, np.float32)))
    return [Planner().det_to_locs(d[1], 320, 320)[0] for d in dets]


def test_row_table_equals_decode_packed_and_det_to_locs_in_fp32():
    from lav_b200.evaluate import detected_rows
    below = float(np.nextafter(np.float32(0.2), np.float32(0)))
    frames = [
        [(1, 0.9, 100, 200, 5, 5), (1, below, 110, 200, 5, 5), (1, 0.2, 120, 200, 5, 5),   # below / exactly float32(0.2): both dropped
         (0, 0.9, 130, 200, 5, 5), (0, 0.5, 90, 90, 0, 0),                                 # class 0: decoded, never a row
         (1, 0.8, 163, 280, 5, 5), (1, 0.8, 164, 280, 5, 5), (1, 0.8, 160, 276, 5, 5),     # within 4 px of the crop centre
         (1, 0.8, 165, 280, 5, 5), (1, 0.7, 160, 281, 5, 5), (1, 0.7, 160, 160, 5, 5),     # 5 px: kept; outside the window
         (1, 0.7, 100, 250, 0.3, 0.3), (1, 0.7, 101, 250, 0.3, 5),                         # size filter: both sides / one side
         (1, 0.6, 140, 250, 2, 2), (1, 0.6, 141, 250, 2, 2)],                                  # score ties
        [],
        [(0, 0.9, 100, 100, 5, 5), (1, 0.3, 200, 240, 1, 1), (1, 0.95, 120, 260, 1, 1)],
    ]
    packed = np.concatenate([E.packed_of(p) for p in frames])
    want = agent_rows(packed)
    frame, col, locs = row_table_ref(packed)
    assert [int((frame == b).sum()) for b in range(3)] == [len(w) for w in want] == [5, 0, 2]
    assert np.array_equal(locs, np.array([x for w in want for x in w], np.float32).reshape(-1, 2))
    assert col.tolist() == [15, 21, 25, 26, 27, 15, 16]
    got = detected_rows(packed, 4, CENTRE)
    assert np.array_equal(got["frame"], frame) and np.array_equal(got["col"], col) and np.array_equal(got["locs"], locs)
    assert got["counts"].tolist() == [5, 0, 2] and np.array_equal(got["score"], packed[frame, 0, col])


def test_row_table_on_random_peaks_in_fp32():
    """Scores rounded to two decimals, so float32(0.2) occurs: those columns are never rows (the reference compares in fp32)."""
    from lav_b200.evaluate import detected_rows
    rs = np.random.RandomState(5)
    packed = np.zeros((40, 7, 30), np.float32)
    packed[:, 0] = np.round(rs.rand(40, 30) * 0.5, 2)
    assert (packed[:, 0] == np.float32(0.2)).any()
    packed[:, 1] = np.where(rs.rand(40, 30) < 0.3, 280 * 320 + 160 + rs.randint(-6, 7, (40, 30)) + 320 * rs.randint(-6, 7, (40, 30)),
                            rs.randint(0, 320 * 320, (40, 30)))
    packed[:, 2:4] = rs.uniform(0, 1, (40, 2, 30))
    packed[:, 6] = 320
    want = agent_rows(packed)
    frame, col, locs = row_table_ref(packed)
    assert [int((frame == b).sum()) for b in range(40)] == [len(w) for w in want] and len(frame) > 20
    assert np.array_equal(locs, np.array([x for w in want for x in w], np.float32).reshape(-1, 2))
    got = detected_rows(packed, 4, CENTRE)
    assert np.array_equal(got["frame"], frame) and np.array_equal(got["col"], col) and np.array_equal(got["locs"], locs)
    assert not (packed[frame, 0, col] <= np.float32(0.2)).any()


# ---------------------------------------------------------------------------------------------------- the match
def labels(B, M=6, T=4, seed=0):
    rs = np.random.RandomState(seed)
    return (rs.randn(B, M, T + 1, 2) * 10).astype(np.float32), (rs.randn(B, T + 1, 2)).astype(np.float32)


def one_sample(peaks, acts, num_objs=None, match_m=MATCH_M):
    """the match of one sample's class-1 peaks [(score, px, py)] against actors ``acts``."""
    packed = E.packed_of([(1, s, x, y, 5, 5) for s, x, y in peaks])
    cols = np.arange(15, 15 + len(peaks))
    locs, ego = labels(1, max(len(acts), 1))
    n = len(acts) if num_objs is None else num_objs
    return match_ref(packed, acts, [0, len(acts)], [0, len(peaks)], cols, [n], locs, ego, match_m), locs, ego


def test_nearest_not_first_and_ties_to_the_lower_row():
    r, *_ = one_sample([(0.9, 100, 200)], [E.actor(106, 200), E.actor(101, 201)])
    assert r["actor"].tolist() == [1] and r["dist"][0] == math.sqrt(2) / 4
    r, *_ = one_sample([(0.9, 100, 200)], [E.actor(103, 200), E.actor(97, 200)])       # 3 px either side
    assert r["actor"].tolist() == [0] and r["dist"][0] == 0.75


def test_a_higher_ranked_row_takes_the_actor_first():
    # row 0 (score 0.5) sits on actor 0; row 1 (score 0.9) is 1 px from it and takes it; row 0 falls back to actor 1, 6 px away
    r, *_ = one_sample([(0.5, 100, 200), (0.9, 101, 200)], [E.actor(100, 200), E.actor(94, 200)])
    assert r["actor"].tolist() == [1, 0] and r["dist"].tolist() == [1.5, 0.25]
    # equal scores: the lower flat index ranks first
    r, *_ = one_sample([(0.7, 101, 200), (0.7, 100, 199)], [E.actor(100, 200)])
    assert r["actor"].tolist() == [-1, 0] and r["flag"].tolist() == [0, 3]


def test_pedestrians_and_vehicles_outside_the_window_never_match():
    acts = [E.actor(100, 200, typ=0), E.actor(160, 281), E.actor(160, 160), E.actor(100, 200, typ=2)]
    r, *_ = one_sample([(0.9, 100, 200), (0.8, 160, 281), (0.7, 160, 160)], acts)
    assert r["actor"].tolist() == [-1, -1, -1] and r["flag"].tolist() == [0, 0, 0] and np.isnan(r["dist"]).all()
    assert np.isnan(r["target"]).all() and r["ngt"].tolist() == [[0, 0]]


def test_match_radius_is_inclusive():
    at = E.actor(108, 200)                                                    # exactly 8 px = 2 m
    r, *_ = one_sample([(0.9, 100, 200)], [at])
    assert r["actor"].tolist() == [0] and r["dist"][0] == 2.0
    beyond = list(at)
    beyond[0] = float(np.float32(at[0]) - np.float32(2e-6))                  # the centre moves a float32 step further away
    assert E.centres([beyond])[0][0] > 108
    r, *_ = one_sample([(0.9, 100, 200)], [beyond])
    assert r["actor"].tolist() == [-1] and r["ngt"].tolist() == [[1, 0]]


def test_untracked_actor_is_matched_and_flagged_and_targets_are_the_tracks():
    acts = [E.actor(100, 200), E.actor(120, 200), E.actor(140, 200)]
    r, locs, ego = one_sample([(0.9, 100, 200), (0.8, 121, 200), (0.7, 140, 201)], acts, num_objs=2)
    assert r["actor"].tolist() == [0, 1, 2] and r["flag"].tolist() == [3, 3, 1] and r["ngt"].tolist() == [[2, 1]]
    assert np.array_equal(r["target"][0], locs[0, 0, 1:] - ego[0, 0]) and np.array_equal(r["target"][1], locs[0, 1, 1:] - ego[0, 0])
    assert np.isnan(r["target"][2]).all() and r["dist"][2] == 0.25


def test_samples_without_rows_or_actors():
    packed = np.concatenate([E.packed_of([(1, 0.9, 100, 200, 5, 5)]), E.packed_of([]), E.packed_of([(1, 0.9, 50, 50, 5, 5)])])
    acts = [E.actor(100, 200), E.actor(100, 220)]
    locs, ego = labels(3)
    r = match_ref(packed, acts, [0, 1, 2, 2], [0, 1, 1, 2], [15, 15], [1, 1, 0], locs, ego)
    assert r["actor"].tolist() == [0, -1] and r["ngt"].tolist() == [[1, 0], [1, 0], [0, 0]]
    r = match_ref(packed[1:2], [], [0, 0], [0, 0], np.zeros(0, np.int64), [0], locs[:1], ego[:1])
    assert r["actor"].shape == (0,) and r["target"].shape == (0, 4, 2) and r["ngt"].tolist() == [[0, 0]]


# ---------------------------------------------------------------------------------------------------- the host reduction
def views(err, flag, ngt, t=4):
    k = len(flag)
    return dict(err=torch.from_numpy(np.asarray(err, np.float64).reshape(k, 6)), flag=torch.from_numpy(np.asarray(flag, np.int32)),
                ngt=torch.from_numpy(np.asarray(ngt, np.int32).reshape(-1, 2)))


def test_host_reduction_known_answers():
    from lav_b200.evaluate import DetectedForecastScores
    err = np.zeros((5, 6))
    err[:, 1] = [1.0, 3.0, 0.5, 0.0, 2.0]                                    # minFDE: row 1 a miss, row 4 exactly 2 m (a hit)
    flag = [3, 3, 0, 1, 3]
    scores = [0.9, 0.8, 0.8, 0.95, 0.8]                                      # ties at 0.8 keep row order: 1 (miss), 2 (FP), 4 (TP)
    ds = DetectedForecastScores()
    ds.add(views(err, flag, [[3, 1], [1, 0]]), scores)
    s = ds.summary()
    assert s == reduce_ref([(scores, flag, err, np.array([[3, 1], [1, 0]]))])
    assert (s["rows"], s["matched"], s["matched_untracked"], s["gt"]) == (5, 3, 1, 4) and s["recall"] == 0.75
    assert s["miss_rate"] == 1 / 3 and s["min_fde"] == 2.0 and s["match_m"] == 2.0
    # ranked: TP (0.9), FP (0.8, miss), FP, TP -> precision envelope 1, 1/2 at recalls 1/4, 2/4
    assert abs(s["ap"] - (1 / 4 + 0.5 / 4)) < 1e-12

    ds = DetectedForecastScores()                                            # rows but no tracked vehicle: null recall and AP
    ds.add(views(np.zeros((2, 6)), [0, 1], [[0, 1]]), [0.5, 0.6])
    s = ds.summary()
    assert s["gt"] == 0 and s["recall"] is None and s["ap"] is None and s["min_ade"] is None and s["matched_untracked"] == 1
    assert s == reduce_ref([([0.5, 0.6], [0, 1], np.zeros((2, 6)), np.array([[0, 1]]))])

    s = DetectedForecastScores().summary()                                   # no batch at all
    assert s == dict(rows=0, matched=0, matched_untracked=0, gt=0, recall=None, min_ade=None, min_fde=None, top_ade=None,
                     top_fde=None, miss_rate=None, ap=None, match_m=2.0)
    ds = DetectedForecastScores()                                            # every row untracked, tracked GT unmatched
    ds.add(views(np.full((3, 6), np.nan), [1, 1, 1], [[2, 3]]), [0.3, 0.4, 0.5])
    s = ds.summary()
    assert s["matched"] == 0 and s["matched_untracked"] == 3 and s["recall"] == 0.0 and s["ap"] == 0.0 and s["min_ade"] is None


def test_host_reduction_equals_the_statement():
    from lav_b200.evaluate import DetectedForecastScores
    rs = np.random.RandomState(2)
    ds, batches = DetectedForecastScores(), []
    for k, b in ((9, 4), (0, 2), (13, 5)):
        cast, score, target, cmd = F.random_rows(k, 6, 10, rs.randint(1000))
        err = F.forecast_eval_ref(cast, score, target, np.full(k, -1))["err"]
        flag = rs.choice([0, 1, 3, 3], k).astype(np.int32)
        s = np.round(rs.rand(k), 1).astype(np.float32)
        ngt = rs.randint(0, 4, (b, 2)).astype(np.int32)
        ds.add(views(err, flag, ngt), s)
        batches.append((s, flag, err, ngt))
    assert ds.summary() == reduce_ref(batches)
