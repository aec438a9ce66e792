"""CPU: the numpy statement of the evaluation metrics (BEV IoU from counts, decode_packed's filters, greedy centre-distance
matching with its tie rules, all-point AP, plan ADE / FDE) on hand-built cases with known answers, the evaluator's host
reduction against it, and the evaluator's ordered, unaugmented batching with a short last batch."""
import numpy as np
import pytest
import torch

from lav_b200.model_inference import score_kept

THRESHOLDS = (0.5, 1.0, 2.0, 4.0)
GRID = dict(ppm=4, cx0=160.0, cy0=320.0, cy1=-40.0)          # ops.det_grid() of the default map


# ---------------------------------------------------------------------------------------------------- the numpy statement
def iou_counts(seg, gt):
    """seg (B,H,W,3) probabilities, gt (B,P,H,W) -> (B,3,2) int64 = per channel (|pred & gt|, |pred | gt|)."""
    pred = np.moveaxis(np.asarray(seg, np.float32), 3, 1) > 0.5
    tgt = np.asarray(gt)[:, :3] != 0
    return np.stack([(pred & tgt).sum((2, 3)), (pred | tgt).sum((2, 3))], -1).astype(np.int64)


def centres(actors, grid=GRID):
    """actor rows [x, y, ori, bx, by, typ] -> pixel centres (cx, cy) float32, with det_heatmaps' fp32 operations."""
    a = np.asarray(actors, np.float32).reshape(-1, 6)
    ppm = np.float32(grid["ppm"])
    cx = (-a[:, 0] * ppm) + np.float32(grid["cx0"])
    cy = ((-a[:, 1] * ppm) + np.float32(grid["cy0"])) + np.float32(grid["cy1"])
    return cx, cy


def window_dist(x, y, grid=GRID):
    wx, wy = float(grid["cx0"]), float(np.float32(grid["cy0"]) + np.float32(grid["cy1"]))
    dx, dy = np.asarray(x, np.float64) - wx, np.asarray(y, np.float64) - wy
    return np.sqrt(dx * dx + dy * dy)


def survivors(packed, w=320, min_score=0.2, grid=GRID):
    """decode_packed's filters on packed peaks (B,7,2*n_det) -> keep (B,cols) bool, x, y (int64), loc (int64)."""
    packed = np.asarray(packed, np.float32)
    ppm = grid["ppm"]
    loc = packed[:, 1].astype(np.int64)
    x, y = loc % w, loc // w
    bw, bh = packed[:, 2], packed[:, 3]
    cls = np.arange(packed.shape[2]) // (packed.shape[2] // 2)
    dist = window_dist(x, y, grid)
    keep = score_kept(packed[:, 0], min_score) & ~((cls[None] == 1) & (np.maximum(bw, bh) < 0.1 * ppm))
    keep &= ~((dist <= 2) | (dist >= 30 * ppm))
    return keep, x, y, loc


def match(packed, actors, offsets, w=320, min_score=0.2, grid=GRID):
    """-> ngt (B,2) int32, flags (B,cols) int32: bit 4 = survivor, bit k = matched at THRESHOLDS[k]."""
    packed = np.asarray(packed, np.float32)
    B, _, cols = packed.shape
    n_det = cols // 2
    keep, x, y, loc = survivors(packed, w, min_score, grid)
    actors = np.asarray(actors, np.float32).reshape(-1, 6)
    cx, cy = centres(actors, grid)
    d = window_dist(cx, cy, grid)
    typ = actors[:, 5]
    gcls = np.where(typ == 0, 0, np.where(typ == 1, 1, -1))
    gkeep = (gcls >= 0) & (d > 2) & (d < 30 * grid["ppm"])
    ngt = np.zeros((B, 2), np.int32)
    flags = np.where(keep, 16, 0).astype(np.int32)
    for b in range(B):
        rows = np.arange(offsets[b], offsets[b + 1])
        for c in range(2):
            g = rows[gkeep[rows] & (gcls[rows] == c)]
            ngt[b, c] = len(g)
            cand = [j for j in range(c * n_det, (c + 1) * n_det) if keep[b, j]]
            cand.sort(key=lambda j: (-packed[b, 0, j], loc[b, j], j))
            for k, t in enumerate(THRESHOLDS):
                used = set()
                for j in cand:
                    best = None
                    for r in g:                                    # ascending rows: a strict < keeps the lower row on a tie
                        if r in used:
                            continue
                        dx, dy = float(x[b, j]) - float(cx[r]), float(y[b, j]) - float(cy[r])
                        d2 = dx * dx + dy * dy
                        if d2 <= (t * grid["ppm"]) ** 2 and (best is None or d2 < best[0]):
                            best = (d2, r)
                    if best is not None:
                        used.add(best[1])
                        flags[b, j] |= 1 << k
    return ngt, flags


def plan_errors(plan, ego_locs):
    """plan (B,T,2), ego_locs (B,T+1,2) -> (B,2) fp64 = (ADE, FDE) against ego_locs[:, 1:]."""
    err = np.sqrt((np.square(np.asarray(plan, np.float64) - np.asarray(ego_locs, np.float64)[:, 1:])).sum(-1))
    return np.stack([err.mean(1), err[:, -1]], 1)


def average_precision(scores, matched, n_gt):
    """all-point interpolation: descending score (stable), precision envelope, sum of precision x recall step."""
    if n_gt == 0:
        return None
    order = sorted(range(len(scores)), key=lambda i: -float(scores[i]))
    tp, ap, prev_r = 0, 0.0, 0.0
    prec, rec = [], []
    for n, i in enumerate(order, 1):
        tp += bool(matched[i])
        prec.append(tp / n)
        rec.append(tp / n_gt)
    for i in range(len(prec)):
        ap += max(prec[i:]) * (rec[i] - prev_r)
        prev_r = rec[i]
    return ap


def eval_batch_ref(seg, gt, packed, actors, offsets, plan, ego_locs, min_score=0.2, grid=GRID):
    """every output of ops.eval_batch, as eval_views names them."""
    ngt, flags = match(packed, actors, offsets, np.asarray(seg).shape[2], min_score, grid)
    return dict(iou=iou_counts(seg, gt), ngt=ngt, flags=flags, score=np.asarray(packed, np.float32)[:, 0],
                plan_err=plan_errors(plan, ego_locs))


# ---------------------------------------------------------------------------------------------------- hand-built cases
def actor(px, py, typ=1):
    """an actor whose centre lies exactly on pixel (px, py) of the default grid."""
    return [(160 - px) / 4, (280 - py) / 4, 0.0, 2.0, 1.0, typ]


def packed_of(peaks, n_det=15, w=320):
    """peaks [(class, score, px, py, bw, bh)] -> (1, 7, 2 * n_det), the unused columns padded as det_peaks pads them."""
    p = np.zeros((1, 7, 2 * n_det), np.float32)
    p[0, 0] = -1e5
    p[0, 6] = w
    used = [0, 0]
    for c, s, x, y, bw, bh in peaks:
        j = c * n_det + used[c]
        used[c] += 1
        p[0, :6, j] = (s, y * w + x, bw, bh, 1.0, 0.0)
    return p


def test_equidistant_prediction_takes_the_lower_row():
    a, b = actor(100, 200), actor(104, 200)
    pk = packed_of([(1, 0.9, 102, 200, 5, 5), (1, 0.8, 101, 200, 5, 5)])   # P1 2 px from a and b; P2 1 px from a, 3 px from b
    ngt, flags = match(pk, [a, b], [0, 2])
    assert ngt.tolist() == [[0, 2]]
    # P1 takes a (the lower row), so P2 can only have b: beyond 0.5 m (2 px), within 1 m
    assert flags[0, 15] == 16 | 0b1111 and flags[0, 16] == 16 | 0b1110
    _, flags = match(pk, [b, a], [0, 2])                                    # rows swapped: P1 takes b, P2 gets a everywhere
    assert flags[0, 15] == 16 | 0b1111 and flags[0, 16] == 16 | 0b1111


def test_two_predictions_on_one_gt_and_equal_scores():
    acts = [actor(100, 200, typ=0)]
    pk = packed_of([(0, 0.5, 101, 200, 0, 0), (0, 0.9, 100, 201, 0, 0)])    # class 0 has no size filter
    _, flags = match(pk, acts, [0, 1])
    assert flags[0, 1] == 16 | 0b1111 and flags[0, 0] == 16        # the higher score takes it, the other is a false positive
    assert average_precision(pk[0, 0, :2], flags[0, :2] & 1, 1) == 1.0
    pk = packed_of([(0, 0.7, 101, 200, 0, 0), (0, 0.7, 100, 199, 0, 0)])    # equal scores: lower flat index ((100, 199)) first
    _, flags = match(pk, acts, [0, 1])
    assert flags[0, 1] & 1 and not flags[0, 0] & 1


def test_no_predictions_no_gt_and_gt_outside_the_window():
    acts = [actor(160, 280), actor(160, 281), actor(160, 280 - 120), actor(100, 200, typ=3), actor(100, 200)]
    pk = packed_of([])
    ngt, flags = match(pk, acts, [0, len(acts)])
    assert ngt.tolist() == [[0, 1]]                                # the ego (d = 0), d = 1 px, d = 30 m and class 3 do not count
    assert not flags.any()
    assert average_precision([], [], 1) == 0.0                     # GT but no prediction
    assert average_precision([0.9], [0], 0) is None                # no GT: null, not 0
    pk = packed_of([(1, 0.9, 160, 281, 5, 5), (1, 0.9, 160, 160, 5, 5), (1, 0.1, 100, 200, 5, 5), (1, 0.9, 100, 200, 0.3, 0.3),
                    (1, 0.9, 100, 200, 0.3, 5)])
    keep, *_ = survivors(pk)
    assert keep[0, 15:20].tolist() == [False, False, False, False, True]   # window, window, score, size (both sides), one side ok


def test_average_precision_and_iou_known_answers():
    ap = average_precision([0.9, 0.8, 0.7], [1, 0, 1], 3)
    assert abs(ap - (1 / 3 + (2 / 3) / 3)) < 1e-12
    seg = np.zeros((1, 4, 4, 3), np.float32)
    gt = np.zeros((1, 9, 4, 4), np.uint8)
    seg[0, :2, :, 0] = 0.9                                          # 8 predicted
    gt[0, 0, 1:3] = 1                                               # 8 true, 4 in common
    seg[0, 0, 0, 1] = 0.5                                           # exactly 0.5 is not a prediction
    assert iou_counts(seg, gt)[0].tolist() == [[4, 12], [0, 0], [0, 0]]
    assert np.allclose(plan_errors(np.ones((1, 2, 2)), np.zeros((1, 3, 2))), [[np.sqrt(2), np.sqrt(2)]])


def test_host_reduction_equals_the_statement():
    """lav_b200.evaluate's AP over a recording equals the statement's on random flags with ties, an empty class included."""
    from lav_b200 import evaluate as E
    from lav_b200.ops import EVAL_THRESHOLDS_M
    assert tuple(EVAL_THRESHOLDS_M) == THRESHOLDS
    rs = np.random.RandomState(0)
    scores = E.Scores()
    all_s, all_f = [], []
    for b in range(3):
        B, cols = 4 - b, 30
        s = np.round(rs.rand(B, cols), 1).astype(np.float32)
        f = (rs.rand(B, cols) < 0.7) * 16 + rs.randint(0, 16, (B, cols))
        f[:, :15] = 0                                                # class 0: nothing survives
        v = dict(iou=torch.from_numpy(rs.randint(0, 100, (B, 3, 2))), ngt=torch.from_numpy(np.stack([np.zeros(B), np.full(B, 9)], 1).astype(np.int32)),
                 score=torch.from_numpy(s), flags=torch.from_numpy(f.astype(np.int32)), plan_err=torch.from_numpy(rs.rand(B, 2)))
        scores.add(v, rs.randint(0, 6, B))
        keep = (f[:, 15:] & 16) != 0
        all_s.append(s[:, 15:][keep])
        all_f.append(f[:, 15:][keep])
    r = scores.summary()
    s, f = np.concatenate(all_s), np.concatenate(all_f)
    assert r["samples"] == 9 and r["det"]["pedestrian"]["ap"]["mean"] is None and r["det"]["vehicle"]["n_gt"] == 81
    for k, t in enumerate(THRESHOLDS):
        assert abs(r["det"]["vehicle"]["ap"][f"{t:g}"] - average_precision(s, (f >> k) & 1, 81)) < 1e-12


class _FakeDataset:
    """the calls TemporalBatchLoader makes, recorded."""

    def __init__(self, n):
        self.n, self.prepared, self.device = n, [], torch.device("cpu")

    def __len__(self):
        return self.n

    def draw(self, rng):
        raise AssertionError("an ordered loader draws no augmentation")

    def no_draw(self):
        return 0.0, [(np.zeros(2), 0.0)] * 3

    def prepare(self, idx, angle, jitters):
        self.prepared.append((idx, angle, [float(np.abs(j[0]).sum()) + j[1] for j in jitters]))
        return idx

    def stage_batch(self, hs, generator=None):
        return dict(idxs=list(hs), maps=None)

    def decode_maps(self, maps):
        return None

    def launch_batch(self, st):
        return tuple(st["idxs"])


def test_ordered_loader_keeps_index_order_and_the_short_last_batch():
    from lav_b200.datasets import TemporalBatchLoader
    ds = _FakeDataset(10)
    loader = TemporalBatchLoader(ds, 4, drop_last=False, num_workers=3, ordered=True)
    assert len(loader) == 3
    got = list(loader.staged_batches())
    assert [b for b, _ in got] == [(0, 1, 2, 3), (4, 5, 6, 7), (8, 9)]
    assert [st["idxs"] for _, st in got] == [[0, 1, 2, 3], [4, 5, 6, 7], [8, 9]]
    assert sorted(i for i, _, _ in ds.prepared) == list(range(10))
    assert all(a == 0.0 and not any(j) for _, a, j in ds.prepared)
    assert [b for b in TemporalBatchLoader(ds, 5, drop_last=False, ordered=True)] == [(0, 1, 2, 3, 4), (5, 6, 7, 8, 9)]
    with pytest.raises(AssertionError):
        list(TemporalBatchLoader(ds, 4))                            # the training mode still draws augmentations
