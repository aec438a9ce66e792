"""The fp64 statement of the inference pillar encoders (tests/util.pillar_forward_ref64), pinned on the CPU: to the oracle's
PointPillarNet on small clouds, and to a hand-worked per-point loop on tiny clouds built around the grid's edges (one point,
pillars that collide on the clamped last row and column, points at exactly min_x, just below max_x and at max_x, a grid
with nx != ny).  tests/test_gpu_pillar_forward_contract.py holds the encoders to this statement."""
import numpy as np
import pytest
import torch

from lav_b200 import synth
from oracle import lav_ref as O
from tests import util

GRID4 = (-10.0, 70.0, -40.0, 40.0, 4.0, 320, 320)            # the LiDAR model's grid
SQUARE = (-40.0, 40.0, -40.0, 40.0, 4.0, 320, 320)           # x and y both round onto index 320 just below max
WIDE = (-10.0, 10.0, -5.0, 5.0, 2.0, 40, 20)                  # nx = 40 != ny = 20: xi 20..40 all clamp onto row 0
MODES = ["fp32", "sorted", "sorted_h16"]


def _weights(seed=0):
    g = torch.Generator().manual_seed(seed)
    w1 = torch.randn(64, 16, generator=g) * 0.25
    w2 = torch.randn(64, 64, generator=g) * 0.125
    s1, s2 = 0.5 + torch.rand(64, generator=g), 0.5 + torch.rand(64, generator=g)
    t1, t2 = torch.randn(64, generator=g) * 0.5, torch.randn(64, generator=g) * 0.5
    return w1, s1, t1, w2, s2, t2


def _below(v):
    return float(np.nextafter(np.float32(v), np.float32(-np.inf)))


def hand_loop(pts, starts, counts, grid, w1, s1, t1, w2, s2, t2, mode):
    """the same statement, one point at a time in numpy scalars: fp32 grid location, a dict of pillars, fp64 MLP, a dict of
    cells holding the running per-channel max."""
    mn_x, mx_x, mn_y, mx_y, ppm, nx, ny = grid
    f32 = np.float32
    W1, S1, T1, W2, S2, T2 = (t.double().numpy() for t in (w1, s1, t1, w2, s2, t2))
    if mode != "fp32":
        W2 = np.clip(W2.astype(np.float32), -65504, 65504).astype(np.float16).astype(np.float64)
    pillars = {}
    for b, (s, c) in enumerate(zip(starts, counts)):
        for r in range(s, s + c):
            p = pts[r, :11].numpy().astype(np.float32)
            x, y = p[0], p[1]
            if not (x >= f32(mn_x) and x < f32(mx_x) and y >= f32(mn_y) and y < f32(mx_y)):
                continue
            xi = int((x - f32(mn_x)) * f32(ppm))
            yi = int((y - f32(mn_y)) * f32(ppm))
            pillars.setdefault((b, xi, yi), []).append(p.astype(np.float64))
    canvas = np.zeros((len(counts), ny, nx, 64))
    for (b, xi, yi), members in pillars.items():
        mean = sum(m[:3] for m in members) / len(members)
        ox = float(f32(f32(yi) / f32(ppm)) + f32(mn_x))
        oy = float(f32(f32(xi) / f32(ppm)) + f32(mn_y))
        row, col = min(max(ny - 1 - xi, 0), ny - 1), min(max(yi, 0), nx - 1)
        for m in members:
            f = np.concatenate([m, m[:3] - mean, [m[0] - ox, m[1] - oy]])
            h = np.maximum(W1 @ f * S1 + T1, 0)
            if mode != "fp32":
                h = np.clip(h.astype(np.float32), -65504, 65504).astype(np.float16).astype(np.float64)
            o = np.maximum(W2 @ h * S2 + T2, 0)
            canvas[b, row, col] = np.maximum(canvas[b, row, col], o)
    if mode == "sorted_h16":
        canvas = np.clip(canvas.astype(np.float32), -65504, 65504).astype(np.float16).astype(np.float64)
    return canvas


def _cloud(xy, seed=1):
    g = torch.Generator().manual_seed(seed)
    p = torch.rand(len(xy), 11, generator=g) * 2 - 1
    p[:, :2] = torch.tensor(xy, dtype=torch.float32)
    p[:, 2] = torch.rand(len(xy), generator=g) * 4 - 2
    return p


def _tiny(name):
    """-> (pts, starts, counts, grid)"""
    if name == "one_point":
        return _cloud([(12.3, -7.7)]), [0], [1], GRID4
    if name == "edges":        # exactly min_x / min_y (kept), just below max_x / max_y (kept), at max_x / max_y (dropped)
        xy = [(-10.0, -40.0), (_below(70.0), 0.5), (3.0, _below(40.0)), (70.0, 0.5), (3.0, 40.0), (-10.0, 3.3), (-9.9, 3.3)]
        return _cloud(xy, 2), [0], [len(xy)], GRID4
    if name == "collide_last_row_and_col":   # (xi, yi) = (320, 320) and (319, 319) both land on row 0, col 319
        hi = _below(40.0)
        xy = [(hi, hi), (hi, hi), (39.9, 39.8), (39.95, 39.76), (hi, 0.1), (39.8, 0.1), (0.2, hi), (0.2, 39.9)]
        return _cloud(xy, 3), [0], [len(xy)], SQUARE
    if name == "wide_grid":
        g = torch.Generator().manual_seed(4)
        xy = torch.stack([torch.rand(60, generator=g) * 22 - 11, torch.rand(60, generator=g) * 11 - 5.5], 1)
        xy[:3] = torch.tensor([[_below(10.0), _below(5.0)], [9.9, 4.9], [0.0, 0.0]])
        return _cloud(xy.tolist(), 5), [0, 30], [30, 30], WIDE
    if name == "two_frames_gap":
        xy = [(float(i % 7) * 0.3 + 1, float(i // 7) * 0.2 - 1) for i in range(40)]
        return _cloud(xy, 6), [25, 0], [15, 20], GRID4
    raise KeyError(name)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", ["one_point", "edges", "collide_last_row_and_col", "wide_grid", "two_frames_gap"])
def test_statement_matches_hand_loop(case, mode):
    pts, starts, counts, grid = _tiny(case)
    ws = _weights()
    want = hand_loop(pts, starts, counts, grid, *ws, mode)
    got, bound = util.pillar_forward_ref64(pts, starts, counts, grid, *ws, mode)
    assert got.shape == want.shape and got.dtype == torch.float64
    np.testing.assert_allclose(got.numpy(), want, rtol=1e-12, atol=1e-12)
    assert bool((bound >= 0).all()) and bool(torch.isfinite(bound).all())
    if case == "one_point":                          # one occupied cell; the empty cells are exactly 0
        assert int((bound.sum(-1) > 0).sum()) == 1 and int((got.sum(-1) > 0).sum()) == 1
    if case == "edges":                               # 5 kept points; (-10, 3.3) and (-9.9, 3.3) share one pillar
        keep, xi, yi = util.pillar_locate(pts[:, 0], pts[:, 1], grid)
        assert keep.tolist() == [True, True, True, False, False, True, True]
        assert (int(xi[0]), int(yi[0]), int(xi[1]), int(yi[2])) == (0, 0, 319, 320)     # y just below 40 rounds onto ny
    if case == "collide_last_row_and_col":           # both pillars of the corner reach the corner cell
        keep, xi, yi = util.pillar_locate(pts[:, 0], pts[:, 1], grid)
        assert (int(xi[0]), int(yi[0]), int(xi[2]), int(yi[2])) == (320, 320, 319, 319)
        corner = hand_loop(pts[:2], [0], [2], grid, *ws, mode)[0, 0, 319]
        other = hand_loop(pts[2:4], [0], [2], grid, *ws, mode)[0, 0, 319]
        np.testing.assert_array_equal(want[0, 0, 319], np.maximum(corner, other))
        assert (want[0, 0, 319] != corner).any() and (want[0, 0, 319] != other).any()


def test_statement_location_is_fp32():
    """xi is trunc of the fp32 product: y = nextafter(40, -inf) on [-40, 40) rounds to 80 in fp32 and lands on 320 = ny;
    an fp64 computation would give 319."""
    y = torch.tensor([_below(40.0)], dtype=torch.float32)
    keep, xi, yi = util.pillar_locate(y, y, SQUARE)
    assert bool(keep[0]) and int(yi[0]) == 320 and int((y.double()[0] + 40) * 4) == 319
    ox, oy = util.pillar_origins((-10.0, 70.0, -40.0, 40.0, 3.0, 240, 240))
    assert float(ox[7]) == float(np.float32(np.float32(7) / np.float32(3)) + np.float32(-10))
    assert float(ox[7]) != 7 / 3 - 10


@pytest.mark.parametrize("clouds", ["pair", "ragged3"])
def test_statement_matches_oracle_pillar_net(clouds):
    """fp32 mode against oracle/lav_ref.pillar_net (fp32, folded BatchNorm) on clouds without a yi == nx collision, where the
    oracle's one-pillar-per-cell assignment and the max over pillars agree."""
    m, sd = util.lidar_model()
    ws = [t.detach() for t in m.point_pillar_net._build("cpu")]
    if clouds == "pair":
        cl = util.pillar_clouds()
    else:
        cl = [synth.stacked_lidar(900, tag="rc0"), synth.stacked_lidar(13, tag="rc1"), synth.stacked_lidar(400, tag="rc2")]
    counts = [len(c) for c in cl]
    buf = torch.cat(cl).contiguous()
    starts = list(np.cumsum([0] + counts[:-1]))
    keep, xi, yi = util.pillar_locate(buf[:, 0], buf[:, 1], GRID4)
    assert not bool((keep & ((xi == 320) | (yi == 320))).any())
    with torch.no_grad():
        want = O.pillar_net(sd, cl, counts, **util.GRID).permute(0, 2, 3, 1).double()
    got, bound = util.pillar_forward_ref64(buf, starts, counts, GRID4, *ws, "fp32")
    err = (got - want).abs()
    scale = float(want.abs().max())
    assert scale > 1 and float((got > 0).sum()) > 1000
    # the oracle is an fp32 computation (GEMM sums, unfolded BatchNorm): within the bound, plus the fp32 rounding of the
    # folded s and t (a few u of the activation scale)
    assert bool((err <= bound + 8 * util.U32 * scale).all()), float((err - bound).max())
    assert float(err.max()) < 1e-5 * scale


def test_bound_covers_a_fp32_evaluation():
    """The statement's own fp32 evaluation (decoration and MLP in fp32, centroid sums in a shuffled order) lies inside the
    "fp32" bound, and the "centroid" part bounds the difference between two shuffled orders."""
    pts = synth.stacked_lidar(3000, tag="bnd")
    pts[:, 0] = pts[:, 0] * 0.05 + 20             # few, crowded pillars: long centroid sums
    ws = _weights(7)
    got, bound = util.pillar_forward_ref64(pts, [0], [len(pts)], GRID4, *ws, "fp32")
    _, cbound = util.pillar_forward_ref64(pts, [0], [len(pts)], GRID4, *ws, "fp32", parts="centroid")
    assert float(cbound.max()) > 0
    outs = []
    for seed in (0, 1):
        perm = torch.randperm(len(pts), generator=torch.Generator().manual_seed(seed))
        p = pts[perm]
        keep, xi, yi = util.pillar_locate(p[:, 0], p[:, 1], GRID4)
        p, xi, yi = p[keep], xi[keep], yi[keep]
        _, inv = torch.unique(xi * 321 + yi, return_inverse=True)
        n = torch.bincount(inv).float()[:, None]
        s = torch.zeros((len(n), 3)).index_add_(0, inv, p[:, :3])
        ox, oy = (o.float() for o in util.pillar_origins(GRID4))
        f = torch.cat([p[:, :11], p[:, :3] - (s / n)[inv], p[:, :1] - ox[yi][:, None], p[:, 1:2] - oy[xi][:, None]], 1)
        w1, s1, t1, w2, s2, t2 = ws
        o = torch.relu(torch.relu(f @ w1.T * s1 + t1) @ w2.T * s2 + t2).double()
        cell = (319 - xi).clamp(0, 319) * 320 + yi.clamp(0, 319)
        c = torch.zeros((320 * 320, 64), dtype=torch.float64).scatter_reduce(0, cell[:, None].expand(-1, 64), o, "amax")
        outs.append(c.view(1, 320, 320, 64))
        assert bool(((c.view(1, 320, 320, 64) - got).abs() <= bound).all())
    assert bool(((outs[0] - outs[1]).abs() <= cbound).all())
