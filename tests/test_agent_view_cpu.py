"""CPU: the numpy statement of the agent's debug view (oracle/view_ref.py) against the reference's frames
(tests/golden/agent_view.npz, written by oracle/pin_view.py from the unmodified LAVAgent.visualize) and its restated OpenCV and
numpy primitives against cv2 and numpy themselves on thousands of random cases."""
import os

import numpy as np
import pytest

from lav_b200 import view
from oracle import view_ref as V

cv2 = pytest.importorskip("cv2")
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "agent_view.npz")


def pixels(img):
    return set(map(tuple, np.argwhere(img.reshape(img.shape[0], img.shape[1], -1).any(-1))[:, ::-1].tolist()))


def test_statement_equals_reference_frames():
    g = np.load(GOLD)
    ppm, thresh = float(g["config"][4]), float(g["config"][5])
    assert list(g["kinds"]) == list(V.VIEW_KINDS)
    for kind, want in zip(g["kinds"], g["frames"]):
        got = V.case_frame(V.view_case(int(g["seed"]), str(kind)), ppm, thresh)
        np.testing.assert_array_equal(got, want, err_msg=str(kind))


@pytest.mark.parametrize("shape", [(288, 768, 320, 853), (192, 480, 320, 800), (320, 2293, 160, 1146), (7, 9, 20, 3)])
def test_resize_equals_cv2(shape):
    h, w, oh, ow = shape
    rng = np.random.default_rng(h * w)
    for seed in range(3):
        for img in (rng.integers(0, 256, (h, w, 3), dtype=np.uint8), (rng.integers(0, 2, (h, w, 3)) * 255).astype(np.uint8),
                    np.full((h, w, 3), 255, np.uint8)):
            np.testing.assert_array_equal(V.resize(img, ow, oh), cv2.resize(img, (ow, oh)), err_msg=f"{shape} seed {seed}")


@pytest.mark.parametrize("r", [1, 2])
def test_circles_equal_cv2_at_every_offset(r):
    for h, w in ((9, 11), (320, 320)):
        xs = list(range(-4, 6)) + list(range(w - 5, w + 4))
        ys = list(range(-4, 6)) + list(range(h - 5, h + 4))
        for cx in xs:
            for cy in ys:
                want = np.zeros((h, w, 3), np.uint8)
                cv2.circle(want, (cx, cy), r, (255, 0, 0), -1)
                got = np.zeros_like(want)
                V.circle(got, cx, cy, r, (255, 0, 0))
                np.testing.assert_array_equal(got, want, err_msg=f"r={r} centre ({cx}, {cy}) on {w}x{h}")


def _quads(rng, n, lo, hi):
    """random quads, vehicle-like boxes at every angle, zero-size boxes and boxes crossing or outside the image"""
    for t in range(n):
        kind = t % 5
        if kind == 0:
            yield rng.integers(lo, hi, (4, 2))
            continue
        x, y = rng.integers(lo, hi, 2)
        w, h = (0.0, 0.0) if kind == 1 else rng.uniform(0, 15, 2) if kind < 4 else rng.uniform(0, 400, 2)
        a = rng.uniform(0, 2 * np.pi)
        yield np.array(V.box_corners((x, y, w, h, np.cos(a), np.sin(a))))


def test_thick_contours_equal_cv2():
    rng = np.random.default_rng(11)
    n = 0
    for (h, w), (lo, hi), count in (((320, 320), (-40, 360), 1200), ((24, 24), (-10, 34), 1200), ((320, 320), (-5000, 5000), 200)):
        for pts in _quads(rng, count, lo, hi):
            want = np.zeros((h, w, 3), np.uint8)
            cv2.drawContours(want, np.array([pts]), 0, (255, 0, 0), 2)
            got = np.zeros_like(want)
            V.thick_polyline(got, [tuple(map(int, p)) for p in pts], (255, 0, 0))
            assert pixels(got) == pixels(want), (pts.tolist(), w, h)
            n += 1
    assert n == 2600


def test_box_corners_equal_numpy():
    rng = np.random.default_rng(3)
    for _ in range(5000):
        x, y = (int(v) for v in rng.integers(0, 320, 2))
        ww, hh = (float(v) for v in rng.uniform(0, 20, 2).astype(np.float32))
        a = rng.uniform(0, 2 * np.pi)
        cos, sin = float(np.float32(np.cos(a))), float(np.float32(np.sin(a)))
        m = np.array([[-sin, cos], [-cos, -sin]])
        want = [tuple(int(v) for v in ([x, y] + np.array(s) @ m).astype(int)) for s in ([-ww, -hh], [-ww, hh], [ww, hh], [ww, -hh])]
        assert V.box_corners((x, y, ww, hh, cos, sin)) == want
    assert V.box_corners((1, 2, np.nan, 3, 1, 0)) is None
    assert V.box_corners((1, 2, 1e300, 3, 1, 0)) is None


def test_points_and_target_equal_numpy():
    rng = np.random.default_rng(5)
    ego = [160, 280]
    locs = np.concatenate([rng.normal(0, 30, (2000, 2)), rng.normal(0, 1e8, (200, 2))]).astype(np.float32)
    for loc in locs:
        want = (ego + loc * 4).astype(int)
        p = V.point_pixel(loc, 4)
        if np.all(np.abs(want) < 2 ** 31):
            assert p == tuple(int(v) for v in want), loc
        else:
            assert p is None
    assert V.point_pixel(np.float32([np.nan, 0]), 4) is None
    for tgt in rng.normal(0, 60, (500, 2)).astype(np.float32):
        assert V.target_pixel(tgt, 4) == tuple(int(v) for v in np.clip(ego + np.array([float(t) for t in tgt]) * 4, 0, 255).astype(int))
    assert V.target_pixel(np.float32([np.nan, 1]), 4) is None


def _edge_values(edges):
    e = edges.astype(np.float32)
    return np.concatenate([e, np.nextafter(e, np.float32(np.inf)), np.nextafter(e, -np.float32(np.inf)),
                           np.float32([edges[-1], edges[0], np.inf, -np.inf, np.nan])])


def test_histogram_equals_histogramdd():
    rng = np.random.default_rng(9)
    xs, ys = _edge_values(V.XBINS), _edge_values(V.YBINS)
    pts = np.concatenate([
        np.stack([xs, rng.uniform(-40, 41, len(xs)).astype(np.float32)], 1),
        np.stack([rng.uniform(-10, 71, len(ys)).astype(np.float32), ys], 1),
        np.stack([rng.choice(xs, 5000), rng.choice(ys, 5000)], 1),
        rng.uniform([-12, -42], [73, 43], (20000, 2)).astype(np.float32)])
    finite = np.isfinite(pts).all(1)            # histogramdd refuses NaN / inf ranges only when it derives them; edges are given
    want = np.histogramdd(pts[finite], bins=(V.XBINS, V.YBINS))[0]
    np.testing.assert_array_equal(V.lidar_counts(pts), want)
    with np.errstate(invalid="ignore"):
        want_all = np.histogramdd(pts, bins=(V.XBINS, V.YBINS))[0]
    np.testing.assert_array_equal(V.lidar_counts(pts), want_all)
    hist = np.minimum(want, 10)
    np.testing.assert_array_equal(V.lidar_bev(pts), (hist / 10 * 255.)[::-1, :].astype(np.uint8))


def test_bev_mean_equals_numpy():
    rng = np.random.default_rng(4)
    for c in (1, 2, 4, 7):
        p = rng.uniform(0, 1, (c, 320, 320)).astype(np.float32)
        p[:, 0, :3] = np.float32([0, 1, np.nextafter(np.float32(1), np.float32(0))])
        np.testing.assert_array_equal(V.bev_mean(p), (255 * p.mean(axis=0)).astype(np.uint8))


def test_jet_tables_agree():
    np.testing.assert_array_equal(view.jet_bytes(), V.jet_bytes())
    assert V.jet_bytes().shape == (259, 3)
    scores = np.float32([0.0, 0.2, 1.0, np.nextafter(np.float32(1), np.float32(0)), 1.5, -0.1, np.nan])
    np.testing.assert_array_equal(V.jet_index(scores), [0, 51, 255, 255, 257, 256, 258])


def test_annotate_equals_statement():
    rng = np.random.default_rng(8)
    frames = rng.integers(0, 256, (3, 160, 1146, 3), dtype=np.uint8)
    speeds, cmds = np.float32([0.5, 3.25, 8.0]), np.int32([0, 4, 5])
    control, bra = rng.uniform(-1, 1, (3, 3)).astype(np.float32), rng.uniform(0, 1, 3).astype(np.float32)
    want = [V.annotate(f.copy(), float(speeds[i]), int(cmds[i]), *(float(v) for v in control[i]), float(bra[i]))
            for i, f in enumerate(frames)]
    got = view.annotate(frames.copy(), speeds, cmds, control, bra)
    np.testing.assert_array_equal(got, np.stack(want))
