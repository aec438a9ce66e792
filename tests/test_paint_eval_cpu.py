"""CPU: the numpy statement of lavb_paint_confusion (used by tests/test_gpu_paint_eval.py) with hand-built known answers, the host
reduction and metrics of lav_b200.evaluate_paint, and the host half of datasets.PaintDataset on a synthetic recording."""
import numpy as np
import pytest

from lav_b200 import ops, synth
from lav_b200 import point_painting as PP
from lav_b200.data_pipeline import roof_keep

H, W = 288, 256
WINDOW = (-10.0, 70.0, -40.0, 40.0)
RANGE_EDGES = np.float32(ops.PAINT_RANGES_M)


# ----------------------------------------------------------------------------- the statement of the kernel
def fma32(a, b, c):
    """fp32 fmaf(a, b, c) with one rounding: a * b is exact in fp64, the fp64 sum's rounding error is recovered (TwoSum) and a sum
    that rounded onto an fp32 midpoint is nudged toward the exact value, so the final fp64 -> fp32 rounding is the only one."""
    p = np.asarray(a, np.float32).astype(np.float64) * np.asarray(b, np.float32).astype(np.float64)
    c = np.asarray(c, np.float32).astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        s = p + c
        bb = s - p
        err = (p - (s - bb)) + (c - bb)
        bits = s.view(np.int64) if isinstance(s, np.ndarray) else np.float64(s).view(np.int64)
        mid = (bits & ((1 << 29) - 1)) == (1 << 28)
        fix = mid & (err != 0) & np.isfinite(s)
        s = np.where(fix, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
        return s.astype(np.float32)


def project_ref(cams, x, y, z, h=H, w=W):
    """project_hit (project_hit.cuh) in fp32, operation for operation: -> (camera or -1, u, v) per point."""
    cams = np.asarray(cams, np.float32)
    x, y, z = (np.asarray(a, np.float32) for a in (x, y, z))
    one = np.float32(1)
    hit, hu, hv = np.full(x.shape, -1), np.zeros(x.shape, np.int64), np.zeros(x.shape, np.int64)

    def dot4(r, a, b, c, d):
        return fma32(r[3], d, fma32(r[2], c, fma32(r[1], b, np.float32(r[0]) * a)))

    def dot3(r, a, b, c):
        return fma32(r[2], c, fma32(r[1], b, np.float32(r[0]) * a))

    def trunc(v):
        with np.errstate(invalid="ignore"):
            ok = np.abs(v) < np.float32(9.2233720368547758e18)
            return np.where(ok, np.trunc(np.where(ok, v, 0)).astype(np.int64), np.int64(-2 ** 63))
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        for c in range(len(cams)):
            K, L, Wc = cams[c, :9], cams[c, 9:25], cams[c, 25:41]
            wv = [dot4(L[4 * r:4 * r + 4], x, y, z, one) for r in range(4)]
            c0, c1, c2 = (dot4(Wc[4 * r:4 * r + 4], *wv) for r in range(3))
            a0, a1, a2 = c1, -c2, c0
            q0, q1, q2 = (dot3(K[3 * r:3 * r + 3], a0, a1, a2) for r in range(3))
            den = np.float32(1e-5) + q2
            u, v, zi = trunc(q0 / den), trunc(q1 / den), trunc(q2)
            ok = (zi >= 0) & (u >= 0) & (u < w) & (v >= 0) & (v < h)
            hit, hu, hv = np.where(ok, c, hit), np.where(ok, u, hu), np.where(ok, v, hv)
    return hit, hu, hv


def logits_ref32(fv, table, pv, pu, c):
    """deconv_logits.cuh in fp32: per point bias[k], then fmaf(f[ch], w[pv][pu][ch][k], .) over ch = 0..15 -> (n, c)."""
    t = np.asarray(table, np.float32)
    w, b = t[:512].reshape(2, 2, 16, 8), t[512:520]
    out = np.empty((len(fv), c), np.float32)
    for k in range(c):
        acc = np.full(len(fv), b[k], np.float32)
        for ch in range(16):
            acc = fma32(fv[:, ch], w[pv, pu, ch, k], acc)
        out[:, k] = acc
    return out


def logits_ref64(fv, table, pv, pu, c):
    """the same logits in fp64 and their scale sum |f w| + |b| (for the near-tie bound)."""
    t = np.asarray(table, np.float64)
    w, b = t[:512].reshape(2, 2, 16, 8)[pv, pu][..., :c], t[512:512 + c]
    f = np.asarray(fv, np.float64)
    return f @ w + b, np.abs(f) @ np.abs(w) + np.abs(b)


def first_argmax(v):
    """the first index of the largest entry of each row (ties to the lower index; rows without NaN)."""
    return np.argmax(v, -1)


def stored_class_ref(rows):
    """the class a lidar_sem row encodes, decoded in fp64 (sequential sum, no contraction) -> (n,) with -1 = stored-invalid."""
    s = np.asarray(rows, np.float32).astype(np.float64)
    n, k = s.shape
    with np.errstate(invalid="ignore", divide="ignore"):
        tot = s[:, 0].copy()
        for j in range(1, k):
            tot = tot + s[:, j]
        q = np.sqrt(tot)
        p = np.concatenate([(1.0 - q)[:, None], s / q[:, None]], 1)
    cls = np.where(np.isnan(p).any(1) | np.isnan(s).any(1), -1, first_argmax(np.where(np.isnan(p), -np.inf, p)))
    return np.where(~np.isnan(s).any(1) & (tot == 0), 0, cls)


def range_bin(x, y):
    x, y = np.float32(x), np.float32(y)
    r = np.sqrt(x * x + y * y)
    return np.searchsorted(RANGE_EDGES, r, side="right")


def paint_confusion_ref(points, tags, lut, cams, window, c, feat=None, table=None, stored=None, meta=None):
    """(F, L) int64 counts of lavb_paint_confusion, and per frame a dict of per-point arrays (cam, u, v, gt, online, stored, win,
    rb; -1 where not defined) plus "logits64" / "scale" of the visible points for the near-tie bound."""
    points = np.asarray(points, np.float32)
    F, N, _ = points.shape
    cams = np.asarray(cams, np.float32)
    ncam = len(cams)
    h, w = np.asarray(tags).shape[1:]
    tags = np.asarray(tags).reshape(F, ncam, h, w)
    online, st_on = feat is not None, stored is not None
    L = ops.paint_confusion_ints(ncam, c, online, st_on)
    out = np.zeros((F, L), np.int64)
    views = ops.paint_confusion_views(out, ncam, c, online, st_on)
    names = {k: i for i, k in enumerate(ops.PAINT_COUNTERS)}
    mn_x, mx_x, mn_y, mx_y = (np.float32(v) for v in window)
    per = []
    for f in range(F):
        rows = N if meta is None else min(max(int(meta[f][0]), 0), N)
        score_st = st_on and (meta is None or int(meta[f][1]) != 0)
        p = points[f, :rows]
        x, y, z = p[:, 0], p[:, 1], p[:, 2]
        cnt = views["counters"][f]
        cnt[names["points"]] += rows
        nan = np.isnan(p[:, :3]).any(1)
        cnt[names["nan"]] += int(nan.sum())
        roof = ~nan & ~roof_keep(p)
        with np.errstate(invalid="ignore"):
            win = ~nan & ~roof & (x >= mn_x) & (x < mx_x) & (y >= mn_y) & (y < mx_y)
        cnt[names["roof"]] += int(roof.sum())
        cnt[names["in_window"]] += int(win.sum())
        cam, u, v = project_ref(cams, x, y, z, h, w)
        cam = np.where(nan, -1, cam)
        vis = cam >= 0
        cnt[names["not_visible"]] += int((~nan & ~vis).sum())
        cnt[names["not_visible_in_window"]] += int((win & ~vis).sum())
        gt = np.full(rows, -1)
        gt[vis] = np.asarray(lut)[tags[f, cam[vis], v[vis], u[vis]]]
        rb = np.where(vis, range_bin(x, y), -1)
        d = dict(cam=cam, u=u, v=v, gt=gt, win=win, rb=rb, online=np.full(rows, -1), stored=np.full(rows, -1),
                 logits64=np.zeros((rows, c)), scale=np.zeros((rows, c)))
        if online:
            fr = np.asarray(feat, np.float32).reshape(F, ncam, h // 2, w // 2, 16)[f]
            idx = np.nonzero(vis)[0]
            for pv in range(2):
                for pu in range(2):
                    sel = idx[((v[idx] & 1) == pv) & ((u[idx] & 1) == pu)]
                    fv = fr[cam[sel], v[sel] >> 1, u[sel] >> 1]
                    lg = logits_ref32(fv, table, pv, pu, c)
                    bad = np.isnan(lg).any(1)
                    d["online"][sel] = np.where(bad, -2, first_argmax(np.where(np.isnan(lg), -np.inf, lg)))
                    d["logits64"][sel], d["scale"][sel] = logits_ref64(fv, table, pv, pu, c)
            cnt[names["invalid"]] += int((d["online"] == -2).sum())
        if score_st:
            cls = stored_class_ref(np.asarray(stored, np.float32)[f, :rows])
            d["stored"] = np.where(vis, np.where(cls < 0, -2, cls), -1)
            cnt[names["stored_invalid"]] += int((d["stored"] == -2).sum())
        for src in ("online", "stored"):
            if src in views:
                pr = d[src]
                ok = pr >= 0
                np.add.at(views[src][f], (cam[ok], rb[ok], win[ok].astype(int), gt[ok], pr[ok]), 1)
        if "agreement" in views:
            ok = (d["online"] >= 0) & (d["stored"] >= 0)
            np.add.at(views["agreement"][f], (cam[ok], d["online"][ok], d["stored"][ok]), 1)
        per.append(d)
    return out, per


# ----------------------------------------------------------------------------- hand-built cases
CAMS = np.stack([cv.packed() for cv in PP.make_converters(1.5, 2.4)])


def pixel_point(u, v, depth=10.0, cam=1):
    """a LiDAR point (sensor at the origin, the cameras 1.5 m ahead at its height) in front of camera ``cam`` of CAMS at depth
    ``depth`` that projects to the centre of pixel (u, v), worked out in fp64."""
    conv = PP.make_converters(1.5, 2.4)[cam]
    f = conv.K[0, 0]
    a0, a1 = (u + 0.5 - W / 2) * depth / f, (v + 0.5 - H / 2) * depth / f
    cam_xyz = np.array([depth, a0, -a1, 1.0])                   # (c0, c1, c2): a0 = c1, a1 = -c2, a2 = c0
    world = np.linalg.inv(conv.world_to_cam) @ cam_xyz
    lidar = np.linalg.inv(conv.lidar_to_world) @ world
    return lidar[:3].astype(np.float32)


def test_projection_known_answers():
    pts = np.array([pixel_point(100, 50), pixel_point(255, 287), pixel_point(0, 0), [-20, 0, 0], [-1.2, 0, -1.25]], np.float32)
    cam, u, v = project_ref(CAMS[1:2], pts[:, 0], pts[:, 1], pts[:, 2])
    assert cam.tolist() == [0, 0, 0, -1, -1]                      # the last column and row are inside; behind is not
    assert (u[:3].tolist(), v[:3].tolist()) == ([100, 255, 0], [50, 287, 0])
    cam, _, _ = project_ref(CAMS, pts[:, 0], pts[:, 1], pts[:, 2])
    assert cam[3] == -1 and cam[4] == -1                          # behind every camera; the roof return too
    nxt = pixel_point(256, 100)                                   # column 256 of the middle camera: outside its image
    assert project_ref(CAMS[1:2], *nxt[:, None])[0][0] == -1


def test_two_cameras_the_last_wins():
    """a point at 30 degrees to the right, inside both the middle and the right camera's field of view: the right one (later in
    the list) paints and scores it."""
    az, r = np.deg2rad(30.0), 12.0
    p = np.array([[1.5 + r * np.cos(az), -r * np.sin(az), -1.0], [1.5 + r * np.cos(az), r * np.sin(az), -1.0]], np.float32)
    alone = [project_ref(CAMS[k:k + 1], p[:, 0], p[:, 1], p[:, 2])[0] for k in range(3)]
    both = project_ref(CAMS, p[:, 0], p[:, 1], p[:, 2])[0]
    for j in range(2):
        seen = [k for k in range(3) if alone[k][j] == 0]
        assert len(seen) == 2 and both[j] == seen[-1], (seen, both[j])


def test_stored_decode_known_answers():
    rows = np.array([[0, 0, 0, 0],                                 # all zero: not seen when painted -> background
                     [0, 1, 0, 0],                                 # one-hot p_2 = 1 -> class 2
                     [0, 0, np.nan, 0],                            # NaN -> stored-invalid
                     [0.234375, 0.15625, 0, 0],                    # p = (0.375, 0.375, 0.25): p_0 ties class 1 -> 0
                     [0.234375, 0.15625 * 2, 0, 0],                # no tie: class 2 is largest
                     [-0.5, 0, 0, 0]], np.float32)                 # negative sum: sqrt is NaN -> stored-invalid
    assert stored_class_ref(rows).tolist() == [0, 2, -1, 0, 2, -1]


def test_counts_known_answers():
    """one frame at C = 3, the middle camera only: the tags make every pixel class 1 except column 255 (class 2)."""
    xyz = [pixel_point(100, 50), pixel_point(255, 287, depth=25.0), [-20, 0, 0], [-1.2, 0, -1.25], [np.nan, 0, 0], [70, 0, 0],
           pixel_point(20, 20, depth=45.0), [0, 5, -2]]
    pts = np.array([np.append(np.asarray(p, np.float32), 0) for p in xyz], np.float32)[None]
    tags = np.full((1, H, W), 4, np.uint8)
    tags[0, :, 255] = 6
    lut = ops.sem_class_table([4, 6])
    stored = np.zeros((1, 8, 2), np.float32)
    stored[0, 1] = [0, 1]                                          # the point on column 255: class 2, right
    stored[0, 6] = [np.nan, 0]
    got, per = paint_confusion_ref(pts, tags, lut, CAMS[1:2], WINDOW, 3, stored=stored)
    v = ops.paint_confusion_views(got, 1, 3, False, True)
    cnt = dict(zip(ops.PAINT_COUNTERS, v["counters"][0].tolist()))
    assert cnt == dict(points=8, nan=1, roof=1, in_window=4, not_visible=3, not_visible_in_window=1, invalid=0, stored_invalid=1)
    # x = 70 = max_x is outside the window (half open); the roof point is outside the window by definition
    assert per[0]["win"].tolist() == [True, True, False, False, False, False, True, True]
    assert per[0]["cam"].tolist() == [0, 0, -1, -1, -1, 0, 0, -1]
    conf = v["stored"][0, 0]                                       # [range bin][in window][recorded][predicted]
    assert conf[1, 1, 1, 0] == 1                                   # 11.5 m ahead: bin 1, in window, class 1, all-zero row -> 0
    assert conf[2, 1, 2, 2] == 1                                   # 26.5 m on the last column: bin 2, class 2, one-hot -> 2
    assert conf[3, 0, 1, 0] == 1                                   # 70 m: bin 3, outside the window
    assert conf.sum() == 3
    meta = np.array([[8, 0]])                                      # a mismatched frame: no stored scores at all
    got2, _ = paint_confusion_ref(pts, tags, lut, CAMS[1:2], WINDOW, 3, stored=stored, meta=meta)
    v2 = ops.paint_confusion_views(got2, 1, 3, False, True)
    assert v2["stored"].sum() == 0 and v2["counters"][0, 7] == 0 and v2["counters"][0, 0] == 8
    got3, _ = paint_confusion_ref(pts, tags, lut, CAMS[1:2], WINDOW, 3, stored=stored, meta=np.array([[3, 1]]))
    assert got3[0, 0] == 3 and got3[0, 1] == 0                     # rows past the frame's count are not read


def test_window_edges():
    x = np.array([-10, np.nextafter(np.float32(-10), np.float32(-20)), np.nextafter(np.float32(70), np.float32(0)), 70, 5, 5],
                 np.float32)
    y = np.array([0, 0, 0, 0, -40, 40], np.float32)
    pts = np.stack([x, y, np.full(6, -1.0, np.float32), np.zeros(6, np.float32)], 1)[None]
    _, per = paint_confusion_ref(pts, np.zeros((3, H, W), np.uint8), np.zeros(256, np.uint8), CAMS, WINDOW, 2,
                                 stored=np.zeros((1, 6, 1), np.float32))
    assert per[0]["win"].tolist() == [True, False, True, False, True, False]


def test_fma32_rounds_once():
    a = np.float32(1 + 2 ** -12)
    b = np.float32(1 + 2 ** -12)
    c = np.float32(-(1 + 2 ** -11))
    assert fma32(a, b, c) == np.float32(2 ** -24)                  # the product's low bits survive: a plain fp32 mul-add gives 0
    rs = np.random.RandomState(0)
    a, b, c = (rs.randn(100000).astype(np.float32) for _ in range(3))
    exact = a.astype(np.float64) * b + c                           # not exact in general, but fma32 must be its fp32 rounding
    assert np.abs(fma32(a, b, c).astype(np.float64) - exact).max() <= np.abs(exact).max() * 2 ** -23


# ----------------------------------------------------------------------------- host reductions
def test_scores_and_metrics_by_hand():
    from lav_b200.evaluate_paint import PaintScores
    c, ncam = 2, 3
    L = ops.paint_confusion_ints(ncam, c, True, True)
    counts = np.zeros((2, L), np.int64)
    v = ops.paint_confusion_views(counts, ncam, c, True, True)
    v["counters"][0] = [10, 1, 1, 6, 2, 1, 1, 0]
    v["counters"][1] = [5, 0, 0, 4, 1, 1, 0, 0]
    v["online"][0, 0, 0, 1] = [[3, 1], [0, 2]]                     # camera 0, 0-10 m, in window
    v["online"][1, 2, 3, 0] = [[1, 0], [0, 0]]                     # camera 2, 40 m+, outside the window
    v["stored"][0, 0, 0, 1] = [[4, 0], [0, 2]]
    v["agreement"][0, 0] = [[3, 0], [1, 2]]
    s = PaintScores(ncam, c, True, True)
    s.add(counts, np.array([[10, 1], [5, 0]]))
    r = s.summary([0, 4])
    assert r["points"] == dict(points=15, nan=1, roof=1, in_window=10, not_visible=3, not_visible_in_window=2, invalid=1,
                               stored_invalid=0)
    assert r["coverage"] == pytest.approx(8 / 10) and r["mismatched_frames"] == 1
    assert r["online"]["confusion"] == [[4, 1], [0, 2]] and r["online"]["invalid_pixels"] == 1
    assert r["online"]["in_window"]["confusion"] == [[3, 1], [0, 2]]
    assert r["online"]["per_range"]["40m+"]["confusion"] == [[1, 0], [0, 0]]
    assert r["online"]["per_camera"][2]["pixel_accuracy"] == 1.0 and r["online"]["per_camera"][1]["pixel_accuracy"] is None
    assert r["online"]["iou"] == [4 / 5, 2 / 3]
    assert r["stored"]["pixel_accuracy"] == 1.0
    assert r["agreement"]["rate"] == pytest.approx(5 / 6) and r["agreement"]["confusion"] == [[3, 0], [1, 2]]


def test_layout_matches_the_library():
    from lav_b200 import capi
    for ncam in (1, 3, 4):
        for c in (2, 5, 8):
            for on, st in ((1, 0), (0, 1), (1, 1)):
                assert capi.lib().lavb_paint_confusion_ints(ncam, c, on, st) == ops.paint_confusion_ints(ncam, c, on, st)
    assert capi.lib().lavb_paint_confusion_ints(3, 5, 0, 0) == -1 and capi.lib().lavb_paint_confusion_ints(5, 5, 1, 0) == -1


# ----------------------------------------------------------------------------- the dataset's host half
def write_paint_config(path, data_dir, num_plan=3, seg_channels=(4, 6, 7, 10)):
    import yaml
    cfg = dict(data_dir=str(data_dir), percentage_data=1.01, all_towns=True, num_plan=num_plan,
               camera_yaws=[-120, -60, 0, 60, 120], seg_channels=list(seg_channels), camera_x=1.5, camera_z=2.4,
               min_x=-10, max_x=70, min_y=-40, max_y=40)
    with open(path, "w") as f:
        yaml.safe_dump(cfg, f)
    return str(path)


@pytest.fixture(scope="module")
def recording(tmp_path_factory):
    root = tmp_path_factory.mktemp("paintrec")
    synth.record_trajectories(str(root), n_traj=2, n_frames=6, n_points=300, images=True, n_cameras=5)
    return root


def test_dataset_reads_what_it_needs_and_flags_mismatched_frames(recording, tmp_path):
    import shutil
    from lav_b200.datasets import CameraBatchLoader, PaintDataset
    from tests.test_camera_eval_cpu import KeyLog, direct
    root = tmp_path / "rec"
    shutil.copytree(recording, root)
    from lav_b200 import data_paint
    env = data_paint.open_env(str(root / "traj_000"))
    env.put("lidar_sem_00001", np.zeros((299, 4), np.float32).tobytes())         # a stale frame: one row short
    import os
    os.remove(str(root / "traj_001" / "kv" / "lidar_sem_00002"))                  # an interrupted run: no row at all
    cfg = write_paint_config(tmp_path / "p.yaml", root)
    for online, stored in ((True, False), (False, True), (True, True)):
        ds = PaintDataset(cfg, online=online, stored=stored, device="cpu")
        assert len(ds) == 2 * 3 and ds.cams == [0, 1, 2]                          # three painting cameras, not the five yaws
        log = []
        envf = ds.env
        ds.env = lambda traj: KeyLog(envf(traj), log)
        batches = [(b, st) for b, st in CameraBatchLoader(ds, 4, num_workers=2).staged_batches()]
        assert [len(b["points"]) for b, _ in batches] == [4, 2]
        read = {k.rsplit("_", 1)[0] for k in log}
        assert read == ({"lidar", "sem_0", "sem_1", "sem_2"} | ({"rgb_0", "rgb_1", "rgb_2"} if online else set())
                        | ({"lidar_sem"} if stored else set()))
        meta = np.concatenate([b["meta"].numpy() for b, _ in batches])
        assert meta[:, 0].tolist() == [300] * 6
        if stored:
            assert meta[:, 1].tolist() == [1, 0, 1, 1, 1, 0]                      # traj 0 frame 1, traj 1 frame 2
        for j, (traj, i) in enumerate(ds.index):
            b, k = divmod(j, 4)
            batch = batches[b][0]
            lidar = np.frombuffer(data_paint.open_env(ds.paths[traj]).get(f"lidar_{i:05d}"), np.float32).reshape(-1, 4)
            assert np.array_equal(batch["points"][k].numpy(), lidar)
            assert np.array_equal(batch["labels"][k, 2].numpy(), direct(ds.paths[traj], f"sem_2_{i:05d}"))
            if online:
                assert np.array_equal(batch["rgbs"][k, 1].numpy(), direct(ds.paths[traj], f"rgb_1_{i:05d}"))


def test_dataset_rejects_other_image_sizes(recording, tmp_path):
    import shutil
    from lav_b200 import data_paint
    from lav_b200.capi import LavbError
    from lav_b200.datasets import PaintDataset
    root = tmp_path / "rec"
    shutil.copytree(recording, root)
    data_paint.open_env(str(root / "traj_000")).put("sem_1_00000", synth.encode_png(np.zeros((144, 128), np.uint8)))
    ds = PaintDataset(write_paint_config(tmp_path / "p.yaml", root), online=False, stored=True, device="cpu")
    with pytest.raises(LavbError, match="sem_1_00000"):
        ds.prepare(0)
    with pytest.raises(LavbError):
        PaintDataset(write_paint_config(tmp_path / "q.yaml", root), online=False, stored=False, device="cpu")
