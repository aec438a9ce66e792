"""GPU: ops.paint_confusion against the numpy statement of tests/test_paint_eval_cpu.py (random sweeps with NaN, roof and ragged
rows, 1 / 3 / 4 cameras, C = 2 / 5 / 8, fp32 and h16 features, every rejection), the painting kernels' visibility against the same
statement, and lav_b200.evaluate_paint on synthetic recordings: online against stored after data_paint, a known-answer
recording, the statement per batch at two batch sizes with a stale frame, its CLI, and the released seg weights when present."""
import ctypes as C
import json
import shutil

import numpy as np
import pytest
import torch

from lav_b200 import capi, ops, synth
from lav_b200 import point_painting as PP
from lav_b200.capi import LavbError
from tests import test_paint_eval_cpu as R
from tests import util

pytestmark = pytest.mark.gpu

# the fp32 fmaf chain of 16 products against fp64: a point whose top two fp64 logits lie within this fraction of its logit scale
# may take either class (the seg_confusion test's bound and budget)
KERNEL_TIE_REL = 1e-5
TIE_BUDGET = 1e-3

YAWS = {1: [0], 3: [-60, 0, 60], 4: [-60, 0, 60, 180]}


def random_case(F, N, c, ncam, half, seed, dev, online=True, stored=True):
    rs = np.random.RandomState(seed)
    cams = np.stack([cv.packed() for cv in PP.make_converters(1.5, 2.4, yaws=YAWS[ncam])])
    pts = np.full((F, N, 4), np.nan, np.float32)
    rows = rs.randint(0, N + 1, F)
    rows[0] = N
    if F > 2:
        rows[1] = 0                                                   # an empty sweep
    for f in range(F):
        p = synth.lidar_sweep(int(rows[f]), seed=seed * 1000 + f, tag="pe").numpy() if rows[f] else np.zeros((0, 4), np.float32)
        k = min(len(p), 40)
        p[:k, :3] = np.array([-1.2, 0.0, -1.25]) + rs.uniform(-0.3, 0.3, (k, 3)) * [1, 1, 0.5]   # roof returns
        p[k:k + 5, rs.randint(0, 3)] = np.nan                                                   # NaN rows
        pts[f, :rows[f]] = p
    meta = np.stack([rows, rs.rand(F) > 0.2], 1).astype(np.int32)
    tags = rs.choice([0, 4, 6, 7, 10, 12, 22, 255], (F * ncam, 288, 256)).astype(np.uint8)
    lut = ops.sem_class_table(list(rs.choice(np.arange(1, 23), c - 1, replace=False)))
    feat = table = st = None
    if online:
        feat = rs.randn(F * ncam, 144, 128, 16).astype(np.float32)
        table = np.zeros(520, np.float32)
        table[:512].reshape(2, 2, 16, 8)[..., :c] = rs.randn(2, 2, 16, c) * 0.5
        table[512:512 + c] = rs.randn(c) * 0.1
        if half:
            feat = torch.from_numpy(feat).to(ops.h16()).float().numpy()         # the values the kernel reads
    if stored:
        prob = rs.dirichlet(np.ones(c), (F, N))
        st = (prob[..., 1:] * (1 - prob[..., :1])).astype(np.float32)
        st[rs.rand(F, N) < 0.2] = 0                                        # unseen when painted
        st[rs.rand(F, N) < 0.01, 0] = np.nan
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    dev_feat = None if feat is None else t(feat).to(ops.h16() if half else torch.float32)
    return dict(points=pts, meta=meta, tags=tags, lut=lut, cams=cams, feat=feat, table=table, stored=st), \
        dict(points=t(pts), meta=t(meta), tags=t(tags), feat=dev_feat, table=t(table), stored=t(st))


def check_against_statement(got, h, c, rel=KERNEL_TIE_REL):
    """counts equal the statement's, except that a point whose top two fp64 logits lie within rel x its scale may sit in either
    class's bin of its recorded row (online confusion) or of its stored column (agreement); those are counted and held to the
    budget.  -> (number of near-tie points, number of visible points)."""
    ncam = len(h["cams"])
    want, per = R.paint_confusion_ref(h["points"], h["tags"], h["lut"], h["cams"], R.WINDOW, c, feat=h["feat"], table=h["table"],
                                      stored=h["stored"], meta=h["meta"])
    online, stored = h["feat"] is not None, h["stored"] is not None
    gv = ops.paint_confusion_views(got.astype(np.int64), ncam, c, online, stored)
    wv = ops.paint_confusion_views(want, ncam, c, online, stored)
    assert np.array_equal(gv["counters"], wv["counters"])
    if stored:
        assert np.array_equal(gv["stored"], wv["stored"])
    n_close = 0
    vis = sum(int((d["cam"] >= 0).sum()) for d in per)
    if online:
        for d in per:
            top2 = np.sort(d["logits64"], -1)[:, -2:]
            n_close += int((((top2[:, 1] - top2[:, 0]) <= rel * d["scale"].max(-1)) & (d["online"] >= 0)).sum())
        for key, axis in (("online", -1), ("agreement", -2)):
            if key in gv:
                diff = gv[key] - wv[key]
                assert np.array_equal(gv[key].sum(axis), wv[key].sum(axis))
                assert np.abs(diff).sum() <= 2 * n_close, (key, np.abs(diff).sum(), n_close)
        assert n_close <= TIE_BUDGET * max(vis, 1), (n_close, vis)
    return n_close, vis


CASES = [(1, 120000, 5, 3, True), (7, 30000, 8, 4, False), (64, 3000, 2, 1, True), (7, 5000, 5, 3, False), (7, 5000, 8, 4, True)]


@pytest.mark.parametrize("F,N,c,ncam,half", CASES)
def test_kernel_equals_the_statement(cuda, F, N, c, ncam, half):
    h, d = random_case(F, N, c, ncam, half, seed=F * 7 + c + ncam, dev=cuda)
    got = ops.paint_confusion(d["points"], d["tags"], h["lut"], h["cams"], R.WINDOW, c, feat=d["feat"], table=d["table"],
                              stored=d["stored"], meta=d["meta"]).cpu().numpy()
    assert got.shape == (F, ops.paint_confusion_ints(ncam, c, True, True))
    n_close, vis = check_against_statement(got, h, c)
    assert vis > 0.05 * h["meta"][:, 0].sum()


@pytest.mark.parametrize("online,stored", [(True, False), (False, True)])
def test_one_source_and_no_frame_table(cuda, online, stored):
    h, d = random_case(5, 4000, 5, 3, False, seed=11, dev=cuda, online=online, stored=stored)
    got = ops.paint_confusion(d["points"], d["tags"], h["lut"], h["cams"], R.WINDOW, 5, feat=d["feat"], table=d["table"],
                              stored=d["stored"], meta=d["meta"]).cpu().numpy()
    check_against_statement(got, h, 5)
    h["meta"] = None                                                    # every row of every frame, stored rows scored
    got = ops.paint_confusion(d["points"], d["tags"], h["lut"], h["cams"], R.WINDOW, 5, feat=d["feat"], table=d["table"],
                              stored=d["stored"]).cpu().numpy()
    check_against_statement(got, h, 5)


def test_exact_integer_logits_give_equal_counts(cuda):
    """integer features and weights: every logit is exact, ties are frequent and go to the lower class; counts bit-equal."""
    h, d = random_case(3, 6000, 5, 3, False, seed=5, dev=cuda)
    rs = np.random.RandomState(3)
    h["feat"] = rs.randint(-2, 3, h["feat"].shape).astype(np.float32)
    h["table"] = np.zeros(520, np.float32)
    h["table"][:512].reshape(2, 2, 16, 8)[..., :5] = rs.randint(-1, 2, (2, 2, 16, 5))
    d["feat"], d["table"] = torch.from_numpy(h["feat"]).to(cuda), torch.from_numpy(h["table"]).to(cuda)
    got = ops.paint_confusion(d["points"], d["tags"], h["lut"], h["cams"], R.WINDOW, 5, feat=d["feat"], table=d["table"],
                              stored=d["stored"], meta=d["meta"]).cpu().numpy()
    want, _ = R.paint_confusion_ref(h["points"], h["tags"], h["lut"], h["cams"], R.WINDOW, 5, feat=h["feat"], table=h["table"],
                                    stored=h["stored"], meta=h["meta"])
    assert np.array_equal(got, want)


def test_malformed_calls_write_nothing(cuda):
    h, d = random_case(4, 1000, 5, 3, False, seed=9, dev=cuda)
    L = ops.paint_confusion_ints(3, 5, True, True)
    out = torch.full((4, L), 0x5A5A5A5A, dtype=torch.int32, device=cuda)
    sentinel = out.clone()
    lib = capi.lib()
    p = lambda t, off=0: C.c_void_p(t.data_ptr() + off)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    bad_lut = h["lut"].copy()
    bad_lut[200] = 5
    other16 = capi.BF16 if ops.h16() == torch.float16 else capi.F16
    calls = [dict(c=1), dict(c=9), dict(ncam=0), dict(ncam=5), dict(h=287), dict(w=0), dict(frames=65536), dict(frames=-1),
             dict(n=-1), dict(lut=bad_lut), dict(dtype=7), dict(dtype=other16), dict(feat=None, stored=None),
             dict(min_x=70.0), dict(max_y=-40.0), dict(pts=p(d["points"], 4)), dict(feat=p(d["feat"], 4)), dict(out=None),
             dict(pts=None), dict(tags=None), dict(table=None), dict(stored=p(d["stored"], 2)), dict(meta=p(d["meta"], 2)),
             dict(lut=None), dict(cams=None)]
    for bad in calls:
        a = dict(pts=p(d["points"]), frames=4, n=1000, meta=p(d["meta"]), feat=p(d["feat"]), dtype=capi.F32, table=p(d["table"]),
                 tags=p(d["tags"]), lut=h["lut"], stored=p(d["stored"]), cams=h["cams"], ncam=3, c=5, h=288, w=256, min_x=-10.0,
                 max_x=70.0, min_y=-40.0, max_y=40.0, out=p(out))
        a.update(bad)
        host = lambda arr, dt: None if arr is None else np.ascontiguousarray(arr, dt).ctypes.data_as(C.c_void_p)
        code = lib.lavb_paint_confusion(a["pts"], a["frames"], a["n"], a["meta"], a["feat"], a["dtype"], a["table"], a["tags"],
                                        host(a["lut"], np.uint8), a["stored"], host(a["cams"], np.float32), a["ncam"], a["c"],
                                        a["h"], a["w"], a["min_x"], a["max_x"], a["min_y"], a["max_y"], a["out"], stream)
        assert code != 0, bad
        torch.cuda.synchronize()
        assert torch.equal(out, sentinel), bad
    with pytest.raises(LavbError):
        ops.paint_confusion(d["points"], d["tags"], bad_lut, h["cams"], R.WINDOW, 5, feat=d["feat"], table=d["table"], out=out)
    with pytest.raises(LavbError):
        ops.paint_confusion(d["points"], d["tags"], h["lut"], h["cams"], R.WINDOW, 5, stored=d["stored"][:, :, :3].contiguous(),
                            out=out)
    assert torch.equal(out, sentinel)
    assert lib.lavb_paint_confusion(p(d["points"]), 0, 1000, p(d["meta"]), p(d["feat"]), capi.F32, p(d["table"]), p(d["tags"]),
                                    h["lut"].ctypes.data_as(C.c_void_p), p(d["stored"]), h["cams"].ctypes.data_as(C.c_void_p), 3,
                                    5, 288, 256, -10.0, 70.0, -40.0, 40.0, p(out), stream) == 0
    torch.cuda.synchronize()
    assert torch.equal(out, sentinel)                                           # frames = 0 writes nothing either
    ops.paint_confusion(d["points"][:, :0].contiguous(), d["tags"], h["lut"], h["cams"], R.WINDOW, 5, feat=d["feat"],
                        table=d["table"], stored=d["stored"][:, :0].contiguous(), out=out)
    assert not out.any()                                                        # no points: every element written, all zero
    out.fill_(0x5A5A5A5A)
    ops.paint_confusion(d["points"], d["tags"], h["lut"], h["cams"], R.WINDOW, 5, feat=d["feat"], table=d["table"],
                        stored=d["stored"], meta=d["meta"], out=out)
    assert not (out == 0x5A5A5A5A).any() and int(out[:, 0].sum()) == int(h["meta"][:, 0].sum())


def test_painting_kernels_see_what_the_statement_sees(cuda):
    """project_hit moved into its own header: the painting kernels' visibility is the statement's, point for point (a painted
    row is zero exactly when no camera sees the point: softmax probabilities of moderate logits are never 0)."""
    h, d = random_case(3, 20000, 5, 3, True, seed=21, dev=cuda, stored=False)
    pts = torch.nan_to_num(d["points"], nan=0.0)                          # the painting kernels take no NaN rows
    out = torch.empty((3, 20000, 4), device=cuda)
    ops.paint_deconv_batched(pts, d["feat"], 5, d["table"], h["cams"], 0, out, (288, 256))
    seen = (out.abs().sum(-1) != 0).cpu().numpy()
    ones = torch.ones((3, 1, 288, 256), device=cuda)
    flat = ops.paint(pts[0].contiguous(), ones, h["cams"], mode=0).cpu().numpy()
    p = np.nan_to_num(h["points"], nan=0.0)
    for f in range(3):
        cam, _, _ = R.project_ref(h["cams"], p[f, :, 0], p[f, :, 1], p[f, :, 2])
        assert np.array_equal(seen[f], cam >= 0), f
        if f == 0:
            assert np.array_equal(flat[:, 0] == 1, cam >= 0)


# ----------------------------------------------------------------------------- the evaluator
@pytest.fixture(scope="module")
def recording(tmp_path_factory):
    root = tmp_path_factory.mktemp("paintrec")
    synth.record_trajectories(str(root), n_traj=2, n_frames=9, n_points=3000, images=True, n_cameras=3)
    return root


def copy_of(recording, tmp_path):
    dst = tmp_path / "rec"
    shutil.copytree(recording, dst)
    return dst


def dataset(root, tmp_path, cuda, online, stored):
    from lav_b200.datasets import PaintDataset
    return PaintDataset(R.write_paint_config(tmp_path / "p.yaml", root), online=online, stored=stored, device=cuda)


def run(seg, ds, batch_size, precision="f16"):
    from lav_b200.evaluate_paint import evaluate_paint
    seen = []
    on_batch = lambda b, feat, counts: seen.append(dict(points=b["points"].cpu().numpy(), meta=b["meta"].cpu().numpy(),
                                                        tags=b["labels"].cpu().numpy().reshape(-1, 288, 256),
                                                        stored=b["stored"].cpu().numpy() if "stored" in b else None,
                                                        feat=None if feat is None else feat.float().cpu().numpy(),
                                                        counts=counts))
    return evaluate_paint(seg, ds, batch_size=batch_size, precision=precision, num_workers=2, on_batch=on_batch), seen


def test_evaluate_paint_per_batch_and_batch_sizes_with_a_stale_frame(cuda, recording, tmp_path):
    from lav_b200 import data_paint
    root = copy_of(recording, tmp_path)
    data_paint.open_env(str(root / "traj_001")).put("lidar_sem_00002", np.zeros((2999, 4), np.float32).tobytes())
    sm, _ = util.seg_model()
    ds = dataset(root, tmp_path, cuda, True, True)
    res, seen = run(sm, ds, 4)                                          # 12 frames: 4 + 4 + 4
    assert [len(s["points"]) for s in seen] == [4, 4, 4] and res["samples"] == 12 and res["mismatched_frames"] == 1
    table = sm.erfnet._plan_get(cuda, sm.erfnet._build)[2].cpu().numpy()
    cams = np.stack([cv.packed() for cv in ds.converters])
    lut = ops.sem_class_table([4, 6, 7, 10])
    for s in seen:
        h = dict(points=s["points"], meta=s["meta"], tags=s["tags"], lut=lut, cams=cams, feat=s["feat"], table=table,
                 stored=s["stored"])
        check_against_statement(s["counts"], h, 5)
    assert sum(int((s["meta"][:, 1] == 0).sum()) for s in seen) == 1
    res5, seen5 = run(sm, ds, 5)                                        # 12 = 5 + 5 + 2
    assert [len(s["points"]) for s in seen5] == [5, 5, 2]
    assert res5 == res
    assert res["points"]["points"] == 12 * 3000 and 0 < res["coverage"] < 1
    v = res["online"]
    assert sum(map(sum, v["confusion"])) + v["invalid_pixels"] == 12 * 3000 - res["points"]["not_visible"] - res["points"]["nan"]


@pytest.mark.parametrize("precision", ["f16", "fp32"])
def test_online_equals_stored_after_data_paint(cuda, recording, tmp_path, precision):
    from lav_b200.data_paint import PointPaintDataset, paint_dataset
    root = copy_of(recording, tmp_path)
    sm, _ = util.seg_model()
    sm.set_precision(precision)
    pp = PointPaintDataset(str(root))
    assert paint_dataset(pp, sm, frames_per_batch=4, device=cuda) == 18
    pp.close()
    res, _ = run(sm, dataset(root, tmp_path, cuda, True, True), 4, precision)
    agree = np.array(res["agreement"]["confusion"])
    off = int(agree.sum() - np.trace(agree))
    assert res["mismatched_frames"] == 0 and agree.sum() > 0
    assert off <= TIE_BUDGET * agree.sum(), (off, agree.sum())
    on, st = np.array(res["online"]["confusion"]), np.array(res["stored"]["confusion"])
    assert np.abs(on - st).sum() <= 2 * off and res["online"]["invalid_pixels"] == res["stored"]["invalid_pixels"] == 0
    assert len(np.unique(np.nonzero(agree)[0])) > 1                                 # the seeded model paints several classes


def one_hot_rows(root, ds):
    """the known answer: lidar_sem of every frame written as the one-hot recorded class at the point's pixel (all zero for the
    background and for points no camera sees), through the statement's projection."""
    from lav_b200 import data_paint
    from lav_b200.datasets import load_img
    lut = ops.sem_class_table(ds.seg_channels)
    cams = np.stack([cv.packed() for cv in ds.converters])
    for path in ds.paths:
        env = data_paint.open_env(path)
        for i in range(int(env.get("len"))):
            p = np.frombuffer(env.get(f"lidar_{i:05d}"), np.float32).reshape(-1, 4)
            tags = np.stack([load_img(env, f"sem_{c}", i) for c in range(3)])
            cam, u, v = R.project_ref(cams, p[:, 0], p[:, 1], p[:, 2])
            cls = np.where(cam >= 0, lut[tags[np.maximum(cam, 0), v, u]], 0)
            rows = np.zeros((len(p), 4), np.float32)
            rows[cls > 0, cls[cls > 0] - 1] = 1
            env.put(f"lidar_sem_{i:05d}", rows.tobytes())


def test_known_answer_recording(cuda, recording, tmp_path):
    from lav_b200 import data_paint
    from lav_b200.datasets import load_img
    root = copy_of(recording, tmp_path)
    ds = dataset(root, tmp_path, cuda, False, True)
    one_hot_rows(root, ds)
    res, seen = run(None, ds, 4)
    conf = np.array(res["stored"]["confusion"])
    assert conf.sum() > 0 and conf.sum() == np.trace(conf) and res["stored"]["pixel_accuracy"] == 1.0
    assert res["precision"] is None and "online" not in res and "agreement" not in res
    # camera 1's recorded tags shifted right by one column: the score drops exactly where the statement says
    for path in ds.paths:
        env = data_paint.open_env(path)
        for i in range(int(env.get("len"))):
            img = load_img(env, "sem_1", i)
            env.put(f"sem_1_{i:05d}", synth.encode_png(np.ascontiguousarray(np.roll(img, 1, axis=1))))
    shifted, seen2 = run(None, dataset(root, tmp_path, cuda, False, True), 4)
    cams = np.stack([cv.packed() for cv in ds.converters])
    want = np.zeros_like(conf)
    for s in seen2:
        got, _ = R.paint_confusion_ref(s["points"], s["tags"], ops.sem_class_table([4, 6, 7, 10]), cams, R.WINDOW, 5,
                                       stored=s["stored"], meta=s["meta"])
        want += ops.paint_confusion_views(got, 3, 5, False, True)["stored"].sum((0, 2, 3))[1]
        assert np.array_equal(s["counts"], got)
    sc = np.array(shifted["stored"]["per_camera"][1]["confusion"])
    assert np.array_equal(sc, want) and sc.sum() > np.trace(sc)
    assert shifted["stored"]["per_camera"][0] == res["stored"]["per_camera"][0]
    assert shifted["stored"]["pixel_accuracy"] < 1.0


def test_cli_writes_json(cuda, recording, tmp_path):
    from lav_b200 import evaluate_paint
    sm, sd = util.seg_model()
    torch.save(sd, tmp_path / "seg.th")
    cfg = R.write_paint_config(tmp_path / "c.yaml", "unused")
    out = tmp_path / "r.json"
    res = evaluate_paint.main(["--config-path", cfg, "--data-dir", str(recording), "--seg-weights", str(tmp_path / "seg.th"),
                               "--stored", "--batch-size", "5", "--num-workers", "2", "--json", str(out)])
    assert json.load(open(out)) == json.loads(json.dumps(res))
    assert res["samples"] == 12 and "agreement" in res and res["mismatched_frames"] == 0
    only = evaluate_paint.main(["--config-path", cfg, "--data-dir", str(recording), "--stored", "--num-workers", "2"])
    assert "online" not in only and only["samples"] == 12
    with pytest.raises(SystemExit):
        evaluate_paint.parse_args(["--data-dir", str(recording)])


@pytest.mark.skipif(not util.have_real_seg(), reason="the released seg_1 weights are not extracted (oracle/_ref)")
def test_released_seg_weights_on_a_synthetic_recording(cuda, recording, tmp_path):
    sm, _ = util.seg_model(real=True)
    res, seen = run(sm, dataset(recording, tmp_path, cuda, True, False), 6)
    v = res["online"]
    assert sum(map(sum, v["confusion"])) + v["invalid_pixels"] == 12 * 3000 - res["points"]["not_visible"] - res["points"]["nan"]
    assert v["invalid_pixels"] == 0 and all(0 <= (m["pixel_accuracy"] or 0) <= 1 for m in v["per_camera"])
