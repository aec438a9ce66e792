"""GPU: ops.det_forecast_match against the numpy statement of tests/test_detected_forecast_cpu.py, its agreement with eval_batch's
2 m matches, its argument checks; lav_b200.evaluate --forecast-detected with a ground-truth detector against a per-sample loop on a
synthetic recording; the unchanged default output; the CLI."""
import ctypes as C
import json

import numpy as np
import pytest
import torch

from lav_b200 import ops
from lav_b200.capi import LavbError, lib
from tests import test_detected_forecast_cpu as R
from tests import test_evaluate_cpu as E
from tests import test_forecast_eval_cpu as F
from tests.test_gpu_evaluate import cfg_dir, random_batch, recording, seeded_models  # noqa: F401  (recording is a fixture)
from tests.test_gpu_forecast_eval import batch_sizes

pytestmark = pytest.mark.gpu


def match_inputs(B, T, seed, big=None):
    """packed, actors, offsets, row_offsets, cols, num_objs, locs, ego_locs of B samples: class-1 peaks scattered around vehicle
    centres (some on them, equal scores), 0..15 rows per sample, actors of classes 0 / 1 / 2 in and out of the window, some with
    a track and some without; sample 0 has no row, sample 1 all 15, sample 2 no actor; sample ``big`` holds 1024 actors."""
    rs = np.random.RandomState(seed)
    M, n_det = 24, 15
    counts = rs.randint(0, 21, B)
    if B > 2:
        counts[2] = 0
    if big is not None:
        counts[big] = 1024
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    actors = np.zeros((offsets[-1], 6), np.float32)
    actors[:, 0] = rs.uniform(-35, 5, len(actors))
    actors[:, 1] = rs.uniform(-10, 50, len(actors))
    actors[::5, :2] = np.round(actors[::5, :2] * 4) / 4
    actors[:, 2:5] = rs.uniform(0, 3, (len(actors), 3))
    actors[:, 5] = rs.choice([0, 1, 1, 1, 2], len(actors))
    packed = np.zeros((B, 7, 2 * n_det), np.float32)
    packed[:, 0] = -1e5
    packed[:, 6] = 320
    rows, cols = [0], []
    for b in range(B):
        cx, cy = E.centres(actors[offsets[b]:offsets[b + 1]])
        for j in range(2 * n_det):
            if len(cx) and rs.rand() < 0.7:
                g = rs.randint(len(cx))
                x = np.clip(np.round(cx[g] + rs.randint(-12, 13) * rs.rand() ** 2), 0, 319)
                y = np.clip(np.round(cy[g] + rs.randint(-12, 13) * rs.rand() ** 2), 0, 319)
            else:
                x, y = rs.randint(0, 320), rs.randint(0, 320)
            packed[b, :6, j] = (np.round(rs.rand(), 1), y * 320 + x, 2.0, 2.0, 1.0, 0.0)
        n_rows = 0 if b == 0 else n_det if b == 1 else rs.randint(0, n_det + 1)
        mine = np.sort(rs.choice(np.arange(n_det, 2 * n_det), n_rows, replace=False))
        cols += mine.tolist()
        rows.append(rows[-1] + len(mine))
    num_objs = np.minimum(rs.randint(0, M + 1, B), counts).astype(np.int32)
    locs = (rs.randn(B, M, T + 1, 2) * 10).astype(np.float32)
    ego = rs.randn(B, T + 1, 2).astype(np.float32)
    return packed, actors, offsets, np.array(rows, np.int32), np.array(cols, np.int32), num_objs, locs, ego


def to_dev(dev, *arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in arrays]


def run(dev, packed, actors, offsets, rows, cols, num_objs, locs, ego, out=None):
    p, a, l, e = to_dev(dev, packed, actors, locs, ego)
    return ops.det_forecast_match(p, a, offsets, rows, cols, num_objs, l, e, out=out)


def check_equal(got, want):
    for k in ("actor", "flag", "ngt"):
        assert np.array_equal(got[k].numpy(), want[k]), (k, np.argwhere(got[k].numpy() != want[k])[:5])
    for k in ("dist", "target"):
        assert np.array_equal(got[k].numpy(), want[k], equal_nan=True), k


@pytest.mark.parametrize("B", [1, 7, 64, 300])
@pytest.mark.parametrize("t", [10, 20])
def test_det_forecast_match_equals_the_numpy_statement(cuda, B, t):
    inputs = match_inputs(B, t, B + t, big=B // 2 if B > 1 else None)
    k = int(inputs[3][-1])
    got = ops.det_match_views(run(cuda, *inputs).cpu(), B, k, t)
    want = R.match_ref(*inputs)
    check_equal(got, want)
    if B > 1:
        f = want["flag"]
        assert (f == 3).any() and (f == 1).any() and (f == 0).any()


def test_matches_equal_eval_batch_at_2m(cuda):
    """on seeded batches with no class-1 survivor within 4 px of the crop centre, a row is matched exactly when eval_batch matches
    its column at 2 m."""
    from lav_b200.evaluate import detected_rows
    from lav_b200.model_inference import peak_filter
    for B, seed in ((7, 1), (64, 2)):
        seg, gt, packed, actors, offsets, plan, ego = random_batch(B, seed, cuda)
        pk = packed.cpu().numpy()
        keep, x, y, cls = peak_filter(pk, 4)
        near = keep & (cls[None] == 1) & ~((x - 160.0) ** 2 + (y - 280.0) ** 2 > 16)
        pk[:, 0][near] = 0.1                                                    # no survivor at the crop centre
        packed = torch.from_numpy(pk).to(cuda)
        flags = ops.eval_views(ops.eval_batch(seg, gt, packed, actors, offsets, plan, ego).cpu(), B, 30)["flags"].numpy()
        rows = detected_rows(pk, 4, R.CENTRE)
        survive = (flags[:, 15:] & 16) != 0
        assert rows["counts"].tolist() == survive.sum(1).tolist()
        row_offsets = np.concatenate([[0], np.cumsum(rows["counts"])]).astype(np.int32)
        n = np.diff(offsets).astype(np.int32)
        locs, egos = R.labels(B, 1, 20, seed)
        v = ops.det_match_views(ops.det_forecast_match(packed, actors, offsets, row_offsets, rows["col"], n * 0, *to_dev(cuda, locs, egos)).cpu(),
                                B, len(rows["col"]), 20)
        want = (flags[rows["frame"], rows["col"]] >> 2) & 1
        assert np.array_equal(v["flag"].numpy() & 1, want) and want.any() and not want.all()
        assert (v["flag"].numpy() & 2 == 0).all() and v["ngt"].numpy()[:, 0].sum() == 0


def test_det_forecast_match_rejects_malformed_arguments_and_writes_nothing(cuda):
    packed, actors, offsets, rows, cols, num_objs, locs, ego = match_inputs(4, 10, 3)
    size = run(cuda, packed, actors, offsets, rows, cols, num_objs, locs, ego).numel()
    out = torch.full((size,), 0xAB, dtype=torch.uint8, device=cuda)
    k = int(rows[-1])
    assert k > 0
    swap = cols.copy()
    i = int(np.nonzero(np.diff(rows))[0][0])
    if rows[i + 1] - rows[i] >= 2:
        swap[rows[i]], swap[rows[i] + 1] = swap[rows[i] + 1], swap[rows[i]]
    else:
        swap = cols.copy()
        swap[rows[i]] = 31
    bad = [dict(offsets=np.array([0, 3, 2, 5, offsets[-1]], np.int32)),                   # not monotone
           dict(offsets=np.array([0, 1, 2, 3, len(actors) + 1], np.int32)),               # past the actor rows
           dict(offsets=offsets[:-1]),
           dict(rows=np.array([1, rows[1], rows[2], rows[3], k], np.int32)),              # rows must start at 0
           dict(rows=np.array([0, 16, 16, 16, 16], np.int32), cols=np.arange(16, dtype=np.int32) + 14),   # over n_det rows
           dict(cols=np.where(np.arange(k) == 0, 3, cols).astype(np.int32)),             # a class-0 column
           dict(cols=np.where(np.arange(k) == 0, 30, cols).astype(np.int32)),            # past the packed columns
           dict(cols=swap),                                                                 # not ascending
           dict(cols=cols[:-1]), dict(cols=cols.astype(np.int64)),
           dict(num_objs=np.array([0, 0, 25, 0], np.int32)),                              # more tracks than label slots
           dict(num_objs=np.array([0, -1, 0, 0], np.int32)),
           dict(packed=packed[:, :6].copy()), dict(packed=np.zeros((4, 7, 130), np.float32)),   # over 64 peaks per class
           dict(actors=actors[:, :5].copy()), dict(locs=locs[:, :, :, :1].copy()), dict(ego=ego[:, :5].copy()),
           dict(locs=np.zeros((4, 24, 34, 2), np.float32), ego=np.zeros((4, 34, 2), np.float32))]   # over 32 steps
    for kw in bad:
        args = dict(packed=packed, actors=actors, offsets=offsets, rows=rows, cols=cols, num_objs=num_objs, locs=locs, ego=ego)
        args.update(kw)
        with pytest.raises(LavbError):
            run(cuda, out=out, **args)
    with pytest.raises(LavbError):
        run(cuda, packed, actors, offsets, rows, cols, num_objs, locs, ego, out=out[:-8])
    with pytest.raises(LavbError):
        ops.det_forecast_match(*to_dev(cuda, packed), torch.from_numpy(actors), offsets, rows, cols, num_objs, *to_dev(cuda, locs, ego), out=out)
    many = np.array([0, 0, 0, 0, 1025], np.int32)                                           # over 1024 actors in one sample
    with pytest.raises(LavbError):
        run(cuda, packed, np.zeros((1025, 6), np.float32), many, rows, cols, num_objs, locs, ego, out=out)
    p, a, l, e = to_dev(cuda, packed, actors, locs, ego)
    v = ops.det_match_views(out, 4, k, 10)
    ptr = lambda t: C.c_void_p(t.data_ptr())
    ip = lambda x: x.ctypes.data_as(C.c_void_p)
    st, null = C.c_void_p(torch.cuda.current_stream().cuda_stream), C.c_void_p(0)
    dev_ptrs = [ptr(p), ptr(a), ptr(l), ptr(e), ptr(v["actor"]), ptr(v["flag"]), ptr(v["dist"]), ptr(v["target"]), ptr(v["ngt"])]

    def call(d, match_m=2.0, t=10, max_objs=24):
        return lib().lavb_det_forecast_match(d[0], 4, 320, 15, d[1], len(actors), ip(offsets), ip(rows), ip(cols), ip(num_objs), d[2],
                                             d[3], max_objs, t, 4.0, 160.0, 320.0, -40.0, match_m, *d[4:], st)
    for i in range(len(dev_ptrs)):                                                          # each device pointer null in turn
        d = list(dev_ptrs)
        d[i] = null
        assert call(d) != 0
    assert call(dev_ptrs, match_m=0.0) != 0 and call(dev_ptrs, match_m=float("nan")) != 0
    assert call(dev_ptrs, t=0) != 0 and call(dev_ptrs, max_objs=-1) != 0
    d = list(dev_ptrs)
    d[7] = C.c_void_p(v["target"].data_ptr() + 4)                                          # target not 8-byte aligned
    assert call(d) != 0
    torch.cuda.synchronize()
    assert bool((out == 0xAB).all())


# ---------------------------------------------------------------------------------------------------- the evaluator
def perturbed(actors, offsets):
    """the actor table a ground-truth detector sees: every third vehicle of a sample dropped (a miss), one decoy vehicle added
    to every sample where none was recorded (a false positive).  Each sample's table depends on that sample alone, so a batch
    sees the detections a B = 1 loop sees."""
    out, offs = [], [0]
    for b in range(len(offsets) - 1):
        a = actors[offsets[b]:offsets[b + 1]]
        veh = np.cumsum(a[:, 5] == 1) * (a[:, 5] == 1)
        a = a[veh % 3 != 2]
        decoy = np.array([[-14.0, 11.5, 0.3, 2.0, 1.0, 1.0]], np.float32)
        out.append(np.concatenate([a, decoy]))
        offs.append(offs[-1] + len(out[-1]))
    return np.concatenate(out).astype(np.float32), np.array(offs, np.int32)


class GroundTruthDetector:
    """ops.det_peaks replaced by the peaks of det_heatmaps on the scored batch's own actor table (perturbed), as logits, with its
    size and orientation maps: deterministic detections with hits, misses and false positives.  The dataset's launch_batch is
    wrapped to see each batch's table; ``table`` may also be set by hand."""

    def __init__(self, ds, dev):
        self.ds, self.dev, self.table = ds, dev, None

    def __enter__(self):
        self.launch, self.peaks = self.ds.launch_batch, ops.det_peaks

        def launch_batch(st):
            self.table = (st["actors"].numpy().copy(), st["offsets"].numpy().copy())
            return self.launch(st)

        def det_peaks(center, box, ori, **k):
            actors, offsets = perturbed(*self.table)
            assert len(offsets) - 1 == center.shape[0]
            grid = dict(min_x=self.ds.min_x, max_x=self.ds.max_x, min_y=self.ds.min_y, max_y=self.ds.max_y,
                        pixels_per_meter=self.ds.pixels_per_meter)
            heat, size, orim = ops.det_heatmaps(*to_dev(self.dev, actors, offsets), grid)
            nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous()
            return self.peaks(nhwc(torch.logit(heat.clamp(1e-6, 1 - 1e-6))), nhwc(size), nhwc(orim), **k)
        self.ds.launch_batch, ops.det_peaks = launch_batch, det_peaks
        return self

    def __exit__(self, *exc):
        del self.ds.launch_batch
        ops.det_peaks = self.peaks


class Recorder:
    """wraps ops.det_forecast_match and ops.forecast_eval: per batch the match's host inputs and result buffer, and the scores'
    inputs."""

    def __init__(self):
        self.matches, self.scores = [], []

    def __enter__(self):
        self.m, self.f = ops.det_forecast_match, ops.forecast_eval

        def det_forecast_match(packed, actors, offsets, row_offsets, cols, num_objs, locs, ego_locs, grid=None, **k):
            buf = self.m(packed, actors, offsets, row_offsets, cols, num_objs, locs, ego_locs, grid, **k)
            host = lambda t: t.cpu().numpy() if torch.is_tensor(t) else np.asarray(t)
            self.matches.append(([host(x) for x in (packed, actors, offsets, row_offsets, cols, num_objs, locs, ego_locs)], buf))
            return buf

        def forecast_eval(cast, score, target, cmd, out=None):
            self.scores.append([t.cpu().numpy() for t in (cast, score, target, cmd)])
            return self.f(cast, score, target, cmd, out)
        ops.det_forecast_match, ops.forecast_eval = det_forecast_match, forecast_eval
        return self

    def __exit__(self, *exc):
        ops.det_forecast_match, ops.forecast_eval = self.m, self.f


def loop_reference(ds, lid, uni, dev):
    """per sample, at B = 1: sample() with the evaluator's zero draws, forward_batch under the ground-truth detector, the row
    table and the match -> rows (frame-local), columns, match outputs, casts, the detection metres and the labels."""
    from lav_b200.agent import infer_model, math_mode
    from lav_b200.datasets import TemporalBatchLoader
    from lav_b200.evaluate import detected_rows, score_detected
    im = infer_model(lid.to(dev).eval(), uni.to(dev).eval(), "fp32", ds.camera_x, ds.camera_z, dev)
    _, gen = TemporalBatchLoader(ds, 1, ordered=True).generators(0)
    grid = dict(min_x=ds.min_x, max_x=ds.max_x, min_y=ds.min_y, max_y=ds.max_y, pixels_per_meter=ds.pixels_per_meter)
    loop = []
    with GroundTruthDetector(ds, dev) as det, math_mode("fp32"), torch.no_grad():
        for idx in range(len(ds)):
            angle, jit = ds.no_draw()
            lidar, num, _, _, _, _, ego, cmd, nxp, _, locs, _, _, n_obj = ds.sample(idx, angle, jit, gen)
            table = ds.stage_batch([ds.prepare(idx, angle, jit)], torch.Generator())
            det.table = (table["actors"].numpy(), table["offsets"].numpy())
            out = im.forward_batch([lidar[:num]], [int(num)], nxp.float()[None], [cmd])
            h, w = out["features"].shape[1:3]
            rows = detected_rows(out["packed"].cpu().numpy(), im.pixels_per_meter, im.uniplanner.crop_centre(2 * h, 2 * w))
            buf = score_detected(out, rows, table["actors"].to(dev), table["offsets"], locs[None], ego.float()[None], [n_obj], grid)
            v = ops.det_match_views(buf.cpu(), 1, len(rows["col"]), locs.shape[1] - 1)
            loop.append(dict(col=rows["col"], locs=rows["locs"], centre=im.uniplanner.crop_centre(2 * h, 2 * w), ppm=im.pixels_per_meter, cast=torch.cat(out["other_cast_locs"]).float().cpu().numpy(),
                             labels=locs.cpu().numpy(), ego=ego.float().cpu().numpy(),
                             **{k: v[k].numpy().copy() for k in ("actor", "flag", "dist", "target", "ngt")}))
    return loop


def test_evaluate_forecast_detected_with_a_ground_truth_detector(cuda, recording):
    import lav_b200.evaluate as EV
    from lav_b200.datasets import TemporalLiDARPaintedDataset
    from lav_b200.evaluate import detected_rows
    ds = TemporalLiDARPaintedDataset(recording[0], device=cuda)
    n = len(ds)
    lid, uni = seeded_models()
    loop = loop_reference(ds, lid, uni, cuda)
    ppm = float(ds.pixels_per_meter)
    for bs in batch_sizes(n):
        with GroundTruthDetector(ds, cuda), Recorder() as rec:
            result = EV.evaluate(lid, uni, ds, batch_size=bs, precision="fp32", num_workers=4, forecast_detected=True)
        sizes = [min(bs, n - k) for k in range(0, n, bs)]
        assert [len(m[0][2]) - 1 for m in rec.matches] == sizes and len(rec.scores) == len(sizes)
        batches, s0, worst, on_pixel = [], 0, 0.0, 0
        for (inp, buf), scored in zip(rec.matches, rec.scores):
            b, k, t = len(inp[0]), int(inp[3][-1]), inp[6].shape[2] - 1
            v = ops.det_match_views(buf.cpu(), b, k, t)
            check_equal(v, R.match_ref(*inp))                                   # the kernels on what the evaluator fed them
            F_want = F.forecast_eval_ref(*scored)
            assert np.array_equal(v["err"].numpy(), F_want["err"], equal_nan=True)
            assert np.array_equal(scored[2], v["target"].numpy(), equal_nan=True) and (scored[3] == -1).all()
            batches.append((inp[0][np.repeat(np.arange(b), np.diff(inp[3])), 0, inp[4]], v["flag"].numpy(), v["err"].numpy(),
                            v["ngt"].numpy()))
            for i in range(b):                                                  # ... sample for sample, the B = 1 loop
                want, r0, r1 = loop[s0 + i], inp[3][i], inp[3][i + 1]
                assert np.array_equal(inp[4][r0:r1], want["col"])
                mine = detected_rows(inp[0][i:i + 1], want["ppm"], want["centre"])
                assert np.array_equal(mine["col"], want["col"]) and np.array_equal(mine["locs"], want["locs"])
                for key in ("actor", "flag", "dist", "target"):
                    assert np.array_equal(v[key].numpy()[r0:r1], want[key], equal_nan=True), key
                assert np.array_equal(v["ngt"].numpy()[i], want["ngt"][0])
                if r1 > r0:
                    worst = max(worst, float(np.abs(scored[0][r0:r1] - want["cast"]).max()) / (1 + float(np.abs(want["cast"]).max())))
                for r in range(r0, r1):                                         # the frame: detection metres on the track's start
                    if v["flag"].numpy()[r] == 3 and v["dist"].numpy()[r] <= np.sqrt(0.5) / ppm:   # on its actor's pixel
                        on_pixel += 1
                        a = v["actor"].numpy()[r]
                        start = want["labels"][a, 0] - want["ego"][0]
                        assert np.hypot(*(want["locs"][r - r0] - start)) <= np.sqrt(0.5) / ppm + 1e-5
            s0 += b
        assert s0 == n and worst <= 1e-3 and on_pixel > 0, (worst, on_pixel)
        got = result["forecast_detected"]
        assert got == R.reduce_ref(batches)
        print(f"evaluate --forecast-detected fp32, batch {bs}: {got}, largest relative cast difference to the loop {worst}")
        assert got["rows"] > got["matched"] > 0 and got["gt"] >= got["matched"]
        flags = np.concatenate([x[1] for x in batches])
        assert ((flags & 1) == 0).any()


def test_default_and_forecast_outputs_keep_their_keys(cuda, recording):
    import lav_b200.evaluate as EV
    from lav_b200.datasets import TemporalLiDARPaintedDataset
    ds = TemporalLiDARPaintedDataset(recording[0], device=cuda)
    lid, uni = seeded_models()
    with GroundTruthDetector(ds, cuda):
        plain = EV.evaluate(lid, uni, ds, batch_size=4, precision="fp32", num_workers=2)
        fc = EV.evaluate(lid, uni, ds, batch_size=4, precision="fp32", num_workers=2, forecast=True)
        both = EV.evaluate(lid, uni, ds, batch_size=4, precision="fp32", num_workers=2, forecast=True, forecast_detected=True)
    assert "forecast_detected" not in plain and "forecast_detected" not in fc
    assert set(both) == set(fc) | {"forecast_detected"} and set(fc) == set(plain) | {"forecast"}
    assert both["det"]["vehicle"]["n_gt"] == fc["det"]["vehicle"]["n_gt"] and both["det"]["vehicle"]["n_det"] == fc["det"]["vehicle"]["n_det"]
    assert both["forecast"]["other"]["rows"] == fc["forecast"]["other"]["rows"]
    assert both["forecast_detected"]["gt"] <= both["det"]["vehicle"]["n_gt"]


def test_cli_forecast_detected_writes_the_json(cuda, recording, tmp_path):
    import yaml
    from lav_b200 import evaluate as EV
    lid, uni = seeded_models()
    torch.save(lid.state_dict(), tmp_path / "lidar_1.th")
    torch.save(uni.state_dict(), tmp_path / "uniplanner_1.th")
    cfg = yaml.safe_load(open(recording[0]))
    cfg["data_dir"] = "/nonexistent"
    yaml.safe_dump(cfg, open(tmp_path / "c.yaml", "w"))
    r = EV.main(["--config-path", str(tmp_path / "c.yaml"), "--data-dir", cfg_dir(recording), "--lidar-weights",
                 str(tmp_path / "lidar_1.th"), "--uniplanner-weights", str(tmp_path / "uniplanner_1.th"), "--batch-size", "5",
                 "--num-workers", "2", "--forecast-detected", "--json", str(tmp_path / "out.json")])
    got = json.load(open(tmp_path / "out.json"))
    assert got == json.loads(json.dumps(r)) and "forecast" not in got
    d = got["forecast_detected"]                                               # the seeded weights detect nothing above 0.2
    assert d["rows"] == d["matched"] == d["matched_untracked"] == 0 and d["match_m"] == 2.0
    assert d["min_ade"] is None and d["min_fde"] is None and d["top_ade"] is None and d["top_fde"] is None and d["miss_rate"] is None
    assert d["recall"] == d["ap"] == (0.0 if d["gt"] else None)
