"""GPU: ops.det_box_eval against the fp64 statement of tests/test_det_boxes_cpu.py, its agreement with eval_batch, its argument
checks; lav_b200.evaluate --det-boxes with the ground-truth detector of test_gpu_detected_forecast against the statement run on
the same peaks and actor tables, across batch sizes, a B = 1 loop and a two-checkpoint sweep."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from lav_b200 import ops
from lav_b200.capi import LavbError, lib
from tests import test_det_boxes_cpu as R
from tests import test_evaluate_cpu as E
from tests.test_gpu_detected_forecast import GroundTruthDetector, perturbed, to_dev
from tests.test_gpu_evaluate import recording, seeded_models  # noqa: F401  (recording is a fixture)
from tests.test_gpu_forecast_eval import batch_sizes

pytestmark = pytest.mark.gpu

PPM = 4.0


def box_inputs(B, n_det, seed, big=None):
    """packed, actors, offsets of B samples: peaks on and around the actors' centres with their boxes, perturbed sizes and headings
    (some turned by pi), equal scores, and NaN scores, NaN or zero extents, NaN headings, peaks outside the window and class-0
    peaks of size zero; actors of classes 0 / 1 / 2 in and out of the window, some with a NaN heading or a zero extent; sample 2
    has no actor, sample ``big`` holds 1024."""
    rs = np.random.RandomState(seed)
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
    actors[:, 2] = rs.uniform(-4, 4, len(actors))
    actors[:, 3] = rs.uniform(0.2, 3, len(actors))
    actors[:, 4] = rs.uniform(0.2, 1.5, len(actors))
    actors[:, 5] = rs.choice([0, 1, 1, 1, 2], len(actors))
    actors[7::29, 2] = np.nan
    actors[11::31, 3] = 0
    packed = np.zeros((B, 7, 2 * n_det), np.float32)
    packed[:, 0] = -1e5
    packed[:, 6] = 320
    for b in range(B):
        a = actors[offsets[b]:offsets[b + 1]]
        cx, cy = E.centres(a)
        for j in range(2 * n_det):
            if len(a) and rs.rand() < 0.75:
                g = rs.randint(len(a))
                jitter = rs.rand() < 0.5
                x = np.clip(np.round(cx[g] + jitter * rs.randint(-6, 7) * rs.rand() ** 2), 0, 319)
                y = np.clip(np.round(cy[g] + jitter * rs.randint(-6, 7) * rs.rand() ** 2), 0, 319)
                ww, hh = a[g, 3] * PPM * (1 + jitter * rs.uniform(-0.4, 0.4)), a[g, 4] * PPM * (1 + jitter * rs.uniform(-0.4, 0.4))
                t = a[g, 2] + jitter * rs.uniform(-0.5, 0.5) + (rs.rand() < 0.1) * np.pi
                c, s = np.cos(t), np.sin(t)
            else:
                x, y = rs.randint(0, 320), rs.randint(0, 320)
                ww, hh, c, s = rs.uniform(0, 12), rs.uniform(0, 6), rs.uniform(-1, 1), rs.uniform(-1, 1)
            packed[b, :6, j] = (np.round(rs.rand(), 1), y * 320 + x, ww, hh, c, s)
        u = rs.rand(2 * n_det)
        packed[b, 0, u < 0.03] = np.nan
        packed[b, 2, (u >= 0.03) & (u < 0.06)] = np.nan
        packed[b, 3, (u >= 0.06) & (u < 0.09)] = 0
        packed[b, 4, (u >= 0.09) & (u < 0.12)] = np.nan
        packed[b, 5, (u >= 0.12) & (u < 0.14)] = np.nan
        packed[b, 1, (u >= 0.14) & (u < 0.17)] = 280 * 320 + 160                        # on the ego: outside the window
        packed[b, 1, (u >= 0.17) & (u < 0.19)] = 2 * 320 + 5                            # beyond 30 m
        zero = np.nonzero((u[:n_det] >= 0.19) & (u[:n_det] < 0.25))[0]
        packed[b, 2:4, zero] = 0                                                         # class-0 peaks of size zero survive
        packed[b, 0, zero] = 0.9
    return packed, actors, offsets


def run(dev, packed, actors, offsets, out=None):
    p, a = to_dev(dev, packed, actors)
    return ops.det_box_eval(p, a, offsets, out=out)


def check_equal(got, want, tol=1e-12):
    for k in ("flags", "actor", "ngt"):
        assert np.array_equal(got[k].numpy(), want[k]), (k, np.argwhere(got[k].numpy() != want[k])[:5])
    assert np.array_equal(got["score"].numpy(), want["score"], equal_nan=True)
    e, w = got["err"].numpy(), want["err"]
    assert np.array_equal(np.isnan(e), np.isnan(w))
    live = ~np.isnan(w)
    diff = float(np.abs(e[live] - w[live]).max()) if live.any() else 0.0
    assert diff <= tol, diff
    return diff


@pytest.mark.parametrize("B", [1, 7, 64])
@pytest.mark.parametrize("n_det", [15, 30])
def test_det_box_eval_equals_the_statement(cuda, B, n_det):
    packed, actors, offsets = box_inputs(B, n_det, B + n_det, big=B // 2 if B > 1 else None)
    got = ops.det_box_views(run(cuda, packed, actors, offsets).cpu(), B, 2 * n_det)
    want = R.det_box_ref(packed, actors, offsets)
    assert want["near"] == 0                                                            # no IoU within 1e-12 of a threshold
    diff = check_equal(got, want)
    f = want["flags"]
    print(f"B {B}, n_det {n_det}: {int(((f & 16) != 0).sum())} survivors, IoU matches {[int(((f >> k) & 1).sum()) for k in range(3)]}, "
          f"{int(((f >> 3) & 1).sum())} at 2 m, largest error difference {diff:.3g}")
    if B > 1:
        assert ((f & 4) != 0).any() and (((f & 8) != 0) & ((f & 1) == 0)).any() and (((f & 16) != 0) & ((f & 8) == 0)).any()
        h = want["err"][..., 3]
        assert (h > math.pi / 2).any() and np.isnan(h[(f & 8) != 0]).any()


def test_ngt_survivors_and_2m_matches_equal_eval_batch(cuda):
    for B, n_det, seed in ((7, 15, 1), (64, 30, 2)):
        packed, actors, offsets = box_inputs(B, n_det, seed, big=3)
        box = ops.det_box_views(run(cuda, packed, actors, offsets).cpu(), B, 2 * n_det)
        seg = torch.zeros((B, 320, 320, 3), device=cuda)
        gt = torch.zeros((B, 3, 320, 320), dtype=torch.uint8, device=cuda)
        plan, ego = torch.zeros((B, 10, 2), device=cuda), torch.zeros((B, 11, 2), device=cuda)
        p, a = to_dev(cuda, packed, actors)
        ev = ops.eval_views(ops.eval_batch(seg, gt, p, a, offsets, plan, ego).cpu(), B, 2 * n_det)
        f, g = box["flags"].numpy(), ev["flags"].numpy()
        assert np.array_equal(box["ngt"].numpy(), ev["ngt"].numpy())
        assert np.array_equal(f & 16, g & 16) and np.array_equal((f >> 3) & 1, (g >> 2) & 1) and ((f >> 3) & 1).any()


def test_det_box_eval_rejects_malformed_arguments_and_writes_nothing(cuda):
    packed, actors, offsets = box_inputs(4, 15, 3)
    size = run(cuda, packed, actors, offsets).numel()
    out = torch.full((size,), 0xAB, dtype=torch.uint8, device=cuda)
    bad = [dict(offsets=np.array([0, 3, 2, 5, offsets[-1]], np.int32)),                  # not monotone
           dict(offsets=np.array([0, 1, 2, 3, len(actors) + 1], np.int32)),              # past the actor rows
           dict(offsets=offsets[:-1]), dict(offsets=offsets.astype(np.int64)),
           dict(packed=packed[:, :6].copy()), dict(packed=packed[:, :, :29].copy()),
           dict(packed=np.zeros((4, 7, 130), np.float32)),                                 # over 64 peaks per class
           dict(actors=actors[:, :5].copy()), dict(actors=actors.astype(np.float64))]
    for kw in bad:
        args = dict(packed=packed, actors=actors, offsets=offsets)
        args.update(kw)
        with pytest.raises(LavbError):
            run(cuda, out=out, **args)
    with pytest.raises(LavbError):
        run(cuda, packed, actors, offsets, out=out[:-8])
    with pytest.raises(LavbError):
        run(cuda, packed, actors, offsets, out=out.view(torch.int8))
    with pytest.raises(LavbError):
        ops.det_box_eval(*to_dev(cuda, packed), torch.from_numpy(actors), offsets, out=out)   # a host actor table
    many = np.array([0, 0, 0, 0, 1025], np.int32)                                        # over 1024 actors in one sample
    with pytest.raises(LavbError):
        run(cuda, packed, np.zeros((1025, 6), np.float32), many, out=out)
    p, a = to_dev(cuda, packed, actors)
    v = ops.det_box_views(out, 4, 30)
    ptr = lambda t: C.c_void_p(t.data_ptr())
    st, null = C.c_void_p(torch.cuda.current_stream().cuda_stream), C.c_void_p(0)
    ip = offsets.ctypes.data_as(C.c_void_p)
    dev_ptrs = [ptr(p), ptr(a), ptr(v["score"]), ptr(v["flags"]), ptr(v["actor"]), ptr(v["err"]), ptr(v["ngt"])]

    def call(d, n_det=15, ppm=4.0, w=320, b=4, offs=ip):
        return lib().lavb_det_box_eval(d[0], b, w, n_det, d[1], len(actors), offs, ppm, 160.0, 320.0, -40.0, 0.2, *d[2:], st)
    for i in range(len(dev_ptrs)):                                                         # each device pointer null in turn
        d = list(dev_ptrs)
        d[i] = null
        assert call(d) != 0
    assert call(dev_ptrs, n_det=0) != 0 and call(dev_ptrs, n_det=65) != 0 and call(dev_ptrs, ppm=0.0) != 0
    assert call(dev_ptrs, ppm=float("nan")) != 0 and call(dev_ptrs, w=0) != 0 and call(dev_ptrs, b=-1) != 0
    assert call(dev_ptrs, offs=null) != 0
    d = list(dev_ptrs)
    d[5] = C.c_void_p(v["err"].data_ptr() + 4)                                            # err not 8-byte aligned
    assert call(d) != 0
    d = list(dev_ptrs)
    d[3] = C.c_void_p(v["flags"].data_ptr() + 2)
    assert call(d) != 0
    torch.cuda.synchronize()
    assert bool((out == 0xAB).all())
    assert call(dev_ptrs, b=0) == 0                                                        # an empty batch writes nothing
    torch.cuda.synchronize()
    assert bool((out == 0xAB).all())


# ---------------------------------------------------------------------------------------------------- the evaluator
class Recorder:
    """wraps ops.det_box_eval: per batch its host inputs and result buffer."""

    def __init__(self):
        self.calls = []

    def __enter__(self):
        self.f = ops.det_box_eval

        def det_box_eval(packed, actors, offsets, grid=None, **k):
            buf = self.f(packed, actors, offsets, grid, **k)
            self.calls.append((packed.cpu().numpy(), actors.cpu().numpy(), np.asarray(offsets).copy(), buf.cpu()))
            return buf
        ops.det_box_eval = det_box_eval
        return self

    def __exit__(self, *exc):
        ops.det_box_eval = self.f


def run_eval(ds, lid, uni, dev, bs, **k):
    import lav_b200.evaluate as EV
    with GroundTruthDetector(ds, dev), Recorder() as rec:
        result = EV.evaluate(lid, uni, ds, batch_size=bs, precision="fp32", num_workers=2, det_boxes=True, **k)
    return result, rec.calls


def test_evaluate_det_boxes_with_a_ground_truth_detector(cuda, recording):
    from lav_b200.datasets import TemporalLiDARPaintedDataset
    ds = TemporalLiDARPaintedDataset(recording[0], device=cuda)
    n = len(ds)
    lid, uni = seeded_models()
    ppm = float(ds.pixels_per_meter)
    results = {}
    for bs in sorted(set(batch_sizes(n)) | {4, 5, 1}):
        result, calls = run_eval(ds, lid, uni, cuda, bs)
        assert [len(c[2]) - 1 for c in calls] == [min(bs, n - k) for k in range(0, n, bs)]
        batches, kept, dropped, on_pixel, decoys = [], 0, 0, 0, 0
        for packed, actors, offsets, buf in calls:
            b, cols = packed.shape[0], packed.shape[2]
            v = ops.det_box_views(buf, b, cols)
            want = R.det_box_ref(packed, actors, offsets, w=320)
            assert want["near"] == 0
            check_equal(v, want)
            batches.append((want["score"], want["flags"], want["err"], want["ngt"]))
            seen, _ = perturbed(actors, offsets)
            cx, cy = E.centres(actors)
            inside = (E.window_dist(cx, cy) > 2) & (E.window_dist(cx, cy) < 30 * ppm)
            f, who, err = want["flags"], want["actor"][..., 3], want["err"]
            for i in range(b):
                rows = np.arange(offsets[i], offsets[i + 1])
                veh = np.cumsum(actors[rows, 5] == 1) * (actors[rows, 5] == 1)
                matched = set(who[i, cols // 2:][who[i, cols // 2:] >= 0].tolist())
                for a in range(len(rows)):
                    if veh[a] == 0 or not inside[rows[a]]:
                        continue
                    if veh[a] % 3 == 2:                                              # dropped by the detector: never matched
                        assert a not in matched
                        dropped += 1
                    else:
                        others = [(cx[rows[o]], cy[rows[o]]) for o in range(len(rows))
                                  if o != a and actors[rows[o], 5] == 1 and veh[o] % 3 != 2] + [(216.0, 234.0)]   # and the decoy
                        sep = min(math.hypot(cx[rows[a]] - x, cy[rows[a]] - y) for x, y in others)
                        on_map = 1 <= cx[rows[a]] < 319 and 1 <= cy[rows[a]] < 319      # the window runs past the map's edge
                        if on_map and sep > 8 and len(others) <= cols // 2:          # its own peak among n_det: matched at 2 m
                            assert a in matched, (i, a)
                        kept += 1
                for j in range(cols // 2, cols):
                    if not f[i, j] & 8:
                        continue
                    a = who[i, j]
                    A = actors[rows[a]]
                    if (packed[i, 2, j] == np.float32(A[3] * ppm) and packed[i, 3, j] == np.float32(A[4] * ppm)
                            and abs(packed[i, 4, j] - math.cos(A[2])) < 1e-6 and abs(packed[i, 5, j] - math.sin(A[2])) < 1e-6):   # its own box
                        assert err[i, j, 1] <= math.sqrt(2) * 0.5 / ppm + 1e-12 and err[i, j, 2] == 0.0 and err[i, j, 3] < 1e-6
                        on_pixel += 1
                dx, dy = E.centres(np.array([[-14.0, 11.5, 0.3, 2.0, 1.0, 1.0]], np.float32))
                at = [j for j in range(cols // 2, cols) if f[i, j] & 16 and packed[i, 1, j] == float(int(dy[0]) * 320 + int(dx[0]))]
                near = any(math.hypot(cx[r] - dx[0], cy[r] - dy[0]) <= 2 * ppm for r in rows if actors[r, 5] == 1 and inside[r])
                if at and not near:                                                  # the decoy: a false positive
                    assert not f[i, at[0]] & 8
                    decoys += 1
        got = result["det_boxes"]
        assert R.close_dicts(got, R.reduce_ref(batches)), (got, R.reduce_ref(batches))
        assert kept > 0 and dropped > 0 and on_pixel > 0 and decoys > 0, (kept, dropped, on_pixel, decoys)
        print(f"evaluate --det-boxes fp32, batch {bs}: vehicle {got['vehicle']}")
        results[bs] = got
    first = results[1]
    for bs, got in results.items():
        assert got == first, bs                                                        # every batch size: the B = 1 loop


def test_sweep_and_default_outputs(cuda, recording):
    import lav_b200.evaluate as EV
    from lav_b200.datasets import TemporalLiDARPaintedDataset
    ds = TemporalLiDARPaintedDataset(recording[0], device=cuda)
    lid, uni = seeded_models()
    single, _ = run_eval(ds, lid, uni, cuda, 4)
    with GroundTruthDetector(ds, cuda), Recorder() as rec:
        plain = EV.evaluate(lid, uni, ds, batch_size=4, precision="fp32", num_workers=2)
        sweep = EV.evaluate_checkpoints([(lid, uni), seeded_models()], ds, batch_size=4, precision="fp32", num_workers=2, det_boxes=True)
    assert len(rec.calls) == 2 * len(range(0, len(ds), 4))                              # the plain run made no box launch
    assert "det_boxes" not in plain and set(single) == set(plain) | {"det_boxes"}
    assert single["det"] == plain["det"]            # the detector's peaks are exact; the BEV is not bit-reproducible across runs
    for r in sweep:
        assert r["det_boxes"] == single["det_boxes"]
    assert "det boxes, vehicle" in EV.format_result(single) and "det boxes" not in EV.format_result(plain)
