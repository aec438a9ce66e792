"""GPU: online painting (lav_b200.evaluate --seg-weights).  ops.lidar_batch_paint bit for bit against its composition,
paint_deconv_batched on each sweep followed by lidar_batch; its refusals; the loader's online batches against the stored path
on a recording painted by data_paint with the same model; evaluate(seg_model=...) on a recording without lidar_sem, against the
stored evaluation, in a sweep and across ranks."""
import ctypes
import os
import shutil
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from lav_b200 import capi, ops, synth
from lav_b200 import point_painting as PP
from lav_b200.capi import LavbError
from tests.test_gpu_sweep_eval import StandIn, seeded_pair
from tests.test_online_paint_cpu import write_recording
from tests.util import canary, is_canary, project_hit32
from tests.util import seg_model as make_seg

pytestmark = pytest.mark.gpu

HW = (288, 256)
YAWS = {1: [0], 3: PP.CAMERA_YAWS, 4: [-60, 0, 60, 180]}


def rot(deg):
    r = np.deg2rad(deg)
    return np.array([[np.cos(r), np.sin(r), 0], [-np.sin(r), np.cos(r), 0], [0, 0, 1]], np.float32)


def batch_inputs(B, n_sweep, n_frames, ncam, c_cls, feat_dtype, angle, seed, max_points):
    """raw (N, 4) rows of B samples of three sweeps (one empty in sample 1), with NaN rows, points behind every camera and dense
    points in the cameras' view; the row table with shuffles, -1 padding and out-of-range rows; sweep records; frame slots (some
    frames shared); features and a deconv table; cams."""
    rs = np.random.RandomState(seed)
    cams = np.stack([c.packed() for c in PP.make_converters(1.5, 2.4, yaws=YAWS[ncam])])
    sizes = [[n_sweep - rs.randint(0, n_sweep // 8 + 1) for _ in range(3)] for _ in range(B)]
    if B > 1:
        sizes[1][1] = 0
    raw, table, rows = [], [], np.full((B, max_points), -1, np.int32)
    r0 = 0
    for b in range(B):
        mine = []
        for t, n in enumerate(sizes[b]):
            p = np.stack([rs.uniform(-20, 60, n), rs.uniform(-50, 50, n), rs.uniform(-4, 3, n), rs.rand(n)], 1).astype(np.float32)
            p[:n // 50, 0] = np.float32(np.nan)
            p[n // 50:n // 25, :3] = (0.0, 0.0, 30.0)                      # above the car: behind every camera's image plane
            raw.append(p)
            a, d = rot(rs.uniform(-5, 5)), rs.uniform(-3, 3, 2)
            table.append((rot(angle).ravel(), a.ravel(), d[0], d[1], t, r0))
            mine.append(np.arange(r0, r0 + n))
            r0 += n
        kept = rs.permutation(np.concatenate(mine))[:max_points - 3]
        rows[b, :len(kept)] = kept
        rows[b, len(kept):len(kept) + 3] = (r0 + 5, -7, 2 ** 31 - 1)        # outside [0, n_raw): zero rows
    sweeps = np.array(table, ops.LIDAR_SWEEP_DTYPE)
    slots = rs.randint(0, n_frames, len(sweeps)).astype(np.int32)
    slots[1::3] = slots[0::3][:len(slots[1::3])]                           # frames shared by several sweeps
    g = torch.Generator().manual_seed(seed)
    feat = (torch.randn((n_frames * ncam, HW[0] // 2, HW[1] // 2, 16), generator=g) * 2).to(feat_dtype)
    deconv = ops.pack_deconv2x2(torch.randn((16, c_cls, 2, 2), generator=g), torch.randn((c_cls,), generator=g))
    return np.concatenate(raw), rows, sweeps, slots, feat, deconv, cams


def composition(raw, rows, sweeps, slots, feat, c_cls, deconv, cams, n_time):
    """paint_deconv_batched on each sweep with its frame's features, then lidar_batch on the painted rows."""
    ncam = len(cams)
    painted = torch.zeros((raw.shape[0], 3 + c_cls), device=raw.device)
    bounds = list(sweeps["row0"]) + [raw.shape[0]]
    for s, f in enumerate(slots.tolist()):
        lo, hi = bounds[s], bounds[s + 1]
        if hi > lo:
            out = torch.empty((1, hi - lo, 3 + c_cls), device=raw.device)
            ops.paint_deconv_batched(raw[lo:hi][None].contiguous(), feat[f * ncam:(f + 1) * ncam].contiguous(), c_cls, deconv, cams,
                                     4, out, HW)
            painted[lo:hi] = out[0]
    return ops.lidar_batch(painted, rows, ops._to_device(sweeps.view(np.uint8), raw.device), cams, HW, n_time), painted


def bits(t):
    return t.contiguous().view(torch.int32).cpu().numpy()


CASES = [  # B, points per sweep, frames, ncam, classes, feature dtype, rotation jitter
    (1, 3000, 1, 3, 5, "h16", 0.0),
    (7, 4000, 5, 1, 2, "fp32", 20.0),
    (7, 4000, 9, 4, 8, "h16", -20.0),
    (32, 40000, 34, 3, 5, "h16", 20.0),
    (32, 40000, 34, 3, 8, "fp32", 0.0),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "-".join(map(str, c)))
def test_kernel_equals_the_composition_bit_for_bit(cuda, case):
    B, n, F_, ncam, C, dt, angle = case
    P = 120000 if n == 40000 else 3 * n
    raw, rows, sweeps, slots, feat, deconv, cams = batch_inputs(B, n, F_, ncam, C, ops.h16() if dt == "h16" else torch.float32,
                                                                angle, CASES.index(case) + 1, P)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    raw_d, rows_d, feat_d, deconv_d = d(raw), d(rows), feat.to(cuda), deconv.to(cuda)
    sweeps_d = ops._to_device(sweeps.view(np.uint8), cuda)
    got = ops.lidar_batch_paint(raw_d, rows_d, sweeps_d, d(slots), feat_d, C, deconv_d, cams, HW, 3)
    want, painted = composition(raw_d, rows_d, sweeps, slots, feat_d, C, deconv_d, cams, 3)
    assert got.shape == want.shape == (B, P, 3 + C + 3)
    assert np.array_equal(bits(got), bits(want))
    g = got.cpu().numpy()
    assert np.isnan(g[..., 0]).any() and (g[..., 4:3 + C] > 0).any() and (g[..., :3] == 0).all(-1).any()
    if n == 40000:                                       # the pixel edges are reached: truncated u, v on 0 and on the last
        cam, u, v = project_hit32(cams, raw[:200000, 0], raw[:200000, 1], raw[:200000, 2], *HW)
        seen = cam >= 0
        assert (u[seen] == 0).any() and (u[seen] == HW[1] - 1).any() and (v[seen] == 0).any() and (v[seen] == HW[0] - 1).any()
    live = (rows >= 0) & (rows < len(raw))
    pre = painted.cpu().numpy()[rows[live]][:, 4:]
    masked = (pre != 0).any(1) & (g[live][:, 4:3 + C] == 0).all(1)
    assert masked.any() == (angle != 0)                  # the re-mask bites only under a rotation


def test_empty_inputs(cuda):
    raw = torch.zeros((0, 4), device=cuda)
    rows = torch.full((2, 5), -1, dtype=torch.int32, device=cuda)
    sweeps = ops._to_device(np.zeros(1, ops.LIDAR_SWEEP_DTYPE).view(np.uint8), cuda)
    slots = torch.zeros(1, dtype=torch.int32, device=cuda)
    feat = torch.zeros((3, 144, 128, 16), device=cuda)
    deconv = torch.zeros(520, device=cuda)
    cams = np.stack([c.packed() for c in PP.make_converters()])
    out = ops.lidar_batch_paint(raw, rows, sweeps, slots, feat, 5, deconv, cams, HW, 3)
    assert out.shape == (2, 5, 11) and (out == 0).all()
    empty = ops.lidar_batch_paint(raw, rows[:0], sweeps, slots, feat, 5, deconv, cams, HW, 3)
    assert empty.shape == (0, 5, 11)


def test_a_bad_frame_slot_gives_nan_columns_and_leaves_the_other_rows(cuda):
    raw, rows, sweeps, slots, feat, deconv, cams = batch_inputs(3, 2000, 4, 3, 5, ops.h16(), 10.0, 11, 6000)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    args = lambda sl: (d(raw), d(rows), ops._to_device(sweeps.view(np.uint8), cuda), d(sl), feat.to(cuda), 5, deconv.to(cuda), cams,
                       HW, 3)
    good = ops.lidar_batch_paint(*args(slots)).cpu().numpy()
    bounds = list(sweeps["row0"]) + [len(raw)]
    for bad in (4, -1, 2 ** 31 - 1):
        sl = slots.copy()
        sl[5] = bad                                                            # sample 1's last sweep (its middle one is empty)
        got = ops.lidar_batch_paint(*args(sl)).cpu().numpy()
        mine = (rows >= bounds[5]) & (rows < bounds[6])
        assert mine.any()
        assert np.array_equal(got[~mine].view(np.int32), good[~mine].view(np.int32))
        assert np.isnan(got[mine][:, 4:8]).all()
        assert np.array_equal(got[mine][:, [0, 1, 2, 3, 8, 9, 10]].view(np.int32), good[mine][:, [0, 1, 2, 3, 8, 9, 10]].view(np.int32))


def test_malformed_calls_are_refused_with_the_output_untouched(cuda):
    raw, rows, sweeps, slots, feat, deconv, cams = batch_inputs(2, 500, 2, 3, 5, torch.float32, 0.0, 3, 1500)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    raw_d, rows_d, sw_d, sl_d, feat_d, dc_d = d(raw), d(rows), ops._to_device(sweeps.view(np.uint8), cuda), d(slots), feat.to(cuda), deconv.to(cuda)
    out = canary((2, 1500, 11), torch.float32, cuda)
    good = dict(raw=raw_d, rows=rows_d, sweeps=sw_d, slots=sl_d, feat=feat_d, n_classes=5, deconv=dc_d, cams=cams, image_hw=HW,
                n_time=3, out=out)
    bad = [dict(raw=raw_d[:, :3].contiguous()), dict(raw=torch.zeros((len(raw) * 4 + 1,), device=cuda)[1:].view(-1, 4)),
           dict(rows=rows_d.long()), dict(slots=sl_d[:-1]), dict(slots=sl_d.cpu()), dict(feat=feat_d[:, :-1]),
           dict(feat=feat_d[:-1]), dict(feat=feat_d.double()), dict(n_classes=1), dict(n_classes=9), dict(deconv=dc_d[:-1]),
           dict(cams=cams[:, :40]), dict(cams=np.concatenate([cams, cams])[:5]), dict(image_hw=(287, 256)), dict(n_time=9),
           dict(out=canary((2, 1500, 10), torch.float32, cuda)), dict(sweeps=sw_d[:-1])]
    for change in bad:
        with pytest.raises(LavbError):
            ops.lidar_batch_paint(**dict(good, **change))
        torch.cuda.synchronize()
        assert is_canary(out).all(), change
    lib, p = capi.lib(), lambda t: ctypes.c_void_p(t.data_ptr())
    h = np.ascontiguousarray(cams)
    base = [p(raw_d), len(raw), p(rows_d), rows_d.numel(), p(sw_d), p(sl_d), len(sweeps), p(feat_d), capi.F32, 2, 5, p(dc_d),
            h.ctypes.data_as(ctypes.c_void_p), 3, 288, 256, 3, p(out), None]
    edits = [(1, -1), (3, -1), (6, -1), (9, -1), (10, 1), (10, 9), (13, 0), (13, 5), (14, 287), (15, 255), (16, 9), (8, 7),
             (0, ctypes.c_void_p(raw_d.data_ptr() + 4)), (7, ctypes.c_void_p(feat_d.data_ptr() + 4)), (2, None), (4, None),
             (5, None), (7, None), (11, None), (12, None), (17, None)]
    for i, v in edits:
        args = list(base)
        args[i] = v
        assert lib.lavb_lidar_batch_paint(*args) != 0, i
        torch.cuda.synchronize()
        assert is_canary(out).all(), i
    assert lib.lavb_lidar_batch_paint(*base) == 0 and capi.lib().lavb_abi_version() == 3
    torch.cuda.synchronize()
    assert not is_canary(out).any()


# ---------------------------------------------------------------------------------------------------- the loader and evaluate
@pytest.fixture(scope="module")
def painted(tmp_path_factory):
    """(config path, the recording without any lidar_sem key, a copy painted by data_paint at f16, one at fp32)."""
    import yaml
    from lav_b200 import data_paint
    root = tmp_path_factory.mktemp("online_paint_gpu")
    cfg = write_recording(str(root))
    data = yaml.safe_load(open(cfg))["data_dir"]
    for t in os.listdir(data):
        for k in os.listdir(os.path.join(data, t, "kv")):
            if k.startswith("lidar_sem_"):
                os.remove(os.path.join(data, t, "kv", k))
    copies = {}
    for prec in ("f16", "fp32"):
        dst = str(root / f"painted_{prec}")
        shutil.copytree(data, dst)
        seg, _ = make_seg()
        seg.set_precision(prec)
        ds = data_paint.PointPaintDataset(dst)
        data_paint.paint_dataset(ds, seg, 1.5, 2.4, device=torch.device("cuda"))
        ds.close()
        copies[prec] = dst
    return cfg, data, copies


@pytest.mark.parametrize("prec", ["f16", "fp32"])
@pytest.mark.parametrize("bs", [4, 5])
def test_loader_online_equals_the_stored_path(cuda, painted, prec, bs):
    from lav_b200.agent import math_mode
    from lav_b200.datasets import TemporalBatchLoader, TemporalLiDARPaintedDataset
    cfg, data, copies = painted
    seg, _ = make_seg(cuda)
    seg.eval().set_precision(prec)
    online = TemporalLiDARPaintedDataset(cfg, device=cuda, overrides=dict(data_dir=data))
    stored = TemporalLiDARPaintedDataset(cfg, device=cuda, overrides=dict(data_dir=copies[prec]))
    assert len(online) == 36
    with math_mode(prec):
        a = list(TemporalBatchLoader(online, bs, drop_last=False, num_workers=3, ordered=True, seg_model=seg).staged_batches())
        b = list(TemporalBatchLoader(stored, bs, drop_last=False, num_workers=3, ordered=True).staged_batches())
    assert len(a) == len(b) == -(-36 // bs)
    for (x, sx), (y, _) in zip(a, b):
        assert len(sx["paint"]["pairs"]) <= bs + 2
        for i, (u, v) in enumerate(zip(x, y)):
            if torch.is_tensor(u):
                assert u.dtype == v.dtype and u.shape == v.shape, i
                assert torch.equal(u.cpu().view(torch.uint8) if u.is_floating_point() else u.cpu(),
                                   v.cpu().view(torch.uint8) if v.is_floating_point() else v.cpu()), i
            else:
                assert u == v, i
        assert (x[0][..., 4:8] != 0).any()


class PaintStandIn(StandIn):
    """StandIn whose ego plan also depends on the painted columns of the batch, so a painting difference changes the result;
    the dataset's launch_batch is wrapped with the loader's segmentation model passed through."""

    def __enter__(self):
        super().__enter__()
        from lav_b200.model_inference import InferModel
        inner, me, launch = InferModel.forward_batch, self, self.launch

        def forward_batch(im, lidars, num_points, nxps, cmds):
            out = inner(im, lidars, num_points, nxps, cmds)
            paint = lidars[:, :, 4:8].double().sum((1, 2)).float()
            out["ego_plan_locs"] = out["ego_plan_locs"] + 1e-3 * paint[:, None, None]
            return out

        def launch_batch(st, *a):
            me.batch = (launch(st, *a), st["actors"].numpy().copy(), st["offsets"].numpy().copy())
            return me.batch[0]
        InferModel.forward_batch, self.ds.launch_batch = forward_batch, launch_batch
        return self


FLAGS = dict(forecast=True, forecast_detected=True, plan_safety=True, det_boxes=True)


def standin_eval(ds, pairs, bs, seg=None):
    import lav_b200.evaluate as E
    with PaintStandIn(ds):
        return E.evaluate_checkpoints(pairs, ds, batch_size=bs, precision="f16", num_workers=3, seg_model=seg, **FLAGS)


def test_evaluate_online_equals_the_stored_evaluation(cuda, painted):
    from lav_b200.datasets import TemporalLiDARPaintedDataset
    cfg, data, copies = painted
    seg, _ = make_seg(cuda)
    online = TemporalLiDARPaintedDataset(cfg, device=cuda, overrides=dict(data_dir=data))
    stored = TemporalLiDARPaintedDataset(cfg, device=cuda, overrides=dict(data_dir=copies["f16"]))
    pair = seeded_pair(3)
    calls = []
    fwd = seg.forward_features_nhwc
    seg.forward_features_nhwc = lambda x: calls.append(x.shape[0]) or fwd(x)
    got = standin_eval(online, [pair], 5, seg)[0]
    n_batches = len(calls)
    want = standin_eval(stored, [pair], 5)[0]
    assert n_batches == 8 and sum(calls) == 3 * got["painting"]["frames"]
    assert got.pop("painting") == dict(frames=sum(calls) // 3, images=sum(calls)) and "painting" not in want
    assert got == want
    zero = TemporalLiDARPaintedDataset(cfg, device=cuda, overrides=dict(data_dir=copies["fp32"]))
    assert standin_eval(zero, [pair], 5)[0]["plan"] != want["plan"]             # the stand-in sees the painting
    calls.clear()
    sweep = standin_eval(online, [pair, seeded_pair(5)], 5, seg)
    assert len(calls) == n_batches                                             # one ERFNet call per batch for both checkpoints
    single = standin_eval(online, [seeded_pair(5)], 5, seg)[0]
    assert sweep[0] == dict(want, painting=sweep[0]["painting"]) and sweep[1] == single


def _worker(rank, world, port, cfg, data, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), LOCAL_RANK=str(rank))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from lav_b200.datasets import TemporalLiDARPaintedDataset
        dev = torch.device("cuda", rank % torch.cuda.device_count())
        torch.cuda.set_device(dev)
        ds = TemporalLiDARPaintedDataset(cfg, device=dev, overrides=dict(data_dir=data))
        res = standin_eval(ds, [seeded_pair(3)], 4, make_seg(dev)[0])
        if rank == 0:
            torch.save(res, out)
    finally:
        dist.destroy_process_group()


def test_two_ranks_equal_one_process(cuda, painted, tmp_path):
    from lav_b200.datasets import TemporalLiDARPaintedDataset
    cfg, data, _ = painted
    one = standin_eval(TemporalLiDARPaintedDataset(cfg, device=cuda, overrides=dict(data_dir=data)), [seeded_pair(3)], 4,
                       make_seg(cuda)[0])
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    out = str(tmp_path / "rank0.pt")
    mp.spawn(_worker, args=(2, port, cfg, data, out), nprocs=2, join=True)
    got = torch.load(out, weights_only=False)
    assert got[0]["samples"] == one[0]["samples"] == 36
    # each rank segments its own shard's frames, so the frames of the shard boundary are segmented twice
    assert got[0]["painting"]["frames"] >= one[0]["painting"]["frames"]
    got[0].pop("painting"), one[0].pop("painting")
    assert got == one
