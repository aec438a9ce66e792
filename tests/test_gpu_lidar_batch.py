"""GPU: the batched training-data kernels against the per-sample path they replace, bit for bit — ops.lidar_batch against
GpuLidarStacker, ops.det_heatmaps against detections_to_heatmap — then TemporalBatchLoader against ds.sample with the loader's
draws replayed, a batch under torch's sync-debug mode, the argument checks, and train_full with --num-workers."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from lav_b200 import ops
from lav_b200.capi import LavbError, lib
from lav_b200.data_pipeline import GpuLidarStacker, detections_to_heatmap
from tests.test_gpu_temporal_dataset import config, gold  # noqa: F401  (fixtures: the golden recording and its config)
from tests.test_lidar_batch_cpu import make_sample

pytestmark = pytest.mark.gpu

SPECIAL = np.array([np.nan, np.inf, -np.inf, -0.0], np.float32)


def bits(t):
    return t.contiguous().view(torch.int32)


def check_batch(stacker, samples, seed=11, ref_samples=None):
    g = torch.Generator().manual_seed(seed)
    want = [stacker(sw, a, j, generator=g) for sw, a, j in (ref_samples or samples)]
    g2 = torch.Generator().manual_seed(seed)
    got, nums = stacker.batch(samples, g2)
    assert nums == [n for _, n in want]
    w = torch.stack([x for x, _ in want])
    diff = (bits(got) != bits(w)).any(-1)
    assert not diff.any(), f"{int(diff.sum())} rows differ, first at {diff.nonzero()[:3].tolist()}"
    assert torch.equal(g.get_state(), g2.get_state())                 # the same draws were taken
    return got, nums


@pytest.mark.parametrize("B", [1, 32])
def test_lidar_batch_matches_stacker(cuda, B):
    """ragged batches: frames 0 and 1 (one or two sweeps), truncation (kept rows > P) and zero padding (far below P)."""
    rs = np.random.RandomState(B)
    P = 6000
    sizes = [[4000], [1500, 1500], [3000, 3000, 3000], [200, 300, 100]]
    samples = [make_sample(rs, sizes[b % 4]) for b in range(B)]
    got, nums = check_batch(GpuLidarStacker(2, 4, P, device=cuda), samples)
    if B > 1:
        assert max(nums) == P and min(nums) < P // 5
        assert not got[3, nums[3]:].any()                              # zero padding is +0.0


def test_lidar_batch_at_training_size(cuda):
    """B = 64 at 30 000-point sweeps and max_lidar_points = 120 000."""
    rs = np.random.RandomState(64)
    samples = [make_sample(rs, [30000] * (1 + min(b % 5, 2))) for b in range(64)]
    check_batch(GpuLidarStacker(2, 4, 120000, device=cuda), samples)


def test_lidar_batch_edge_rows(cuda):
    """an all-roof sweep, an empty sweep, NaN / +-inf / -0.0 in coordinates and painted columns, points no camera sees."""
    rs = np.random.RandomState(5)
    samples = [make_sample(rs, [3000, 0, 2000]), make_sample(rs, [2000, 500]), make_sample(rs, [3000, 3000, 3000], angle=0.0)]
    samples[1][0][1][0][:, :3] = [-1.0, 0.0, -1.2]                     # every point of this sweep on the ego roof
    xyzr, painted = samples[2][0][0][0], samples[2][0][0][1]
    for k, v in enumerate(SPECIAL):
        xyzr[k * 50:(k + 1) * 50, k % 3] = v                           # coordinates
        painted[1000 + k * 50:1000 + (k + 1) * 50, k] = v              # painted columns
    xyzr[2000:2100, :3] = [0.0, 0.0, 80.0]                              # straight up: no camera
    xyzr[2100:2200, :3] = [-30.0, 0.5, -1.0]                            # behind the ego, between the rear cameras
    xyzr[2200:2300, 0] = -0.0                                           # -0.0 + 0.0 = +0.0 after the first rotation (angle 0)
    # the per-sample stacker cannot take a zero-row sweep (ops.roof_filter rejects it); a sweep whose every point is on the
    # roof keeps no row either and draws the same permutation size, so it stands in for the empty sweep in the reference
    roof = (np.array([[-1.0, 0.0, -1.2, 0.5]], np.float32), np.ones((1, 4), np.float32))
    ref = [([roof + sw[2:] if len(sw[0]) == 0 else sw for sw in sweeps], a, j) for sweeps, a, j in samples]
    got, _ = check_batch(GpuLidarStacker(2, 4, 12000, device=cuda), samples, ref_samples=ref)
    assert torch.isnan(got).any() and torch.isinf(got).any()
    unseen = (got[..., 4:8] == 0).all(-1) & (got[..., 8:].sum(-1) == 1)
    assert unseen.sum() >= 100                                         # the FOV re-mask zeroed the painted columns of some rows


def actors(rs, n, typ, lo=-20, hi=20):
    locs = rs.uniform(lo, hi, (n, 2))
    return locs, rs.uniform(-math.pi, math.pi, n), rs.uniform(0.5, 3, (n, 2)), np.full(n, typ, np.float64)


def cat(*parts):
    return tuple(np.concatenate([p[k] for p in parts]) for k in range(4))


def test_det_heatmaps_match_torch(cuda):
    rs = np.random.RandomState(3)
    empty = actors(rs, 0, 0)
    tie = actors(rs, 2, 1)
    tie[0][:] = [-5.0, 3.0]                                             # two coincident vehicles, different boxes and yaws,
    cx, cy = 180, 268                                                   # centred on pixel (row 268, column 180)
    dets = [empty, actors(rs, 7, 0), actors(rs, 9, 1), cat(actors(rs, 4, 0), actors(rs, 5, 1)),
            cat(actors(rs, 3, 0, 200, 300), actors(rs, 3, 1, -300, -200)),                     # outside the window
            cat(tie, actors(rs, 1, 0)), cat(actors(rs, 50, 0), actors(rs, 50, 1)),             # 100 actors in one sample
            cat(actors(rs, 3, 0, -1, 1), actors(rs, 3, 1, -1, 1), actors(rs, 2, 2))]          # crowded; an unknown type
    grid = dict(min_x=-10, max_x=70, min_y=-40, max_y=40, pixels_per_meter=4)
    want = [detections_to_heatmap(*d, device=cuda, **grid) for d in dets]
    table = np.concatenate([np.column_stack([d[0], d[1], d[2], d[3]]) for d in dets]).astype(np.float32)
    offsets = np.cumsum([0] + [len(d[0]) for d in dets]).astype(np.int32)
    got = ops.det_heatmaps(torch.from_numpy(table).to(cuda), torch.from_numpy(offsets).to(cuda), grid)
    for name, g, w in zip(("heat", "size", "ori"), got, zip(*want)):
        w = torch.stack(w)
        bad = bits(g) != bits(w)
        assert not bad.any(), (name, int(bad.sum()), bad.nonzero()[:4].tolist())
    heat, size, orim = got
    assert not heat[0].any() and not heat[1, 1].any() and not heat[2, 0].any() and not heat[4].any()
    # the tie goes to the first of the two coincident vehicles (torch's max(dim) rule)
    cos = torch.cos(torch.tensor(tie[1], dtype=torch.float32, device=cuda))
    assert heat[5, 1, cy, cx] == 1 and cos[0] != cos[1] and orim[5, 0, cy, cx] == cos[0]
    assert size[5, 0, cy, cx] == np.float32(tie[2][0, 0]) * 4


def replay(ds, loader, epoch):
    """the batches of ``loader`` at ``epoch``, stacked from ds.sample with the loader's draws, in sample order."""
    rng, gen = loader.generators(epoch)
    order = loader.shard(epoch)
    out = []
    for k in range(len(loader)):
        samples = [ds.sample(int(i), *ds.draw(rng), generator=gen) for i in order[k * loader.B:(k + 1) * loader.B]]
        cols = list(zip(*samples))
        out.append([torch.stack([torch.as_tensor(v) for v in c]) if torch.is_tensor(c[0]) else torch.tensor(c) for c in cols])
    return out


def assert_batches_equal(got, want):
    for b, (g, w) in enumerate(zip(got, want)):
        assert len(g) == len(w) == 14
        for k, (x, y) in enumerate(zip(g, w)):
            x, y = x.cpu(), y.cpu()
            if y.dtype == torch.float64:
                y = y.float()                                           # ego_locs and nxp: the loader's fp32 copies
            assert x.shape == y.shape and x.dtype == y.dtype, (b, k, x.shape, y.shape, x.dtype, y.dtype)
            if x.dtype == torch.float32:
                assert torch.equal(bits(x), bits(y)), (b, k)
            else:
                assert torch.equal(x, y), (b, k)


@pytest.mark.parametrize("num_workers,rank", [(1, 0), (8, 0), (8, 1)])
def test_loader_batches_equal_sample_replay(cuda, gold, config, num_workers, rank):  # noqa: F811
    from lav_b200.datasets import TemporalBatchLoader, TemporalLiDARPaintedDataset
    ds = TemporalLiDARPaintedDataset(config, seed=int(gold["seed"]), device=cuda)
    loader = TemporalBatchLoader(ds, 2, seed=5, rank=rank, world=2, num_workers=num_workers)
    got = list(loader)
    assert len(got) == len(loader) >= 2
    assert_batches_equal(got, replay(ds, loader, 0))


def test_sample_batch_does_not_synchronise(cuda, gold, config):  # noqa: F811
    from lav_b200.datasets import TemporalLiDARPaintedDataset
    ds = TemporalLiDARPaintedDataset(config, seed=int(gold["seed"]), device=cuda)
    rng = np.random.RandomState(0)
    idxs = list(range(min(4, len(ds))))
    draws = [ds.draw(rng) for _ in idxs]
    ds.sample_batch(idxs, draws, torch.Generator().manual_seed(0))     # warm-up: module loads, pinned pool
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = ds.sample_batch(idxs, draws, torch.Generator().manual_seed(0))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert out[0].shape[0] == len(idxs)


def test_bad_arguments_are_rejected_before_launch(cuda):
    canary = torch.full((2, 8, 11), float("nan"), device=cuda)
    maps = [torch.full((1, 2, 320, 320), 7.0, device=cuda) for _ in range(3)]
    before = [bits(canary).clone()] + [m.clone() for m in maps]
    raw = torch.zeros((10, 8), device=cuda)
    rows = torch.zeros((2, 8), dtype=torch.int32, device=cuda)
    sweeps = torch.zeros((88,), dtype=torch.uint8, device=cuda)
    cams = GpuLidarStacker(device=cuda).cams
    with pytest.raises(LavbError):
        ops.lidar_batch(raw, rows.long(), sweeps, cams, (288, 256), 3, out=canary)
    with pytest.raises(LavbError):
        ops.lidar_batch(raw[:, :3], rows, sweeps, cams, (288, 256), 3)
    with pytest.raises(LavbError):
        ops.lidar_batch(raw, rows, sweeps[:80], cams, (288, 256), 3, out=canary)
    with pytest.raises(LavbError):
        ops.lidar_batch(raw, rows, sweeps, cams, (288, 256), 4, out=canary)     # out shape
    actors = torch.zeros((1, 6), device=cuda)
    offsets = torch.tensor([0, 1], dtype=torch.int32, device=cuda)
    with pytest.raises(LavbError):
        ops.det_heatmaps(actors[:, :5].contiguous(), offsets, out=maps)
    with pytest.raises(LavbError):
        ops.det_heatmaps(actors, offsets.long(), out=maps)
    p = lambda t: C.c_void_p(t.data_ptr())
    cam = np.ascontiguousarray(cams, np.float32).ctypes.data_as(C.c_void_p)
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    L = lib()
    assert L.lavb_lidar_batch(p(raw), 10, 4, p(rows), 16, p(sweeps), 1, cam, 4, 288, 256, 9, p(canary), s) != 0   # 17 columns
    assert L.lavb_lidar_batch(p(raw), 10, 4, p(rows), 16, p(sweeps), 1, cam, 5, 288, 256, 3, p(canary), s) != 0   # 5 cameras
    assert L.lavb_lidar_batch(p(raw), 10, 4, p(rows), -1, p(sweeps), 1, cam, 4, 288, 256, 3, p(canary), s) != 0
    assert L.lavb_lidar_batch(p(raw), 10, 4, p(rows), 16, None, 0, cam, 4, 288, 256, 3, p(canary), s) != 0       # no sweeps
    assert L.lavb_lidar_batch(p(raw), 10, 4, p(rows), 16, p(sweeps), 1, None, 4, 288, 256, 3, p(canary), s) != 0
    hm = [p(m) for m in maps]
    assert L.lavb_det_heatmaps(p(actors), p(offsets), 70000, 320, 320, 4.0, 160.0, 320.0, -40.0, 1.0, *hm, s) != 0
    assert L.lavb_det_heatmaps(p(actors), p(offsets), 1, 0, 320, 4.0, 160.0, 320.0, -40.0, 1.0, *hm, s) != 0
    assert L.lavb_det_heatmaps(p(actors), None, 1, 320, 320, 4.0, 160.0, 320.0, -40.0, 1.0, *hm, s) != 0
    torch.cuda.synchronize()
    assert torch.equal(bits(canary), before[0]) and all(torch.equal(m, b) for m, b in zip(maps, before[1:]))


def test_train_full_with_workers(cuda, gold, config, tmp_path):  # noqa: F811
    import yaml
    import bench
    from lav_b200 import train_full
    (_, lid, uni, _), _ = bench.build_models()
    cfg = yaml.safe_load(open(config))
    cfg.update(num_features=[64, 64], backbone="cnn", crop_size=96, feature_x_jitter=1.5, feature_angle_jitter=20, num_cmds=6,
               num_plan_iter=5, point_painting=True)
    for name, m in (("lidar", lid), ("uniplanner", uni), ("bev", uni.bev_planner)):
        torch.save(m.state_dict(), tmp_path / f"{name}.th")
        cfg[f"{name}_model_dir" if name != "uniplanner" else "uniplanner_dir"] = str(tmp_path / f"{name}.th")
    path = tmp_path / "train.yaml"
    yaml.safe_dump(cfg, open(path, "w"))
    train_full.main(["--config-path", str(path), "--batch-size", "2", "--max-steps", "2", "--num-per-log", "1", "--num-workers", "4",
                     "--save-dir", str(tmp_path / "ckpt")])
    assert (tmp_path / "ckpt" / "lidar_1.th").exists() and (tmp_path / "ckpt" / "uniplanner_1.th").exists()
