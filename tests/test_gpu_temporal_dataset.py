"""GPU: the temporal BEV target kernel (ops.bev_targets) against the fixed-point OpenCV restatement, the device-side
TemporalLiDARPaintedDataset against the reference's outputs in tests/golden/temporal_dataset.npz, the batch loader, and a
two-step run of lav_b200.train_full."""
import json
import math
import os

import numpy as np
import pytest
import torch

from lav_b200 import ops, synth
from lav_b200.capi import LavbError
from oracle import dataset_ref as D
from tests.test_temporal_dataset_cpu import write_config

pytestmark = pytest.mark.gpu


def test_bev_targets_bit_identical_to_opencv_chain(cuda):
    """32 samples x 9 planes: jitter +-20 deg, yaw change up to +-0.3 rad, shifts 0 / +-32 / random, frames missing."""
    rs = np.random.RandomState(0)
    B = 32
    src, rows, want = [], [], np.zeros((B, 9, 320, 320), np.uint8)
    for b in range(B):
        jitter = float(rs.uniform(-20, 20))
        n_frames = 1 + b % 3                                                  # 1, 2 or 3 frames present: the rest missing
        groups = [((0, 1, 2), 0.0, (0, 0))]
        for t in range(n_frames):
            yaw = float(rs.uniform(-0.3, 0.3))
            shift = [(0, 0), (32, -32), (-32, 32), (32, 32)][b % 4] if t == 1 else tuple(int(v) for v in rs.uniform(-32.99, 32.99, 2))
            groups.append(((3 + 2 * t, 4 + 2 * t), yaw, shift))
        for dsts, yaw, (dx, dy) in groups:
            planes = ((rs.rand(320, 320, len(dsts)) > 0.8) * 255).astype(np.uint8)
            want[b, list(dsts)] = D.load_bev_channels(planes, yaw, jitter, (dx, dy))
            for c, d in enumerate(dsts):
                rows.append((len(src), b * 9 + d, -yaw * 180 / math.pi, jitter, dx, dy))
                src.append(planes[..., c])
        rows += [(-1, b * 9 + 3 + 2 * t + c, 0.0, 0.0, 0, 0) for t in range(n_frames, 3) for c in (0, 1)]
    out = torch.full((B, 9, 320, 320), 0xAB, dtype=torch.uint8, device=cuda)           # canary
    ops.bev_targets(torch.from_numpy(np.stack(src)).to(cuda), ops.bev_jobs(rows), out)
    got = out.cpu().numpy()
    assert set(np.unique(got).tolist()) <= {0, 1}
    assert np.array_equal(got, want), int((got != want).sum())
    assert want[:, 3:].any() and not want[0::3, 5:].any()                              # planes of missing frames are zeros
    with pytest.raises(LavbError):
        ops.bev_targets(torch.from_numpy(np.stack(src[:1])).to(cuda), ops.bev_jobs([(0, 0, 0.0, 0.0, 33, 0)]))
    with pytest.raises(LavbError):
        ops.bev_targets(torch.from_numpy(np.stack(src[:1])).to(cuda), ops.bev_jobs([(0, 0, 0.0, 0.0, 0, -33)]))


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, "temporal_dataset.npz"))


@pytest.fixture(scope="module")
def config(gold, tmp_path_factory):
    root = tmp_path_factory.mktemp("gpu_rec")
    synth.record_trajectories(str(root / "data"), int(gold["n_traj"]), int(gold["n_frames"]), int(gold["seed"]))
    return write_config(gold, str(root / "data"), root / "config.yaml")


def test_dataset_matches_reference_golden(cuda, gold, config):
    from lav_b200.datasets import TemporalLiDARPaintedDataset
    ds = TemporalLiDARPaintedDataset(config, seed=int(gold["seed"]), device=cuda)
    assert len(ds) == len(gold["map_traj"])
    for k, idx in enumerate(gold["samples"].tolist()):
        jit = gold[f"s{k}_jitters"]
        got = ds.sample(idx, float(gold[f"s{k}_angle"]), [(j[:2], j[2]) for j in jit], torch.Generator().manual_seed(k))
        g = {n: (v.cpu().numpy() if torch.is_tensor(v) else np.asarray(v)) for n, v in zip(
            ["lidar", "num_points", "heatmaps", "sizemaps", "orimaps", "bev", "ego_locs", "cmd", "nxp", "bra", "locs", "oris", "typs",
             "num_objs"], got)}
        w = {n: gold[f"s{k}_{n}"] for n in g}
        assert g["bev"].dtype == np.uint8 and np.array_equal(g["bev"], w["bev"]), (k, int((g["bev"] != w["bev"]).sum()))
        for n in ("heatmaps", "sizemaps", "orimaps", "ego_locs", "nxp", "locs", "oris"):
            assert g[n].shape == w[n].shape and np.abs(g[n].astype(np.float64) - w[n]).max() <= 1e-5, (k, n)
        for n in ("cmd", "bra", "typs", "num_objs", "num_points"):
            assert np.array_equal(g[n], w[n]), (k, n)
        num = int(w["num_points"])
        gl, wl = g["lidar"][:num], w["lidar"][:num]
        assert not g["lidar"][num:].any()
        assert np.array_equal(gl[:, 8:].sum(0), wl[:, 8:].sum(0))                       # rows per stacked frame
        key = lambda a: np.lexsort((a[:, 3], a[:, 8], a[:, 9], a[:, 10]))              # raw intensity is unique within a sweep
        gl, wl = gl[key(gl)], wl[key(wl)]
        assert np.abs(gl[:, :4] - wl[:, :4]).max() < 2e-4                               # fp32 rotation chain vs fp64 numpy
        flips = (np.abs(gl[:, 4:8] - wl[:, 4:8]).max(1) > 1e-6).sum()
        assert flips <= max(2, num // 2000), flips                                      # FOV-boundary flips of the fp32 projection


def test_loader_batches_for_the_trainer(cuda, gold, config):
    import bench
    from lav_b200.datasets import TemporalBatchLoader, TemporalLiDARPaintedDataset
    from lav_b200.train import LAVTrainer
    ds = TemporalLiDARPaintedDataset(config, seed=int(gold["seed"]), device=cuda)
    a, b = TemporalBatchLoader(ds, 2, seed=3, rank=0, world=2), TemporalBatchLoader(ds, 2, seed=3, rank=1, world=2)
    assert np.array_equal(a.shard(0), TemporalBatchLoader(ds, 2, seed=3, rank=0, world=2).shard(0))     # the seed fixes the order
    assert not np.array_equal(a.shard(0), a.shard(1))                                                     # a new order per epoch
    assert not set(a.shard(0)) & set(b.shard(0)) and set(a.shard(0)) | set(b.shard(0)) == set(range(len(ds)))
    loader = TemporalBatchLoader(ds, 4, seed=3)
    batches = list(loader)
    assert len(batches) == len(loader) == len(ds) // 4
    cfg = json.loads(str(gold["config"]))
    P, M, T = cfg["max_lidar_points"], cfg["max_objs"], cfg["num_plan"] + 1
    shapes = [(4, P, 11), (4,), (4, 2, 320, 320), (4, 2, 320, 320), (4, 2, 320, 320), (4, 9, 320, 320), (4, T, 2), (4,), (4, 2), (4,),
              (4, M, T, 2), (4, M), (4, M), (4,)]
    dtypes = [torch.float32, torch.int64, torch.float32, torch.float32, torch.float32, torch.uint8, torch.float32, torch.int64,
              torch.float32, torch.int64, torch.float32, torch.float32, torch.int32, torch.int64]
    for t, s, d in zip(batches[0], shapes, dtypes):
        assert tuple(t.shape) == s and t.dtype == d, (tuple(t.shape), s, t.dtype, d)
    assert set(torch.unique(batches[0][5]).tolist()) <= {0, 1}
    (_, lid, uni, _), _ = bench.build_models()
    tr = LAVTrainer(lid.to(cuda), uni.to(cuda), device=cuda)
    loss, parts = tr.train_lidar(*batches[0])
    assert math.isfinite(float(loss)) and all(math.isfinite(float(v)) for v in parts.values())


def test_train_full_two_steps(cuda, gold, config, tmp_path):
    import yaml
    import bench
    from lav_b200 import train_full
    from lav_b200.heads import UniPlanner, BEVPlanner
    from lav_b200.lidar import LiDARModel
    (_, lid, uni, _), _ = bench.build_models()
    cfg = yaml.safe_load(open(config))
    cfg.update(num_features=[64, 64], backbone="cnn", crop_size=96, feature_x_jitter=1.5, feature_angle_jitter=20, num_cmds=6,
               num_plan_iter=5, point_painting=True)
    for name, m in (("lidar", lid), ("uniplanner", uni), ("bev", uni.bev_planner)):
        torch.save(m.state_dict(), tmp_path / f"{name}.th")
        cfg[f"{name}_model_dir" if name != "uniplanner" else "uniplanner_dir"] = str(tmp_path / f"{name}.th")
    path = tmp_path / "train.yaml"
    yaml.safe_dump(cfg, open(path, "w"))
    train_full.main(["--config-path", str(path), "--batch-size", "2", "--max-steps", "2", "--num-per-log", "1",
                     "--save-dir", str(tmp_path / "ckpt")])
    kw = dict(pixels_per_meter=4, crop_size=96, feature_x_jitter=1.5, feature_angle_jitter=20, x_offset=0,
              y_offset=1 + (-10) / ((70 + 10) / 2), num_cmds=6, num_plan=20, num_plan_iter=5)
    LiDARModel(num_input=16, num_features=[64, 64], backbone="cnn").load_state_dict(
        torch.load(tmp_path / "ckpt" / "lidar_1.th"), strict=True)
    up = UniPlanner(BEVPlanner(num_frame_stack=2, **kw), num_input_feature=384, **kw)
    sd = torch.load(tmp_path / "ckpt" / "uniplanner_1.th")
    up.load_state_dict(sd, strict=True)
    trained = torch.load(tmp_path / "ckpt" / "lidar_1.th")
    moved = [k for k, v in lid.state_dict().items() if v.is_floating_point() and not torch.equal(v.cpu(), trained[k])]
    assert moved, "two Adam steps changed no LiDAR-model parameter"
