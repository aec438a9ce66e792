"""GPU: the uint8 BEV crop kernel (ops.crop_bilinear_u8) against the fp32 crop kernel and F.grid_sample, BEVPlanner.forward on a
uint8 map against the reference golden, the device-side TemporalBEVDataset and its loader, one BEVTrainer step, and a two-step
run of lav_b200.train_bev whose checkpoint then serves as train_full's teacher."""
import json
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F
import yaml

from lav_b200 import ops, synth
from lav_b200.capi import LavbError
from tests.test_bev_train_cpu import PLANNER, _planner

pytestmark = pytest.mark.gpu


def _poses(K, B, gen):
    """K random crop poses: rotations of any angle, scales 0.3 .. 1.2, centres up to 1.6 half-widths out (crops that leave the map)."""
    ang = (torch.rand(K, generator=gen) * 2 - 1) * math.pi
    s = 0.3 + 0.9 * torch.rand(K, generator=gen)
    t = (torch.rand(K, 2, generator=gen) * 2 - 1) * 1.6
    theta = torch.stack([torch.stack([s * torch.cos(ang), -s * torch.sin(ang), t[:, 0]], -1),
                         torch.stack([s * torch.sin(ang), s * torch.cos(ang), t[:, 1]], -1)], -2)
    theta[:4] = torch.tensor([[1.0, 0, 0], [0, 1.0, 0]])                      # identity, exact pixel centres
    theta[4] = torch.tensor([[1.0, 0, 3.0], [0, 1.0, 0]])                     # entirely off the map
    frame = torch.randint(0, B, (K,), generator=gen, dtype=torch.int32)
    return theta, frame


@pytest.mark.parametrize("C", [9, 5, 1])
@pytest.mark.parametrize("S", [192, 37])
def test_crop_u8_bit_identical_to_fp32_kernel(cuda, C, S):
    g = torch.Generator().manual_seed(100 * C + S)
    B, H, W, K = 3, 320, 288, 300
    bev = (torch.rand(B, C, H, W, generator=g) * 256).to(torch.uint8)
    bev[:, :, :5] = torch.randint(0, 2, (B, C, 5, W), generator=g).to(torch.uint8)
    theta, frame = _poses(K, B, g)
    bev_d, theta_d, frame_d = bev.to(cuda), theta.to(cuda), frame.to(cuda)
    out = torch.full((K, C, S, S), float("nan"), device=cuda)                 # canary: every element must be written
    ops.crop_bilinear_u8(bev_d, frame_d, theta_d, S, out=out)
    assert not torch.isnan(out).any()
    feats = torch.zeros(B, H, W, 16, device=cuda)                             # the float copy, zero-padded to 16 channels
    feats[..., :C] = bev_d.permute(0, 2, 3, 1).float()
    want = ops.crop_bilinear(feats, frame_d, theta_d, S)[..., :C].permute(0, 3, 1, 2)
    assert torch.equal(out, want), float((out - want).abs().max())
    grids = F.affine_grid(theta_d, (K, C, S, S), align_corners=True)
    ref = F.grid_sample(bev_d.float()[frame_d.long()], grids, align_corners=True)
    assert float((out - ref).abs().max()) <= 1e-4 * 255
    assert float((out[4]).abs().max()) == 0.0 and float(out.abs().max()) > 0
    assert torch.equal(ops.crop_bilinear_u8(bev_d, frame_d, theta_d, S), out)    # allocating form


def test_crop_u8_clamps_frames_and_rejects_bad_arguments(cuda):
    bev = (torch.rand(2, 9, 64, 64) > 0.5).to(torch.uint8).to(cuda)
    theta = torch.tensor([[[0.5, 0, 0], [0, 0.5, 0]]] * 2, device=cuda)
    a = ops.crop_bilinear_u8(bev, torch.tensor([-5, 7], dtype=torch.int32, device=cuda), theta, 16)
    b = ops.crop_bilinear_u8(bev, torch.tensor([0, 1], dtype=torch.int32, device=cuda), theta, 16)
    assert torch.equal(a, b)
    fi = torch.zeros(2, dtype=torch.int32, device=cuda)
    with pytest.raises(LavbError):
        ops.crop_bilinear_u8(bev.float(), fi, theta, 16)                      # not uint8
    with pytest.raises(LavbError):
        ops.crop_bilinear_u8(bev.permute(0, 1, 3, 2), fi, theta, 16)          # not contiguous
    with pytest.raises(LavbError):
        ops.crop_bilinear_u8(bev[:, :0], fi, theta, 16)                       # C < 1
    with pytest.raises(LavbError):
        ops.crop_bilinear_u8(bev, fi, theta, 1)                               # crop < 2
    with pytest.raises(LavbError):
        ops.crop_bilinear_u8(bev, torch.zeros(65536, dtype=torch.int32, device=cuda), theta[:1].expand(65536, 2, 3), 2)
    with pytest.raises(LavbError):
        ops.crop_bilinear_u8(bev, fi, theta, 16, out=torch.empty(2, 9, 16, 15, device=cuda))
    assert ops.crop_bilinear_u8(bev, fi[:0], theta[:0], 16).shape == (0, 9, 16, 16)


@pytest.mark.parametrize("tag", ["mixed", "none"])
def test_planner_forward_on_uint8_map_matches_reference(cuda, golden_dir, tag):
    gold = np.load(os.path.join(golden_dir, "bev_planner_train.npz"))
    m = _planner(int(gold["seed"])).to(cuda)
    batch = [t.to(cuda) for t in synth.bev_planner_batch(no_vehicles=tag == "none")]
    bev, ego_locs, cmds, nxps, bras, locs, oris, typs = batch
    assert bev.dtype == torch.uint8
    torch.manual_seed(int(gold["fwd_seed"]))
    out = m(bev, ego_locs, locs, oris, nxps, typs)
    for n, got in zip(gold["names_fwd"].tolist(), out):
        want = gold[f"{tag}_{n}"]
        got = got.detach().cpu().numpy()
        assert got.shape == want.shape and got.dtype == np.float32, (n, got.shape, want.shape)
        assert np.abs(got.astype(np.float64) - want).max() <= 2e-4 * (np.abs(want).max() + 1), n


@pytest.fixture(scope="module")
def gold_ds(golden_dir):
    return np.load(os.path.join(golden_dir, "temporal_bev_dataset.npz"))


@pytest.fixture(scope="module")
def bev_config(gold_ds, tmp_path_factory):
    root = tmp_path_factory.mktemp("gpu_bevrec")
    synth.record_trajectories(str(root / "data"), int(gold_ds["n_traj"]), int(gold_ds["n_frames"]), int(gold_ds["seed"]))
    cfg = dict(json.loads(str(gold_ds["config"])), data_dir=str(root / "data"))
    with open(root / "config.yaml", "w") as f:
        yaml.safe_dump(cfg, f)
    return str(root / "config.yaml")


def test_dataset_matches_reference_golden(cuda, gold_ds, bev_config):
    from lav_b200.datasets import TemporalBEVDataset
    ds = TemporalBEVDataset(bev_config, seed=int(gold_ds["seed"]), device=cuda)
    assert len(ds) == len(gold_ds["map_traj"])
    names = ["bev", "ego_locs", "cmd", "nxp", "bra", "locs", "oris", "typs", "num_objs"]
    for k, idx in enumerate(gold_ds["samples"].tolist()):
        ds.gen.manual_seed(int(gold_ds[f"s{k}_torch_seed"]))                  # __getitem__ replays the reference's draws
        for got in (ds.sample(idx, int(gold_ds[f"s{k}_offset"]), float(gold_ds[f"s{k}_angle"])), ds[idx]):
            g = {n: (v.cpu().numpy() if torch.is_tensor(v) else np.asarray(v)) for n, v in zip(names, got)}
            assert g["bev"].dtype == np.uint8 and np.array_equal(g["bev"], gold_ds[f"s{k}_bev"]), (k, int((g["bev"] != gold_ds[f"s{k}_bev"]).sum()))
            for n in ("ego_locs", "nxp", "locs", "oris"):
                assert g[n].shape == gold_ds[f"s{k}_{n}"].shape and np.abs(g[n].astype(np.float64) - gold_ds[f"s{k}_{n}"]).max() <= 1e-5, (k, n)
            for n in ("cmd", "bra", "typs", "num_objs"):
                assert np.array_equal(g[n], gold_ds[f"s{k}_{n}"]), (k, n)
    with pytest.raises(LavbError):                                            # a shift past the 32-pixel margin
        ds.prepare(int(gold_ds["samples"][0]), 33, 0.0)


def test_loader_batches_and_one_trainer_step(cuda, gold_ds, bev_config):
    from lav_b200.datasets import TemporalBEVBatchLoader, TemporalBEVDataset, get_data_loader
    from lav_b200.train import BEVTrainer
    from types import SimpleNamespace
    ds = TemporalBEVDataset(bev_config, seed=int(gold_ds["seed"]), device=cuda)
    a, b = TemporalBEVBatchLoader(ds, 2, seed=3, rank=0, world=2), TemporalBEVBatchLoader(ds, 2, seed=3, rank=1, world=2)
    assert not set(a.shard(0)) & set(b.shard(0)) and set(a.shard(0)) | set(b.shard(0)) == set(range(len(ds)))
    loader = get_data_loader("temporal_bev", SimpleNamespace(config_path=bev_config, seed=3, batch_size=4, device=cuda, num_workers=3))
    assert isinstance(loader, TemporalBEVBatchLoader) and loader.num_workers == 3
    batches = list(loader)
    assert len(batches) == len(loader) == len(ds) // 4
    cfg = json.loads(str(gold_ds["config"]))
    M, T = cfg["max_objs"], cfg["num_plan"] + 1
    shapes = [(4, 9, 320, 320), (4, T, 2), (4,), (4, 2), (4,), (4, M, T, 2), (4, M), (4, M), (4,)]
    dtypes = [torch.uint8, torch.float32, torch.int64, torch.float32, torch.int64, torch.float32, torch.float32, torch.int32, torch.int64]
    for t, s, d in zip(batches[0], shapes, dtypes):
        assert tuple(t.shape) == s and t.dtype == d, (tuple(t.shape), s, t.dtype, d)
    assert set(torch.unique(batches[0][0]).tolist()) <= {0, 1}
    again = list(get_data_loader("temporal_bev", SimpleNamespace(config_path=bev_config, seed=3, batch_size=4, device=cuda,
                                                                 num_workers=1)))
    assert all(torch.equal(x, y) for x, y in zip(batches[0], again[0]))       # the worker count does not change the data
    m = _planner(2021).to(cuda)
    tr = BEVTrainer(m, device=cuda)
    before = [p.detach().clone() for p in m.parameters()]
    loss, parts = tr.train_bev(*batches[0], other_weight=tr.other_weight(4000))
    assert math.isfinite(float(loss)) and all(math.isfinite(float(v)) for v in parts.values())
    assert any(not torch.equal(p0, p) for p0, p in zip(before, m.parameters()))


def test_train_bev_two_steps_feeds_train_full(cuda, gold_ds, bev_config, tmp_path):
    import bench
    from lav_b200 import train_bev, train_full
    from lav_b200.heads import BEVPlanner
    cfg = yaml.safe_load(open(bev_config))
    cfg.update(crop_size=96, feature_x_jitter=1.5, feature_angle_jitter=20, num_cmds=6, num_plan_iter=5, branch_weights=[5, 5, 5, 1, 1, 1],
               cmd_weight=0.1, cmd_smooth=0.2, use_others_to_train=True)
    path = tmp_path / "bev.yaml"
    yaml.safe_dump(cfg, open(path, "w"))
    torch.manual_seed(2021)
    init = train_bev.build_planner(cfg).state_dict()
    train_bev.main(["--config-path", str(path), "--batch-size", "2", "--max-steps", "2", "--num-per-log", "1", "--num-workers", "2",
                    "--save-dir", str(tmp_path / "ckpt")])
    sd = torch.load(tmp_path / "ckpt" / "bev_1.th")
    m = BEVPlanner(**PLANNER)
    m.load_state_dict(sd, strict=True)
    assert any(v.is_floating_point() and not torch.equal(v, init[k]) for k, v in sd.items() if "running" not in k)

    # the checkpoint is a teacher for train_full
    (_, lid, uni, _), _ = bench.build_models()
    full = yaml.safe_load(open(bev_config))
    full.update(seg_channels=[4, 6, 7, 10], max_lidar_points=2000, camera_x=1.5, camera_z=2.4, stack_loc_jitter=0.4, stack_ori_jitter=0.1,
                num_features=[64, 64], backbone="cnn", crop_size=96, feature_x_jitter=1.5, feature_angle_jitter=20, num_cmds=6,
                num_plan_iter=5, point_painting=True, bev_model_dir=str(tmp_path / "ckpt" / "bev_1.th"))
    for name, mod in (("lidar_model_dir", lid), ("uniplanner_dir", uni)):
        torch.save(mod.state_dict(), tmp_path / f"{name}.th")
        full[name] = str(tmp_path / f"{name}.th")
    fpath = tmp_path / "full.yaml"
    yaml.safe_dump(full, open(fpath, "w"))
    _, up = train_full.build_models(yaml.safe_load(open(fpath)), motion_only=True)
    assert all(torch.equal(up.bev_planner.state_dict()[k], v) for k, v in sd.items())
    train_full.main(["--config-path", str(fpath), "--batch-size", "2", "--max-steps", "1", "--num-per-log", "1", "--motion-only",
                     "--save-dir", str(tmp_path / "full")])
    assert os.path.exists(tmp_path / "full" / "uniplanner_1.th")
