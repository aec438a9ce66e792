"""CPU: the synthetic recorder, the dataset's index mapping and the oracle's TemporalLiDARPaintedDataset.__getitem__ against
tests/golden/temporal_dataset.npz (the reference's own outputs on the same seeded recording, oracle/pin_dataset.py)."""
import json
import os

import numpy as np
import pytest
import torch

from lav_b200 import synth
from lav_b200.data_paint import DirEnv
from lav_b200.datasets import TRAIN_TOWNS, index_trajectories
from oracle import dataset_ref as D
from oracle import lav_ref as O

NAMES = ["lidar", "num_points", "heatmaps", "sizemaps", "orimaps", "bev", "ego_locs", "cmd", "nxp", "bra", "locs", "oris", "typs",
         "num_objs"]


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, "temporal_dataset.npz"))


@pytest.fixture(scope="module")
def recording(gold, tmp_path_factory):
    root = tmp_path_factory.mktemp("rec")
    synth.record_trajectories(str(root), int(gold["n_traj"]), int(gold["n_frames"]), int(gold["seed"]))
    return str(root)


def test_recorder_round_trip(tmp_path):
    paths = synth.record_trajectories(str(tmp_path), 1, 22, seed=5)
    env = DirEnv(paths[0])
    assert int(env.get("len")) == 22 and env.get("town").decode() in TRAIN_TOWNS
    for i in (0, 21):
        ids = np.frombuffer(env.get(f"id_{i:05d}"), np.int32)
        n = len(ids)
        assert np.frombuffer(env.get(f"loc_{i:05d}"), np.float32).shape == (2 * n,)
        assert np.frombuffer(env.get(f"ori_{i:05d}"), np.float32).shape == (n,)
        assert np.frombuffer(env.get(f"bbox_{i:05d}"), np.float32).shape == (2 * n,)
        assert np.frombuffer(env.get(f"type_{i:05d}"), np.uint8).shape == (n,)
        assert ids[0] == ids.min()                                                 # the ego comes first
        assert np.frombuffer(env.get(f"nxp_{i:05d}"), np.float32).shape == (2,)
        pts = np.frombuffer(env.get(f"lidar_{i:05d}"), np.float32).reshape(-1, 4)
        assert np.frombuffer(env.get(f"lidar_sem_{i:05d}"), np.float32).shape == (len(pts) * 4,)
        for c in range(12):
            plane = synth.decode_png(env.get(f"map_{c}_{i:05d}"))
            assert plane.shape == (320, 320) and set(np.unique(plane)) <= {0, 255}
    n0 = len(np.frombuffer(env.get("id_00000"), np.int32))
    assert len(np.frombuffer(env.get("id_00021"), np.int32)) < n0                   # some actors leave
    img = (np.random.RandomState(0).rand(37, 53) * 255).astype(np.uint8)
    assert np.array_equal(synth.decode_png(synth.encode_png(img)), img)


def test_png_writer_without_cv2(monkeypatch):
    import sys
    img = (np.random.RandomState(1).rand(64, 80) > 0.5).astype(np.uint8) * 255
    monkeypatch.setitem(sys.modules, "cv2", None)                                   # import cv2 raises ImportError
    data = synth.encode_png(img)
    assert np.array_equal(synth.decode_png(data), img)


def test_index_mapping_matches_reference(gold, recording):
    cfg = json.loads(str(gold["config"]))
    paths, index = index_trajectories(recording, cfg["percentage_data"], cfg["all_towns"], cfg["num_plan"], int(gold["seed"]))
    got = [(os.path.basename(paths[t]), i) for t, i in index]
    want = list(zip(gold["map_traj"].tolist(), gold["map_index"].tolist()))
    assert got == want
    assert len({t for t, _ in want}) < int(gold["n_traj"])                           # the coin tosses / town filter dropped some


def test_oracle_getitem_reproduces_reference(gold, recording):
    cfg = dict(json.loads(str(gold["config"])), data_dir=recording)
    convs = O.default_converters(cfg["camera_x"], cfg["camera_z"])
    for k in range(len(gold["samples"])):
        env = DirEnv(os.path.join(recording, str(gold[f"s{k}_traj"])))
        jit = gold[f"s{k}_jitters"]
        got = D.get_item(env.get, int(gold[f"s{k}_index"]), cfg, float(gold[f"s{k}_angle"]), [(j[:2], j[2]) for j in jit],
                         gold[f"s{k}_perm"], convs)
        for n, g in zip(NAMES, got):
            want = gold[f"s{k}_{n}"]
            g = g.numpy() if torch.is_tensor(g) else np.asarray(g)
            assert g.shape == want.shape, (k, n)
            if n in ("bev", "num_points", "cmd", "bra", "typs", "num_objs"):
                assert np.array_equal(g, want), (k, n)
            else:
                assert np.abs(g.astype(np.float64) - want).max() <= 1e-5, (k, n)
    assert {int(gold[f"s{k}_index"]) for k in range(3)} >= {0, 1}


def write_config(gold, data_dir, path):
    import yaml
    cfg = dict(json.loads(str(gold["config"])), data_dir=data_dir)
    with open(path, "w") as f:
        yaml.safe_dump(cfg, f)
    return str(path)


def test_dataset_host_labels_match_reference(gold, recording, tmp_path):
    """the host half of the product dataset (record reads, vectorised actor filter / ego transform / padding) on the CPU."""
    from lav_b200.datasets import TemporalLiDARPaintedDataset
    ds = TemporalLiDARPaintedDataset(write_config(gold, recording, tmp_path / "c.yaml"), seed=int(gold["seed"]), device="cpu")
    assert len(ds) == len(gold["map_traj"])
    for k, idx in enumerate(gold["samples"].tolist()):
        jit = gold[f"s{k}_jitters"]
        h = ds.prepare(idx, float(gold[f"s{k}_angle"]), [(j[:2], j[2]) for j in jit])
        for n in ("ego_locs", "nxp", "locs", "oris", "typs", "num_objs", "cmd", "bra"):
            assert np.abs(np.asarray(h[n], dtype=np.float64) - gold[f"s{k}_{n}"]).max() <= 1e-5, (k, n)
        assert len(h["sweeps"]) == min(int(gold[f"s{k}_index"]), 2) + 1


def test_train_full_parses_arguments_and_config(tmp_path):
    import yaml
    import bench
    from lav_b200 import train_full
    args = train_full.parse_args(["--config-path", "c.yaml", "--batch-size", "4", "--max-steps", "2", "--perceive-only"])
    assert (args.batch_size, args.max_steps, args.perceive_only, args.motion_only, args.num_epoch, args.lr, args.seed) == \
        (4, 2, True, False, 64, 3e-4, 2021)
    with pytest.raises(SystemExit):
        train_full.parse_args(["--perceive-only", "--motion-only"])
    (_, lid, uni, _), _ = bench.build_models()
    cfg = dict(seg_channels=[4, 6, 7, 10], num_frame_stack=2, num_features=[64, 64], backbone="cnn", min_x=-10, max_x=70, min_y=-40,
               max_y=40, pixels_per_meter=4, crop_size=96, feature_x_jitter=1.5, feature_angle_jitter=20, num_cmds=6, num_plan=20,
               num_plan_iter=5, point_painting=True)
    for key, m in (("lidar_model_dir", lid), ("uniplanner_dir", uni), ("bev_model_dir", uni.bev_planner)):
        torch.save(m.state_dict(), tmp_path / key)
        cfg[key] = str(tmp_path / key)
    l2, u2 = train_full.build_models(yaml.safe_load(yaml.safe_dump(cfg)))
    for a, b in ((lid, l2), (uni, u2)):
        sa, sb = a.state_dict(), b.state_dict()
        assert sa.keys() == sb.keys() and all(torch.equal(sa[k], sb[k]) for k in sa)
