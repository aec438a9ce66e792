"""Pin oracle/dataset_ref.py against the REFERENCE's TemporalLiDARPaintedDataset and write tests/golden/temporal_dataset.npz.

Runs only where the reference sources are readable.  It
  1. writes a small seeded synthetic recording with lav_b200.synth.record_trajectories (plus the empty data.mdb placeholder
     BasicDataset looks for in each trajectory directory),
  2. runs the reference's own TemporalLiDARPaintedDataset.__getitem__ on it (lmdb = oracle/refshim/lmdb, which reads the
     directory store; the trajectory directories are listed in sorted order), seeding torch and numpy before each call so the
     draws can be replayed,
  3. replays the draws through oracle.dataset_ref.get_item and asserts agreement,
  4. stores the recording's seed and config, the index mapping, the draws and the reference's 14 outputs.

    python oracle/pin_dataset.py
"""
import glob as _glob
import json
import os
import shutil
import sys
import tempfile

import numpy as np
import torch
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("LAV_REFERENCE", "/root/reference")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "refshim"))
sys.path.insert(0, REF)

from lav_b200 import synth  # noqa: E402
from lav_b200.data_paint import DirEnv  # noqa: E402
from oracle import dataset_ref as D  # noqa: E402
from oracle import lav_ref as O  # noqa: E402

SEED = 2021
N_TRAJ, N_FRAMES = 5, 25
# config_v2.yaml values, except a small max_lidar_points (3 sweeps of <= 600 points never exceed it) and a data filter that
# drops trajectories: percentage_data < 1 and the TRAIN_TOWNS filter
CONFIG = dict(num_plan=20, num_frame_stack=2, seg_channels=[4, 6, 7, 10], max_lidar_points=2000, camera_x=1.5, camera_z=2.4,
              camera_yaws=[-120, -60, 0, 60, 120], angle_jitter=20, stack_loc_jitter=0.4, stack_ori_jitter=0.1,
              max_pedestrian_radius=10, max_vehicle_radius=25, max_mot_vehicle_radius=15, max_objs=20, min_x=-10, max_x=70,
              min_y=-40, max_y=40, pixels_per_meter=4, percentage_data=0.7, all_towns=False)
OUT = os.path.join(ROOT, "tests", "golden", "temporal_dataset.npz")


def main():
    tmp = tempfile.mkdtemp(prefix="lavb_pin_ds_")
    data_dir = os.path.join(tmp, "data")
    for p in synth.record_trajectories(data_dir, N_TRAJ, N_FRAMES, SEED):
        open(os.path.join(p, "data.mdb"), "wb").close()
    cfg = dict(CONFIG, data_dir=data_dir)
    cfg_path = os.path.join(tmp, "config.yaml")
    with open(cfg_path, "w") as f:
        yaml.safe_dump(cfg, f)

    import types
    import lav.utils
    pkg = types.ModuleType("lav.utils.datasets")       # the package __init__ imports every dataset (imgaug, ...): load the three
    pkg.__path__ = [os.path.join(REF, "lav", "utils", "datasets")]                # modules this needs without it
    sys.modules["lav.utils.datasets"] = pkg
    import lav.utils.datasets.basic_dataset as BD
    from lav.utils.datasets.temporal_lidar_painted_dataset import TemporalLiDARPaintedDataset

    class _SortedGlob:                                   # the reference lists trajectories in file-system order; pin sorted order
        @staticmethod
        def glob(pattern):
            return sorted(_glob.glob(pattern))
    BD.glob = _SortedGlob
    ds = TemporalLiDARPaintedDataset(cfg_path, seed=SEED)
    mapping = [(os.path.basename(ds.nam_map[i]), ds.idx_map[i]) for i in range(len(ds))]
    print(f"reference: {len(ds)} samples from {sorted(set(m[0] for m in mapping))}")

    # index 0 and 1 (missing previous frames), and a later frame of another trajectory (shift + yaw change)
    trajs = sorted(set(m[0] for m in mapping))
    picks = [mapping.index((trajs[0], 0)), mapping.index((trajs[0], 1)), mapping.index((trajs[-1], 4))]
    convs = O.default_converters(cfg["camera_x"], cfg["camera_z"])
    gold = dict(seed=SEED, n_traj=N_TRAJ, n_frames=N_FRAMES, config=json.dumps(CONFIG), samples=np.array(picks),
                map_traj=np.array([m[0] for m in mapping]), map_index=np.array([m[1] for m in mapping]))
    names = ["lidar", "num_points", "heatmaps", "sizemaps", "orimaps", "bev", "ego_locs", "cmd", "nxp", "bra", "locs", "oris",
             "typs", "num_objs"]
    for k, idx in enumerate(picks):
        torch.manual_seed(1000 + k)
        np.random.seed(1000 + k)
        ref = ds[idx]
        torch.manual_seed(1000 + k)                      # replay the draws in the order __getitem__ makes them
        angle = float(torch.rand(1) * 2 - 1) * cfg["angle_jitter"]
        np.random.seed(1000 + k)
        index = ds.idx_map[idx]
        nfr = min(index, cfg["num_frame_stack"]) + 1
        jit = np.zeros((3, 3))
        for t in range(1, nfr):
            jit[t, :2] = np.random.uniform(low=-cfg["stack_loc_jitter"], high=cfg["stack_loc_jitter"], size=2)
            jit[t, 2] = np.random.uniform(low=-cfg["stack_ori_jitter"], high=cfg["stack_ori_jitter"])
        total = int(ref[1])
        assert total < cfg["max_lidar_points"]
        perm = np.arange(total)
        np.random.shuffle(perm)
        env = DirEnv(ds.nam_map[idx])
        got = D.get_item(env.get, index, cfg, angle, [(j[:2], j[2]) for j in jit], perm, convs)
        for n, r, g in zip(names, ref, got):
            r, g = np.asarray(r, dtype=np.float64), np.asarray(g, dtype=np.float64)
            assert r.shape == g.shape, (n, r.shape, g.shape)
            d = float(np.abs(r - g).max()) if r.size else 0.0
            tol = 0.0 if n in ("bev", "num_points", "cmd", "bra", "typs", "num_objs") else 1e-5
            print(f"  sample {idx} (frame {index}) {n:10s} max|ref-oracle| = {d:.2e}")
            assert d <= tol, (idx, n, d)
        dl = [D.filter_actors(env.get, i, T=cfg["num_plan"])[1][0] for i in (index, max(index - 2, 0))]
        print(f"  sample {idx}: ego moved {np.linalg.norm(dl[0] - dl[1]):.2f} m over the stack")
        gold.update({f"s{k}_angle": angle, f"s{k}_jitters": jit, f"s{k}_perm": perm, f"s{k}_traj": mapping[idx][0],
                     f"s{k}_index": index})
        for n, r in zip(names, ref):
            gold[f"s{k}_{n}"] = r.numpy() if torch.is_tensor(r) else np.asarray(r)
    np.savez_compressed(OUT, **gold)
    shutil.rmtree(tmp, True)
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1e6:.2f} MB)")


if __name__ == "__main__":
    main()
