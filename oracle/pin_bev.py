"""Pin the privileged-planner stage (TemporalBEVDataset, BEVPlanner.forward, LAV.train_bev) against the REFERENCE and write
tests/golden/temporal_bev_dataset.npz and tests/golden/bev_planner_train.npz.  Every other golden is left untouched.

Runs only where the reference sources are readable.  It
  1. writes a small seeded synthetic recording (lav_b200.synth.record_trajectories, plus the empty data.mdb placeholder
     BasicDataset looks for), runs the reference's own TemporalBEVDataset on it (lmdb = oracle/refshim/lmdb, trajectories in
     sorted order), seeding torch before each item, replays the draws through oracle.bev_dataset_ref.get_bev_item and asserts
     agreement; stores the seed, config, index mapping, draws and the reference's 9 outputs;
  2. runs the reference bev_planner_v2.BEVPlanner in train mode with synth.fill_state_dict_ weights on
     synth.bev_planner_batch (a sample with more than max_num_cars vehicles ahead, and a call where none qualifies), checks
     lav_b200.heads.BEVPlanner against it and stores the 6 outputs of each call (the inputs are regenerated from the seed);
  3. calls the reference's own LAV.train_bev on a stub instance for two other_weight values, checks lav_b200.train.BEVTrainer
     against it, and stores the 4 losses and a digest of the parameters after the Adam step.

    python oracle/pin_bev.py
"""
import glob as _glob
import importlib
import json
import os
import shutil
import sys
import tempfile
import types

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
from oracle.bev_dataset_ref import get_bev_item  # noqa: E402

SEED = 2021
N_TRAJ, N_FRAMES = 5, 25
# config_v2.yaml's dataset values, with a data filter that drops trajectories (percentage_data < 1, the TRAIN_TOWNS filter)
CONFIG = dict(num_plan=20, num_frame_stack=2, crop_size=96, x_jitter=10, angle_jitter=20, max_pedestrian_radius=10,
              max_vehicle_radius=25, max_objs=20, min_x=-10, max_x=70, min_y=-40, max_y=40, pixels_per_meter=4, percentage_data=0.7,
              all_towns=False)
# the planner of config_v2.yaml (lav_privileged_v2.py:32-42)
PLANNER = dict(pixels_per_meter=4, crop_size=96, feature_x_jitter=1.5, feature_angle_jitter=20, x_offset=0,
               y_offset=1 + (-10) / ((70 + 10) / 2), num_cmds=6, num_plan=20, num_plan_iter=5, num_frame_stack=2)
GOLD = os.path.join(ROOT, "tests", "golden")
NAMES_DS = ["bev", "ego_locs", "cmd", "nxp", "bra", "locs", "oris", "typs", "num_objs"]
NAMES_FWD = ["other_locs", "other_cast_locs", "other_cast_cmds", "ego_plan_locs", "ego_cast_locs", "ego_cast_cmds"]
NAMES_LOSS = ["plan_loss", "ego_cast_loss", "other_cast_loss", "cmd_loss"]
FWD_SEED = 1234
OTHER_WEIGHTS = (0.0, 0.5)


def param_digest(sd):
    """per-tensor (sum, sum of squares) in fp64 of the floating-point entries of a state_dict, in key order."""
    return np.array([[float(v.double().sum()), float((v.double() ** 2).sum())] for v in sd.values() if v.is_floating_point()])


def pin_dataset():
    tmp = tempfile.mkdtemp(prefix="lavb_pin_bev_")
    data_dir = os.path.join(tmp, "data")
    for p in synth.record_trajectories(data_dir, N_TRAJ, N_FRAMES, SEED):
        open(os.path.join(p, "data.mdb"), "wb").close()
    cfg = dict(CONFIG, data_dir=data_dir)
    cfg_path = os.path.join(tmp, "config.yaml")
    with open(cfg_path, "w") as f:
        yaml.safe_dump(cfg, f)
    import lav.utils
    pkg = types.ModuleType("lav.utils.datasets")       # the package __init__ imports every dataset: load only what this needs
    pkg.__path__ = [os.path.join(REF, "lav", "utils", "datasets")]
    sys.modules["lav.utils.datasets"] = pkg
    import lav.utils.datasets.basic_dataset as BD
    from lav.utils.datasets.temporal_bev_dataset import TemporalBEVDataset

    class _SortedGlob:
        @staticmethod
        def glob(pattern):
            return sorted(_glob.glob(pattern))
    BD.glob = _SortedGlob
    ds = TemporalBEVDataset(cfg_path, seed=SEED)
    mapping = [(os.path.basename(ds.nam_map[i]), ds.idx_map[i]) for i in range(len(ds))]
    trajs = sorted(set(m[0] for m in mapping))
    print(f"[dataset] reference: {len(ds)} samples from {trajs}")
    picks = [mapping.index((trajs[0], 0)), mapping.index((trajs[0], 1)), mapping.index((trajs[-1], 4)), mapping.index((trajs[1], 3))]
    gold = dict(seed=SEED, n_traj=N_TRAJ, n_frames=N_FRAMES, config=json.dumps(CONFIG), samples=np.array(picks),
                map_traj=np.array([m[0] for m in mapping]), map_index=np.array([m[1] for m in mapping]))
    for k, idx in enumerate(picks):
        torch.manual_seed(1000 + k)
        ref = ds[idx]
        torch.manual_seed(1000 + k)                      # replay the draws in the order __getitem__ makes them
        offset = int(np.clip(int((torch.rand(1) * 2 - 1) * cfg["x_jitter"]), -32, 32))
        angle = float(torch.rand(1) * 2 - 1) * cfg["angle_jitter"]
        index = ds.idx_map[idx]
        got = get_bev_item(DirEnv(ds.nam_map[idx]).get, index, cfg, offset, angle)
        for n, r, g in zip(NAMES_DS, ref, got):
            r, g = np.asarray(r, dtype=np.float64), np.asarray(g, dtype=np.float64)
            assert r.shape == g.shape, (n, r.shape, g.shape)
            d = float(np.abs(r - g).max()) if r.size else 0.0
            tol = 0.0 if n in ("bev", "cmd", "bra", "typs", "num_objs") else 1e-5
            print(f"  sample {idx} (frame {index}, offset {offset}, angle {angle:.2f}) {n:9s} max|ref-oracle| = {d:.2e}")
            assert d <= tol, (idx, n, d)
        gold.update({f"s{k}_offset": offset, f"s{k}_angle": angle, f"s{k}_torch_seed": 1000 + k, f"s{k}_traj": mapping[idx][0],
                     f"s{k}_index": index})
        for n, r in zip(NAMES_DS, ref):
            gold[f"s{k}_{n}"] = np.asarray(r)
    out = os.path.join(GOLD, "temporal_bev_dataset.npz")
    np.savez_compressed(out, **gold)
    shutil.rmtree(tmp, True)
    print(f"wrote {out} ({os.path.getsize(out) / 1e6:.2f} MB)")


def pin_planner():
    pkg = types.ModuleType("lavm")                      # lav/models as a package without running its __init__
    pkg.__path__ = [os.path.join(REF, "lav", "models")]
    sys.modules["lavm"] = pkg
    RefBP = importlib.import_module("lavm.bev_planner_v2").BEVPlanner
    from lav.lav_privileged_v2 import LAV
    from lav_b200.heads import BEVPlanner
    from lav_b200.train import BEVTrainer

    ref_cfg = yaml.safe_load(open(os.path.join(REF, "config_v2.yaml")))
    ref = RefBP(**PLANNER).train()
    # a copy: state_dict() tensors alias the module's, and train-mode forwards update the BatchNorm running statistics
    sd = {k: v.clone() for k, v in synth.fill_state_dict_(ref.state_dict()).items()}
    ref.load_state_dict(sd)
    mine = BEVPlanner(**PLANNER).train()
    mine.load_state_dict(sd)
    gold = dict(seed=synth.SEED, fwd_seed=FWD_SEED, names_fwd=np.array(NAMES_FWD), names_loss=np.array(NAMES_LOSS),
                other_weights=np.array(OTHER_WEIGHTS))
    print("[planner forward]")
    for tag, no_veh in (("mixed", False), ("none", True)):
        bev, ego_locs, cmds, nxps, bras, locs, oris, typs = synth.bev_planner_batch(no_vehicles=no_veh)
        torch.manual_seed(FWD_SEED)
        r = ref(bev.float(), ego_locs, locs, oris, nxps, typs)
        torch.manual_seed(FWD_SEED)
        m = mine(bev.float(), ego_locs, locs, oris, nxps, typs)
        for n, a, b in zip(NAMES_FWD, r, m):
            a, b = a.detach(), b.detach()
            assert a.shape == b.shape, (tag, n, a.shape, b.shape)
            d = float((a.double() - b.double()).abs().max()) if a.numel() else 0.0
            tol = 2e-4 * (float(a.abs().max()) + 1) if a.numel() else 0.0
            print(f"  {tag:5s} {n:16s} {tuple(a.shape)} max|ref-mine| = {d:.2e} (tol {tol:.1e})")
            assert d <= tol, (tag, n)
            gold[f"{tag}_{n}"] = a.numpy()
    print("[train_bev]")
    batch = synth.bev_planner_batch()
    for w in OTHER_WEIGHTS:
        model = RefBP(**PLANNER)
        model.load_state_dict(sd)
        obj = object.__new__(LAV)                       # LAV.__init__ builds every model and loads weights: set what train_bev reads
        for k in ("use_others_to_train", "num_plan", "num_plan_iter", "num_cmds", "cmd_smooth", "cmd_weight", "pixels_per_meter"):
            setattr(obj, k, ref_cfg[k])
        obj.device = torch.device("cpu")
        obj.branch_weights = torch.tensor(ref_cfg["branch_weights"]).float()
        obj.bev_center = [160.0, 280.0]
        obj.bev_planner = model.train()
        obj.bev_optim = torch.optim.Adam(model.parameters(), lr=3e-4)
        bev, ego_locs, cmds, nxps, bras, locs, oris, typs = batch
        torch.manual_seed(FWD_SEED)
        res = LAV.train_bev(obj, bev, ego_locs, cmds, nxps, bras, locs, oris, typs, torch.full((3,), 8), other_weight=w)
        ref_l = np.array([res[k] for k in NAMES_LOSS])
        ref_d = param_digest(model.state_dict())

        my_model = BEVPlanner(**PLANNER)
        my_model.load_state_dict(sd)
        tr = BEVTrainer(my_model, lr=3e-4, device=torch.device("cpu"), branch_weights=ref_cfg["branch_weights"],
                        cmd_weight=ref_cfg["cmd_weight"], cmd_smooth=ref_cfg["cmd_smooth"],
                        use_others_to_train=ref_cfg["use_others_to_train"])
        torch.manual_seed(FWD_SEED)
        _, parts = tr.train_bev(*batch, other_weight=w)
        my_l = np.array([float(parts[k]) for k in NAMES_LOSS])
        my_d = param_digest(my_model.state_dict())
        dl = float(np.abs(ref_l - my_l).max() / np.abs(ref_l).max())
        dd = float(np.abs(ref_d - my_d).max() / (np.abs(ref_d).max()))
        print(f"  other_weight={w}: losses {ref_l}, max rel |ref-mine| = {dl:.2e}; parameter digest max rel diff {dd:.2e}")
        assert dl < 1e-5 and dd < 1e-5
        gold[f"w{w}_losses"] = ref_l
        gold[f"w{w}_digest"] = ref_d
    out = os.path.join(GOLD, "bev_planner_train.npz")
    np.savez_compressed(out, **gold)
    print(f"wrote {out} ({os.path.getsize(out) / 1e6:.2f} MB)")


if __name__ == "__main__":
    pin_dataset()
    pin_planner()
