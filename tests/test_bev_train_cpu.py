"""CPU: the privileged-planner stage against the reference's own outputs (oracle/pin_bev.py) — the oracle's
TemporalBEVDataset.__getitem__ and the dataset's index mapping and host labels (tests/golden/temporal_bev_dataset.npz),
BEVPlanner.forward on the grid_sample path, bev_losses and one BEVTrainer step (tests/golden/bev_planner_train.npz) — plus the
state_dict keys, the other_weight schedule and the train_bev arguments."""
import json
import math
import os

import numpy as np
import pytest
import torch
import yaml

from lav_b200 import synth
from lav_b200.data_paint import DirEnv
from oracle.bev_dataset_ref import get_bev_item

NAMES_DS = ["bev", "ego_locs", "cmd", "nxp", "bra", "locs", "oris", "typs", "num_objs"]
EXACT = ("bev", "cmd", "bra", "typs", "num_objs")
PLANNER = dict(pixels_per_meter=4, crop_size=96, feature_x_jitter=1.5, feature_angle_jitter=20, x_offset=0,
               y_offset=1 + (-10) / ((70 + 10) / 2), num_cmds=6, num_plan=20, num_plan_iter=5, num_frame_stack=2)


@pytest.fixture(scope="module")
def gold_ds(golden_dir):
    return np.load(os.path.join(golden_dir, "temporal_bev_dataset.npz"))


@pytest.fixture(scope="module")
def gold_tr(golden_dir):
    return np.load(os.path.join(golden_dir, "bev_planner_train.npz"))


@pytest.fixture(scope="module")
def bev_config(gold_ds, tmp_path_factory):
    root = tmp_path_factory.mktemp("bevrec")
    synth.record_trajectories(str(root / "data"), int(gold_ds["n_traj"]), int(gold_ds["n_frames"]), int(gold_ds["seed"]))
    cfg = dict(json.loads(str(gold_ds["config"])), data_dir=str(root / "data"))
    with open(root / "config.yaml", "w") as f:
        yaml.safe_dump(cfg, f)
    return str(root / "config.yaml")


def _planner(seed):
    from lav_b200.heads import BEVPlanner
    m = BEVPlanner(**PLANNER).train()
    m.load_state_dict(synth.fill_state_dict_(m.state_dict(), seed))
    return m


def test_oracle_getitem_reproduces_reference(gold_ds, bev_config):
    cfg = yaml.safe_load(open(bev_config))
    for k in range(len(gold_ds["samples"])):
        env = DirEnv(os.path.join(cfg["data_dir"], str(gold_ds[f"s{k}_traj"])))
        got = get_bev_item(env.get, int(gold_ds[f"s{k}_index"]), cfg, int(gold_ds[f"s{k}_offset"]), float(gold_ds[f"s{k}_angle"]))
        for n, g in zip(NAMES_DS, got):
            want, g = gold_ds[f"s{k}_{n}"], np.asarray(g)
            assert g.shape == want.shape, (k, n)
            if n in EXACT:
                assert np.array_equal(g, want), (k, n)
            else:
                assert np.abs(g.astype(np.float64) - want).max() <= 1e-5, (k, n)
    assert {int(gold_ds[f"s{k}_index"]) for k in range(len(gold_ds["samples"]))} >= {0, 1}
    assert any(int(gold_ds[f"s{k}_offset"]) != 0 for k in range(len(gold_ds["samples"])))


def test_index_mapping_and_host_labels(gold_ds, bev_config):
    from lav_b200.datasets import TemporalBEVDataset
    ds = TemporalBEVDataset(bev_config, seed=int(gold_ds["seed"]), device="cpu")
    got = [(os.path.basename(ds.paths[t]), i) for t, i in ds.index]
    assert got == list(zip(gold_ds["map_traj"].tolist(), gold_ds["map_index"].tolist())) and len(ds) == len(got)
    for k, idx in enumerate(gold_ds["samples"].tolist()):
        ds.gen.manual_seed(int(gold_ds[f"s{k}_torch_seed"]))
        offset, angle = ds.draw(ds.gen)                                              # the reference's stream replays
        assert offset == int(gold_ds[f"s{k}_offset"]) and angle == float(gold_ds[f"s{k}_angle"])
        h = ds.prepare(idx, offset, angle)
        for n in ("ego_locs", "nxp", "locs", "oris", "typs", "num_objs", "cmd", "bra"):
            assert np.abs(np.asarray(h[n], dtype=np.float64) - gold_ds[f"s{k}_{n}"]).max() <= 1e-5, (k, n)


def test_duplicate_x_jitter_key_takes_the_later_value(tmp_path):
    """config_v2.yaml sets x_jitter twice (5, then 10); yaml.safe_load keeps the later one, as the reference does."""
    from lav_b200.datasets import TemporalBEVDataset
    (tmp_path / "data").mkdir()
    text = ("x_jitter: 5\nangle_jitter: 20\nnum_plan: 20\nx_jitter: 10 # In pixels\n"
            f"data_dir: {tmp_path / 'data'}\npercentage_data: 1.01\nall_towns: True\n")
    (tmp_path / "c.yaml").write_text(text)
    ds = TemporalBEVDataset(str(tmp_path / "c.yaml"), device="cpu")
    assert ds.x_jitter == 10 and len(ds) == 0
    offsets = {ds.draw(ds.gen)[0] for _ in range(400)}
    assert max(offsets) >= 8 and min(offsets) <= -8 and max(abs(o) for o in offsets) <= 10


@pytest.mark.parametrize("tag", ["mixed", "none"])
def test_planner_forward_matches_reference(gold_tr, tag):
    m = _planner(int(gold_tr["seed"]))
    bev, ego_locs, cmds, nxps, bras, locs, oris, typs = synth.bev_planner_batch(no_vehicles=tag == "none")
    torch.manual_seed(int(gold_tr["fwd_seed"]))
    out = m(bev.float(), ego_locs, locs, oris, nxps, typs)
    assert len(out) == 6
    for n, got in zip(gold_tr["names_fwd"].tolist(), out):
        want = gold_tr[f"{tag}_{n}"]
        got = got.detach().numpy()
        assert got.shape == want.shape, (n, got.shape, want.shape)
        assert np.abs(got.astype(np.float64) - want).max() <= 2e-4 * (np.abs(want).max() + 1), n
    if tag == "mixed":
        assert len(out[0]) == 5 + int(((typs[1, 1:] == 1) & (locs[1, 1:, 0, 1] < ego_locs[1, 0, 1])).sum())   # the cap of 5 applied


def test_bev_losses_and_one_step_match_reference(gold_tr):
    from lav_b200.train import BEVTrainer, bev_losses
    batch = synth.bev_planner_batch()
    bev, ego_locs, cmds, nxps, bras, locs, oris, typs = batch
    names = gold_tr["names_loss"].tolist()
    for w in gold_tr["other_weights"].tolist():
        m = _planner(int(gold_tr["seed"]))
        torch.manual_seed(int(gold_tr["fwd_seed"]))
        out = m(bev, ego_locs, locs, oris, nxps, typs)
        bw = torch.tensor([5, 5, 5, 1, 1, 1]).float()
        total, parts = bev_losses(out, ego_locs, cmds, bras, bw, other_weight=w, cmd_weight=0.1, cmd_smooth=0.2)
        got = np.array([float(parts[k]) for k in names])
        want = gold_tr[f"w{w}_losses"]
        assert np.abs(got - want).max() / np.abs(want).max() <= 1e-5, (w, got, want)
        assert math.isclose(float(total), want[0] + want[1] + w * want[2] + 0.1 * want[3], rel_tol=1e-5)

        m = _planner(int(gold_tr["seed"]))
        tr = BEVTrainer(m, lr=3e-4, device=torch.device("cpu"))
        torch.manual_seed(int(gold_tr["fwd_seed"]))
        tr.train_bev(*batch, other_weight=w)
        digest = np.array([[float(v.double().sum()), float((v.double() ** 2).sum())] for v in m.state_dict().values()
                           if v.is_floating_point()])
        ref = gold_tr[f"w{w}_digest"]
        assert np.abs(digest - ref).max() / np.abs(ref).max() <= 1e-5, w


def test_plan_loss_is_nan_when_every_sample_brakes():
    """as in the reference: the plan loss is a mean over the non-braking samples only."""
    from lav_b200.train import bev_losses
    B, T = 2, 20
    out = (torch.zeros(3, T, 2), torch.zeros(3, 6, T, 2), torch.full((3, 6), 0.5), torch.zeros(B, 5, 6, T, 2),
           torch.zeros(B, 6, T, 2), torch.full((B, 6), 0.5))
    _, parts = bev_losses(out, torch.ones(B, T + 1, 2), torch.tensor([0, 3]), torch.ones(B, dtype=torch.int64), torch.ones(6))
    assert math.isnan(float(parts["plan_loss"])) and math.isfinite(float(parts["ego_cast_loss"]))


def test_state_dict_keys_match_the_teacher_in_the_uniplanner_checkpoint(golden_dir):
    want = {k[len("bev_planner."):]: v for k, v in json.load(open(os.path.join(golden_dir, "keys_uniplanner.json"))).items()
            if k.startswith("bev_planner.")}
    m = _planner(2021)
    assert {k: list(v.shape) for k, v in m.state_dict().items()} == want
    assert m.max_num_cars == 5 and math.isclose(m.feature_angle_jitter, math.radians(20)) and m.feature_x_jitter == 1.5


def test_other_weight_schedule():
    from lav_b200.train import BEVTrainer, other_weight_schedule
    assert other_weight_schedule(0) == 0.0
    assert math.isclose(other_weight_schedule(4000), 0.2) and math.isclose(other_weight_schedule(8000), 1 - 0.64)
    assert 0.99 < other_weight_schedule(100000) < 1.0
    m = _planner(2021)
    assert BEVTrainer(m, device=torch.device("cpu")).other_weight(4000) == pytest.approx(0.2)
    assert BEVTrainer(m, device=torch.device("cpu"), use_others_to_train=False).other_weight(4000) == 0.0


def test_train_bev_parses_arguments():
    from lav_b200 import train_bev
    a = train_bev.parse_args([])
    assert (a.config_path, a.num_epoch, a.batch_size, a.lr, a.seed, a.num_per_log, a.num_per_save, a.weight_decay, a.max_steps) == \
        ("config_v2.yaml", 160, 256, 3e-4, 2021, 100, 1, 2e-4, 0)
    a = train_bev.parse_args(["--config-path", "c.yaml", "--batch-size", "4", "--max-steps", "2", "--save-dir", "out",
                              "--num-workers", "3"])
    assert (a.config_path, a.batch_size, a.max_steps, a.save_dir, a.num_workers) == ("c.yaml", 4, 2, "out", 3)
    cfg = dict(pixels_per_meter=4, crop_size=96, feature_x_jitter=1.5, feature_angle_jitter=20, min_x=-10, max_x=70, num_cmds=6,
               num_plan=20, num_plan_iter=5, num_frame_stack=2)
    m = train_bev.build_planner(cfg)
    assert math.isclose(float(m.offset_y), PLANNER["y_offset"]) and m.bev_conv_emb[0].conv1.in_channels == 9
