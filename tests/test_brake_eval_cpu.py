"""CPU: the host half of evaluate --brake: BrakeScores against a hand count, its rank merge, the expert-track row builder against
a loop over the label slots, the CLI's refusal of --brake without weights, and the brake model's camera reads of
TemporalLiDARPaintedDataset against CameraDataset's on a synthetic 5-camera recording (PNG and JPEG trajectories)."""
import os

import numpy as np
import pytest
import torch

from lav_b200 import synth
from lav_b200.capi import LavbError
from lav_b200.control import FLAG_BRAKE_MODEL, FLAG_COLLIDE, FLAG_PID_BRAKE, FLAG_PLAN_INVALID, FLAG_SPEED_CAP
import lav_b200.evaluate as E

REASONS = (("brake_model", FLAG_BRAKE_MODEL), ("plan_stop", FLAG_PID_BRAKE), ("collide", FLAG_COLLIDE))


# ----------------------------------------------------------------------------- the host reduction
def hand_summary(res, cmds, bras, num_cmds):
    """BrakeScores.summary written out sample by sample."""
    def table(rows):
        n = dict(tp=0, fp=0, fn=0, tn=0)
        for fire, y in rows:
            n[("t" if fire == y else "f") + ("p" if fire else "n")] += 1
        div = lambda a, b: a / b if b else None
        return dict(n, precision=div(n["tp"], n["tp"] + n["fp"]), recall=div(n["tp"], n["tp"] + n["fn"]),
                    false_brake_rate=div(n["fp"], n["fp"] + n["tn"]), missed_brake_rate=div(n["fn"], n["tp"] + n["fn"]))

    def verdicts(r):
        f, fe, brake = (int(x) for x in r)
        return dict(agent=brake != 0, brake_model=bool(f & FLAG_BRAKE_MODEL), plan_stop=bool(f & FLAG_PID_BRAKE),
                    collide=bool(f & FLAG_COLLIDE), collide_expert_tracks=bool(fe & FLAG_COLLIDE))

    def tables(idx):
        return {name: table([(verdicts(res[i])[name], bras[i] != 0) for i in idx]) for name in E.BRAKE_VERDICTS}

    n = len(res)
    by_reason = {}
    for combo in ("brake_model", "plan_stop", "brake_model+plan_stop", "collide", "brake_model+collide", "plan_stop+collide",
                  "brake_model+plan_stop+collide"):
        names = combo.split("+")
        brakes = false = 0
        for i in range(n):
            fired = [name for name, bit in REASONS if res[i][0] & bit]
            if res[i][2] and fired == names:
                brakes += 1
                false += bras[i] == 0
        by_reason[combo] = dict(brakes=brakes, false_brakes=false)
    cmd_set = sorted(set(range(num_cmds)) | set(int(c) for c in cmds))
    return dict(samples=n, positives=sum(int(b != 0) for b in bras), invalid_plans=sum(int(r[0] & FLAG_PLAN_INVALID != 0) for r in res),
                verdicts=tables(range(n)),
                per_cmd={str(c): dict(samples=sum(int(x == c) for x in cmds), verdicts=tables([i for i in range(n) if cmds[i] == c]))
                         for c in cmd_set},
                by_reason=by_reason)


def flag_patterns(n, seed, num_cmds=6, skip_cmd=2):
    """n samples of score_brake results whose agent brake follows the kernel's rule (any of the three reasons), with
    PLAN_INVALID plans (no PID brake), the speed-cap bit as noise, every command but ``skip_cmd`` (4 and 5 included)."""
    rs = np.random.RandomState(seed)
    f = np.zeros(n, np.int32)
    invalid = rs.rand(n) < 0.2
    f |= np.where(invalid, FLAG_PLAN_INVALID, 0)
    f |= np.where(~invalid & (rs.rand(n) < 0.3), FLAG_PID_BRAKE, 0)
    f |= np.where(rs.rand(n) < 0.3, FLAG_BRAKE_MODEL, 0)
    f |= np.where(rs.rand(n) < 0.3, FLAG_COLLIDE, 0)
    f |= np.where(rs.rand(n) < 0.1, FLAG_SPEED_CAP, 0)
    fe = np.where(rs.rand(n) < 0.4, FLAG_COLLIDE, 0) | (f & ~FLAG_COLLIDE)
    brake = ((f & (FLAG_BRAKE_MODEL | FLAG_PID_BRAKE | FLAG_COLLIDE)) != 0).astype(np.int32)
    cmds = rs.choice([c for c in range(num_cmds) if c != skip_cmd], n)
    cmds[:2] = (4, 5)
    bras = (rs.rand(n) < 0.35).astype(np.int64)
    return np.stack([f, fe, brake], 1), cmds, bras


@pytest.mark.parametrize("labels", ["mixed", "all_negative", "all_positive"])
def test_reduction_equals_a_hand_count(labels):
    res, cmds, bras = flag_patterns(200, 7)
    if labels != "mixed":
        bras[:] = labels == "all_positive"
    acc = E.BrakeScores(6)
    for k in range(0, 200, 33):                                          # uneven batches
        acc.add(res[k:k + 33], cmds[k:k + 33], bras[k:k + 33])
    got = acc.summary()
    assert got == hand_summary(res, cmds, bras, 6)
    assert got["per_cmd"]["2"]["samples"] == 0
    assert all(d["precision"] is None and d["false_brake_rate"] is None for d in got["per_cmd"]["2"]["verdicts"].values())
    assert got["invalid_plans"] > 0 and got["per_cmd"]["4"]["samples"] > 0 and got["per_cmd"]["5"]["samples"] > 0
    a = got["verdicts"]["agent"]
    if labels == "all_negative":
        assert a["recall"] is None and a["missed_brake_rate"] is None and a["false_brake_rate"] is not None
    if labels == "all_positive":
        assert a["false_brake_rate"] is None and a["missed_brake_rate"] is not None
    assert sum(d["brakes"] for d in got["by_reason"].values()) == a["tp"] + a["fp"]
    assert sum(d["false_brakes"] for d in got["by_reason"].values()) == a["fp"]


def test_reduction_known_answer():
    P, B, C = FLAG_PID_BRAKE, FLAG_BRAKE_MODEL, FLAG_COLLIDE
    res = np.array([[B, 0, 1], [C, 0, 1], [P | C, C, 1], [0, C, 0], [FLAG_PLAN_INVALID, 0, 0], [B | C, C, 1]], np.int32)
    bras = np.array([0, 1, 1, 1, 0, 0])
    acc = E.BrakeScores(6)
    acc.add(res, [0, 1, 4, 5, 3, 0], bras)
    s = acc.summary()
    assert {k: s["verdicts"]["agent"][k] for k in ("tp", "fp", "fn", "tn")} == dict(tp=2, fp=2, fn=1, tn=1)
    assert s["verdicts"]["agent"]["false_brake_rate"] == 2 / 3 and s["verdicts"]["agent"]["missed_brake_rate"] == 1 / 3
    assert {k: s["verdicts"]["collide_expert_tracks"][k] for k in ("tp", "fp", "fn", "tn")} == dict(tp=2, fp=1, fn=1, tn=2)
    assert s["by_reason"]["brake_model"] == dict(brakes=1, false_brakes=1)
    assert s["by_reason"]["collide"] == dict(brakes=1, false_brakes=0)
    assert s["by_reason"]["plan_stop+collide"] == dict(brakes=1, false_brakes=0)
    assert s["by_reason"]["brake_model+collide"] == dict(brakes=1, false_brakes=1)
    assert s["invalid_plans"] == 1 and s["positives"] == 3 and s["samples"] == 6
    assert E.BrakeScores(6).summary()["verdicts"]["agent"]["precision"] is None


def test_rank_split_accumulators_merge_to_one_stream():
    from lav_b200.eval_sweep import merge_ranks
    res, cmds, bras = flag_patterns(97, 3)
    one = E.BrakeScores(6)
    for k in range(0, 97, 10):
        one.add(res[k:k + 10], cmds[k:k + 10], bras[k:k + 10])
    for world in (2, 3, 5):
        parts = []
        for r in range(world):
            lo, hi = r * 97 // world, (r + 1) * 97 // world
            acc = E.BrakeScores(6)
            for k in range(lo, hi, 10):
                acc.add(res[k:min(k + 10, hi)], cmds[k:min(k + 10, hi)], bras[k:min(k + 10, hi)])
            parts.append((acc,))
        assert merge_ranks(parts)[0].summary() == one.summary()


# ----------------------------------------------------------------------------- the expert-track rows
def rows_loop(locs, ego_locs, typs, num_objs, C):
    B, M = typs.shape
    T = locs.shape[2] - 1
    rows = np.full((B * (M - 1), C, T, 2), np.nan, np.float32)
    scores = np.zeros((B * (M - 1), C), np.float32)
    for b in range(B):
        for a in range(1, M):
            if a < num_objs[b] and typs[b, a] == 1:
                r = b * (M - 1) + a - 1
                rows[r, 0] = locs[b, a, 1:] - ego_locs[b, 0]
                scores[r, 0] = 1
    return rows, scores


@pytest.mark.parametrize("B,M,T", [(1, 1, 4), (3, 5, 4), (7, 20, 20)])
def test_expert_rows_equal_a_loop_over_the_label_slots(B, M, T):
    rs = np.random.RandomState(B * 100 + M)
    locs = rs.normal(0, 10, (B, M, T + 1, 2)).astype(np.float32)
    ego = rs.normal(0, 1, (B, T + 1, 2)).astype(np.float32)
    typs = rs.choice([0, 1, 1, 2], (B, M)).astype(np.int32)
    num_objs = rs.randint(0, M + 1, B)
    num_objs[0] = M                                                     # the cap: every slot filled
    rows, scores, offsets = E.expert_track_rows(torch.from_numpy(locs), torch.from_numpy(ego), torch.from_numpy(typs),
                                                torch.from_numpy(num_objs), 6)
    want_rows, want_scores = rows_loop(locs, ego, typs, num_objs, 6)
    assert rows.dtype == scores.dtype == torch.float32
    assert np.array_equal(rows.numpy(), want_rows, equal_nan=True) and np.array_equal(scores.numpy(), want_scores)
    assert offsets.dtype == np.int32 and offsets.tolist() == [b * (M - 1) for b in range(B + 1)]


# ----------------------------------------------------------------------------- the CLI
def test_brake_without_weights_is_refused(capsys):
    base = ["--data-dir", "d", "--lidar-weights", "l.th", "--uniplanner-weights", "u.th"]
    with pytest.raises(SystemExit):
        E.parse_args(base + ["--brake"])
    assert "--bra-weights" in capsys.readouterr().err
    args = E.parse_args(base + ["--brake", "--bra-weights", "b.th"])
    assert args.brake and args.bra_weights == "b.th" and args.agent_config is None
    assert not E.parse_args(base).brake


# ----------------------------------------------------------------------------- the camera reads
@pytest.fixture(scope="module")
def camera_recording(tmp_path_factory):
    root = tmp_path_factory.mktemp("brake_cams")
    synth.record_trajectories(str(root / "data"), n_traj=2, n_frames=7, n_points=64, images=True, n_cameras=5)
    return root


def configs(root, tmp_path):
    import json
    import yaml
    from tests.test_camera_eval_cpu import write_camera_config
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", "temporal_dataset.npz"))
    cfg = dict(json.loads(str(gold["config"])), data_dir=str(root / "data"), num_plan=3, crop_tel_bottom=96,
               percentage_data=1.01, all_towns=True)
    with open(tmp_path / "t.yaml", "w") as f:
        yaml.safe_dump(cfg, f)
    return str(tmp_path / "t.yaml"), write_camera_config(tmp_path / "c.yaml", root / "data", 5, num_plan=3)


class KeyLog:
    def __init__(self, env, log):
        self.env, self.log = env, log

    def get(self, key):
        self.log.append(key)
        return self.env.get(key)


def test_camera_staging_equals_camera_datasets(camera_recording, tmp_path):
    from lav_b200.datasets import CameraDataset, TemporalBatchLoader, TemporalLiDARPaintedDataset
    t_cfg, c_cfg = configs(camera_recording, tmp_path)
    ds = TemporalLiDARPaintedDataset(t_cfg, device="cpu")
    cam = CameraDataset(c_cfg, seg=False, brake=True, device="cpu")
    assert ds.index == cam.index and len(ds) == 8
    assert {p.rsplit("/", 1)[-1] for p in ds.paths} == {"traj_000", "traj_001"}         # PNG and JPEG colour images
    log = []
    env = ds.env
    ds.env = lambda traj: KeyLog(env(traj), log)
    for cameras in (False, True):
        log.clear()
        staged = [st for _, st in _staged(TemporalBatchLoader(ds, 3, ordered=True, drop_last=False, num_workers=2, cameras=cameras))]
        read = {k.rsplit("_", 1)[0] for k in log}
        assert ("rgb_1" in read) == cameras and ("tel_rgb" in read) == cameras
        assert not any(k.startswith(("rgb_0", "rgb_4", "sem_")) for k in log)
        if not cameras:
            assert all("cameras" not in st for st in staged)
            continue
        for k, st in enumerate(staged):
            want = cam.stage_batch([cam.prepare(i) for i in range(3 * k, min(3 * k + 3, len(ds)))])
            got = st["cameras"]
            assert set(got) == {"rgbs", "tel"}
            for key in ("rgbs", "tel"):
                assert got[key].dtype == want[key].dtype == torch.uint8 and got[key].shape == want[key].shape
                assert torch.equal(got[key], want[key])
            assert got["rgbs"].shape[1:] == (3, 288, 256, 3) and got["tel"].shape[1:] == (192, 480, 3)


def _staged(loader):
    """the loader's host tables per batch, without the device half."""
    from concurrent.futures import ThreadPoolExecutor
    rng, gen = loader.generators(0)
    order = loader.shard(0)
    with ThreadPoolExecutor(2) as pool:
        for k in range(len(loader)):
            idxs = order[k * loader.B:(k + 1) * loader.B]
            hs = loader._prepare(pool, idxs, [loader.ds.no_draw() for _ in idxs])
            yield hs, loader.ds.stage_batch(hs, gen)


def test_a_missing_tel_rgb_is_named(camera_recording, tmp_path):
    import shutil
    from lav_b200.datasets import TemporalLiDARPaintedDataset
    root = tmp_path / "rec"
    shutil.copytree(camera_recording / "data", root / "data")
    os.remove(root / "data" / "traj_001" / "kv" / "tel_rgb_00002")
    t_cfg, _ = configs(root, tmp_path)
    ds = TemporalLiDARPaintedDataset(t_cfg, device="cpu")
    idx = ds.index.index((1, 2))
    ds.prepare(idx, *ds.no_draw())                                       # without the cameras nothing is missing
    with pytest.raises(LavbError, match="tel_rgb_00002"):
        ds.prepare(idx, *ds.no_draw(), cameras=True)
