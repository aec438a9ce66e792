"""CPU: the host half of online painting (lav_b200.evaluate --seg-weights): the frame table and staged images of
TemporalLiDARPaintedDataset.stage_batch against load_img, the sweeps' frame slots, a recording without any lidar_sem key, the
errors for a missing or wrongly sized camera image, and the CLI flag, on a synthetic 3-camera recording (PNG and JPEG
trajectories)."""
import os
import shutil

import numpy as np
import pytest
import torch
import yaml

from lav_b200 import synth
from lav_b200.capi import LavbError
from lav_b200.datasets import TemporalBatchLoader, TemporalLiDARPaintedDataset, load_img

CONFIG = dict(num_plan=20, num_frame_stack=2, seg_channels=[4, 6, 7, 10], max_lidar_points=2000, camera_x=1.5, camera_z=2.4,
              camera_yaws=[-120, -60, 0, 60, 120], angle_jitter=20, stack_loc_jitter=0.4, stack_ori_jitter=0.1,
              max_pedestrian_radius=10, max_vehicle_radius=25, max_mot_vehicle_radius=15, max_objs=20, min_x=-10, max_x=70,
              min_y=-40, max_y=40, pixels_per_meter=4, percentage_data=1.0, all_towns=True)


def write_recording(root, n_traj=3, n_frames=32):
    """a recording with the painting cameras' images; -> its config path."""
    synth.record_trajectories(os.path.join(root, "data"), n_traj, n_frames, images=True, n_cameras=3)
    path = os.path.join(root, "config.yaml")
    with open(path, "w") as f:
        yaml.safe_dump(dict(CONFIG, data_dir=os.path.join(root, "data")), f)
    return path


@pytest.fixture(scope="module")
def rec(tmp_path_factory):
    return write_recording(str(tmp_path_factory.mktemp("online_paint")))


def staged_batches(ds, bs, n_batches=None):
    """the ordered loader's host tables of the first batches, built as the loader builds them (prepare with paint, then
    stage_batch), without any device work."""
    loader = TemporalBatchLoader(ds, bs, drop_last=False, num_workers=3, ordered=True, seg_model=object())
    order = loader.shard(0)
    batches = [order[k:k + bs] for k in range(0, len(order), bs)][:n_batches]
    _, gen = loader.generators(0)
    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(3) as pool:
        for idxs in batches:
            hs = loader._prepare(pool, idxs, [ds.no_draw() for _ in idxs])
            yield idxs, hs, ds.stage_batch(hs, gen, pool)


@pytest.mark.parametrize("bs", [1, 4, 5, 32])
def test_frame_table_lists_each_frame_once_and_stages_its_images(rec, bs):
    ds = TemporalLiDARPaintedDataset(rec, device="cpu")
    assert len(ds) == 36 and len(ds.paths) == 3
    seen_boundary = False
    for idxs, hs, st in staged_batches(ds, bs, None if bs >= 5 else 10):
        pairs, imgs = st["paint"]["pairs"], st["paint"]["images"].numpy()
        assert len(set(pairs)) == len(pairs) and imgs.shape == (len(pairs), 3, 288, 256, 3) and imgs.dtype == np.uint8
        want = []
        for idx in idxs:
            traj, i = ds.index[int(idx)]
            want += [(traj, f) for f in range(i, i - 3, -1) if f >= 0]
        assert pairs == list(dict.fromkeys(want))                                   # first-use order, each pair once
        seen_boundary |= len({t for t, _ in pairs}) > 1
        slots = st["lidar"]["slots"].numpy()
        assert len(slots) == len(want) == len(st["lidar"]["sweeps"])
        assert [pairs[s] for s in slots] == want                                    # each sweep's slot names its own frame
        assert st["lidar"]["raw"].shape == (sum(len(sw[0]) for h in hs for sw in h["sweeps"]), 4)
        for f, (traj, i) in enumerate(pairs):
            env = ds.env(traj)
            for c in range(3):
                assert np.array_equal(imgs[f, c], load_img(env, f"rgb_{c}", i)), (traj, i, c)
    if bs >= 5:
        assert seen_boundary
    if bs == 32:                                                                    # consecutive samples share frames
        _, _, st = next(staged_batches(ds, bs, 1))
        assert len(st["paint"]["pairs"]) < 3 * 32


def test_the_raw_rows_are_the_stored_paths_first_columns(rec):
    ds = TemporalLiDARPaintedDataset(rec, device="cpu")
    idxs = [0, 1, 2, 3, 14]
    gen = lambda: torch.Generator().manual_seed(5)
    stored = ds.stage_batch([ds.prepare(i, *ds.no_draw()) for i in idxs], gen())["lidar"]
    online = ds.stage_batch([ds.prepare(i, *ds.no_draw(), paint=True) for i in idxs], gen())["lidar"]
    assert np.array_equal(online["raw"].numpy(), stored["raw"].numpy()[:, :4])
    assert np.array_equal(online["rows"].numpy(), stored["rows"].numpy()) and online["nums"] == stored["nums"]
    assert online["sweeps"].tobytes() == stored["sweeps"].tobytes() and "slots" not in stored


def test_prepare_paint_reads_no_lidar_sem(rec, tmp_path):
    data = str(tmp_path / "data")
    shutil.copytree(yaml.safe_load(open(rec))["data_dir"], data)
    removed = 0
    for kv in (os.path.join(data, t, "kv") for t in os.listdir(data)):
        for k in os.listdir(kv):
            if k.startswith("lidar_sem_"):
                os.remove(os.path.join(kv, k))
                removed += 1
    assert removed > 0
    ds = TemporalLiDARPaintedDataset(rec, device="cpu", overrides=dict(data_dir=data))
    with pytest.raises(TypeError):                                                  # the stored path needs lidar_sem
        ds.prepare(3, *ds.no_draw())
    h = ds.prepare(3, *ds.no_draw(), paint=True)
    assert [sw[1] for sw in h["sweeps"]] == [3, 2, 1] and all(sw[0].shape[1] == 4 for sw in h["sweeps"])
    _, _, st = next(staged_batches(ds, 6, 1))
    assert len(st["paint"]["pairs"]) == 6


@pytest.mark.parametrize("fault", ["missing", "size"])
def test_a_bad_camera_image_is_refused_naming_the_key(rec, tmp_path, fault):
    import cv2
    src = yaml.safe_load(open(rec))["data_dir"]
    data = str(tmp_path / "data")
    shutil.copytree(src, data)
    traj = sorted(os.listdir(data))[1]
    key = os.path.join(data, traj, "kv", "rgb_1_00004")
    if fault == "missing":
        os.remove(key)
    else:
        img = cv2.imdecode(np.fromfile(key, np.uint8), cv2.IMREAD_COLOR)
        with open(key, "wb") as f:
            f.write(cv2.imencode(".png", img[:, :255])[1].tobytes())
    ds = TemporalLiDARPaintedDataset(rec, device="cpu", overrides=dict(data_dir=data))
    with pytest.raises(LavbError, match=rf"{traj}.*rgb_1_00004" + (" is missing" if fault == "missing" else " is 255 x 288")):
        for _ in staged_batches(ds, 5):
            pass
    ok = TemporalLiDARPaintedDataset(rec, device="cpu", overrides=dict(data_dir=data))
    for idxs, hs, st in staged_batches(ok, 4, 1):                                   # trajectory 0 does not need that frame
        assert len(st["paint"]["pairs"]) == 4


def test_cli_parses_seg_weights_and_a_plain_result_has_no_painting():
    import lav_b200.evaluate as E
    base = ["--data-dir", "d", "--lidar-weights", "l.th", "--uniplanner-weights", "u.th"]
    assert E.parse_args(base).seg_weights is None
    args = E.parse_args(base + ["--seg-weights", "seg_1.th", "--brake", "--bra-weights", "b.th", "--forecast"])
    assert args.seg_weights == "seg_1.th" and args.brake and args.forecast
    acc = (E.Scores(), E.ForecastScores(), E.DetectedForecastScores(), E.PlanSafetyScores(), E.DetBoxScores(), E.BrakeScores(),
           E.PaintingCount())
    assert "painting" not in E.summarize(acc, "f16", False, False, False, 20)
    acc[6].frames = 7
    other = E.PaintingCount()
    other.frames = 5
    acc[6].extend(other)
    assert E.summarize(acc, "f16", False, False, False, 20, painting=True)["painting"] == dict(frames=12, images=36)
