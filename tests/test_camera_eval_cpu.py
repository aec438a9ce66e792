"""CPU: the numpy statement of lavb_seg_confusion (used by tests/test_gpu_camera_eval.py) with known answers, the tag -> class
table against filter_sem, the host reductions of lav_b200.evaluate_rgb on hand-worked cases, and the host half of
datasets.CameraDataset / CameraBatchLoader against a direct cv2.imdecode loop over a synthetic recording."""
import math

import numpy as np
import pytest

from lav_b200 import ops, synth
from lav_b200.evaluate_rgb import brake_metrics, seg_metrics


# ----------------------------------------------------------------------------- the statement of the kernel
def seg_logits_ref(feat, table, n_classes):
    """fp64 logits of output_conv from the packed 520-float table: feat (N, h, w, 16) -> (N, 2h, 2w, C), and the scale
    sum_c |f_c w_ck| + |b_k| of each logit (for error bounds)."""
    f = np.asarray(feat, np.float64)
    t = np.asarray(table, np.float64)
    w, b = t[:512].reshape(2, 2, 16, 8)[..., :n_classes], t[512:512 + n_classes]
    n, h, wd, _ = f.shape
    logits = np.zeros((n, 2 * h, 2 * wd, n_classes))
    scale = np.zeros_like(logits)
    for pv in range(2):
        for pu in range(2):
            logits[:, pv::2, pu::2] = np.einsum("nyxc,ck->nyxk", f, w[pv, pu]) + b
            scale[:, pv::2, pu::2] = np.einsum("nyxc,ck->nyxk", np.abs(f), np.abs(w[pv, pu])) + np.abs(b)
    return logits, scale


def seg_confusion_ref(feat, table, labels, lut, n_classes, logits=None):
    """(N, C*C + 1) int64: per image confusion[lut[label]][argmax logit] (first index of the maximum: ties to the lower class), then
    the pixels with a NaN logit, which count nowhere else."""
    if logits is None:
        logits, _ = seg_logits_ref(feat, table, n_classes)
    c = n_classes
    invalid = np.isnan(logits).any(-1)
    pred = np.argmax(np.where(np.isnan(logits), -np.inf, logits), -1)
    gt = np.asarray(lut)[np.asarray(labels)]
    out = np.zeros((len(logits), c * c + 1), np.int64)
    for i in range(len(logits)):
        ok = ~invalid[i]
        out[i, :c * c] = np.bincount((gt[i][ok] * c + pred[i][ok]).ravel(), minlength=c * c)
        out[i, c * c] = int(invalid[i].sum())
    return out


def filter_sem_loop(sem, labels):
    """filter_sem (lav/utils/__init__.py:3-8), restated."""
    resem = np.zeros_like(sem)
    for i, label in enumerate(labels):
        resem[sem == label] = i + 1
    return resem


def integer_case():
    """one feature pixel, C = 3, logits small exact integers: phase (0,0) -> [0, 2, 1], (0,1) -> [3, 3, 1] (a tie), (1,0) ->
    [0, 0, 5], (1,1) -> [1, 1, 1]; tags [[4, 6], [6, 200]] with seg_channels [4, 6]."""
    feat = np.zeros((1, 1, 1, 16), np.float32)
    feat[..., 0] = 1
    w = np.zeros((2, 2, 16, 8), np.float32)
    w[0, 0, 0, :3], w[0, 1, 0, :3], w[1, 0, 0, :3], w[1, 1, 0, :3] = [0, 2, 1], [3, 3, 1], [0, 0, 5], [1, 1, 1]
    table = np.concatenate([w.ravel(), np.zeros(8, np.float32)])
    labels = np.array([[[4, 6], [6, 200]]], np.uint8)
    return feat, table, labels, ops.sem_class_table([4, 6])


def test_statement_known_answers():
    feat, table, labels, lut = integer_case()
    got = seg_confusion_ref(feat, table, labels, lut, 3)
    want = np.zeros((1, 10), np.int64)
    want[0, 1 * 3 + 1] += 1          # tag 4 -> class 1, predicted 1
    want[0, 2 * 3 + 0] += 1          # tag 6 -> class 2, a tie of classes 0 and 1 -> 0
    want[0, 2 * 3 + 2] += 1          # tag 6 -> class 2, predicted 2
    want[0, 0 * 3 + 0] += 1          # tag 200 (unlisted) -> background, a three-way tie -> 0
    assert np.array_equal(got, want)
    feat[..., 5] = np.nan            # NaN * 0 is NaN: every logit of the pixel is NaN
    assert np.array_equal(seg_confusion_ref(feat, table, labels, lut, 3), np.array([[0] * 9 + [4]]))


def test_statement_bias_and_phases():
    """bias only (zero features): every pixel takes the largest bias; the phases pick their own weights."""
    feat = np.zeros((2, 2, 3, 16), np.float32)
    table = np.zeros(520, np.float32)
    table[512:517] = [0.5, -1, 2, 2, 0]          # classes 2 and 3 tie: 2
    labels = np.zeros((2, 4, 6), np.uint8)
    got = seg_confusion_ref(feat, table, labels, np.zeros(256, np.uint8), 5)
    assert got[:, 0 * 5 + 2].tolist() == [24, 24] and got.sum() == 48
    feat[0, 0, 0, 3] = 1
    w = table[:512].reshape(2, 2, 16, 8)
    w[1, 0, 3, 4] = 10                            # only output pixel (1, 0) of feature pixel (0, 0) of image 0 changes class
    got = seg_confusion_ref(feat, table, labels, np.zeros(256, np.uint8), 5)
    assert got[0, 4] == 1 and got[0, 2] == 23 and got[1, 2] == 24


@pytest.mark.parametrize("channels", [[4, 6, 7, 10], [4, 10, 18], [7, 4, 7], [0, 255, 3], [], [12, 12, 12, 1, 2, 3, 4]])
def test_class_table_is_filter_sem(channels):
    tags = np.arange(256, dtype=np.uint8)
    assert np.array_equal(ops.sem_class_table(channels)[tags], filter_sem_loop(tags, channels))


# ----------------------------------------------------------------------------- host reductions
def test_seg_metrics_by_hand():
    m = seg_metrics([[5, 1, 0], [2, 3, 0], [0, 0, 0]], invalid=7)
    assert m["iou"] == [5 / 8, 3 / 6, None]                     # class 2 never recorded nor predicted: null
    assert m["miou"] == pytest.approx((5 / 8 + 3 / 6) / 2)    # over the non-null classes only
    assert m["miou_fg"] == pytest.approx(0.5)
    assert m["pixel_accuracy"] == pytest.approx(8 / 11)
    assert m["precision"] == [5 / 7, 3 / 4, None] and m["recall"] == [5 / 6, 3 / 5, None]
    assert m["invalid_pixels"] == 7 and m["confusion"] == [[5, 1, 0], [2, 3, 0], [0, 0, 0]]
    empty = seg_metrics(np.zeros((2, 2), np.int64))
    assert empty["iou"] == [None, None] and empty["miou"] is None and empty["pixel_accuracy"] is None
    assert seg_metrics([[4, 0], [0, 0]])["miou_fg"] is None


def test_brake_metrics_by_hand():
    p = [0.1, 0.6, 0.2, 0.0, 1.0, 0.6, 0.0, 1.0]
    y = [1, 1, 0, 0, 1, 0, 1, 0]
    m = brake_metrics(p, y)
    assert m["frames"] == 8 and m["positives"] == 4
    # p > 0.1 strictly: 0.1 itself does not brake
    assert m["at_0.1"] == dict(precision=2 / 5, recall=0.5, accuracy=3 / 8, false_brake_rate=3 / 4)
    assert m["at_0.5"] == dict(precision=0.5, recall=0.5, accuracy=0.5, false_brake_rate=0.5)
    # the clamp: log(0) and log(1 - 1) count as -100
    assert m["bce"] == pytest.approx((-math.log(0.1) - math.log(0.6) - math.log(0.8) - math.log(0.4) + 200) / 8, rel=1e-12)
    # ranked 1.0 (y), 1.0 (n), 0.6 (y), 0.6 (n), 0.2, 0.1 (y), 0.0, 0.0 (y): ties keep frame order
    assert m["ap"] == pytest.approx(0.25 * (1 + 2 / 3 + 0.5 + 0.5))


def test_brake_rule_on_fp32_probabilities():
    """the model's probabilities are fp32: the fp32 number nearest 0.1 is above 0.1 and brakes, as float(pred_bra) > 0.1 does in
    the agent; the one below it does not."""
    near = np.float32(0.1)
    below = np.nextafter(near, np.float32(0))
    m = brake_metrics(np.array([near, below], np.float32), [1, 1])
    assert m["at_0.1"]["recall"] == 0.5
    none = brake_metrics(np.zeros(0, np.float32), np.zeros(0, np.int64))
    assert none["ap"] is None and none["bce"] is None and none["at_0.1"]["accuracy"] is None
    assert brake_metrics([0.3], [0])["ap"] is None and brake_metrics([0.3], [0])["at_0.1"]["false_brake_rate"] == 1.0


# ----------------------------------------------------------------------------- the loader's host half
def write_camera_config(path, data_dir, n_cameras, num_plan=3, seg_channels=(4, 6, 7, 10)):
    import yaml
    yaws = {3: [-60, 0, 60], 5: [-120, -60, 0, 60, 120]}[n_cameras]
    cfg = dict(data_dir=str(data_dir), percentage_data=1.01, all_towns=True, num_plan=num_plan, camera_yaws=yaws,
               crop_tel_bottom=96, seg_channels=list(seg_channels))
    with open(path, "w") as f:
        yaml.safe_dump(cfg, f)
    return str(path)


@pytest.fixture(scope="module", params=[3, 5])
def camera_recording(request, tmp_path_factory):
    root = tmp_path_factory.mktemp(f"cams{request.param}")
    synth.record_trajectories(str(root), n_traj=2, n_frames=7, n_points=64, images=True, n_cameras=request.param)
    return root, request.param


def direct(path, key):
    import cv2
    from lav_b200 import data_paint
    data = data_paint.open_env(path).get(key)
    img = cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR if "rgb" in key else cv2.IMREAD_GRAYSCALE)
    return img[..., ::-1] if img.ndim == 3 else img


class KeyLog:
    def __init__(self, env, log):
        self.env, self.log = env, log

    def get(self, key):
        self.log.append(key)
        return self.env.get(key)


@pytest.mark.parametrize("seg,brake", [(True, True), (True, False), (False, True)])
def test_loader_equals_a_direct_decode_loop(camera_recording, tmp_path, seg, brake):
    from lav_b200.datasets import CameraBatchLoader, CameraDataset
    root, ncam = camera_recording
    ds = CameraDataset(write_camera_config(tmp_path / "c.yaml", root, ncam), seg=seg, brake=brake, device="cpu")
    assert len(ds) == 2 * (7 - 3)
    mid = [ncam // 2 - 1, ncam // 2, ncam // 2 + 1]
    assert mid == ([0, 1, 2] if ncam == 3 else [1, 2, 3])
    assert ds.cams == (list(range(ncam)) if seg else mid)
    log = []
    env = ds.env
    ds.env = lambda traj: KeyLog(env(traj), log)
    batches = [b for b, _ in CameraBatchLoader(ds, 3, num_workers=2).staged_batches()]
    assert [len(b["rgbs"]) for b in batches] == [3, 3, 2]                   # frame order, the last batch short
    got = {k: np.concatenate([b[k].numpy() for b in batches]) for k in batches[0]}
    for j, (traj, i) in enumerate(ds.index):
        path = ds.paths[traj]
        for p, c in enumerate(ds.cams):
            assert np.array_equal(got["rgbs"][j, p], direct(path, f"rgb_{c}_{i:05d}"))      # BGR -> RGB
            if seg:
                assert np.array_equal(got["labels"][j, p], direct(path, f"sem_{c}_{i:05d}"))
        if brake:
            assert [ds.cams[p] for p in ds.brake_cams] == mid
            tel = direct(path, f"tel_rgb_{i:05d}")
            assert tel.shape == (288, 480, 3) and np.array_equal(got["tel"][j], tel[:-96])
            assert got["tel"].shape[1:] == (192, 480, 3)
            assert got["bra"][j] == np.frombuffer(ds.env(traj).env.get(f"bra_{i:05d}"), np.uint8)[0]
    read = {k.rsplit("_", 1)[0] for k in log}
    assert read == ({f"rgb_{c}" for c in ds.cams} | ({f"sem_{c}" for c in ds.cams} if seg else set())
                    | ({"tel_rgb", "bra"} if brake else set()))
    assert got["rgbs"].dtype == np.uint8 and got["rgbs"].shape[2:] == (288, 256, 3)


def test_jpeg_trajectory_and_label_tags(camera_recording):
    """trajectory 1 stores its colour images as JPEG, trajectory 0 as PNG; the label images hold listed tags, unlisted tags and
    background."""
    from lav_b200 import data_paint
    root, _ = camera_recording
    envs = [data_paint.open_env(str(root / f"traj_{k:03d}")) for k in range(2)]
    assert envs[0].get("rgb_0_00000")[:4] == b"\x89PNG" and envs[0].get("tel_rgb_00000")[:4] == b"\x89PNG"
    assert envs[1].get("rgb_0_00000")[:2] == b"\xff\xd8" and envs[1].get("tel_rgb_00000")[:2] == b"\xff\xd8"
    tags = set(np.unique(np.concatenate([direct(str(root / "traj_000"), f"sem_0_{i:05d}").ravel() for i in range(7)])).tolist())
    assert 0 in tags and tags & {4, 6, 7, 10} and tags - {0, 4, 6, 7, 10}


def test_images_leave_the_other_keys_unchanged(tmp_path):
    import os
    a = synth.record_trajectories(str(tmp_path / "a"), n_traj=2, n_frames=3, n_points=32)
    b = synth.record_trajectories(str(tmp_path / "b"), n_traj=2, n_frames=3, n_points=32, images=True)
    for pa, pb in zip(a, b):
        ka, kb = sorted(os.listdir(os.path.join(pa, "kv"))), sorted(os.listdir(os.path.join(pb, "kv")))
        assert set(ka) < set(kb)
        for k in ka:
            assert open(os.path.join(pa, "kv", k), "rb").read() == open(os.path.join(pb, "kv", k), "rb").read(), k
