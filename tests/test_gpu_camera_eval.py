"""GPU: ops.seg_confusion against the numpy statement of tests/test_camera_eval_cpu.py (random, exact-integer and NaN inputs, every
rejection), against argmax + bincount of RGBSegmentationModel.forward_nhwc's materialised logits, and lav_b200.evaluate_rgb on a
synthetic recording with seeded models, against the statement, the agent's brake branch and itself at another batch size; plus
its CLI."""
import ctypes as C
import json

import numpy as np
import pytest
import torch

from lav_b200 import capi, ops, synth
from lav_b200.capi import LavbError
from tests import test_camera_eval_cpu as R
from tests import util

pytestmark = pytest.mark.gpu

# the fp32 fmaf chain of 16 products against fp64: a pixel whose top two fp64 logits lie within this fraction of its logit
# scale sum_c |f w| + |b| may take either class
KERNEL_TIE_REL = 1e-5


def random_inputs(n, h, w, c, half, seed, dev):
    rs = np.random.RandomState(seed)
    feat = rs.randn(n, h // 2, w // 2, 16).astype(np.float32)
    table = np.zeros(520, np.float32)
    table[:512].reshape(2, 2, 16, 8)[..., :c] = rs.randn(2, 2, 16, c) * 0.5
    table[512:512 + c] = rs.randn(c) * 0.1
    labels = rs.randint(0, 23, (n, h, w)).astype(np.uint8)
    labels[:, ::5, ::3] = 255
    channels = list(rs.choice(np.arange(1, 23), c - 1, replace=False))
    f = torch.from_numpy(feat).to(dev)
    if half:
        f = f.to(ops.h16())
    return f, torch.from_numpy(table).to(dev), torch.from_numpy(labels).to(dev), ops.sem_class_table(channels)


def check_against_statement(got, feat, table, labels, lut, c, rel=KERNEL_TIE_REL, budget=1e-3):
    """counts equal the statement's except at the pixels whose top two fp64 logits lie within rel x their scale: those are
    counted, held to ``budget`` of the pixels, and may sit in either class's bin of their recorded row."""
    logits, scale = R.seg_logits_ref(feat, table, c)
    top2 = np.sort(logits, -1)[..., -2:]
    close = (top2[..., 1] - top2[..., 0]) <= rel * scale.max(-1)
    want = R.seg_confusion_ref(feat, table, labels, lut, c, logits=logits)
    gt = lut[labels]
    amb = np.zeros_like(want)
    for i in range(len(want)):
        for g in range(c):
            amb[i, g * c:(g + 1) * c] = int((close[i] & (gt[i] == g)).sum())
    assert np.all(np.abs(got - want) <= amb), np.argwhere(np.abs(got - want) > amb)[:5]
    assert np.array_equal(got.reshape(len(got), -1)[:, :c * c].reshape(-1, c, c).sum(-1),
                          want[:, :c * c].reshape(-1, c, c).sum(-1))              # each recorded row keeps its pixel count
    assert np.array_equal(got[:, -1], want[:, -1])
    assert close.sum() <= budget * close.size, close.sum()
    return int(close.sum())


SHAPES = [(1, 288, 256), (7, 288, 256), (7, 2, 2), (7, 2, 256)]


@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("c", [2, 5, 8])
@pytest.mark.parametrize("shape", SHAPES + [(96, 288, 256)])
def test_kernel_equals_the_statement(cuda, shape, c, half):
    n, h, w = shape
    if n == 96 and c != 5:
        pytest.skip("96 images at C = 5 only")
    feat, table, labels, lut = random_inputs(n, h, w, c, half, seed=n * 100 + c * 10 + h + half, dev=cuda)
    got = ops.seg_confusion(feat, table, labels, lut, c).cpu().numpy()
    assert got.shape == (n, c * c + 1) and got[:, :-1].sum() == n * h * w
    check_against_statement(got, feat.float().cpu().numpy(), table.cpu().numpy(), labels.cpu().numpy(), lut, c)


@pytest.mark.parametrize("half", [False, True])
def test_exact_integer_logits_give_equal_counts(cuda, half):
    """small integer features, weights and biases: every logit is exact in fp32 (and h16), so the counts are bit-equal, ties
    (frequent here) going to the lower class."""
    feat, table, labels, lut = R.integer_case()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    f = t(feat).to(ops.h16()) if half else t(feat)
    assert np.array_equal(ops.seg_confusion(f, t(table), t(labels), lut, 3).cpu().numpy(),
                          R.seg_confusion_ref(feat, table, labels, lut, 3))
    rs = np.random.RandomState(7)
    for c in (2, 5, 8):
        feat = rs.randint(-2, 3, (5, 24, 40, 16)).astype(np.float32)
        table = np.zeros(520, np.float32)
        table[:512].reshape(2, 2, 16, 8)[..., :c] = rs.randint(-1, 2, (2, 2, 16, c))
        table[512:512 + c] = rs.randint(-1, 2, c)
        labels = rs.choice([0, 4, 6, 7, 10, 12, 255], (5, 48, 80)).astype(np.uint8)
        lut = ops.sem_class_table([4, 6, 7, 10, 6, 12, 4][:c - 1])
        f = t(feat).to(ops.h16()) if half else t(feat)
        got = ops.seg_confusion(f, t(table), t(labels), lut, c).cpu().numpy()
        want = R.seg_confusion_ref(feat, table, labels, lut, c)
        logits, _ = R.seg_logits_ref(feat, table, c)
        assert (np.sort(logits, -1)[..., -1] == np.sort(logits, -1)[..., -2]).mean() > 0.05      # ties occur
        assert np.array_equal(got, want), c


@pytest.mark.parametrize("half", [False, True])
def test_nan_features_are_invalid(cuda, half):
    feat, table, labels, lut = random_inputs(3, 16, 32, 5, half, seed=3, dev=cuda)
    f = feat.float().cpu().numpy()
    f[0, 1, 2, 7] = np.nan
    f[2, :, 5, 0] = np.nan                  # a whole column of feature pixels
    f[2, 3, 9, :] = np.inf                  # inf * w of both signs sums to NaN
    feat = torch.from_numpy(f).to(cuda).to(feat.dtype)
    got = ops.seg_confusion(feat, table, labels, lut, 5).cpu().numpy()
    logits, _ = R.seg_logits_ref(f, table.cpu().numpy(), 5)
    assert got[:, -1].tolist() == np.isnan(logits).any(-1).sum((1, 2)).tolist() and got[0, -1] == 4 and got[1, -1] == 0
    assert got[2, -1] >= 4 * 8
    check_against_statement(got, f, table.cpu().numpy(), labels.cpu().numpy(), lut, 5)


def test_malformed_calls_write_nothing(cuda):
    feat, table, labels, lut = random_inputs(4, 8, 12, 5, False, seed=9, dev=cuda)
    out = torch.full((4, 26), 0x5A5A5A5A, dtype=torch.int32, device=cuda)
    sentinel = out.clone()
    lib = capi.lib()
    p = lambda t: C.c_void_p(t.data_ptr())
    lutp = lambda a: np.ascontiguousarray(a, np.uint8).ctypes.data_as(C.c_void_p)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    bad_lut = lut.copy()
    bad_lut[200] = 5
    calls = [dict(c=1), dict(c=9), dict(h=7), dict(w=13), dict(h=0), dict(n=65536), dict(n=-1), dict(lut=bad_lut),
             dict(dtype=7), dict(dtype=capi.BF16 if ops.h16() == torch.float16 else capi.F16), dict(feat=0), dict(out=0),
             dict(labels_off=1), dict(feat_off=4)]
    for bad in calls:
        a = dict(dtype=capi.F32, n=4, c=5, h=8, w=12, lut=lut, feat=p(feat), out=p(out))
        a.update(bad)
        fptr = a["feat"] if not isinstance(a["feat"], int) else C.c_void_p(a["feat"])
        if "feat_off" in bad:
            fptr = C.c_void_p(feat.data_ptr() + 4)
        lab = C.c_void_p(labels.data_ptr() + bad.get("labels_off", 0))
        optr = a["out"] if not isinstance(a["out"], int) else C.c_void_p(a["out"])
        code = lib.lavb_seg_confusion(fptr, a["dtype"], p(table), lab, lutp(a["lut"]), a["n"], a["c"], a["h"], a["w"], optr, stream)
        assert code != 0, bad
        torch.cuda.synchronize()
        assert torch.equal(out, sentinel), bad
    with pytest.raises(LavbError):
        ops.seg_confusion(feat, table, labels, bad_lut, 5, out=out)
    assert torch.equal(out, sentinel)
    assert lib.lavb_seg_confusion(p(feat), capi.F32, p(table), p(labels), lutp(lut), 0, 5, 8, 12, p(out), stream) == 0
    torch.cuda.synchronize()
    assert torch.equal(out, sentinel)                                             # n = 0 writes nothing either
    ops.seg_confusion(feat, table, labels, lut, 5, out=out)
    assert int(out[:, :25].sum()) == 4 * 8 * 12 and not (out == 0x5A5A5A5A).any()   # every element of the rows written


# the documented difference between the kernel's logits and forward_nhwc's materialised ones, relative to the logit scale
MATERIALISED_TIE_REL = {"fp32": 1e-5, "f16": 5e-3}


@pytest.mark.parametrize("precision", ["fp32", "f16"])
def test_kernel_equals_argmax_of_the_materialised_logits(cuda, precision):
    sm, _ = util.seg_model(cuda)
    sm.set_precision(precision)
    imgs = torch.cat([synth.rgb_frames(tag=f"mat{k}", smooth=True) for k in range(4)]).to(cuda)
    labels = torch.from_numpy(np.random.RandomState(5).choice([0, 4, 6, 7, 10, 1, 22], (12, 288, 256)).astype(np.uint8)).to(cuda)
    lut = ops.sem_class_table([4, 6, 7, 10])
    with torch.no_grad():
        feat, table, c = sm.forward_features_nhwc(imgs)
        logits = sm.forward_nhwc(imgs)
    got = ops.seg_confusion(feat, table, labels, lut, c).cpu().numpy()
    lg = logits.double().cpu().numpy()
    top2 = np.sort(lg, -1)[..., -2:]
    close = (top2[..., 1] - top2[..., 0]) < MATERIALISED_TIE_REL[precision] * np.abs(lg).max()
    pred = torch.from_numpy(lg).argmax(-1)
    gt = torch.from_numpy(lut[labels.cpu().numpy()]).long()
    want = np.stack([torch.bincount((gt[i] * c + pred[i])[~torch.from_numpy(close[i])], minlength=c * c).numpy() for i in range(12)])
    diff = got[:, :c * c] - want
    assert np.all(diff >= 0) and np.array_equal(diff.sum(1), close.sum((1, 2))) and not got[:, -1].any()
    assert close.mean() < 5e-2, close.mean()
    assert len(np.unique(pred.numpy())) > 1                                 # the seeded model predicts more than one class


# ----------------------------------------------------------------------------- the evaluator
@pytest.fixture(scope="module")
def recording(tmp_path_factory):
    root = tmp_path_factory.mktemp("camrec")
    synth.record_trajectories(str(root), n_traj=2, n_frames=9, n_points=64, images=True, n_cameras=3)
    return root


def brake_model():
    from lav_b200.heads import RGBBrakePredictionModel
    m = RGBBrakePredictionModel([4, 6, 7, 10]).eval()
    m.load_state_dict(synth.fill_state_dict_(m.state_dict(), seed=13))
    return m


def run(recording, tmp_path, precision, batch_size, cuda):
    from lav_b200.datasets import CameraDataset
    from lav_b200.evaluate_rgb import evaluate_rgb
    sm, _ = util.seg_model()
    ds = CameraDataset(R.write_camera_config(tmp_path / "c.yaml", recording, 3), device=cuda)
    seen = []
    on_batch = lambda b, feat, counts, p: seen.append(dict(rgbs=b["rgbs"].clone(), tel=b["tel"].clone(), labels=b["labels"].cpu().numpy(),
                                                           feat=feat.float().cpu().numpy(), counts=counts, probs=p))
    res = evaluate_rgb(sm, brake_model(), ds, batch_size=batch_size, precision=precision, num_workers=2, on_batch=on_batch)
    return res, seen, sm


@pytest.mark.parametrize("precision", ["fp32", "f16"])
def test_evaluate_rgb_against_statement_agent_and_batch_size(cuda, recording, tmp_path, precision):
    from lav_b200.agent import StaticFramePipeline, math_mode
    res, seen, sm = run(recording, tmp_path, precision, 4, cuda)       # 12 frames: 4 + 4 + 4
    assert res["samples"] == 12 and res["precision"] == precision and [len(s["rgbs"]) for s in seen] == [4, 4, 4]
    table = sm.erfnet._plan_get(cuda, sm.erfnet._build)[2].cpu().numpy()
    lut = ops.sem_class_table([4, 6, 7, 10])
    conf = np.zeros((3, 5, 5), np.int64)
    for s in seen:                                                      # each batch's counts = the statement on its features
        check_against_statement(s["counts"], s["feat"], table, s["labels"].reshape(-1, 288, 256), lut, 5)
        conf += s["counts"][:, :25].reshape(-1, 3, 5, 5).sum(0)
    assert res["seg"]["confusion"] == conf.sum(0).tolist()
    assert [d["confusion"] for d in res["seg"]["per_camera"]] == conf.tolist() and res["seg"]["classes"] == [0, 4, 6, 7, 10]
    # the brake probabilities are the agent's: the brake branch of the frame pipeline on the same frames
    lm, _ = util.lidar_model()
    from tests.test_heads_cpu import uniplanner
    pipe = StaticFramePipeline(util.seg_model()[0], lm, uniplanner()[0], brake_model(), batch=4, n_points=256, device=cuda,
                               precision=precision, use_graphs=False)
    for s in seen:
        pipe.rgbs.copy_(s["rgbs"])
        pipe.tels.copy_(s["tel"])
        with torch.no_grad(), math_mode(precision):
            want = pipe._brake().float().cpu().numpy()
        assert np.array_equal(s["probs"], want), np.abs(s["probs"] - want).max()
    # another batch size (12 = 5 + 5 + 2): the same counts; the brake probabilities within the batch-size dependence of cuBLAS
    res5, seen5, _ = run(recording, tmp_path, precision, 5, cuda)
    assert [len(s["rgbs"]) for s in seen5] == [5, 5, 2]
    assert res5["seg"] == res["seg"]
    p4, p5 = np.concatenate([s["probs"] for s in seen]), np.concatenate([s["probs"] for s in seen5])
    assert np.abs(p4 - p5).max() <= (1e-6 if precision == "fp32" else 2e-3)
    assert res5["brake"]["frames"] == res["brake"]["frames"] == 12


def test_cli_writes_json(cuda, recording, tmp_path):
    from lav_b200 import evaluate_rgb
    sm, sd = util.seg_model()
    torch.save(sd, tmp_path / "seg.th")
    torch.save(brake_model().state_dict(), tmp_path / "bra.th")
    cfg = R.write_camera_config(tmp_path / "c.yaml", "unused", 3)
    out = tmp_path / "r.json"
    res = evaluate_rgb.main(["--config-path", cfg, "--data-dir", str(recording), "--seg-weights", str(tmp_path / "seg.th"),
                             "--bra-weights", str(tmp_path / "bra.th"), "--batch-size", "5", "--num-workers", "2", "--json", str(out)])
    assert json.load(open(out)) == json.loads(json.dumps(res))
    assert res["samples"] == 12 and 0 <= res["seg"]["pixel_accuracy"] <= 1 and res["brake"]["positives"] >= 0
    only = evaluate_rgb.main(["--config-path", cfg, "--data-dir", str(recording), "--bra-weights", str(tmp_path / "bra.th"),
                              "--precision", "fp32", "--num-workers", "2"])
    assert "seg" not in only and only["brake"]["frames"] == 12
