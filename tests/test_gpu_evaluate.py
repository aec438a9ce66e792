"""GPU: ops.eval_batch against the numpy statement of tests/test_evaluate_cpu.py, its argument checks and known answers, and
lav_b200.evaluate against a plain per-sample loop on a synthetic recording, plus its CLI."""
import json

import numpy as np
import pytest
import torch

from lav_b200 import ops, synth
from lav_b200.capi import LavbError
from tests import test_evaluate_cpu as R
from tests.test_temporal_dataset_cpu import write_config

pytestmark = pytest.mark.gpu


def random_batch(B, seed, dev):
    """seg, gt, packed, actors, offsets, plan, ego_locs of B samples: peaks scattered around the actors' centres (some exactly on
    them, equal scores, small boxes), actors of classes 0 / 1 / 2 inside and outside the window; sample 0 has no actor and
    sample 1 no surviving peak (when B > 1)."""
    rs = np.random.RandomState(seed)
    seg = rs.rand(B, 320, 320, 3).astype(np.float32)
    seg[:, ::7] = 0.5                                                      # exactly 0.5 is not a prediction
    gt = (rs.rand(B, 9, 320, 320) < 0.3).astype(np.uint8)
    counts = rs.randint(0, 13, B)
    counts[0] = 0
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    actors = np.zeros((offsets[-1], 6), np.float32)
    actors[:, 0] = rs.uniform(-35, 5, len(actors))
    actors[:, 1] = rs.uniform(-10, 50, len(actors))
    actors[::5, :2] = np.round(actors[::5, :2] * 4) / 4                   # centres exactly on a pixel
    actors[:, 2:5] = rs.uniform(0, 3, (len(actors), 3))
    actors[:, 5] = rs.choice([0, 1, 1, 2], len(actors))
    n_det = 15
    packed = np.zeros((B, 7, 2 * n_det), np.float32)
    packed[:, 6] = 320
    for b in range(B):
        cx, cy = R.centres(actors[offsets[b]:offsets[b + 1]])
        for j in range(2 * n_det):
            if len(cx) and rs.rand() < 0.7:
                g = rs.randint(len(cx))
                x, y = np.clip(np.round(cx[g] + rs.randint(-20, 21) * rs.rand() ** 2), 0, 319), np.clip(np.round(cy[g] + rs.randint(-20, 21) * rs.rand() ** 2), 0, 319)
            else:
                x, y = rs.randint(0, 320), rs.randint(0, 320)
            packed[b, :6, j] = (np.round(rs.rand(), 1), y * 320 + x, rs.uniform(0, 2), rs.uniform(0, 2), 1.0, 0.0)
        packed[b, 0, rs.rand(2 * n_det) < 0.1] = -1e5
    if B > 1:
        packed[1, 0] = 0.1
    plan = rs.randn(B, 20, 2).astype(np.float32) * 5
    ego_locs = rs.randn(B, 21, 2).astype(np.float32) * 5
    t = lambda a: torch.from_numpy(a).to(dev)
    return t(seg), t(gt), t(packed), t(actors), offsets, t(plan), t(ego_locs)


def check_equal(got, want):
    """counts, scores and flags identical; ADE / FDE within 1e-6."""
    for k in ("iou", "ngt", "flags", "score"):
        g = got[k].numpy()
        assert np.array_equal(g, want[k]), (k, np.argwhere(g != want[k])[:5])
    assert np.abs(got["plan_err"].numpy() - want["plan_err"]).max() <= 1e-6


@pytest.mark.parametrize("B", [1, 7, 64])
@pytest.mark.parametrize("half", [False, True])
def test_eval_batch_equals_the_fp32_threshold_statement(cuda, B, half):
    """The kernel equals the numpy statement, whose score threshold is model_inference.score_kept: a packed score of exactly
    float32(0.2) (random_batch rounds scores to one decimal) is not a survivor, as in the reference."""
    seg, gt, packed, actors, offsets, plan, ego = random_batch(B, B + 100 * half, cuda)
    if half:
        seg = seg.to(ops.h16())
    v = ops.eval_views(ops.eval_batch(seg, gt, packed, actors, offsets, plan, ego).cpu(), B, packed.shape[2])
    want = R.eval_batch_ref(seg.float().cpu().numpy(), gt.cpu().numpy(), packed.cpu().numpy(), actors.cpu().numpy(), offsets,
                            plan.cpu().numpy(), ego.cpu().numpy())
    check_equal(v, want)
    f = v["flags"].numpy()
    at = packed.cpu().numpy()[:, 0] == np.float32(0.2)
    assert at.any() and not (f[at] & 16).any()
    if B > 1:
        assert (f & 1).any() and ((f & 16) & ~(f & 1)).any()              # matches and misses both occur
        assert not (f[1] & 16).any() and v["ngt"].numpy()[0].sum() == 0


def test_eval_batch_rejects_malformed_arguments_and_writes_nothing(cuda):
    seg, gt, packed, actors, offsets, plan, ego = random_batch(4, 5, cuda)
    size = ops.eval_batch(seg, gt, packed, actors, offsets, plan, ego).numel()
    out = torch.full((size,), 0xAB, dtype=torch.uint8, device=cuda)
    bad = [dict(offsets=np.array([0, 3, 2, 5, offsets[-1]], np.int32)),                   # not monotone
           dict(offsets=np.array([0, 1, 2, 3, len(actors) + 1], np.int32)),               # past the row count
           dict(offsets=np.array([-1, 1, 2, 3, 4], np.int32)),
           dict(offsets=offsets[:-1]),
           dict(seg=seg.double()), dict(seg=seg[..., :2].contiguous()), dict(seg=seg.permute(0, 2, 1, 3)),
           dict(gt=gt.float()), dict(gt=gt[:, :, :160].contiguous()), dict(gt=gt[:3]),
           dict(packed=packed[:, :6].contiguous()), dict(packed=packed[:, :, :29].contiguous()),
           dict(packed=torch.zeros((4, 7, 130), device=cuda)),                                 # more than 64 peaks per class
           dict(actors=actors[:, :5].contiguous()), dict(plan=plan[:, :19].contiguous()), dict(ego_locs=ego.double()),
           dict(plan=torch.zeros((4, 40, 2), device=cuda), ego_locs=torch.zeros((4, 41, 2), device=cuda)),   # more than 32 steps
           dict(actors=actors.cpu())]
    for kw in bad:
        args = dict(seg=seg, gt=gt, packed=packed, actors=actors, offsets=offsets, plan=plan, ego_locs=ego)
        args.update(kw)
        with pytest.raises(LavbError):
            ops.eval_batch(args["seg"], args["gt"], args["packed"], args["actors"], args["offsets"], args["plan"], args["ego_locs"],
                           out=out)
    torch.cuda.synchronize()
    assert bool((out == 0xAB).all())
    many = np.array([0, 0, 0, 0, 1025], np.int32)                                             # over 1024 actors in one sample
    with pytest.raises(LavbError):
        ops.eval_batch(seg, gt, packed, torch.zeros((1025, 6), device=cuda), many, plan, ego, out=out)
    torch.cuda.synchronize()
    assert bool((out == 0xAB).all())


def test_known_answers(cuda):
    from lav_b200.evaluate import average_precision
    B = 3
    seg, gt, packed, actors, offsets, plan, ego = random_batch(B, 9, cuda)
    gt[:, 1] = 0                                                            # a channel with no target, predicted nowhere
    perfect = gt[:, :3].permute(0, 2, 3, 1).float().contiguous()
    rs = np.random.RandomState(3)
    acts, offs, pk = [], [0], np.zeros((B, 7, 30), np.float32)
    pk[:, 0] = -1e5
    for b in range(B):
        n = 6 + b
        px, py = rs.choice(np.arange(40, 280, 7), n, replace=False), rs.randint(60, 250, n)
        typ = np.arange(n) % 2
        acts += [R.actor(x, y, t) for x, y, t in zip(px, py, typ)]
        offs.append(offs[-1] + n)
        used = [0, 0]
        for x, y, t in zip(px, py, typ):
            j = t * 15 + used[t]
            used[t] += 1
            pk[b, :6, j] = (0.3 + 0.1 * rs.rand(), y * 320 + x, 5, 5, 1, 0)
    pk[:, 6] = 320
    res = ops.eval_views(ops.eval_batch(perfect, gt, torch.from_numpy(pk).to(cuda), torch.tensor(acts, dtype=torch.float32, device=cuda),
                                        np.array(offs, np.int32), plan, ego).cpu(), B, 30)
    iou = res["iou"].numpy().sum(0)
    assert iou[0, 0] == iou[0, 1] > 0 and iou[2, 0] == iou[2, 1] > 0 and iou[1].tolist() == [0, 0]
    f = res["flags"].numpy()
    for c in range(2):
        s, fl = res["score"].numpy()[:, c * 15:(c + 1) * 15], f[:, c * 15:(c + 1) * 15]
        keep = (fl & 16) != 0
        n_gt = int(res["ngt"].numpy()[:, c].sum())
        assert keep.sum() == n_gt > 0
        for k in range(4):
            assert average_precision(s[keep], (fl[keep] >> k) & 1, n_gt) == 1.0


@pytest.fixture(scope="module")
def recording(tmp_path_factory, golden_dir):
    import os
    import yaml
    gold = np.load(os.path.join(golden_dir, "temporal_dataset.npz"))
    root = tmp_path_factory.mktemp("eval_rec")
    synth.record_trajectories(str(root / "data"), int(gold["n_traj"]), int(gold["n_frames"]), int(gold["seed"]))
    path = write_config(gold, str(root / "data"), root / "config.yaml")
    cfg = yaml.safe_load(open(path))
    cfg.update(num_features=[64, 64], backbone="cnn", crop_size=96, feature_x_jitter=1.5, feature_angle_jitter=20, num_cmds=6,
               num_plan_iter=5, point_painting=True)
    yaml.safe_dump(cfg, open(path, "w"))
    return path, str(root)


def seeded_models():
    import bench
    (_, lid, uni, _), _ = bench.build_models()
    return lid, uni


def loop_reference(ds, lid, uni, precision, dev):
    """a plain loop over the samples: sample() with the evaluator's zero draws and LiDAR shuffle stream, then InferModel.forward.
    -> per sample the inputs of the scoring: the data (GT BEV, actor table, ego_locs) and the model outputs (NHWC probabilities,
    packed peaks, plan), as numpy arrays."""
    from lav_b200.agent import infer_model, math_mode
    from lav_b200.datasets import TemporalBatchLoader
    im = infer_model(lid.to(dev).eval(), uni.to(dev).eval(), precision, ds.camera_x, ds.camera_z, dev)
    _, gen = TemporalBatchLoader(ds, 1, ordered=True).generators(0)
    seen = []
    det_peaks = ops.det_peaks

    def recording_peaks(*a, **k):
        seen.append(det_peaks(*a, **k))
        return seen[-1]

    out = []
    ops.det_peaks = recording_peaks
    try:
        with math_mode(precision):
            for idx in range(len(ds)):
                angle, jit = ds.no_draw()
                lidar, num, _, _, _, bev, ego_locs, cmd, nxp = ds.sample(idx, angle, jit, gen)[:9]
                _, plan, _, _, _, pred_bev, _ = im.forward(lidar[:num], nxp.float(), cmd)
                table = ds.stage_batch([ds.prepare(idx, angle, jit)], torch.Generator())
                out.append(dict(seg=pred_bev.permute(0, 2, 3, 1).float().cpu().numpy()[0], gt=bev.cpu().numpy(),
                                packed=seen[-1].cpu().numpy()[0], actors=table["actors"].numpy(), plan=plan.float().cpu().numpy(),
                                ego_locs=ego_locs.float().cpu().numpy()))
    finally:
        ops.det_peaks = det_peaks
    return out


@pytest.mark.parametrize("precision", ["fp32", "f16"])
def test_evaluate_equals_a_plain_loop(cuda, recording, precision):
    """Each batch's results equal the numpy statement on the inputs the evaluator scored, exactly; those inputs are, sample for
    sample and in index order, what a plain loop over the recording reads and what the models compute for it; the summary is the
    reduction of the batch results."""
    import lav_b200.evaluate as E
    from lav_b200.datasets import TemporalLiDARPaintedDataset
    ds = TemporalLiDARPaintedDataset(recording[0], device=cuda)
    n = len(ds)
    lid, uni = seeded_models()
    loop = loop_reference(ds, lid, uni, precision, cuda)
    divisor = next(d for d in range(min(n, 8), 0, -1) if n % d == 0)
    other = next(d for d in range(3, n) if n % d)
    for bs in sorted({divisor, other}):
        scored = []
        eval_batch = ops.eval_batch

        def recording_eval(seg, gt, packed, actors, offsets, plan, ego_locs, grid=None, **k):
            res = eval_batch(seg, gt, packed, actors, offsets, plan, ego_locs, grid, **k)
            host = lambda t: t.float().cpu().numpy() if t.dtype != torch.uint8 else t.cpu().numpy()
            scored.append((dict(seg=host(seg), gt=host(gt), packed=host(packed), actors=host(actors), offsets=np.asarray(offsets.numpy() if torch.is_tensor(offsets) else offsets),
                                plan=host(plan), ego_locs=host(ego_locs)), ops.eval_views(res.cpu(), len(seg), packed.shape[2])))
            return res

        ops.eval_batch = recording_eval
        try:
            result = E.evaluate(lid, uni, ds, batch_size=bs, precision=precision, num_workers=4)
        finally:
            ops.eval_batch = eval_batch
        assert [len(inp["seg"]) for inp, _ in scored] == [min(bs, n - k) for k in range(0, n, bs)]
        for inp, got in scored:                                             # the kernel on what the evaluator fed it
            check_equal(got, R.eval_batch_ref(inp["seg"], inp["gt"], inp["packed"], inp["actors"], inp["offsets"], inp["plan"],
                                              inp["ego_locs"]))
        i = 0
        for inp, _ in scored:                                               # ... which is the loop's samples, in index order
            for b in range(len(inp["seg"])):
                want = loop[i]
                a0, a1 = inp["offsets"][b], inp["offsets"][b + 1]
                assert np.array_equal(inp["gt"][b], want["gt"]) and np.array_equal(inp["actors"][a0:a1], want["actors"])
                assert np.array_equal(inp["ego_locs"][b], want["ego_locs"])
                # model outputs: the same network on the same input; the fp32 pillar encoder sums its centroids with float
                # atomics and the planner's reductions depend on the batch size, so these agree to fp32 rounding, not bit for bit
                assert np.abs(inp["seg"][b] - want["seg"]).max() <= 1e-4
                live = want["packed"][0] > 0.2
                assert np.array_equal(inp["packed"][b][1][live], want["packed"][1][live])
                assert np.abs(inp["packed"][b][[0, 2, 3, 4, 5]] - want["packed"][[0, 2, 3, 4, 5]]).max() <= 1e-4
                assert np.abs(inp["plan"][b] - want["plan"]).max() <= 1e-5 * (1 + np.abs(want["plan"]).max())
                i += 1
        assert i == n
        got = {k: np.concatenate([v[k].numpy() for _, v in scored]) for k in ("iou", "ngt", "flags", "score", "plan_err")}
        assert result["samples"] == n and result["bev_counts"] == got["iou"].sum(0).tolist()
        assert [result["det"][c]["n_gt"] for c in E.CLASSES] == got["ngt"].sum(0).tolist()
        for c, name in enumerate(E.CLASSES):
            f, s = got["flags"][:, c * 15:(c + 1) * 15], got["score"][:, c * 15:(c + 1) * 15]
            keep = (f & 16) != 0
            for k, t in enumerate(R.THRESHOLDS):
                ap, want_ap = result["det"][name]["ap"][f"{t:g}"], R.average_precision(s[keep], (f[keep] >> k) & 1, int(got["ngt"][:, c].sum()))
                assert (ap is None and want_ap is None) or abs(ap - want_ap) <= 1e-12
        assert abs(result["plan"]["ade"] - got["plan_err"][:, 0].mean()) <= 1e-9
        assert got["flags"].any() and got["ngt"].any()


def test_cli_writes_the_json(cuda, recording, tmp_path):
    import yaml
    from lav_b200 import evaluate as E
    lid, uni = seeded_models()
    torch.save(lid.state_dict(), tmp_path / "lidar_1.th")
    torch.save(uni.state_dict(), tmp_path / "uniplanner_1.th")
    cfg = yaml.safe_load(open(recording[0]))
    cfg["data_dir"] = "/nonexistent"                                       # --data-dir replaces it
    yaml.safe_dump(cfg, open(tmp_path / "c.yaml", "w"))
    r = E.main(["--config-path", str(tmp_path / "c.yaml"), "--data-dir", cfg_dir(recording), "--lidar-weights",
                str(tmp_path / "lidar_1.th"), "--uniplanner-weights", str(tmp_path / "uniplanner_1.th"), "--batch-size", "5",
                "--num-workers", "2", "--json", str(tmp_path / "out.json")])
    got = json.load(open(tmp_path / "out.json"))
    assert got == json.loads(json.dumps(r))
    assert got["samples"] > 0 and len(got["bev_iou"]) == 3 and set(got["det"]) == {"pedestrian", "vehicle"}
    assert set(got["det"]["vehicle"]["ap"]) == {"0.5", "1", "2", "4", "mean"} and got["plan"]["ade"] > 0


def cfg_dir(recording):
    import os
    return os.path.join(recording[1], "data")
