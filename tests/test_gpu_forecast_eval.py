"""GPU: ops.forecast_eval against the numpy statement of tests/test_forecast_eval_cpu.py, its argument checks and known answers;
lav_b200.evaluate --forecast and lav_b200.evaluate_bev against a plain per-sample loop on a synthetic recording; the ordered BEV
loader; both CLIs."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from lav_b200 import ops
from lav_b200.capi import LavbError, lib
from tests import test_forecast_eval_cpu as R
from tests.test_bev_train_cpu import _planner
from tests.test_gpu_evaluate import cfg_dir, recording, seeded_models  # noqa: F401  (recording is a fixture)

pytestmark = pytest.mark.gpu


def to_dev(dev, *arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in arrays]


def check_equal(got, want):
    """every error and branch identical, NaN where the statement has NaN."""
    assert np.array_equal(got["err"].numpy(), want["err"], equal_nan=True), np.argwhere(~((got["err"].numpy() == want["err"]) |
                                                                                          np.isnan(want["err"])))[:5]
    assert np.array_equal(got["branch"].numpy(), want["branch"])


@pytest.mark.parametrize("k", [0, 1, 33, 5000])
@pytest.mark.parametrize("t", [10, 20])
def test_forecast_eval_equals_the_numpy_statement(cuda, k, t):
    cast, score, target, cmd = R.random_rows(k, 6, t, 10 * k + t)
    got = ops.forecast_views(ops.forecast_eval(*to_dev(cuda, cast, score, target, cmd)).cpu(), k)
    want = R.forecast_eval_ref(cast, score, target, cmd)
    check_equal(got, want)
    if k >= 33:
        b = want["branch"]
        assert np.isnan(want["err"][:, 4]).any() and not np.isnan(want["err"][:, 4]).all()
        assert (b[:, 0] != b[:, 1]).any() and (b[:, 1] == 0).any()


def test_known_answers(cuda):
    target = np.zeros((4, 10, 2), np.float32)
    cast = np.repeat(target[:, None], 6, 1)
    cast[1:, :, :, 0] += 1.0                                                # rows 1..3: every branch 1 m off
    cast[2, 3] = 0.0                                                        # row 2: branch 3 exact
    score = np.zeros((4, 6), np.float32)
    score[1] = np.nan                                                       # every score NaN: branch 0 is the top
    score[2, 5] = 0.9
    score[3, [1, 4]] = 0.8                                                  # tie: the lower branch
    cmd = np.array([2, -1, 3, 4], np.int32)
    v = ops.forecast_views(ops.forecast_eval(*to_dev(cuda, cast, score, target, cmd)).cpu(), 4)
    err, branch = v["err"].numpy(), v["branch"].numpy()
    assert err[0].tolist() == [0.0] * 6 and branch[0].tolist() == [0, 0]
    assert err[1, :4].tolist() == [1.0] * 4 and np.isnan(err[1, 4:]).all() and branch[1].tolist() == [0, 0]
    assert err[2].tolist() == [0.0, 0.0, 1.0, 1.0, 0.0, 0.0] and branch[2].tolist() == [3, 5]
    assert err[3].tolist() == [1.0] * 6 and branch[3].tolist() == [0, 1]


def test_forecast_eval_rejects_malformed_arguments_and_writes_nothing(cuda):
    cast, score, target, cmd = to_dev(cuda, *R.random_rows(8, 6, 10, 3))
    out = torch.full((8 * 56,), 0xAB, dtype=torch.uint8, device=cuda)
    bad = [dict(cast=cast.double()), dict(cast=cast.transpose(1, 2).contiguous().transpose(1, 2)), dict(cast=cast[..., :1].contiguous()),
           dict(score=score[:, :5].contiguous()), dict(score=score.double()), dict(target=target[:, :9].contiguous()),
           dict(target=target[:7].contiguous()), dict(cmd=cmd.long()), dict(cmd=cmd[:7].contiguous()), dict(cmd=cmd.cpu()),
           dict(cast=torch.zeros((8, 33, 10, 2), device=cuda), score=torch.zeros((8, 33), device=cuda)),          # over 32 branches
           dict(cast=torch.zeros((8, 6, 33, 2), device=cuda), target=torch.zeros((8, 33, 2), device=cuda))]       # over 32 steps
    for kw in bad:
        args = dict(cast=cast, score=score, target=target, cmd=cmd)
        args.update(kw)
        with pytest.raises(LavbError):
            ops.forecast_eval(args["cast"], args["score"], args["target"], args["cmd"], out=out)
    with pytest.raises(LavbError):
        ops.forecast_eval(cast, score, target, cmd, out=out[:-8])
    v = ops.forecast_views(out, 8)
    p = lambda t: C.c_void_p(t.data_ptr())
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    null = C.c_void_p(0)
    fn = lib().lavb_forecast_eval
    assert fn(p(cast), p(score), p(target), p(cmd), -1, 6, 10, p(v["err"]), p(v["branch"]), st) != 0         # negative k
    assert fn(p(cast), p(score), p(target), p(cmd), 8, 0, 10, p(v["err"]), p(v["branch"]), st) != 0          # no branch
    assert fn(p(cast), p(score), p(target), p(cmd), 8, 6, 0, p(v["err"]), p(v["branch"]), st) != 0           # no step
    for i in range(6):                                                      # each pointer null in turn, k > 0
        ptrs = [p(cast), p(score), p(target), p(cmd), p(v["err"]), p(v["branch"])]
        ptrs[i] = null
        assert fn(*ptrs[:4], 8, 6, 10, *ptrs[4:], st) != 0
    assert fn(null, null, null, null, 0, 6, 10, null, null, st) == 0        # k = 0: nothing to do, nothing read
    torch.cuda.synchronize()
    assert bool((out == 0xAB).all())


# ---------------------------------------------------------------------------------------------------- the evaluators
class Recorder:
    """wraps score_forecasts (in ``module``) and ops.forecast_eval: per batch the forecast_recorded dict and the recorded commands,
    the kernel's inputs and its results, on the host."""

    def __init__(self, module):
        self.module, self.fcs, self.scored = module, [], []

    def __enter__(self):
        self.sf, self.fe = self.module.score_forecasts, ops.forecast_eval

        def score_forecasts(fc, cmds, plan=False):
            self.fcs.append(({k: v.float().cpu().numpy() if v.is_floating_point() else v.cpu().numpy() for k, v in fc.items()},
                             cmds.cpu().numpy()))
            return self.sf(fc, cmds, plan)

        def forecast_eval(cast, score, target, cmd, out=None):
            res = self.fe(cast, score, target, cmd, out)
            inputs = [t.cpu().numpy() for t in (cast, score, target, cmd)]
            self.scored.append((inputs, ops.forecast_views(res.cpu(), len(cast))))
            return res
        self.module.score_forecasts, ops.forecast_eval = score_forecasts, forecast_eval
        return self

    def __exit__(self, *exc):
        self.module.score_forecasts, ops.forecast_eval = self.sf, self.fe


def check_against_loop(rec, loop, result, sizes, plan, cast_tol):
    """each batch's results equal the statement on its inputs; those inputs are the batch's forecast_recorded rows and commands;
    rows, slots and targets equal the per-sample loop bit for bit, casts and scores to ``cast_tol`` (relative to the largest);
    the summary is the reduction of the batch results.  -> the largest cast / score / plan differences seen."""
    assert [len(c) for _, c in rec.fcs] == sizes and len(rec.scored) == len(sizes)
    batches, s0, worst = [], 0, dict(cast=0.0, score=0.0, plan=0.0)
    for (fc, cmds), (inputs, got) in zip(rec.fcs, rec.scored):
        check_equal(got, R.forecast_eval_ref(*inputs))
        k, b = len(fc["frame"]), len(cmds)
        parts = [("cast", "score", "target"), ("ego_cast", "ego_score", "ego_target")] + ([("ego_plan", "ego_score", "ego_target")] if plan else [])
        for i in range(3):
            assert np.array_equal(inputs[i], np.concatenate([fc[p[i]] for p in parts]))
        assert inputs[3].tolist() == [-1] * k + cmds.tolist() * (len(parts) - 1)
        batches.append((got["err"].numpy(), got["branch"].numpy(), k, cmds))
        want = [loop[i] for i in range(s0, s0 + b)]
        frames = np.concatenate([np.full(len(w["frame"]), i) for i, w in enumerate(want)]) if want else np.zeros(0)
        assert np.array_equal(fc["frame"], frames) and np.array_equal(fc["slot"], np.concatenate([w["slot"] for w in want]))
        for key in ("target", "ego_target"):
            assert np.array_equal(fc[key], np.concatenate([w[key] for w in want])), key
        for key, kind in (("cast", "cast"), ("ego_cast", "cast"), ("score", "score"), ("ego_score", "score")) + ((("ego_plan", "plan"),) if plan else ()):
            w = np.concatenate([x[key] for x in want])
            d = float(np.abs(fc[key] - w).max()) if w.size else 0.0
            worst[kind] = max(worst[kind], d / (1 + float(np.abs(w).max())) if w.size else 0.0)
        s0 += b
    assert worst["cast"] <= cast_tol and worst["score"] <= cast_tol and worst["plan"] <= cast_tol, worst
    assert result == R.reduce_ref(batches, plan)
    assert result["other"]["rows"] == sum(len(w["frame"]) for w in loop) > 0
    return worst


def batch_sizes(n):
    divisor = next(d for d in range(min(n, 8), 0, -1) if n % d == 0)
    other = next(d for d in range(3, n) if n % d)
    return sorted({divisor, other})


def test_evaluate_forecast_equals_a_plain_loop(cuda, recording):
    """evaluate(forecast=True) at fp32 against sample() + forward_batch + forecast_recorded one sample at a time."""
    import lav_b200.evaluate as E
    from lav_b200.agent import infer_model, math_mode
    from lav_b200.datasets import TemporalBatchLoader, TemporalLiDARPaintedDataset
    ds = TemporalLiDARPaintedDataset(recording[0], device=cuda)
    n = len(ds)
    lid, uni = seeded_models()
    im = infer_model(lid.to(cuda).eval(), uni.to(cuda).eval(), "fp32", ds.camera_x, ds.camera_z, cuda)
    _, gen = TemporalBatchLoader(ds, 1, ordered=True).generators(0)
    loop = []
    with math_mode("fp32"), torch.no_grad():
        for idx in range(n):
            angle, jit = ds.no_draw()
            lidar, num, _, _, _, _, ego, cmd, nxp, _, locs, oris, typs = ds.sample(idx, angle, jit, gen)[:13]
            o = im.forward_batch([lidar[:num]], [int(num)], nxp.float()[None], [cmd])
            fc = im.uniplanner.forecast_recorded(o["features"].permute(0, 3, 1, 2), ego.float()[None], locs[None], oris[None], typs[None])
            loop.append({k: v.cpu().numpy() for k, v in fc.items()})
    for bs in batch_sizes(n):
        with Recorder(E) as rec:
            result = E.evaluate(lid, uni, ds, batch_size=bs, precision="fp32", num_workers=4, forecast=True)
        sizes = [min(bs, n - k) for k in range(0, n, bs)]
        # the LiDAR features differ from run to run (the pillar encoder sums centroids with float atomics) and the embedder's
        # reductions depend on the batch size, so the casts agree to that variation, not bit for bit
        worst = check_against_loop(rec, loop, result["forecast"], sizes, plan=False, cast_tol=1e-3)
        print(f"evaluate --forecast fp32, batch {bs}: largest relative difference to the loop {worst}")
        assert result["samples"] == n and "plan" in result
    assert "forecast" not in E.evaluate(lid, uni, ds, batch_size=batch_sizes(n)[0], precision="fp32", num_workers=4)


def test_evaluate_bev_equals_a_plain_loop(cuda, recording):
    """evaluate_bev against sample(idx, 0, 0.0) + forecast_recorded one sample at a time."""
    import lav_b200.evaluate_bev as EB
    from lav_b200.agent import math_mode
    from lav_b200.datasets import TemporalBEVDataset
    ds = TemporalBEVDataset(recording[0], device=cuda)
    n = len(ds)
    planner = _planner(2021).to(cuda).eval()
    loop = []
    with math_mode("fp32"):
        for idx in range(n):
            bev, ego, _, nxp, _, locs, oris, typs, _ = ds.sample(idx, 0, 0.0)
            fc = planner.forecast_recorded(bev[None], ego.float()[None], locs[None], oris[None], typs[None], nxp.float()[None])
            loop.append({k: v.cpu().numpy() for k, v in fc.items()})
    for bs in batch_sizes(n):
        with Recorder(EB) as rec:
            result = EB.evaluate_bev(planner, ds, batch_size=bs, num_workers=4)
        sizes = [min(bs, n - k) for k in range(0, n, bs)]
        worst = check_against_loop(rec, loop, result["forecast"], sizes, plan=True, cast_tol=1e-4)
        print(f"evaluate_bev, batch {bs}: largest relative difference to the loop {worst}")
        assert result["samples"] == n and set(result["forecast"]) == {"other", "ego_cast", "ego_plan"}


def test_ordered_bev_loader_equals_unaugmented_samples(cuda, recording):
    from lav_b200.datasets import TemporalBEVBatchLoader, TemporalBEVDataset
    ds = TemporalBEVDataset(recording[0], device=cuda)
    n = len(ds)

    def no_random_draw(gen):
        raise AssertionError("an ordered loader draws no augmentation")
    ds.draw = no_random_draw
    loader = TemporalBEVBatchLoader(ds, 3, drop_last=False, num_workers=2, ordered=True)
    got = list(loader.staged_batches())
    assert len(got) == len(loader) == -(-n // 3)
    i = 0
    for batch, hs in got:
        for b in range(len(hs)):
            want = ds.sample(i, 0, 0.0)
            assert torch.equal(batch[0][b], want[0])
            assert torch.equal(batch[1][b], want[1].float()) and torch.equal(batch[3][b], want[3].float())
            assert int(batch[2][b]) == want[2] == hs[b]["cmd"] and int(batch[4][b]) == want[4]
            for j in (5, 6, 7):
                assert torch.equal(batch[j][b], want[j])
            assert int(batch[8][b]) == want[8]
            i += 1
    assert i == n
    assert [len(b[0]) for b in TemporalBEVBatchLoader(ds, 4, drop_last=False, num_workers=2, ordered=True)] == \
        [min(4, n - k) for k in range(0, n, 4)]


def test_clis_write_the_json(cuda, recording, tmp_path):
    import yaml
    from lav_b200 import evaluate as E
    from lav_b200 import evaluate_bev as EB
    lid, uni = seeded_models()
    torch.save(lid.state_dict(), tmp_path / "lidar_1.th")
    torch.save(uni.state_dict(), tmp_path / "uniplanner_1.th")
    torch.save(_planner(2021).state_dict(), tmp_path / "bev_1.th")
    cfg = yaml.safe_load(open(recording[0]))
    cfg["data_dir"] = "/nonexistent"                                       # --data-dir replaces it
    yaml.safe_dump(cfg, open(tmp_path / "c.yaml", "w"))
    common = ["--config-path", str(tmp_path / "c.yaml"), "--data-dir", cfg_dir(recording), "--batch-size", "4", "--num-workers", "2"]
    r = E.main(common + ["--lidar-weights", str(tmp_path / "lidar_1.th"), "--uniplanner-weights", str(tmp_path / "uniplanner_1.th"),
                         "--forecast", "--json", str(tmp_path / "out.json")])
    got = json.load(open(tmp_path / "out.json"))
    assert got == json.loads(json.dumps(r)) and got["precision"] == "f16"
    assert got["forecast"]["other"]["rows"] > 0 and got["forecast"]["ego_cast"]["samples"] == got["samples"]
    assert "ego_plan" not in got["forecast"]
    r = EB.main(common + ["--bev-weights", str(tmp_path / "bev_1.th"), "--json", str(tmp_path / "bev.json")])
    got = json.load(open(tmp_path / "bev.json"))
    assert got == json.loads(json.dumps(r)) and got["samples"] > 0
    f = got["forecast"]
    assert f["other"]["rows"] > 0 and f["ego_cast"]["samples"] == f["ego_plan"]["samples"] == got["samples"]
    assert os.path.getsize(tmp_path / "bev.json") > 0
