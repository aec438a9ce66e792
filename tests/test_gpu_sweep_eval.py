"""GPU: checkpoint sweeps of lav_b200.evaluate and lav_b200.evaluate_bev against single-checkpoint runs, evaluation across gloo
ranks against one process (exactly, with a deterministic stand-in for the models; within the models' run-to-run variation with
the real ones), and the refusal of a sweep that does not fit on the device, on the synthetic recording of test_gpu_evaluate."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from lav_b200 import ops, synth
from lav_b200.capi import LavbError
from tests.test_bev_train_cpu import _planner
from tests.test_gpu_detected_forecast import perturbed, to_dev
from tests.test_gpu_evaluate import recording, seeded_models  # noqa: F401  (recording is a fixture)
from tests.test_gpu_forecast_eval import batch_sizes

pytestmark = pytest.mark.gpu

FLAGS = dict(forecast=True, forecast_detected=True, plan_safety=True)


def seeded_pair(seed):
    """bench's LiDAR model and UniPlanner with the weights of synth seed ``seed``: distinct checkpoints of one architecture."""
    lid, uni = seeded_models()
    for m in (lid, uni):
        m.load_state_dict(synth.fill_state_dict_(m.state_dict(), seed))
    return lid, uni


class Launches:
    """the inputs of every eval_batch, forecast_eval and plan_safety launch, on the host, per checkpoint: evaluate.score_batch
    is wrapped to know which checkpoint (by the order of its InferModel in the first batch) is being scored."""

    def __init__(self):
        self.by_model, self.current = {}, self.record()

    @staticmethod
    def record():
        return dict(eval=[], views=[], forecast=[], safety=[])

    def __enter__(self):
        import lav_b200.evaluate as E
        self.E, self.sb, self.fns = E, E.score_batch, (ops.eval_batch, ops.forecast_eval, ops.plan_safety)

        def score_batch(im, *a, **k):
            self.current = self.by_model.setdefault(id(im), self.record())
            return self.sb(im, *a, **k)

        host = lambda t: (t.float() if t.is_floating_point() else t).cpu().numpy() if torch.is_tensor(t) else np.asarray(t)
        eb, fe, ps = self.fns

        def eval_batch(*a, **k):
            self.current["eval"].append([host(x) for x in a[:7]])
            res = eb(*a, **k)
            self.current["views"].append(ops.eval_views(res.cpu(), len(a[0]), a[2].shape[2]))
            return res

        def forecast_eval(cast, score, target, cmd, out=None):
            self.current["forecast"].append([host(x) for x in (cast, score, target, cmd)])
            return fe(cast, score, target, cmd, out)

        def plan_safety(*a, **k):
            res = ps(*a, **k)
            self.current["safety"].append(([host(x) for x in a[:5]], res.cpu().numpy()))
            return res
        E.score_batch, ops.eval_batch, ops.forecast_eval, ops.plan_safety = score_batch, eval_batch, forecast_eval, plan_safety
        return self

    def __exit__(self, *exc):
        self.E.score_batch = self.sb
        ops.eval_batch, ops.forecast_eval, ops.plan_safety = self.fns

    def checkpoints(self):
        return list(self.by_model.values())


def close(a, b, tol):
    return a.shape == b.shape and (a.size == 0 or float(np.abs(a - b).max()) <= tol * (1 + float(np.abs(b).max())))


def check_launches(got, want):
    """one checkpoint's launches in a sweep against those of its single run: the data bit for bit, the model outputs to the
    tolerances of test_evaluate_equals_a_plain_loop (the pillar encoder sums with float atomics)."""
    assert len(got["eval"]) == len(want["eval"]) and len(got["safety"]) == len(want["safety"])
    for g, w in zip(got["eval"], want["eval"]):
        seg, gt, packed, actors, offsets, plan, ego = range(7)
        for i in (gt, actors, offsets, ego):
            assert np.array_equal(g[i], w[i])
        assert close(g[seg], w[seg], 1e-4) and close(g[plan], w[plan], 1e-5)
        live = w[packed][:, 0] > 0.2
        assert np.array_equal(g[packed][:, 1][live], w[packed][:, 1][live])
    assert len(got["forecast"]) == len(want["forecast"])
    for g, w in zip(got["forecast"], want["forecast"]):
        assert np.array_equal(g[2], w[2], equal_nan=True) and np.array_equal(g[3], w[3])          # targets and commands
        assert close(g[0], w[0], 1e-3) and close(g[1], w[1], 1e-3)                               # casts and scores
    for (g, gres), (w, wres) in zip(got["safety"], want["safety"]):
        assert np.array_equal(g[0][:, 1], w[0][:, 1])                                             # the expert trajectories
        assert close(g[0][:, 0], w[0][:, 0], 1e-5)
        for i in (1, 2, 3, 4):
            assert np.array_equal(g[i], w[i])
        assert np.array_equal(gres[:, 1], wres[:, 1])                                             # the expert's outcomes


def check_reduction(result, launches):
    """the summary is the reduction of the checkpoint's own eval_batch results."""
    iou = np.concatenate([v["iou"].numpy() for v in launches["views"]]).sum(0)
    ngt = np.concatenate([v["ngt"].numpy() for v in launches["views"]]).sum(0)
    plan_err = np.concatenate([v["plan_err"].numpy() for v in launches["views"]])
    assert result["bev_counts"] == iou.tolist() and [result["det"][c]["n_gt"] for c in ("pedestrian", "vehicle")] == ngt.tolist()
    assert result["plan"]["ade"] == float(np.array(plan_err[:, 0].tolist()).mean())
    assert result["samples"] == sum(len(x[0]) for x in launches["eval"])


def test_sweep_equals_single_runs(cuda, recording):
    import lav_b200.evaluate as E
    from lav_b200.datasets import TemporalLiDARPaintedDataset
    ds = TemporalLiDARPaintedDataset(recording[0], device=cuda)
    n = len(ds)
    pairs = [seeded_pair(s) for s in (3, 5, 8)]
    for bs in batch_sizes(n):
        singles = []
        for lid, uni in pairs:
            with Launches() as rec:
                r = E.evaluate(lid, uni, ds, batch_size=bs, precision="fp32", num_workers=4, **FLAGS)
            singles.append((r, rec.checkpoints()[0]))
        with Launches() as rec:
            sweep = E.evaluate_checkpoints(pairs, ds, batch_size=bs, precision="fp32", num_workers=4, **FLAGS)
        assert len(sweep) == 3 and len(rec.checkpoints()) == 3
        for got, launches, (single, want) in zip(sweep, rec.checkpoints(), singles):
            check_launches(launches, want)
            check_reduction(got, launches)
            assert set(got) == set(single) and got["samples"] == single["samples"] == n
            assert abs(got["plan"]["ade"] - single["plan"]["ade"]) <= 1e-5 * (1 + abs(single["plan"]["ade"]))
            assert got["plan_safety"]["expert"] == single["plan_safety"]["expert"]
        assert sweep[0]["plan"]["ade"] != sweep[1]["plan"]["ade"]                                 # distinct checkpoints
        assert sweep[0]["plan_safety"]["expert"] == sweep[1]["plan_safety"]["expert"] == sweep[2]["plan_safety"]["expert"]


def test_a_sweep_of_one_checkpoint_twice(cuda, recording):
    import lav_b200.evaluate as E
    from lav_b200.datasets import TemporalLiDARPaintedDataset
    ds = TemporalLiDARPaintedDataset(recording[0], device=cuda)
    pair = seeded_pair(3)
    with Launches() as rec:
        a, b = E.evaluate_checkpoints([pair, pair], ds, batch_size=5, precision="fp32", num_workers=4, **FLAGS)
    check_launches(*rec.checkpoints())
    assert a["samples"] == b["samples"] and a["det"]["vehicle"]["n_gt"] == b["det"]["vehicle"]["n_gt"]
    # a pixel within the model's run-to-run variation of 0.5 may flip, so the counts agree to that, not exactly
    assert np.abs(np.array(a["bev_counts"]) - np.array(b["bev_counts"])).max() <= 1e-4 * np.array(b["bev_counts"]).max()
    assert abs(a["plan"]["ade"] - b["plan"]["ade"]) <= 1e-5 * (1 + abs(a["plan"]["ade"]))
    assert a["plan_safety"]["expert"] == b["plan_safety"]["expert"]


def test_bev_sweep_equals_single_runs(cuda, recording):
    import lav_b200.evaluate_bev as EB
    from lav_b200.datasets import TemporalBEVDataset
    ds = TemporalBEVDataset(recording[0], device=cuda)
    n = len(ds)
    planners = [_planner(s) for s in (2021, 7, 99)]
    for bs in batch_sizes(n):
        singles = []
        for p in planners:
            with Launches() as rec:
                singles.append((EB.evaluate_bev(p, ds, batch_size=bs, num_workers=4, plan_safety=True), rec.current))
        with Launches() as rec:
            sweep = EB.evaluate_bev_checkpoints(planners + [planners[0]], ds, batch_size=bs, num_workers=4, plan_safety=True)
        per = len(rec.current["forecast"]) // 4                                                   # one launch per planner per batch
        for j, (got, (single, want)) in enumerate(zip(sweep, singles + [singles[0]])):
            mine = dict(eval=[], views=[], forecast=rec.current["forecast"][j::4], safety=rec.current["safety"][j::4])
            assert len(mine["forecast"]) == per == len(want["forecast"])
            check_launches(mine, want)
            assert got["samples"] == single["samples"] == n and got["forecast"]["other"]["rows"] == single["forecast"]["other"]["rows"]
            for key in ("min_ade", "min_fde"):
                assert abs(got["forecast"]["other"][key] - single["forecast"]["other"][key]) <= 1e-4
            assert got["plan_safety"]["expert"] == single["plan_safety"]["expert"] == sweep[0]["plan_safety"]["expert"]


def test_a_sweep_that_does_not_fit_is_refused_before_the_first_batch(cuda, recording):
    import lav_b200.evaluate as E
    import lav_b200.evaluate_bev as EB
    from lav_b200.datasets import TemporalBEVDataset, TemporalLiDARPaintedDataset
    calls = []
    fns = ops.eval_batch, ops.forecast_eval
    ops.eval_batch = ops.forecast_eval = lambda *a, **k: calls.append(1)
    try:
        ds = TemporalLiDARPaintedDataset(recording[0], device=cuda)
        ds.launch_batch = lambda st: calls.append(1)
        with pytest.raises(LavbError, match="at most [0-9]+ fit"):
            E.evaluate_checkpoints([seeded_pair(3)] * 100_000, ds, batch_size=4, num_workers=2)
        bds = TemporalBEVDataset(recording[0], device=cuda)
        bds.prepare = lambda *a, **k: calls.append(1)
        with pytest.raises(LavbError, match="at most [0-9]+ fit"):
            EB.evaluate_bev_checkpoints([_planner(1)] * 1_000_000, bds, batch_size=4, num_workers=2)
    finally:
        ops.eval_batch, ops.forecast_eval = fns
    assert not calls


# ---------------------------------------------------------------------------------------------------- ranks
class StandIn:
    """InferModel.forward_batch and UniPlanner.forecast_recorded replaced by deterministic functions of the batch's own labels:
    the BEV from the recorded one, the peaks of det_heatmaps on the perturbed actor table (test_gpu_detected_forecast's
    ground-truth detector), forecasts of those detections and of the recorded rows offset from their targets, the plan from the
    expert.  The dataset's launch_batch is wrapped to see each batch."""

    def __init__(self, ds):
        self.ds, self.batch = ds, None

    def __enter__(self):
        from lav_b200.evaluate import detected_rows
        from lav_b200.model_inference import InferModel
        from lav_b200.heads import UniPlanner
        self.fb, self.fr, self.launch = InferModel.forward_batch, UniPlanner.forecast_recorded, self.ds.launch_batch
        ds, me = self.ds, self
        grid = dict(min_x=ds.min_x, max_x=ds.max_x, min_y=ds.min_y, max_y=ds.max_y, pixels_per_meter=ds.pixels_per_meter)

        def launch_batch(st):
            me.batch = (me.launch(st), st["actors"].numpy().copy(), st["offsets"].numpy().copy())
            return me.batch[0]

        def forward_batch(im, lidars, num_points, nxps, cmds):
            batch, actors, offsets = me.batch
            bev, ego = batch[5], batch[6]
            dev = bev.device
            seg = (bev[:, :3].permute(0, 2, 3, 1).float() * 0.5 + 0.25 + 0.01 * bev[:, 3:6].permute(0, 2, 3, 1).float()).contiguous()
            heat, size, orim = ops.det_heatmaps(*to_dev(dev, *perturbed(actors, offsets)), grid)
            nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous()
            packed = ops.det_peaks(nhwc(torch.logit(heat.clamp(1e-6, 1 - 1e-6))), nhwc(size), nhwc(orim))
            feats = torch.nn.functional.avg_pool2d(bev[:, :4].float(), 2).permute(0, 2, 3, 1).repeat(1, 1, 1, 96).contiguous()
            h, w = feats.shape[1:3]
            rows = detected_rows(packed.cpu().numpy(), im.pixels_per_meter, im.uniplanner.crop_centre(2 * h, 2 * w))
            T, C = ego.shape[1] - 1, 6
            steps = torch.arange(1, T + 1, device=dev, dtype=torch.float32)[None, None, :, None]
            branch = torch.arange(C, device=dev, dtype=torch.float32)[None, :, None, None]
            locs = torch.from_numpy(rows["locs"]).to(dev)[:, None, None] + steps * torch.tensor([0.1, -0.7], device=dev) * (1 + 0.1 * branch)
            score = torch.from_numpy(rows["score"]).to(dev)[:, None] - 0.05 * branch[:, :, 0, 0]
            counts = rows["counts"].tolist()
            plan = ego[:, 1:] * 0.9 + cmds.to(dev).float()[:, None, None] * 0.3
            return dict(pred_bev=seg.permute(0, 3, 1, 2), packed=packed, ego_plan_locs=plan, features=feats,
                        other_cast_locs=torch.split(locs, counts), other_cast_cmds=torch.split(score, counts))

        def forecast_recorded(up, *a, **k):
            fc = dict(me.fr(up, *a, **k))
            for rows, tgt in (("cast", "target"), ("ego_cast", "ego_target")):
                t = fc[tgt].float()
                C = fc[rows].shape[1]
                fc[rows] = t[:, None] * (1 + 0.05 * torch.arange(C, device=t.device, dtype=torch.float32)[None, :, None, None])
                fc["score" if rows == "cast" else "ego_score"] = -t[:, -1:, 0].repeat(1, C) + torch.arange(C, device=t.device) * 0.01
            return fc
        InferModel.forward_batch, UniPlanner.forecast_recorded, ds.launch_batch = forward_batch, forecast_recorded, launch_batch
        return self

    def __exit__(self, *exc):
        from lav_b200.heads import UniPlanner
        from lav_b200.model_inference import InferModel
        InferModel.forward_batch, UniPlanner.forecast_recorded = self.fb, self.fr
        del self.ds.launch_batch


def odd_dataset(path, dev):
    """the recording, cut to a sample count divisible by neither 2 nor 3."""
    from lav_b200.datasets import TemporalLiDARPaintedDataset
    ds = TemporalLiDARPaintedDataset(path, device=dev)
    m = max(k for k in range(1, len(ds) + 1) if k % 6 in (1, 5))
    ds.index = ds.index[:m]
    return ds


def run(path, stand_in, pairs_seeds, bs):
    import lav_b200.evaluate as E
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", 0)) % torch.cuda.device_count())
    torch.cuda.set_device(dev)
    ds = odd_dataset(path, dev)
    pairs = [seeded_pair(s) for s in pairs_seeds]
    shards = []
    prepare = ds.prepare
    ds.prepare = lambda idx, *a, **k: shards.append(idx) or prepare(idx, *a, **k)
    if stand_in:
        with StandIn(ds):
            out = E.evaluate_checkpoints(pairs, ds, batch_size=bs, precision="fp32", num_workers=2, **FLAGS)
    else:
        out = E.evaluate_checkpoints(pairs, ds, batch_size=bs, precision="fp32", num_workers=2, **FLAGS)
    return out, sorted(shards), len(ds)


def _worker(rank, world, port, path, stand_in, seeds, bs, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), LOCAL_RANK=str(rank))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        res, shard, n = run(path, stand_in, seeds, bs)
        lo, hi = rank * n // world, (rank + 1) * n // world
        assert shard == list(range(lo, hi)), (rank, shard)
        assert (res is None) == (rank != 0)
        if rank == 0:
            torch.save(res, out)
    finally:
        dist.destroy_process_group()


def spawn(world, path, stand_in, seeds, bs, tmp_path):
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    out = str(tmp_path / f"rank0_{world}_{stand_in}.pt")
    mp.spawn(_worker, args=(world, port, path, stand_in, seeds, bs, out), nprocs=world, join=True)
    return torch.load(out, weights_only=False)


def test_ranks_equal_one_process_exactly(cuda, recording, tmp_path):
    one, shard, n = run(recording[0], True, (3, 5), 3)
    assert shard == list(range(n)) and n % 2 and n % 3
    assert one[0]["forecast_detected"]["matched"] > 0 and one[0]["det"]["vehicle"]["n_det"] > 0
    assert one[0]["forecast"]["other"]["rows"] > 0
    for world in (2, 3):
        got = spawn(world, recording[0], True, (3, 5), 3, tmp_path)
        assert got == one, world


def test_ranks_with_the_real_models(cuda, recording, tmp_path):
    one, _, n = run(recording[0], False, (3,), 4)
    got = spawn(2, recording[0], False, (3,), 4, tmp_path)
    a, b = got[0], one[0]
    assert a["samples"] == b["samples"] == n
    assert a["forecast"]["ego_cast"]["samples"] == b["forecast"]["ego_cast"]["samples"] == n
    assert a["plan_safety"]["expert"] == b["plan_safety"]["expert"]
    assert a["det"]["vehicle"]["n_gt"] == b["det"]["vehicle"]["n_gt"] and a["forecast"]["other"]["rows"] == b["forecast"]["other"]["rows"]
    assert abs(a["plan"]["ade"] - b["plan"]["ade"]) <= 1e-4 * (1 + abs(b["plan"]["ade"]))
    for x, y in zip(a["bev_iou"], b["bev_iou"]):
        assert (x is None and y is None) or abs(x - y) <= 1e-3
    assert abs(a["forecast"]["other"]["min_ade"] - b["forecast"]["other"]["min_ade"]) <= 1e-3
