"""GPU: evaluate --brake.  score_brake's two ops.agent_control launches against oracle/control_ref.ControlTail (fresh, speed 0) on
hand-made batches with NaN plans and commands 4 and 5; evaluate(brake=True) against that statement on the inputs each batch
scored, with the real seeded models on a synthetic 5-camera recording; a sweep against its single runs, one brake-model call per
batch, the ranks against one process and the unchanged result without --brake under the deterministic stand-in of
test_gpu_sweep_eval; the CLI."""
import json
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from lav_b200 import ops, synth
from oracle.control_ref import ControlTail
from tests.test_brake_eval_cpu import rows_loop

pytestmark = pytest.mark.gpu

CFG = json.loads(str(np.load(os.path.join(os.path.dirname(__file__), "golden", "agent_control.npz"))["config"]))


def statement(plan, cast, rows, scores, offsets, pred_bra, cmds):
    """ControlTail's flags and brake for one fresh tick at speed 0 on host copies of an agent_control launch's inputs."""
    B = len(plan)
    tail = ControlTail(B, CFG)
    per = lambda a: [a[offsets[b]:offsets[b + 1]] for b in range(B)]
    r = tail.step(plan, cast, per(rows), per(scores), pred_bra, np.zeros(B, np.float32), cmds)
    return r["flags"], r["control"][:, 2]


def synthetic_batch(B, seed, dev, M=8, T=20, C=6):
    """forward_batch-like outputs, brake probabilities and labels: plans stepping 0..1.1 m (some below the PID brake speed),
    NaN plans and casts, 0..6 detected rows per sample placed around the plan, label tracks some of which cross the plan."""
    rs = np.random.RandomState(seed)
    step = rs.uniform(0.0, 1.1, (B, 1, 1)) * rs.uniform(0.6, 1.0, (B, T, 1))
    plan = np.cumsum(np.concatenate([np.zeros((B, T, 1)) + 0.05 * rs.randn(B, T, 1), -np.ones((B, T, 1))], -1) * step, 1)
    plan = plan.astype(np.float32)
    cast = (plan * rs.uniform(0.5, 1.5, (B, 1, 1))).astype(np.float32)
    plan[rs.rand(B) < 0.15, rs.randint(0, T)] = np.nan
    cast[rs.rand(B) < 0.15, rs.randint(0, T), 1] = np.nan
    counts = rs.randint(0, 7, B)
    counts[0] = 0
    K = int(counts.sum())
    start = plan[np.repeat(np.arange(B), counts), rs.randint(0, T, K)] + rs.normal(0, 3, (K, 2))
    start = np.nan_to_num(start)
    v = rs.uniform(0, 0.5, (K, C, 1, 1))
    other = (start[:, None, None] + np.arange(T)[None, None, :, None] * v * rs.normal(0, 1, (K, C, 1, 2))).astype(np.float32)
    other_s = rs.uniform(0, 0.5, (K, C)).astype(np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    out = dict(ego_plan_locs=t(plan), ego_cast_locs=t(cast), other_cast_locs=torch.split(t(other), counts.tolist()),
               other_cast_cmds=torch.split(t(other_s), counts.tolist()))
    pred = rs.uniform(0, 0.15, B).astype(np.float32)
    pred[::9] = np.float32(0.1)
    cmds = rs.randint(0, C, B).astype(np.int32)
    cmds[:2] = (4, 5)[:B]
    ego = np.zeros((B, T + 1, 2), np.float32)
    ego[:, 1:] = np.nan_to_num(plan)
    locs = np.nan_to_num(plan)[:, None].repeat(M, 1) + rs.normal(0, 2.5, (B, M, 1, 2))
    locs = np.concatenate([locs[:, :, :1], locs], 2).astype(np.float32)                       # (B, M, T + 1, 2)
    typs = rs.choice([0, 1, 1], (B, M)).astype(np.int32)
    num_objs = rs.randint(0, M + 1, B)
    return out, t(pred), cmds, t(locs), t(ego), t(typs), torch.from_numpy(num_objs)


@pytest.mark.parametrize("B", [1, 7, 64])
def test_score_brake_equals_the_statement(cuda, B):
    import lav_b200.evaluate as E
    from lav_b200.control import FLAG_BRAKE_MODEL, FLAG_COLLIDE, FLAG_PID_BRAKE, FLAG_PLAN_INVALID, control_config
    out, pred, cmds, locs, ego, typs, num_objs = synthetic_batch(B, B + 11, cuda)
    expert = E.expert_track_rows(locs, ego, typs, num_objs, 6)
    res = E.score_brake(out, pred, expert, cmds, control_config(CFG)).cpu().numpy()
    host = lambda x: x.float().cpu().numpy()
    plan, cast, p = host(out["ego_plan_locs"]), host(out["ego_cast_locs"]), host(pred)
    counts = [len(o) for o in out["other_cast_locs"]]
    offs = np.concatenate([[0], np.cumsum(counts)])
    det = (host(torch.cat(out["other_cast_locs"])), host(torch.cat(out["other_cast_cmds"])), offs)
    want_rows, want_scores = rows_loop(locs.cpu().numpy(), ego.cpu().numpy(), typs.cpu().numpy(), num_objs.numpy(), 6)
    assert np.array_equal(host(expert[0]), want_rows, equal_nan=True)
    for j, (rows, scores, o) in enumerate((det, (want_rows, want_scores, expert[2]))):
        flags, brake = statement(plan, cast, rows, scores, o, p, cmds)
        assert np.array_equal(res[:, j], flags), (j, np.nonzero(res[:, j] != flags))
        if j == 0:
            assert np.array_equal(res[:, 2], (brake == 1).astype(np.int32))
    reasons = (res[:, 0] & (FLAG_BRAKE_MODEL | FLAG_PID_BRAKE | FLAG_COLLIDE)) != 0
    assert np.array_equal(res[:, 2] != 0, reasons)                              # speed 0, fresh state: the three rules only
    if B == 64:
        for bit in (FLAG_PLAN_INVALID, FLAG_PID_BRAKE, FLAG_BRAKE_MODEL, FLAG_COLLIDE):
            assert (res[:, 0] & bit).any() and not (res[:, 0] & bit).all(), bit
        assert (res[:, 1] & FLAG_COLLIDE).any()


# ---------------------------------------------------------------------------------------------------- evaluate
@pytest.fixture(scope="module")
def recording(tmp_path_factory, golden_dir):
    import yaml
    from tests.test_temporal_dataset_cpu import write_config
    gold = np.load(os.path.join(golden_dir, "temporal_dataset.npz"))
    root = tmp_path_factory.mktemp("brake_rec")
    synth.record_trajectories(str(root / "data"), int(gold["n_traj"]), int(gold["n_frames"]), int(gold["seed"]), images=True,
                              n_cameras=5)
    path = write_config(gold, str(root / "data"), root / "config.yaml")
    cfg = yaml.safe_load(open(path))
    cfg.update(num_features=[64, 64], backbone="cnn", crop_size=96, feature_x_jitter=1.5, feature_angle_jitter=20, num_cmds=6,
               num_plan_iter=5, point_painting=True, crop_tel_bottom=96, **CFG)
    yaml.safe_dump(cfg, open(path, "w"))
    return path, str(root)


def seeded_models(seed=None):
    import bench
    (_, lid, uni, bra), _ = bench.build_models()
    if seed is not None:
        for m in (lid, uni):
            m.load_state_dict(synth.fill_state_dict_(m.state_dict(), seed))
    return lid, uni, bra


class Recorder:
    """the inputs and outputs of every agent_control launch and every brake_probs call of the evaluator, on the host."""

    def __enter__(self):
        import lav_b200.evaluate as E
        self.E, self.fns = E, (ops.agent_control, E.brake_probs)
        self.control, self.brake = [], []
        ac, bp = self.fns
        host = lambda t: (t.float() if t.is_floating_point() else t).cpu().numpy() if torch.is_tensor(t) else np.asarray(t).copy()

        def agent_control(*a, **k):
            control, flags = ac(*a, **k)
            self.control.append(([host(x) for x in a[:8]], host(control), host(flags)))
            return control, flags

        def brake_probs(bra, rgbs, tel, *a, **k):
            p = bp(bra, rgbs, tel, *a, **k)
            self.brake.append((host(rgbs), host(tel), host(p)))
            return p
        ops.agent_control, E.brake_probs = agent_control, brake_probs
        return self

    def __exit__(self, *exc):
        ops.agent_control, self.E.brake_probs = self.fns


def test_evaluate_brake_equals_the_statement(cuda, recording, tmp_path):
    import lav_b200.evaluate as E
    from lav_b200.datasets import CameraDataset, TemporalLiDARPaintedDataset
    ds = TemporalLiDARPaintedDataset(recording[0], device=cuda)
    n = len(ds)
    lid, uni, bra = seeded_models()
    with Recorder() as rec:
        result = E.evaluate(lid, uni, ds, batch_size=8, precision="f16", num_workers=4, brake=True, bra_model=bra)
    nb = -(-n // 8)
    assert len(rec.brake) == nb and len(rec.control) == 2 * nb
    acc = E.BrakeScores(6)
    cams = CameraDataset(recording[0], seg=False, brake=True, device="cpu")
    assert cams.index == ds.index
    seen_cmds = set()
    for k in range(nb):
        idx = range(8 * k, min(8 * k + 8, n))
        want_cams = cams.stage_batch([cams.prepare(i) for i in idx])
        rgbs, tel, p = rec.brake[k]
        assert np.array_equal(rgbs, want_cams["rgbs"].numpy()) and np.array_equal(tel, want_cams["tel"].numpy())
        res = []
        for j in (0, 1):
            (plan, cast, rows, scores, offsets, pred, speed, cmds), control, flags = rec.control[2 * k + j]
            assert np.array_equal(pred, p.astype(np.float32)) and not speed.any()
            assert np.array_equal(cmds, [ds.prepare(i, *ds.no_draw())["cmd"] for i in idx])
            want_flags, want_brake = statement(plan, cast, rows, scores, offsets, pred, cmds)
            assert np.array_equal(flags, want_flags) and np.array_equal(control[:, 2], want_brake.astype(np.float32))
            res.append(flags)
            seen_cmds |= set(cmds.tolist())
        acc.add(np.stack([res[0], res[1], (rec.control[2 * k][1][:, 2] == 1).astype(np.int32)], 1), cmds,
                [ds.prepare(i, *ds.no_draw())["bra"] for i in idx])
    assert {4, 5} <= seen_cmds
    assert result["brake"] == acc.summary()
    b = result["brake"]
    assert b["samples"] == n and 0 < b["positives"] < n
    assert "brake" in E.format_result(result)


# ---------------------------------------------------------------------------------------------------- deterministic stand-in
class BrakeStandIn:
    """test_gpu_sweep_eval.StandIn with an ego cast (the plan bent by the command) and a brake model replaced by an exact
    function of the camera bytes (their integer sum, scaled so that the probabilities straddle 0.1)."""

    def __init__(self, ds):
        from tests.test_gpu_sweep_eval import StandIn
        self.inner = StandIn(ds)

    def __enter__(self):
        import lav_b200.evaluate as E
        from lav_b200.model_inference import InferModel
        self.inner.__enter__()
        self.E, self.fb, self.bp = E, InferModel.forward_batch, E.brake_probs
        fb = self.fb

        def forward_batch(im, lidars, num_points, nxps, cmds):
            out = fb(im, lidars, num_points, nxps, cmds)
            plan = out["ego_plan_locs"].float()
            return dict(out, ego_plan_locs=plan, ego_cast_locs=plan * 1.2 + 0.1)

        def brake_probs(bra, rgbs, tel, *a, **k):
            s = rgbs.to(torch.int64).sum((1, 2, 3, 4)) + tel.to(torch.int64).sum((1, 2, 3))
            n = rgbs[0].numel() + tel[0].numel()
            return (s.double() / (n * 255.0) * 0.2).float()
        InferModel.forward_batch, E.brake_probs = forward_batch, brake_probs
        return self

    def __exit__(self, *exc):
        from lav_b200.model_inference import InferModel
        InferModel.forward_batch, self.E.brake_probs = self.fb, self.bp
        self.inner.__exit__(*exc)


def run(path, seeds, bs, brake=True):
    import lav_b200.evaluate as E
    from lav_b200.datasets import TemporalLiDARPaintedDataset
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", 0)) % torch.cuda.device_count())
    torch.cuda.set_device(dev)
    ds = TemporalLiDARPaintedDataset(path, device=dev)
    models = [seeded_models(s) for s in seeds]
    log, calls = [], []
    env = ds.env
    ds.env = lambda traj: _KeyLog(env(traj), log)
    with BrakeStandIn(ds):
        bp = E.brake_probs
        E.brake_probs = lambda *a, **k: calls.append(1) or bp(*a, **k)
        try:
            out = E.evaluate_checkpoints([m[:2] for m in models], ds, batch_size=bs, precision="fp32", num_workers=2,
                                         plan_safety=True, brake=brake, bra_model=models[0][2] if brake else None)
        finally:
            E.brake_probs = bp
    return out, len(calls), {k.rsplit("_", 1)[0] for k in log}, len(ds)


class _KeyLog:
    def __init__(self, env, log):
        self.env, self.log = env, log

    def get(self, key):
        self.log.append(key)
        return self.env.get(key)


def test_sweep_equals_single_runs_with_one_brake_call_per_batch(cuda, recording):
    n = None
    singles = []
    for s in (3, 5):
        r, calls, _, n = run(recording[0], (s,), 5)
        assert calls == -(-n // 5)
        singles.append(r[0])
    sweep, calls, _, _ = run(recording[0], (3, 5), 5)
    assert calls == -(-n // 5)
    assert sweep == singles
    v = sweep[0]["brake"]["verdicts"]
    assert v["brake_model"]["tp"] + v["brake_model"]["fp"] > 0 and v["brake_model"]["fn"] + v["brake_model"]["tn"] > 0


def test_without_brake_the_result_and_the_reads_are_unchanged(cuda, recording):
    with_brake, _, read_b, _ = run(recording[0], (3,), 4, brake=True)
    plain, calls, read, _ = run(recording[0], (3,), 4, brake=False)
    assert calls == 0 and "brake" not in plain[0]
    assert {k: v for k, v in with_brake[0].items() if k != "brake"} == plain[0]
    assert not any(k.startswith(("rgb_", "tel_rgb")) for k in read)
    assert read_b - read == {"rgb_1", "rgb_2", "rgb_3", "tel_rgb"}


def _worker(rank, world, port, path, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), LOCAL_RANK=str(rank))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        res = run(path, (3,), 3)[0]
        if rank == 0:
            torch.save(res, out)
    finally:
        dist.destroy_process_group()


def test_two_ranks_equal_one_process(cuda, recording, tmp_path):
    one = run(recording[0], (3,), 3)[0]
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    out = str(tmp_path / "rank0.pt")
    mp.spawn(_worker, args=(2, port, recording[0], out), nprocs=2, join=True)
    got = torch.load(out, weights_only=False)
    assert got[0]["brake"] == one[0]["brake"] and got == one


def test_cli_prints_the_brake_block(cuda, recording, tmp_path, capsys):
    import yaml
    from lav_b200 import evaluate as E
    lid, uni, bra = seeded_models()
    for name, m in (("lidar_1.th", lid), ("uniplanner_1.th", uni), ("bra.th", bra)):
        torch.save(m.state_dict(), tmp_path / name)
    cfg = yaml.safe_load(open(recording[0]))
    for k in CFG:                                                            # the controls come from --agent-config
        if k not in ("pixels_per_meter",):
            cfg.pop(k, None)
    cfg["aim_point"] = 4                                                     # config_v2.yaml's scalar
    yaml.safe_dump(cfg, open(tmp_path / "c.yaml", "w"))
    yaml.safe_dump(CFG, open(tmp_path / "agent.yaml", "w"))
    base = ["--config-path", str(tmp_path / "c.yaml"), "--data-dir", os.path.join(recording[1], "data"), "--lidar-weights",
            str(tmp_path / "lidar_1.th"), "--uniplanner-weights", str(tmp_path / "uniplanner_1.th"), "--batch-size", "6",
            "--num-workers", "2", "--brake", "--bra-weights", str(tmp_path / "bra.th")]
    from lav_b200.capi import LavbError
    with pytest.raises(LavbError, match="aim_point"):
        E.main(base)
    r = E.main(base + ["--agent-config", str(tmp_path / "agent.yaml"), "--json", str(tmp_path / "out.json")])
    printed = capsys.readouterr().out
    assert "brake decision" in printed and "collide_expert_tracks" in printed
    got = json.load(open(tmp_path / "out.json"))
    assert got == json.loads(json.dumps(r)) and got["brake"]["samples"] == got["samples"] > 0
    assert set(got["brake"]["verdicts"]) == {"agent", "brake_model", "plan_stop", "collide", "collide_expert_tracks"}
