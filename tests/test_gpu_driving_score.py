"""GPU: ops.driving_score against the numpy statement of tests/test_driving_score_cpu.py on random inputs and on its known
answers, its argument checks, and lav_b200.evaluate / evaluate_bev --driving-score against the statement and a per-sample loop on
the synthetic recording; DAC against plan_safety's off-road verdict; the unchanged default outputs; both CLIs and a sweep."""
import ctypes as C
import json

import numpy as np
import pytest
import torch

from lav_b200 import ops
from lav_b200.capi import LavbError, lib
from tests import test_driving_score_cpu as R
from tests.test_bev_train_cpu import _planner
from tests.test_gpu_evaluate import cfg_dir, recording, seeded_models  # noqa: F401  (recording is a fixture)
from tests.test_gpu_forecast_eval import batch_sizes

pytestmark = pytest.mark.gpu
DTYPE = ops.PLAN_SAFETY_ACTOR_DTYPE
F = R.FIELDS


def random_inputs(B, T, n, seed, big=None, actors=None):
    """traj (B, n, T, 2) fp32, expert (B, T, 2) fp32, actor records (T + 1 per row), offsets, ego_ext (B, 2), bev (B, 2, 320, 320)
    uint8: paths at 0 .. 12 m/s with stopped, short and turning steps, NaN and inf points; actors of classes 0 / 1 / 2 moving around
    the paths (some overtaking from behind, some crossing), absent at some steps; a blotchy road.  Sample 0 has no actor, sample
    ``big`` 2000; with ``actors`` every other sample has that many."""
    rs = np.random.RandomState(seed)
    counts = rs.randint(0, 40, B) if actors is None else np.full(B, actors)
    counts[0] = 0
    if big is not None:
        counts[big] = 2000
    speed = rs.choice([0.0, 0.01, 1.0, 5.0, 12.0], (B, n, 1)) * rs.uniform(0.5, 1.5, (B, n, T))
    step = speed * 0.25
    step[rs.rand(B, n, T) < 0.1] = 0.0
    yaw = -np.pi / 2 + rs.uniform(-0.3, 0.3, (B, n, 1)) + np.cumsum(rs.randn(B, n, T) * rs.choice([0.02, 0.3], (B, n, 1)), 2)
    traj = np.cumsum(np.stack([step * np.cos(yaw), step * np.sin(yaw)], 3), 2).astype(np.float32)
    bad = rs.rand(B, n, T) < 0.01
    traj[bad] = np.where(rs.rand(int(bad.sum()), 1) < 0.8, np.nan, np.inf)
    expert = traj[:, -1].copy()                                                       # the last trajectory, or a longer copy
    alt = rs.rand(B) < 0.3
    expert[alt] = traj[alt, 0] * np.float32(1.7)
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    rec = np.zeros((offsets[-1], T + 1), DTYPE)
    for b in range(B):
        a = rec[offsets[b]:offsets[b + 1]]
        m = len(a)
        if not m:
            continue
        j = rs.randint(0, n, m)
        anchor = np.nan_to_num(traj[b, j, rs.randint(0, T, m)].astype(np.float64), nan=0.0, posinf=0.0, neginf=0.0)
        base = anchor + rs.uniform(-6, 6, (m, 2))
        vel = rs.uniform(-3, 3, (m, 1, 2)) * rs.choice([0.0, 1.0], (m, 1, 1))
        a["x"] = base[:, None, 0] + vel[..., 0] * np.arange(T + 1)
        a["y"] = base[:, None, 1] + vel[..., 1] * np.arange(T + 1)
        psi = rs.uniform(-np.pi, np.pi, (m, 1)) + rs.randn(m, T + 1) * 0.05
        psi[::4] = np.round(psi[::4] / (np.pi / 2)) * (np.pi / 2)
        a["cos"], a["sin"] = np.cos(psi), np.sin(psi)
        a["e1"], a["e2"] = rs.uniform(0.2, 2.6, (m, 1)), rs.uniform(0.2, 1.2, (m, 1))
        a["typ"] = rs.choice([0, 1, 1, 2], (m, 1))
        a["present"] = rs.rand(m, T + 1) > 0.15
    ext = np.where(rs.rand(B, 1) < 0.5, [[2.4, 1.1]], rs.uniform(0.5, 3.0, (B, 2)))
    road = np.kron(rs.rand(B, 20, 20) > 0.04, np.ones((16, 16))).astype(np.uint8)
    bev = np.stack([road, rs.randint(0, 2, (B, 320, 320))], 1).astype(np.uint8)
    return traj, expert, rec.reshape(-1), offsets, ext.astype(np.float64), bev


def to_dev(dev, *arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in arrays]


def run(dev, traj, expert, rec, offsets, ext, bev, dt=R.DT, out=None):
    t, e, a, x, m = to_dev(dev, traj, expert, rec.view(np.uint8), ext, bev)
    return ops.driving_score(t, e, a, offsets, x, m, dt=dt, out=out)


def host(buf, b, n):
    """(res (b, n, 16) int32, ep (b, n, 2) fp64) of a result buffer."""
    v = ops.driving_score_views(buf.cpu(), b, n)
    return (np.stack([v[k].numpy() for k in ops.DRIVING_SCORE_FIELDS], -1),
            np.stack([v["progress"].numpy(), v["length"].numpy()], -1))


def check_equal(got, want):
    """integer fields equal but a comfort term within NEAR of its bound; s and L within 1e-12 relative (NaN to NaN, inf to
    inf)."""
    (res, ep), (wres, wep, near) = got, want
    diff = res != wres
    comfort = np.zeros_like(diff)
    comfort[..., F["comfort_mask"]] = True
    comfort[..., 10:15] = True
    assert not (diff & ~comfort).any(), np.argwhere(diff & ~comfort)[:5]
    for q in range(5):
        d = ((res[..., F["comfort_mask"]] ^ wres[..., F["comfort_mask"]]) >> q) & 1 | (res[..., 10 + q] != wres[..., 10 + q])
        assert not (d.astype(bool) & ~near[..., q]).any(), (q, np.argwhere(d.astype(bool) & ~near[..., q])[:5])
    assert np.array_equal(np.isnan(ep), np.isnan(wep))
    got, want = ep[~np.isnan(wep)], wep[~np.isnan(wep)]
    with np.errstate(invalid="ignore"):
        close = (got == want) | (np.abs(got - want) <= 1e-12 * np.abs(want))
    assert close.all(), (got[~close][:5], want[~close][:5])


@pytest.mark.parametrize("B", [1, 32, 256])
@pytest.mark.parametrize("T", [1, 2, 3, 20])
def test_driving_score_equals_the_numpy_statement(cuda, B, T):
    big = B // 2 if B > 1 else 0 if T == 20 else None                                  # B = 1: 2000 actors or none
    inputs = random_inputs(B, T, 2, 1000 * B + T, big=big)
    traj, expert, rec, offsets, ext, bev = inputs
    got = host(run(cuda, *inputs), B, 2)
    want = R.driving_score_ref(traj, expert, rec, offsets, ext, bev[:, 0])
    check_equal(got, want)
    if B == 256 and T == 20:
        res = want[0]
        for k in ("fault_step", "exempt_step", "ttc_step", "off_road_step", "invalid_step"):
            assert (res[..., F[k]] > 0).any() and (res[..., F[k]] < 0).any(), k
        assert (res[..., F["comfort_mask"]] > 0).any() and (res[..., F["comfort_mask"]] == 0).any()
        assert set(res[..., F["fault_class"]].ravel().tolist()) >= {0, 1}


@pytest.mark.parametrize("dt", [0.1, 0.5, 2.0])
def test_other_step_periods(cuda, dt):
    inputs = random_inputs(16, 10, 2, 77)
    traj, expert, rec, offsets, ext, bev = inputs
    check_equal(host(run(cuda, *inputs, dt=dt), 16, 2), R.driving_score_ref(traj, expert, rec, offsets, ext, bev[:, 0], dt=dt))


@pytest.mark.parametrize("name", ["moving_ego", "from_behind", "stopped_ego", "crossing", "progress", "braking", "zig_zag",
                                  "off_road", "nan", "overlap_at_0", "classes"])
def test_known_answers(cuda, name, monkeypatch):
    """each hand-built case of the CPU statement, run through the kernel instead."""
    def kernel(traj, expert, actors, offsets, ext, road):
        b, n = traj.shape[:2]
        res, ep = host(run(cuda, traj, expert, actors, offsets, ext, road[:, None]), b, n)
        return res, ep, np.zeros((b, n, 5), bool)
    monkeypatch.setattr(R, "driving_score_ref", kernel)
    case = {"moving_ego": R.test_moving_ego_runs_into_a_stopped_car, "from_behind": R.test_a_faster_car_from_behind_is_exempt,
            "stopped_ego": R.test_a_stopped_ego_that_is_hit_keeps_nc, "progress": R.test_progress_along_the_expert,
            "braking": R.test_hard_braking_fails_only_the_acceleration, "zig_zag": R.test_a_two_step_zig_zag_fails_only_the_yaw_rate,
            "off_road": R.test_an_off_road_corner_gives_dac_0, "nan": R.test_a_nan_step_makes_the_trajectory_invalid,
            "overlap_at_0": R.test_an_overlap_present_at_step_0_is_not_new,
            "classes": R.test_classes_other_than_vehicles_and_pedestrians_are_ignored}
    if name == "crossing":
        R.test_a_car_crossing_ahead(2, 1)
        R.test_a_car_crossing_ahead(8, -1)
    else:
        case[name]()


def test_driving_score_rejects_malformed_arguments_and_writes_nothing(cuda):
    traj, expert, rec, offsets, ext, bev = random_inputs(4, 10, 2, 5, actors=3)
    nbytes = ops._layout(ops._driving_parts(4, 2))[1]
    out = torch.full((nbytes,), 0x7B, dtype=torch.uint8, device=cuda)
    bad = [dict(offsets=np.array([0, 3, 2, 5, offsets[-1]], np.int32)),                  # not monotone
           dict(offsets=np.array([0, 1, 2, 3, offsets[-1] + 1], np.int32)),              # past the actor rows
           dict(offsets=offsets[:-1]), dict(offsets=offsets.astype(np.int64)),
           dict(traj=traj[:, :, :, :1].copy()), dict(traj=np.zeros((4, 9, 10, 2), np.float32)),   # over 8 trajectories
           dict(traj=np.zeros((4, 2, 33, 2), np.float32), expert=np.zeros((4, 33, 2), np.float32),
                rec=np.zeros(offsets[-1] * 34, DTYPE)),                                   # over 32 steps
           dict(expert=expert[:, :9].copy()), dict(expert=expert.astype(np.float64)),
           dict(rec=rec[:-1]), dict(rec=rec.reshape(-1, 11)[:, :10].copy().reshape(-1)),  # T records per row, not T + 1
           dict(ext=ext[:, :1].copy()), dict(ext=ext.astype(np.float32)),
           dict(bev=bev[:, 0].copy()), dict(bev=bev[:3].copy()),
           dict(dt=0.0), dict(dt=-0.25), dict(dt=float("nan")), dict(dt=float("inf")), dict(dt=0.01)]   # 100 projections
    for kw in bad:
        args = dict(traj=traj, expert=expert, rec=rec, offsets=offsets, ext=ext, bev=bev)
        args.update(kw)
        with pytest.raises(LavbError):
            run(cuda, out=out, **args)
    with pytest.raises(LavbError):
        run(cuda, traj, expert, rec, offsets, ext, bev, out=out[:-1])
    t, e, a, x, m = to_dev(cuda, traj, expert, rec.view(np.uint8), ext, bev)
    with pytest.raises(LavbError):
        ops.driving_score(t.cpu(), e, a, offsets, x, m, out=out)
    with pytest.raises(LavbError):                                                           # out over an input
        ops.driving_score(t, e, a, offsets, x, m, out=a[:nbytes] if a.numel() >= nbytes else m.view(-1)[:nbytes])
    ptr = lambda v: C.c_void_p(v.data_ptr())
    st, null = C.c_void_p(torch.cuda.current_stream().cuda_stream), C.c_void_p(0)
    v = ops._views(out, ops._driving_parts(4, 2))
    dev_ptrs = [ptr(t), ptr(e), ptr(a), ptr(x), ptr(m), ptr(v["ep"]), ptr(v["res"])]

    def call(d, n=2, T=10, stride=2 * 320 * 320, ppm=4.0, dt=0.25, offs=offsets):
        return lib().lavb_driving_score(d[0], d[1], 4, n, T, d[2], len(rec) // 11, offs.ctypes.data_as(C.c_void_p), d[3], d[4], stride,
                                        320, 320, ppm, 160.0, 320.0, -40.0, dt, d[5], d[6], st)
    for i in range(len(dev_ptrs)):                                                          # each device pointer null in turn
        d = list(dev_ptrs)
        d[i] = null
        assert call(d) != 0
    assert call(dev_ptrs, n=0) != 0 and call(dev_ptrs, n=9) != 0 and call(dev_ptrs, T=0) != 0 and call(dev_ptrs, T=33) != 0
    assert call(dev_ptrs, stride=320 * 320 - 1) != 0 and call(dev_ptrs, ppm=0.0) != 0 and call(dev_ptrs, ppm=float("nan")) != 0
    assert call(dev_ptrs, dt=0.0) != 0 and call(dev_ptrs, dt=float("inf")) != 0 and call(dev_ptrs, dt=1 / 65) != 0
    for k in (0, 1, 2, 3, 5):                                                               # 8-byte inputs and ep misaligned
        d = list(dev_ptrs)
        d[k] = C.c_void_p(d[k].value + 4)
        assert call(d) != 0
    torch.cuda.synchronize()
    assert bool((out == 0x7B).all())


# ---------------------------------------------------------------------------------------------------- the evaluators
class Recorder:
    """wraps ops.driving_score (and ops.plan_safety): per batch their host inputs and results."""

    def __init__(self):
        self.calls, self.safety = [], []

    def __enter__(self):
        self.f, self.g = ops.driving_score, ops.plan_safety
        hostv = lambda t: t.cpu().numpy() if torch.is_tensor(t) else np.asarray(t)

        def driving_score(traj, expert, actors, offsets, ego_ext, bev, grid=None, dt=ops.DRIVING_SCORE_STEP_S, out=None):
            buf = self.f(traj, expert, actors, offsets, ego_ext, bev, grid, dt, out)
            b, n = traj.shape[:2]
            self.calls.append(([hostv(traj), hostv(expert), hostv(actors).view(DTYPE), hostv(offsets), hostv(ego_ext),
                                hostv(bev[:, 0])], dt, host(buf, b, n)))
            return buf

        def plan_safety(traj, actors, offsets, ego_ext, bev, grid=None, out=None):
            res = self.g(traj, actors, offsets, ego_ext, bev, grid, out)
            self.safety.append(hostv(res))
            return res
        ops.driving_score, ops.plan_safety = driving_score, plan_safety
        return self

    def __exit__(self, *exc):
        ops.driving_score, ops.plan_safety = self.f, self.g


def expert_loop(ds, prepare_args):
    """per sample at B = 1: ops.driving_score on the unaugmented sample's expert alone, against its own table and road."""
    from lav_b200.datasets import stage_plan_safety
    dev, out = ds.device, []
    for idx in range(len(ds)):
        h = ds.prepare(idx, *prepare_args, driving_score=True)
        table = stage_plan_safety([h["driving_score"]], False)
        bev = ds.bev_batch([h])
        expert = torch.as_tensor(h["ego_locs"][1:], dtype=torch.float32, device=dev)[None].contiguous()
        buf = ops.driving_score(expert[:, None].contiguous(), expert, table["actors"].to(dev), table["offsets"],
                                table["ego_ext"].to(dev), bev)
        res, ep = host(buf, 1, 1)
        out.append((res[0, 0], ep[0, 0], h["cmd"]))
    return out


def check_evaluator(rec, loop, result, sizes, dt=R.DT):
    from lav_b200.evaluate import DrivingScores
    assert [len(c[0][0]) for c in rec.calls] == sizes
    s0, red = 0, DrivingScores(dt=dt)
    for inputs, got_dt, (res, ep) in rec.calls:
        assert got_dt == dt
        check_equal((res, ep), R.driving_score_ref(*inputs, dt=dt))
        b = len(res)
        for i in range(b):
            assert np.array_equal(res[i, 1], loop[s0 + i][0]), (s0 + i, res[i, 1], loop[s0 + i][0])
            assert np.array_equal(ep[i, 1], loop[s0 + i][1], equal_nan=True)
        buf = torch.zeros(ops._layout(ops._driving_parts(b, 2))[1], dtype=torch.uint8)
        v = ops._views(buf, ops._driving_parts(b, 2))
        v["res"].copy_(torch.from_numpy(res))
        v["ep"].copy_(torch.from_numpy(ep))
        red.add(buf, [c for _, _, c in loop[s0:s0 + b]])
        s0 += b
    assert s0 == len(loop)
    assert result["driving_score"] == red.summary()
    return np.concatenate([r for _, _, (r, _) in rec.calls]), np.concatenate([e for _, _, (_, e) in rec.calls])


def check_dac_and_expert(rec, res, ep):
    """DAC is plan_safety's off-road verdict sample for sample; the expert's EP is 1."""
    from lav_b200.evaluate import driving_terms
    safety = np.concatenate(rec.safety)
    assert np.array_equal(res[..., F["off_road_step"]], safety[..., 4])
    v = {k: res[..., i] for k, i in F.items()}
    v["progress"], v["length"] = ep[..., 0], ep[..., 1]
    t = driving_terms(v)
    valid = ~t["invalid"][:, 1]
    assert valid.any() and (t["ep"][valid, 1] == 1.0).all()


def test_evaluate_driving_score(cuda, recording):
    import lav_b200.evaluate as EV
    from lav_b200.datasets import TemporalLiDARPaintedDataset
    ds = TemporalLiDARPaintedDataset(recording[0], device=cuda)
    n = len(ds)
    lid, uni = seeded_models()
    loop = expert_loop(ds, ds.no_draw())
    for bs in batch_sizes(n):
        with Recorder() as rec:
            result = EV.evaluate(lid, uni, ds, batch_size=bs, precision="fp32", num_workers=4, plan_safety=True, driving_score=True)
        res, ep = check_evaluator(rec, loop, result, [min(bs, n - k) for k in range(0, n, bs)])
        check_dac_and_expert(rec, res, ep)
        print(f"evaluate --driving-score, batch {bs}: {json.dumps(result['driving_score']['plan'])}")
    with Recorder() as rec:                                                   # another step period, without --plan-safety
        result = EV.evaluate(lid, uni, ds, batch_size=8, precision="fp32", num_workers=4, driving_score=True, step_seconds=0.1)
    assert "plan_safety" not in result and result["driving_score"]["step_seconds"] == 0.1 and not rec.safety
    for inputs, dt, got in rec.calls:
        check_equal(got, R.driving_score_ref(*inputs, dt=0.1))


def test_evaluate_bev_driving_score(cuda, recording):
    import lav_b200.evaluate_bev as EB
    from lav_b200.datasets import TemporalBEVDataset
    ds = TemporalBEVDataset(recording[0], device=cuda)
    n = len(ds)
    planner = _planner(2021).to(cuda).eval()
    loop = expert_loop(ds, ds.no_draw())
    for bs in batch_sizes(n):
        with Recorder() as rec:
            result = EB.evaluate_bev(planner, ds, batch_size=bs, num_workers=4, plan_safety=True, driving_score=True)
        res, ep = check_evaluator(rec, loop, result, [min(bs, n - k) for k in range(0, n, bs)])
        check_dac_and_expert(rec, res, ep)
        assert set(result) == {"samples", "forecast", "plan_safety", "driving_score"}
        assert set(result["driving_score"]) == {"plan", "expert", "step_seconds"}


def test_default_outputs_have_no_new_key(cuda, recording):
    import lav_b200.evaluate as EV
    import lav_b200.evaluate_bev as EB
    from lav_b200.datasets import TemporalBEVDataset, TemporalLiDARPaintedDataset
    lid, uni = seeded_models()
    ds = TemporalLiDARPaintedDataset(recording[0], device=cuda)
    plain = EV.evaluate(lid, uni, ds, batch_size=4, precision="fp32", num_workers=2)
    both = EV.evaluate(lid, uni, ds, batch_size=4, precision="fp32", num_workers=2, driving_score=True)
    assert "driving_score" not in plain and set(both) == set(plain) | {"driving_score"}
    assert both["samples"] == plain["samples"] and both["driving_score"]["plan"]["samples"] == plain["samples"]
    bds = TemporalBEVDataset(recording[0], device=cuda)
    planner = _planner(2021).to(cuda).eval()
    bplain = EB.evaluate_bev(planner, bds, batch_size=4, num_workers=2)
    bboth = EB.evaluate_bev(planner, bds, batch_size=4, num_workers=2, driving_score=True)
    assert set(bplain) == {"samples", "forecast"} and set(bboth) == {"samples", "forecast", "driving_score"}


def test_clis_driving_score_write_the_json_and_a_sweep_prints_pdms(cuda, recording, tmp_path, capsys):
    import yaml
    from lav_b200 import evaluate as EV
    from lav_b200 import evaluate_bev as EB
    lid, uni = seeded_models()
    torch.save(lid.state_dict(), tmp_path / "lidar_1.th")
    torch.save(uni.state_dict(), tmp_path / "uniplanner_1.th")
    torch.save(_planner(2021).state_dict(), tmp_path / "bev_1.th")
    torch.save(_planner(7).state_dict(), tmp_path / "bev_2.th")
    cfg = yaml.safe_load(open(recording[0]))
    cfg["data_dir"] = "/nonexistent"
    yaml.safe_dump(cfg, open(tmp_path / "c.yaml", "w"))
    common = ["--config-path", str(tmp_path / "c.yaml"), "--data-dir", cfg_dir(recording), "--batch-size", "5", "--num-workers", "2",
              "--driving-score"]
    r = EV.main(common + ["--lidar-weights", str(tmp_path / "lidar_1.th"), "--uniplanner-weights", str(tmp_path / "uniplanner_1.th"),
                          "--json", str(tmp_path / "out.json")])
    got = json.load(open(tmp_path / "out.json"))
    assert got == json.loads(json.dumps(r)) and set(got["driving_score"]) == {"plan", "expert", "step_seconds"}
    assert got["driving_score"]["expert"]["samples"] == got["samples"]
    assert "driving score, plan" in capsys.readouterr().out
    rb = EB.main(common + ["--bev-weights", str(tmp_path / "bev_1.th"), "--json", str(tmp_path / "bev.json")])
    gotb = json.load(open(tmp_path / "bev.json"))
    assert gotb == json.loads(json.dumps(rb)) and gotb["driving_score"]["expert"] == got["driving_score"]["expert"]
    capsys.readouterr()
    sweep = EB.main(common + ["--bev-weights", str(tmp_path / "bev_1.th"), str(tmp_path / "bev_2.th")])
    text = capsys.readouterr().out
    assert "PDMS" in text.splitlines()[1] and len(sweep["checkpoints"]) == 2
    assert sweep["checkpoints"][0]["result"]["driving_score"] == gotb["driving_score"]
