"""GPU: ops.plan_safety against the numpy statement of tests/test_plan_safety_cpu.py and its known answers, its argument checks, a
world-coordinate recording with known answers for the expert, and lav_b200.evaluate / evaluate_bev --plan-safety against the
statement and a per-sample loop on the synthetic recording; the unchanged default outputs; both CLIs."""
import ctypes as C
import json
import math
import os

import numpy as np
import pytest
import torch

from lav_b200 import ops
from lav_b200.capi import LavbError, lib
from tests import test_plan_safety_cpu as R
from tests.test_bev_train_cpu import _planner
from tests.test_gpu_evaluate import cfg_dir, recording, seeded_models  # noqa: F401  (recording is a fixture)
from tests.test_gpu_forecast_eval import batch_sizes

pytestmark = pytest.mark.gpu
DTYPE = ops.PLAN_SAFETY_ACTOR_DTYPE


def random_inputs(B, T, n, seed, big=None, actors=None):
    """traj (B, n, T, 2) fp32, actor records, offsets, ego_ext (B, 2), bev (B, 2, 320, 320) uint8 of B samples: turning paths
    with short and stationary steps, points on pixel edges, NaN and inf points; actors of classes 0 / 1 / 2 around the paths,
    some absent at some steps; a blotchy road plane.  Sample 0 has no actor, sample 1 one, sample ``big`` 2000; with ``actors``
    every sample has that many instead."""
    rs = np.random.RandomState(seed)
    counts = rs.randint(0, 40, B)
    counts[0] = 0
    if B > 1:
        counts[1] = 1
    if actors is not None:
        counts[:] = actors
    if big is not None:
        counts[big] = 2000
    step = rs.uniform(0.0, 2.0, (B, n, T))
    step[rs.rand(B, n, T) < 0.15] = rs.uniform(0.0, 0.12)
    yaw = -np.pi / 2 + rs.uniform(-0.5, 0.5, (B, n, 1)) + np.cumsum(rs.randn(B, n, T) * 0.2, 2)
    traj = np.cumsum(np.stack([step * np.cos(yaw), step * np.sin(yaw)], 3), 2)
    traj[:, :, ::3] = np.round(traj[:, :, ::3] * 4) / 4                               # on pixel edges
    traj = traj.astype(np.float32)
    bad = rs.rand(B, n, T) < 0.02
    traj[bad] = np.where(rs.rand(int(bad.sum()), 1) < 0.8, np.nan, np.inf)
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    rec = np.zeros((offsets[-1], T), DTYPE)
    for b in range(B):
        a = rec[offsets[b]:offsets[b + 1]]
        m = len(a)
        if not m:
            continue
        anchor = np.nan_to_num(traj[b, rs.randint(0, n, m), rs.randint(0, T, m)].astype(np.float64), nan=0.0, posinf=0.0)
        base = anchor + rs.uniform(-4, 4, (m, 2))
        base[::4] = np.round(base[::4] * 4) / 4
        drift = rs.uniform(-0.3, 0.3, (m, 1, 2)) * np.arange(1, T + 1)[None, :, None]
        psi = rs.uniform(-np.pi, np.pi, (m, 1)) + rs.randn(m, T) * 0.05
        psi[::5] = np.round(psi[::5] / (np.pi / 2)) * (np.pi / 2)
        a["x"], a["y"] = base[:, None, 0] + drift[..., 0], base[:, None, 1] + drift[..., 1]
        a["cos"], a["sin"] = np.cos(psi), np.sin(psi)
        a["e1"], a["e2"] = rs.uniform(0.2, 2.6, (m, 1)), rs.uniform(0.2, 1.2, (m, 1))
        a["typ"] = rs.choice([0, 1, 1, 2], (m, 1))
        a["present"] = rs.rand(m, T) > 0.2
    ext = np.where(rs.rand(B, 1) < 0.5, [[2.4, 1.1]], rs.uniform(0.5, 3.0, (B, 2)))
    road = np.kron(rs.rand(B, 20, 20) > 0.06, np.ones((16, 16))).astype(np.uint8)
    bev = np.stack([road, rs.randint(0, 2, (B, 320, 320))], 1).astype(np.uint8)
    return traj, rec.reshape(-1), offsets, ext.astype(np.float64), bev


def to_dev(dev, *arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in arrays]


def run(dev, traj, rec, offsets, ext, bev, out=None):
    t, a, e, m = to_dev(dev, traj, rec.view(np.uint8), ext, bev)
    return ops.plan_safety(t, a, offsets, e, m, out=out)


@pytest.mark.parametrize("B", [1, 7, 64, 300])
@pytest.mark.parametrize("T", [10, 20])
@pytest.mark.parametrize("n", [1, 2])
def test_plan_safety_equals_the_numpy_statement(cuda, B, T, n):
    inputs = random_inputs(B, T, n, 1000 * B + 10 * T + n, big=B // 2 if B > 2 else None)
    got = run(cuda, *inputs).cpu().numpy()
    traj, rec, offsets, ext, bev = inputs
    want = R.plan_safety_ref(traj, rec, offsets, ext, bev[:, 0])
    assert np.array_equal(got, want), np.argwhere(got != want)[:5]
    if B >= 64:
        assert (want[..., 0] > 0).any() and (want[..., 2] > 0).any() and (want[..., 4] > 0).any() and (want[..., 6] > 0).any()
        assert (want[..., 0] < 0).any() and (want[..., 4] < 0).any()


@pytest.mark.parametrize("case", R.case_table(), ids=lambda c: c[0])
def test_known_answers(cuda, case):
    name, traj, rows, road, want = case

    def kernel(traj, actors, offsets, ext, road):
        return run(cuda, traj, actors, offsets, ext, road[:, None]).cpu().numpy()
    assert R.run_case(traj, rows, road, kernel).tolist() == want, name


def test_plan_safety_rejects_malformed_arguments_and_writes_nothing(cuda):
    traj, rec, offsets, ext, bev = random_inputs(4, 10, 2, 5)
    out = torch.full((4, 2, 8), 0x7B7B7B7B, dtype=torch.int32, device=cuda)
    bad = [dict(offsets=np.array([0, 3, 2, 5, offsets[-1]], np.int32)),                  # not monotone
           dict(offsets=np.array([0, 1, 2, 3, offsets[-1] + 1], np.int32)),              # past the actor rows
           dict(offsets=offsets[:-1]), dict(offsets=offsets.astype(np.int64)),
           dict(traj=traj[:, :, :, :1].copy()), dict(traj=np.zeros((4, 9, 10, 2), np.float32)),   # over 8 trajectories
           dict(traj=np.zeros((4, 2, 33, 2), np.float32), rec=np.zeros(offsets[-1] * 33, DTYPE)),  # over 32 steps
           dict(rec=rec[:-1]), dict(ext=ext[:, :1].copy()), dict(ext=ext.astype(np.float32)),
           dict(bev=bev[:, 0].copy()), dict(bev=bev[:3].copy())]
    for kw in bad:
        args = dict(traj=traj, rec=rec, offsets=offsets, ext=ext, bev=bev)
        args.update(kw)
        with pytest.raises(LavbError):
            run(cuda, out=out, **args)
    with pytest.raises(LavbError):
        run(cuda, traj, rec, offsets, ext, bev, out=out[:3])
    t, a, e, m = to_dev(cuda, traj, rec.view(np.uint8), ext, bev)
    with pytest.raises(LavbError):
        ops.plan_safety(t.cpu(), a, offsets, e, m, out=out)
    ptr = lambda x: C.c_void_p(x.data_ptr())
    st, null = C.c_void_p(torch.cuda.current_stream().cuda_stream), C.c_void_p(0)
    dev_ptrs = [ptr(t), ptr(a), ptr(e), ptr(m), ptr(out)]

    def call(d, n=2, T=10, stride=2 * 320 * 320, ppm=4.0, offs=offsets):
        return lib().lavb_plan_safety(d[0], 4, n, T, d[1], len(rec) // 10, offs.ctypes.data_as(C.c_void_p), d[2], d[3], stride, 320,
                                      320, ppm, 160.0, 320.0, -40.0, d[4], st)
    for i in range(len(dev_ptrs)):                                                          # each device pointer null in turn
        d = list(dev_ptrs)
        d[i] = null
        assert call(d) != 0
    assert call(dev_ptrs, n=0) != 0 and call(dev_ptrs, n=9) != 0 and call(dev_ptrs, T=0) != 0 and call(dev_ptrs, T=33) != 0
    assert call(dev_ptrs, stride=320 * 320 - 1) != 0 and call(dev_ptrs, ppm=0.0) != 0 and call(dev_ptrs, ppm=float("nan")) != 0
    assert lib().lavb_plan_safety(dev_ptrs[0], 4, 2, 10, dev_ptrs[1], 0, null, dev_ptrs[2], dev_ptrs[3], 2 * 320 * 320, 320, 320,
                                  4.0, 160.0, 320.0, -40.0, dev_ptrs[4], st) != 0                  # no host offsets
    for k in (0, 1, 2):                                                                     # traj, actors, ego_ext misaligned
        d = list(dev_ptrs)
        d[k] = C.c_void_p([t, a, e][k].data_ptr() + 4)
        assert call(d) != 0
    torch.cuda.synchronize()
    assert bool((out == 0x7B7B7B7B).all())


# ---------------------------------------------------------------------------------------------------- a world-coordinate fixture
SPEED = 1.5          # metres per frame along the ego's heading
PARKED_M = 28.0      # a car parked ahead, beyond the 25 m vehicle radius of the labels
SIDE_M = (5.0, 3.0)  # a car 5 m ahead and 3 m to the side


def write_fixture(root, turned, yaw_deg=37.0, n_frames=22):
    """one trajectory through data_paint.DirEnv, in the record layout synth.record_trajectories writes: the ego (2.4 x 1.1 half
    extents) driving straight at SPEED m per frame along yaw_deg, a 2.0 x 0.9 car parked PARKED_M ahead along the same heading,
    and one at SIDE_M beside the path, along it or, with ``turned``, across it; map plane 0 a road band |x| < 3 m around the
    path, every other plane empty."""
    from lav_b200.data_paint import DirEnv
    from lav_b200.synth import encode_png
    env = DirEnv(os.path.join(root, f"traj_{int(turned)}"))
    env.put("len", str(n_frames).encode())
    env.put("town", b"Town01")
    y = math.radians(yaw_deg)
    fwd, left = np.array([math.cos(y), math.sin(y)]), np.array([-math.sin(y), math.cos(y)])
    start = np.array([50.0, -20.0])
    road = np.zeros((320, 320), np.uint8)
    road[:, 148:172] = 255
    empty = np.zeros((320, 320), np.uint8)
    for f in range(n_frames):
        locs = [start + SPEED * f * fwd, start + PARKED_M * fwd, start + SIDE_M[0] * fwd + SIDE_M[1] * left]
        env.put(f"id_{f:05d}", np.array([5, 60, 11], np.int32).tobytes())
        env.put(f"loc_{f:05d}", np.array(locs, np.float32).tobytes())
        env.put(f"ori_{f:05d}", np.array([yaw_deg, yaw_deg, yaw_deg + (90.0 if turned else 0.0)], np.float32).tobytes())
        env.put(f"bbox_{f:05d}", np.array([[2.4, 1.1], [2.0, 0.9], [2.0, 0.9]], np.float32).tobytes())
        env.put(f"type_{f:05d}", np.array([1, 1, 1], np.uint8).tobytes())
        env.put(f"cmd_{f:05d}", np.array([3], np.uint8).tobytes())
        env.put(f"bra_{f:05d}", np.array([0], np.uint8).tobytes())
        env.put(f"nxp_{f:05d}", (start + (SPEED * f + 20) * fwd).astype(np.float32).tobytes())
        for c in range(12):
            env.put(f"map_{c}_{f:05d}", encode_png(road if c == 0 else empty))


def first_step(index, lo, hi):
    """by hand: the first step t (1..20) whose ego box, [SPEED t - 2.4, SPEED t + 2.4] metres ahead of the ego of frame
    ``index``, overlaps a box spanning (lo, hi) metres ahead of the first frame's ego."""
    for t in range(1, 21):
        if SPEED * t - 2.4 < hi - SPEED * index and SPEED * t + 2.4 > lo - SPEED * index:
            return t
    return -1


def test_world_fixture_known_answers(cuda, recording, tmp_path):
    from lav_b200.datasets import TemporalBEVDataset, stage_plan_safety
    root = str(tmp_path / "fixture")
    write_fixture(root, turned=False)
    write_fixture(root, turned=True)
    ds = TemporalBEVDataset(recording[0], device=cuda, overrides=dict(data_dir=root, percentage_data=1.0, all_towns=True))
    assert len(ds) == 4 and ds.num_plan == 20
    for idx in range(len(ds)):
        traj_no, index = ds.index[idx]
        turned = ds.paths[traj_no].endswith("traj_1")
        h = ds.prepare(idx, 0, 0.0, plan_safety=True)
        assert len(h["plan_safety"]["locs"]) == 2 and h["plan_safety"]["present"].all()      # the ego is not an actor
        bev = ds.bev_batch([h])
        expert = torch.as_tensor(h["ego_locs"][1:], dtype=torch.float32, device=cuda)
        traj = torch.stack([expert, expert + torch.tensor([6.0, 0.0], device=cuda)])[None].contiguous()
        table = stage_plan_safety([h["plan_safety"]], False)
        res = ops.plan_safety(traj, table["actors"].to(cuda), table["offsets"], table["ego_ext"].to(cuda), bev)
        v = {k: x.cpu().numpy()[0] for k, x in ops.plan_safety_views(res).items()}
        parked = first_step(index, PARKED_M - 2.0, PARKED_M + 2.0)
        side = first_step(index, SIDE_M[0] - 0.9, SIDE_M[0] + 0.9) if turned else -1
        assert parked == (16 if index == 0 else 15) and side in ((-1,) if not turned else (2,) if index == 0 else (1,))
        rows = {60: 1, 11: 0}                                                             # actor rows in id order: 11, 60
        want_step, want_row = (side, rows[11]) if turned else (parked, rows[60])
        assert (v["veh_step"][0], v["veh_row"][0]) == (want_step, want_row), (idx, turned, v)
        assert v["ped_step"][0] == -1 and v["off_road_step"][0] == -1 and v["invalid_steps"][0] == 0 and v["off_map_steps"][0] == 0
        assert v["off_road_step"][1] == 1                                                 # 6 m beside the road band
        assert np.array_equal(res.cpu().numpy(), R.plan_safety_ref(traj.cpu().numpy(), table["actors"].numpy().view(DTYPE),
                                                                    table["offsets"].numpy(), table["ego_ext"].numpy(),
                                                                    bev[:, 0].cpu().numpy()))


# ---------------------------------------------------------------------------------------------------- the evaluators
class Recorder:
    """wraps ops.plan_safety: per batch its host inputs and result."""

    def __init__(self):
        self.calls = []

    def __enter__(self):
        self.f = ops.plan_safety

        def plan_safety(traj, actors, offsets, ego_ext, bev, grid=None, out=None):
            res = self.f(traj, actors, offsets, ego_ext, bev, grid, out)
            host = lambda t: t.cpu().numpy() if torch.is_tensor(t) else np.asarray(t)
            self.calls.append(([host(traj), host(actors).view(DTYPE), host(offsets), host(ego_ext), host(bev[:, 0])], host(res)))
            return res
        ops.plan_safety = plan_safety
        return self

    def __exit__(self, *exc):
        ops.plan_safety = self.f


def expert_loop(ds, prepare_args):
    """per sample at B = 1: the unaugmented sample's table and road plane, and ops.plan_safety on its expert alone."""
    from lav_b200.datasets import stage_plan_safety
    dev, out = ds.device, []
    for idx in range(len(ds)):
        h = ds.prepare(idx, *prepare_args, plan_safety=True)
        table = stage_plan_safety([h["plan_safety"]], False)
        bev = ds.bev_batch([h])
        expert = torch.as_tensor(h["ego_locs"][1:], dtype=torch.float32, device=dev)[None, None].contiguous()
        res = ops.plan_safety(expert, table["actors"].to(dev), table["offsets"], table["ego_ext"].to(dev), bev)
        out.append((res.cpu().numpy()[0, 0], h["cmd"]))
    return out


def check_evaluator(rec, loop, result, sizes, T):
    from lav_b200.evaluate import PlanSafetyScores
    assert [len(c[0][0]) for c in rec.calls] == sizes
    s0, red = 0, PlanSafetyScores()
    for inputs, res in rec.calls:
        assert np.array_equal(res, R.plan_safety_ref(*inputs)), "the kernel on what the evaluator fed it"
        b = len(res)
        for i in range(b):
            assert np.array_equal(res[i, 1], loop[s0 + i][0]), (s0 + i, res[i, 1], loop[s0 + i][0])
        red.add(res, [c for _, c in loop[s0:s0 + b]])
        s0 += b
    assert s0 == len(loop)
    assert result["plan_safety"] == red.summary(T)
    return np.concatenate([r for _, r in rec.calls])


def test_evaluate_plan_safety(cuda, recording):
    import lav_b200.evaluate as EV
    from lav_b200.datasets import TemporalLiDARPaintedDataset
    ds = TemporalLiDARPaintedDataset(recording[0], device=cuda)
    n = len(ds)
    lid, uni = seeded_models()
    loop = expert_loop(ds, ds.no_draw())
    for bs in batch_sizes(n):
        with Recorder() as rec:
            result = EV.evaluate(lid, uni, ds, batch_size=bs, precision="fp32", num_workers=4, plan_safety=True)
        allres = check_evaluator(rec, loop, result, [min(bs, n - k) for k in range(0, n, bs)], ds.num_plan)
        print(f"evaluate --plan-safety, batch {bs}: expert first collisions {allres[:, 1, 7].tolist()}, off-road "
              f"{allres[:, 1, 4].tolist()}; {json.dumps(result['plan_safety']['plan'])}")


def test_evaluate_bev_plan_safety(cuda, recording):
    import lav_b200.evaluate_bev as EB
    from lav_b200.datasets import TemporalBEVDataset
    ds = TemporalBEVDataset(recording[0], device=cuda)
    n = len(ds)
    planner = _planner(2021).to(cuda).eval()
    loop = expert_loop(ds, ds.no_draw())
    for bs in batch_sizes(n):
        with Recorder() as rec:
            result = EB.evaluate_bev(planner, ds, batch_size=bs, num_workers=4, plan_safety=True)
        check_evaluator(rec, loop, result, [min(bs, n - k) for k in range(0, n, bs)], ds.num_plan)
        assert set(result) == {"samples", "forecast", "plan_safety"} and set(result["plan_safety"]) == {"plan", "expert"}


def test_recorded_branch_picks_the_command():
    from lav_b200.evaluate_bev import recorded_branch
    plan = torch.arange(3 * 4 * 2 * 2, dtype=torch.float32).view(3, 4, 2, 2)
    got = recorded_branch(plan, torch.tensor([2, 0, 7]))
    assert torch.equal(got[0], plan[0, 2]) and torch.equal(got[1], plan[1, 0]) and bool(got[2].isnan().all())


def test_default_outputs_have_no_new_key(cuda, recording):
    import lav_b200.evaluate as EV
    import lav_b200.evaluate_bev as EB
    from lav_b200.datasets import TemporalBEVDataset, TemporalLiDARPaintedDataset
    lid, uni = seeded_models()
    ds = TemporalLiDARPaintedDataset(recording[0], device=cuda)
    plain = EV.evaluate(lid, uni, ds, batch_size=4, precision="fp32", num_workers=2)
    both = EV.evaluate(lid, uni, ds, batch_size=4, precision="fp32", num_workers=2, plan_safety=True)
    assert "plan_safety" not in plain and set(both) == set(plain) | {"plan_safety"}
    assert both["samples"] == plain["samples"] and both["plan_safety"]["plan"]["samples"] == plain["samples"]
    bds = TemporalBEVDataset(recording[0], device=cuda)
    bplain = EB.evaluate_bev(_planner(2021).to(cuda).eval(), bds, batch_size=4, num_workers=2)
    assert set(bplain) == {"samples", "forecast"}


def test_clis_plan_safety_write_the_json(cuda, recording, tmp_path):
    import yaml
    from lav_b200 import evaluate as EV
    from lav_b200 import evaluate_bev as EB
    lid, uni = seeded_models()
    torch.save(lid.state_dict(), tmp_path / "lidar_1.th")
    torch.save(uni.state_dict(), tmp_path / "uniplanner_1.th")
    torch.save(_planner(2021).state_dict(), tmp_path / "bev_1.th")
    cfg = yaml.safe_load(open(recording[0]))
    cfg["data_dir"] = "/nonexistent"
    yaml.safe_dump(cfg, open(tmp_path / "c.yaml", "w"))
    common = ["--config-path", str(tmp_path / "c.yaml"), "--data-dir", cfg_dir(recording), "--batch-size", "5", "--num-workers", "2",
              "--plan-safety"]
    r = EV.main(common + ["--lidar-weights", str(tmp_path / "lidar_1.th"), "--uniplanner-weights", str(tmp_path / "uniplanner_1.th"),
                          "--json", str(tmp_path / "out.json")])
    got = json.load(open(tmp_path / "out.json"))
    assert got == json.loads(json.dumps(r)) and set(got["plan_safety"]) == {"plan", "expert"}
    assert got["plan_safety"]["expert"]["samples"] == got["samples"] and len(got["plan_safety"]["plan"]["collision_rate_by_step"]) == 20
    rb = EB.main(common + ["--bev-weights", str(tmp_path / "bev_1.th"), "--json", str(tmp_path / "bev.json")])
    gotb = json.load(open(tmp_path / "bev.json"))
    assert gotb == json.loads(json.dumps(rb)) and gotb["plan_safety"]["expert"] == got["plan_safety"]["expert"]
