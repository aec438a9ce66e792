"""CPU: the numpy statement of the forecast scores (per-row errors in sequential fp64 sums, branch selections with their tie and NaN
rules, the host reduction over a recording) on hand-built cases with known answers, ForecastScores against it, and the forecast
rows and targets of heads.recorded_rows against a hand-built label batch and against the training forward at zero jitter."""
import math

import numpy as np
import torch

MISS_M = 2.0


# ---------------------------------------------------------------------------------------------------- the numpy statement
def forecast_eval_ref(cast, score, target, cmd):
    """every output of ops.forecast_eval, as forecast_views names them: err (k,6) fp64, branch (k,2) int32."""
    cast, score = np.asarray(cast, np.float32), np.asarray(score, np.float32)
    target, cmd = np.asarray(target, np.float32), np.asarray(cmd, np.int64)
    k, c, t, _ = cast.shape
    dx = cast[..., 0].astype(np.float64) - target[:, None, :, 0].astype(np.float64)
    dy = cast[..., 1].astype(np.float64) - target[:, None, :, 1].astype(np.float64)
    d = np.sqrt(dx * dx + dy * dy)                                          # (k, c, t); numpy never contracts
    s = np.zeros((k, c))
    for i in range(t):                                                     # ascending steps
        s = s + d[..., i]
    ade, fde = s / t, d[..., t - 1]
    err = np.full((k, 6), np.nan)
    branch = np.zeros((k, 2), np.int32)
    for r in range(k):
        a_best, f_best, s_best, arg, top = ade[r, 0], fde[r, 0], score[r, 0], 0, 0
        for j in range(1, c):                                              # a NaN never wins; the first of equals stays
            if ade[r, j] < a_best or (math.isnan(a_best) and not math.isnan(ade[r, j])):
                a_best, arg = ade[r, j], j
            if fde[r, j] < f_best or (math.isnan(f_best) and not math.isnan(fde[r, j])):
                f_best = fde[r, j]
            if score[r, j] > s_best or (math.isnan(s_best) and not math.isnan(score[r, j])):
                s_best, top = score[r, j], j
        err[r, :4] = a_best, f_best, ade[r, top], fde[r, top]
        if 0 <= cmd[r] < c:
            err[r, 4:] = ade[r, cmd[r]], fde[r, cmd[r]]
        branch[r] = arg, top
    return dict(err=err, branch=branch)


def reduce_ref(batches, plan=False):
    """the host reduction over a recording of [(err, branch, n_other, cmds)] (each batch: the vehicle rows, the B ego casts, then
    with ``plan`` the B ego plans) -> ForecastScores.summary()'s dict."""
    other = [e[:n] for e, _, n, _ in batches]
    ego = [e[n:n + len(c)] for e, _, n, c in batches]
    top = [b[n:n + len(c), 1] for _, b, n, c in batches]
    cmd = np.concatenate([np.asarray(c, np.int64) for *_, c in batches])
    o, e, top = np.concatenate(other), np.concatenate(ego), np.concatenate(top)

    def mean(a):
        return float(np.mean(a)) if len(a) else None

    def ego_stats(m):
        return dict(samples=int(m.sum()), ade=mean(e[m, 4]), fde=mean(e[m, 5]), min_ade=mean(e[m, 0]), min_fde=mean(e[m, 1]),
                    cmd_accuracy=mean(top[m] == cmd[m]))
    everything = np.ones(len(cmd), bool)
    r = dict(other=dict(rows=len(o), min_ade=mean(o[:, 0]), min_fde=mean(o[:, 1]), top_ade=mean(o[:, 2]), top_fde=mean(o[:, 3]),
                        miss_rate=mean(o[:, 1] > MISS_M)),
             ego_cast=dict(ego_stats(everything), per_cmd={str(c): ego_stats(cmd == c) for c in sorted(set(cmd.tolist()))}))
    if plan:
        p = np.concatenate([e[n + len(c):n + 2 * len(c)] for e, _, n, c in batches])
        stats = lambda m: dict(samples=int(m.sum()), ade=mean(p[m, 4]), fde=mean(p[m, 5]))
        r["ego_plan"] = dict(stats(everything), per_cmd={str(c): stats(cmd == c) for c in sorted(set(cmd.tolist()))})
    return r


def random_rows(k, c, t, seed):
    """seeded cast, score, target, cmd of k rows: offsets of a few metres, repeated branches (ties in ADE), rounded scores (ties),
    NaN scores, and commands -1 / in range."""
    rs = np.random.RandomState(seed)
    target = np.cumsum(rs.randn(k, t, 2), 1).astype(np.float32)
    cast = (target[:, None] + rs.randn(k, c, t, 2) * rs.uniform(0.1, 3, (k, c, 1, 1))).astype(np.float32)
    if c > 2:
        cast[::3, 2] = cast[::3, 0]                                        # equal ADE and FDE in branches 0 and 2
    score = np.round(rs.rand(k, c), 1).astype(np.float32)
    score[::5, rs.randint(c)] = np.nan
    score[::7] = np.nan
    cmd = np.where(rs.rand(k) < 0.5, -1, rs.randint(0, c, k)).astype(np.int32)
    return cast, score, target, cmd


# ---------------------------------------------------------------------------------------------------- hand-built cases
def test_exact_forecast_gives_zeros_and_constant_offset_gives_one():
    rs = np.random.RandomState(0)
    target = rs.randn(3, 10, 2).astype(np.float32)
    cast = np.repeat(target[:, None], 6, 1)
    r = forecast_eval_ref(cast, np.full((3, 6), 0.5, np.float32), target, np.array([0, 5, 3]))
    assert (r["err"] == 0).all() and (r["branch"] == 0).all()
    target_i = np.zeros((3, 10, 2), np.float32)                           # integer coordinates: a 1 m offset is exactly 1
    cast_i = np.repeat(target_i[:, None], 6, 1) + np.array([1.0, 0.0], np.float32)
    cast_i[1, 4] = 0
    r = forecast_eval_ref(cast_i, np.zeros((3, 6), np.float32), target_i, np.array([-1, 4, 2]))
    assert r["err"][0, :4].tolist() == [1.0, 1.0, 1.0, 1.0] and np.isnan(r["err"][0, 4:]).all()
    assert r["err"][1].tolist() == [0.0, 0.0, 1.0, 1.0, 0.0, 0.0] and r["branch"][1].tolist() == [4, 0]
    assert r["err"][2, 4:].tolist() == [1.0, 1.0]


def test_ties_go_to_the_lower_branch_and_nan_scores_count_lowest():
    t = np.zeros((1, 4, 2), np.float32)
    cast = np.zeros((1, 3, 4, 2), np.float32)
    cast[0, 0, :, 0] = 2.0
    cast[0, 1, :, 0] = 1.0                                                 # branches 1 and 2 tie in ADE
    cast[0, 2, :, 0] = 1.0
    r = forecast_eval_ref(cast, np.array([[0.3, 0.7, 0.7]], np.float32), t, [1])
    assert r["branch"][0].tolist() == [1, 1]
    r = forecast_eval_ref(cast, np.array([[np.nan, 0.1, np.nan]], np.float32), t, [-1])
    assert r["branch"][0, 1] == 1 and r["err"][0, 2] == 1.0
    r = forecast_eval_ref(cast, np.full((1, 3), np.nan, np.float32), t, [-1])
    assert r["branch"][0, 1] == 0 and r["err"][0, 2] == 2.0                # every score NaN: branch 0
    # minADE and minFDE are taken independently: branch 0 is worse on average but ends on the target
    cast[0, 0, -1] = 0.0
    r = forecast_eval_ref(cast, np.zeros((1, 3), np.float32), t, [0])
    assert r["branch"][0, 0] == 1 and r["err"][0, 0] == 1.0 and r["err"][0, 1] == 0.0 and r["err"][0, 5] == 0.0


def test_sums_are_sequential_in_fp64():
    cast, score, target, cmd = random_rows(50, 6, 20, 1)
    r = forecast_eval_ref(cast, score, target, cmd)
    j = 3
    for row in range(50):
        s = 0.0
        for i in range(20):
            dx = float(cast[row, j, i, 0]) - float(target[row, i, 0])
            dy = float(cast[row, j, i, 1]) - float(target[row, i, 1])
            s += math.sqrt(dx * dx + dy * dy)
        if cmd[row] == j:
            assert r["err"][row, 4] == s / 20


def test_empty_batch_and_miss_threshold():
    from lav_b200.evaluate import FORECAST_MISS_M, ForecastScores
    assert FORECAST_MISS_M == MISS_M
    r = forecast_eval_ref(np.zeros((0, 6, 10, 2)), np.zeros((0, 6)), np.zeros((0, 10, 2)), np.zeros(0))
    assert r["err"].shape == (0, 6) and r["branch"].shape == (0, 2)
    # three vehicle rows ending at exactly 2 m, just over it and below it; one ego row
    t = np.zeros((4, 1, 2), np.float32)
    cast = np.zeros((4, 2, 1, 2), np.float32)
    cast[0, :, 0, 0] = 2.0
    cast[1, :, 0, 0] = np.nextafter(np.float32(2.0), np.float32(3.0))
    cast[2, :, 0, 0] = 1.5
    got = forecast_eval_ref(cast, np.zeros((4, 2), np.float32), t, [-1, -1, -1, 1])
    fs = ForecastScores()
    fs.add(dict(err=torch.from_numpy(got["err"]), branch=torch.from_numpy(got["branch"])), 3, [1])
    s = fs.summary()
    assert s["other"]["rows"] == 3 and s["other"]["miss_rate"] == 1 / 3
    assert s == reduce_ref([(got["err"], got["branch"], 3, [1])])
    fs = ForecastScores(plan=True)                                          # no batch at all
    assert fs.summary()["other"] == dict(rows=0, min_ade=None, min_fde=None, top_ade=None, top_fde=None, miss_rate=None)


def test_host_reduction_equals_the_statement():
    from lav_b200.evaluate import ForecastScores
    rs = np.random.RandomState(4)
    for plan in (False, True):
        fs, batches = ForecastScores(plan=plan), []
        for b, n_other in ((4, 7), (3, 0), (2, 5)):
            cmds = rs.randint(0, 6, b)
            rows = n_other + b * (2 if plan else 1)
            cast, score, target, _ = random_rows(rows, 6, 10, rs.randint(1000))
            cmd = np.concatenate([np.full(n_other, -1), cmds] + ([cmds] if plan else []))
            got = forecast_eval_ref(cast, score, target, cmd)
            fs.add(dict(err=torch.from_numpy(got["err"]), branch=torch.from_numpy(got["branch"])), n_other, cmds)
            batches.append((got["err"], got["branch"], n_other, cmds))
        assert fs.summary() == reduce_ref(batches, plan)
        assert ("ego_plan" in fs.summary()) == plan


# ---------------------------------------------------------------------------------------------------- rows and targets
def label_batch():
    """B = 3 samples of 9 slots (slot 0 the ego): sample 0 holds 7 vehicles ahead (more than max_num_cars), a pedestrian ahead,
    nothing padded; sample 1 vehicles ahead and behind, a pedestrian, padded slots (typ 0 at the origin); sample 2 at most
    max_num_cars = 5 vehicles ahead."""
    g = torch.Generator().manual_seed(7)
    B, N, T = 3, 9, 11
    ego = torch.cumsum(torch.rand(B, T, 2, generator=g) * torch.tensor([0.2, -1.0]), 1)
    locs = torch.randn(B, N, T, 2, generator=g) * torch.tensor([4.0, 3.0]) + torch.tensor([0.0, -10.0])
    locs[:, 0] = ego
    oris = torch.rand(B, N, generator=g) * 0.6 - 0.3
    typs = torch.ones(B, N, dtype=torch.int32)
    typs[0, 5] = 0                                                          # a pedestrian ahead
    locs[1, 2, :, 1] = locs[1, 2, :, 1].abs() + 1.0                         # behind the ego
    locs[1, 4, :, 1] = locs[1, 4, :, 1].abs() + 1.0
    typs[1, 3] = 0
    typs[1, 6:] = 0                                                         # padding
    locs[1, 6:] = 0
    oris[1, 6:] = 0
    locs[2, 6:, :, 1] = locs[2, 6:, :, 1].abs() + 1.0                       # 5 vehicles ahead, 3 behind
    return ego, locs, oris, typs


def test_recorded_rows_select_every_vehicle_ahead():
    from lav_b200.heads import recorded_rows, transform_points
    ego, locs, oris, typs = label_batch()
    rows = recorded_rows(ego, locs, oris, typs)
    got = list(zip(rows["frame"].tolist(), rows["slot"].tolist()))
    want = [(0, s) for s in (1, 2, 3, 4, 6, 7, 8)] + [(1, 1), (1, 5)] + [(2, s) for s in range(1, 6)]
    assert got == want
    for k, (f, s) in enumerate(got):
        heading = oris[f, s] - oris[f, 0]
        assert torch.equal(rows["start"][k], locs[f, s, 0] - ego[f, 0]) and torch.equal(rows["heading"][k], heading)
        # one row at a time, through the same batched product (a 2-D matmul may round differently)
        assert torch.equal(rows["target"][k], transform_points((locs[f, s, 1:] - locs[f, s, :1])[None], -heading[None])[0])


def test_rows_and_targets_equal_the_training_forward_at_zero_jitter():
    """with at most max_num_cars vehicles ahead in every sample, BEVPlanner.forward keeps every row: its other_locs at zero jitter
    are the recorded_rows targets, and forecast_recorded returns those rows."""
    from lav_b200.heads import BEVPlanner, recorded_rows
    ego, locs, oris, typs = label_batch()
    ego, locs, oris, typs = ego[1:], locs[1:], oris[1:], typs[1:]
    torch.manual_seed(0)
    m = BEVPlanner(pixels_per_meter=4, crop_size=32, feature_x_jitter=0, feature_angle_jitter=0, num_plan=10,
                   num_frame_stack=2).eval()
    bev = (torch.rand(2, 9, 320, 320) > 0.7).to(torch.uint8)
    nxps = torch.tensor([[0.0, -20.0], [1.0, -15.0]])
    with torch.no_grad():
        other_locs = m(bev, ego, locs, oris, nxps, typs)[0]
    rows = recorded_rows(ego, locs, oris, typs)
    assert rows["target"].shape == other_locs.shape == (7, 10, 2)
    assert np.array_equal(rows["target"].numpy(), other_locs.numpy())
    fc = m.forecast_recorded(bev, ego, locs, oris, typs, nxps)
    assert torch.equal(fc["frame"], rows["frame"]) and torch.equal(fc["slot"], rows["slot"])
    assert torch.equal(fc["target"], rows["target"]) and torch.equal(fc["ego_target"], ego[:, 1:])
    assert fc["cast"].shape == (7, 6, 10, 2) and fc["score"].shape == (7, 6) and fc["ego_cast"].shape == (2, 6, 10, 2)
    assert fc["ego_plan"].shape == (2, 6, 10, 2)
