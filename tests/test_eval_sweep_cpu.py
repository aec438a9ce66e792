"""CPU: the evaluators' rank sharding (contiguous, disjoint, covering, the training shard unchanged), the merge of per-rank
accumulators against one stream of the same per-sample results, checkpoint selection for sweeps, the sweep's memory check and
its printout."""
import itertools
import os
import pickle

import numpy as np
import pytest
import torch

from lav_b200 import eval_sweep as S
from lav_b200 import evaluate as E
from lav_b200 import evaluate_bev as EB
from lav_b200.capi import LavbError
from lav_b200.datasets import TemporalBatchLoader, TemporalBEVBatchLoader


class _Sized:
    def __init__(self, n):
        self.n = n

    def __len__(self):
        return self.n


# ---------------------------------------------------------------------------------------------------- shards
@pytest.mark.parametrize("n", [1, 7, 64, 101])
@pytest.mark.parametrize("world", [1, 2, 3, 5])
def test_ordered_shards_are_contiguous_disjoint_and_cover_the_recording(n, world):
    for cls in (TemporalBatchLoader, TemporalBEVBatchLoader):
        shards = [cls(_Sized(n), 4, rank=r, world=world, drop_last=False, ordered=True).shard(0) for r in range(world)]
        for s in shards:
            assert np.array_equal(s, np.arange(s[0], s[0] + len(s))) if len(s) else True
        assert np.array_equal(np.concatenate(shards), np.arange(n))       # disjoint, in rank order, every sample once
        assert max(map(len, shards)) - min(map(len, shards)) <= 1
        lens = [len(cls(_Sized(n), 4, rank=r, world=world, drop_last=False, ordered=True)) for r in range(world)]
        assert lens == [-(-len(s) // 4) for s in shards]                   # the last batch of a rank may be short


@pytest.mark.parametrize("n", [1, 7, 64, 101])
@pytest.mark.parametrize("world", [1, 2, 3, 5])
def test_training_shard_is_unchanged(n, world):
    for r in range(world):
        loader = TemporalBatchLoader(_Sized(n), 2, seed=11, rank=r, world=world)
        for epoch in (0, 3):
            want = np.random.RandomState([11, epoch]).permutation(n)[r::world][:n // world]
            assert np.array_equal(loader.shard(epoch), want)
        assert len(loader) == n // world // 2


# ---------------------------------------------------------------------------------------------------- the merge
N_COLS, T = 30, 20


def per_sample(n, seed):
    """seeded per-sample results of eval_batch, forecast_eval (vehicle rows, ego cast, ego plan), det_match and plan_safety;
    detection scores rounded to one decimal, so ties run across every rank boundary."""
    rs = np.random.RandomState(seed)
    out = []
    for i in range(n):
        k_other, k_det = rs.randint(0, 4), rs.randint(0, 4)
        flags = ((rs.rand(N_COLS) < 0.7) * 16 + rs.randint(0, 16, N_COLS)).astype(np.int32)
        out.append(dict(
            iou=rs.randint(0, 100, (3, 2)), ngt=rs.randint(0, 5, 2).astype(np.int32), score=np.round(rs.rand(N_COLS), 1).astype(np.float32),
            flags=flags, plan_err=rs.rand(2), cmd=int(rs.randint(0, 4)),
            other=rs.rand(k_other, 6), ego=rs.rand(6), ego_plan=rs.rand(6), branch=rs.randint(0, 6, 2).astype(np.int32),
            other_branch=rs.randint(0, 6, (k_other, 2)).astype(np.int32),
            det_score=np.round(rs.rand(k_det), 1).astype(np.float32), det_flag=rs.choice([0, 1, 3, 3], k_det).astype(np.int32),
            det_err=rs.rand(k_det, 6), det_ngt=rs.randint(0, 4, (1, 2)).astype(np.int32),
            safety=rs.randint(-1, T + 1, (2, 8)).astype(np.int32)))
    return out


def add_batch(acc, samples):
    """one batch of ``samples`` into evaluate's accumulator tuple, as score_batch adds the views of its launches."""
    scores, forecasts, detected, safety = acc
    cat = lambda k: torch.from_numpy(np.stack([s[k] for s in samples]))
    cmds = np.array([s["cmd"] for s in samples])
    scores.add(dict(iou=cat("iou"), ngt=cat("ngt"), score=cat("score"), flags=cat("flags"), plan_err=cat("plan_err")), cmds)
    other = np.concatenate([s["other"] for s in samples])
    err = np.concatenate([other, np.stack([s["ego"] for s in samples]), np.stack([s["ego_plan"] for s in samples])])
    branch = np.concatenate([np.concatenate([s["other_branch"] for s in samples]), np.stack([s["branch"] for s in samples]),
                             np.stack([s["branch"] for s in samples])])
    forecasts.add(dict(err=torch.from_numpy(err), branch=torch.from_numpy(branch)), len(other), cmds)
    detected.add(dict(flag=torch.from_numpy(np.concatenate([s["det_flag"] for s in samples])),
                      err=torch.from_numpy(np.concatenate([s["det_err"] for s in samples])),
                      ngt=torch.from_numpy(np.concatenate([s["det_ngt"] for s in samples]))),
                 np.concatenate([s["det_score"] for s in samples]))
    safety.add(np.stack([s["safety"] for s in samples]), cmds)


def accumulate(samples, batch, plan=False):
    acc = (E.Scores(), E.ForecastScores(plan), E.DetectedForecastScores(), E.PlanSafetyScores())
    for k in range(0, len(samples), batch):
        add_batch(acc, samples[k:k + batch])
    return acc


def splits(n, world, rs):
    """uneven contiguous cuts of range(n) into ``world`` ranks (some possibly empty)."""
    cuts = np.sort(rs.randint(0, n + 1, world - 1))
    return [(a, b) for a, b in zip(np.concatenate([[0], cuts]), np.concatenate([cuts, [n]]))]


@pytest.mark.parametrize("world", [1, 2, 3, 4, 5])
def test_ranks_merge_to_the_single_stream_summary(world):
    n, rs = 37, np.random.RandomState(world)
    samples = per_sample(n, 7)
    flat_scores = np.concatenate([s["score"] for s in samples])
    assert len(set(flat_scores.tolist())) < len(flat_scores)                # tied scores throughout
    for cut in (splits(n, world, rs), [(r * n // world, (r + 1) * n // world) for r in range(world)]):
        for plan in (False, True):
            one = accumulate(samples, 4, plan)
            # each rank batches its own range (a short last batch of its own) and its accumulators travel pickled, as
            # gather_object sends them
            parts = [pickle.loads(pickle.dumps([accumulate(samples[a:b], 3, plan)])) for a, b in cut]
            merged = S.merge_ranks(parts)[0]
            for flags in itertools.product([False, True], repeat=3):
                assert E.summarize(merged, "f16", *flags, T) == E.summarize(one, "f16", *flags, T)
            for ps in (False, True):
                assert EB.summarize((merged[1], merged[3]), n, ps, T) == EB.summarize((one[1], one[3]), n, ps, T)


def test_merge_refuses_mismatched_structures():
    with pytest.raises(LavbError):
        S.merge_ranks([[E.Scores()], [E.Scores(), E.Scores()]])
    assert S.gather_merged([1, 2]) == [1, 2]                                # no process group: the accumulators themselves


# ---------------------------------------------------------------------------------------------------- checkpoint selection
def touch(d, *names):
    for n in names:
        open(os.path.join(d, n), "wb").close()


def test_run_dir_pairs_sorted_by_epoch_and_epoch_ranges(tmp_path):
    d = str(tmp_path)
    touch(d, *[f"{n}_{e}.th" for e in (1, 2, 8, 16, 17, 64) for n in ("lidar", "uniplanner")], "bev_3.th", "lidar_x.th", "notes.txt")
    got = S.find_checkpoints(d, ("lidar", "uniplanner"))
    assert [e for e, _ in got] == [1, 2, 8, 16, 17, 64]
    assert got[2][1] == dict(lidar=os.path.join(d, "lidar_8.th"), uniplanner=os.path.join(d, "uniplanner_8.th"))
    assert S.parse_epochs("1,8,16-64") == [1, 8] + list(range(16, 65))
    assert S.parse_epochs("17, 2,2-2") == [2, 17]
    assert [e for e, _ in S.find_checkpoints(d, ("lidar", "uniplanner"), [2, 16, 17])] == [2, 16, 17]
    assert [e for e, _ in S.find_checkpoints(d, ("bev",))] == [3]
    for bad in ("", "1-", "a", "5-3"):
        with pytest.raises(LavbError):
            S.parse_epochs(bad)
    with pytest.raises(LavbError, match="lidar_9.th"):                   # an epoch of the selection with no file
        S.find_checkpoints(d, ("lidar", "uniplanner"), S.parse_epochs("8-9"))


def test_missing_partner_and_empty_selection_are_refused(tmp_path):
    d = str(tmp_path)
    touch(d, "lidar_1.th", "uniplanner_1.th", "lidar_2.th", "uniplanner_3.th")
    with pytest.raises(LavbError, match="uniplanner_2.th"):
        S.find_checkpoints(d, ("lidar", "uniplanner"))
    with pytest.raises(LavbError, match="lidar_3.th"):
        S.find_checkpoints(d, ("lidar", "uniplanner"), [3])
    assert [e for e, _ in S.find_checkpoints(d, ("lidar", "uniplanner"), [1])] == [1]
    with pytest.raises(LavbError, match="bev_"):
        S.find_checkpoints(d, ("bev",))
    with pytest.raises(LavbError, match="not a directory"):
        S.find_checkpoints(os.path.join(d, "nowhere"), ("bev",))


def test_weight_lists_pair_by_position_and_unequal_counts_are_refused(tmp_path):
    assert S.pair_paths(dict(lidar=["a", "b"], uniplanner=["c", "d"])) == [(None, dict(lidar="a", uniplanner="c")),
                                                                           (None, dict(lidar="b", uniplanner="d"))]
    with pytest.raises(LavbError, match="lidar_3.th"):
        S.pair_paths(dict(lidar=["lidar_1.th", "lidar_3.th"], uniplanner=["uniplanner_1.th"]))
    common = ["--data-dir", str(tmp_path), "--config-path", str(tmp_path / "absent.yaml")]
    with pytest.raises(LavbError, match="uniplanner_2.th"):              # refused before the config or a device is touched
        E.main(common + ["--lidar-weights", "lidar_1.th", "--uniplanner-weights", "uniplanner_1.th", "uniplanner_2.th"])
    with pytest.raises(LavbError, match="--uniplanner-weights"):
        E.main(common + ["--lidar-weights", "lidar_1.th"])
    with pytest.raises(LavbError, match="not both"):
        E.main(common + ["--lidar-weights", "l.th", "--uniplanner-weights", "u.th", "--run-dir", str(tmp_path)])
    with pytest.raises(LavbError, match="bev_"):
        EB.main(common + ["--run-dir", str(tmp_path)])
    args = E.parse_args(common + ["--lidar-weights", "l.th", "--uniplanner-weights", "u.th"])
    assert S.select_checkpoints(args, ("lidar", "uniplanner")) == [(None, dict(lidar="l.th", uniplanner="u.th"))]


# ---------------------------------------------------------------------------------------------------- memory and printout
def test_sweep_capacity_and_refusal():
    gib, mib = 2 ** 30, 2 ** 20
    assert S.sweep_capacity(100 * mib, 10 * gib, 2 * gib) == 81
    assert S.sweep_capacity(100 * mib, gib, 2 * gib) == 0
    ws = S.EVAL_WORKSPACE_BYTES_PER_SAMPLE * 32
    cap = S.check_sweep_fits(16, gib, 20 * gib + ws, 32)
    assert cap == 20
    with pytest.raises(LavbError, match="at most 20 fit"):
        S.check_sweep_fits(21, gib, 20 * gib + ws, 32)
    S.check_sweep_fits(1, 100 * gib, gib, 32)                             # one checkpoint is never refused


def fake_result(seed, extra=True):
    samples = per_sample(9, seed)
    acc = accumulate(samples, 4)
    return E.summarize(acc, "f16", extra, extra, extra, T)


def test_one_checkpoint_prints_as_a_single_run_and_a_sweep_prints_a_table():
    r = fake_result(1)
    ck = [(None, dict(lidar="l.th", uniplanner="u.th"))]
    assert E.report(ck, [r], 1) == (E.format_result(r), r)
    rs = [fake_result(s) for s in (1, 2, 3)]
    ck = [(e, dict(lidar=f"lidar_{e}.th", uniplanner=f"uniplanner_{e}.th")) for e in (1, 8, 16)]
    text, doc = E.report(ck, rs, 2)
    lines = text.splitlines()
    assert lines[0].startswith("9 samples, precision f16, 3 checkpoints, 2 rank(s)")
    assert len(lines) == 5 and all(f"epoch {e}" in lines[2 + i] for i, e in enumerate((1, 8, 16)))
    for col in ("IoU0", "ped mAP", "veh mAP", "ADE", "FDE", "fc minADE", "det fc AP", "collision", "off-road"):
        assert col in lines[1]
    assert doc == dict(samples=9, ranks=2, checkpoints=[dict(epoch=e, weights=w, result=r) for (e, w), r in zip(ck, rs)])
    plain = E.report(ck, [fake_result(s, extra=False) for s in (1, 2, 3)], 1)[0]
    assert "fc minADE" not in plain and "collision" not in plain
    by_path = E.report([(None, dict(lidar="a/l.th", uniplanner="u.th"))] * 2, rs[:2], 1)[0]
    assert by_path.splitlines()[2].startswith("a/l.th")


def test_bev_report_keeps_the_single_run_printout():
    acc = accumulate(per_sample(9, 4), 4, plan=True)
    r = EB.summarize((acc[1], acc[3]), 9, True, T)
    assert EB.report([(None, dict(bev="b.th"))], [r], 1) == (EB.format_result(r), r)
    text, doc = EB.report([(3, dict(bev="bev_3.th")), (5, dict(bev="bev_5.th"))], [r, r], 1)
    assert "plan ADE" in text.splitlines()[1] and doc["checkpoints"][1]["epoch"] == 5
