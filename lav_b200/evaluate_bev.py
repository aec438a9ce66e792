"""Score a privileged BEV planner checkpoint (train_bev's bev_{epoch}.th) on a held-out recording: its motion forecasts of the
recorded vehicles and of the ego, its command scores and its ego plan, under the protocol of lav_b200.evaluate --forecast.

    python -m lav_b200.evaluate_bev --config-path config_v2.yaml --data-dir VALDIR --bev-weights bev_7.th [--batch-size 64] \
        [--num-workers 16] [--json out.json] [--plan-safety] [--driving-score [--step-seconds 0.25]]
    python -m lav_b200.evaluate_bev ... --bev-weights bev_40.th bev_80.th bev_160.th
    python -m lav_b200.evaluate_bev ... --run-dir RUN [--epochs 40-160]
    torchrun --nproc-per-node N -m lav_b200.evaluate_bev ...

Every sample is taken once, in index order, unaugmented (TemporalBEVBatchLoader's ordered mode); the last batch may be short.
Per batch, BEVPlanner.forecast_recorded runs the planner in fp32 on crops of the ground-truth BEV at the recorded poses and one
ops.forecast_eval launch scores the vehicle rows, the ego casts and the ego plans; the one device-to-host copy is that launch's
result buffer.  The result is dict(samples, forecast) with ``forecast`` as ForecastScores.summary(plan=True) gives it; a student
UniPlanner scored by lav_b200.evaluate --forecast on the same recording is comparable row for row.  With --plan-safety the result
also holds ``plan_safety``: the recorded command's branch of the ego plan and the expert, checked against the recorded traffic and
the road plane by one ops.plan_safety launch per batch, under lav_b200.evaluate's plan-safety protocol.  With --driving-score it
holds ``driving_score``: the same two trajectories scored by one ops.driving_score launch per batch, under lav_b200.evaluate's
driving-score protocol.

Sweeps of several planners (paths, or train_bev's bev_{e}.th found by --run-dir) and torchrun ranks work as in
lav_b200.evaluate (lav_b200.eval_sweep): each batch is loaded once for every planner, and rank 0 merges the ranks' records.
"""
import argparse
import json

import torch

from . import ops
from .agent import math_mode
from .datasets import TemporalBEVBatchLoader, TemporalBEVDataset, stage_plan_safety
from .eval_sweep import (ResidentMeter, add_checkpoint_args, check_sweep_fits, eval_device, gather_merged, init_ranks,
                         rank_and_world, select_checkpoints, sweep_json, sweep_table)
from .evaluate import (DrivingScores, ForecastScores, PlanSafetyScores, add_driving_score_args, format_driving_score, format_forecast,
                       format_plan_safety, score_driving, score_forecasts, score_plan_safety)


def recorded_branch(ego_plan, cmds):
    """the (B,T,2) branch of the recorded command of a (B,C,T,2) ego plan, the one score_forecasts(..., plan=True) scores; NaN
    where the command is outside [0, C) (forecast_eval scores no branch there)."""
    c = ego_plan.shape[1]
    ok = (cmds >= 0) & (cmds < c)
    picked = ego_plan[torch.arange(len(cmds), device=ego_plan.device), cmds.clamp(0, c - 1)].float()
    return torch.where(ok[:, None, None], picked, torch.full_like(picked, float("nan")))


def evaluate_bev(bev_planner, dataset, batch_size=64, num_workers=16, plan_safety=False, driving_score=False,
                 step_seconds=ops.DRIVING_SCORE_STEP_S):
    """Forecast scores of ``bev_planner`` over every sample of ``dataset`` (a TemporalBEVDataset); with ``plan_safety`` also the
    collision and off-road rates of its ego plan and of the expert, with ``driving_score`` their driving score at a step period
    of ``step_seconds``.  -> dict(samples, forecast[, plan_safety][, driving_score]); None on a rank other than 0 of a process
    group."""
    results = evaluate_bev_checkpoints([bev_planner], dataset, batch_size, num_workers, plan_safety, driving_score, step_seconds)
    return None if results is None else results[0]


@torch.no_grad()
def evaluate_bev_checkpoints(planners, dataset, batch_size=64, num_workers=16, plan_safety=False, driving_score=False,
                             step_seconds=ops.DRIVING_SCORE_STEP_S):
    """evaluate_bev() of every BEVPlanner of ``planners`` in one pass over ``dataset``: each batch is loaded once, then every
    planner runs forecast_recorded and its scoring launches on it into its own accumulators.  All planners stay resident; a
    sweep that would not fit on the device is refused before any data is loaded.  In a process group each rank scores its
    contiguous shard and rank 0 merges the records (eval_sweep.gather_merged).  -> one result per planner on rank 0, None on
    the other ranks."""
    dev = dataset.device
    rank, world = rank_and_world()
    for i, planner in enumerate(planners):
        meter = ResidentMeter(dev, planner) if i == 0 and len(planners) > 1 else None
        planner.to(dev).eval()
        if meter is not None:
            check_sweep_fits(len(planners), meter.resident(), meter.available, batch_size, "BEV planners")
    loader = TemporalBEVBatchLoader(dataset, batch_size, rank=rank, world=world, drop_last=False, num_workers=num_workers,
                                    ordered=True, plan_safety=plan_safety, driving_score=driving_score)
    accs = [(ForecastScores(plan=True), PlanSafetyScores(), DrivingScores(dt=step_seconds)) for _ in planners]
    grid = dict(min_x=dataset.min_x, max_x=dataset.max_x, min_y=dataset.min_y, max_y=dataset.max_y,
                pixels_per_meter=dataset.pixels_per_meter)
    with math_mode("fp32"):
        for (bev, ego_locs, cmds, nxps, _, locs, oris, typs, _), hs in loader.staged_batches():
            host_cmds = [h["cmd"] for h in hs]
            table = stage_plan_safety([h["plan_safety"] for h in hs], dev.type == "cuda") if plan_safety else None
            driving = stage_plan_safety([h["driving_score"] for h in hs], dev.type == "cuda") if driving_score else None
            for planner, (scores, safety, drive) in zip(planners, accs):
                fc = planner.forecast_recorded(bev, ego_locs, locs, oris, typs, nxps)
                k, b = fc["cast"].shape[0], len(hs)
                scores.add(ops.forecast_views(score_forecasts(fc, cmds, plan=True).cpu(), k + 2 * b), k, host_cmds)
                if plan_safety:
                    res = score_plan_safety(recorded_branch(fc["ego_plan"], cmds), ego_locs, table, bev, grid)
                    safety.add(res.cpu().numpy(), host_cmds)
                if driving_score:
                    res = score_driving(recorded_branch(fc["ego_plan"], cmds), ego_locs, driving, bev, grid, step_seconds)
                    drive.add(res.cpu(), host_cmds)
    accs = gather_merged(accs)
    if accs is None:
        return None
    return [summarize(acc, len(dataset), plan_safety, dataset.num_plan, driving_score) for acc in accs]


def summarize(acc, samples, plan_safety, num_plan, driving_score=False):
    """the evaluate_bev() result of one planner's accumulators ``acc`` = (ForecastScores, PlanSafetyScores[, DrivingScores]); the
    DrivingScores is read only with ``driving_score``."""
    scores, safety = acc[:2]
    result = dict(samples=samples, forecast=scores.summary())
    if plan_safety:
        result["plan_safety"] = safety.summary(num_plan)
    if driving_score:
        result["driving_score"] = acc[2].summary()
    return result


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--config-path", default="config_v2.yaml")
    ap.add_argument("--data-dir", required=True, help="the held-out recording (replaces the YAML's data_dir)")
    add_checkpoint_args(ap, ("bev",), dict(bev="a BEVPlanner state_dict (train_bev's bev_{epoch}.th)"))
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--num-workers", type=int, default=16, help="host threads of the loader (record reads, PNG chunk walks)")
    ap.add_argument("--json", default=None, help="also write the result here")
    ap.add_argument("--plan-safety", action="store_true",
                    help="also score the ego plan and the expert for collisions with the recorded traffic and for leaving the road")
    add_driving_score_args(ap)
    return ap.parse_args(argv)


def format_result(r):
    return "\n".join([f"{r['samples']} samples"] + format_forecast(r["forecast"]) +
                     (format_plan_safety(r["plan_safety"]) if "plan_safety" in r else []) +
                     (format_driving_score(r["driving_score"]) if "driving_score" in r else []))


def headline(r):
    """the (column, value) pairs of a result in a sweep's table."""
    f = r["forecast"]
    cols = [("fc minADE", f["other"]["min_ade"]), ("fc minFDE", f["other"]["min_fde"]), ("ego minADE", f["ego_cast"]["min_ade"]),
            ("cmd acc", f["ego_cast"]["cmd_accuracy"]), ("plan ADE", f["ego_plan"]["ade"]), ("plan FDE", f["ego_plan"]["fde"])]
    if "plan_safety" in r:
        cols += [("collision", r["plan_safety"]["plan"]["collision_rate"]), ("off-road", r["plan_safety"]["plan"]["off_road_rate"])]
    if "driving_score" in r:
        cols.append(("PDMS", r["driving_score"]["plan"]["pdms"]))
    return cols


def report(checkpoints, results, world):
    """(printout, --json document): one checkpoint's as always, a sweep's as a table and sweep_json."""
    if len(results) == 1:
        return format_result(results[0]), results[0]
    text = (f"{results[0]['samples']} samples, {len(results)} checkpoints, {world} rank(s)\n" +
            sweep_table(checkpoints, [headline(r) for r in results]))
    return text, sweep_json(checkpoints, results, results[0]["samples"], world)


def main(argv=None):
    import torch.distributed as dist
    import yaml
    from .train_bev import build_planner
    args = parse_args(argv)
    checkpoints = select_checkpoints(args, ("bev",))
    with open(args.config_path) as f:
        cfg = yaml.safe_load(f)
    own_group = init_ranks()
    dev = eval_device()
    torch.cuda.set_device(dev)
    planners = []
    for _, paths in checkpoints:
        planner = build_planner(cfg)
        planner.load_state_dict(torch.load(paths["bev"], map_location="cpu"))
        planners.append(planner)
    ds = TemporalBEVDataset(args.config_path, device=dev, overrides=dict(data_dir=args.data_dir))
    results = evaluate_bev_checkpoints(planners, ds, args.batch_size, args.num_workers, args.plan_safety, args.driving_score,
                                       args.step_seconds)
    out = None
    if results is not None:
        text, out = report(checkpoints, results, rank_and_world()[1])
        print(text)
        if args.json:
            with open(args.json, "w") as f:
                json.dump(out, f, indent=1)
    if own_group:
        dist.destroy_process_group()
    return out


if __name__ == "__main__":
    main()
