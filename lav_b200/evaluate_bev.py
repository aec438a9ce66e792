"""Score a privileged BEV planner checkpoint (train_bev's bev_{epoch}.th) on a held-out recording: its motion forecasts of the
recorded vehicles and of the ego, its command scores and its ego plan, under the protocol of lav_b200.evaluate --forecast.

    python -m lav_b200.evaluate_bev --config-path config_v2.yaml --data-dir VALDIR --bev-weights bev_7.th [--batch-size 64] \
        [--num-workers 16] [--json out.json] [--plan-safety]

Every sample is taken once, in index order, unaugmented (TemporalBEVBatchLoader's ordered mode); the last batch may be short.
Per batch, BEVPlanner.forecast_recorded runs the planner in fp32 on crops of the ground-truth BEV at the recorded poses and one
ops.forecast_eval launch scores the vehicle rows, the ego casts and the ego plans; the one device-to-host copy is that launch's
result buffer.  The result is dict(samples, forecast) with ``forecast`` as ForecastScores.summary(plan=True) gives it; a student
UniPlanner scored by lav_b200.evaluate --forecast on the same recording is comparable row for row.  With --plan-safety the result
also holds ``plan_safety``: the recorded command's branch of the ego plan and the expert, checked against the recorded traffic and
the road plane by one ops.plan_safety launch per batch, under lav_b200.evaluate's plan-safety protocol.
"""
import argparse
import json

import torch

from . import ops
from .agent import math_mode
from .datasets import TemporalBEVBatchLoader, TemporalBEVDataset, stage_plan_safety
from .evaluate import ForecastScores, PlanSafetyScores, format_forecast, format_plan_safety, score_forecasts, score_plan_safety


def recorded_branch(ego_plan, cmds):
    """the (B,T,2) branch of the recorded command of a (B,C,T,2) ego plan, the one score_forecasts(..., plan=True) scores; NaN
    where the command is outside [0, C) (forecast_eval scores no branch there)."""
    c = ego_plan.shape[1]
    ok = (cmds >= 0) & (cmds < c)
    picked = ego_plan[torch.arange(len(cmds), device=ego_plan.device), cmds.clamp(0, c - 1)].float()
    return torch.where(ok[:, None, None], picked, torch.full_like(picked, float("nan")))


@torch.no_grad()
def evaluate_bev(bev_planner, dataset, batch_size=64, num_workers=16, plan_safety=False):
    """Forecast scores of ``bev_planner`` over every sample of ``dataset`` (a TemporalBEVDataset); with ``plan_safety`` also the
    collision and off-road rates of its ego plan and of the expert.  -> dict(samples, forecast[, plan_safety])."""
    dev = dataset.device
    bev_planner.to(dev).eval()
    loader = TemporalBEVBatchLoader(dataset, batch_size, drop_last=False, num_workers=num_workers, ordered=True,
                                    plan_safety=plan_safety)
    scores, safety = ForecastScores(plan=True), PlanSafetyScores()
    grid = dict(min_x=dataset.min_x, max_x=dataset.max_x, min_y=dataset.min_y, max_y=dataset.max_y,
                pixels_per_meter=dataset.pixels_per_meter)
    with math_mode("fp32"):
        for (bev, ego_locs, cmds, nxps, _, locs, oris, typs, _), hs in loader.staged_batches():
            fc = bev_planner.forecast_recorded(bev, ego_locs, locs, oris, typs, nxps)
            k, b = fc["cast"].shape[0], len(hs)
            host_cmds = [h["cmd"] for h in hs]
            scores.add(ops.forecast_views(score_forecasts(fc, cmds, plan=True).cpu(), k + 2 * b), k, host_cmds)
            if plan_safety:
                table = stage_plan_safety([h["plan_safety"] for h in hs], dev.type == "cuda")
                res = score_plan_safety(recorded_branch(fc["ego_plan"], cmds), ego_locs, table, bev, grid)
                safety.add(res.cpu().numpy(), host_cmds)
    result = dict(samples=len(dataset), forecast=scores.summary())
    if plan_safety:
        result["plan_safety"] = safety.summary(dataset.num_plan)
    return result


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--config-path", default="config_v2.yaml")
    ap.add_argument("--data-dir", required=True, help="the held-out recording (replaces the YAML's data_dir)")
    ap.add_argument("--bev-weights", required=True, help="a BEVPlanner state_dict (train_bev's bev_{epoch}.th)")
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--num-workers", type=int, default=16, help="host threads of the loader (record reads, PNG chunk walks)")
    ap.add_argument("--json", default=None, help="also write the result here")
    ap.add_argument("--plan-safety", action="store_true",
                    help="also score the ego plan and the expert for collisions with the recorded traffic and for leaving the road")
    return ap.parse_args(argv)


def main(argv=None):
    import yaml
    from .train_bev import build_planner
    args = parse_args(argv)
    with open(args.config_path) as f:
        cfg = yaml.safe_load(f)
    dev = torch.device("cuda")
    planner = build_planner(cfg)
    planner.load_state_dict(torch.load(args.bev_weights, map_location="cpu"))
    ds = TemporalBEVDataset(args.config_path, device=dev, overrides=dict(data_dir=args.data_dir))
    result = evaluate_bev(planner, ds, args.batch_size, args.num_workers, args.plan_safety)
    print("\n".join([f"{result['samples']} samples"] + format_forecast(result["forecast"]) +
                    (format_plan_safety(result["plan_safety"]) if "plan_safety" in result else [])))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)
    return result


if __name__ == "__main__":
    main()
