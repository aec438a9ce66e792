"""Measurements of the forecast scores (DESIGN §4): forecast_eval_kernel time per batch, lav_b200.evaluate samples/s with and
without --forecast, and lav_b200.evaluate_bev samples/s against its loader alone, on a synthetic recording of realistic size.

    python scripts/forecast_measure.py --out-dir OUT [--batch 32] [--bev-batch 64] [--num-workers 16] [--detected]

Seeded models (bench.build_models, a seeded BEVPlanner), a seeded recording in a temporary directory (30 000-point sweeps); the
GPU's name, power limit and clocks are read in the same run.  Each rate is a list over alternating rounds (the two evaluate
variants alternate).  Results go to OUT/forecast_measure.json.

With --detected it measures the forecasts on detected vehicles instead: the det_forecast_match + forecast_eval launches of one
batch at 32 and 256 samples, and lav_b200.evaluate samples/s with and without --forecast-detected, alternating; results go to
OUT/forecast_detected_measure.json.
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import yaml  # noqa: E402

from eval_measure import gpu_info  # noqa: E402


def kernel_ms(sizes, t, rounds, reps, dev):
    """median over ``rounds`` of the per-launch time of ``reps`` launches, the sizes alternating round by round."""
    from lav_b200 import ops
    from tests.test_forecast_eval_cpu import random_rows
    args = {k: [torch.from_numpy(a).to(dev) for a in random_rows(k, 6, t, k)] for k in sizes}
    outs = {k: ops.forecast_eval(*args[k]) for k in sizes}
    times = {k: [] for k in sizes}
    for _ in range(rounds):
        for k in sizes:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                ops.forecast_eval(*args[k], out=outs[k])
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) / reps)
    return {str(k): dict(rows=k, steps=t, branches=6, ms_median=float(np.median(v)), ms_min=float(min(v)), ms_max=float(max(v)))
            for k, v in times.items()}


def detected_kernel_ms(sizes, t, rounds, reps, dev):
    """median over ``rounds`` of the time of one batch's det_forecast_match + forecast_eval launches (seeded batches of ``sizes``
    samples, 0..15 rows each), repeated ``reps`` times, the sizes alternating round by round."""
    from lav_b200 import ops
    from tests.test_forecast_eval_cpu import random_rows
    from tests.test_gpu_detected_forecast import match_inputs
    args = {}
    for b in sizes:
        packed, actors, offsets, rows, cols, num_objs, locs, ego = match_inputs(b, t, b)
        k = int(rows[-1])
        cast, score, _, _ = random_rows(k, 6, t, b)
        d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        args[b] = (d(packed), d(actors), offsets, rows, cols, num_objs, d(locs), d(ego), d(cast), d(score),
                   torch.full((k,), -1, dtype=torch.int32, device=dev), k)

    def launch(b, out=None):
        packed, actors, offsets, rows, cols, num_objs, locs, ego, cast, score, cmd, k = args[b]
        buf = ops.det_forecast_match(packed, actors, offsets, rows, cols, num_objs, locs, ego, out=out)
        ops.forecast_eval(cast, score, ops.det_match_views(buf, b, k, t)["target"], cmd, out=buf[:56 * k])
        return buf
    outs = {b: launch(b) for b in sizes}
    times = {b: [] for b in sizes}
    for _ in range(rounds):
        for b in sizes:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                launch(b, outs[b])
            e1.record()
            torch.cuda.synchronize()
            times[b].append(e0.elapsed_time(e1) / reps)
    return {str(b): dict(samples=b, rows=args[b][-1], steps=t, ms_median=float(np.median(v)), ms_min=float(min(v)),
                         ms_max=float(max(v))) for b, v in times.items()}


def timed(fn, n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return n / (time.perf_counter() - t0), r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", required=True)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--bev-batch", type=int, default=64)
    ap.add_argument("--num-workers", type=int, default=16)
    ap.add_argument("--frames", type=int, default=61, help="frames per trajectory (4 trajectories; 20 fewer samples each)")
    ap.add_argument("--detected", action="store_true", help="measure the forecasts on detected vehicles instead")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import bench
    from lav_b200 import synth
    from lav_b200.datasets import TemporalBEVBatchLoader, TemporalBEVDataset, TemporalLiDARPaintedDataset
    from lav_b200.evaluate import evaluate
    from lav_b200.evaluate_bev import evaluate_bev
    from lav_b200.train_bev import build_planner
    dev = torch.device("cuda:0")
    res = dict(gpu_before=gpu_info(), batch=args.batch, bev_batch=args.bev_batch, num_workers=args.num_workers)
    if args.detected:
        res["kernel"] = detected_kernel_ms((32, 256), 20, 9, 200, dev)
    else:
        res["kernel"] = kernel_ms((256, 5000), 20, 9, 200, dev)
    tmp = tempfile.mkdtemp(prefix="lavb_forecast_")
    rec = os.path.join(tmp, "recording")
    synth.record_trajectories(rec, 4, args.frames, seed=2021, n_points=30000)
    cfg = dict(num_plan=20, num_frame_stack=2, seg_channels=[4, 6, 7, 10], max_lidar_points=120000, camera_x=1.5, camera_z=2.4,
               camera_yaws=[-120, -60, 0, 60, 120], angle_jitter=20, stack_loc_jitter=0.4, stack_ori_jitter=0.1, x_jitter=10,
               max_pedestrian_radius=10, max_vehicle_radius=25, max_mot_vehicle_radius=15, max_objs=20, min_x=-10, max_x=70,
               min_y=-40, max_y=40, pixels_per_meter=4, percentage_data=1.01, all_towns=True, data_dir=rec, crop_size=96,
               feature_x_jitter=1.5, feature_angle_jitter=20, num_cmds=6, num_plan_iter=5)
    cfg_path = os.path.join(tmp, "config.yaml")
    yaml.safe_dump(cfg, open(cfg_path, "w"))
    ds = TemporalLiDARPaintedDataset(cfg_path, device=dev)
    n = len(ds)
    res["samples"] = n
    (_, lid, uni, _), _ = bench.build_models()
    if args.detected:
        evaluate(lid, uni, ds, args.batch, "f16", args.num_workers, forecast_detected=True)      # warm-up
        for detected in (False, True, False, True):
            rate, r = timed(lambda: evaluate(lid, uni, ds, args.batch, "f16", args.num_workers, forecast_detected=detected), n)
            res.setdefault(f"evaluate_samples_per_s_forecast_detected_{detected}", []).append(rate)
            if detected:
                res["evaluate_forecast_detected"] = r["forecast_detected"]
        return finish(res, tmp, args.out_dir, "forecast_detected_measure.json")
    evaluate(lid, uni, ds, args.batch, "f16", args.num_workers, forecast=True)      # warm-up: plans, cuDNN algorithms, pages
    for forecast in (False, True, False, True):
        rate, r = timed(lambda: evaluate(lid, uni, ds, args.batch, "f16", args.num_workers, forecast=forecast), n)
        res.setdefault(f"evaluate_samples_per_s_forecast_{forecast}", []).append(rate)
        if forecast:
            res["evaluate_forecast"] = r["forecast"]
    bds = TemporalBEVDataset(cfg_path, device=dev)
    torch.manual_seed(2021)
    planner = build_planner(cfg)
    planner.load_state_dict(synth.fill_state_dict_(planner.state_dict(), 2021))
    evaluate_bev(planner, bds, args.bev_batch, args.num_workers)                     # warm-up
    for _ in range(2):
        rate, r = timed(lambda: evaluate_bev(planner, bds, args.bev_batch, args.num_workers), n)
        res.setdefault("evaluate_bev_samples_per_s", []).append(rate)
        res["evaluate_bev_forecast"] = r["forecast"]
        rate, _ = timed(lambda: list(TemporalBEVBatchLoader(bds, args.bev_batch, drop_last=False, num_workers=args.num_workers,
                                                            ordered=True)), n)
        res.setdefault("bev_loader_alone_samples_per_s", []).append(rate)
    finish(res, tmp, args.out_dir, "forecast_measure.json")


def finish(res, tmp, out_dir, name):
    res["gpu_after"] = gpu_info()
    shutil.rmtree(tmp, True)
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, name), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: v for k, v in res.items() if not k.endswith("forecast") and not k.endswith("detected")}))


if __name__ == "__main__":
    main()
