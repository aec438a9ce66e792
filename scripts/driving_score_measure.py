"""Measurements of the driving score (DESIGN §4): the lavb_driving_score time per batch and lav_b200.evaluate samples/s with and
without --driving-score, on a synthetic recording.

    python scripts/driving_score_measure.py --out-dir OUT [--batch 32] [--num-workers 16]

Seeded models (bench.build_models) and a seeded recording in a temporary directory (30 000-point sweeps); the GPU's name, power
limit and clocks are read in the same run.  Kernel times are CUDA-event medians over alternating rounds of seeded batches of 32
and 256 samples with 100 actors x 21 steps each, two trajectories of 20 steps and dt = 0.25 s; the evaluate variants alternate.
Results go to OUT/driving_score_measure.json.
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
    from tests.test_gpu_driving_score import random_inputs
    args = {}
    for b in sizes:
        traj, expert, rec, offsets, ext, bev = random_inputs(b, t, 2, b, actors=100)
        d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        args[b] = (d(traj), d(expert), d(rec.view(np.uint8)), offsets, d(ext), d(bev))
    outs = {b: ops.driving_score(*args[b]) for b in sizes}
    times = {b: [] for b in sizes}
    for _ in range(rounds):
        for b in sizes:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                ops.driving_score(*args[b], out=outs[b])
            e1.record()
            torch.cuda.synchronize()
            times[b].append(e0.elapsed_time(e1) / reps)
    return {str(b): dict(samples=b, actors_per_sample=100, steps=t, trajectories=2, ms_median=float(np.median(v)),
                         ms_min=float(min(v)), ms_max=float(max(v))) for b, v in times.items()}


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
    ap.add_argument("--num-workers", type=int, default=16)
    ap.add_argument("--frames", type=int, default=61, help="frames per trajectory (4 trajectories; 20 fewer samples each)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import bench
    from lav_b200 import synth
    from lav_b200.datasets import TemporalLiDARPaintedDataset
    from lav_b200.evaluate import evaluate
    dev = torch.device("cuda:0")
    res = dict(gpu_before=gpu_info(), batch=args.batch, num_workers=args.num_workers)
    res["kernel"] = kernel_ms((32, 256), 20, 9, 200, dev)
    tmp = tempfile.mkdtemp(prefix="lavb_driving_score_")
    rec = os.path.join(tmp, "recording")
    synth.record_trajectories(rec, 4, args.frames, seed=2021, n_points=30000, n_actors=100)
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
    evaluate(lid, uni, ds, args.batch, "f16", args.num_workers, driving_score=True)   # warm-up: plans, cuDNN algorithms, pages
    for drive in (False, True, False, True, False, True):
        rate, r = timed(lambda: evaluate(lid, uni, ds, args.batch, "f16", args.num_workers, driving_score=drive), n)
        res.setdefault(f"evaluate_samples_per_s_driving_score_{drive}", []).append(rate)
        if drive:
            res["evaluate_driving_score"] = r["driving_score"]
    res["gpu_after"] = gpu_info()
    shutil.rmtree(tmp, True)
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "driving_score_measure.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k != "evaluate_driving_score"}))


if __name__ == "__main__":
    main()
