"""Measurements of evaluate --brake (DESIGN §4): evaluation samples/s with and without --brake, and the loader alone with and
without the brake model's camera reads, on a synthetic recording with five cameras.

    python scripts/brake_eval_measure.py --out-dir OUT [--batch 32] [--num-workers 16] [--rounds 3]

Seeded models (bench.build_models: the LiDAR model, the UniPlanner and the brake model) at f16; a seeded recording in a temporary
directory (record_trajectories(images=True, n_cameras=5), 30 000-point sweeps); the agent controls of team_code_v2/config.yaml.
After one warm-up run of each, every round times the four runs in turn (evaluate without and with --brake, then the loader
without and with the camera reads), so the two sides of each comparison alternate.  The GPU's name, power limit and clocks are
read in the same run.  Results go to OUT/brake_eval_measure.json.
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
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import yaml  # noqa: E402

from eval_measure import gpu_info  # noqa: E402

# team_code_v2/config.yaml: the CONTROLLER section, cmd_thresh and pixels_per_meter
AGENT = dict(aim_point=[4, 4, 4, 3, 6, 6], speed_ratio=[0.8, 0.8, 0.8, 0.6, 0.8, 0.8], turn_KP=0.8, turn_KI=0.5, turn_KD=0.2,
             turn_n=40, speed_KP=5.0, speed_KI=0.5, speed_KD=1.0, speed_n=40, brake_speed=0.2, clip_delta=0.25, max_throttle=0.8,
             max_speed=35, cmd_thresh=0.2, pixels_per_meter=4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", required=True)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--num-workers", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--frames", type=int, default=61, help="frames per trajectory (4 trajectories; 20 fewer samples each)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import bench
    from lav_b200 import synth
    from lav_b200.datasets import TemporalBatchLoader, TemporalLiDARPaintedDataset
    from lav_b200.evaluate import evaluate
    dev = torch.device("cuda:0")
    res = dict(gpu_before=gpu_info(), batch=args.batch, num_workers=args.num_workers)
    tmp = tempfile.mkdtemp(prefix="lavb_brake_eval_")
    rec = os.path.join(tmp, "recording")
    synth.record_trajectories(rec, 4, args.frames, seed=2021, n_points=30000, images=True, n_cameras=5)
    cfg = dict(num_plan=20, num_frame_stack=2, seg_channels=[4, 6, 7, 10], max_lidar_points=120000, camera_x=1.5, camera_z=2.4,
               camera_yaws=[-120, -60, 0, 60, 120], angle_jitter=20, stack_loc_jitter=0.4, stack_ori_jitter=0.1,
               max_pedestrian_radius=10, max_vehicle_radius=25, max_mot_vehicle_radius=15, max_objs=20, min_x=-10, max_x=70,
               min_y=-40, max_y=40, pixels_per_meter=4, percentage_data=1.01, all_towns=True, crop_tel_bottom=96, data_dir=rec)
    cfg_path = os.path.join(tmp, "config.yaml")
    yaml.safe_dump(cfg, open(cfg_path, "w"))
    ds = TemporalLiDARPaintedDataset(cfg_path, device=dev)
    n = len(ds)
    res["samples"] = n
    (_, lid, uni, bra), _ = bench.build_models()

    def run_eval(brake):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = evaluate(lid, uni, ds, args.batch, "f16", args.num_workers, brake=brake, bra_model=bra if brake else None,
                     agent_config=AGENT)
        torch.cuda.synchronize()
        return n / (time.perf_counter() - t0), r

    def run_loader(cameras):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        loader = TemporalBatchLoader(ds, args.batch, drop_last=False, num_workers=args.num_workers, ordered=True, cameras=cameras)
        for _ in loader.staged_batches():
            pass
        torch.cuda.synchronize()
        return n / (time.perf_counter() - t0)

    run_eval(False), run_eval(True), run_loader(False), run_loader(True)          # warm-up: plans, cuDNN algorithms, pages
    for _ in range(args.rounds):
        for brake in (False, True):
            rate, r = run_eval(brake)
            res.setdefault(f"evaluate{'_brake' if brake else ''}_samples_per_s", []).append(rate)
        for cameras in (False, True):
            res.setdefault(f"loader{'_cameras' if cameras else ''}_samples_per_s", []).append(run_loader(cameras))
    res["brake"] = r["brake"]
    res["gpu_after"] = gpu_info()
    shutil.rmtree(tmp, True)
    for k in [k for k in res if k.endswith("_per_s")]:
        res[k + "_median"] = float(np.median(res[k]))
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "brake_eval_measure.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k != "brake"}))


if __name__ == "__main__":
    main()
