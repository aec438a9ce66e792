"""Measurements of the evaluator (DESIGN §4): eval_batch_kernel time per batch, evaluation samples/s on a synthetic recording of
realistic size against the loader alone, and the metric differences between the 16-bit and the fp32 path.

    python scripts/eval_measure.py --out-dir OUT [--batch 32] [--num-workers 16]

Seeded models (bench.build_models), a seeded recording in a temporary directory (30 000-point sweeps); the GPU's name, power limit
and clocks are read in the same run.  Results go to OUT/eval_measure.json.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import yaml  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def kernel_ms(B, half, reps, dev):
    from lav_b200 import ops
    from tests.test_gpu_evaluate import random_batch
    seg, gt, packed, actors, offsets, plan, ego = random_batch(B, 1, dev)
    if half:
        seg = seg.to(ops.h16())
    out = ops.eval_batch(seg, gt, packed, actors, offsets, plan, ego)
    times = []
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            ops.eval_batch(seg, gt, packed, actors, offsets, plan, ego, out=out)
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / reps)
    nbytes = seg.numel() * seg.element_size() + B * 3 * 320 * 320
    return dict(ms_median=float(np.median(times)), ms_min=float(min(times)), ms_max=float(max(times)), bytes_read=nbytes,
                gb_per_s=nbytes / (np.median(times) * 1e-3) / 1e9)


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
    from lav_b200.datasets import TemporalBatchLoader, TemporalLiDARPaintedDataset
    from lav_b200 import synth
    from lav_b200.evaluate import evaluate
    dev = torch.device("cuda:0")
    res = dict(gpu_before=gpu_info(), batch=args.batch, num_workers=args.num_workers)
    res["kernel_b32_fp32_seg"] = kernel_ms(args.batch, False, 200, dev)
    res["kernel_b32_h16_seg"] = kernel_ms(args.batch, True, 200, dev)
    tmp = tempfile.mkdtemp(prefix="lavb_eval_")
    rec = os.path.join(tmp, "recording")
    synth.record_trajectories(rec, 4, args.frames, seed=2021, n_points=30000)
    cfg = dict(num_plan=20, num_frame_stack=2, seg_channels=[4, 6, 7, 10], max_lidar_points=120000, camera_x=1.5, camera_z=2.4,
               camera_yaws=[-120, -60, 0, 60, 120], angle_jitter=20, stack_loc_jitter=0.4, stack_ori_jitter=0.1,
               max_pedestrian_radius=10, max_vehicle_radius=25, max_mot_vehicle_radius=15, max_objs=20, min_x=-10, max_x=70,
               min_y=-40, max_y=40, pixels_per_meter=4, percentage_data=1.01, all_towns=True, data_dir=rec)
    cfg_path = os.path.join(tmp, "config.yaml")
    yaml.safe_dump(cfg, open(cfg_path, "w"))
    ds = TemporalLiDARPaintedDataset(cfg_path, device=dev)
    res["samples"] = len(ds)
    (_, lid, uni, _), _ = bench.build_models()
    evaluate(lid, uni, ds, args.batch, "f16", args.num_workers)            # warm-up: plans, cuDNN algorithms, the recording's pages
    results = {}
    for precision in ("f16", "fp32", "f16", "fp32"):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = evaluate(lid, uni, ds, args.batch, precision, args.num_workers)
        torch.cuda.synchronize()
        res.setdefault(f"samples_per_s_{precision}", []).append(len(ds) / (time.perf_counter() - t0))
        results[precision] = r
    loader_rates = []
    for _ in range(2):
        t0 = time.perf_counter()
        for _batch in TemporalBatchLoader(ds, args.batch, drop_last=False, num_workers=args.num_workers, ordered=True):
            pass
        torch.cuda.synchronize()
        loader_rates.append(len(ds) / (time.perf_counter() - t0))
    res["loader_alone_samples_per_s"] = loader_rates
    res["results"] = results
    a, b = results["f16"], results["fp32"]
    diff = dict(bev_iou=[None if x is None or y is None else x - y for x, y in zip(a["bev_iou"], b["bev_iou"])],
                bev_counts=(np.array(a["bev_counts"]) - np.array(b["bev_counts"])).tolist(),
                det_ap={c: {k: None if a["det"][c]["ap"][k] is None else a["det"][c]["ap"][k] - b["det"][c]["ap"][k]
                            for k in a["det"][c]["ap"]} for c in a["det"]},
                n_det={c: a["det"][c]["n_det"] - b["det"][c]["n_det"] for c in a["det"]},
                ade=a["plan"]["ade"] - b["plan"]["ade"], fde=a["plan"]["fde"] - b["plan"]["fde"])
    res["f16_minus_fp32"] = diff
    res["gpu_after"] = gpu_info()
    shutil.rmtree(tmp, True)
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "eval_measure.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k != "results"}))


if __name__ == "__main__":
    main()
