"""Measurements of the painting scores (DESIGN §3, §4): the lavb_paint_confusion time at F = 32 sweeps of 30 k and 120 k points,
and lav_b200.evaluate_paint frames/s next to the loader alone, on a synthetic recording.

    python scripts/paint_eval_measure.py --out-dir OUT [--batch 32] [--num-workers 16] [--points 30000]

Kernel: seeded sweeps (synth.lidar_sweep), the three painting cameras, h16 decoder features of seeded frames (tests/util.py's
ERFNet weights at f16), seeded tags, C = 5 and both sources (online and stored rows); CUDA-event medians over rounds of 50
launches.  The bytes it must read are 16 B of point, the 32 B feature pixel, 1 tag byte and 16 B of stored row per visible
point, and 16 B per point that no camera sees.  Evaluator: online and stored at f16 over a recording of 4 trajectories with
--points points per sweep; the loader rate is CameraBatchLoader's alone over the same PaintDataset (record reads and cv2
decodes, no model).  The GPU's name, power limit and clocks are read in the same run.  Results go to OUT/paint_eval_measure.json.
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

from eval_measure import gpu_info  # noqa: E402

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet


def kernel_ms(sm, sizes, frames, rounds, reps, dev):
    from lav_b200 import ops, synth
    from lav_b200 import point_painting as PP
    lut = ops.sem_class_table([4, 6, 7, 10])
    cams = np.stack([cv.packed() for cv in PP.make_converters(1.5, 2.4)])
    imgs = torch.cat([synth.rgb_frames(tag=f"pmeas{k}", smooth=True) for k in range(frames)]).to(dev)
    with torch.no_grad():
        feat, table, c = sm.forward_features_nhwc(imgs)
    tags = torch.from_numpy(np.random.RandomState(3).randint(0, 23, (frames * 3, 288, 256)).astype(np.uint8)).to(dev)
    res = {}
    for n in sizes:
        pts = torch.stack([synth.lidar_sweep(n, tag=f"pmeas{f}") for f in range(frames)]).to(dev)
        rs = np.random.RandomState(n)
        prob = rs.dirichlet(np.ones(c), (frames, n))
        stored = torch.from_numpy((prob[..., 1:] * (1 - prob[..., :1])).astype(np.float32)).to(dev)
        call = lambda: ops.paint_confusion(pts, tags, lut, cams, (-10, 70, -40, 40), c, feat=feat, table=table, stored=stored)
        counts = call()
        cnt = dict(zip(ops.PAINT_COUNTERS, counts[:, :8].sum(0).tolist()))
        times = []
        for _ in range(rounds):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                call()
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1) / reps)
        visible = cnt["points"] - cnt["not_visible"] - cnt["nan"]
        nbytes = visible * (16 + 32 + 1 + 16) + (cnt["points"] - visible) * 16
        med = float(np.median(times))
        res[f"F{frames}_N{n}"] = dict(ms_median=med, ms_min=float(min(times)), ms_max=float(max(times)), points=cnt["points"],
                                      visible=visible, hbm_bytes=nbytes, hbm_bound_ms=nbytes / HBM_BYTES_PER_S * 1e3,
                                      hbm_share=nbytes / HBM_BYTES_PER_S * 1e3 / med)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", required=True)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--num-workers", type=int, default=16)
    ap.add_argument("--frames", type=int, default=43, help="frames per trajectory (4 trajectories; 3 fewer samples each)")
    ap.add_argument("--points", type=int, default=30000, help="points per recorded sweep")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import yaml
    from lav_b200 import synth
    from lav_b200.data_paint import PointPaintDataset, paint_dataset
    from lav_b200.datasets import CameraBatchLoader, PaintDataset
    from lav_b200.evaluate_paint import evaluate_paint
    from tests import util
    dev = torch.device("cuda:0")
    res = dict(gpu_before=gpu_info(), batch=args.batch, num_workers=args.num_workers, points_per_sweep=args.points)
    sm, _ = util.seg_model(dev)
    sm.set_precision("f16")
    res["kernel"] = kernel_ms(sm, (30000, 120000), 32, 7, 50, dev)
    tmp = tempfile.mkdtemp(prefix="lavb_paint_eval_")
    rec = os.path.join(tmp, "recording")
    synth.record_trajectories(rec, 4, args.frames, seed=2021, n_points=args.points, images=True, n_cameras=3)
    pp = PointPaintDataset(rec)
    paint_dataset(pp, sm, frames_per_batch=args.batch, device=dev)          # lidar_sem rows of this model, as data_paint writes them
    pp.close()
    cfg = dict(data_dir=rec, percentage_data=1.01, all_towns=True, num_plan=3, seg_channels=[4, 6, 7, 10], camera_x=1.5,
               camera_z=2.4, min_x=-10, max_x=70, min_y=-40, max_y=40)
    cfg_path = os.path.join(tmp, "config.yaml")
    yaml.safe_dump(cfg, open(cfg_path, "w"))
    ds = PaintDataset(cfg_path, online=True, stored=True, device=dev)
    n = len(ds)
    res["frames"] = n
    evaluate_paint(sm, ds, args.batch, "f16", args.num_workers)              # warm-up: plans, pages
    for _ in range(3):
        t0 = time.perf_counter()
        for _ in CameraBatchLoader(ds, args.batch, args.num_workers).staged_batches():
            pass
        torch.cuda.synchronize()
        res.setdefault("loader_frames_per_s", []).append(n / (time.perf_counter() - t0))
        t0 = time.perf_counter()
        r = evaluate_paint(sm, ds, args.batch, "f16", args.num_workers)
        torch.cuda.synchronize()
        res.setdefault("evaluate_paint_frames_per_s", []).append(n / (time.perf_counter() - t0))
    res["evaluate_paint"] = r
    res["gpu_after"] = gpu_info()
    shutil.rmtree(tmp, True)
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "paint_eval_measure.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k != "evaluate_paint"}))


if __name__ == "__main__":
    main()
