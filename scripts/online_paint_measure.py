"""Measurements of online painting (DESIGN §3, §4): ops.lidar_batch_paint against its composition (paint_deconv_batched per
sweep, then lidar_batch) at B = 32 with 30 k- and 120 k-point samples, the ERFNet call on the distinct frames of a 32-sample
ordered batch, lav_b200.evaluate samples/s stored and online (alternated), and the peak device memory of both.

    python scripts/online_paint_measure.py --out-dir OUT [--batch 32] [--num-workers 16] [--points 30000] [--rounds 2]

Kernel: tests/test_gpu_online_paint.batch_inputs (three sweeps per sample, 34 frame slots, h16 features, C = 5, T = 3, a 20
degree rotation), CUDA-event medians over rounds of 20 calls after a warm-up.  The bytes a row needs: 4 B of row index and 16 B of
raw point per row, 32 B of features per row a camera sees, and the (3 + C + T) * 4 B output row; the share is of the H100 SXM's
3.35 TB/s.  ERFNet: 34 x 3 uint8 frames at f16 through forward_features_nhwc.  Evaluator: tests/util.py's seeded models
(bench's LiDAR model and UniPlanner, the seeded ERFNet) at f16 over a synthetic recording of 2 trajectories with --points points
per sweep; the stored run reads a copy painted by data_paint with the same ERFNet.  The GPU's name, power limit and clocks are
read in the same run.  Results go to OUT/online_paint_measure.json.
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

from eval_measure import gpu_info  # noqa: E402

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet


def events_ms(call, rounds=7, reps=20):
    for _ in range(3):
        call()
    times = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            call()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / reps)
    return float(np.median(times)), float(min(times)), float(max(times))


def kernel(dev):
    from lav_b200 import ops
    from tests.test_gpu_online_paint import HW, batch_inputs, composition
    res = {}
    C, T = 5, 3
    for n in (10000, 40000):
        raw, rows, sweeps, slots, feat, deconv, cams = batch_inputs(32, n, 34, 3, C, ops.h16(), 20.0, n, 3 * n)
        d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        raw_d, rows_d, feat_d, deconv_d, slots_d = d(raw), d(rows), feat.to(dev), deconv.to(dev), d(slots)
        sweeps_d = ops._to_device(sweeps.view(np.uint8), dev)
        out = torch.empty((32, 3 * n, 3 + C + T), device=dev)
        fused = lambda: ops.lidar_batch_paint(raw_d, rows_d, sweeps_d, slots_d, feat_d, C, deconv_d, cams, HW, T, out=out)
        comp = lambda: composition(raw_d, rows_d, sweeps, slots, feat_d, C, deconv_d, cams, T)
        assert torch.equal(fused().view(torch.int32), comp()[0].view(torch.int32))
        live = rows[(rows >= 0) & (rows < len(raw))]
        seen = ops.paint(raw_d, torch.ones((len(cams), 1) + HW, device=dev), cams, mode=0)[:, 0].cpu().numpy()
        visible = int(seen[live].sum())
        n_rows = rows.size
        nbytes = n_rows * 4 + len(live) * 16 + visible * 32 + n_rows * (3 + C + T) * 4
        f_med, f_min, f_max = events_ms(fused)
        c_med, c_min, c_max = events_ms(comp, rounds=5, reps=3)
        res[f"B32_N{3 * n}"] = dict(rows=n_rows, visible_rows=visible, bytes=nbytes, bytes_per_row=nbytes / n_rows,
                                    fused_ms=f_med, fused_ms_min=f_min, fused_ms_max=f_max, composition_ms=c_med,
                                    composition_ms_min=c_min, composition_ms_max=c_max,
                                    hbm_share=nbytes / HBM_BYTES_PER_S * 1e3 / f_med)
    return res


def erfnet_ms(sm, dev):
    from lav_b200 import synth
    imgs = torch.cat([synth.rgb_frames(tag=f"opm{k}", smooth=True) for k in range(34)]).to(dev)
    with torch.no_grad():
        med, lo, hi = events_ms(lambda: sm.forward_features_nhwc(imgs), rounds=5, reps=5)
    return dict(images=int(imgs.shape[0]), ms=med, ms_min=lo, ms_max=hi)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", required=True)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--num-workers", type=int, default=16)
    ap.add_argument("--frames", type=int, default=60, help="frames per trajectory (2 trajectories; 20 fewer samples each)")
    ap.add_argument("--points", type=int, default=30000, help="points per recorded sweep")
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import yaml
    import lav_b200.evaluate as E
    from lav_b200 import synth
    from lav_b200.data_paint import PointPaintDataset, paint_dataset
    from lav_b200.datasets import TemporalLiDARPaintedDataset
    from tests import util
    from tests.test_gpu_evaluate import seeded_models
    from tests.test_online_paint_cpu import CONFIG
    dev = torch.device("cuda:0")
    res = dict(gpu_before=gpu_info(), batch=args.batch, num_workers=args.num_workers, points_per_sweep=args.points)
    res["kernel"] = kernel(dev)
    sm, _ = util.seg_model(dev)
    sm.eval().set_precision("f16")
    res["erfnet_34_frames"] = erfnet_ms(sm, dev)
    tmp = tempfile.mkdtemp(prefix="lavb_online_paint_")
    rec, stored = os.path.join(tmp, "recording"), os.path.join(tmp, "painted")
    synth.record_trajectories(rec, 2, args.frames, seed=2021, n_points=args.points, images=True, n_cameras=3)
    shutil.copytree(rec, stored)
    pp = PointPaintDataset(stored)
    paint_dataset(pp, sm, frames_per_batch=args.batch, device=dev)
    pp.close()
    cfg_path = os.path.join(tmp, "config.yaml")
    yaml.safe_dump(dict(CONFIG, data_dir=rec, max_lidar_points=120000), open(cfg_path, "w"))
    lid, uni = seeded_models()
    runs = dict(stored=(stored, None), online=(rec, sm))
    for rnd in range(args.rounds + 1):                                       # round 0 warms up plans and pages
        for name, (data, seg) in runs.items():
            ds = TemporalLiDARPaintedDataset(cfg_path, device=dev, overrides=dict(data_dir=data))
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated(dev)
            torch.cuda.reset_peak_memory_stats(dev)
            t0 = time.perf_counter()
            r = E.evaluate(lid, uni, ds, args.batch, "f16", args.num_workers, forecast=True, plan_safety=True, seg_model=seg)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            if rnd:
                res.setdefault(f"{name}_samples_per_s", []).append(r["samples"] / dt)
                res[f"{name}_peak_bytes_above_resident"] = torch.cuda.max_memory_allocated(dev) - base
                res["samples"] = r["samples"]
                if seg is not None:
                    res["painting"] = r["painting"]
    res["peak_bytes_per_sample"] = {k: res[f"{k}_peak_bytes_above_resident"] / args.batch for k in runs}
    res["gpu_after"] = gpu_info()
    shutil.rmtree(tmp, True)
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "online_paint_measure.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
