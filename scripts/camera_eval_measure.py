"""Measurements of the camera-model scores (DESIGN §3, §4): the lavb_seg_confusion time against the materialised route
(output_conv's fp32 logits, then argmax and bincount in ATen) on the same features, lav_b200.evaluate_rgb frames/s, and the
loader's host decode rate, on a synthetic recording.

    python scripts/camera_eval_measure.py --out-dir OUT [--batch 32] [--num-workers 16]

Seeded models (tests/util.py's ERFNet weights, a seeded brake model) at f16; the GPU's name, power limit and clocks are read in the
same run.  Kernel times are CUDA-event medians over rounds in which the kernel and the materialised route alternate, on the h16
decoder features of 96 and 160 seeded 288 x 256 frames.  The HBM bound counts 32 B of features per feature pixel and 1 label byte
per pixel.  The loader rate is CameraBatchLoader's alone (record reads and cv2 decodes, no model).  Results go to
OUT/camera_eval_measure.json.
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


def kernel_ms(sm, sizes, rounds, reps, dev):
    from lav_b200 import ops, synth
    lut = ops.sem_class_table([4, 6, 7, 10])
    lut_d = torch.from_numpy(lut).long().to(dev)
    out_conv = sm.erfnet._plan_get(dev, sm.erfnet._build)[1]
    args = {}
    for n in sizes:
        imgs = torch.cat([synth.rgb_frames(tag=f"meas{k}", smooth=True) for k in range(-(-n // 3))])[:n].to(dev)
        with torch.no_grad():
            feat, table, c = sm.forward_features_nhwc(imgs)
        labels = torch.from_numpy(np.random.RandomState(n).randint(0, 23, (n, 288, 256)).astype(np.uint8)).to(dev)
        args[n] = (feat, table, labels, c)

    def kernel(n):
        feat, table, labels, c = args[n]
        return ops.seg_confusion(feat, table, labels, lut, c)

    def materialised(n):
        feat, table, labels, c = args[n]
        logits = out_conv(feat, out_dtype=torch.float32)
        idx = (lut_d[labels.long()] * c + logits.argmax(-1)) + torch.arange(n, device=dev)[:, None, None] * (c * c)
        return torch.bincount(idx.view(-1), minlength=n * c * c).view(n, c * c)

    res = {}
    for n in sizes:
        a, b = kernel(n)[:, :-1].long(), materialised(n)
        res[f"{n}_max_count_difference"] = int((a - b).abs().max())
    times = {(n, k): [] for n in sizes for k in ("seg_confusion", "materialised")}
    with torch.no_grad():
        for _ in range(rounds):
            for n in sizes:
                for k, fn in (("seg_confusion", kernel), ("materialised", materialised)):
                    fn(n)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(reps):
                        fn(n)
                    e1.record()
                    torch.cuda.synchronize()
                    times[(n, k)].append(e0.elapsed_time(e1) / reps)
    for (n, k), v in times.items():
        nbytes = n * (144 * 128 * 32 + 288 * 256)
        res[f"{n}_{k}"] = dict(ms_median=float(np.median(v)), ms_min=float(min(v)), ms_max=float(max(v)))
        if k == "seg_confusion":
            res[f"{n}_{k}"].update(hbm_bytes=nbytes, hbm_bound_ms=nbytes / HBM_BYTES_PER_S * 1e3,
                                   hbm_share=nbytes / HBM_BYTES_PER_S * 1e3 / float(np.median(v)))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", required=True)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--num-workers", type=int, default=16)
    ap.add_argument("--frames", type=int, default=43, help="frames per trajectory (4 trajectories; 3 fewer samples each)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import yaml
    from lav_b200 import synth
    from lav_b200.datasets import CameraBatchLoader, CameraDataset
    from lav_b200.evaluate_rgb import evaluate_rgb
    from lav_b200.heads import RGBBrakePredictionModel
    from tests import util
    dev = torch.device("cuda:0")
    res = dict(gpu_before=gpu_info(), batch=args.batch, num_workers=args.num_workers)
    sm, _ = util.seg_model(dev)
    sm.set_precision("f16")
    res["kernel"] = kernel_ms(sm, (96, 160), 7, 20, dev)
    tmp = tempfile.mkdtemp(prefix="lavb_camera_eval_")
    rec = os.path.join(tmp, "recording")
    synth.record_trajectories(rec, 4, args.frames, seed=2021, n_points=64, images=True, n_cameras=3)
    cfg = dict(data_dir=rec, percentage_data=1.01, all_towns=True, num_plan=3, camera_yaws=[-60, 0, 60], crop_tel_bottom=96,
               seg_channels=[4, 6, 7, 10])
    cfg_path = os.path.join(tmp, "config.yaml")
    yaml.safe_dump(cfg, open(cfg_path, "w"))
    ds = CameraDataset(cfg_path, device=dev)
    n = len(ds)
    res["frames"] = n
    bra = RGBBrakePredictionModel([4, 6, 7, 10]).eval()
    bra.load_state_dict(synth.fill_state_dict_(bra.state_dict(), seed=13))
    evaluate_rgb(sm, bra, ds, args.batch, "f16", args.num_workers)          # warm-up: plans, cuDNN algorithms, pages
    for _ in range(3):
        t0 = time.perf_counter()
        for _ in CameraBatchLoader(ds, args.batch, args.num_workers).staged_batches():
            pass
        torch.cuda.synchronize()
        res.setdefault("loader_frames_per_s", []).append(n / (time.perf_counter() - t0))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = evaluate_rgb(sm, bra, ds, args.batch, "f16", args.num_workers)
        torch.cuda.synchronize()
        res.setdefault("evaluate_rgb_frames_per_s", []).append(n / (time.perf_counter() - t0))
    res["evaluate_rgb"] = r
    res["gpu_after"] = gpu_info()
    shutil.rmtree(tmp, True)
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "camera_eval_measure.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k != "evaluate_rgb"}))


if __name__ == "__main__":
    main()
