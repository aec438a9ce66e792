"""Training-data throughput: the device-side TemporalLiDARPaintedDataset against one CPU worker of the reference's pipeline.

    python scripts/loader_throughput.py --out-dir OUT [--batch 32] [--batches 6]

Writes a seeded recording to a temporary directory and measures, with the GPU name and power limit read in the same run:
  1. loader batches/s at --batch (device events + synchronize, after a warm-up batch);
  2. ops.bev_targets on one batch (one 128-byte-per-plane job-table copy + the launch): time, and algorithmic bytes (planes
     read + written) over it;
  3. one sample of the CPU path (numpy / OpenCV restatement of __getitem__, oracle/dataset_ref.py) on one host core — what one
     of the reference's DataLoader workers does per sample;
  4. LAVTrainer.train_lidar samples/s with the loader in the loop, against the same trainer on one pre-staged batch;
  5. a breakdown per batch at B = 32 and 64: host `prepare` on 1 and on --num-workers threads, the host tables of the batched
     path (stage_batch), and the device build of the per-sample path (one GpuLidarStacker and detections_to_heatmap call per
     sample, as the loader did before the batched kernels) against the batched path (launch_batch), both ending in a
     synchronize, alternating on the same prepared batch.
Results go to OUT/loader_throughput.json.
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
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def per_sample_device(ds, hs, decoded, gen):
    """the device part of a batch as the loader built it before the batched kernels: per sample GpuLidarStacker and
    detections_to_heatmap, one bev_targets launch, and the label copies."""
    dev = ds.device
    parts = [ds.lidar_and_maps(h, gen) for h in hs]
    bev = ds.bev_batch(hs, decoded)
    st = lambda i: torch.stack([p[i] for p in parts])
    f32 = lambda key: torch.as_tensor(np.stack([h[key] for h in hs]), dtype=torch.float32).to(dev)
    ints = lambda key: torch.tensor([h[key] for h in hs], dtype=torch.int64)
    return (st(0), torch.tensor([p[1] for p in parts]), st(2), st(3), st(4), bev, f32("ego_locs"), ints("cmd").to(dev), f32("nxp"),
            ints("bra").to(dev), f32("locs"), f32("oris"), torch.as_tensor(np.stack([h["typs"] for h in hs])).to(dev),
            ints("num_objs"))


def breakdown(ds, B, workers, reps):
    """seconds per batch of B samples: host prepare (1 and `workers` threads), host tables, the two device paths."""
    from concurrent.futures import ThreadPoolExecutor
    from lav_b200.datasets import stage_maps
    rng = np.random.RandomState(B)
    idxs = list(range(B))
    draws = [ds.draw(rng) for _ in idxs]
    out = {k: [] for k in ("prepare_1_thread_s", "prepare_workers_s", "stage_batch_s", "device_per_sample_s", "device_batched_s")}
    with ThreadPoolExecutor(workers) as pool:
        for r in range(reps + 1):                                      # the first round warms up and is not kept
            t0 = time.perf_counter()
            hs = [ds.prepare(i, *d) for i, d in zip(idxs, draws)]
            t1 = time.perf_counter()
            list(pool.map(lambda a: ds.prepare(a[0], *a[1]), zip(idxs, draws)))
            t2 = time.perf_counter()
            st = ds.stage_batch(hs, torch.Generator().manual_seed(r))
            t3 = time.perf_counter()
            decoded = ds.decode_maps(stage_maps(hs, True))
            torch.cuda.synchronize()
            t4 = time.perf_counter()
            old = per_sample_device(ds, hs, decoded, torch.Generator().manual_seed(r))
            torch.cuda.synchronize()
            t5 = time.perf_counter()
            new = ds.launch_batch(st)
            torch.cuda.synchronize()
            t6 = time.perf_counter()
            if r == 0:
                assert all(torch.equal(a.cpu(), b.cpu()) for a, b in zip(old, new))
                continue
            for k, v in zip(out, (t1 - t0, t2 - t1, t3 - t2, t5 - t4, t6 - t5)):
                out[k].append(v)
    return {k: float(np.median(v)) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", required=True)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--batches", type=int, default=6)
    ap.add_argument("--train-steps", type=int, default=4)
    ap.add_argument("--num-workers", type=int, default=16)
    ap.add_argument("--breakdown-reps", type=int, default=3)
    args = ap.parse_args()
    os.makedirs(args.out_dir, exist_ok=True)
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import bench
    from lav_b200 import ops, synth
    from lav_b200.datasets import TemporalBatchLoader, TemporalLiDARPaintedDataset
    from lav_b200.train import LAVTrainer
    from oracle import dataset_ref as D
    from oracle import lav_ref as O
    dev = torch.device("cuda:0")
    res = dict(gpu=gpu_info(), batch=args.batch, num_workers=args.num_workers)
    tmp = tempfile.mkdtemp(prefix="lavb_loader_")                      # the recording (~1 MB per frame) stays out of --out-dir
    rec = os.path.join(tmp, "recording")
    n_traj, n_frames = 4, 21 + max(args.batch * (args.batches + 1), 64) // 4 + 1
    t0 = time.time()
    synth.record_trajectories(rec, n_traj, n_frames, seed=2021, n_points=30000)
    res["record_s"] = time.time() - t0
    cfg = dict(num_plan=20, num_frame_stack=2, seg_channels=[4, 6, 7, 10], max_lidar_points=120000, camera_x=1.5, camera_z=2.4,
               camera_yaws=[-120, -60, 0, 60, 120], angle_jitter=20, stack_loc_jitter=0.4, stack_ori_jitter=0.1,
               max_pedestrian_radius=10, max_vehicle_radius=25, max_mot_vehicle_radius=15, max_objs=20, min_x=-10, max_x=70,
               min_y=-40, max_y=40, pixels_per_meter=4, percentage_data=1.01, all_towns=True, data_dir=rec)
    cfg_path = os.path.join(tmp, "config.yaml")
    yaml.safe_dump(cfg, open(cfg_path, "w"))
    ds = TemporalLiDARPaintedDataset(cfg_path, seed=2021, device=dev)
    res["samples"] = len(ds)

    # 1. loader batches/s
    loader = TemporalBatchLoader(ds, args.batch, seed=1, num_workers=args.num_workers)
    it = iter(loader)
    staged = next(it)                                                  # warm-up (and the trainer's pre-staged batch below)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 0
    t0 = time.time()
    e0.record()
    for _ in range(args.batches):
        next(it)
        n += 1
    e1.record()
    torch.cuda.synchronize()
    res["loader_batches_per_s"] = n / (time.time() - t0)
    res["loader_samples_per_s"] = res["loader_batches_per_s"] * args.batch

    # 2. bev_targets alone
    hs = [ds.prepare(i, *ds.draw(ds.rng)) for i in range(args.batch)]
    from lav_b200.datasets import stage_maps
    planes = ds.planes_on_stream(ds.decode_maps(stage_maps(hs, True)))
    n_bev = 3 + 2 * (ds.num_frame_stack + 1)
    jobs = ops.bev_jobs([(s + sum(len(x["pngs"]) for x in hs[:b]) if s >= 0 else -1, b * n_bev + d, a1, a2, dx, dy)
                         for b, h in enumerate(hs) for s, d, a1, a2, dx, dy in h["rows"]])
    out = torch.empty((len(hs), n_bev, 320, 320), dtype=torch.uint8, device=dev)
    assert torch.equal(ops.bev_targets(planes, jobs, out), ds.bev_batch(hs))
    torch.cuda.synchronize()
    reps = 50
    e0.record()
    for _ in range(reps):
        ops.bev_targets(planes, jobs, out)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    nbytes = planes.numel() + out.numel()
    res.update(bev_batch_ms=ms, bev_bytes=nbytes, bev_gb_per_s=nbytes / (ms * 1e-3) / 1e9,
               bev_note="per call: job table build on the host + one H2D copy + one launch")

    # 3. CPU path per sample on one host core (the reference's per-worker work, numpy / fixed-point warp restatement)
    torch.set_num_threads(1)
    convs = O.default_converters()
    k = 3
    t0 = time.time()
    for i in range(k):
        traj, index = ds.index[i]
        env = ds.env(traj)
        D.get_item(env.get, index, cfg, 5.0, [(np.zeros(2), 0.0)] * 3, None, convs)
    res["cpu_oracle_s_per_sample"] = (time.time() - t0) / k
    try:
        import cv2
        img = np.zeros((320, 320, 2), np.uint8)
        t0 = time.time()
        for _ in range(100):
            cv2.warpAffine(img, cv2.getRotationMatrix2D((160, 280), 5.0, 1.0), (320, 320), flags=cv2.INTER_LINEAR)
        res["cpu_cv2_warp_ms"] = (time.time() - t0) * 10
    except ImportError:
        res["cpu_cv2_warp_ms"] = None

    # 4. trainer with the loader in the loop vs a pre-staged batch
    (_, lid, uni, _), _ = bench.build_models()
    tr = LAVTrainer(lid.to(dev), uni.to(dev), device=dev)
    tr.train_lidar(*staged)
    torch.cuda.synchronize()
    t0 = time.time()
    for _ in range(args.train_steps):
        tr.train_lidar(*staged)
    torch.cuda.synchronize()
    res["train_staged_samples_per_s"] = args.train_steps * args.batch / (time.time() - t0)
    loader = TemporalBatchLoader(ds, args.batch, seed=2, num_workers=args.num_workers)
    it = iter(loader)
    tr.train_lidar(*next(it))
    torch.cuda.synchronize()
    t0 = time.time()
    for _ in range(args.train_steps):
        tr.train_lidar(*next(it))
    torch.cuda.synchronize()
    res["train_loader_samples_per_s"] = args.train_steps * args.batch / (time.time() - t0)
    res["breakdown"] = {B: breakdown(ds, B, args.num_workers, args.breakdown_reps) for B in (32, 64)}
    shutil.rmtree(tmp, True)
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "loader_throughput.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
