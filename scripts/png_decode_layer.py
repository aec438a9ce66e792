"""The recordings' map PNG decode: ops.png_decode_gray8 on the GPU against cv2 on the host, and where `prepare` spends its time.

    python scripts/png_decode_layer.py --out-dir OUT [--reps 50]

Writes a seeded recording (synth.record_trajectories, 30 000-point sweeps) to a temporary directory and measures, with the GPU
name and power limit read in the same run:
  1. the kernel on the 288 maps of a 32-sample train_full batch and the 2 304 of a 256-sample train_bev batch: CUDA events
     around each launch, after a warm-up, median and min-max over --reps; GB/s of planes written (h * w bytes per plane);
  2. cv2.imdecode(IMREAD_GRAYSCALE) of the same planes on 1 and 16 host threads;
  3. bytes copied host-to-device per batch: the decoded planes (what the loaders copied before) against the packed zlib streams
     and the 32-byte job records;
  4. TemporalLiDARPaintedDataset.prepare per sample, and its pieces: record reads (LiDAR sweeps, poses, labels), the chunk walk
     of the 9 map PNGs (png.parse), actor_tracks, and the host decode of the same 9 maps (cv2, what prepare did before).
Results go to OUT/png_decode_layer.json.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import yaml  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def stats(xs):
    return dict(median=float(np.median(xs)), min=float(np.min(xs)), max=float(np.max(xs)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", required=True)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--prepare-samples", type=int, default=64)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import cv2
    from lav_b200 import ops, png, synth
    from lav_b200.datasets import _frame, actor_tracks, ego_pose, stage_maps, TemporalLiDARPaintedDataset
    dev = torch.device("cuda:0")
    res = dict(gpu=gpu_info(), cv2=cv2.__version__, host_cpus=os.cpu_count())
    tmp = tempfile.mkdtemp(prefix="lavb_png_")
    rec = os.path.join(tmp, "recording")
    synth.record_trajectories(rec, 4, 21 + 256 // 4 + 2, seed=2021, n_points=30000)
    cfg = dict(num_plan=20, num_frame_stack=2, seg_channels=[4, 6, 7, 10], max_lidar_points=120000, camera_x=1.5, camera_z=2.4,
               camera_yaws=[-120, -60, 0, 60, 120], angle_jitter=20, stack_loc_jitter=0.4, stack_ori_jitter=0.1,
               max_pedestrian_radius=10, max_vehicle_radius=25, max_mot_vehicle_radius=15, max_objs=20, min_x=-10, max_x=70,
               min_y=-40, max_y=40, pixels_per_meter=4, percentage_data=1.01, all_towns=True, data_dir=rec)
    cfg_path = os.path.join(tmp, "config.yaml")
    yaml.safe_dump(cfg, open(cfg_path, "w"))
    ds = TemporalLiDARPaintedDataset(cfg_path, seed=2021, device=dev)
    rng = np.random.RandomState(0)

    # 1-3: the maps of a 32- and a 256-sample batch
    for B in (32, 256):
        idxs = rng.permutation(len(ds))[:B]
        hs = [ds.prepare(int(i), *ds.draw(rng)) for i in idxs]
        maps = stage_maps(hs, True)
        datas = [ds.env(ds.index[int(i)][0]).get(k.rsplit(": ", 1)[-1]) for i, h in zip(idxs, hs) for k, _ in h["pngs"]]
        n = maps["n_planes"]
        src = maps["src"].to(dev)
        out = torch.empty((n, 320, 320), dtype=torch.uint8, device=dev)
        status = ops.png_decode_gray8(src, maps["jobs"], out)
        torch.cuda.synchronize()
        want = np.stack([cv2.imdecode(np.frombuffer(d, np.uint8), cv2.IMREAD_GRAYSCALE) for d in datas])
        assert not status.any() and np.array_equal(out.cpu().numpy(), want)
        ms = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            ops.png_decode_gray8(src, maps["jobs"], out, status)
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        row = dict(planes=n, kernel_ms=stats(ms), planes_written_gb_per_s=n * 320 * 320 / (np.median(ms) * 1e-3) / 1e9,
                   note="per launch: the job-table H2D copy (pinned) + the kernel")
        bufs = [np.frombuffer(d, np.uint8) for d in datas]
        for threads in (1, 16):
            with ThreadPoolExecutor(threads) as pool:
                list(pool.map(lambda b: cv2.imdecode(b, cv2.IMREAD_GRAYSCALE), bufs))
                t = []
                for _ in range(5):
                    t0 = time.perf_counter()
                    list(pool.map(lambda b: cv2.imdecode(b, cv2.IMREAD_GRAYSCALE), bufs))
                    t.append((time.perf_counter() - t0) * 1e3)
            row[f"cv2_{threads}_threads_ms"] = stats(t)
        row["h2d_bytes_decoded_planes"] = n * 320 * 320
        row["h2d_bytes_streams_and_jobs"] = int(maps["src"].numel() + maps["jobs"].nbytes)
        res[f"batch_{B}"] = row

    # 4: prepare per sample and its pieces
    samples = [(int(i), ds.draw(rng)) for i in rng.permutation(len(ds))[:args.prepare_samples]]
    t = dict(prepare=0.0, record_reads=0.0, png_parse=0.0, actor_tracks=0.0, cv2_decode_9_maps=0.0)
    for idx, d in samples:
        traj, index = ds.index[idx]
        env = ds.env(traj)
        frames = [i for i in range(index, index - ds.num_frame_stack - 1, -1) if i >= 0]
        t0 = time.perf_counter()
        h = ds.prepare(idx, *d)
        t1 = time.perf_counter()
        poses = {i: ego_pose(env, i) for i in frames}
        [(_frame(env, "lidar", i), _frame(env, "lidar_sem", i)) for i in frames]
        _frame(env, "nxp", index), _frame(env, "cmd", index, np.uint8), _frame(env, "bra", index, np.uint8)
        t2 = time.perf_counter()
        keys = [k.rsplit(": ", 1)[-1] for k, _ in h["pngs"]]
        datas = [env.get(k) for k in keys]
        t3 = time.perf_counter()
        [png.parse(x, "k", 320) for x in datas]
        t4 = time.perf_counter()
        actor_tracks(env, index, ds.num_plan, ds.max_pedestrian_radius, ds.max_vehicle_radius)
        t5 = time.perf_counter()
        [cv2.imdecode(np.frombuffer(x, np.uint8), cv2.IMREAD_GRAYSCALE) for x in datas]
        t6 = time.perf_counter()
        for k, v in zip(t, (t1 - t0, (t2 - t1) + (t3 - t2), t4 - t3, t5 - t4, t6 - t5)):
            t[k] += v * 1e3 / len(samples)
        del poses
    t["rest"] = t["prepare"] - t["record_reads"] - t["png_parse"] - t["actor_tracks"]
    t["prepare_before_estimate"] = t["prepare"] - t["png_parse"] + t["cv2_decode_9_maps"]
    res["prepare_ms_per_sample"] = t
    shutil.rmtree(tmp, True)
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "png_decode_layer.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
