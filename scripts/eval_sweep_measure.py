"""Measurements of checkpoint sweeps and multi-rank evaluation (DESIGN §4): evaluate samples/s at K = 1, 4, 16 and 64 resident
checkpoints with --forecast --plan-safety off and on, evaluate_bev at K = 1 and 16, one rank against every GPU of the machine at
K = 1, the device memory of one resident LiDAR + UniPlanner pair and of one BEVPlanner, and the peak memory of a batch.

    python scripts/eval_sweep_measure.py --out-dir OUT [--batch 32] [--num-workers 16] [--frames 61]

Seeded models (bench.build_models; the K checkpoints of a sweep are copies of one, each resident with its own packed copy), a seeded recording in a temporary
directory (30 000-point sweeps).  Runs alternate between the settings and each is repeated twice; the GPU's name, power limit
and clocks are read in the same run.  Results go to OUT/eval_sweep_measure.json.
"""
import argparse
import copy
import json
import os
import shutil
import socket
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import yaml  # noqa: E402

from scripts.eval_measure import gpu_info  # noqa: E402


def write_recording(tmp, frames):
    from lav_b200 import synth
    rec = os.path.join(tmp, "recording")
    synth.record_trajectories(rec, 4, frames, seed=2021, n_points=30000)
    cfg = dict(num_plan=20, num_frame_stack=2, seg_channels=[4, 6, 7, 10], max_lidar_points=120000, camera_x=1.5, camera_z=2.4,
               camera_yaws=[-120, -60, 0, 60, 120], angle_jitter=20, stack_loc_jitter=0.4, stack_ori_jitter=0.1,
               max_pedestrian_radius=10, max_vehicle_radius=25, max_mot_vehicle_radius=15, max_objs=20, min_x=-10, max_x=70,
               min_y=-40, max_y=40, pixels_per_meter=4, percentage_data=1.01, all_towns=True, data_dir=rec, x_jitter=3,
               crop_size=96)
    path = os.path.join(tmp, "config.yaml")
    yaml.safe_dump(cfg, open(path, "w"))
    return path


def pairs(k):
    """k resident copies of the seeded pair (their weights do not change the work)."""
    import bench
    (_, lid, uni, _), _ = bench.build_models()
    return [(copy.deepcopy(lid), copy.deepcopy(uni)) for _ in range(k)]


def planners(k):
    from tests.test_bev_train_cpu import _planner
    p = _planner(2021)
    return [copy.deepcopy(p) for _ in range(k)]


def resident_bytes(dev):
    """device bytes of one resident LiDAR + UniPlanner pair at f16 (the models and the packed inference copy) and of one
    BEVPlanner, as the sweep's memory check measures them."""
    from lav_b200.agent import infer_model
    from lav_b200.eval_sweep import ResidentMeter
    (lid, uni), = pairs(1)
    m = ResidentMeter(dev, lid, uni)
    im = infer_model(lid.to(dev).eval(), uni.to(dev).eval(), "f16", 1.5, 2.4, dev)
    pair = m.resident()
    p, = planners(1)
    m = ResidentMeter(dev, p)
    p.to(dev)
    bev = m.resident()
    del im, lid, uni, p
    torch.cuda.empty_cache()
    return pair, bev


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def _rank(rank, world, port, cfg_path, batch, workers, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), LOCAL_RANK=str(rank))
    import torch.distributed as dist
    from lav_b200.datasets import TemporalLiDARPaintedDataset
    from lav_b200.evaluate import evaluate_checkpoints
    dist.init_process_group("gloo", rank=rank, world_size=world)
    dev = torch.device("cuda", rank % torch.cuda.device_count())
    torch.cuda.set_device(dev)
    ds = TemporalLiDARPaintedDataset(cfg_path, device=dev)
    ps = pairs(1)
    evaluate_checkpoints(ps, ds, batch, "f16", workers)                    # warm-up
    dist.barrier()
    dt, _ = timed(lambda: evaluate_checkpoints(ps, ds, batch, "f16", workers))
    times = [None] * world
    dist.all_gather_object(times, dt)
    if rank == 0:
        json.dump(dict(world=world, seconds=max(times), samples_per_s=len(ds) / max(times)), open(out, "w"))
    dist.destroy_process_group()


def ranks(world, cfg_path, batch, workers, tmp):
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    out = os.path.join(tmp, f"ranks_{world}.json")
    mp.spawn(_rank, args=(world, port, cfg_path, batch, workers, out), nprocs=world, join=True)
    return json.load(open(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", required=True)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--num-workers", type=int, default=16)
    ap.add_argument("--frames", type=int, default=61, help="frames per trajectory (4 trajectories; 20 fewer samples each)")
    ap.add_argument("--ks", default="1,4,16,64")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from lav_b200.datasets import TemporalBEVDataset, TemporalLiDARPaintedDataset
    from lav_b200.evaluate import evaluate_checkpoints
    from lav_b200.evaluate_bev import evaluate_bev_checkpoints
    dev = torch.device("cuda:0")
    res = dict(gpu_before=gpu_info(), batch=args.batch, num_workers=args.num_workers, gpus=torch.cuda.device_count())
    res["resident_bytes_lidar_uniplanner_pair_f16"], res["resident_bytes_bev_planner"] = resident_bytes(dev)
    tmp = tempfile.mkdtemp(prefix="lavb_sweep_")
    try:
        cfg_path = write_recording(tmp, args.frames)
        ds = TemporalLiDARPaintedDataset(cfg_path, device=dev)
        n = res["samples"] = len(ds)
        ks = [int(k) for k in args.ks.split(",")]
        models = pairs(max(ks))
        evaluate_checkpoints(models[:1], ds, args.batch, "f16", args.num_workers, forecast=True, plan_safety=True)   # warm-up
        for extra in (False, True):
            torch.cuda.reset_peak_memory_stats(dev)
            base = torch.cuda.memory_allocated(dev)
            evaluate_checkpoints(models[:1], ds, args.batch, "f16", args.num_workers, forecast=extra, plan_safety=extra)
            res[f"peak_batch_bytes_above_resident_{'fc_ps' if extra else 'plain'}"] = torch.cuda.max_memory_allocated(dev) - base
        rates = {}
        for _ in range(2):                                              # alternate the settings, each twice
            for k in ks:
                for extra in (False, True):
                    dt, _ = timed(lambda: evaluate_checkpoints(models[:k], ds, args.batch, "f16", args.num_workers, forecast=extra,
                                                               plan_safety=extra))
                    rates.setdefault(f"K{k}_{'fc_ps' if extra else 'plain'}", []).append(n / dt)
                    print(f"evaluate K={k} forecast+plan_safety={extra}: {n / dt:.2f} samples/s", flush=True)
        res["evaluate_samples_per_s"] = rates
        del models
        torch.cuda.empty_cache()
        bds = TemporalBEVDataset(cfg_path, device=dev)
        ps = planners(16)
        evaluate_bev_checkpoints(ps[:1], bds, args.batch, args.num_workers, plan_safety=True)                     # warm-up
        brates = {}
        for _ in range(2):
            for k in (1, 16):
                dt, _ = timed(lambda: evaluate_bev_checkpoints(ps[:k], bds, args.batch, args.num_workers, plan_safety=True))
                brates.setdefault(f"K{k}_ps", []).append(len(bds) / dt)
                print(f"evaluate_bev K={k} plan_safety: {len(bds) / dt:.2f} samples/s", flush=True)
        res["evaluate_bev_samples_per_s"] = brates
        del ps
        torch.cuda.empty_cache()
        worlds = sorted({1, torch.cuda.device_count()})
        res["ranks_k1"] = [ranks(w, cfg_path, args.batch, args.num_workers, tmp) for w in worlds]
        if len(worlds) == 1:
            res["ranks_note"] = "one GPU on this machine: several GPUs not measured"
    finally:
        shutil.rmtree(tmp, True)
    res["gpu_after"] = gpu_info()
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "eval_sweep_measure.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
