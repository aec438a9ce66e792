"""Profile the privileged-planner stage (python -m lav_b200.train_bev) at the reference batch of 256 on one GPU:
  * TemporalBEVBatchLoader samples/s on a synthetic recording (record reads + PNG decodes on --num-workers threads, one
    bev_targets launch per batch);
  * the uint8 crop kernel (ops.crop_bilinear_u8) against the torch path it replaces (bev.float(), gather, affine_grid, grid_sample)
    for the ego crop and 5 vehicle crops per sample, 9 x 192 x 192 each;
  * one BEVTrainer.train_bev step, and its parts timed on their own: crops, embedder forward + backward, cast / plan GRUs forward
    + backward, Adam;
  * peak device memory of the step.
Prints the GPU name and power limit of the run, and writes JSON with --out.

    python scripts/bev_train_profile.py [--batch 256] [--out bev_profile.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch
import torch.nn.functional as F
import yaml

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lav_b200 import ops, synth  # noqa: E402
from lav_b200.heads import BEVPlanner, crop_theta  # noqa: E402
from lav_b200.train import BEVTrainer  # noqa: E402

PLANNER = dict(pixels_per_meter=4, crop_size=96, feature_x_jitter=1.5, feature_angle_jitter=20, x_offset=0,
               y_offset=1 + (-10) / ((70 + 10) / 2), num_cmds=6, num_plan=20, num_plan_iter=5, num_frame_stack=2)


def timed(fn, reps, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def gpu_info():
    name = torch.cuda.get_device_name()
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                               text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def loader_rate(B, workers, dev):
    from types import SimpleNamespace
    from lav_b200.datasets import get_data_loader
    tmp = tempfile.mkdtemp(prefix="lavb_bevprof_")
    n_traj = -(-2 * B // 40)                                        # 40 samples per 60-frame trajectory, two batches
    synth.record_trajectories(os.path.join(tmp, "data"), n_traj, 60, 7)
    cfg = dict(num_plan=20, num_frame_stack=2, crop_size=96, x_jitter=10, angle_jitter=20, max_pedestrian_radius=10,
               max_vehicle_radius=25, max_objs=20, min_x=-10, max_x=70, min_y=-40, max_y=40, pixels_per_meter=4,
               percentage_data=1.01, all_towns=True, data_dir=os.path.join(tmp, "data"))
    path = os.path.join(tmp, "c.yaml")
    yaml.safe_dump(cfg, open(path, "w"))
    loader = get_data_loader("temporal_bev", SimpleNamespace(config_path=path, seed=1, batch_size=B, device=dev, num_workers=workers))
    torch.cuda.synchronize()
    t0 = time.time()
    n = 0
    for batch in loader:
        n += batch[0].shape[0]
    torch.cuda.synchronize()
    return n / (time.time() - t0), n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--num-workers", type=int, default=16)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda")
    name, limit = gpu_info()
    print(f"GPU: {name}, power limit {limit}")
    res = dict(gpu=name, power_limit=limit, batch=args.batch)

    rate, n = loader_rate(args.batch, args.num_workers, dev)
    res["loader_samples_per_s"] = rate
    print(f"loader: {rate:.1f} samples/s ({n} samples, batch {args.batch}, {args.num_workers} threads)")

    batch = [t.to(dev) for t in synth.bev_planner_batch(B=args.batch)]
    bev, ego_locs, cmds, nxps, bras, locs, oris, typs = batch
    m = BEVPlanner(**PLANNER).to(dev).train()
    B, S = args.batch, 2 * PLANNER["crop_size"]
    K = B * 6                                                       # the ego + max_num_cars = 5 vehicles per sample
    g = torch.Generator().manual_seed(0)
    rel = ((torch.rand(K, 2, generator=g) * 2 - 1) * 20).to(dev)
    ori = ((torch.rand(K, generator=g) * 2 - 1) * 3.14).to(dev)
    frame = (torch.arange(K) % B).to(torch.int32).to(dev)
    theta = crop_theta(rel, ori, 320, 320, 4, S, m.offset_x, m.offset_y).float().contiguous()
    out = torch.empty((K, 9, S, S), device=dev)
    t_kernel = timed(lambda: ops.crop_bilinear_u8(bev, frame, theta, S, out=out), args.reps)

    def torch_path():
        feats = bev.float()[frame.long()]
        grids = F.affine_grid(theta, (K, 9, S, S), align_corners=True)
        return F.grid_sample(feats, grids, align_corners=True)
    t_torch = timed(torch_path, args.reps)
    gb = out.numel() * 4 / 1e9
    res.update(crops=K, crop_out_GB=gb, crop_kernel_ms=t_kernel, crop_torch_ms=t_torch, crop_kernel_TBps=gb / t_kernel)
    print(f"crops: {K} x 9 x {S} x {S} ({gb:.2f} GB fp32): kernel {t_kernel:.2f} ms ({gb / t_kernel:.2f} TB/s), "
          f"torch path {t_torch:.2f} ms")

    tr = BEVTrainer(m, device=dev)
    torch.cuda.reset_peak_memory_stats()
    t_step = timed(lambda: tr.train_bev(*batch, other_weight=0.5), args.reps, warmup=1)
    peak = torch.cuda.max_memory_allocated() / 1e9
    with torch.no_grad():
        probe = m(*[batch[i] for i in (0, 1, 5, 6, 3, 7)])
    n_other = probe[0].shape[0]
    res.update(step_ms=t_step, peak_GB=peak, vehicle_crops=n_other)
    print(f"train_bev step: {t_step:.1f} ms ({B / t_step * 1e3:.0f} samples/s), {n_other} vehicle crops + {B} ego crops, "
          f"peak {peak:.1f} GB")

    crops_other = out[:n_other].clone()
    crops_ego = out[:B].clone()
    t_crops = timed(lambda: (ops.crop_bilinear_u8(bev, frame[:n_other], theta[:n_other], S),
                             ops.crop_bilinear_u8(bev, frame[:B], theta[:B], S)), args.reps)

    def embed():
        e1 = m.bev_conv_emb(crops_other)
        e2 = m.bev_conv_emb(crops_ego)
        (e1.sum() + e2.sum()).backward()
    t_embed = timed(embed, args.reps, warmup=1)
    emb_o = torch.randn(n_other, 512, device=dev, requires_grad=True)
    emb_e = torch.randn(B, 512, device=dev, requires_grad=True)

    def grus():
        oc = m.cast(emb_o)
        ec = m.cast(emb_e)
        ep = m.plan(emb_e, nxps, cast_locs=ec, pixels_per_meter=4, crop_size=S)
        (oc.sum() + ec.sum() + ep.sum()).backward()
    t_gru = timed(grus, args.reps, warmup=1)
    t_adam = timed(lambda: tr.optim.step(), args.reps)
    res.update(part_crops_ms=t_crops, part_embedder_fwd_bwd_ms=t_embed, part_grus_fwd_bwd_ms=t_gru, part_adam_ms=t_adam)
    print(f"parts: crops {t_crops:.2f} ms, embedder fwd+bwd {t_embed:.1f} ms, GRUs fwd+bwd {t_gru:.1f} ms, Adam {t_adam:.2f} ms")
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
