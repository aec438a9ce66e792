"""Train the LiDAR perception model and the UniPlanner student from a recording — lav/train_full_v2.py with lav/lav_final_v2.py's
model set-up (:26-89) on LAVTrainer and the device-side TemporalLiDARPaintedDataset (lav_b200/datasets.py).

    python -m lav_b200.train_full --config-path config_v2.yaml [--perceive-only | --motion-only] [--batch-size 32]
    torchrun --nproc-per-node 8 -m lav_b200.train_full --config-path config_v2.yaml

One process per GPU (NCCL, LOCAL_RANK) instead of nn.DataParallel; --batch-size is per rank.  StepLR steps once per epoch;
rank 0 writes lidar_{epoch}.th and uniplanner_{epoch}.th (plain state_dicts, the reference's keys) to --save-dir.
"""
import argparse
import os
import time
from types import SimpleNamespace

import torch
import torch.distributed as dist
import yaml

from .datasets import get_data_loader
from .heads import BEVPlanner, UniPlanner
from .lidar import LiDARModel
from .train import LAVTrainer


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--config-path", default="config_v2.yaml")
    ap.add_argument("--perceive-only", action="store_true")
    ap.add_argument("--motion-only", action="store_true")
    ap.add_argument("--num-epoch", type=int, default=64)
    ap.add_argument("--num-per-log", type=int, default=100, help="print the losses every N steps")
    ap.add_argument("--num-per-save", type=int, default=1, help="save every N epochs")
    ap.add_argument("--batch-size", type=int, default=32, help="samples per GPU (per rank under torchrun), as bench.py --train-batch")
    ap.add_argument("--lr", type=float, default=3e-4)
    ap.add_argument("--seed", type=int, default=2021)
    ap.add_argument("--save-dir", default=".", help="directory of the checkpoints")
    ap.add_argument("--max-steps", type=int, default=0, help="stop after this many steps (0 = run every epoch)")
    ap.add_argument("--num-workers", type=int, default=16, help="host threads of the loader (record reads, PNG decodes)")
    args = ap.parse_args(argv)
    if args.perceive_only and args.motion_only:
        ap.error("--perceive-only and --motion-only exclude each other")
    return args


def make_models(cfg):
    """LAV.__init__'s models (lav_final_v2.py:31-72), freshly initialised: (LiDARModel, BEVPlanner teacher, UniPlanner student
    holding that teacher)."""
    if not cfg.get("point_painting", True):
        raise NotImplementedError("only the point-painted LiDAR model (point_painting: True) is provided")
    lid = LiDARModel(num_input=len(cfg["seg_channels"]) + cfg["num_frame_stack"] + 10, num_features=cfg["num_features"],
                     backbone=cfg["backbone"], min_x=cfg["min_x"], max_x=cfg["max_x"], min_y=cfg["min_y"], max_y=cfg["max_y"],
                     pixels_per_meter=cfg["pixels_per_meter"])
    kw = dict(pixels_per_meter=cfg["pixels_per_meter"], crop_size=cfg["crop_size"], feature_x_jitter=cfg["feature_x_jitter"],
              feature_angle_jitter=cfg["feature_angle_jitter"], x_offset=0,
              y_offset=1 + cfg["min_x"] / ((cfg["max_x"] - cfg["min_x"]) / 2), num_cmds=cfg["num_cmds"], num_plan=cfg["num_plan"],
              num_plan_iter=cfg["num_plan_iter"])
    bev = BEVPlanner(num_frame_stack=cfg["num_frame_stack"], **kw)
    return lid, bev, UniPlanner(bev, num_input_feature=cfg["num_features"][-1] * 6, **kw)


def build_models(cfg, perceive_only=False, motion_only=False):
    """make_models with lidar_model_dir / bev_model_dir / uniplanner_dir loaded as the reference loads them."""
    lid, bev, uni = make_models(cfg)
    if not perceive_only:
        lid.load_state_dict(torch.load(cfg["lidar_model_dir"], map_location="cpu"))
    bev.load_state_dict(torch.load(cfg["bev_model_dir"], map_location="cpu"))
    bev.eval()
    if not perceive_only and not motion_only:
        uni.load_state_dict(torch.load(cfg["uniplanner_dir"], map_location="cpu"))
    return lid, uni


def main(argv=None):
    args = parse_args(argv)
    with open(args.config_path) as f:
        cfg = yaml.safe_load(f)
    rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    torch.manual_seed(args.seed)
    lid, uni = build_models(cfg, args.perceive_only, args.motion_only)
    weights = {k: cfg[k] for k in ("box_weight", "ori_weight", "seg_weight", "perception_weight", "other_weight", "cmd_weight",
                                   "cmd_smooth", "branch_weights") if k in cfg}
    tr = LAVTrainer(lid.to(dev), uni.to(dev), lr=args.lr, device=dev, distill=cfg.get("distill", True),
                    perceive_only=args.perceive_only, motion_only=args.motion_only, **weights)
    loader = get_data_loader("temporal_lidar_painted", SimpleNamespace(config_path=args.config_path, seed=args.seed,
                                                                      batch_size=args.batch_size, rank=rank, world_size=world,
                                                                      device=dev, num_workers=args.num_workers))
    if rank == 0:
        print(f"{len(loader.ds)} samples, {len(loader)} steps per epoch per rank, {world} rank(s) x {args.batch_size}")
        os.makedirs(args.save_dir, exist_ok=True)
    step, t0 = 0, time.time()
    for epoch in range(args.num_epoch):
        for batch in loader:
            loss, parts = tr.train_lidar(*batch)
            if rank == 0 and step % args.num_per_log == 0:
                terms = " ".join(f"{k}={float(v):.4f}" for k, v in parts.items())
                print(f"epoch {epoch} step {step} loss={float(loss):.4f} {terms} ({time.time() - t0:.1f} s)", flush=True)
            step += 1
            if args.max_steps and step >= args.max_steps:
                break
        tr.sched.step()
        stop = bool(args.max_steps) and step >= args.max_steps
        if rank == 0 and ((epoch + 1) % args.num_per_save == 0 or stop):
            for name, m in (("lidar", lid), ("uniplanner", uni)):
                path = os.path.join(args.save_dir, f"{name}_{epoch + 1}.th")
                torch.save({k: v.detach().cpu().contiguous() for k, v in m.state_dict().items()}, path)
                print(f"saved to {path}")
        if stop:
            break
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
