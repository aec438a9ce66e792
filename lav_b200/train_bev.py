"""Train the privileged BEV planner from a recording — stage 1 of the v2 recipe, lav/train_bev_v2.py with lav/lav_privileged_v2.py's
model set-up (:32-62) on BEVTrainer and the TemporalBEVDataset loader (lav_b200/datasets.py).

    python -m lav_b200.train_bev --config-path config_v2.yaml [--batch-size 256]
    torchrun --nproc-per-node 8 -m lav_b200.train_bev --config-path config_v2.yaml

One process per GPU (NCCL, LOCAL_RANK) instead of nn.DataParallel; --batch-size is per rank.  StepLR steps once per epoch;
rank 0 writes bev_{epoch}.th (a plain state_dict with the reference's keys) to --save-dir, usable as train_full's
bev_model_dir.  --weight-decay is accepted for command-line compatibility and NOT applied: the reference's bev_optim is built
without it (lav_privileged_v2.py:61).
"""
import argparse
import os
import time
from types import SimpleNamespace

import torch
import torch.distributed as dist
import yaml

from .datasets import get_data_loader
from .heads import BEVPlanner
from .train import BEVTrainer


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--config-path", default="config_v2.yaml")
    ap.add_argument("--num-epoch", type=int, default=160)
    ap.add_argument("--num-per-log", type=int, default=100, help="print the losses every N steps")
    ap.add_argument("--num-per-save", type=int, default=1, help="save every N epochs")
    ap.add_argument("--batch-size", type=int, default=256, help="samples per GPU (per rank under torchrun)")
    ap.add_argument("--lr", type=float, default=3e-4)
    ap.add_argument("--weight-decay", type=float, default=2e-4, help="accepted, not applied (as in the reference)")
    ap.add_argument("--num-workers", type=int, default=16, help="threads reading and decoding the records of a batch")
    ap.add_argument("--seed", type=int, default=2021)
    ap.add_argument("--save-dir", default=".", help="directory of the checkpoints")
    ap.add_argument("--max-steps", type=int, default=0, help="stop after this many steps (0 = run every epoch)")
    return ap.parse_args(argv)


def build_planner(cfg):
    """LAV.__init__'s BEVPlanner (lav_privileged_v2.py:32-42), freshly initialised."""
    return BEVPlanner(pixels_per_meter=cfg["pixels_per_meter"], crop_size=cfg["crop_size"], feature_x_jitter=cfg["feature_x_jitter"],
                      feature_angle_jitter=cfg["feature_angle_jitter"], x_offset=0,
                      y_offset=1 + cfg["min_x"] / ((cfg["max_x"] - cfg["min_x"]) / 2), num_cmds=cfg["num_cmds"],
                      num_plan=cfg["num_plan"], num_plan_iter=cfg["num_plan_iter"], num_frame_stack=cfg["num_frame_stack"])


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
    planner = build_planner(cfg).to(dev)
    weights = {k: cfg[k] for k in ("branch_weights", "cmd_weight", "cmd_smooth", "use_others_to_train") if k in cfg}
    tr = BEVTrainer(planner, lr=args.lr, device=dev, **weights)
    loader = get_data_loader("temporal_bev", SimpleNamespace(config_path=args.config_path, seed=args.seed, batch_size=args.batch_size,
                                                            rank=rank, world_size=world, device=dev, num_workers=args.num_workers))
    if rank == 0:
        print(f"{len(loader.ds)} samples, {len(loader)} steps per epoch per rank, {world} rank(s) x {args.batch_size}")
        os.makedirs(args.save_dir, exist_ok=True)
    step, t0 = 0, time.time()
    for epoch in range(args.num_epoch):
        for batch in loader:
            loss, parts = tr.train_bev(*batch, other_weight=tr.other_weight(step))
            if rank == 0 and step % args.num_per_log == 0:
                terms = " ".join(f"{k}={float(v):.4f}" for k, v in parts.items())
                print(f"epoch {epoch} step {step} loss={float(loss):.4f} {terms} ({time.time() - t0:.1f} s)", flush=True)
            step += 1
            if args.max_steps and step >= args.max_steps:
                break
        tr.sched.step()
        stop = bool(args.max_steps) and step >= args.max_steps
        if rank == 0 and ((epoch + 1) % args.num_per_save == 0 or stop):
            path = os.path.join(args.save_dir, f"bev_{epoch + 1}.th")
            torch.save({k: v.detach().cpu().contiguous() for k, v in planner.state_dict().items()}, path)
            print(f"saved to {path}")
        if stop:
            break
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
