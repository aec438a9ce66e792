"""Score LiDAR and planner checkpoints on a held-out recording: the comparisons LAV.train_lidar draws for wandb
(lav/lav_final_v2.py:226-258) — predicted BEV against the recorded one, detections against the recorded actors, the ego plan
against the expert's future — as numbers over every sample of the recording, through the agent's eval-mode inference path.

    python -m lav_b200.evaluate --config-path config_v2.yaml --data-dir VALDIR --lidar-weights lidar_7.th \
        --uniplanner-weights uniplanner_7.th [--batch-size 32] [--precision f16|fp32] [--num-workers 16] [--json out.json]

Every sample is taken once, in index order, unaugmented (TemporalBatchLoader's ordered mode); the last batch may be short.  Per
batch, InferModel.forward_batch runs the models and one ops.eval_batch launch scores its outputs; the one device-to-host copy
is that launch's result buffer.  The host sums the counts and computes AP over the whole recording.

Metrics:
  bev_iou[c]      intersection / union of (pred > 0.5, gt != 0) over all pixels of BEV channel c (null without any union)
  det[cls].ap[t]  all-point-interpolated AP of class cls (pedestrian, vehicle) at centre distance t metres: the surviving
                  detections of the recording sorted by descending score (ties keep sample order, then column order), the
                  precision envelope summed over the recall steps; null for a class with no actor in the window; "mean" is the
                  mean over the thresholds
  plan            ADE (mean over the steps of the Euclidean error) and FDE (error at the last step) in metres, over all samples
                  and per recorded command
"""
import argparse
import json

import numpy as np
import torch

from . import ops
from .agent import infer_model, math_mode
from .datasets import TemporalBatchLoader, TemporalLiDARPaintedDataset

CLASSES = ("pedestrian", "vehicle")


def average_precision(scores, matched, n_gt):
    """all-point-interpolated AP of detections (scores, matched flags) against n_gt ground-truth objects; None when n_gt is 0."""
    if n_gt == 0:
        return None
    order = np.argsort(-np.asarray(scores, np.float64), kind="stable")
    tp = np.cumsum(np.asarray(matched, bool)[order])
    precision = tp / np.arange(1, len(tp) + 1)
    recall = tp / n_gt
    envelope = np.maximum.accumulate(precision[::-1])[::-1]
    return float((envelope * np.diff(np.concatenate([[0.0], recall]))).sum())


class Scores:
    """host accumulation of eval_batch results over a recording."""

    def __init__(self):
        self.iou = np.zeros((3, 2), np.int64)
        self.ngt = np.zeros(2, np.int64)
        self.det = [[] for _ in CLASSES]             # per class: (score, flags) arrays of the surviving detections, in order
        self.ade, self.fde, self.cmd = [], [], []

    def add(self, v, cmds):
        """v = ops.eval_views of a host copy of one batch's result buffer; cmds (B,) the recorded commands."""
        self.iou += v["iou"].numpy().sum(0)
        self.ngt += v["ngt"].numpy().sum(0)
        score, flags = v["score"].numpy(), v["flags"].numpy()
        n_det = score.shape[1] // 2
        for c in range(2):
            s, f = score[:, c * n_det:(c + 1) * n_det], flags[:, c * n_det:(c + 1) * n_det]
            keep = (f & 16) != 0
            self.det[c].append((s[keep], f[keep]))
        pe = v["plan_err"].numpy()
        self.ade += pe[:, 0].tolist()
        self.fde += pe[:, 1].tolist()
        self.cmd += [int(c) for c in cmds]

    def summary(self):
        inter, union = self.iou[:, 0], self.iou[:, 1]
        det = {}
        for c, name in enumerate(CLASSES):
            s = np.concatenate([a for a, _ in self.det[c]] or [np.zeros(0, np.float32)])
            f = np.concatenate([b for _, b in self.det[c]] or [np.zeros(0, np.int32)])
            aps = {f"{t:g}": average_precision(s, (f >> k) & 1, int(self.ngt[c])) for k, t in enumerate(ops.EVAL_THRESHOLDS_M)}
            aps["mean"] = None if self.ngt[c] == 0 else float(np.mean(list(aps.values())))
            det[name] = dict(ap=aps, n_gt=int(self.ngt[c]), n_det=int(len(s)))
        ade, fde, cmd = np.array(self.ade), np.array(self.fde), np.array(self.cmd, np.int64)
        plan = dict(ade=float(ade.mean()) if len(ade) else None, fde=float(fde.mean()) if len(fde) else None,
                    per_cmd={str(c): dict(samples=int((cmd == c).sum()), ade=float(ade[cmd == c].mean()), fde=float(fde[cmd == c].mean()))
                             for c in sorted(set(cmd.tolist()))})
        return dict(samples=len(self.ade), bev_iou=[float(i) / float(u) if u else None for i, u in zip(inter, union)],
                    bev_counts=self.iou.tolist(), det=det, plan=plan)


@torch.no_grad()
def evaluate(lidar_model, uniplanner, dataset, batch_size=32, precision="f16", num_workers=16):
    """Scores of ``lidar_model`` and ``uniplanner`` over every sample of ``dataset`` (a TemporalLiDARPaintedDataset), the models
    run as the agent runs them at ``precision``.  -> dict (see the module docstring)."""
    dev = dataset.device
    lidar_model.to(dev).eval()
    uniplanner.to(dev).eval()
    im = infer_model(lidar_model, uniplanner, precision, dataset.camera_x, dataset.camera_z, dev)
    grid = dict(min_x=dataset.min_x, max_x=dataset.max_x, min_y=dataset.min_y, max_y=dataset.max_y,
                pixels_per_meter=dataset.pixels_per_meter)
    loader = TemporalBatchLoader(dataset, batch_size, drop_last=False, num_workers=num_workers, ordered=True)
    scores = Scores()
    with math_mode(precision):
        for batch, staged in loader.staged_batches():
            lidars, num_points, bev, ego_locs, cmds, nxps = batch[0], batch[1], batch[5], batch[6], batch[7], batch[8]
            out = im.forward_batch(lidars, num_points, nxps, cmds)
            res = ops.eval_batch(out["pred_bev"].permute(0, 2, 3, 1), bev, out["packed"], staged["actors"].to(dev, non_blocking=True),
                                 staged["offsets"], out["ego_plan_locs"].float().contiguous(), ego_locs, grid)
            scores.add(ops.eval_views(res.cpu(), len(num_points), out["packed"].shape[2]), staged["labels"]["cmd"].numpy())
    result = scores.summary()
    result["precision"] = precision
    return result


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--config-path", default="config_v2.yaml")
    ap.add_argument("--data-dir", required=True, help="the held-out recording (replaces the YAML's data_dir)")
    ap.add_argument("--lidar-weights", required=True)
    ap.add_argument("--uniplanner-weights", required=True)
    ap.add_argument("--batch-size", type=int, default=32)
    ap.add_argument("--precision", default="f16", choices=["f16", "fp32"])
    ap.add_argument("--num-workers", type=int, default=16, help="host threads of the loader (record reads, PNG chunk walks)")
    ap.add_argument("--json", default=None, help="also write the result here")
    return ap.parse_args(argv)


def format_result(r):
    fmt = lambda v: "n/a" if v is None else f"{v:.4f}"
    lines = [f"{r['samples']} samples, precision {r['precision']}",
             "BEV IoU per channel: " + " ".join(fmt(v) for v in r["bev_iou"])]
    for name, d in r["det"].items():
        lines.append(f"{name} AP ({d['n_gt']} GT, {d['n_det']} detections): " + " ".join(f"{k}={fmt(v)}" for k, v in d["ap"].items()))
    p = r["plan"]
    lines.append(f"plan ADE {fmt(p['ade'])} m, FDE {fmt(p['fde'])} m")
    lines += [f"  cmd {c}: {d['samples']} samples, ADE {fmt(d['ade'])} m, FDE {fmt(d['fde'])} m" for c, d in p["per_cmd"].items()]
    return "\n".join(lines)


def main(argv=None):
    import yaml
    from .train_full import make_models
    args = parse_args(argv)
    with open(args.config_path) as f:
        cfg = yaml.safe_load(f)
    dev = torch.device("cuda")
    # inference never runs the nested BEVPlanner: a freshly initialised one fills its place, and no bev_model_dir is read
    lid, _, uni = make_models(cfg)
    lid.load_state_dict(torch.load(args.lidar_weights, map_location="cpu"))
    uni.load_state_dict(torch.load(args.uniplanner_weights, map_location="cpu"))
    ds = TemporalLiDARPaintedDataset(args.config_path, device=dev, overrides=dict(data_dir=args.data_dir))
    result = evaluate(lid, uni, ds, args.batch_size, args.precision, args.num_workers)
    print(format_result(result))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)
    return result


if __name__ == "__main__":
    main()
