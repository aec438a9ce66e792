"""Score the point painting on a held-out recording: the class each LiDAR point is painted with, by a segmentation checkpoint run
as the agent runs it (online) and / or as a recording's lidar_sem rows hold it (stored), against the recorded semantic cameras
at the pixel the point hits.  The reference has no such numbers: data_paint (lav/data_paint.py:44-107) writes the rows and
nothing checks them.

    python -m lav_b200.evaluate_paint --config-path config_v2.yaml --data-dir VALDIR [--seg-weights seg_1.th] [--stored] \
        [--batch-size 32] [--precision f16|fp32] [--num-workers 16] [--json out.json]

At least one of --seg-weights and --stored is given; only the keys the run needs are read.

Samples.  The frames of the recording as BasicDataset lists them (index_trajectories: the n - num_plan frames of each
  trajectory), in order, unaugmented, through datasets.PaintDataset and CameraBatchLoader; the last batch may be short.
Points.  Every row of the recorded sweep lidar_%05d, in record order.  A row with a NaN x, y or z is counted (nan) and scored
  nowhere.  A row is roof when data_pipeline.roof_keep drops it (the training loader's roof filter) and in window when it is not
  roof and lies inside the pillar grid's [min_x, max_x) x [min_y, max_y), tested as the voxeliser tests it (pillar_grid.cuh:
  in_window, which pillar.cu's locate calls).  Roof points are scored, outside the window.
Cameras.  The painting cameras: point_painting.make_converters(camera_x, camera_z) with CAMERA_YAWS (-60, 0, 60) and the records
  rgb_{c} / sem_{c} for c = 0 .. 2, what data_paint and the agent paint with.  config_v2.yaml's camera_yaws lists five cameras
  (the ones evaluate_rgb scores); the painting uses three, and this module does not take the config's list.
Visibility.  project_hit (project_hit.cuh), the projection every painting kernel runs: the last camera whose truncated pixel lies
  inside the 288 x 256 image wins.  A point no camera sees is counted (not_visible) and scored nowhere; its painted row is zero.
Ground truth.  The hit camera's recorded tag at the hit pixel, sem_c[v, u], through ops.sem_class_table(seg_channels) (filter_sem
  as a table): classes 0 .. C - 1, 0 the background.
Online prediction.  ERFNet at ``precision`` (set_precision) on the painting cameras' uint8 frames, forward_features_nhwc, then
  the hit pixel's logits through deconv_logits.cuh, the chain paint_deconv_kernel and seg_confusion_kernel share; the class is
  the first index of the largest logit (ties to the lower class); a NaN logit makes the point invalid.
Stored prediction.  The class the lidar_sem row encodes: the row holds s_k = p_k (1 - p_0), k = 1 .. C - 1, so sum s_k =
  (1 - p_0)^2; decoded in fp64 without contraction, q = sqrt(sum s_k), p_0 = 1 - q, p_k = s_k / q, the first index of the
  largest of (p_0, p_1, ...); a row summing to 0 (all zero: the point was not seen when painted) is class 0; a NaN entering the
  decode makes the point stored-invalid.  A frame whose lidar_sem is missing or does not hold the sweep's rows x (C - 1)
  floats counts in mismatched_frames and is left out of the stored scores.
Counts.  One ops.paint_confusion launch per batch and one copy of its int32 counts: confusion [recorded][predicted] per source,
  hit camera, range bin (horizontal distance sqrt(x^2 + y^2) in fp32, [0, 10), [10, 20), [20, 40), [40, inf) m) and window
  flag; agreement [online][stored] per camera over the points both sources score; the counters of ops.PAINT_COUNTERS.  All
  integers, so the result does not depend on the schedule.

Metrics.  For each scored source: evaluate_rgb.seg_metrics (IoU, mIoU, foreground mIoU, accuracy, precision and recall per class;
  its invalid_pixels are invalid points) over all visible points, over the in-window points, per range bin and per camera.
  points (the counters), coverage = the share of in-window points a camera sees, agreement (rate = trace / total, confusion)
  with both sources, mismatched_frames with --stored, classes (0, then the seg_channels tags), precision and samples (frames).
"""
import argparse
import json

import numpy as np
import torch

from . import ops
from .agent import math_mode
from .datasets import CameraBatchLoader, PaintDataset
from .evaluate_rgb import seg_metrics

RANGE_NAMES = ("0-10m", "10-20m", "20-40m", "40m+")


class PaintScores:
    """host accumulation of paint_confusion results over a recording."""

    def __init__(self, ncam, n_classes, online, stored):
        self.ncam, self.c, self.online, self.stored = ncam, n_classes, online, stored
        self.counters = np.zeros(len(ops.PAINT_COUNTERS), np.int64)
        shape = (ncam, len(RANGE_NAMES), 2, n_classes, n_classes)
        self.conf = {s: np.zeros(shape, np.int64) for s, on in (("online", online), ("stored", stored)) if on}
        self.agreement = np.zeros((ncam, n_classes, n_classes), np.int64)
        self.mismatched_frames = 0
        self.frames = 0

    def add(self, counts, meta):
        """counts (B, L) int32 and meta (B, 2) int32, host copies of one batch's paint_confusion result and its frame table."""
        v = ops.paint_confusion_views(np.asarray(counts, np.int64), self.ncam, self.c, self.online, self.stored)
        self.counters += v["counters"].sum(0)
        for s in self.conf:
            self.conf[s] += v[s].sum(0)
        if "agreement" in v:
            self.agreement += v["agreement"].sum(0)
        self.frames += len(counts)
        if self.stored:
            self.mismatched_frames += int((np.asarray(meta)[:, 1] == 0).sum())

    def summary(self, classes):
        cnt = dict(zip(ops.PAINT_COUNTERS, (int(x) for x in self.counters)))
        out = dict(classes=list(classes), points=cnt)
        in_win = cnt["in_window"]
        out["coverage"] = (in_win - cnt["not_visible_in_window"]) / in_win if in_win else None
        for s, conf in self.conf.items():
            invalid = cnt["invalid" if s == "online" else "stored_invalid"]
            out[s] = dict(seg_metrics(conf.sum((0, 1, 2)), invalid), in_window=seg_metrics(conf[:, :, 1].sum((0, 1))),
                          per_range={r: seg_metrics(conf[:, k].sum((0, 1))) for k, r in enumerate(RANGE_NAMES)},
                          per_camera=[seg_metrics(cf.sum((0, 1))) for cf in conf])
        if self.online and self.stored:
            total = int(self.agreement.sum())
            out["agreement"] = dict(rate=float(np.trace(self.agreement.sum(0))) / total if total else None,
                                    confusion=self.agreement.sum(0).tolist(), per_camera=[a.tolist() for a in self.agreement])
        if self.stored:
            out["mismatched_frames"] = self.mismatched_frames
        return out


@torch.no_grad()
def evaluate_paint(seg_model, dataset, batch_size=32, precision="f16", num_workers=16, on_batch=None):
    """Scores of the painting over every frame of ``dataset`` (a PaintDataset): online with ``seg_model`` at ``precision`` when it
    is given (the dataset then loads the colour images), stored when the dataset loads lidar_sem.  ``on_batch(batch, feat,
    counts)`` (tests) sees each batch's device inputs, the features it scored (or None) and the host copy of its counts.
    -> dict (see the module docstring)."""
    online = seg_model is not None
    if not (online or dataset.stored):
        raise ValueError("evaluate_paint: nothing to score (no seg model and no stored rows)")
    if online and not dataset.online:
        raise ValueError("evaluate_paint: the dataset does not load the colour images the seg model needs")
    dev = dataset.device
    ncam, c = len(dataset.cams), dataset.n_classes
    if online:
        seg_model.to(dev).eval().set_precision(precision)
        if seg_model.erfnet.decoder.output_conv.out_channels != c:
            raise ValueError(f"evaluate_paint: the seg model has {seg_model.erfnet.decoder.output_conv.out_channels} classes, "
                             f"seg_channels gives {c}")
    scores = PaintScores(ncam, c, online, dataset.stored)
    lut = ops.sem_class_table(dataset.seg_channels)
    cams = np.stack([cv.packed() for cv in dataset.converters])
    loader = CameraBatchLoader(dataset, batch_size, num_workers=num_workers)
    with math_mode(precision):
        for batch, staged in loader.staged_batches():
            labels = batch["labels"]
            B, _, H, W = labels.shape
            feat = table = None
            if online:
                feat, table, _ = seg_model.forward_features_nhwc(batch["rgbs"].view(B * ncam, H, W, 3))
            counts = ops.paint_confusion(batch["points"], labels.view(B * ncam, H, W), lut, cams, dataset.window, c, feat=feat,
                                         table=table, stored=batch.get("stored"), meta=batch["meta"]).cpu().numpy()
            scores.add(counts, staged["meta"].numpy())
            if on_batch is not None:
                on_batch(batch, feat, counts)
    return dict(scores.summary([0] + [int(t) for t in dataset.seg_channels]), precision=precision if online else None,
                samples=scores.frames)


def format_result(r):
    fmt = lambda v: "n/a" if v is None else f"{v:.4f}"
    p = r["points"]
    lines = [f"{r['samples']} frames, {p['points']} points: {p['nan']} NaN, {p['roof']} roof, {p['in_window']} in window, "
             f"{p['not_visible']} seen by no camera; coverage of the window {fmt(r['coverage'])}"]
    for s in ("online", "stored"):
        if s in r:
            d = r[s]
            lines.append(f"{s} (classes {r['classes']}): mIoU {fmt(d['miou'])}, foreground mIoU {fmt(d['miou_fg'])}, accuracy "
                         f"{fmt(d['pixel_accuracy'])}, {d['invalid_pixels']} invalid points; in window mIoU "
                         f"{fmt(d['in_window']['miou'])}")
            lines.append("  IoU per class: " + " ".join(fmt(v) for v in d["iou"]))
            lines.append("  by range: " + ", ".join(f"{k} mIoU {fmt(m['miou'])}" for k, m in d["per_range"].items()))
            lines.append("  by camera: " + ", ".join(f"{k} mIoU {fmt(m['miou'])}" for k, m in enumerate(d["per_camera"])))
    if "agreement" in r:
        lines.append(f"online / stored agreement {fmt(r['agreement']['rate'])}")
    if "mismatched_frames" in r:
        lines.append(f"{r['mismatched_frames']} frames without matching lidar_sem rows (left out of the stored scores)")
    return "\n".join(lines)


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--config-path", default="config_v2.yaml")
    ap.add_argument("--data-dir", required=True, help="the held-out recording (replaces the YAML's data_dir)")
    ap.add_argument("--seg-weights", default=None, help="RGBSegmentationModel weights (seg_1.th): score its online painting")
    ap.add_argument("--stored", action="store_true", help="score the recording's lidar_sem rows")
    ap.add_argument("--batch-size", type=int, default=32)
    ap.add_argument("--precision", default="f16", choices=["f16", "fp32"])
    ap.add_argument("--num-workers", type=int, default=16, help="host threads of the loader (record reads, image decodes)")
    ap.add_argument("--json", default=None, help="also write the result here")
    args = ap.parse_args(argv)
    if args.seg_weights is None and not args.stored:
        ap.error("give --seg-weights, --stored or both")
    return args


def main(argv=None):
    import yaml
    from .rgb import RGBSegmentationModel
    args = parse_args(argv)
    with open(args.config_path) as f:
        cfg = yaml.safe_load(f)
    seg = None
    if args.seg_weights:
        seg = RGBSegmentationModel(cfg["seg_channels"])
        seg.load_state_dict(torch.load(args.seg_weights, map_location="cpu"))
    ds = PaintDataset(args.config_path, online=seg is not None, stored=args.stored, device=torch.device("cuda"),
                      overrides=dict(data_dir=args.data_dir))
    result = evaluate_paint(seg, ds, args.batch_size, args.precision, args.num_workers)
    print(format_result(result))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)
    return result


if __name__ == "__main__":
    main()
