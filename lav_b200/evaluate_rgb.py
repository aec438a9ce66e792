"""Score the camera models on a held-out recording: ERFNet (RGBSegmentationModel) against the recorded semantic camera images and
the brake classifier (RGBBrakePredictionModel) against the recorded brake labels, run as the agent runs them.  The reference has
no such numbers: train_seg / train_bra only log an argmax image (lav/lav_privileged_v2.py:162-216).

    python -m lav_b200.evaluate_rgb --config-path config_v2.yaml --data-dir VALDIR [--seg-weights seg_1.th] \
        [--bra-weights bra_v2_9.th] [--batch-size 32] [--precision f16|fp32] [--num-workers 16] [--json out.json]

At least one of the two weights files is given; only the keys its model needs are read.

Samples.  The frames of the recording as BasicDataset lists them (index_trajectories: the n - num_plan frames of each
  trajectory), in order, unaugmented, through datasets.CameraBatchLoader; the last batch may be short.  Images are decoded on the
  host as BasicDataset.load_img decodes them (cv2.imdecode; colour images flipped BGR -> RGB).
Segmentation.  Every (frame, camera) pair for cameras 0 .. len(camera_yaws) - 1, SegmentationDataset's samples.  Ground truth:
  the recorded tags sem_{c} through filter_sem(sem, seg_channels) as a table (ops.sem_class_table: an unlisted tag is class 0,
  the background; a later duplicate wins).  Prediction: the model at ``precision`` (set_precision) on the uint8 frames,
  forward_features_nhwc (the fused stem), then one ops.seg_confusion launch per batch over all B x ncam images: output_conv's
  logits computed as the painting gather computes them, the first index of the largest logit; a pixel with a NaN logit is
  invalid and counted apart.  Per batch one copy of the (B * ncam, C * C + 1) count buffer.
Brake.  Every frame, with the three middle cameras ncam//2 - 1 .. ncam//2 + 1 side by side and the telephoto view tel_rgb cut by
  [:-crop_tel_bottom] (BrakePredictionDataset).  The model is agent.brake_model's private copy at ``precision``, called through
  agent.brake_probs as the agent calls it: forward_u8 on the uint8 frames at f16, the float model under math_mode("fp32") at
  fp32.  Per batch one copy of the (B,) probabilities.

Metrics.
  seg, overall and per camera: confusion (C x C, [recorded class][predicted class], int64 over the recording); iou[k] =
    TP / (TP + FP + FN), null when that union is empty; miou = mean over the non-null classes, miou_fg = the same over classes
    1 .. C-1 (null when none); pixel_accuracy = trace / total; per-class precision TP / (TP + FP) and recall TP / (TP + FN), null
    over an empty denominator; invalid_pixels.  classes = the seg_channels tags, with 0 for the background.
  brake: frames, positives; ap = evaluate.average_precision ranked by probability (ties keep frame order) against the
    positives; at the agent's rule p > 0.1 (strictly, compared in fp64 as float(pred_bra) > 0.1) and at p > 0.5: precision,
    recall, accuracy and false_brake_rate (the share of frames without a recorded brake on which it fires), null over an empty
    denominator; bce = mean binary cross-entropy in fp64, each log clamped at -100 as F.binary_cross_entropy clamps it.
  precision (the compute path) and samples (frames).
"""
import argparse
import json

import numpy as np
import torch

from . import ops
from .agent import brake_model, brake_probs, math_mode
from .datasets import CameraBatchLoader, CameraDataset
from .evaluate import average_precision

BRAKE_THRESHOLDS = (0.1, 0.5)       # the agent's rule (lav_agent_fast.py:340-341), and the classifier's midpoint


def seg_metrics(conf, invalid=0):
    """the seg metrics of one confusion matrix (C x C, [recorded][predicted])."""
    conf = np.asarray(conf, np.int64)
    tp = np.diag(conf)
    fp, fn = conf.sum(0) - tp, conf.sum(1) - tp
    ratio = lambda a, b: [float(x) / float(y) if y else None for x, y in zip(a, b)]
    iou = ratio(tp, tp + fp + fn)
    mean = lambda v: float(np.mean([x for x in v if x is not None])) if any(x is not None for x in v) else None
    total = int(conf.sum())
    return dict(confusion=conf.tolist(), iou=iou, miou=mean(iou), miou_fg=mean(iou[1:]),
                pixel_accuracy=float(tp.sum()) / total if total else None, precision=ratio(tp, tp + fp), recall=ratio(tp, tp + fn),
                invalid_pixels=int(invalid))


class SegScores:
    """host accumulation of seg_confusion results over a recording, per camera."""

    def __init__(self, n_classes, n_cams):
        self.c = n_classes
        self.conf = np.zeros((n_cams, n_classes, n_classes), np.int64)
        self.invalid = np.zeros(n_cams, np.int64)

    def add(self, counts):
        """counts (B * ncam, C * C + 1) int32, a host copy of one batch's seg_confusion result, frame-major."""
        c = self.c
        counts = np.asarray(counts, np.int64).reshape(-1, self.conf.shape[0], c * c + 1)
        self.conf += counts[..., :c * c].sum(0).reshape(-1, c, c)
        self.invalid += counts[..., c * c].sum(0)

    def summary(self, classes):
        return dict(seg_metrics(self.conf.sum(0), self.invalid.sum()), classes=list(classes),
                    per_camera=[seg_metrics(cf, iv) for cf, iv in zip(self.conf, self.invalid)])


def brake_metrics(probs, labels):
    """the brake metrics of probabilities ``probs`` (the model's fp32, widened exactly) against the recorded labels (0 / 1)."""
    p = np.asarray(probs).astype(np.float64)
    y = np.asarray(labels, np.int64) != 0
    n, pos = len(y), int(y.sum())
    div = lambda a, b: float(a) / float(b) if b else None

    def rule(t):
        fire = p > t
        tp, fp = int((fire & y).sum()), int((fire & ~y).sum())
        return dict(precision=div(tp, tp + fp), recall=div(tp, pos), accuracy=div(int((fire == y).sum()), n),
                    false_brake_rate=div(fp, n - pos))
    with np.errstate(divide="ignore"):
        bce = -(np.where(y, np.maximum(np.log(p), -100.0), 0.0) + np.where(y, 0.0, np.maximum(np.log(1.0 - p), -100.0)))
    return dict(frames=n, positives=pos, ap=average_precision(p, y, pos), **{f"at_{t:g}": rule(t) for t in BRAKE_THRESHOLDS},
                bce=float(bce.mean()) if n else None)


@torch.no_grad()
def evaluate_rgb(seg_model, bra_model, dataset, batch_size=32, precision="f16", num_workers=16, on_batch=None):
    """Scores of ``seg_model`` and / or ``bra_model`` (either may be None) over every frame of ``dataset`` (a CameraDataset loading
    what they need), run as the agent runs them at ``precision``.  ``on_batch(batch, feat, counts, probs)`` (tests) sees each
    batch's device inputs, the features it scored and the host copies of its results.  -> dict (see the module docstring)."""
    if seg_model is None and bra_model is None:
        raise ValueError("evaluate_rgb: no model to score")
    dev = dataset.device
    ncam = len(dataset.cams)
    seg = bra = None
    if seg_model is not None:
        seg_model.to(dev).eval().set_precision(precision)
        n_classes = seg_model.erfnet.decoder.output_conv.out_channels
        seg = SegScores(n_classes, ncam)
        lut = ops.sem_class_table(dataset.seg_channels)
    if bra_model is not None:
        bra_copy = brake_model(bra_model.to(dev).eval(), precision)
        probs, labels = [], []
    frames = 0
    loader = CameraBatchLoader(dataset, batch_size, num_workers=num_workers)
    with math_mode(precision):
        for batch, _ in loader.staged_batches():
            rgbs = batch["rgbs"]
            B, _, H, W, _ = rgbs.shape
            frames += B
            feat = counts = p = None
            if seg is not None:
                feat, table, _ = seg_model.forward_features_nhwc(rgbs.view(B * ncam, H, W, 3))
                counts = ops.seg_confusion(feat, table, batch["labels"].view(B * ncam, H, W), lut, n_classes).cpu().numpy()
                seg.add(counts)
            if bra_model is not None:
                cams = rgbs[:, dataset.brake_cams]
                p = brake_probs(bra_copy, cams.contiguous(), batch["tel"]).float().cpu().numpy()
                probs.append(p)
                labels.append(batch["bra"].cpu().numpy())
            if on_batch is not None:
                on_batch(batch, feat, counts, p)
    result = dict(precision=precision, samples=frames)
    if seg is not None:
        result["seg"] = seg.summary([0] + [int(t) for t in dataset.seg_channels])
    if bra_model is not None:
        result["brake"] = brake_metrics(np.concatenate(probs) if probs else np.zeros(0, np.float32),
                                        np.concatenate(labels) if labels else np.zeros(0, np.int64))
    return result


def format_result(r):
    fmt = lambda v: "n/a" if v is None else f"{v:.4f}"
    lines = [f"{r['samples']} frames, precision {r['precision']}"]
    if "seg" in r:
        s = r["seg"]
        lines.append(f"segmentation (classes {s['classes']}): mIoU {fmt(s['miou'])}, foreground mIoU {fmt(s['miou_fg'])}, pixel "
                     f"accuracy {fmt(s['pixel_accuracy'])}, {s['invalid_pixels']} invalid pixels")
        lines.append("  IoU per class: " + " ".join(fmt(v) for v in s["iou"]))
        lines += [f"  camera {c}: mIoU {fmt(d['miou'])}, foreground mIoU {fmt(d['miou_fg'])}, pixel accuracy "
                  f"{fmt(d['pixel_accuracy'])}" for c, d in enumerate(s["per_camera"])]
    if "brake" in r:
        b = r["brake"]
        lines.append(f"brake ({b['frames']} frames, {b['positives']} braking): AP {fmt(b['ap'])}, BCE {fmt(b['bce'])}")
        for t in BRAKE_THRESHOLDS:
            d = b[f"at_{t:g}"]
            lines.append(f"  p > {t:g}: precision {fmt(d['precision'])}, recall {fmt(d['recall'])}, accuracy {fmt(d['accuracy'])}, "
                         f"false brake rate {fmt(d['false_brake_rate'])}")
    return "\n".join(lines)


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--config-path", default="config_v2.yaml")
    ap.add_argument("--data-dir", required=True, help="the held-out recording (replaces the YAML's data_dir)")
    ap.add_argument("--seg-weights", default=None, help="RGBSegmentationModel weights (seg_1.th)")
    ap.add_argument("--bra-weights", default=None, help="RGBBrakePredictionModel weights (bra_v2_9.th)")
    ap.add_argument("--batch-size", type=int, default=32)
    ap.add_argument("--precision", default="f16", choices=["f16", "fp32"])
    ap.add_argument("--num-workers", type=int, default=16, help="host threads of the loader (record reads, image decodes)")
    ap.add_argument("--json", default=None, help="also write the result here")
    args = ap.parse_args(argv)
    if args.seg_weights is None and args.bra_weights is None:
        ap.error("give --seg-weights, --bra-weights or both")
    return args


def main(argv=None):
    import yaml
    from .heads import RGBBrakePredictionModel
    from .rgb import RGBSegmentationModel
    args = parse_args(argv)
    with open(args.config_path) as f:
        cfg = yaml.safe_load(f)
    dev = torch.device("cuda")
    seg = bra = None
    if args.seg_weights:
        seg = RGBSegmentationModel(cfg["seg_channels"])
        seg.load_state_dict(torch.load(args.seg_weights, map_location="cpu"))
    if args.bra_weights:
        bra = RGBBrakePredictionModel(cfg["seg_channels"])
        bra.load_state_dict(torch.load(args.bra_weights, map_location="cpu"))
    ds = CameraDataset(args.config_path, seg=seg is not None, brake=bra is not None, device=dev,
                       overrides=dict(data_dir=args.data_dir))
    result = evaluate_rgb(seg, bra, ds, args.batch_size, args.precision, args.num_workers)
    print(format_result(result))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)
    return result


if __name__ == "__main__":
    main()
