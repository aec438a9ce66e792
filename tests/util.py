"""Shared builders for the tests: seeded weights (identical in the pin script) and inputs."""
import os

import numpy as np
import torch

from lav_b200 import synth

GRID = dict(min_x=-10, max_x=70, min_y=-40, max_y=40)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def lidar_model(device=None):
    from lav_b200.lidar import LiDARModel
    m = LiDARModel(num_input=16, num_features=[64, 64], backbone="cnn", pixels_per_meter=4, **GRID).eval()
    sd = synth.fill_state_dict_(m.state_dict())
    m.load_state_dict(sd)
    if device is not None:
        m = m.to(device)
    return m, {k: v.clone() for k, v in sd.items()}


def seg_model(device=None, real=False):
    from lav_b200.rgb import RGBSegmentationModel
    m = RGBSegmentationModel([4, 6, 7, 10]).eval()
    if real:
        sd = torch.load(os.path.join(ROOT, "oracle", "_ref", "seg_1.state_dict.pt"), map_location="cpu")
    else:
        sd = synth.fill_state_dict_(m.state_dict())
    m.load_state_dict(sd)
    if device is not None:
        m = m.to(device)
    return m, {k: v.clone() for k, v in sd.items()}


def have_real_seg():
    return os.path.exists(os.path.join(ROOT, "oracle", "_ref", "seg_1.state_dict.pt"))


def pillar_clouds():
    return [synth.stacked_lidar(2000, tag="pp0"), synth.stacked_lidar(1500, tag="pp1")]


def paint_inputs():
    gold = np.load(os.path.join(ROOT, "tests", "golden", "paint.npz"))
    lidar = torch.cat([synth.lidar_sweep(8192, tag="paint"), torch.from_numpy(gold["edge"])]).contiguous()
    return lidar, synth.sem_probs(tag="paint"), gold


def rel_err(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def crop_ref64(feats_nchw, frame_idx, theta, S, padding="zeros"):
    """lavb_crop_bilinear in float64: frame indices clamped to [0, B) as the kernel clamps them, then
    F.affine_grid(theta, align_corners=True) + F.grid_sample(bilinear, align_corners=True).  feats (B,C,H,W), frame_idx (K,),
    theta (K,2,3) -> (K,C,S,S) float64.  The bilinear weights are >= 0, so crop_ref64(|f|) is the per-element sum |w f| of
    the forward.  ``padding`` other than the kernel's "zeros" is for error bounds (tests/test_gpu_crop_contract.py)."""
    import torch.nn.functional as F
    B, C = feats_nchw.shape[:2]
    fi = frame_idx.long().cpu().clamp(0, B - 1)
    grid = F.affine_grid(theta.double().cpu(), [theta.shape[0], C, S, S], align_corners=True)
    return F.grid_sample(feats_nchw.double().cpu()[fi], grid, mode="bilinear", padding_mode=padding, align_corners=True)


def crop_ref64_adjoint(gout_nchw, frame_idx, theta, feat_shape):
    """the adjoint of crop_ref64 (the crop's gradient with respect to the (B,C,H,W) map) by float64 autograd through the same
    call: gout (K,C,S,S) -> (B,C,H,W) float64.  Applied to |gout| it gives the per-element sum |w g| of the backward."""
    f = torch.zeros(feat_shape, dtype=torch.float64, requires_grad=True)
    out = crop_ref64(f, frame_idx, theta, gout_nchw.shape[-1])
    return torch.autograd.grad(out, f, gout_nchw.double().cpu())[0]


def seg_logit_err(got_prob, ref_feats, sd):
    """error of the seg head measured BEFORE its sigmoid, as a fraction of the logit scale: the reference module returns
    sigmoid(logits) with logits of O(30-90) on seeded weights, so a probability-space max-norm would measure the sigmoid's slope.
    ref_feats: oracle features (B,384,h,w); got_prob: our sigmoid output (B,3,H,W).  Compared where our sigmoid is invertible
    (|reference logit| < 10), normalised by max |reference logit|."""
    from oracle import lav_ref as O
    with torch.no_grad():
        ref_logit = O.head(sd, ref_feats, "seg_head.", sigmoid=False)
    got_logit = torch.logit(got_prob.double().cpu().clamp(1e-9, 1 - 1e-9))
    live = ref_logit.abs() < 10
    assert float(live.float().mean()) > 0.05
    return float((got_logit - ref_logit.double())[live].abs().max() / ref_logit.abs().max())
