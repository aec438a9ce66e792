"""InferModel — drop-in mirror of team_code_v2/model_inference.py:14-187 (same constructor, forward_paint,
forward, point_painting, det_inference, uniplanner_infer), plus ``forward_batch`` for B independent frames.

What changed underneath: painting is one CUDA kernel (background suppression fused), the LiDAR model is
the lav_b200 CUDA path, detection decode does ONE device->host copy per batch (the reference does ~60
blocking ``float()`` reads per frame, model_inference.py:100-112), crops are one CUDA kernel for all
vehicles of all frames, and the six command branches of the plan GRU run as one batch.
"""
import numpy as np
import torch
from torch import nn
from torch.nn import functional as F

from . import point_painting as PP

CAMERA_YAWS = PP.CAMERA_YAWS


def extract_peak_batch(heat, max_pool_ks=7, max_det=15):
    """extract_peak (model_inference.py:189-202) for heat (M,H,W): -> score (M,max_det), loc (M,max_det)."""
    max_cls = F.max_pool2d(heat[:, None], kernel_size=max_pool_ks, padding=max_pool_ks // 2, stride=1)[:, 0]
    possible = heat - (max_cls > heat).float() * 1e5
    return torch.topk(possible.flatten(1), min(max_det, possible[0].numel()), dim=1)


def score_kept(score, min_score=0.2):
    """det_inference's score test (model_inference.py:101-103): the reference compares each fp32 score, a 0-d tensor, with the
    Python float min_score, and torch does that in fp32.  So a score of exactly float32(min_score) is dropped, and so is NaN."""
    return np.asarray(score, np.float32) > np.float32(min_score)


def peak_filter(packed, pixels_per_meter, ncls=2, min_score=0.2):
    """decode_packed's filters on host packed peaks (B, 7, ncls * n) (det_inference, model_inference.py:98-121): score threshold
    (score_kept), the class-1 size filter, the ego-distance window.  -> keep (B, cols) bool, x, y (B, cols) int64 pixel, cls
    (cols,)."""
    W = int(packed[0, 6, 0])
    nd = packed.shape[2] // ncls
    loc = packed[:, 1].astype(np.int64)
    x, y = loc % W, loc // W
    w, h = packed[:, 2], packed[:, 3]
    cls = np.arange(packed.shape[2]) // nd
    dist = np.sqrt(((x - 160) ** 2 + (y - 280) ** 2).astype(np.float64))     # TODO hard-code of the reference kept
    keep = score_kept(packed[:, 0], min_score) & ~((cls[None] == 1) & (np.maximum(w, h) < 0.1 * pixels_per_meter))
    keep &= ~((dist <= 2) | (dist >= 30 * pixels_per_meter))
    return keep, x, y, cls


class InferModel(nn.Module):
    def __init__(self, lidar_model, uniplanner, camera_x, camera_z, device=torch.device("cuda")):
        super().__init__()
        self.uniplanner = uniplanner
        self.lidar_model = lidar_model
        self.coord_converters = PP.make_converters(camera_x, camera_z, rgb_h=288, rgb_w=256, fov=64, yaws=CAMERA_YAWS)
        # attribute names of the reference, so code that reaches into them keeps working
        self.lidar_model_point_pillar = lidar_model.point_pillar_net
        self.lidar_mode_backbone = lidar_model.backbone
        self.lidar_center_head, self.lidar_box_head = lidar_model.center_head, lidar_model.box_head
        self.lidar_ori_head, self.lidar_seg_head = lidar_model.ori_head, lidar_model.seg_head
        self.lidar_conv_emb = uniplanner.lidar_conv_emb
        self.plan, self.cast, self.cast_cmd_pred = uniplanner.plan, uniplanner.cast, uniplanner.cast_cmd_pred
        self.pixels_per_meter = uniplanner.pixels_per_meter
        self.offset_x, self.offset_y = uniplanner.offset_x, uniplanner.offset_y
        self.crop_size, self.num_cmds, self.num_plan = uniplanner.crop_size, uniplanner.num_cmds, uniplanner.num_plan
        self.to(device)

    # ---- painting ------------------------------------------------------------------------------------
    def forward_paint(self, cur_lidar, pred_sem, logits=False):
        """(N,4) + softmaxed (3,5,H,W) -> fused (N,8)  (model_inference.py:44-50).  logits=True also fuses the softmax."""
        return PP.forward_paint(cur_lidar, pred_sem, self.coord_converters, logits=logits)

    def point_painting(self, lidar, sems):
        return PP.point_painting(lidar, sems, self.coord_converters)

    # ---- detection decode ----------------------------------------------------------------------------
    @staticmethod
    def pack_peaks(heatmaps, sizemaps, orimaps):
        """device part of the decode: top-15 NMS peaks per class with the size/orientation values at the peaks,
        packed as (B, 6, ncls*15) = score | flat index | w | h | cos | sin.  Capturable in a CUDA graph."""
        B, ncls, H, W = heatmaps.shape
        score, loc = extract_peak_batch(heatmaps.reshape(B * ncls, H, W).float())
        score, loc = score.view(B, ncls, -1), loc.view(B, ncls, -1)
        flat = lambda t: t.reshape(B, 2, H * W).float()
        sz, ori = flat(sizemaps), flat(orimaps)
        idx = loc.reshape(B, 1, -1).expand(B, 2, -1)                      # (B,2,ncls*max_det)
        packed = torch.cat([score.reshape(B, 1, -1), loc.reshape(B, 1, -1).float(), sz.gather(2, idx), ori.gather(2, idx)], 1)
        return torch.cat([packed, packed.new_full((B, 1, packed.shape[2]), float(W))], 1)     # row 6 carries W

    def det_inference_batch(self, heatmaps, sizemaps, orimaps, min_score=0.2):
        """heatmaps (B,2,H,W) already sigmoided; sizemaps/orimaps (B,2,H,W).  Same filters as
        det_inference (model_inference.py:95-121); one D2H copy for the whole batch."""
        return self.decode_packed(self.pack_peaks(heatmaps, sizemaps, orimaps), heatmaps.shape[1], min_score)

    def decode_packed(self, packed, ncls=2, min_score=0.2):
        """host part of det_inference (model_inference.py:98-121), vectorised over the batch: score threshold, the
        class-1 size filter, the ego-distance window; survivors keep the reference's order (descending score)."""
        packed = packed.cpu().numpy()                                     # the ONE device->host copy of the decode
        B = packed.shape[0]
        if B == 0:
            return []
        keep, x, y, cls = peak_filter(packed, self.pixels_per_meter, ncls, min_score)
        out = []
        for b in range(B):
            dets = [[] for _ in range(ncls)]
            for j in np.nonzero(keep[b])[0]:
                dets[int(cls[j])].append((int(x[b, j]), int(y[b, j]), float(packed[b, 2, j]), float(packed[b, 3, j]),
                                          float(packed[b, 4, j]), float(packed[b, 5, j])))
            out.append(dets)
        return out

    def det_inference(self, heatmaps, sizemaps, orimaps, min_score=0.2):
        return self.det_inference_batch(heatmaps[None], sizemaps[None], orimaps[None], min_score)[0]

    # ---- planner -------------------------------------------------------------------------------------
    def uniplanner_infer(self, features, det, cmd_value, nxp):
        ee, epl, ecl, ocl, occ = self.uniplanner.infer_batch(features[None], [det], [cmd_value], nxp[None])
        if len(ocl[0]) == 0:
            return ee, epl[0], ecl[0], torch.zeros((0, self.num_cmds, self.num_plan, 2)), torch.zeros((0, self.num_cmds))
        return ee, epl[0], ecl[0], ocl[0], occ[0]

    # ---- whole frame ---------------------------------------------------------------------------------
    @torch.no_grad()
    def forward_batch(self, lidars, num_points, nxps, cmd_values):
        """B independent frames.  lidars: list of (P_b,11) tensors or (B,P,11); nxps (B,2); cmd_values (B,).
        Returns dict of batched outputs; 'det' is the per-frame detection list of the reference, 'packed' the device peaks it
        was decoded from (ops.det_peaks)."""
        from . import ops
        feats, center, box, ori, seg = self.lidar_model.forward_nhwc(lidars, num_points)
        packed = ops.det_peaks(center, box, ori)
        dets = self.decode_packed(packed)
        ee, epl, ecl, ocl, occ = self.uniplanner.infer_batch(feats.permute(0, 3, 1, 2), [d[1] for d in dets], cmd_values, nxps)
        return dict(ego_embd=ee, ego_plan_locs=epl, ego_cast_locs=ecl, other_cast_locs=ocl, other_cast_cmds=occ,
                    pred_bev=seg.permute(0, 3, 1, 2), det=dets, features=feats, packed=packed)

    @torch.no_grad()
    def forward(self, lidar_points, nxps, cmd_value):
        """InferModel.forward (model_inference.py:53-73): one frame."""
        o = self.forward_batch([lidar_points], [len(lidar_points)], nxps[None], [cmd_value])
        ocl, occ = o["other_cast_locs"][0], o["other_cast_cmds"][0]
        if len(ocl) == 0:   # the reference returns CPU zero tensors when nothing is detected (model_inference.py:160-161)
            ocl, occ = torch.zeros((0, self.num_cmds, self.num_plan, 2)), torch.zeros((0, self.num_cmds))
        return o["ego_embd"], o["ego_plan_locs"][0], o["ego_cast_locs"][0], ocl, occ, o["pred_bev"], o["det"][0]
