"""PyTorch heads of the LAV frame path (north_star: "autograd on the heads" stays PyTorch):
ResNet-18 embedder, UniPlanner (+ its frozen BEVPlanner teacher as a weight container), the
brake predictor.  Written fresh against the reference's behaviour with identical ``state_dict``
keys (tests/golden/keys_uniplanner.json, keys_brake.json):

  resnet18            lav/models/resnet.py:144-283 (num_channels stem, returns the layer4 map)
  UniPlanner          team_code_v2/models/uniplanner.py (infer path) — crop -> embed -> cast/plan GRUs
  BEVPlanner          lav/models/bev_planner_v2.py (training forward; the frozen teacher of UniPlanner's distillation)
  RGBBrakePredictionModel, Attention, SegmentationHead
                      team_code_v2/models/rgb.py:48-83, lav/models/attention.py, segmentation.py

Only the crop (bilinear rotated window gather) is a lav_b200 CUDA kernel; convs/GRUs here are cuDNN, except the
flag-selected kernels below (STEM_KERNEL, CAST_KERNEL) and the brake stem of forward_u8.
"""
import math

import numpy as np
import torch
from torch import nn
from torch.nn import functional as F

from . import ops


# ----------------------------------------------------------------------------- ResNet-18
TRAIN_CROP_KERNEL = True      # UniPlanner.crop_feature with gradients: lav_b200 crop kernel + its gather backward (ops.CropBilinear)
                              # instead of F.grid_sample (cudnn bilinear_sampler_bw)
# Eval f16 stems with 7x7 / s2 / p3 -> 64 and cin % 64 == 0 (the planner embedder's 384-channel crop stem) run on the lav_b200
# wgmma kernel (ops.conv7x7s2_umma).  cuDNN gives this shape a generic engine on H100 that is >10x slower.  False: cuDNN.
STEM_KERNEL = True


class BasicBlock(nn.Module):
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 3, stride, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.relu = nn.ReLU(inplace=True)
        self.conv2 = nn.Conv2d(planes, planes, 3, 1, 1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.downsample = downsample

    def forward(self, x):
        idt = x if self.downsample is None else self.downsample(x)
        out = self.relu(self.bn1(self.conv1(x)))
        out = self.bn2(self.conv2(out))
        return self.relu(out + idt)


class ResNet18(nn.Module):
    def __init__(self, num_channels=3, num_classes=1000):
        super().__init__()
        self.conv1 = nn.Conv2d(num_channels, 64, 7, 2, 3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(3, 2, 1)
        inpl = 64
        for i, (planes, stride) in enumerate(((64, 1), (128, 2), (256, 2), (512, 2)), 1):
            ds = None
            if stride != 1 or inpl != planes:
                ds = nn.Sequential(nn.Conv2d(inpl, planes, 1, stride, bias=False), nn.BatchNorm2d(planes))
            setattr(self, f"layer{i}", nn.Sequential(BasicBlock(inpl, planes, stride, ds), BasicBlock(planes, planes)))
            inpl = planes
        self.avgpool = nn.AdaptiveAvgPool2d((1, 1))       # present in the reference module tree, unused
        self.fc = nn.Linear(512, num_classes)             # keys exist in the checkpoints, unused (resnet.py:235-247)

    def forward(self, x):
        if not self.training and x.is_cuda and not torch.is_grad_enabled():
            return self._forward_folded(x)
        x = self.maxpool(self.relu(self.bn1(self.conv1(x))))
        return self.layer4(self.layer3(self.layer2(self.layer1(x))))

    # ---- eval fast path: BatchNorm folded into the conv weights, conv+bias+ReLU and conv+bias+add+ReLU as single cuDNN
    # fused ops (no separate BN / ReLU / add passes over the activations).  Folded weights are cached per (dtype, device).
    def _fold_sig(self):
        """identity + in-place version of every tensor the folded weights derive from: optimizer steps, copy_ (any
        load_state_dict, also a parent's), .to() and re-assignment all change it, so stale folds cannot survive."""
        return tuple((t.data_ptr(), t._version) for t in list(self.parameters()) + list(self.buffers()))

    def _cache(self):
        cache = self.__dict__.setdefault("_fold_cache", {})
        sig = self._fold_sig()
        if cache.get("sig") != sig:
            cache.clear()
            cache["sig"] = sig
        return cache

    def _folded(self, dtype, device):
        key = (dtype, str(device))
        cache = self._cache()
        if key not in cache:
            def fold(conv, bn):
                s = bn.weight.double() / torch.sqrt(bn.running_var.double() + bn.eps)
                w = (conv.weight.double() * s[:, None, None, None]).to(dtype).contiguous(memory_format=torch.channels_last)
                b = (bn.bias.double() - bn.running_mean.double() * s).to(dtype)
                return w, b
            f = {"stem": fold(self.conv1, self.bn1)}
            for li in range(1, 5):
                for bi, blk in enumerate(getattr(self, f"layer{li}")):
                    f[(li, bi, 1)] = fold(blk.conv1, blk.bn1)
                    f[(li, bi, 2)] = fold(blk.conv2, blk.bn2)
                    if blk.downsample is not None:
                        f[(li, bi, "d")] = fold(blk.downsample[0], blk.downsample[1])
            cache[key] = f
        return cache[key]

    def _forward_folded(self, x):
        dt = self.conv1.weight.dtype
        x = x.to(dt).contiguous(memory_format=torch.channels_last)
        f = self._folded(dt, x.device)
        c1 = self.conv1
        if (STEM_KERNEL and dt == ops.h16() and c1.kernel_size == (7, 7) and c1.stride == (2, 2) and c1.padding == (3, 3)
                and c1.out_channels == 64 and c1.in_channels % 64 == 0):
            # the planner embedder's 384-channel stem on the lav_b200 wgmma kernel (csrc/stem_umma.cu)
            if "stem_umma" not in f:
                w, b = self._folded(torch.float32, x.device)["stem"]                # fold in fp32, round once
                f["stem_umma"] = (ops.pack_conv7x7s2_weights(w), b.float().contiguous())
            wk, b = f["stem_umma"]
            x = ops.conv7x7s2_umma(x.permute(0, 2, 3, 1).contiguous(), wk, b)
            return self._trunk_folded(ops.maxpool3x3s2_nhwc(x).permute(0, 3, 1, 2), f)
        w, b = f["stem"]
        x = torch.cudnn_convolution_relu(x, w, b, (2, 2), (3, 3), (1, 1), 1)
        if dt == ops.h16():                        # lav_b200 pool kernel on the channels-last memory (ATen's is ~5x slower)
            return self._trunk_folded(ops.maxpool3x3s2_nhwc(x.permute(0, 2, 3, 1).contiguous()).permute(0, 3, 1, 2), f)
        return self._trunk_folded(self.maxpool(x), f)

    def forward_u8(self, img_u8, mean, std):
        """Eval fast path from raw camera bytes: img_u8 (B, ncam, H, cam_w, 3) uint8 (cameras side by side) -> layer4 map.
        Normalisation + conv1 + bn1 + ReLU run in the lav_b200 tensor-core stem kernel and the max-pool in its companion
        (csrc/stem.cu): in cuDNN/ATen these two are 64 % of the brake model's GPU time (3 input channels).  f16 only."""
        dt = self.conv1.weight.dtype
        assert dt == ops.h16() and self.conv1.in_channels == 3, "forward_u8: f16 3-channel stem only"
        f = self._folded(dt, img_u8.device)
        if "stem_u8" not in f:
            w, b = self._folded(torch.float32, img_u8.device)["stem"]                  # fold in fp32, round once
            f["stem_u8"] = (ops.pack_stem_weights(w), b.float().contiguous())
        wk, b = f["stem_u8"]
        x = ops.maxpool3x3s2_nhwc(ops.stem7x7s2_u8(img_u8, wk, b, mean, std))
        return self._trunk_folded(x.permute(0, 3, 1, 2), f)                            # NCHW view of channels-last memory

    def _trunk_folded(self, x, f):
        for li in range(1, 5):
            for bi, blk in enumerate(getattr(self, f"layer{li}")):
                st = blk.conv1.stride
                w1, b1 = f[(li, bi, 1)]
                w2, b2 = f[(li, bi, 2)]
                idt = x
                if blk.downsample is not None:
                    wd, bd = f[(li, bi, "d")]
                    idt = F.conv2d(x, wd, bd, blk.downsample[0].stride)
                y = torch.cudnn_convolution_relu(x, w1, b1, st, (1, 1), (1, 1), 1)
                x = torch.cudnn_convolution_add_relu(y, w2, idt, 1.0, b2, (1, 1), (1, 1), (1, 1), 1)
        return x

    def _apply(self, fn, *a, **k):
        self.__dict__["_fold_cache"] = {}
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, *a, **k):
        self.__dict__["_fold_cache"] = {}
        return super().load_state_dict(*a, **k)

    def train(self, mode=True):
        self.__dict__["_fold_cache"] = {}
        return super().train(mode)


def resnet18(pretrained=False, num_channels=3, **kw):
    return ResNet18(num_channels=num_channels)


# The cast branches (6 x GRU(512, 64) + Linear(64, 2) + cumsum over the repeated embedding) as ONE fp32 kernel (csrc/cast_gru.cu)
# instead of ~100 dependent cuDNN / ATen launches per call.  Inference only.
CAST_KERNEL = True


def _cast_branches(owner, grus, mlps, embd, num_plan):
    """cast() of both planners.  Kernel path for CUDA fp32 inference (transposed weights packed once per parameter version);
    the module path otherwise (training, CPU, non-fp32)."""
    w0 = grus[0].weight_ih_l0
    if (CAST_KERNEL and embd.is_cuda and not torch.is_grad_enabled() and embd.dtype == torch.float32 and w0.dtype == torch.float32
            and grus[0].hidden_size == 64 and grus[0].input_size == 512 and mlps[0].out_features == 2):
        params = [p for g in grus for p in (g.weight_ih_l0, g.weight_hh_l0, g.bias_ih_l0, g.bias_hh_l0)] + [p for m in mlps for p in (m.weight, m.bias)]
        key = tuple((p.data_ptr(), p._version) for p in params) + (str(embd.device),)
        cached = owner.__dict__.get("_cast_pack")
        if cached is None or cached[0] != key:                       # re-pack after load_state_dict / .to() / an optimizer step
            with torch.no_grad():
                pack = (torch.stack([g.weight_ih_l0.t() for g in grus]).contiguous(), torch.stack([g.weight_hh_l0.t() for g in grus]).contiguous(),
                        torch.stack([g.bias_ih_l0 for g in grus]).contiguous(), torch.stack([g.bias_hh_l0 for g in grus]).contiguous(),
                        torch.stack([m.weight for m in mlps]).contiguous(), torch.stack([m.bias for m in mlps]).contiguous())
            cached = owner.__dict__["_cast_pack"] = (key, pack)
        return ops.cast_gru(embd.contiguous(), *cached[1], num_plan)
    B = embd.size(0)
    u = embd.expand(num_plan, B, -1).permute(1, 0, 2).contiguous()
    return torch.stack([torch.cumsum(mlp(gru(u)[0]), dim=1) for gru, mlp in zip(grus, mlps)], dim=1)


# ----------------------------------------------------------------------------- planners
def transform_points(locs, oris):
    """rotate row-vector points by `oris` (right-multiplication by [[c, s], [-s, c]], uniplanner.py:319-326):
    locs (..., T, 2), oris (...)."""
    c, s_ = torch.cos(oris), torch.sin(oris)
    rot = torch.stack([c, s_, -s_, c], dim=-1).unflatten(-1, (2, 2))
    return torch.matmul(locs, rot)


def crop_theta(rel_locs, rel_oris, H, W, pixels_per_meter, crop_size, offset_x, offset_y):
    """affine theta (K,2,3) of UniPlanner.crop_feature (team_code_v2/models/uniplanner.py:303-333)."""
    rel_locs = rel_locs.view(-1, 2) * pixels_per_meter        # then / [H/2, W/2] per column (no host tensor: graph-capturable)
    cos, sin = torch.cos(rel_oris), torch.sin(rel_oris)
    rel_x, rel_y = rel_locs[..., 0] / (H / 2), rel_locs[..., 1] / (W / 2)
    k = crop_size / H
    rot_x_offset = -k * offset_x * cos + k * offset_y * sin + offset_x
    rot_y_offset = -k * offset_x * sin - k * offset_y * cos + offset_y
    return torch.stack([torch.stack([k * cos, k * -sin, rot_x_offset + rel_x], dim=-1),
                        torch.stack([k * sin, k * cos, rot_y_offset + rel_y], dim=-1)], dim=-2)


def _pose_jitter(n, x_jitter, angle_jitter, device):
    """augmentation of a crop's pose: lateral offset U(-x_jitter, x_jitter) metres (no longitudinal part) and heading
    U(-angle_jitter, angle_jitter) radians.  Drawn on the CPU generator as rand(n,2) then rand(n): the reference's stream order
    (uniplanner.py:83-86,118-121, bev_planner_v2.py:100-102)."""
    shift = (torch.rand(n, 2) * 2 - 1) * x_jitter
    shift[:, 1] = 0
    turn = (torch.rand(n) * 2 - 1) * angle_jitter
    return shift.to(device), turn.to(device)


def _cap_rows_host(mask, limit):
    """cap_per_sample(mask, limit) with ONE device->host copy of the mask instead of one synchronisation per row: the same
    multinomial draws in the same row order, so the same actors are kept.  -> (frame, slot) index tensors on the mask's device,
    in row-major order (the order of a boolean-mask gather)."""
    m = mask.cpu()
    for b in range(m.shape[0]):
        on = m[b].nonzero().flatten()
        if on.numel() > limit:
            keep = on[torch.multinomial(torch.ones(on.numel()), limit)]
            m[b] = False
            m[b, keep] = True
    frame, slot = m.nonzero(as_tuple=True)
    return frame.to(mask.device), slot.to(mask.device)


class BEVPlanner(nn.Module):
    """The privileged planner (lav/models/bev_planner_v2.py): the teacher nested in the UniPlanner checkpoint (bev_planner.*),
    and trained on its own from ground-truth BEV maps by ``forward`` (stage 1 of the v2 recipe, lav_b200.train_bev)."""

    def __init__(self, pixels_per_meter=2, crop_size=64, x_offset=0, y_offset=0.75, feature_x_jitter=1, feature_angle_jitter=10,
                 num_plan=10, k=16, num_out_feature=64, num_cmds=6, max_num_cars=5, num_plan_iter=1, num_frame_stack=0):
        super().__init__()
        self.num_cmds, self.num_plan, self.num_plan_iter, self.max_num_cars = num_cmds, num_plan, num_plan_iter, max_num_cars
        self.num_out_feature = num_out_feature
        self.pixels_per_meter, self.crop_size = pixels_per_meter, crop_size
        self.feature_x_jitter = feature_x_jitter
        self.feature_angle_jitter = np.deg2rad(feature_angle_jitter)
        self.offset_x = nn.Parameter(torch.tensor(x_offset).float(), requires_grad=False)
        self.offset_y = nn.Parameter(torch.tensor(y_offset).float(), requires_grad=False)
        self.bev_conv_emb = nn.Sequential(resnet18(num_channels=3 + 2 * (num_frame_stack + 1)), nn.AdaptiveAvgPool2d((1, 1)), nn.Flatten())
        self.plan_gru = nn.GRU(4, 512, batch_first=True)
        self.plan_mlp = nn.Linear(512, 2)
        self.cast_grus = nn.ModuleList([nn.GRU(512, 64, batch_first=True) for _ in range(num_cmds)])
        self.cast_mlps = nn.ModuleList([nn.Linear(64, 2) for _ in range(num_cmds)])
        self.cast_cmd_pred = nn.Sequential(nn.Linear(512, num_cmds), nn.Sigmoid())

    def crop_feature(self, features, rel_locs, rel_oris, pixels_per_meter=4, crop_size=96, frame_idx=None):
        """BEVPlanner.crop_feature (bev_planner_v2.py:222-264).  A uint8 CUDA map (B,C,H,W) goes through the lav_b200 kernel
        (ops.crop_bilinear_u8): crop k reads frame ``frame_idx[k]`` (default k) straight from the bytes, -> fp32 NCHW crops.
        Every other input takes F.affine_grid + F.grid_sample (the frozen teacher of train_lidar passes fp32 maps), after
        gathering ``features[frame_idx]`` when frame indices are given."""
        B, C, H, W = features.size()
        theta = crop_theta(rel_locs, rel_oris, H, W, pixels_per_meter, crop_size, self.offset_x, self.offset_y)
        if features.is_cuda and features.dtype == torch.uint8:
            if frame_idx is None:
                frame_idx = torch.arange(theta.shape[0], device=features.device, dtype=torch.int32)
            return ops.crop_bilinear_u8(features.contiguous(), frame_idx, theta.detach(), crop_size)
        if frame_idx is not None:
            features = features[frame_idx.long()]
            B = features.shape[0]
        grids = F.affine_grid(theta, torch.Size((B, C, crop_size, crop_size)), align_corners=True)
        return F.grid_sample(features, grids, align_corners=True)

    def forward(self, bev, ego_locs, locs, oris, nxps, typs):
        """Training forward of the privileged planner (bev_planner_v2.py:72-174): from crops of the ground-truth BEV ``bev``
        (B,C,H,W) — uint8 on the GPU takes the lav_b200 crop kernel, anything else is cast to fp32 and takes grid_sample —
        forecast the vehicles ahead of each ego (at most max_num_cars per sample, pose jittered) and plan for the ego (no jitter).
        locs / oris / typs slot 0 is the ego.  Returns the reference's 6-tuple
            (other_locs, other_cast_locs, other_cast_cmds, ego_plan_locs, ego_cast_locs, ego_cast_cmds).
        Random draws keep the reference's order on the CPU generator: the per-row multinomial cap, then rand(K,2), rand(K).
        Others and egos go through the embedder in two calls, so BatchNorm sees the reference's two batches."""
        if not (bev.is_cuda and bev.dtype == torch.uint8):
            bev = bev.float()
        dev = bev.device
        dt = torch.float32 if bev.dtype == torch.uint8 else bev.dtype
        ppm, crop = self.pixels_per_meter, 2 * self.crop_size
        ego_heading = oris[:, :1]
        act_locs, act_oris = locs[:, 1:], oris[:, 1:]
        slots = act_locs.shape[1]
        chosen = vehicles_ahead(ego_locs, act_locs, typs[:, 1:] == 1)
        if bool(chosen.any()):
            frame, slot = _cap_rows_host(chosen, self.max_num_cars)
            future = act_locs[frame, slot, 1:] - act_locs[frame, slot, :1]
            start = act_locs[frame, slot, 0] - ego_locs[frame, 0]
            heading = act_oris[frame, slot] - ego_heading[frame, 0]
            shift, turn = _pose_jitter(frame.numel(), self.feature_x_jitter, self.feature_angle_jitter, dev)
            crops = self.crop_feature(bev, start + shift, heading + turn, pixels_per_meter=ppm, crop_size=crop, frame_idx=frame)
            other_locs = transform_points(future - shift[:, None], -heading - turn)
            other_embd = self.bev_conv_emb(crops)
            other_cast, other_cmds = self.cast(other_embd), self.cast_cmd_pred(other_embd)
        else:                                                               # no vehicle ahead: zero placeholders, one per slot
            other_locs = torch.zeros((slots, self.num_plan, 2), dtype=dt, device=dev)
            other_cast = torch.zeros((slots, self.num_cmds, self.num_plan, 2), dtype=dt, device=dev)
            other_cmds = torch.zeros((slots, self.num_cmds), dtype=dt, device=dev)
        B = bev.shape[0]
        zero = torch.zeros((B, 2), dtype=dt, device=dev)
        ego_embd = self.bev_conv_emb(self.crop_feature(bev, zero, zero[:, 0], pixels_per_meter=ppm, crop_size=crop))
        ego_cast = self.cast(ego_embd)
        ego_plan = self.plan(ego_embd, nxps, cast_locs=ego_cast, pixels_per_meter=ppm, crop_size=crop)
        return other_locs, other_cast, other_cmds, ego_plan, ego_cast, self.cast_cmd_pred(ego_embd)

    @torch.no_grad()
    def forecast_recorded(self, bev, ego_locs, locs, oris, typs, nxps):
        """Forecasts of every recorded_rows row and of each ego, from crops of the ground-truth BEV ``bev`` at the recorded poses
        (forward's crops at zero jitter; a uint8 map on the GPU takes the lav_b200 crop kernel), all through one embedder call.
        -> dict: frame, slot, cast (K,C,T,2), score (K,C), target (K,T,2) of the rows; ego_cast (B,C,T,2), ego_score (B,C),
        ego_target (B,T,2) = ego_locs[:, 1:]; ego_plan (B,C,T,2) = the last plan iteration from the ego's cast and ``nxps``."""
        if not (bev.is_cuda and bev.dtype == torch.uint8):
            bev = bev.float()
        B, dev = bev.shape[0], bev.device
        ppm, crop = self.pixels_per_meter, 2 * self.crop_size
        rows = recorded_rows(ego_locs, locs, oris, typs)
        at, facing, fidx = _forecast_poses(rows, B, dev)
        embd = self.bev_conv_emb(self.crop_feature(bev, at, facing, pixels_per_meter=ppm, crop_size=crop, frame_idx=fidx))
        cast, score = self.cast(embd), self.cast_cmd_pred(embd)
        out = _forecast_result(rows, cast, score, ego_locs)
        K = rows["frame"].numel()
        out["ego_plan"] = self.plan(embd[K:], nxps, cast_locs=cast[K:], pixels_per_meter=ppm, crop_size=crop)[:, -1]
        return out

    def cast(self, embd):
        return _cast_branches(self, self.cast_grus, self.cast_mlps, embd, self.num_plan)

    def plan(self, embd, nxp, cast_locs=None, pixels_per_meter=4, crop_size=96):
        return _plan_rollout(self.plan_gru, self.plan_mlp, self.num_cmds, self.num_plan, self.num_plan_iter, embd, nxp,
                             (self.cast(embd) if cast_locs is None else cast_locs).detach(), pixels_per_meter, crop_size)


def _plan_rollout(plan_gru, plan_mlp, num_cmds, num_plan, num_plan_iter, embd, nxp, plan_loc, pixels_per_meter, crop_size):
    """plan/_plan of both planners (uniplanner.py:227-259): the six command branches share the GRU, so one call rolls
    6*B sequences; repeated num_plan_iter times feeding its own output."""
    B = embd.size(0)
    u0 = nxp * pixels_per_meter / crop_size * 2 - 1
    h0 = embd[:, None].expand(B, num_cmds, -1).reshape(1, B * num_cmds, -1).contiguous()
    outs = []
    for _ in range(num_plan_iter):
        u = torch.cat([u0[:, None, None].expand(B, num_cmds, num_plan, 2), plan_loc], dim=3)
        out, _ = plan_gru(u.reshape(B * num_cmds, num_plan, 4), h0)
        plan_loc = torch.cumsum(plan_mlp(out), dim=1).view(B, num_cmds, num_plan, 2) + plan_loc
        outs.append(plan_loc)
    return torch.stack(outs, dim=1)


def vehicles_ahead(ego_locs, locs, is_vehicle):
    """mask of the actors a sample may forecast: vehicles whose current position lies ahead of the ego (negative y in the ego
    frame) — the selection rule of lav/models/uniplanner.py:329-333.  ego_locs (B,T,2), locs (B,N,T,2), is_vehicle (B,N) bool."""
    ahead = (locs[:, :, 0, 1] - ego_locs[:, None, 0, 1]) < 0
    return is_vehicle & ahead


def recorded_rows(ego_locs, locs, oris, typs):
    """the forecast rows of an evaluation over recorded poses: every actor the training selection accepts
    (vehicles_ahead(ego_locs, locs[:, 1:], typs[:, 1:] == 1), slot order, no max_num_cars cap) with the training forward's pose
    and target at zero jitter.  locs (B,N,T+1,2), oris (B,N), typs (B,N), slot 0 the ego.  -> dict: frame, slot (K,) int64 with
    slot >= 1 the index into locs; start (K,2) = locs[f, s, 0] - ego_locs[f, 0]; heading (K,) = oris[f, s] - oris[f, 0]; target
    (K,T,2) = the actor's recorded future in its crop frame, transform_points(locs[f, s, 1:] - locs[f, s, :1], -heading)."""
    frame, slot = vehicles_ahead(ego_locs, locs[:, 1:], typs[:, 1:] == 1).nonzero(as_tuple=True)
    slot = slot + 1
    heading = oris[frame, slot] - oris[frame, 0]
    return dict(frame=frame, slot=slot, start=locs[frame, slot, 0] - ego_locs[frame, 0], heading=heading,
                target=transform_points(locs[frame, slot, 1:] - locs[frame, slot, :1], -heading))


def _forecast_poses(rows, B, device):
    """(locations, headings, frame indices) of the crops of forecast_recorded: the K rows, then the B egos at the origin."""
    at = torch.cat([rows["start"], torch.zeros((B, 2), dtype=rows["start"].dtype, device=device)])
    facing = torch.cat([rows["heading"], torch.zeros((B,), dtype=rows["heading"].dtype, device=device)])
    fidx = torch.cat([rows["frame"], torch.arange(B, device=device)]).to(torch.int32)
    return at, facing, fidx


def _forecast_result(rows, cast, score, ego_locs):
    K = rows["frame"].numel()
    return dict(frame=rows["frame"], slot=rows["slot"], cast=cast[:K], score=score[:K], target=rows["target"], ego_cast=cast[K:],
                ego_score=score[K:], ego_target=ego_locs[:, 1:])


def off_centre(x, y, center_x, center_y):
    """det_to_locs' centre test (uniplanner.py:203-204): a detection at pixel (x, y) (scalars or arrays) is forecast when it lies
    more than 4 px from the crop centre."""
    dx, dy = np.asarray(x, np.float64) - center_x, np.asarray(y, np.float64) - center_y
    return np.sqrt(dx * dx + dy * dy) > 4


def cap_per_sample(mask, limit):
    """at most `limit` True entries per row of a (B,N) bool mask; rows over the limit keep a uniformly random subset.  One
    torch.multinomial draw per over-full row, in row order — the random stream consumption of uniplanner.py:336-347, so a
    seeded run selects the same actors as the reference."""
    out = mask.clone()
    for b in range(mask.shape[0]):
        on = mask[b].nonzero().flatten()
        if on.numel() > limit:
            keep = on[torch.multinomial(torch.ones(on.numel()), limit).to(on.device)]
            out[b] = False
            out[b, keep] = True
    return out


class UniPlanner(nn.Module):
    def __init__(self, bev_planner, pixels_per_meter=2, crop_size=64, x_offset=0, y_offset=0.75, feature_x_jitter=1,
                 feature_angle_jitter=10, num_plan=10, k=16, num_input_feature=96, num_out_feature=64, num_cmds=6,
                 max_num_cars=4, num_plan_iter=1):
        super().__init__()
        self.num_cmds, self.num_plan, self.num_plan_iter, self.max_num_cars = num_cmds, num_plan, num_plan_iter, max_num_cars
        self.bev_planner = bev_planner
        self.num_out_feature = num_out_feature
        self.pixels_per_meter, self.crop_size = pixels_per_meter, crop_size
        self.feature_x_jitter = feature_x_jitter
        self.feature_angle_jitter = np.deg2rad(feature_angle_jitter)
        self.offset_x = nn.Parameter(torch.tensor(x_offset).float(), requires_grad=False)
        self.offset_y = nn.Parameter(torch.tensor(y_offset).float(), requires_grad=False)
        self.lidar_conv_emb = nn.Sequential(resnet18(num_channels=num_input_feature), nn.AdaptiveAvgPool2d((1, 1)), nn.Flatten())
        self.plan_gru = nn.GRU(4, 512, batch_first=True)
        self.plan_mlp = nn.Linear(512, 2)
        self.cast_grus_ego = nn.ModuleList([nn.GRU(512, 64, batch_first=True) for _ in range(num_cmds)])
        self.cast_mlps_ego = nn.ModuleList([nn.Linear(64, 2) for _ in range(num_cmds)])
        self.cast_grus_other = nn.ModuleList([nn.GRU(512, 64, batch_first=True) for _ in range(num_cmds)])   # dead weights, kept
        self.cast_mlps_other = nn.ModuleList([nn.Linear(64, 2) for _ in range(num_cmds)])
        self.cast_cmd_pred = nn.Sequential(nn.Linear(512, num_cmds), nn.Sigmoid())

    # -- crop: one CUDA kernel on channels-last features (or grid_sample for generic callers)
    def crop_feature(self, features, rel_locs, rel_oris, pixels_per_meter=4, crop_size=96, frame_idx=None):
        """features: logical (B,C,H,W).  With ``frame_idx`` (K,) the K crops read features[frame_idx[k]] without
        materialising an expanded copy.  A map the crop kernel cannot take as it is (see ops.crop_supported) goes through
        F.affine_grid + F.grid_sample."""
        B, C, H, W = features.size()
        theta = crop_theta(rel_locs, rel_oris, H, W, pixels_per_meter, crop_size, self.offset_x, self.offset_y)
        if features.is_cuda and not (torch.is_grad_enabled() and features.requires_grad):
            feats_nhwc = features.permute(0, 2, 3, 1)
            if ops.crop_supported(feats_nhwc):
                if frame_idx is None:
                    frame_idx = torch.arange(theta.shape[0], device=features.device, dtype=torch.int32) % B
                return ops.crop_bilinear(feats_nhwc, frame_idx, theta, crop_size).permute(0, 3, 1, 2)
        if TRAIN_CROP_KERNEL and features.is_cuda and features.dtype == torch.float32:
            # training: same kernel forward, hand-written gather backward (ops.CropBilinear) instead of cudnn's atomics
            feats_nhwc = features.permute(0, 2, 3, 1).contiguous()           # no copy when `features` is channels-last
            if ops.crop_supported(feats_nhwc):
                if frame_idx is None:
                    frame_idx = torch.arange(theta.shape[0], device=features.device, dtype=torch.int32) % B
                return ops.CropBilinear.apply(feats_nhwc, frame_idx, theta, crop_size).permute(0, 3, 1, 2)
        if frame_idx is not None:
            features = features[frame_idx.long()]
        grids = F.affine_grid(theta, torch.Size((theta.shape[0], C, crop_size, crop_size)), align_corners=True)
        return F.grid_sample(features, grids, align_corners=True)

    def cast(self, embd, mode='ego'):
        # 'other' re-uses the ego GRUs (uniplanner.py:296-300)
        return _cast_branches(self, self.cast_grus_ego, self.cast_mlps_ego, embd, self.num_plan)

    def plan(self, embd, nxp, cast_locs=None, pixels_per_meter=4, crop_size=96):
        return _plan_rollout(self.plan_gru, self.plan_mlp, self.num_cmds, self.num_plan, self.num_plan_iter, embd, nxp,
                             (self.cast(embd) if cast_locs is None else cast_locs).detach(), pixels_per_meter, crop_size)

    # ---- training forward ------------------------------------------------------------------------------------------------
    def _jitter(self, n, device):
        """augmentation of a crop's pose: lateral offset U(-jx, jx) metres (no longitudinal part) and heading U(-ja, ja).
        Drawn on the CPU generator as rand(n,2) then rand(n): the reference's stream order (uniplanner.py:83-86,118-121)."""
        return _pose_jitter(n, self.feature_x_jitter, self.feature_angle_jitter, device)

    def _student(self, crops):
        """crops (n,C,crop,crop) -> (embedding, cast (n,cmds,T,2), command scores (n,cmds)); one call = one BatchNorm batch."""
        embd = self.lidar_conv_emb(crops)
        return embd, self.cast(embd), self.cast_cmd_pred(embd)

    def forward(self, features, bev, ego_locs, locs, oris, nxps, typs):
        """Distillation forward of train_lidar (lav/models/uniplanner.py:56-151): the student forecasts the selected other
        vehicles and plans for the ego from jittered crops of the LiDAR features; the frozen BEVPlanner teacher does the same
        from crops of the ground-truth BEV, under no_grad.  Returns the reference's 11-tuple
            (other_locs, other_cast_locs, other_cast_cmds, other_cast_locs_expert, other_cast_cmds_expert,
             ego_locs, ego_plan_locs, ego_cast_locs, ego_cast_cmds, ego_cast_locs_expert, ego_plan_locs_expert).
        Others and egos go through the embedder in two separate calls (two BatchNorm batches) and the random draws keep the
        reference's order, so a seeded run is bit-identical to the reference module (tests/golden/uniplanner_train.npz)."""
        teacher = self.bev_planner.eval()
        dev = features.device
        if TRAIN_CROP_KERNEL and features.is_cuda and features.dtype == torch.float32:
            features = features.contiguous(memory_format=torch.channels_last)   # one transposition serves both crop calls
        ppm, crop = self.pixels_per_meter, self.crop_size
        ego_now, ego_heading = ego_locs[:, 0], oris[:, :1]
        act_locs, act_oris = locs[:, 1:], oris[:, 1:]                       # slot 0 of locs / oris / typs is the ego itself
        slots = act_locs.shape[1]
        chosen = vehicles_ahead(ego_locs, act_locs, typs[:, 1:] == 1)
        if bool(chosen.any()):
            chosen = cap_per_sample(chosen, self.max_num_cars)
            frame, slot = chosen.nonzero(as_tuple=True)                     # row-major = the order of a boolean-mask gather
            start = act_locs[frame, slot, 0] - ego_now[frame]               # actor pose in the ego frame
            heading = act_oris[frame, slot] - ego_heading[frame, 0]
            future = act_locs[frame, slot, 1:] - act_locs[frame, slot, :1]
            shift, turn = self._jitter(frame.numel(), dev)
            at, facing = start + shift, heading + turn
            other_locs = transform_points(future - shift[:, None], -facing)
            _, other_cast, other_cmds = self._student(self.crop_feature(features, at, facing, pixels_per_meter=ppm / 2, crop_size=crop,
                                                                        frame_idx=frame))
            with torch.no_grad():
                t_embd = teacher.bev_conv_emb(teacher.crop_feature(bev[frame], at, facing, pixels_per_meter=ppm, crop_size=2 * crop))
                other_cast_t, other_cmds_t = teacher.cast(t_embd), teacher.cast_cmd_pred(t_embd)
        else:                                                               # no actor to forecast: zero placeholders, one per slot
            blank = lambda *shape: torch.zeros(shape, dtype=features.dtype, device=dev)
            other_locs = blank(slots, self.num_plan, 2)
            other_cast, other_cast_t = blank(slots, self.num_cmds, self.num_plan, 2), blank(slots, self.num_cmds, self.num_plan, 2)
            other_cmds, other_cmds_t = blank(slots, self.num_cmds), blank(slots, self.num_cmds)
        shift, turn = self._jitter(features.shape[0], dev)
        ego_future = transform_points(ego_locs[:, 1:] - shift[:, None], -turn)
        goal = transform_points(nxps[:, None] - shift[:, None], -turn)[:, 0]
        ego_embd, ego_cast, ego_cmds = self._student(self.crop_feature(features, shift, turn, pixels_per_meter=ppm / 2, crop_size=crop))
        with torch.no_grad():
            t_embd = teacher.bev_conv_emb(teacher.crop_feature(bev, shift, turn, pixels_per_meter=ppm, crop_size=2 * crop))
            ego_cast_t = teacher.cast(t_embd)
            ego_plan_t = teacher.plan(t_embd, goal, cast_locs=ego_cast_t, pixels_per_meter=ppm, crop_size=2 * crop)
        ego_plan = self.plan(ego_embd, goal, cast_locs=ego_cast, pixels_per_meter=ppm, crop_size=2 * crop)
        return (other_locs, other_cast, other_cmds, other_cast_t, other_cmds_t,
                ego_future, ego_plan, ego_cast, ego_cmds, ego_cast_t, ego_plan_t)

    def crop_centre(self, H, W):
        """(center_x, center_y) in map pixels of the agent's crop frame, for features of logical size (H/2, W/2)."""
        return float(W / 2 + self.offset_x * W / 2), float(H / 2 + self.offset_y * H / 2)

    def det_to_locs(self, det, H, W):
        """detections -> (locs list, oris list) in ego metres (uniplanner.py:195-214)."""
        center_x, center_y = self.crop_centre(H, W)
        locs, oris = [], []
        for X, Y, h, w, cos, sin in det:
            if not off_centre(X, Y, center_x, center_y):
                continue
            locs.append([(X - center_x) / self.pixels_per_meter, (Y - center_y) / self.pixels_per_meter])
            oris.append(float(np.arctan2(sin, cos)))
        return locs, oris

    @torch.no_grad()
    def infer_batch(self, features, dets, cmds, nxps):
        """Batched UniPlanner.infer: features logical (B,C,h,w); dets[b] = vehicle detections of frame b;
        cmds (B,) ints; nxps (B,2).  All crops of the batch go through one embed / GRU roll-out.
        Returns per-frame lists like infer(): (ego_embd, ego_plan_locs, ego_cast_locs, other_cast_locs, other_cast_cmds)."""
        B = features.size(0)
        dev = features.device
        H, W = features.size(2) * 2, features.size(3) * 2
        locs, oris, fidx, counts = [], [], [], []
        for b, det in enumerate(dets):
            l, o = self.det_to_locs(det, H, W)
            locs += l
            oris += o
            fidx += [b] * len(l)
            counts.append(len(l))
        K = len(locs)
        all_locs = torch.tensor(locs + [[0.0, 0.0]] * B, dtype=torch.float32).view(-1, 2).to(dev)
        all_oris = torch.tensor(oris + [0.0] * B, dtype=torch.float32).to(dev)
        all_fidx = torch.tensor(fidx + list(range(B)), dtype=torch.int32).to(dev)
        cmds = torch.as_tensor(cmds, device=dev).long()
        ee, epl, ecl, o_cast, o_cmds = self.infer_device(features, all_locs, all_oris, all_fidx, K, nxps.to(dev).float(), cmds)
        return ee, epl, ecl, torch.split(o_cast, counts), torch.split(o_cmds, counts)

    @torch.no_grad()
    def infer_device(self, features, all_locs, all_oris, all_fidx, K, nxps, cmds):
        """Device-only part of infer (capturable in a CUDA graph): rows [0,K) of all_* are detected vehicles, rows
        [K,K+B) the egos.  Returns (ego_embd, ego_plan_locs (B,T,2), ego_cast_locs (B,T,2), other_cast_locs (K,6,T,2),
        other_cast_cmds (K,6))."""
        B = features.size(0)
        dev = features.device
        crops = self.crop_feature(features, all_locs, all_oris, pixels_per_meter=self.pixels_per_meter / 2,
                                  crop_size=self.crop_size, frame_idx=all_fidx)
        embd = self.lidar_conv_emb(crops.to(self.lidar_conv_emb[0].conv1.weight.dtype)).float()
        cast = self.cast(embd)
        ego_embd, ego_cast = embd[K:], cast[K:]
        ego_plan = self.plan(ego_embd, nxps, cast_locs=ego_cast, pixels_per_meter=self.pixels_per_meter,
                             crop_size=self.crop_size * 2)[:, -1]
        ar = torch.arange(B, device=dev)
        ego_plan_locs, ego_cast_locs = ego_plan[ar, cmds], ego_cast[ar, cmds]
        if K > 0:
            o_cast = transform_points(cast[:K], all_oris[:K, None].repeat(1, self.num_cmds)) + all_locs[:K].view(K, 1, 1, 2)
            o_cmds = self.cast_cmd_pred(embd[:K])
        else:
            o_cast = torch.zeros((0, self.num_cmds, self.num_plan, 2), device=dev)
            o_cmds = torch.zeros((0, self.num_cmds), device=dev)
        return ego_embd, ego_plan_locs, ego_cast_locs, o_cast, o_cmds

    @torch.no_grad()
    def forecast_recorded(self, features, ego_locs, locs, oris, typs):
        """Forecasts of every recorded_rows row and of each ego from crops of the LiDAR ``features`` (logical (B,C,h,w)) at the
        recorded poses: infer_device's crop -> embed (at the embedder's dtype) -> cast / cast_cmd_pred chain, without its
        transform to the ego frame, all rows through one embedder call.  -> dict: frame, slot, cast (K,C,T,2), score (K,C), target
        (K,T,2) of the rows; ego_cast (B,C,T,2), ego_score (B,C), ego_target (B,T,2) = ego_locs[:, 1:]."""
        rows = recorded_rows(ego_locs, locs, oris, typs)
        at, facing, fidx = _forecast_poses(rows, features.shape[0], features.device)
        crops = self.crop_feature(features, at, facing, pixels_per_meter=self.pixels_per_meter / 2, crop_size=self.crop_size,
                                  frame_idx=fidx)
        embd = self.lidar_conv_emb(crops.to(self.lidar_conv_emb[0].conv1.weight.dtype)).float()
        return _forecast_result(rows, self.cast(embd), self.cast_cmd_pred(embd), ego_locs)

    @torch.no_grad()
    def infer(self, features, det, cmd, nxp):
        """UniPlanner.infer (team_code_v2/models/uniplanner.py:186-247): features (C,h,w), B = 1."""
        ee, epl, ecl, ocl, occ = self.infer_batch(features[None], [det], [cmd], nxp[None])
        if len(ocl[0]) == 0:   # reference returns CPU zeros here (uniplanner.py:234-235)
            return epl[0], ecl[0], torch.zeros((0, self.num_cmds, self.num_plan, 2)), torch.zeros((0, self.num_cmds))
        return epl[0], ecl[0], ocl[0], occ[0]


# ----------------------------------------------------------------------------- brake predictor
def positionalencoding1d(d_model, length):
    """sinusoidal table (length, d_model): even columns sin, odd columns cos of position / 10000^(2i/d_model) — the
    positional-encodings package formula the reference's attention pool uses (lav/models/attention.py:41-56)."""
    phase = torch.arange(length, dtype=torch.float32)[:, None] * torch.exp(torch.arange(0, d_model, 2, dtype=torch.float) * -(math.log(10000.0) / d_model))
    return torch.stack([torch.sin(phase), torch.cos(phase)], dim=-1).flatten(1)


class Attention(nn.Module):
    def __init__(self, dim, num_heads=8):
        super().__init__()
        dim_head = dim // num_heads
        self.q = nn.Parameter(torch.randn(1, num_heads, 1, dim_head))
        self.linear_kv = nn.Linear(dim, dim * 2)
        self.num_heads, self.dim_head, self.scale = num_heads, dim_head, dim_head ** -0.5
        self._pe = {}

    def forward(self, x):
        b, d, h, w = x.shape
        x = x.flatten(2).transpose(1, 2)
        k, v = self.linear_kv(x).chunk(2, dim=-1)
        key = (h * w, x.device, x.dtype)
        if key not in self._pe:
            self._pe[key] = positionalencoding1d(d // self.num_heads, h * w).to(x.device, x.dtype)
        k = k.view(b, h * w, self.num_heads, -1).transpose(1, 2) + self._pe[key]
        v = v.view(b, h * w, self.num_heads, -1).transpose(1, 2)
        dots = torch.matmul(self.q.to(x.dtype).expand(b, -1, -1, -1), k.transpose(-1, -2)) * self.scale
        return torch.matmul(torch.softmax(dots, dim=-1), v).transpose(1, 2).reshape(b, d)


class SegmentationHead(nn.Module):
    def __init__(self, input_channels, num_labels):
        super().__init__()
        self.upconv = nn.Sequential(
            nn.ConvTranspose2d(input_channels, 256, 3, 2, 1, 1), nn.BatchNorm2d(256), nn.ReLU(True),
            nn.ConvTranspose2d(256, 128, 3, 2, 1, 1), nn.BatchNorm2d(128), nn.ReLU(True),
            nn.ConvTranspose2d(128, 64, 3, 2, 1, 1), nn.BatchNorm2d(64), nn.ReLU(True),
            nn.Conv2d(64, num_labels, 1, 1, 0))

    def forward(self, x):
        return self.upconv(x)


class Normalize(nn.Module):
    def __init__(self, mean, std):
        super().__init__()
        self.mean = nn.Parameter(torch.tensor(mean), requires_grad=False)
        self.std = nn.Parameter(torch.tensor(std), requires_grad=False)

    def forward(self, x):
        return (x - self.mean[None, :, None, None]) / self.std[None, :, None, None]


class RGBBrakePredictionModel(nn.Module):
    def __init__(self, seg_channels, pretrained=False):
        super().__init__()
        self.conv_backbone = resnet18(pretrained=pretrained)
        self.normalize = Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])
        self.seg_head = SegmentationHead(512, len(seg_channels) + 1)
        self.attn1 = Attention(512, num_heads=8)
        self.attn2 = Attention(512, num_heads=8)
        self.classifier = nn.Sequential(nn.Linear(1024, 1), nn.Sigmoid())

    def forward(self, rgb1, rgb2, mask=False):
        dt = self.conv_backbone.conv1.weight.dtype
        x1 = self.conv_backbone(self.normalize(rgb1 / 255.).to(dt))
        x2 = self.conv_backbone(self.normalize(rgb2 / 255.).to(dt))
        pred_bra = self.classifier(torch.cat([self.attn1(x1), self.attn2(x2)], dim=1).float())
        if mask:
            return (pred_bra[:, 0], F.interpolate(self.seg_head(x1), scale_factor=4), F.interpolate(self.seg_head(x2), scale_factor=4))
        return pred_bra[:, 0]

    @torch.no_grad()
    def forward_u8(self, rgbs_u8, tel_u8):
        """Same as forward(wide, tel) (team_code_v2/lav_agent_fast.py:257-262,318-321) from the raw camera bytes:
        rgbs_u8 (B, 3, 288, 256, 3) — the three cameras, stitched side by side inside the stem kernel — and tel_u8
        (B, 192, 480, 3).  f16 eval only; the mean/std constants are read once (host) and cached."""
        ms = self.__dict__.get("_ms")
        if ms is None:
            ms = self.__dict__["_ms"] = (self.normalize.mean.float().tolist(), self.normalize.std.float().tolist())
        x1 = self.conv_backbone.forward_u8(rgbs_u8, *ms)
        x2 = self.conv_backbone.forward_u8(tel_u8.unsqueeze(1), *ms)
        return self.classifier(torch.cat([self.attn1(x1), self.attn2(x2)], dim=1).float())[:, 0]
