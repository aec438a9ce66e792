"""Training path of the LiDAR perception stack — the ``--perceive-only`` branch of LAV.train_lidar
(lav/lav_final_v2.py:140-259, loss = det_loss + seg_loss at :249-250) — as one process per GPU with an
NCCL gradient all-reduce (SURVEY §8e), replacing nn.DataParallel (lav_final_v2.py:91-94).

What runs where (round 1):
  * voxelise + decorate, pillar max-pool forward and its arg-routed backward: lav_b200 CUDA kernels
    (lavb_pillar_decorate / lavb_pillar_scatter_max / _bwd); the BatchNorm1d in between uses batch statistics over
    all in-window points of the rank's sub-batch, exactly like a DataParallel replica (SURVEY §5).
  * conv / BatchNorm2d forward+backward of the backbone and heads: the module tree's own nn layers (cuDNN) under
    autograd on channels-last tensors — hand-written dgrad/wgrad kernels are the next step of this row.
  * gradient exchange: ``GradAllReducer`` — bucketed (25 MB) asynchronous all-reduce launched from
    post-accumulate-grad hooks while backward is still running; BN statistics stay per rank (as DataParallel).
The full step (``LAVTrainer.train_lidar``) adds the UniPlanner distillation branch — student crops/GRUs with autograd,
frozen BEVPlanner teacher under no_grad (lav_b200/heads.py, pinned bit-exact against the reference on CPU) — and the
motion losses of lav_final_v2.py:190-225.
"""
import contextlib
import dataclasses

import torch
import torch.distributed as dist
from torch import nn
from torch.nn import functional as F


# --------------------------------------------------------------------------- training-mode forward
def lidar_model_train_forward(model, lidars, num_points):
    """LiDARModel.forward in train mode (lidar.py:34-45) -> (features, center, box, ori, seg), logical NCHW."""
    canvas = model.point_pillar_net(lidars, num_points)            # CUDA pillar path with autograd (point_pillar.py)
    bb = model.backbone
    x1 = bb.conv1(canvas)
    x2 = bb.conv2(x1)
    x3 = bb.conv3(x2)
    feats = torch.cat([bb.upconv1(x1), bb.upconv2(x2), bb.upconv3(x3)], dim=1)
    heads = (model.center_head, model.box_head, model.ori_head, model.seg_head)
    hidden = _heads_trunk_fused(heads, feats) if FUSE_HEADS_TRAIN else None
    outs = []
    for i, h in enumerate(heads):
        y = h.net(feats) if hidden is None else h.net[3](hidden[i])
        outs.append(h.output_activation(y) if h.output_activation else y)
    return (feats, *outs)


FUSE_HEADS_TRAIN = True


def _heads_trunk_fused(heads, feats):
    """Conv(384->64) -> ReLU -> BatchNorm of the four heads (lidar.py:14-27) as ONE 384->256 convolution and one 256-channel
    batch norm (statistics are per channel, so this is the same function): the 1.26 GB feature map is read by one fprop and
    one wgrad instead of four, and one dgrad writes its gradient instead of four dgrads + three full-size additions.  The
    parameters stay the heads' own (state_dict unchanged); running statistics are written back to each head's BatchNorm.
    Returns the per-head hidden maps, or None when the heads do not share one configuration."""
    convs, bns = [h.net[0] for h in heads], [h.net[2] for h in heads]
    c0, b0 = convs[0], bns[0]
    same = all(isinstance(c, nn.Conv2d) and c.bias is None and c.weight.shape == c0.weight.shape and c.stride == c0.stride and
               c.padding == c0.padding and c.dilation == c0.dilation and c.groups == 1 for c in convs)
    same = same and all(isinstance(b, nn.BatchNorm2d) and b.training and b.affine and b.track_running_stats and b.momentum is not None
                        and b.momentum == b0.momentum and b.eps == b0.eps for b in bns)
    same = same and all(isinstance(h.net[1], nn.ReLU) and len(h.net) == 4 for h in heads)
    if not same:
        return None
    y = F.conv2d(feats, torch.cat([c.weight for c in convs]), None, c0.stride, c0.padding, c0.dilation)
    y = F.relu_(y)
    mean, var = torch.cat([b.running_mean for b in bns]), torch.cat([b.running_var for b in bns])
    y = F.batch_norm(y, mean, var, torch.cat([b.weight for b in bns]), torch.cat([b.bias for b in bns]), True, b0.momentum, b0.eps)
    with torch.no_grad():
        n = b0.num_features
        for i, b in enumerate(bns):
            b.running_mean.copy_(mean[i * n:(i + 1) * n])
            b.running_var.copy_(var[i * n:(i + 1) * n])
            b.num_batches_tracked += 1
    return y.split(b0.num_features, dim=1)


# --------------------------------------------------------------------------- losses
# The eight loss terms of LAV.train_lidar (lav/lav_final_v2.py:177-225 + lav/models/loss.py:5-27), written as pure functions
# of the model outputs so they can be pinned against the reference's own train_lidar (oracle/pin_against_reference.py runs
# it on stub sub-models -> tests/golden/train_losses.npz).
@dataclasses.dataclass
class LossConfig:
    """config_v2.yaml:14-18,48,57-62 (`distill` is read by train_lidar but absent from the released configs: explicit here)."""
    box_weight: float = 1.0
    ori_weight: float = 1.0
    seg_weight: float = 2.0
    perception_weight: float = 4.0
    other_weight: float = 0.5
    cmd_weight: float = 0.1
    cmd_smooth: float = 0.2
    branch_weights: tuple = (5, 5, 5, 1, 1, 1)
    distill: bool = True
    perceive_only: bool = False
    motion_only: bool = False


def _weighted_ratio(values, weights):
    """mean(values * weights) / mean(weights): the focal-style normalisation of loss.py:21-24 (the weights broadcast over
    channels, so the two means run over different element counts — kept as two means on purpose)."""
    return (values * weights).mean() / weights.mean()


def detection_losses(pred_heat, heat, pred_size, size, pred_ori, ori):
    """DetLoss.forward (lav/models/loss.py:14-27) -> (heat-map, box, orientation) losses.
    Heat-map: per-pixel BCE-with-logits weighted by the probability of being WRONG, sigmoid(logit * (1 - 2 target));
    box / orientation: smooth-L1 weighted by the per-pixel peak of the target heat-maps."""
    wrong = torch.sigmoid(pred_heat * (1.0 - 2.0 * heat))
    peak = heat.amax(dim=1, keepdim=True)
    hm = _weighted_ratio(F.binary_cross_entropy_with_logits(pred_heat, heat, reduction="none"), wrong)
    box = _weighted_ratio(F.smooth_l1_loss(pred_size, size, reduction="none"), peak)
    ang = _weighted_ratio(F.smooth_l1_loss(pred_ori, ori, reduction="none"), peak)
    return hm, box, ang


class DetLoss(nn.Module):
    """module form with the reference's name and call signature (lav/models/loss.py:5)."""

    def forward(self, pred_heatmaps, heatmaps, pred_sizemaps, sizemaps, pred_orimaps, orimaps):
        return detection_losses(pred_heatmaps, heatmaps, pred_sizemaps, sizemaps, pred_orimaps, orimaps)


def build_seg_mask(w=320, h=320, cx=160, cy=280, radius_x=240, radius_y=240):
    """LAV.build_seg_mask (lav_final_v2.py:261-271): an (h, w) Gaussian bump centred on the ego (the reference builds it as a
    max over a trailing singleton axis of the outer product of the two 1-D profiles)."""
    gx = torch.exp(-((torch.arange(w, dtype=torch.float32) - cx) / radius_x) ** 2)
    gy = torch.exp(-((torch.arange(h, dtype=torch.float32) - cy) / radius_y) ** 2)
    return gy[:, None] * gx[None, :]


def train_losses(outs, planner_out, heatmaps, sizemaps, orimaps, bev, ego_locs, cmds, bras, seg_mask, cfg=None, branch_weights=None):
    """-> (total loss, dict of the 8 terms).  outs = LiDARModel outputs (features, heat logits, sizes, orientations, sigmoid BEV);
    planner_out = the 11 UniPlanner.forward outputs; targets as LAV.train_lidar receives them."""
    cfg = cfg or LossConfig()
    _, pred_heat, pred_size, pred_ori, pred_bev = outs
    (other_next, other_cast, other_cmds, other_cast_teacher, other_cmds_teacher, _ego_next, ego_plan, ego_cast, ego_cmds,
     ego_cast_teacher, ego_plan_teacher) = planner_out
    cmds = cmds.long()
    rows = torch.arange(cmds.shape[0], device=cmds.device)
    hm, box, ang = detection_losses(pred_heat, heatmaps, pred_size, sizemaps, pred_ori, orimaps)
    det = hm + cfg.box_weight * box + cfg.ori_weight * ang
    seg = (F.binary_cross_entropy(pred_bev, bev.float()[:, :3], reduction="none") * seg_mask).mean() * cfg.seg_weight
    # plan: every refinement iteration and every command branch regresses the teacher's LAST-iteration plan of the COMMANDED
    # branch; per-sample mean, weighted by the branch weight of that sample's command
    bw = branch_weights if branch_weights is not None else torch.tensor(cfg.branch_weights, dtype=torch.float32, device=ego_plan.device)
    goal = ego_plan_teacher[rows, -1, cmds]                                                   # (B, T, 2)
    plan = ((ego_plan - goal[:, None, None]).abs().flatten(1).mean(1) * bw[cmds]).mean()
    if cfg.distill:
        ego_c = (ego_cast - ego_cast_teacher).abs().mean()
        other_c = (other_cast - other_cast_teacher).abs().mean()
        cmd = F.binary_cross_entropy(other_cmds, other_cmds_teacher)
    else:
        moving = (1 - bras).bool().to(cmds.device)                                             # samples without a brake label
        ego_c = (ego_cast[rows, cmds] - ego_locs[:, 1:].float()).abs().flatten(1).mean(1)[moving].mean()
        other_c = (other_cast - other_next[:, None]).abs().mean(dim=(2, 3)).amin(dim=1).mean()   # best branch per vehicle
        k = ego_cmds.shape[1]
        cmd = F.binary_cross_entropy(ego_cmds, (1.0 - cfg.cmd_smooth) * F.one_hot(cmds, k) + cfg.cmd_smooth / k)
    motion = plan + ego_c + cfg.other_weight * other_c + cfg.cmd_weight * cmd
    if cfg.perceive_only:
        total = det + seg
    elif cfg.motion_only:
        total = motion
    else:
        total = motion + cfg.perception_weight * (det + seg)
    return total, dict(hm_loss=hm, box_loss=box, ori_loss=ang, seg_loss=seg, plan_loss=plan, ego_cast_loss=ego_c,
                       other_cast_loss=other_c, cmd_loss=cmd)


def perception_loss(outs, heatmaps, sizemaps, orimaps, seg_bev, seg_mask, box_weight=1.0, ori_weight=1.0, seg_weight=2.0):
    """det_loss + seg_loss only (the --perceive-only branch, lav_final_v2.py:177-188,249-250)."""
    _, ph, ps, po, pb = outs
    hm, box, ang = detection_losses(ph, heatmaps, ps, sizemaps, po, orimaps)
    seg = (F.binary_cross_entropy(pb, seg_bev, reduction="none") * seg_mask).mean() * seg_weight
    return hm + box_weight * box + ori_weight * ang + seg, dict(hm_loss=hm.detach(), box_loss=box.detach(), ori_loss=ang.detach(),
                                                                seg_loss=seg.detach())


# --------------------------------------------------------------------------- data-parallel gradient exchange
class GradAllReducer:
    """Bucketed, overlapped gradient all-reduce (mean) for one-process-per-GPU data parallelism.

    Parameters are packed into flat buckets in reverse registration order (the order autograd finishes them);
    when the last gradient of a bucket has been accumulated — and every earlier bucket has been launched — its all-reduce
    starts asynchronously (NCCL on GPUs, gloo in the CPU tests); ``finish()`` waits for all buckets and scatters the averaged
    values back.

    Normalisation note: the reference trains under nn.DataParallel, whose losses see the GATHERED full batch, so its ratio terms
    (``(...).mean() / p_det.mean()``, ``/ size_w.mean()``, ``[idxs].mean()``, lav/models/loss.py:14-24, lav_final_v2.py:205) are
    normalised over all samples.  Here every rank normalises over its own sub-batch and the gradients are averaged: identical
    when the per-rank normalisers are equal, a per-rank re-weighting of those loss terms otherwise (standard DDP behaviour).
    """

    def __init__(self, params, bucket_bytes=25 << 20, group=None):
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.params = [p for p in params if p.requires_grad]
        self.buckets, cur, size = [], [], 0
        for p in reversed(self.params):
            cur.append(p)
            size += p.numel() * p.element_size()
            if size >= bucket_bytes:
                self.buckets.append(cur)
                cur, size = [], 0
        if cur:
            self.buckets.append(cur)
        self._flat = [torch.zeros(sum(p.numel() for p in b), dtype=b[0].dtype, device=b[0].device) for b in self.buckets]
        self._where, self._views = {}, []
        for bi, b in enumerate(self.buckets):
            off, views = 0, []
            for p in b:
                self._where[p] = (bi, off)
                views.append(self._flat[bi][off:off + p.numel()].view_as(p))
                off += p.numel()
            self._views.append(views)
        self._pending = [0] * len(self.buckets)
        self._works = [None] * len(self.buckets)
        self._hooks = [p.register_post_accumulate_grad_hook(self._on_grad) for p in self.params]
        self.reset()

    def reset(self):
        self._pending = [len(b) for b in self.buckets]
        self._works = [None] * len(self.buckets)
        self._next = 0            # buckets are reduced STRICTLY in index order: every rank issues the same collectives in the
                                  # same order even when the set of parameters that received a gradient differs between ranks

    def _pack(self, bi):
        """gradients of bucket bi -> its flat buffer: ONE multi-tensor copy (zeros for parameters that received no gradient)"""
        have = [(v, p.grad) for v, p in zip(self._views[bi], self.buckets[bi]) if p.grad is not None]
        for v, p in zip(self._views[bi], self.buckets[bi]):
            if p.grad is None:
                v.zero_()
        if have:
            torch._foreach_copy_([v for v, _ in have], [g for _, g in have])

    def _launch_ready(self):
        while self._next < len(self.buckets) and self._pending[self._next] == 0:
            bi = self._next
            if self.world > 1:
                self._pack(bi)
                self._works[bi] = dist.all_reduce(self._flat[bi], op=dist.ReduceOp.SUM, group=self.group, async_op=True)
            self._next += 1

    def _on_grad(self, p):
        bi, _ = self._where[p]
        self._pending[bi] -= 1
        if self._pending[bi] == 0:
            self._launch_ready()

    def finish(self):
        """wait for the exchanges and write the averaged gradients back into ``p.grad``; call before optimizer.step().
        Buckets with a parameter that received no gradient this step are completed with zeros and reduced here, still in
        index order.  With one rank nothing is copied or reduced: the gradients stay where autograd put them."""
        for bi in range(len(self.buckets)):
            self._pending[bi] = 0
        self._launch_ready()
        if self.world > 1:
            for bi, b in enumerate(self.buckets):
                if self._works[bi] is not None:
                    self._works[bi].wait()
                self._flat[bi].div_(self.world)
                for v, p in zip(self._views[bi], b):
                    if p.grad is None:
                        p.grad = torch.empty_like(p)
                torch._foreach_copy_([p.grad for p in b], self._views[bi])
        self.reset()

    def close(self):
        for h in self._hooks:
            h.remove()


class PerceptionTrainer:
    """Adam + StepLR on the LiDAR model as in LAV.__init__ (lav_final_v2.py:74-89), one process per GPU."""

    def __init__(self, lidar_model, lr=3e-4, device=None, bucket_bytes=25 << 20):
        self.model = lidar_model.train()
        self.device = device or next(lidar_model.parameters()).device
        self.optim = torch.optim.Adam(self.model.parameters(), lr=lr)
        self.sched = torch.optim.lr_scheduler.StepLR(self.optim, step_size=4, gamma=0.5)
        self.reducer = GradAllReducer(self.model.parameters(), bucket_bytes)
        self.seg_mask = build_seg_mask().to(self.device)

    def train_step(self, lidars, num_points, heatmaps, sizemaps, orimaps, bev):
        """one train_lidar step on this rank's sub-batch (perceive-only losses)."""
        seg_bev = bev[:, [0, 1, 2]].float()
        outs = lidar_model_train_forward(self.model, lidars, num_points)
        loss, parts = perception_loss(outs, heatmaps, sizemaps, orimaps, seg_bev, self.seg_mask)
        self.optim.zero_grad(set_to_none=True)
        loss.backward()
        self.reducer.finish()
        self.optim.step()
        return loss.detach(), parts


class LAVTrainer:
    """LAV.train_lidar (lav/lav_final_v2.py:140-259) as one process per GPU: LiDAR model + UniPlanner student trained
    against the frozen BEVPlanner teacher; Adam over the same parameter set (:74-86), gradients averaged across ranks by
    GradAllReducer.  Config values default to config_v2.yaml / team_code_v2/config.yaml."""

    def __init__(self, lidar_model, uniplanner, lr=3e-4, device=None, box_weight=1.0, ori_weight=1.0, seg_weight=2.0,
                 perception_weight=4.0, other_weight=0.5, cmd_weight=0.1, branch_weights=(5, 5, 5, 1, 1, 1), distill=True,
                 cmd_smooth=0.2, perceive_only=False, motion_only=False, bucket_bytes=25 << 20, amp=False, channels_last=True):
        self.lidar_model, self.uniplanner = lidar_model.train(), uniplanner.train()
        if channels_last and next(lidar_model.parameters()).is_cuda:
            # NHWC convolution weights (values and state_dict unchanged): cuDNN's tensor-core kernels are NHWC — this removes most of
            # the nchw<->nhwc conversion kernels around them
            lidar_model.to(memory_format=torch.channels_last)
            uniplanner.to(memory_format=torch.channels_last)
        uniplanner.bev_planner.eval()
        for p in uniplanner.bev_planner.parameters():
            p.requires_grad_(False)
        self.device = device or next(lidar_model.parameters()).device
        up = uniplanner
        params = (list(up.plan_gru.parameters()) + list(up.plan_mlp.parameters()) + list(up.cast_grus_ego.parameters()) +
                  list(up.cast_mlps_ego.parameters()) + list(up.cast_grus_other.parameters()) + list(up.cast_mlps_other.parameters()) +
                  list(up.cast_cmd_pred.parameters()) + list(up.lidar_conv_emb.parameters()))
        if not motion_only:
            params += list(lidar_model.parameters())
        self.params = params
        self.optim = torch.optim.Adam(params, lr=lr)
        self.sched = torch.optim.lr_scheduler.StepLR(self.optim, step_size=4, gamma=0.5)
        self.reducer = GradAllReducer(params, bucket_bytes)
        self.seg_mask = build_seg_mask().to(self.device)
        self.branch_weights = torch.tensor(branch_weights).float().to(self.device)
        self.cfg = LossConfig(box_weight, ori_weight, seg_weight, perception_weight, other_weight, cmd_weight, cmd_smooth,
                              tuple(branch_weights), distill, perceive_only, motion_only)
        self.perceive_only, self.motion_only = perceive_only, motion_only
        # amp=True: LiDAR-model forward under bf16 autocast (fp32 master weights; planner, losses and Adam in fp32).  The
        # reference trains in fp32 (cuDNN TF32); opt-in, off by default: measured no faster (the step is not conv-bound).
        self.amp = bool(amp)

    def losses(self, lidars, num_points, heatmaps, sizemaps, orimaps, bev, ego_locs, cmds, nxps, bras, locs, oris, typs):
        up = self.uniplanner
        bev = bev.float()
        # amp: only the LiDAR model (pillars, backbone, heads — the convolutions) runs under bf16 autocast; the planner (cuDNN
        # GRUs, crops, embedder) and every loss stay fp32 — cuDNN's bf16 RNN path faulted on these shapes (cuDNN 9)
        ctx = torch.autocast("cuda", dtype=torch.bfloat16) if self.amp else contextlib.nullcontext()
        with ctx:
            outs = self.lidar_model(lidars, num_points)
        if self.amp:
            outs = tuple(t.float() for t in outs)
        planner_out = up(outs[0], bev, ego_locs.float(), locs.float(), oris.float(), nxps.float(), typs)
        loss, parts = train_losses(outs, planner_out, heatmaps, sizemaps, orimaps, bev, ego_locs, cmds, bras, self.seg_mask, self.cfg,
                                   self.branch_weights)
        return loss, {k: v.detach() for k, v in parts.items()}

    def train_lidar(self, *batch):
        """batch = the 14-tuple of TemporalLiDARPaintedDataset (temporal_lidar_painted_dataset.py:172-179) minus num_objs:
        lidars, num_points, heatmaps, sizemaps, orimaps, bev, ego_locs, cmds, nxps, bras, locs, oris, typs"""
        loss, parts = self.losses(*batch[:13])
        self.optim.zero_grad(set_to_none=True)
        loss.backward()
        self.reducer.finish()
        self.optim.step()
        return loss.detach(), parts


# --------------------------------------------------------------------------- privileged planner (stage 1 of the v2 recipe)
def bev_losses(planner_out, ego_locs, cmds, bras, branch_weights, other_weight=0.0, cmd_weight=0.1, cmd_smooth=0.2):
    """LAV.train_bev's losses (lav/lav_privileged_v2.py:131-142) term for term -> (total loss, dict of the 4 terms).
    planner_out = the 6 BEVPlanner.forward outputs; ego_locs (B,T+1,2), cmds (B,), bras (B,) 0/1.
      plan_loss      L1 of every iteration and command branch of the plan against the ego's future, mean per sample over the
                     samples WITHOUT a brake label only, weighted by the branch weight of the command (NaN when all brake)
      ego_cast_loss  L1 of the commanded cast branch against the ego's future, over all samples
      other_cast_loss L1 of the best command branch per forecast vehicle, scaled by ``other_weight`` in the total
      cmd_loss       BCE of the command scores against smoothed one-hot targets, scaled by ``cmd_weight`` in the total"""
    other_next, other_cast, _other_cmds, ego_plan, ego_cast, ego_cmds = planner_out
    cmds = cmds.long()
    moving = (1 - bras).bool().to(cmds.device)
    n_iter, n_cmds, T = ego_plan.shape[1], ego_plan.shape[2], ego_plan.shape[3]
    future = ego_locs[:, 1:]
    plan = torch.mean(F.l1_loss(ego_plan, future[:, None, None].repeat(1, n_iter, n_cmds, 1, 1), reduction="none")
                      .mean(dim=[1, 2, 3, 4])[moving] * branch_weights[cmds[moving]])
    commanded = ego_cast.gather(1, cmds.expand(T, 2, 1, -1).permute(3, 2, 0, 1)).squeeze(1)
    ego_c = F.l1_loss(commanded, future, reduction="none").mean(dim=[1, 2]).mean()
    other_c = F.l1_loss(other_cast, other_next.unsqueeze(1).repeat(1, n_cmds, 1, 1), reduction="none").mean(dim=[2, 3]).min(1)[0].mean()
    cmd = F.binary_cross_entropy(ego_cmds, (1.0 - cmd_smooth) * F.one_hot(cmds, n_cmds) + cmd_smooth / n_cmds)
    total = plan + ego_c + other_c * other_weight + cmd * cmd_weight
    return total, dict(plan_loss=plan, ego_cast_loss=ego_c, other_cast_loss=other_c, cmd_loss=cmd)


def other_weight_schedule(it, beta=0.8):
    """weight of the other-vehicle forecast loss at global step ``it`` (lav/train_bev_v2.py:36-37): 0 at the start, -> 1."""
    return 1 - beta ** (it / 4000)


class BEVTrainer:
    """LAV.train_bev (lav/lav_privileged_v2.py:110-160) as one process per GPU: Adam at ``lr`` over every BEVPlanner parameter,
    StepLR(32, 0.5) stepped once per epoch by the caller (``sched``), gradients averaged across ranks by GradAllReducer.
    Precision as LAVTrainer: fp32 tensors under PyTorch's defaults (cuDNN convolutions may use TF32, as in the reference).
    The map may stay uint8 on the GPU: BEVPlanner.forward crops it with the lav_b200 kernel instead of a float copy."""

    def __init__(self, bev_planner, lr=3e-4, device=None, branch_weights=(5, 5, 5, 1, 1, 1), cmd_weight=0.1, cmd_smooth=0.2,
                 use_others_to_train=True, bucket_bytes=25 << 20):
        self.model = bev_planner.train()
        self.device = device or next(bev_planner.parameters()).device
        self.optim = torch.optim.Adam(self.model.parameters(), lr=lr)
        self.sched = torch.optim.lr_scheduler.StepLR(self.optim, step_size=32, gamma=0.5)
        self.reducer = GradAllReducer(self.model.parameters(), bucket_bytes)
        self.branch_weights = torch.tensor(branch_weights).float().to(self.device)
        self.cmd_weight, self.cmd_smooth, self.use_others_to_train = cmd_weight, cmd_smooth, bool(use_others_to_train)

    def other_weight(self, it):
        return other_weight_schedule(it) if self.use_others_to_train else 0.0

    def losses(self, bev, ego_locs, cmds, nxps, bras, locs, oris, typs, other_weight=0.0):
        dev = self.device
        if not self.use_others_to_train:
            other_weight = 0.0
        ego_locs = ego_locs.float().to(dev)
        out = self.model(bev.to(dev), ego_locs, locs.float().to(dev), oris.float().to(dev), nxps.float().to(dev), typs.to(dev))
        loss, parts = bev_losses(out, ego_locs, cmds.to(dev), bras.to(dev), self.branch_weights, other_weight, self.cmd_weight,
                                 self.cmd_smooth)
        return loss, {k: v.detach() for k, v in parts.items()}

    def train_bev(self, bev, ego_locs, cmds, nxps, bras, locs, oris, typs, num_objs=None, other_weight=0.0):
        """one step on this rank's sub-batch: the 9-tuple of TemporalBEVDataset (num_objs unused, as in the reference)."""
        loss, parts = self.losses(bev, ego_locs, cmds, nxps, bras, locs, oris, typs, other_weight)
        self.optim.zero_grad(set_to_none=True)
        loss.backward()
        self.reducer.finish()
        self.optim.step()
        return loss.detach(), parts


def synthetic_train_batch(B, device, seed=2021, n_points=(60000, 120000), n_obj=6):
    """seeded batch with the shapes of SURVEY 8(a) a18: lidar (B,120000,11), maps (B,2,320,320), bev (B,9,320,320) ..."""
    from . import synth
    g = synth._gen(seed, f"train{B}")
    P = 120000
    lid = torch.zeros(B, P, 11)
    npts = []
    for b in range(B):
        n = int(torch.randint(n_points[0], n_points[1] + 1, (1,), generator=g))
        pts = synth.stacked_lidar(40000, seed=seed, tag=f"tb{b}")[:n]
        lid[b, :len(pts)] = pts
        npts.append(len(pts))
    yy, xx = torch.meshgrid(torch.arange(320.), torch.arange(320.), indexing="ij")
    heat = torch.zeros(B, 2, 320, 320)
    for b in range(B):
        for k in range(6):
            cx, cy = (torch.rand(2, generator=g) * 320).tolist()
            heat[b, k % 2] = torch.maximum(heat[b, k % 2], torch.exp(-((xx - cx) ** 2 + (yy - cy) ** 2) / 18.0))
    size = torch.rand(B, 2, 320, 320, generator=g) * 3
    ori = torch.randn(B, 2, 320, 320, generator=g)
    bev = (torch.rand(B, 9, 320, 320, generator=g) > 0.7).to(torch.uint8)
    ego_locs = torch.cumsum(torch.rand(B, 21, 2, generator=g) * torch.tensor([0.2, -1.0]), dim=1)
    locs = torch.randn(B, n_obj, 21, 2, generator=g) * 6 + torch.tensor([0.0, -8.0])
    locs[:, 0] = ego_locs
    oris = torch.rand(B, n_obj, generator=g) * 0.6 - 0.3
    typs = (torch.rand(B, n_obj, generator=g) > 0.3).long()
    cmds = torch.randint(0, 6, (B,), generator=g)
    nxps = torch.tensor([[0.0, -20.0]]).repeat(B, 1) + torch.randn(B, 2, generator=g)
    bras = (torch.rand(B, generator=g) > 0.8).long()
    to = lambda t: t.to(device)
    return (to(lid), torch.tensor(npts), to(heat), to(size), to(ori), to(bev), to(ego_locs), to(cmds), to(nxps), to(bras), to(locs),
            to(oris), to(typs))
