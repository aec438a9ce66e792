"""Device-side pieces of the training data pipeline — the per-sample LiDAR work and the detection-target rasterisation of
`TemporalLiDARPaintedDataset.__getitem__` (lav/utils/datasets/temporal_lidar_painted_dataset.py:13-179) and
`LiDARDataset.detections_to_heatmap` (lav/utils/datasets/lidar_dataset.py:92-127).

In the reference these run in 16 numpy / OpenCV DataLoader workers per GPU; at 8 x H100 the loader, not the GPUs, bounds the
training step (SURVEY 8f rank 4).  Here the record reads stay on the host (key-value store, see data_paint.py) and everything that
touches the points runs on the GPU with the frame path's own kernels:

    roof filter (order-preserving)         LiDARDataset.preprocess, lidar_dataset.py:14-23          lavb_roof_filter
    rotation jitter                        rotate_lidar(-angle), :175-182                           lavb_stack_sweep (R only)
    re-mask painted features by camera FOV point_painting(xyzr, ones) after the rotation, :58-60     lavb_paint (mode 0 on a ones map)
    ego-motion + jitter + time one-hot     move_lidar_points, :159-177 / :62-66,80-87                lavb_stack_sweep
    shuffle, truncate to max_lidar_points, zero-pad  :89-91,131-133                                  torch.randperm + copies
    heat / size / orientation maps         detections_to_heatmap                                    vectorised torch on the device
A training batch takes the batched path instead: GpuLidarStacker.batch_tables does the roof filter, the shuffle, the truncation
and the padding on row indices on the host, and one lavb_lidar_batch launch builds every LiDAR row of the batch; one
lavb_det_heatmaps launch builds every sample's maps.  Both are bit-identical to the per-sample path above, which stays as their
reference.
Not here (host, as in the reference): LMDB reads, the actor filter, BEV image loading and its cv2 rotation.
"""
import math

import numpy as np
import torch

from . import ops
from . import point_painting as PP


class GpuLidarStacker:
    """The LiDAR half of TemporalLiDARPaintedDataset.__getitem__ for one sample, on ``device``."""

    def __init__(self, num_frame_stack=2, seg_channels=4, max_lidar_points=120000, camera_x=1.5, camera_z=2.4, rgb_hw=(288, 256),
                 device=torch.device("cuda")):
        self.T, self.C, self.max_points, self.device, self.rgb_hw = num_frame_stack + 1, seg_channels, max_lidar_points, device, rgb_hw
        self.cams = np.stack([c.packed() for c in PP.make_converters(camera_x, camera_z, rgb_hw[0], rgb_hw[1])])
        self.ones = torch.ones((len(self.cams), 1, rgb_hw[0], rgb_hw[1]), device=device)       # `self.dummy` of the reference

    @torch.no_grad()
    def __call__(self, sweeps, angle_deg, jitters=None, generator=None):
        """sweeps: [(xyzr (n,4), painted (n,C), ego_loc (2,), ego_ori)] newest first (index, index-1, ...), numpy or tensors;
        angle_deg: the sample's rotation jitter; jitters[i] = (loc_jitter (2,), ori_jitter) of sweep i (zeros for i = 0).
        Returns (lidar (max_points, 4+C+T) fp32 zero-padded, num_points)."""
        dev = self.device
        R_aug, moves = sweep_transforms(sweeps, angle_deg, jitters)
        rows = []
        for i, (xyzr, painted, loc, ori) in enumerate(sweeps):
            raw = torch.cat([torch.as_tensor(xyzr, dtype=torch.float32), torch.as_tensor(painted, dtype=torch.float32)], 1).to(dev).contiguous()
            kept, cnt = ops.roof_filter(raw)                                                 # preprocess (both arrays, same rows)
            kept = kept[:int(cnt[0])].contiguous()
            n = kept.shape[0]
            rot = torch.empty((n, 4 + self.C), device=dev)
            ops.stack_sweep(kept, R_aug, 0.0, 0.0, 0, 0, rot)                                # rotate_lidar(xyzr, -angle)
            vis = ops.paint(rot, self.ones, self.cams, mode=0)                               # 1 where some camera still sees the point
            rot[:, 4:] *= vis
            R_mv, dloc = moves[i]
            out = torch.empty((n, 4 + self.C + self.T), device=dev)
            ops.stack_sweep(rot, R_mv, dloc[0], dloc[1], i, self.T, out)                     # move_lidar_points + one-hot(t)
            rows.append(out)
        lidar = torch.cat(rows)
        total = lidar.shape[0]
        perm = torch.randperm(total, generator=generator, device=dev if generator is None or generator.device.type == "cuda" else "cpu").to(dev)
        lidar = lidar[perm[:self.max_points]]
        padded = torch.zeros((self.max_points, lidar.shape[1]), device=dev)
        num = min(self.max_points, total)
        padded[:num] = lidar[:num]
        return padded, num

    def batch_tables(self, samples, generator=None, paint=False):
        """The host half of a batch: samples = [(sweeps, angle_deg, jitters)] as __call__ takes them, sweeps numpy.  Draws each
        sample's permutation from ``generator`` (a CPU torch.Generator; None = torch's default CPU generator) with the sizes and in
        the order of one __call__ per sample, and composes it with the kept rows of the roof filter.  No device work.
        -> dict(raw (N, 4+C) fp32, rows (B, P) int32, sweeps LIDAR_SWEEP_DTYPE records, nums list): raw and rows are pinned
        CPU tensors when the stacker's device is CUDA.  With ``paint`` (online painting) the second entry of each sweep is its
        frame slot instead of its painted rows: raw is (N, 4) and the dict also holds slots (n_sweeps,) int32, pinned likewise."""
        pin = torch.device(self.device).type == "cuda"
        n_raw = sum(len(sw[0]) for sweeps, _, _ in samples for sw in sweeps)
        raw = torch.empty((n_raw, 4 if paint else 4 + self.C), dtype=torch.float32, pin_memory=pin)
        rows = torch.full((len(samples), self.max_points), -1, dtype=torch.int32, pin_memory=pin)
        a, r = raw.numpy(), rows.numpy()
        table = np.zeros(sum(len(sweeps) for sweeps, _, _ in samples), ops.LIDAR_SWEEP_DTYPE)
        slots = torch.zeros(len(table), dtype=torch.int32, pin_memory=pin) if paint else None
        r0, s, nums = 0, 0, []
        for b, (sweeps, angle_deg, jitters) in enumerate(samples):
            R_aug, moves = sweep_transforms(sweeps, angle_deg, jitters)
            kept = []
            for i, (xyzr, painted, _, _) in enumerate(sweeps):
                n = len(xyzr)
                if paint:
                    a[r0:r0 + n], slots[s] = xyzr, int(painted)
                else:
                    a[r0:r0 + n, :4], a[r0:r0 + n, 4:] = xyzr, painted
                kept.append(r0 + np.flatnonzero(roof_keep(a[r0:r0 + n])))
                R_mv, dloc = moves[i]
                table[s] = (R_aug.ravel(), R_mv.ravel(), dloc[0], dloc[1], i, r0)
                r0, s = r0 + n, s + 1
            kept = np.concatenate(kept)
            perm = torch.randperm(len(kept), generator=generator, device="cpu").numpy()
            num = min(self.max_points, len(kept))
            r[b, :num] = kept[perm[:num]]
            nums.append(num)
        out = dict(raw=raw, rows=rows, sweeps=table, nums=nums)
        if paint:
            out["slots"] = slots
        return out

    @torch.no_grad()
    def batch_launch(self, t, painting=None):
        """The device half: H2D copies of the tables and one lavb_lidar_batch launch -> (B, P, 4+C+T) fp32.  Tables made with
        ``paint`` take painting = (features of the frame slots' images, their deconv table, n_classes) of forward_features_nhwc
        and one lavb_lidar_batch_paint launch instead."""
        dev = self.device
        raw, rows = t["raw"].to(dev, non_blocking=True), t["rows"].to(dev, non_blocking=True)
        sweeps = ops._to_device(t["sweeps"].view(np.uint8), dev)
        if "slots" in t:
            feat, table, n_classes = painting
            return ops.lidar_batch_paint(raw, rows, sweeps, t["slots"].to(dev, non_blocking=True), feat, n_classes, table,
                                         self.cams, self.rgb_hw, self.T)
        return ops.lidar_batch(raw, rows, sweeps, self.cams, self.rgb_hw, self.T)

    def batch(self, samples, generator=None):
        """__call__ for every sample of a batch, in one launch: -> (lidar (B, P, 4+C+T) fp32, nums list), bit-identical to
        stacking one __call__ per sample in order with the same generator."""
        t = self.batch_tables(samples, generator)
        return self.batch_launch(t), t["nums"]


def sweep_transforms(sweeps, angle_deg, jitters):
    """GpuLidarStacker's per-sample rotation R_aug (rotate_lidar(-angle)) and per-sweep (R_mv, dloc) (move_lidar_points to the
    newest sweep's ego frame, with the stack jitters): 3x3 fp32 matrices, dloc (2,) fp64."""
    loc0, ori0 = np.asarray(sweeps[0][2], dtype=np.float64), float(sweeps[0][3])
    rad = math.radians(-angle_deg)
    R_aug = np.array([[math.cos(rad), math.sin(rad), 0], [-math.sin(rad), math.cos(rad), 0], [0, 0, 1]], dtype=np.float32)
    moves = []
    for i, (_, _, loc, ori) in enumerate(sweeps):
        lj, oj = (np.zeros(2), 0.0) if (jitters is None or i == 0) else jitters[i]
        dloc = (np.asarray(loc, dtype=np.float64) - loc0 + np.asarray(lj)) @ np.array([[math.cos(ori0), -math.sin(ori0)], [math.sin(ori0), math.cos(ori0)]])
        d = float(ori) + float(oj) - ori0
        R_mv = np.array([[math.cos(d), math.sin(d), 0], [-math.sin(d), math.cos(d), 0], [0, 0, 1]], dtype=np.float32)
        moves.append((R_mv, dloc))
    return R_aug, moves


_ROOF = tuple(np.float32(v) for v in (-2.4, 0, -0.8, 0.8, -1.5, -1))


def roof_keep(rows):
    """LAVAgent.preprocess's keep mask on (n, >=3) fp32 rows: lavb_roof_filter's fp32 predicate (NaN rows are kept)."""
    x, y, z = rows[:, 0], rows[:, 1], rows[:, 2]
    x0, x1, y0, y1, z0, z1 = _ROOF
    return ~((x > x0) & (x < x1) & (y > y0) & (y < y1) & (z > z0) & (z < z1))


@torch.no_grad()
def detections_to_heatmap(locs, oris, bbox, typs, min_x=-10, max_x=70, min_y=-40, max_y=40, pixels_per_meter=4, radius=1,
                          device=torch.device("cuda")):
    """LiDARDataset.detections_to_heatmap (lidar_dataset.py:92-127) on the device.  locs (N,2) ego-frame metres, oris (N,),
    bbox (N,2), typs (N,) in {0: pedestrian, 1: vehicle} -> heatmap (2,h,w), sizemap (2,h,w), orimap (2,h,w)."""
    h, w = (max_y - min_y) * pixels_per_meter, (max_x - min_x) * pixels_per_meter              # len(y_edges), len(x_edges)
    heat = torch.zeros((2, h, w), device=device)
    size = torch.zeros((2, h, w), device=device)
    orim = torch.zeros((2, h, w), device=device)
    locs, oris, bbox = (torch.as_tensor(np.asarray(t), dtype=torch.float32, device=device) for t in (locs, oris, bbox))
    typs = torch.as_tensor(np.asarray(typs), device=device)
    x = torch.arange(w, device=device, dtype=torch.float32)
    y = torch.arange(h, device=device, dtype=torch.float32)
    for i in (0, 1):
        sel = typs == i
        if int(sel.sum()) == 0:
            continue
        loc, ori, box = locs[sel], oris[sel], bbox[sel]
        cx = -loc[:, 0] * pixels_per_meter + (max_y - min_y) * pixels_per_meter / 2
        cy = -loc[:, 1] * pixels_per_meter + h + min_x * pixels_per_meter
        gx = torch.exp(-((x[:, None] - cx[None, :]) / radius) ** 2)                              # (w, K)
        gy = torch.exp(-((y[:, None] - cy[None, :]) / radius) ** 2)                              # (h, K)
        gaussian, who = (gx[None] * gy[:, None]).max(dim=-1)                                     # (h, w): best actor per pixel
        mask = gaussian > heat.max(dim=0)[0]
        size[:, mask] = box.T[:, who[mask]] * pixels_per_meter
        orim[0, mask] = torch.cos(ori[who[mask]])
        orim[1, mask] = torch.sin(ori[who[mask]])
        heat[i] = gaussian
    return heat, size, orim
