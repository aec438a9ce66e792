"""PointPillarNet / DynamicPointNet — drop-in mirrors of lav/models/point_pillar.py.

Same constructor arguments, ``forward(lidar_list, num_points)`` signature and ``state_dict``
keys (``point_net.net.{0,1,3,4}.*``).  The forward is the hand-written CUDA voxeliser + pillar
encoder (csrc/pillar.cu) — no torch_scatter, no ``unique``; there is no CPU path.

Returned canvas: logical shape (B, C, ny, nx) like the reference, stored channels-last.
"""
import torch
from torch import nn

from . import ops
from .capi import LavbError
from .layers import PlanMixin


class DynamicPointNet(nn.Module):
    """Parameter container with the reference layout (point_pillar.py:12-35)."""

    def __init__(self, num_input=9, num_features=[32, 32]):
        super().__init__()
        L = []
        for num_feature in num_features:
            L += [nn.Linear(num_input, num_feature), nn.BatchNorm1d(num_feature), nn.ReLU(inplace=True)]
            num_input = num_feature
        self.net = nn.Sequential(*L)

    def forward(self, points, inverse_indices):
        raise LavbError("DynamicPointNet is fused into PointPillarNet.forward in lav_b200; call the parent module")


class _PillarScatterMax(torch.autograd.Function):
    """scatter_max over canvas cells with arg-routed backward (torch_scatter.scatter_max semantics)."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)     # under autocast the point MLP hands over f16
    def forward(ctx, h, cell, n_cells):
        canvas, arg = ops.pillar_scatter_max(h, cell, n_cells, want_argmax=True)
        ctx.save_for_backward(arg, cell)
        ctx.m = h.shape[0]
        return canvas

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, g):
        arg, cell = ctx.saved_tensors
        return ops.pillar_scatter_max_bwd(g, arg, cell, ctx.m), None, None


class PointPillarNet(PlanMixin, nn.Module):
    def __init__(self, num_input=9, num_features=[32, 32], min_x=-10, max_x=70, min_y=-40, max_y=40, pixels_per_meter=4):
        super().__init__()
        self.point_net = DynamicPointNet(num_input, num_features)
        self.nx = (max_x - min_x) * pixels_per_meter
        self.ny = (max_y - min_y) * pixels_per_meter
        self.min_x, self.min_y, self.max_x, self.max_y = min_x, min_y, max_x, max_y
        self.pixels_per_meter = pixels_per_meter
        self.num_point_dims = num_input - 5
        self.precision = "fp32"      # 'f16' selects the sorted / tensor-core encoder (set by LiDARModel.set_precision)

    def _grid(self):
        return (float(self.min_x), float(self.max_x), float(self.min_y), float(self.max_y), float(self.pixels_per_meter),
                int(self.nx), int(self.ny))

    def _build(self, device):
        net = self.point_net.net
        assert len(net) == 6, "lav_b200 builds the 2-layer point MLP of the v2 config"
        out = []
        for lin, bn in ((net[0], net[1]), (net[3], net[4])):
            s = bn.weight.double() / torch.sqrt(bn.running_var.double() + bn.eps)
            t = (lin.bias.double() - bn.running_mean.double()) * s + bn.bias.double()
            out += [lin.weight.detach().float().contiguous(), s.float().contiguous(), t.float().contiguous()]
        return out

    @staticmethod
    def _as_buffer(lidar_list, num_points):
        """-> (2-D row buffer, starts, counts) without copying when the input is already one tensor."""
        if torch.is_tensor(num_points):
            num_points = num_points.tolist()
        counts = [int(n) for n in num_points]
        if torch.is_tensor(lidar_list):
            assert lidar_list.dim() == 3
            B, P, D = lidar_list.shape
            buf = lidar_list.contiguous().view(B * P, D)
            starts = [b * P for b in range(B)]
            counts = [min(c, P) for c in counts]
        else:
            counts = [min(c, len(t)) for c, t in zip(counts, lidar_list)]
            if len(lidar_list) == 1:
                buf = lidar_list[0].contiguous()
                starts = [0]
            else:
                buf = torch.cat([t[:c] for t, c in zip(lidar_list, counts)], dim=0)
                starts, acc = [], 0
                for c in counts:
                    starts.append(acc)
                    acc += c
        if buf.dtype != torch.float32:
            buf = buf.float()
        return buf, starts, counts

    def forward(self, lidar_list, num_points):
        buf, starts, counts = self._as_buffer(lidar_list, num_points)
        if not buf.is_cuda:
            raise LavbError("lav_b200.PointPillarNet needs CUDA tensors (no CPU fallback)")
        B = len(counts)
        if self.training:
            with torch.no_grad():
                feat, cell = ops.pillar_decorate(buf, starts, counts, self._grid(), self.num_point_dims)
            h = self.point_net.net(feat)
            canvas = _PillarScatterMax.apply(h, cell, B * self.ny * self.nx)
            return canvas.view(B, self.ny, self.nx, -1).permute(0, 3, 1, 2)
        return self.forward_nhwc(lidar_list, num_points, _buf=(buf, starts, counts)).permute(0, 3, 1, 2)

    def forward_nhwc(self, lidar_list, num_points, _buf=None, canvas16=False):
        """eval forward returning the raw NHWC canvas buffer.  fp32 precision: exact kernel (fp32 FFMA + atomicMax).
        f16 precision: sorted / tensor-core kernel; the canvas comes as fp32 (B,ny,nx,C), or with canvas16 as the saturating
        h16 (B,ny,nx,C) that ConvBackbone's first tensor-core conv consumes."""
        buf, starts, counts = _buf if _buf is not None else self._as_buffer(lidar_list, num_points)
        if not buf.is_cuda:
            raise LavbError("lav_b200.PointPillarNet needs CUDA tensors (no CPU fallback)")
        w1, s1, t1, w2, s2, t2 = self._plan_get(buf.device, self._build)
        if self.precision == "f16":
            return ops.pillar_forward_sorted(buf, starts, counts, self._grid(), w1, s1, t1, w2, s2, t2, canvas16=canvas16)
        return ops.pillar_forward(buf, starts, counts, self._grid(), w1, s1, t1, w2, s2, t2)
