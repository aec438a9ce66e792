"""LiDARModel / ConvBackbone / Head — drop-in mirrors of lav/models/lidar.py.

Same constructors, forward signatures and ``state_dict`` keys; every conv / transposed conv
(+ReLU+BatchNorm epilogue) runs in hand-written CUDA (csrc/conv_taps.cu; csrc/conv_umma.cu and, for
the large 3x3 layers, csrc/stem_umma.cu on the f16 path).  Tensors keep the reference's logical NCHW shapes but are stored channels-last.
``precision`` = 'fp32' (exact path, default) or 'f16' (tensor-core path).
"""
import torch
from torch import nn

from . import ops
from .capi import LavbError
from .layers import PlanMixin, TapConv, bn_affine
from .point_pillar import PointPillarNet


def _dt(precision):
    return torch.float32 if precision == "fp32" else ops.h16()


def _nhwc(x):
    """logical NCHW tensor -> contiguous NHWC buffer (free for channels-last inputs)."""
    if not x.is_cuda:
        raise LavbError("lav_b200 modules need CUDA tensors (no CPU fallback)")
    return x.permute(0, 2, 3, 1).contiguous()


class ConvBackbone(PlanMixin, nn.Module):
    def __init__(self, num_feature=64, norm_cfg={'eps': 1e-3, 'momentum': 0.01}):
        super().__init__()
        nf = num_feature

        def stage(cin, cout, n):
            L = []
            for i in range(n):
                L += [nn.Conv2d(cin if i == 0 else cout, cout, 3, 2 if i == 0 else 1, 1, bias=False), nn.ReLU(inplace=True),
                      nn.BatchNorm2d(cout, **norm_cfg)]
            return nn.Sequential(*L)
        self.conv1 = stage(nf, nf, 4)
        self.conv2 = stage(nf, 2 * nf, 6)
        self.conv3 = stage(2 * nf, 2 * nf, 6)
        self.upconv1 = nn.Sequential(nn.ConvTranspose2d(nf, 2 * nf, 1, 1, bias=False), nn.ReLU(inplace=True),
                                     nn.BatchNorm2d(2 * nf, **norm_cfg))
        self.upconv2 = nn.Sequential(nn.ConvTranspose2d(2 * nf, 2 * nf, 4, 2, 1, bias=False), nn.ReLU(inplace=True),
                                     nn.BatchNorm2d(2 * nf, **norm_cfg))
        self.upconv3 = nn.Sequential(nn.ConvTranspose2d(2 * nf, 2 * nf, 4, 4, 1, 2, bias=False), nn.ReLU(inplace=True),
                                     nn.BatchNorm2d(2 * nf, **norm_cfg))
        self.precision = "fp32"

    def _build(self, device):
        def crb(conv, bn):
            s, t = bn_affine(bn)
            return TapConv(conv.weight, isinstance(conv, nn.ConvTranspose2d), conv.stride, conv.padding, conv.dilation,
                           getattr(conv, "output_padding", 0), None, pre_relu=True, scale=s, shift=t)
        plan = {}
        for name in ("conv1", "conv2", "conv3"):
            seq = getattr(self, name)
            plan[name] = [crb(seq[i], seq[i + 2]) for i in range(0, len(seq), 3)]
        for name in ("upconv1", "upconv2", "upconv3"):
            seq = getattr(self, name)
            plan[name] = crb(seq[0], seq[2])
        return plan

    def forward_nhwc(self, x):
        """x: NHWC canvas buffer -> NHWC (B, H/2, W/2, 6*nf) feature buffer."""
        if self.training:
            raise LavbError("ConvBackbone: training-mode forward goes through lav_b200.train (autograd path)")
        plan = self._plan_get(x.device, self._build)
        dt = _dt(self.precision)
        if dt == ops.h16() and x.dtype == torch.float32:
            # an fp32 canvas gets the saturating round-to-nearest the encoder's h16 canvas (out_mode 2) applies
            x = ops.convert(x, dt)
        xs = []
        for name in ("conv1", "conv2", "conv3"):
            for layer in plan[name]:
                x = layer(x, out_dtype=dt)
            xs.append(x)
        n, h, w, _ = xs[0].shape
        ctot = plan["upconv1"].cout + plan["upconv2"].cout + plan["upconv3"].cout
        out = torch.empty((n, h, w, ctot), dtype=dt, device=x.device)
        off = 0
        for name, xi in zip(("upconv1", "upconv2", "upconv3"), xs):
            plan[name](xi, out=out, out_coff=off)
            off += plan[name].cout
        return out

    def forward(self, x):
        if self.training:    # autograd path: the module tree's own layers (cuDNN) — see lav_b200/train.py
            x1 = self.conv1(x)
            x2 = self.conv2(x1)
            x3 = self.conv3(x2)
            return torch.cat([self.upconv1(x1), self.upconv2(x2), self.upconv3(x3)], dim=1)
        return self.forward_nhwc(_nhwc(x)).permute(0, 3, 1, 2)


class Head(PlanMixin, nn.Module):
    def __init__(self, num_input, num_output, num_hidden=64, norm_cfg={'eps': 1e-3, 'momentum': 0.01}, output_activation=None):
        super().__init__()
        self.net = nn.Sequential(
            nn.Conv2d(num_input, num_hidden, 3, 1, 1, bias=False),
            nn.ReLU(inplace=True),
            nn.BatchNorm2d(num_hidden, **norm_cfg),
            nn.ConvTranspose2d(num_hidden, num_output, 3, 2, 1, 1),
        )
        self.output_activation = output_activation
        self.precision = "fp32"

    def _is_sigmoid(self):
        if self.output_activation is None:
            return False
        if self.output_activation is torch.sigmoid or self.output_activation is torch.nn.functional.sigmoid:
            return True
        raise LavbError("Head: only output_activation in (None, torch.sigmoid) is built (lidar.py:29-32)")

    def _build(self, device):
        s, t = bn_affine(self.net[2])
        conv = TapConv(self.net[0].weight, False, 1, 1, pre_relu=True, scale=s, shift=t)
        up = TapConv(self.net[3].weight, True, 2, 1, 1, 1, bias=self.net[3].bias, sigmoid=self._is_sigmoid())
        return conv, up

    def forward_nhwc(self, x):
        if self.training:
            raise LavbError("Head: training-mode forward goes through lav_b200.train (autograd path)")
        conv, up = self._plan_get(x.device, self._build)
        return up(conv(x, out_dtype=_dt(self.precision)), out_dtype=torch.float32)

    def forward(self, x):
        if self.training:
            y = self.net(x)
            return self.output_activation(y) if self.output_activation else y
        return self.forward_nhwc(_nhwc(x)).permute(0, 3, 1, 2)


class LiDARModel(PlanMixin, nn.Module):
    def __init__(self, num_input=9, num_features=[32, 32], backbone='swin', min_x=-10, max_x=70, min_y=-40, max_y=40,
                 pixels_per_meter=4):
        super().__init__()
        self.point_pillar_net = PointPillarNet(num_input, num_features, min_x=min_x, max_x=max_x, min_y=min_y, max_y=max_y,
                                               pixels_per_meter=pixels_per_meter)
        num_feature = num_features[-1]
        if backbone == 'cnn':
            self.backbone = ConvBackbone(num_feature=num_feature)
        else:
            raise NotImplementedError
        self.center_head = Head(6 * num_feature, 2)
        self.box_head = Head(6 * num_feature, 2)
        self.ori_head = Head(6 * num_feature, 2)
        self.seg_head = Head(6 * num_feature, 3, output_activation=torch.sigmoid)
        self.precision = "fp32"

    def set_precision(self, precision):
        assert precision in ("fp32", "f16"), precision
        for m in self.modules():
            if hasattr(m, "precision"):
                m.precision = precision
        self.invalidate_plan()
        return self

    def _heads(self):
        return (self.center_head, self.box_head, self.ori_head, self.seg_head)

    def _build(self, device):
        """one 384->256 conv for the four heads (reads the feature map once), then four small ConvT."""
        ws, ss, ts = [], [], []
        for h in self._heads():
            s, t = bn_affine(h.net[2])
            ws.append(h.net[0].weight)
            ss.append(s)
            ts.append(t)
        conv = TapConv(torch.cat(ws, 0), False, 1, 1, pre_relu=True, scale=torch.cat(ss), shift=torch.cat(ts))
        # the four ConvTranspose2d(64 -> 2/2/2/3, k3 s2 p1 op1) output layers
        nh = self.center_head.net[0].out_channels
        wd = torch.zeros((4, nh, 9, 4), dtype=torch.float32, device=device)
        bd = torch.zeros((4, 4), dtype=torch.float32, device=device)
        n_outs, d2s = [], []
        for g, h in enumerate(self._heads()):
            ct = h.net[3]
            assert ct.kernel_size == (3, 3) and ct.stride == (2, 2) and ct.padding == (1, 1) and ct.output_padding == (1, 1)
            no = ct.out_channels
            wd[g, :, :, :no] = ct.weight.detach().float().permute(0, 2, 3, 1).reshape(nh, 9, no)   # (cin,cout,ky,kx)->(cin,tap,cout)
            bd[g, :no] = ct.bias.detach().float()
            n_outs.append(no)
            # tensor-core form (f16 path): a 2x2-tap GEMM over the input grid with 4*no (<=32) columns and a
            # depth-to-space epilogue.  out(2y+a, 2x+b) gathers input pixel (y+dy, x+dx) through kernel tap (ky,kx):
            #   a=0 -> (dy=0,ky=1);  a=1 -> (dy=0,ky=2) and (dy=1,ky=0)      (same for b / dx / kx)
            w = ct.weight.detach().float()                                      # (cin, cout, ky, kx)
            wu = torch.zeros((4, 32, nh), dtype=torch.float32, device=device)   # [tap=(dy,dx)][col=pos*no+k][cin]
            opts = {0: [(0, 1)], 1: [(0, 2), (1, 0)]}
            for pa in (0, 1):
                for pb in (0, 1):
                    for dy, ky in opts[pa]:
                        for dx, kx in opts[pb]:
                            wu[dy * 2 + dx, (pa * 2 + pb) * no:(pa * 2 + pb) * no + no] = w[:, :, ky, kx].t()
            bias32 = torch.zeros(32, dtype=torch.float32, device=device)
            bias32[:4 * no] = ct.bias.detach().float().repeat(4)
            d2s.append((wu.to(ops.h16()).contiguous(), bias32))
        return conv, (wd.contiguous(), bd.contiguous(), n_outs, [h._is_sigmoid() for h in self._heads()], nh, d2s)

    def heads_nhwc(self, feats):
        conv, (wd, bd, n_outs, sig, nh, d2s) = self._plan_get(feats.device, self._build)
        if self.precision == "f16":
            hid = conv(feats, out_dtype=ops.h16())
            n, h, w, _ = hid.shape
            outs = []
            for g, (wu, b32) in enumerate(d2s):
                out = torch.empty((n, 2 * h, 2 * w, n_outs[g]), dtype=torch.float32, device=hid.device)
                ops.conv_taps(hid, nh, g * nh, out, 32, 0, h, w, (1, 1), (2, 2), (0, 0), [(0, 0), (0, 1), (1, 0), (1, 1)], wu,
                              bias=b32, sigmoid=sig[g], umma=True, d2s_nout=n_outs[g])
                outs.append(out)
            return outs
        hid = conv(feats, out_dtype=torch.float32)
        return ops.deconv3x3s2_small(hid, 4, nh, wd, bd, n_outs, sig)

    def forward_nhwc(self, lidars, num_points):
        # 16-bit path: the canvas is an h16 activation like every other layer's input (64 ch, 128 B per cell).  With half storage
        # its rounding (2^-12) is the same as everywhere else in the stack.
        canvas = self.point_pillar_net.forward_nhwc(lidars, num_points, canvas16=self.precision == "f16")
        feats = self.backbone.forward_nhwc(canvas)
        return (feats, *self.heads_nhwc(feats))

    def forward(self, lidars, num_points):
        if self.training:
            from .train import lidar_model_train_forward
            return lidar_model_train_forward(self, lidars, num_points)
        return tuple(t.permute(0, 3, 1, 2) for t in self.forward_nhwc(lidars, num_points))
