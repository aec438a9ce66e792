"""ResNet-18 trunk (layer1..layer4) on the lav_b200 tensor-core conv kernel — used by the brake predictor on the
f16 path (SURVEY §8f rank 2: "brake model on the same conv kernels").

Each BasicBlock (lav/models/resnet.py:41-84) becomes two (three with a downsample branch) tap-list convolutions whose
epilogue carries the eval-mode BatchNorm as scale/shift, the residual add and the ReLU — no separate BN / add / ReLU
passes over the activations.  The 7x7/2 stem on 3 input channels and the 3x3/2 max-pool stay on cuDNN (BN folded,
`ResNet18._forward_folded`); the parameters are read from the untouched reference-layout module.
"""
import torch

from . import ops
from .layers import TapConv, bn_affine


class _WideTapConv:
    """TapConv for cout > 256: the wgmma kernel holds at most 256 accumulator columns, so wider layers are issued as
    column chunks that write adjacent channel slices."""

    def __init__(self, weight, stride, padding, scale, shift, post_relu, chunk=256):
        self.cout = weight.shape[0]
        self.parts = []
        for c0 in range(0, self.cout, chunk):
            c1 = min(self.cout, c0 + chunk)
            self.parts.append((c0, TapConv(weight[c0:c1], False, stride, padding, 1, 0, None, scale=scale[c0:c1].clone(),
                                           shift=shift[c0:c1].clone(), post_relu=post_relu)))
        self.out_size = self.parts[0][1].out_size

    def __call__(self, x, res=None):
        n, h, w, _ = x.shape
        ho, wo = self.out_size(h, w)
        out = torch.empty((n, ho, wo, self.cout), dtype=x.dtype, device=x.device)
        for c0, part in self.parts:
            part(x, out=out, out_coff=c0, res=res, res_coff=c0)
        return out


class ResNetTrunkUMMA:
    def __init__(self, resnet):
        self.blocks = []
        for li in range(1, 5):
            for blk in getattr(resnet, f"layer{li}"):
                s1, t1 = bn_affine(blk.bn1)
                s2, t2 = bn_affine(blk.bn2)
                c1 = _WideTapConv(blk.conv1.weight, blk.conv1.stride, 1, s1, t1, post_relu=True)
                c2 = _WideTapConv(blk.conv2.weight, 1, 1, s2, t2, post_relu=True)          # relu(bn2(conv2) + identity)
                ds = None
                if blk.downsample is not None:
                    sd, td = bn_affine(blk.downsample[1])
                    ds = _WideTapConv(blk.downsample[0].weight, blk.downsample[0].stride, 0, sd, td, post_relu=False)
                self.blocks.append((c1, c2, ds))

    def __call__(self, x):
        """x: NHWC f16 (N,H,W,64) = stem + max-pool output -> NHWC f16 (N,H/8,W/8,512)."""
        for c1, c2, ds in self.blocks:
            idt = x if ds is None else ds(x)
            x = c2(c1(x), res=idt)
        return x
