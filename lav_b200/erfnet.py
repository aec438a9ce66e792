"""ERFNet — drop-in mirror of lav/models/erfnet.py (same class names, constructors, state_dict keys).

The module tree only holds parameters; ``ERFNet.forward_nhwc`` runs the whole network as a
sequence of tap-list convolutions with fused epilogues (bias / folded eval BatchNorm / residual /
ReLU) in hand-written CUDA.  Eval mode only (the seg model is frozen on the LAV frame path,
lav_agent.py:116-124); no CPU path.
"""
import torch
from torch import nn

from . import ops
from .capi import LavbError
from .layers import PlanMixin, TapConv, bn_affine

def _dt(precision):
    return torch.float32 if precision == "fp32" else ops.h16()


class DownsamplerBlock(nn.Module):
    def __init__(self, ninput, noutput):
        super().__init__()
        self.conv = nn.Conv2d(ninput, noutput - ninput, (3, 3), stride=2, padding=1, bias=True)
        self.pool = nn.MaxPool2d(2, stride=2)
        self.bn = nn.BatchNorm2d(noutput, eps=1e-3)


class non_bottleneck_1d(nn.Module):
    def __init__(self, chann, dropprob, dilated):
        super().__init__()
        self.conv3x1_1 = nn.Conv2d(chann, chann, (3, 1), stride=1, padding=(1, 0), bias=True)
        self.conv1x3_1 = nn.Conv2d(chann, chann, (1, 3), stride=1, padding=(0, 1), bias=True)
        self.bn1 = nn.BatchNorm2d(chann, eps=1e-03)
        self.conv3x1_2 = nn.Conv2d(chann, chann, (3, 1), stride=1, padding=(1 * dilated, 0), bias=True, dilation=(dilated, 1))
        self.conv1x3_2 = nn.Conv2d(chann, chann, (1, 3), stride=1, padding=(0, 1 * dilated), bias=True, dilation=(1, dilated))
        self.bn2 = nn.BatchNorm2d(chann, eps=1e-03)
        self.dropout = nn.Dropout2d(dropprob)


class Encoder(nn.Module):
    def __init__(self, num_classes):
        super().__init__()
        self.initial_block = DownsamplerBlock(3, 16)
        self.layers = nn.ModuleList()
        self.layers.append(DownsamplerBlock(16, 64))
        for x in range(0, 5):
            self.layers.append(non_bottleneck_1d(64, 0.03, 1))
        self.layers.append(DownsamplerBlock(64, 128))
        for x in range(0, 2):
            self.layers.append(non_bottleneck_1d(128, 0.3, 2))
            self.layers.append(non_bottleneck_1d(128, 0.3, 4))
            self.layers.append(non_bottleneck_1d(128, 0.3, 8))
            self.layers.append(non_bottleneck_1d(128, 0.3, 16))
        # present in the checkpoint, unused by the decoder path (erfnet.py:85, predict=False)
        self.output_conv = nn.Conv2d(128, num_classes, 1, stride=1, padding=0, bias=True)


class UpsamplerBlock(nn.Module):
    def __init__(self, ninput, noutput):
        super().__init__()
        self.conv = nn.ConvTranspose2d(ninput, noutput, 3, stride=2, padding=1, output_padding=1, bias=True)
        self.bn = nn.BatchNorm2d(noutput, eps=1e-3)


class Decoder(nn.Module):
    def __init__(self, num_classes):
        super().__init__()
        self.layers = nn.ModuleList()
        self.layers.append(UpsamplerBlock(128, 64))
        self.layers.append(non_bottleneck_1d(64, 0, 1))
        self.layers.append(non_bottleneck_1d(64, 0, 1))
        self.layers.append(UpsamplerBlock(64, 16))
        self.layers.append(non_bottleneck_1d(16, 0, 1))
        self.layers.append(non_bottleneck_1d(16, 0, 1))
        self.output_conv = nn.ConvTranspose2d(16, num_classes, 2, stride=2, padding=0, output_padding=0, bias=True)


class _Down:
    def __init__(self, m):
        s, t = bn_affine(m.bn)
        nconv = m.conv.out_channels
        cin = m.conv.in_channels
        self.cin, self.nconv, self.nout = cin, nconv, m.bn.num_features
        self.conv = TapConv(m.conv.weight, False, 2, 1, bias=m.conv.bias, scale=s[:nconv].clone(), shift=t[:nconv].clone(),
                            post_relu=True, cin_pad=(cin + 3) // 4 * 4)
        self.ps, self.pt = s[nconv:].contiguous(), t[nconv:].contiguous()
        self.down16 = None
        if cin == 16 and nconv == 48 and tuple(m.conv.kernel_size) == (3, 3):
            w9 = m.conv.weight.detach().float().permute(2, 3, 1, 0).reshape(9, 16, 48).contiguous()          # [ky*3+kx][cin][cout]
            tt = t.detach().clone()
            tt[:48] += m.conv.bias.detach().float() * s.detach()[:48]
            self.down16 = (w9, torch.stack([s.detach(), tt], 1).contiguous())

    def __call__(self, x, dt):
        if FUSE_DOWN16 and self.down16 is not None and x.dtype == ops.h16() and dt == x.dtype and x.shape[2] <= 128 and x.shape[1] % 2 == 0 and x.shape[2] % 2 == 0:
            return ops.erf_down16(x, *self.down16)
        n, h, w, _ = x.shape
        out = torch.empty((n, h // 2, w // 2, self.nout), dtype=dt, device=x.device)
        self.conv(x, out=out)
        if x.dtype != dt:   # pool kernel is single-dtype; only the fp32 RGB ingest of a f16 net hits this
            x = ops.convert(x, dt)
        ops.pool2_affine_relu(x, self.cin, 0, self.ps, self.pt, out, self.nconv)
        return out


FUSE_PAIRS = True     # fused (3x1 -> 1x3) wgmma kernel (csrc/conv_pair_umma.cu)


FUSE_STEM = True      # normalize + initial DownsamplerBlock(3,16) as one kernel on the uint8 frames (csrc/erf16.cu: erf_stem_kernel)
FUSE_DOWN16 = True    # DownsamplerBlock(16, 64) as one kernel (csrc/erf16.cu: erf_down16_kernel) instead of conv_c16_mma<9> + pool2
FUSE_NB16 = True      # the 16-channel decoder blocks as ONE kernel each (csrc/erf16.cu) instead of four conv_c16_mma launches


class _NB1D:
    def __init__(self, m):
        d = m.conv3x1_2.dilation[0]
        s1, t1 = bn_affine(m.bn1)
        s2, t2 = bn_affine(m.bn2)
        self.nb16 = self.pair = None
        if m.conv3x1_1.in_channels == 16 and d == 1:
            # [conv][tap][cin][cout] and (scale, shift) with the bias folded: relu(a*s + t)
            ws = [m.conv3x1_1.weight[:, :, :, 0], m.conv1x3_1.weight[:, :, 0, :], m.conv3x1_2.weight[:, :, :, 0], m.conv1x3_2.weight[:, :, 0, :]]
            w4 = torch.stack([w.detach().float().permute(2, 1, 0) for w in ws]).contiguous()
            one, zero = torch.ones_like(s1), torch.zeros_like(t1)
            bs = [m.conv3x1_1.bias, m.conv1x3_1.bias, m.conv3x1_2.bias, m.conv1x3_2.bias]
            st = torch.stack([torch.stack([s, b.detach().float() * s + t], 1)
                              for s, t, b in zip((one, s1, one, s2), (zero, t1, zero, t2), bs)]).contiguous()
            self.nb16 = (w4, st)
        self.a = TapConv(m.conv3x1_1.weight, False, 1, (1, 0), bias=m.conv3x1_1.bias, post_relu=True)
        self.b = TapConv(m.conv1x3_1.weight, False, 1, (0, 1), bias=m.conv1x3_1.bias, scale=s1, shift=t1, post_relu=True)
        self.c = TapConv(m.conv3x1_2.weight, False, 1, (d, 0), (d, 1), bias=m.conv3x1_2.bias, post_relu=True)
        self.d = TapConv(m.conv1x3_2.weight, False, 1, (0, d), (1, d), bias=m.conv1x3_2.bias, scale=s2, shift=t2, post_relu=True)

    def __call__(self, x, dt):
        if FUSE_NB16 and self.nb16 is not None and x.dtype == ops.h16() and x.shape[2] % 16 == 0 and x.shape[2] <= 256:
            return ops.erf_nb16(x, *self.nb16)
        if FUSE_PAIRS and x.dtype == ops.h16() and self.a.umma_ok and x.shape[3] in (64, 128) and x.shape[2] in (32, 64, 128):
            # each (3x1 -> 1x3) pair in one wgmma kernel, the intermediate stays in shared memory
            if self.pair is None:
                def folded(t):       # (conv + b) * s + t' = conv_{w*s} + (b*s + t'): scale into the weights (fp32, rounded once)
                    w = t.phases[0]["w"][:, :, :t.cout] * t.scale[None, None, :]
                    return w.permute(0, 2, 1).to(ops.h16()).contiguous(), ((t.bias if t.bias is not None else 0) * t.scale + t.shift).contiguous()
                self.pair = (self.a.phases[0]["w_umma"], self.a.bias, *folded(self.b), self.c.phases[0]["w_umma"], self.c.bias, *folded(self.d))
            a, ab, b, bt, c, cb, d, dt_ = self.pair
            y = ops.conv_pair_umma(x, a, ab, b, bt, 1)
            return ops.conv_pair_umma(y, c, cb, d, dt_, self.c.dilation[0], res=x)
        y = self.a(x)
        y = self.b(y)
        y = self.c(y)
        return self.d(y, res=x)   # relu(bn2(conv) + x), erfnet.py:61


class _Up:
    def __init__(self, m):
        s, t = bn_affine(m.bn)
        self.conv = TapConv(m.conv.weight, True, 2, 1, 1, 1, bias=m.conv.bias, scale=s, shift=t, post_relu=True)

    def __call__(self, x, dt):
        return self.conv(x)


class ERFNet(PlanMixin, nn.Module):
    def __init__(self, num_classes):
        super().__init__()
        self.encoder = Encoder(num_classes)
        self.decoder = Decoder(num_classes)
        self.precision = "fp32"

    def _build(self, device):
        def wrap(m):
            if isinstance(m, DownsamplerBlock):
                return _Down(m)
            if isinstance(m, non_bottleneck_1d):
                return _NB1D(m)
            return _Up(m)
        seq = [wrap(self.encoder.initial_block)] + [wrap(m) for m in self.encoder.layers] + [wrap(m) for m in self.decoder.layers]
        oc = self.decoder.output_conv
        table = ops.pack_deconv2x2(oc.weight, oc.bias) if tuple(oc.weight.shape[2:]) == (2, 2) and oc.weight.shape[0] == 16 else None
        stem = None
        ib = self.encoder.initial_block
        if ib.conv.in_channels == 3 and ib.bn.num_features == 16:
            # host-side constants of erf_stem_kernel: w[(ky*3+kx)*3+c][co], epi relu(acc*s + t) (conv bias folded), pool channels last
            s, t = (v.detach() for v in bn_affine(ib.bn))
            w27 = torch.zeros((27, 16))
            w27[:, :13] = ib.conv.weight.detach().float().cpu().permute(2, 3, 1, 0).reshape(27, 13)
            t = t.cpu().clone()
            t[:13] += ib.conv.bias.detach().float().cpu() * s.cpu()[:13]
            stem = (w27.numpy(), s.cpu().numpy(), t.numpy())
        return seq, TapConv(oc.weight, True, 2, 0, 1, 0, bias=oc.bias), table, stem

    def forward_features_nhwc(self, x):
        """x: (N,H,W,4) normalised RGB, or the raw uint8 frames (N,H,W,3) -> (features NHWC (N,H/2,W/2,16) = the input of
        Decoder.output_conv, deconv table).
        The frame pipeline evaluates output_conv inside the point-painting gather (ops.paint_deconv_batched), for the hit
        pixels only; forward_nhwc materialises the full logit maps for everyone else."""
        if self.training:
            raise LavbError("lav_b200.ERFNet is inference-only (the seg model is frozen on the frame path)")
        seq, _, table, stem = self._plan_get(x.device, self._build)
        dt = _dt(self.precision)
        if x.dtype == torch.uint8:            # raw camera frames (N,H,W,3): fused normalize + initial block
            if not (FUSE_STEM and stem is not None):
                raise LavbError("uint8 input needs the fused stem (v2 ERFNet: DownsamplerBlock(3, 16))")
            x = ops.erf_stem(x, *stem, dt)
            seq = seq[1:]
        for blk in seq:
            x = blk(x, dt)
        return x, table

    def forward_nhwc(self, x):
        """x: (N,H,W,4) normalised RGB (4th channel ignored) -> logits NHWC (N,H,W,num_classes) fp32."""
        if self.training:
            raise LavbError("lav_b200.ERFNet is inference-only (the seg model is frozen on the frame path)")
        out_conv = self._plan_get(x.device, self._build)[1]
        x, _ = self.forward_features_nhwc(x)
        return out_conv(x, out_dtype=torch.float32)

    def forward(self, input):
        """input: normalised NCHW float (as erfnet.py:144-146)."""
        if not input.is_cuda:
            raise LavbError("lav_b200.ERFNet needs CUDA tensors (no CPU fallback)")
        n, c, h, w = input.shape
        x = torch.zeros((n, h, w, 4), dtype=torch.float32, device=input.device)
        x[..., :3] = input.permute(0, 2, 3, 1)
        return self.forward_nhwc(x).permute(0, 3, 1, 2)
