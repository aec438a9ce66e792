"""Host-side packing of reference layers into tap-list convolutions (lavb_conv_taps).

A ``TapConv`` is built once from an ``nn.Conv2d`` / ``nn.ConvTranspose2d`` weight (reference
layout, untouched in the state_dict) plus the epilogue that follows it in the reference graph.
ConvTranspose2d is decomposed into stride*stride output phases, each an ordinary tap list, so
no multiply-by-zero work is issued.
"""
import torch

from . import ops

USE_UMMA = True   # tests flip this to compare the wgmma path with the CUDA-core path
UMMA_STRIDED = True   # stride-2 convs through the tensor map's element strides


def bn_affine(bn, eps=None):
    """eval-mode BatchNorm as y*scale+shift (fp64 math, fp32 result)."""
    eps = bn.eps if eps is None else eps
    var = bn.running_var.double()
    scale = bn.weight.double() / torch.sqrt(var + eps)
    shift = bn.bias.double() - bn.running_mean.double() * scale
    return scale.float().contiguous(), shift.float().contiguous()


def _pad_cout(w_tco):
    """(ntaps, cin, cout) -> (ntaps, cin, cout_pad16) contiguous fp32"""
    t, ci, co = w_tco.shape
    cp = (co + 15) // 16 * 16
    out = torch.zeros((t, ci, cp), dtype=torch.float32, device=w_tco.device)
    out[:, :, :co] = w_tco
    return out.contiguous()


def cmajor_wins(hout, wout):
    """whether a 3x3 / pad-1 layer runs faster on lavb_conv3x3_umma (output channels in M) than on lavb_conv_umma.
    `scripts/conv_umma_ab.py`, B = 32, H100 SXM at 700 W, median of 5 rounds (conv_umma -> conv3x3_umma):
      64->64 s1 160^2   0.218 -> 0.137 ms     64->64 s2 320->160   0.242 -> 0.197 ms     heads 384->256 160^2  2.58 -> 2.12 ms
      64->128 s2 160->80  0.107 -> 0.085 ms   128->128 s1 80^2     0.146 -> 0.121 ms
      128->128 s2 80->40  0.053 -> 0.061 ms   128->128 s1 40^2     0.049 -> 0.053 ms
    At 40 x 40 the 16 x 16 tiles cover 48 x 48 and a B = 32 layer has 288 of them for 132 SMs (3 rounds, the last a fifth
    full), against 8 x 16 tiles at two CTAs per SM; so maps of 80 x 80 and more go to the channel-major kernel."""
    return hout >= 80 and wout >= 80


class TapConv:
    def __init__(self, weight, transposed=False, stride=1, padding=0, dilation=1, output_padding=0, bias=None,
                 pre_relu=False, scale=None, shift=None, post_relu=False, sigmoid=False, cin_pad=None):
        pair = lambda v: (v, v) if isinstance(v, int) else tuple(v)
        self.stride, self.padding, self.dilation, self.opad = pair(stride), pair(padding), pair(dilation), pair(output_padding)
        self.transposed = transposed
        w = weight.detach().float()
        if transposed:
            self.cin, self.cout, self.kh, self.kw = w.shape
        else:
            self.cout, self.cin, self.kh, self.kw = w.shape
        self.cin_k = cin_pad or self.cin      # channels the kernel reads (zero weights for the padding)
        self.bias = bias.detach().float().contiguous() if bias is not None else None
        self.scale = scale.contiguous() if scale is not None else None
        self.shift = shift.contiguous() if shift is not None else None
        self.pre_relu, self.post_relu, self.sigmoid = pre_relu, post_relu, sigmoid
        sy, sx = self.stride
        py_, px_ = self.padding
        dy_, dx_ = self.dilation
        self.phases = []
        if not transposed:
            taps, blocks = [], []
            for ky in range(self.kh):
                for kx in range(self.kw):
                    taps.append((ky * dy_ - py_, kx * dx_ - px_))
                    blocks.append(self._block(w[:, :, ky, kx].t()))          # (cin, cout)
            self.phases.append(dict(taps=taps, w=_pad_cout(torch.stack(blocks)), in_s=(sy, sx), out_s=(1, 1), out_o=(0, 0)))
        else:
            for oy in range(sy):
                for ox in range(sx):
                    taps, blocks = [], []
                    for ky in range(self.kh):
                        if (oy + py_ - ky * dy_) % sy:
                            continue
                        for kx in range(self.kw):
                            if (ox + px_ - kx * dx_) % sx:
                                continue
                            taps.append(((oy + py_ - ky * dy_) // sy, (ox + px_ - kx * dx_) // sx))
                            blocks.append(self._block(w[:, :, ky, kx]))       # (cin, cout)
                    if not taps:   # phase that no kernel tap reaches: epilogue of 0
                        taps, blocks = [(0, 0)], [torch.zeros((self.cin_k, self.cout), device=w.device)]
                    self.phases.append(dict(taps=taps, w=_pad_cout(torch.stack(blocks)), in_s=(1, 1), out_s=(sy, sx),
                                            out_o=(oy, ox)))
        for ph in self.phases:
            assert len(ph["taps"]) <= 16, "tap list longer than the kernel's table"
        # wgmma path (f16 activations): weights [ntaps][cout][cin] f16, K contiguous
        # (cout that is a multiple of 8 but not of 32 is zero-padded to the MMA width; only the real channels are stored)
        self.umma_ok = USE_UMMA and self.cin_k % 64 == 0 and self.cout % 8 == 0 and self.cout <= 256
        # the 3x3 / pad-1 convolutions lavb_conv3x3_umma takes (output channels in M, 16 x 16 pixel tiles)
        self.cmajor_ok = (self.umma_ok and not transposed and (self.kh, self.kw) == (3, 3) and self.padding == (1, 1)
                          and self.dilation == (1, 1) and self.stride in ((1, 1), (2, 2)) and self.cin_k in (64, 128, 384)
                          and self.cout in (64, 128, 256) and not post_relu and not sigmoid)
        if self.umma_ok:
            cm = (self.cout + 31) // 32 * 32
            for ph in self.phases:
                wu = torch.zeros((len(ph["taps"]), cm, self.cin_k), dtype=ops.h16(), device=ph["w"].device)
                wu[:, :self.cout] = ph["w"][:, :, :self.cout].permute(0, 2, 1).to(ops.h16())
                ph["w_umma"] = wu.contiguous()

    def _block(self, w_ci_co):
        if self.cin_k == self.cin:
            return w_ci_co
        out = torch.zeros((self.cin_k, self.cout), dtype=w_ci_co.dtype, device=w_ci_co.device)
        out[:self.cin] = w_ci_co
        return out

    def out_size(self, hin, win):
        (sy, sx), (py_, px_), (dy_, dx_), (oy, ox) = self.stride, self.padding, self.dilation, self.opad
        if self.transposed:
            return ((hin - 1) * sy - 2 * py_ + dy_ * (self.kh - 1) + oy + 1, (win - 1) * sx - 2 * px_ + dx_ * (self.kw - 1) + ox + 1)
        return ((hin + 2 * py_ - dy_ * (self.kh - 1) - 1) // sy + 1, (win + 2 * px_ - dx_ * (self.kw - 1) - 1) // sx + 1)

    def __call__(self, x, out=None, in_coff=0, out_coff=0, out_channels=None, res=None, res_coff=0, out_dtype=None):
        """x: NHWC buffer whose channels [in_coff, in_coff+cin_k) feed the conv.  Writes channels
        [out_coff, out_coff+cout) of ``out`` (allocated with ``out_channels`` total channels if None)."""
        n, hin, win, _ = x.shape
        hout, wout = self.out_size(hin, win)
        if out is None:
            out = torch.empty((n, hout, wout, out_channels or self.cout), dtype=out_dtype or x.dtype, device=x.device)
        if (self.cmajor_ok and cmajor_wins(hout, wout) and x.dtype == ops.h16()
                and out.dtype == ops.h16() and x.shape[3] == self.cin_k and in_coff == 0 and out.shape[3] == self.cout
                and out_coff == 0 and res is None):
            ph = self.phases[0]
            return ops.conv3x3_umma(x, ph["w_umma"], self.cout, self.stride[0], self.bias, self.scale, self.shift, self.pre_relu,
                                    out=out)
        for ph in self.phases:
            osy, osx = ph["out_s"]
            ooy, oox = ph["out_o"]
            hog, wog = (hout - ooy + osy - 1) // osy, (wout - oox + osx - 1) // osx
            umma = (self.umma_ok and x.dtype == ops.h16() and (res is None or (res.dtype == ops.h16() and self.cout % 32 == 0))
                    and (UMMA_STRIDED or ph["in_s"] == (1, 1)))
            ops.conv_taps(x, self.cin_k, in_coff, out, self.cout, out_coff, hog, wog, ph["in_s"], ph["out_s"], ph["out_o"],
                          ph["taps"], ph["w_umma"] if umma else ph["w"], self.bias, self.scale, self.shift, res, res_coff,
                          self.pre_relu, self.post_relu, self.sigmoid, umma=umma)
        return out


class PlanMixin:
    """Cache of packed kernels per device; dropped whenever parameters may have changed."""

    def _plan_get(self, device, builder):
        plans = self.__dict__.setdefault("_lavb_plans", {})
        key = (str(device), getattr(self, "precision", "fp32"))
        if key not in plans:
            with torch.no_grad():
                plans[key] = builder(device)
        return plans[key]

    def invalidate_plan(self):
        for m in self.modules():
            if isinstance(m, PlanMixin):
                m.__dict__["_lavb_plans"] = {}

    def _apply(self, fn, *a, **k):
        self.__dict__["_lavb_plans"] = {}
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, *a, **k):
        self.invalidate_plan()
        return super().load_state_dict(*a, **k)

    def train(self, mode=True):
        self.__dict__["_lavb_plans"] = {}
        return super().train(mode)
