"""GPU: lavb_conv3x3_umma (3x3 / pad 1 / stride 1 or 2, output channels in M) against its C-ABI contract, and against
lavb_conv_umma on the BEV layers LiDARModel routes to it.

Contract cases compare with fp64 F.conv2d on h16-rounded operands, 1e-3 of the output scale (h16 output).  Output buffers are
filled with a canary bit pattern (a NaN) and carry a spare image past the end: every output element must be written, and the
spare image must still hold the canary bit for bit.
"""
import pytest
import torch
import torch.nn.functional as F

from lav_b200 import capi, ops, synth
from lav_b200.layers import TapConv, cmajor_wins

pytestmark = pytest.mark.gpu

CANARY = {torch.float16: 0x7E5A, torch.bfloat16: 0x7FDA}


def canary(shape, device):
    t = torch.empty(shape, dtype=ops.h16(), device=device)
    t.view(torch.int16).fill_(CANARY[ops.h16()])
    return t


def is_canary(t):
    return t.contiguous().view(torch.int16) == CANARY[t.dtype]


def q(x):
    return x.to(ops.h16()).double()


def rel(got, want):
    return float((got.double() - want.double()).abs().max() / want.double().abs().max())


def pack(wt):
    """(cout, cin, 3, 3) -> (9, cout, cin) h16 [tap = ky*3 + kx][cout][cin]"""
    return wt.permute(2, 3, 0, 1).reshape(9, wt.shape[0], wt.shape[1]).to(ops.h16()).contiguous()


def run_case(cuda, seed, n, h, w, cin, cout, stride, bias=True, affine=True, pre_relu=True):
    g = synth._gen(37, seed)
    x = q(torch.randn(n, h, w, cin, generator=g)).to(cuda)
    wt = q(torch.randn(cout, cin, 3, 3, generator=g) / (9 * cin) ** 0.5).to(cuda)
    b = torch.randn(cout, generator=g).to(cuda) if bias else None
    sc = (torch.rand(cout, generator=g) + 0.5).to(cuda) if affine else None
    sh = torch.randn(cout, generator=g).to(cuda) if affine else None
    a = F.conv2d(x.permute(0, 3, 1, 2), wt, None, stride, 1).permute(0, 2, 3, 1)
    if b is not None:
        a = a + b.double()
    if pre_relu:
        a = F.relu(a)
    if sc is not None:
        a = a * sc.double() + sh.double()
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    full = canary((n + 1, ho, wo, cout), cuda)
    out = ops.conv3x3_umma(x.to(ops.h16()), pack(wt), cout, stride, b, sc, sh, pre_relu, out=full[:n])
    torch.cuda.synchronize()
    assert not bool(is_canary(out).any()), f"{int(is_canary(out).sum())} outputs never written"
    assert bool(is_canary(full[n:]).all()), "written past the end of the output"
    assert rel(out, a) < 1e-3, rel(out, a)


@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("cin", [64, 128, 384])
@pytest.mark.parametrize("cout", [64, 128, 256])
def test_conv3x3_umma_contract(cuda, stride, cin, cout):
    """every (stride, cin, cout) the header allows, on a map whose sides are not multiples of the 16-pixel tile (odd at
    stride 2), with bias, pre-ReLU and the BatchNorm affine"""
    h, w = (37, 45) if stride == 2 else (20, 35)
    run_case(cuda, f"c{stride}_{cin}_{cout}", 2, h, w, cin, cout, stride)


EPILOGUES = {
    "fold_bias": dict(pre_relu=False),                  # (a + b) s + t folded into a s + (b s + t)
    "bias_only": dict(affine=False, pre_relu=False),
    "affine_only": dict(bias=False),
    "relu_only": dict(bias=False, affine=False),
    "plain": dict(bias=False, affine=False, pre_relu=False),
}


@pytest.mark.parametrize("name", list(EPILOGUES))
def test_conv3x3_umma_epilogue(cuda, name):
    run_case(cuda, "e" + name, 2, 18, 21, 64, 128, 1, **EPILOGUES[name])


@pytest.mark.parametrize("n,h,w,cin,cout,stride", [
    (2, 40, 40, 128, 128, 1),     # the backbone's conv3 size: 16 x 16 tiles cover 48 x 48
    (1, 40, 40, 128, 128, 1),     # n = 1
    (1, 1, 1, 64, 64, 1),         # one pixel: every tap but the centre is padding
    (1, 3, 2, 64, 256, 2),        # stride 2 below one tile
    (1, 81, 17, 64, 64, 2),       # odd, a tall map at stride 2
    (12, 64, 64, 64, 64, 1),      # 192 tiles: more than one per CTA of the persistent loop
    (6, 64, 48, 384, 256, 1),     # 144 tiles x 2 CTA columns, 6 K chunks
])
def test_conv3x3_umma_shapes(cuda, n, h, w, cin, cout, stride):
    run_case(cuda, f"s{n}_{h}_{w}_{cin}_{cout}_{stride}", n, h, w, cin, cout, stride)


def test_conv3x3_umma_rejects(cuda):
    x = torch.zeros(1, 8, 8, 96, dtype=ops.h16(), device=cuda)
    wt = torch.zeros(9, 64, 96, dtype=ops.h16(), device=cuda)
    with pytest.raises(capi.LavbError):
        ops.conv3x3_umma(x, wt, 64, 1)
    x = torch.zeros(1, 8, 8, 64, dtype=ops.h16(), device=cuda)
    with pytest.raises(capi.LavbError):
        ops.conv3x3_umma(x, torch.zeros(9, 96, 64, dtype=ops.h16(), device=cuda), 96, 1)
    with pytest.raises(capi.LavbError):
        ops.conv3x3_umma(x, torch.zeros(9, 64, 64, dtype=ops.h16(), device=cuda), 64, 3)


def bev_layer(cuda, seed, cin, cout, stride):
    g = synth._gen(38, seed)
    wt = torch.randn(cout, cin, 3, 3, generator=g) * (2.0 / (9 * cin)) ** 0.5
    s, t = torch.rand(cout, generator=g) + 0.5, torch.randn(cout, generator=g) * 0.1
    return TapConv(wt.to(cuda), False, stride, 1, pre_relu=True, scale=s.to(cuda), shift=t.to(cuda)), g


def conv_umma(layer, x):
    n, h, w, cin = x.shape
    ho, wo = layer.out_size(h, w)
    ph = layer.phases[0]
    y = torch.empty(n, ho, wo, layer.cout, dtype=ops.h16(), device=x.device)
    return ops.conv_taps(x, cin, 0, y, layer.cout, 0, ho, wo, ph["in_s"], (1, 1), (0, 0), ph["taps"], ph["w_umma"], layer.bias,
                         layer.scale, layer.shift, pre_relu=True, umma=True)


# the ConvBackbone layers LiDARModel sends to lavb_conv3x3_umma, at B = 32: (cin, cout, stride, input side)
ROUTED = [(64, 64, 2, 320), (64, 64, 1, 160), (64, 128, 2, 160), (128, 128, 1, 80)]


@pytest.mark.parametrize("cin,cout,stride,side", ROUTED)
def test_conv3x3_umma_bitwise_backbone(cuda, cin, cout, stride, side):
    """with cin <= 128 the kernel walks K tap-major, chunk-minor as conv_umma_kernel does and applies the same fp32 epilogue,
    so TapConv's routing changes no output bit"""
    layer, g = bev_layer(cuda, f"bb{cin}{cout}{stride}", cin, cout, stride)
    ho = (side - 1) // stride + 1
    assert cmajor_wins(ho, ho)
    x = torch.randn(32, side, side, cin, generator=g).to(cuda).to(ops.h16())
    got = layer(x)
    assert got.dtype == ops.h16() and got.shape == (32, ho, ho, cout)
    assert torch.equal(got, conv_umma(layer, x))


def test_conv3x3_umma_heads_conv(cuda):
    """the fused 384 -> 256 heads conv at 160 x 160, B = 32: K walked chunk-major (a tile's input window stays in L2), so the
    sums are reordered against conv_umma_kernel and agree to h16 rounding"""
    layer, g = bev_layer(cuda, "heads", 384, 256, 1)
    assert cmajor_wins(160, 160)
    x = torch.randn(32, 160, 160, 384, generator=g).to(cuda).to(ops.h16())
    got, want = layer(x), conv_umma(layer, x)
    assert rel(got, want) < 1e-3, rel(got, want)
