"""GPU: the wgmma kernels against their whole C-ABI contract (include/lav_b200.h), called through ops directly so that every
descriptor field is set here rather than by TapConv.

Each case compares with fp64 F.conv2d / F.conv_transpose2d on h16-rounded operands (2e-5 of the output scale with fp32
output, 1e-3 with h16 output, 1e-2 for the fused pair).  Output buffers are filled beforehand with a canary bit pattern
(a NaN), and every element outside the slice the call is documented to write — other channels, a spare image past the
end — must still hold it bit for bit.
"""
import subprocess
import sys
import textwrap

import pytest
import torch
import torch.nn.functional as F

from lav_b200 import ops, synth
from oracle import lav_ref as O
from tests import util

pytestmark = pytest.mark.gpu

CANARY = {torch.float32: 0x7FC0DEAD, torch.float16: 0x7E5A, torch.bfloat16: 0x7FDA}
INT = {torch.float32: torch.int32, torch.float16: torch.int16, torch.bfloat16: torch.int16}


def canary(shape, dtype, device):
    t = torch.empty(shape, dtype=dtype, device=device)
    t.view(INT[dtype]).fill_(CANARY[dtype])
    return t


def is_canary(t):
    return t.contiguous().view(INT[t.dtype]) == CANARY[t.dtype]


def q(x):
    return x.to(ops.h16()).double()


def rel(got, want):
    return float((got.double() - want.double()).abs().max() / want.double().abs().max())


def nhwc(t):
    return t.permute(0, 2, 3, 1)


def nchw(t):
    return t.permute(0, 3, 1, 2)


# ------------------------------------------------------------------------------------------------------------------ conv_umma
UMMA_CASES = {
    # MMA widths kNC = cout / 32 that the product never launches, with the full epilogue and a residual
    "cout32": dict(cout=32), "cout96": dict(cout=96), "cout160": dict(cout=160), "cout192": dict(cout=192), "cout224": dict(cout=224),
    # stores narrower than the MMA (zero weight rows past cout; a residual needs cout % 32 == 0)
    "cout8": dict(cout=8, res=False), "cout24": dict(cout=24, res=False), "cout40": dict(cout=40, res=False),
    # channel slices: read [64, 128) of a 192-channel buffer; write [32, 96) of 160; residual [64, 128) of 192
    "in_slice": dict(cout=64, in_cs=192, in_off=64),
    "out_slice": dict(cout=64, out_cs=160, out_off=32),
    "res_slice": dict(cout=64, res_cs=192, res_off=64),
    "all_slices": dict(cin=128, cout=96, in_cs=256, in_off=64, out_cs=256, out_off=136, res_cs=104, res_off=8),
    # epilogues
    "fold_bias": dict(cout=64, pre_relu=False),                          # (a + b) s + t folded into a s + (b s + t)
    "bias_only": dict(cout=64, pre_relu=False, affine=False, res=False, post_relu=False),
    "affine_only": dict(cout=64, bias=False),
    "no_post_relu": dict(cout=128, post_relu=False),
    "sigmoid": dict(cout=64, post_relu=False, sigmoid=True),
    "pre_relu_no_bias": dict(cout=64, bias=False, affine=False, res=False),
    # the tap table's maximum: 4 x 4 kernel
    "taps16": dict(cout=64, k=4, pad=1),
    # stride 2 on odd sizes (TMA element strides, ragged last tile)
    "stride2_odd": dict(cout=64, stride=2, hw=(33, 35)),
    "stride2_odd_wide": dict(cin=128, cout=256, stride=2, hw=(17, 49)),
    # several tiles per CTA of the persistent loop (more tiles than 2 x SMs)
    "persistent64": dict(cout=64, n=12, hw=(64, 64)),
    "persistent256": dict(cout=256, n=6, hw=(64, 64)),
}


@pytest.mark.parametrize("name", list(UMMA_CASES))
def test_conv_umma_descriptor(cuda, name):
    cfg = dict(cin=64, n=2, hw=(20, 24), k=3, pad=1, stride=1, bias=True, affine=True, res=True, pre_relu=True, post_relu=True,
               sigmoid=False, in_off=0, out_off=0, res_off=0)
    cfg.update(UMMA_CASES[name])
    cin, cout, n, (h, w), k, pad, s = cfg["cin"], cfg["cout"], cfg["n"], cfg["hw"], cfg["k"], cfg["pad"], cfg["stride"]
    in_cs, out_cs, res_cs = cfg.get("in_cs", cin), cfg.get("out_cs", cout), cfg.get("res_cs", cout)
    g = synth._gen(33, "umma" + name)
    xbuf = q(torch.randn(n, h, w, in_cs, generator=g)).to(cuda)
    x = xbuf[..., cfg["in_off"]:cfg["in_off"] + cin]
    wt = q(torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5).to(cuda)
    b = torch.randn(cout, generator=g).to(cuda) if cfg["bias"] else None
    sc = (torch.rand(cout, generator=g) + 0.5).to(cuda) if cfg["affine"] else None
    sh = torch.randn(cout, generator=g).to(cuda) if cfg["affine"] else None
    a = nhwc(F.conv2d(nchw(x), wt, None, s, pad))
    ho, wo = a.shape[1:3]
    rbuf = q(torch.randn(n, ho, wo, res_cs, generator=g)).to(cuda) if cfg["res"] else None
    if b is not None:
        a = a + b.double()
    if cfg["pre_relu"]:
        a = F.relu(a)
    if sc is not None:
        a = a * sc.double() + sh.double()
    if rbuf is not None:
        a = a + rbuf[..., cfg["res_off"]:cfg["res_off"] + cout]
    if cfg["post_relu"]:
        a = F.relu(a)
    if cfg["sigmoid"]:
        a = torch.sigmoid(a)
    cout_mma = (cout + 31) // 32 * 32
    wu = torch.zeros(k * k, cout_mma, cin, dtype=torch.float64, device=cuda)
    wu[:, :cout] = wt.permute(2, 3, 0, 1).reshape(k * k, cout, cin)
    wu = wu.to(ops.h16()).contiguous()
    taps = [(ky - pad, kx - pad) for ky in range(k) for kx in range(k)]
    xin = xbuf.to(ops.h16()).contiguous()
    rin = None if rbuf is None else rbuf.to(ops.h16()).contiguous()
    for odt, tol in ((torch.float32, 2e-5), (ops.h16(), 1e-3)):
        full = canary((n + 1, ho, wo, out_cs), odt, cuda)        # one spare image past the end
        out = full[:n]
        ops.conv_taps(xin, cin, cfg["in_off"], out, cout, cfg["out_off"], ho, wo, (s, s), (1, 1), (0, 0), taps, wu, bias=b, scale=sc,
                      shift=sh, res=rin, res_coff=cfg["res_off"], pre_relu=cfg["pre_relu"], post_relu=cfg["post_relu"],
                      sigmoid=cfg["sigmoid"], umma=True)
        torch.cuda.synchronize()
        sl = slice(cfg["out_off"], cfg["out_off"] + cout)
        got = out[..., sl]
        assert not bool(is_canary(got).any()), f"{int(is_canary(got).sum())} outputs never written ({odt})"
        assert rel(got, a) < tol, (odt, rel(got, a))
        untouched = torch.ones(full.shape, dtype=torch.bool, device=cuda)
        untouched[:n, ..., sl] = False
        assert bool(is_canary(full)[untouched].all()), f"{int((~is_canary(full))[untouched].sum())} elements written outside the slice ({odt})"


def pack_d2s(wt, no):
    """ConvTranspose2d(cin, no, 3, stride 2, padding 1, output_padding 1) weight (cin, no, 3, 3) -> the 2x2-tap GEMM operand
    [tap = dy*2 + dx][column = pos*no + k][cin] of the depth-to-space epilogue (as LiDARModel packs its detection heads)"""
    cin = wt.shape[0]
    wu = torch.zeros((4, 32, cin), dtype=wt.dtype, device=wt.device)
    opts = {0: [(0, 1)], 1: [(0, 2), (1, 0)]}
    for pa in (0, 1):
        for pb in (0, 1):
            for dy, ky in opts[pa]:
                for dx, kx in opts[pb]:
                    wu[dy * 2 + dx, (pa * 2 + pb) * no:(pa * 2 + pb + 1) * no] = wt[:, :, ky, kx].t()
    return wu


@pytest.mark.parametrize("no,sigmoid", [(2, False), (3, True), (8, False)])
def test_conv_umma_depth_to_space(cuda, no, sigmoid):
    """d2s_nout in {2, 3, 8}: ConvTranspose2d(64 -> no, k3, s2, p1, op1) as a 2x2-tap GEMM with 4 * no columns, reading channels
    [64, 128) of a 128-channel h16 map, against fp64 F.conv_transpose2d; every output element written, nothing past the end."""
    g = synth._gen(34, f"d2s{no}")
    n, h, w, cin = 2, 13, 18, 64
    xbuf = q(torch.randn(n, h, w, 2 * cin, generator=g)).to(cuda)
    wt = q(torch.randn(cin, no, 3, 3, generator=g) / (9 * cin) ** 0.5).to(cuda)
    b = torch.randn(no, generator=g).to(cuda)
    want = nhwc(F.conv_transpose2d(nchw(xbuf[..., cin:]), wt, b.double(), 2, 1, 1))
    if sigmoid:
        want = torch.sigmoid(want)
    b32 = torch.zeros(32, device=cuda)
    b32[:4 * no] = b.repeat(4)
    full = canary((n + 1, 2 * h, 2 * w, no), torch.float32, cuda)
    out = full[:n]
    ops.conv_taps(xbuf.to(ops.h16()).contiguous(), cin, cin, out, 32, 0, h, w, (1, 1), (2, 2), (0, 0), [(0, 0), (0, 1), (1, 0), (1, 1)],
                  pack_d2s(wt, no).to(ops.h16()).contiguous(), bias=b32, sigmoid=sigmoid, umma=True, d2s_nout=no)
    torch.cuda.synchronize()
    assert not bool(is_canary(out).any())
    assert bool(is_canary(full[n:]).all())
    assert rel(out, want) < 2e-5, rel(out, want)


# ------------------------------------------------------------------------------------------------------------- conv_pair_umma
def pair_want(x, w1, b1, w2, t2, dil, res, relu):
    """relu(conv3x1 + b1) stored as h16 -> conv1x3 + shift2 -> h16 [+ res] [relu]; w1 / w2 [cout][cin][tap]"""
    mid = q(F.relu(F.conv2d(nchw(x), w1[:, :, :, None], b1.double(), padding=(dil, 0), dilation=(dil, 1))))
    a = nhwc(F.conv2d(mid, w2[:, :, None, :], t2.double(), padding=(0, dil), dilation=(1, dil)))
    if res is not None:
        a = q(a) + res
    return F.relu(a) if relu else a


PAIR_VARIANTS = ["d1_res_relu", "dmid_norelu", "dmax_res_norelu", "dmax_relu", "ragged", "persistent"]


@pytest.mark.parametrize("variant", PAIR_VARIANTS)
@pytest.mark.parametrize("c,w", [(c, w) for c in (64, 128) for w in (32, 64, 128)])
def test_conv_pair_umma_contract(cuda, c, w, variant):
    """the header's whole grid c in {64, 128} x w in {32, 64, 128}: dilation 1, a middle value and w - 1 (every tap but the
    centre falls off the row), post_relu 0 / 1, with and without the residual, a ragged last tile (h not a multiple of
    128 / w; w = 128 tiles are single rows), and more tiles than CTAs"""
    tile_h = 128 // w
    n, h, dil, res, relu = 2, 3 * tile_h, 1, True, True
    if variant == "dmid_norelu":
        dil, res, relu = w // 4 + 1, False, False
    elif variant == "dmax_res_norelu":
        dil, relu = w - 1, False
    elif variant == "dmax_relu":
        dil, res = w - 1, False
    elif variant == "ragged":
        h, dil = 3 * tile_h + 1 if tile_h > 1 else 5, 3
    elif variant == "persistent":
        h = 4 * tile_h
        n = 2 * 132 // 4 * 2 + 3             # ~2.3 x 264 tiles: several per CTA for both CTA counts
    g = synth._gen(35, f"pair{c}{w}{variant}")
    x = q(torch.randn(n, h, w, c, generator=g)).to(cuda)
    w1 = q(torch.randn(c, c, 3, generator=g) / (3 * c) ** 0.5).to(cuda)
    w2 = q(torch.randn(c, c, 3, generator=g) / (3 * c) ** 0.5).to(cuda)
    b1, t2 = (torch.randn(c, generator=g) * 0.1).to(cuda), (torch.randn(c, generator=g) * 0.1).to(cuda)
    r = q(torch.randn(n, h, w, c, generator=g)).to(cuda) if res else None
    want = pair_want(x, w1, b1, w2, t2, dil, r, relu)
    full = canary((n + 1, h, w, c), ops.h16(), cuda)
    out = ops.conv_pair_umma(x.to(ops.h16()), w1.permute(2, 0, 1).to(ops.h16()).contiguous(), b1,
                             w2.permute(2, 0, 1).to(ops.h16()).contiguous(), t2, dil,
                             res=None if r is None else r.to(ops.h16()), post_relu=relu, out=full[:n])
    torch.cuda.synchronize()
    assert not bool(is_canary(out).any()), f"{int(is_canary(out).sum())} outputs never written"
    assert bool(is_canary(full[n:]).all()), "written past the end of the output"
    if not relu:
        assert float(want.min()) < 0
    assert rel(out, want) < 1e-2, rel(out, want)


# ------------------------------------------------------------------------------------------------------------- conv7x7s2_umma
@pytest.mark.parametrize("shape", [(2, 20, 24, 128), (1, 22, 18, 192), (2, 49, 51, 64), (3, 7, 7, 64), (2, 9, 30, 128), (1, 31, 8, 64)])
def test_conv7x7s2_umma_contract(cuda, shape):
    """2 and 3 K chunks (cin 128, 192), odd h and w, the minimum 7 x 7, h != w both ways; nothing written past the end"""
    n, h, w, cin = shape
    g = synth._gen(36, str(shape))
    x = q(torch.randn(n, h, w, cin, generator=g)).to(cuda)
    wt = q(torch.randn(64, cin, 7, 7, generator=g) / (49 * cin) ** 0.5).to(cuda)
    b = (torch.randn(64, generator=g) * 0.5).to(cuda)
    want = F.relu(nhwc(F.conv2d(nchw(x), wt, b.double(), 2, 3)))
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    full = canary((n + 1, ho, wo, 64), ops.h16(), cuda)
    out = ops.conv7x7s2_umma(x.to(ops.h16()), ops.pack_conv7x7s2_weights(wt), b, out=full[:n])
    torch.cuda.synchronize()
    assert not bool(is_canary(out).any())
    assert bool(is_canary(full[n:]).all())
    assert rel(out, want) < 2e-3, rel(out, want)


# ------------------------------------------------------------------------------------- per-launch shared memory of erf_nb16
def test_erf_nb16_wide_rows_after_narrow_rows(cuda):
    """erf_nb16's dynamic shared memory grows with the image width, and the limit a kernel may use is raised once per process:
    a first call on 16-pixel rows must not cap a later call on 256-pixel rows (the widest the header allows).  Runs in a fresh
    process so that no earlier test has raised the limit already."""
    code = textwrap.dedent("""
        import torch
        from lav_b200 import ops
        w4 = torch.randn(4, 3, 16, 16, device="cuda") * 0.2
        st = torch.stack([torch.ones(4, 16, device="cuda"), torch.zeros(4, 16, device="cuda")], 2).contiguous()
        for w in (16, 256):
            y = ops.erf_nb16(torch.randn(2, 9, w, 16, device="cuda").to(ops.h16()), w4, st)
            assert bool(torch.isfinite(y.float()).all())
        torch.cuda.synchronize()
        print("nb16 ok")
    """)
    r = subprocess.run([sys.executable, "-c", code], cwd=util.ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "nb16 ok" in r.stdout, r.stdout[-1000:] + r.stderr[-3000:]


# ------------------------------------------------------------------------------------------------------ 16-bit ERFNet vs oracle
@pytest.mark.parametrize("weights", ["seeded", "real"])
def test_erfnet_f16_matches_oracle(cuda, weights):
    """RGBSegmentationModel.set_precision('f16') — the network the agent runs (fused stem, nb16 blocks, wgmma convs and pairs) —
    on uint8 frames through forward_u8, against the fp32 oracle: logit rms and max-norm within 1e-2 of the logit scale, and
    the per-pixel argmax with real weights.  Measured on one H100 SXM 80 GB (400 W power limit): seeded weights rms 1.34e-3,
    max-norm 1.82e-3, argmax agreement 0.99940; real weights rms 3.35e-4, max-norm 8.89e-4, argmax agreement 0.99985."""
    if weights == "real" and not util.have_real_seg():
        pytest.skip("oracle/_ref/seg_1.state_dict.pt not staged")
    m, sd = util.seg_model(cuda, real=(weights == "real"))
    m.set_precision("f16")
    rgb_u8 = synth.rgb_frames(smooth=True)
    with torch.no_grad():
        want = O.erfnet(sd, rgb_u8.permute(0, 3, 1, 2).float()).double()
        got = m.forward_u8(rgb_u8.to(cuda)).double().cpu()
    assert got.shape == want.shape == (3, 5, 288, 256)
    assert bool(torch.isfinite(got).all())
    rms = float(((got - want) ** 2).mean().sqrt() / (want ** 2).mean().sqrt())
    mx = rel(got, want)
    agree = float((got.argmax(1) == want.argmax(1)).double().mean())
    print(f"erfnet f16 vs oracle ({weights}): rms {rms:.2e}  max {mx:.2e}  argmax agreement {agree:.5f}")
    assert rms < 1e-2, rms
    assert mx < 1e-2, mx
    if weights == "real":
        assert agree > 0.99, agree
