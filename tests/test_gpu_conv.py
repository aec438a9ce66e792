"""GPU parity: tap-list convolution layers, the BEV backbone + heads and ERFNet against the oracle."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from lav_b200 import ops, synth
from oracle import lav_ref as O
from tests import util

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("cfg", [
    dict(cin=64, cout=64, k=(3, 3), s=1, p=(1, 1), d=(1, 1)),
    dict(cin=64, cout=128, k=(3, 3), s=2, p=(1, 1), d=(1, 1)),
    dict(cin=128, cout=128, k=(3, 1), s=1, p=(4, 0), d=(4, 1)),
    dict(cin=16, cout=16, k=(1, 3), s=1, p=(0, 1), d=(1, 1)),
    dict(cin=4, cout=13, k=(3, 3), s=2, p=(1, 1), d=(1, 1)),
    dict(cin=128, cout=128, k=(4, 4), s=2, p=(1, 1), d=(1, 1), t=True, op=0),
    dict(cin=128, cout=128, k=(4, 4), s=4, p=(1, 1), d=(1, 1), t=True, op=2),
    dict(cin=64, cout=3, k=(3, 3), s=2, p=(1, 1), d=(1, 1), t=True, op=1),
    dict(cin=16, cout=5, k=(2, 2), s=2, p=(0, 0), d=(1, 1), t=True, op=0),
    dict(cin=64, cout=128, k=(1, 1), s=1, p=(0, 0), d=(1, 1), t=True, op=0),
])
@pytest.mark.parametrize("dtype", ["fp32", "f16"])
def test_tapconv_vs_torch(cuda, cfg, dtype):
    from lav_b200.layers import TapConv
    g = synth._gen(9, str(cfg))
    t = cfg.get("t", False)
    cin, cout, (kh, kw) = cfg["cin"], cfg["cout"], cfg["k"]
    w = torch.randn((cin, cout, kh, kw) if t else (cout, cin, kh, kw), generator=g) / (cin * kh * kw) ** 0.5
    b = torch.randn(cout, generator=g)
    sc, sh = torch.rand(cout, generator=g) + 0.5, torch.randn(cout, generator=g)
    x = torch.randn(2, cin, 22, 26, generator=g)
    if t:
        y = F.conv_transpose2d(x, w, b, cfg["s"], cfg["p"], cfg["op"], 1, cfg["d"])
    else:
        y = F.conv2d(x, w, b, cfg["s"], cfg["p"], cfg["d"])
    res = torch.randn(y.shape, generator=g)
    want = F.relu(F.relu(y) * sc[None, :, None, None] + sh[None, :, None, None] + res)
    layer = TapConv(w.to(cuda), t, cfg["s"], cfg["p"], cfg["d"], cfg.get("op", 0), bias=b.to(cuda), pre_relu=True,
                    scale=sc.to(cuda), shift=sh.to(cuda), post_relu=True)
    tdt = torch.float32 if dtype == "fp32" else ops.h16()
    xin = x.permute(0, 2, 3, 1).contiguous().to(cuda).to(tdt)
    rin = res.permute(0, 2, 3, 1).contiguous().to(cuda).to(tdt)
    got = layer(xin, res=rin).float().cpu().permute(0, 3, 1, 2)
    tol = 1e-5 if dtype == "fp32" else 5e-3
    assert got.shape == want.shape
    assert util.rel_err(got, want) < tol


def test_lidar_model_matches_oracle_fp32(cuda, golden_dir):
    m, sd = util.lidar_model(cuda)
    clouds = util.pillar_clouds()
    npts = [len(c) for c in clouds]
    with torch.no_grad():
        want = O.lidar_model(sd, clouds, npts, **util.GRID)
        got = m([c.to(cuda) for c in clouds], npts)
    names = ["features", "center", "box", "ori", "seg"]
    for n, a, b in zip(names, got, want):
        assert a.shape == b.shape, n
        assert util.rel_err(a, b) < 1e-3, (n, util.rel_err(a, b))       # north_star: 1e-3 fp32
    gold = np.load(os.path.join(golden_dir, "lidar_model.npz"))           # REFERENCE outputs
    assert util.rel_err(got[0][:, :, ::8, ::8], torch.from_numpy(gold["features_s8"])) < 1e-3
    for n, t in zip(names[1:], got[1:]):
        assert util.rel_err(t[:, :, ::4, ::4], torch.from_numpy(gold[n + "_s4"])) < 1e-3
    # sub-modules are individually callable like the reference's (InferModel reaches into them)
    with torch.no_grad():
        feats = m.backbone(m.point_pillar_net([c.to(cuda) for c in clouds], npts))
        assert util.rel_err(feats, want[0]) < 1e-3
        assert util.rel_err(m.seg_head(feats), want[4]) < 1e-3
        assert util.rel_err(m.center_head(feats), want[1]) < 1e-3


def _assert_f16_close(outputs, ref_feats, sd):
    """outputs: (name, got, want) triples of the LiDAR model, ref_feats: the oracle's features"""
    for n, a, b in outputs:
        a = a.float().cpu()
        # north_star tolerance of the 16-bit tensor-core path: 1e-2 (max-norm AND rms, of the tensor scale).  With IEEE-half
        # storage + fp32 accumulation the 12 chained layers measure 1-2e-3 on these seeded, non-contractive weights
        # (bfloat16 storage measured 1.0-1.7e-2, which is why the path is half — DESIGN.md §5).
        rms = float(((a - b) ** 2).mean().sqrt() / (b ** 2).mean().sqrt())
        assert rms < 1e-2, (n, rms)
        if n != "seg":
            assert util.rel_err(a, b) < 1e-2, (n, util.rel_err(a, b))
        else:
            e = util.seg_logit_err(a, ref_feats, sd)        # pre-sigmoid error over the logit scale (see util.seg_logit_err)
            assert e < 1e-2, (n, e)


def test_lidar_model_f16(cuda):
    m, sd = util.lidar_model(cuda)
    m.set_precision("f16")
    clouds = util.pillar_clouds()
    npts = [len(c) for c in clouds]
    with torch.no_grad():
        want = O.lidar_model(sd, clouds, npts, **util.GRID)
        got = m([c.to(cuda) for c in clouds], npts)
    _assert_f16_close(zip(["features", "center", "box", "ori", "seg"], got, want), want[0], sd)


def test_lidar_model_f16_submodules(cuda):
    """the f16 sub-modules called one by one, as InferModel may: PointPillarNet.forward returns the fp32 canvas, which the
    backbone rounds to h16 exactly as the encoder's h16 canvas is rounded, so the chain runs the product path's layers."""
    m, sd = util.lidar_model(cuda)
    m.set_precision("f16")
    clouds = util.pillar_clouds()
    npts = [len(c) for c in clouds]
    with torch.no_grad():
        want = O.lidar_model(sd, clouds, npts, **util.GRID)
        feats = m.backbone(m.point_pillar_net([c.to(cuda) for c in clouds], npts))
        got = [("features", feats, want[0]), ("seg", m.seg_head(feats), want[4]), ("center", m.center_head(feats), want[1])]
    _assert_f16_close(got, want[0], sd)


@pytest.mark.parametrize("weights", ["seeded", "real"])
def test_erfnet_matches_oracle(cuda, weights, golden_dir):
    if weights == "real" and not util.have_real_seg():
        pytest.skip("oracle/_ref/seg_1.state_dict.pt not staged")
    m, sd = util.seg_model(cuda, real=(weights == "real"))
    rgb_u8 = synth.rgb_frames(smooth=True)
    rgb = rgb_u8.permute(0, 3, 1, 2).float()
    with torch.no_grad():
        want = O.erfnet(sd, rgb)
        got = m(rgb.to(cuda)).cpu()
        got_u8 = m.forward_u8(rgb_u8.to(cuda)).cpu()
    assert got.shape == want.shape == (3, 5, 288, 256)
    assert util.rel_err(got, want) < 1e-3
    assert util.rel_err(got_u8, got) < 1e-5          # uint8 frames take the fused normalize + initial-block kernel: same math, other FMA order
    gold = np.load(os.path.join(golden_dir, "erfnet.npz"))
    key = "real_s4" if weights == "real" else "seeded_s4"
    if key in gold:
        assert util.rel_err(got[:, :, ::4, ::4], torch.from_numpy(gold[key])) < 1e-3
    if weights == "real":
        agree = float((got.argmax(1) == want.argmax(1)).float().mean())
        assert agree > 0.999


@pytest.mark.parametrize("cfg", [
    dict(cin=64, cout=64, k=(3, 3), p=(1, 1), d=(1, 1), hw=(24, 32)),
    dict(cin=128, cout=128, k=(3, 3), p=(1, 1), d=(1, 1), hw=(40, 40)),      # ragged tiles (40 % 16 != 0)
    dict(cin=384, cout=256, k=(3, 3), p=(1, 1), d=(1, 1), hw=(16, 48)),
    dict(cin=128, cout=128, k=(3, 1), p=(8, 0), d=(8, 1), hw=(36, 32)),      # ERFNet dilated factorised conv
    dict(cin=64, cout=64, k=(1, 3), p=(0, 1), d=(1, 1), hw=(72, 64)),
    dict(cin=128, cout=128, k=(4, 4), p=(1, 1), d=(1, 1), hw=(20, 24), t=True, s=2, op=0),
    dict(cin=128, cout=128, k=(4, 4), p=(1, 1), d=(1, 1), hw=(10, 10), t=True, s=4, op=2),
    dict(cin=64, cout=128, k=(1, 1), p=(0, 0), d=(1, 1), hw=(24, 32), t=True, s=1, op=0),
    dict(cin=64, cout=16, k=(3, 3), p=(1, 1), d=(1, 1), hw=(20, 24), t=True, s=2, op=1, nores=True),   # cout padded to the MMA width
    dict(cin=64, cout=64, k=(3, 3), p=(1, 1), d=(1, 1), hw=(32, 64), cs=2),           # strided conv: TMA element strides
    dict(cin=64, cout=128, k=(3, 3), p=(1, 1), d=(1, 1), hw=(40, 36), cs=2),
])
def test_umma_conv_vs_torch(cuda, cfg):
    """wgmma implicit-GEMM conv against fp32 torch on f16-rounded operands (so only accumulation order differs)."""
    from lav_b200 import layers
    from lav_b200.layers import TapConv
    g = synth._gen(21, str(cfg))
    t = cfg.get("t", False)
    s = cfg.get("s", 1)
    cin, cout, (kh, kw) = cfg["cin"], cfg["cout"], cfg["k"]
    w = (torch.randn((cin, cout, kh, kw) if t else (cout, cin, kh, kw), generator=g) / (cin * kh * kw) ** 0.5).to(ops.h16()).float()
    b = torch.randn(cout, generator=g)
    sc, sh = torch.rand(cout, generator=g) + 0.5, torch.randn(cout, generator=g)
    x = torch.randn(3, cin, *cfg["hw"], generator=g).to(ops.h16()).float()
    if t:
        y = F.conv_transpose2d(x, w, b, s, cfg["p"], cfg["op"], 1, cfg["d"])
    else:
        s = cfg.get("cs", 1)
        y = F.conv2d(x, w, b, s, cfg["p"], cfg["d"])
    res = torch.randn(y.shape, generator=g).to(ops.h16()).float()
    if cfg.get("nores"):
        res = torch.zeros_like(res)
    want = F.relu(F.relu(y) * sc[None, :, None, None] + sh[None, :, None, None] + res)
    assert layers.USE_UMMA
    layer = TapConv(w.to(cuda), t, s, cfg["p"], cfg["d"], cfg.get("op", 0), bias=b.to(cuda), pre_relu=True,
                    scale=sc.to(cuda), shift=sh.to(cuda), post_relu=True)
    assert layer.umma_ok
    xin = x.permute(0, 2, 3, 1).contiguous().to(cuda).to(ops.h16())
    rin = None if cfg.get("nores") else res.permute(0, 2, 3, 1).contiguous().to(cuda).to(ops.h16())
    got32 = layer(xin, res=rin, out_dtype=torch.float32).cpu().permute(0, 3, 1, 2)
    assert util.rel_err(got32, want) < 2e-5          # fp32 output: only accumulation-order noise
    got16 = layer(xin, res=rin).float().cpu().permute(0, 3, 1, 2)
    assert util.rel_err(got16, want) < 1e-3          # f16 output rounding (2^-11)
    # linearity in the input batch: concatenating images must not mix them (tile scheduler / TMA image coordinate)
    one = layer(xin[1:2].contiguous(), res=None if rin is None else rin[1:2].contiguous(), out_dtype=torch.float32).cpu()
    assert torch.equal(one, layer(xin, res=rin, out_dtype=torch.float32).cpu()[1:2])


@pytest.mark.parametrize("dtype", ["fp32", "h16"])
def test_grouped_head_deconv_vs_torch(cuda, dtype):
    """the four Head.net[3] ConvTranspose2d(64->2/2/2/3,k3,s2,p1,op1) as one grouped launch"""
    dtype = torch.float32 if dtype == "fp32" else ops.h16()
    g = synth._gen(31, "deconv")
    hid = torch.randn(2, 256, 13, 17, generator=g)
    if dtype == ops.h16():
        hid = hid.to(ops.h16()).float()
    n_outs, sig = [2, 2, 2, 3], [False, False, False, True]
    ws = [torch.randn(64, no, 3, 3, generator=g) * 0.1 for no in n_outs]
    bs = [torch.randn(no, generator=g) for no in n_outs]
    wd, bd = torch.zeros(4, 64, 9, 4), torch.zeros(4, 4)
    for i, (w, b) in enumerate(zip(ws, bs)):
        wd[i, :, :, :n_outs[i]] = w.permute(0, 2, 3, 1).reshape(64, 9, n_outs[i])
        bd[i, :n_outs[i]] = b
    x = hid.permute(0, 2, 3, 1).contiguous().to(cuda).to(dtype)
    outs = ops.deconv3x3s2_small(x, 4, 64, wd.to(cuda), bd.to(cuda), n_outs, sig)
    for i in range(4):
        want = F.conv_transpose2d(hid[:, 64 * i:64 * i + 64], ws[i], bs[i], 2, 1, 1)
        if sig[i]:
            want = torch.sigmoid(want)
        got = outs[i].cpu().permute(0, 3, 1, 2)
        assert got.shape == want.shape
        assert util.rel_err(got, want) < 2e-5


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(2, 3, 32, 24), (1, 1, 31, 52), (1, 3, 9, 88), (1, 3, 288, 256), (2, 1, 192, 480)])
def test_stem_u8_vs_torch(cuda, shape):
    """lavb_stem7x7s2_u8 == Normalize + conv 7x7/s2/p3 (3->64) + bias + ReLU on the side-by-side camera image
    (team_code_v2/models/rgb.py:66-70, lav/models/resnet.py:235-238); operands rounded to f16 on both sides, tol 1e-2."""
    b, ncam, h, cw = shape
    g = torch.Generator().manual_seed(5)
    img = torch.randint(0, 256, (b, ncam, h, cw, 3), generator=g, dtype=torch.uint8)
    w = torch.randn(64, 3, 7, 7, generator=g) * 0.1
    bias = torch.randn(64, generator=g) * 0.1
    mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
    out = ops.stem7x7s2_u8(img.cuda(), ops.pack_stem_weights(w.cuda()), bias.cuda(), mean, std).float().cpu()
    wide = img.permute(0, 2, 1, 3, 4).reshape(b, h, ncam * cw, 3).permute(0, 3, 1, 2).float()
    x = (wide / 255. - torch.tensor(mean)[None, :, None, None]) / torch.tensor(std)[None, :, None, None]
    ref = F.relu(F.conv2d(x.to(ops.h16()).float(), w.to(ops.h16()).float(), bias, stride=2, padding=3))
    ref = ref.permute(0, 2, 3, 1)
    assert out.shape == ref.shape
    err = (out - ref).abs().max().item() / ref.abs().max().item()
    assert err < 1e-2, err


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(2, 7, 9, 64), (3, 144, 384, 64), (1, 1, 1, 8), (2, 96, 240, 64)])
def test_maxpool_nhwc_vs_torch(cuda, shape):
    """lavb_maxpool3x3s2_nhwc == MaxPool2d(3, 2, 1) (lav/models/resnet.py:181), bit-exact (values include negatives)."""
    x = torch.randn(shape, generator=torch.Generator().manual_seed(2)).to(ops.h16()).cuda()
    out = ops.maxpool3x3s2_nhwc(x)
    ref = F.max_pool2d(x.permute(0, 3, 1, 2).float(), 3, 2, 1).permute(0, 2, 3, 1).to(ops.h16())
    assert out.shape == ref.shape and torch.equal(out, ref)


@pytest.mark.gpu
def test_brake_forward_u8_matches_forward(cuda):
    """RGBBrakePredictionModel.forward_u8 (stem kernel on raw bytes) == forward(wide, tel) in f16."""
    from lav_b200.heads import RGBBrakePredictionModel
    torch.manual_seed(3)
    m = RGBBrakePredictionModel([4, 6, 7, 10]).eval()
    m.load_state_dict(synth.fill_state_dict_(m.state_dict(), seed=11))
    m = m.cuda()                                   # as FramePipeline.set_precision('f16'): trunk + attention in f16
    m.conv_backbone.to(ops.h16()).to(memory_format=torch.channels_last)
    m.attn1.to(ops.h16()); m.attn2.to(ops.h16())
    g = torch.Generator().manual_seed(9)
    rgbs = torch.randint(0, 256, (3, 3, 288, 256, 3), generator=g, dtype=torch.uint8).cuda()
    tel = torch.randint(0, 256, (3, 192, 480, 3), generator=g, dtype=torch.uint8).cuda()
    with torch.no_grad():
        wide = rgbs.permute(0, 2, 1, 3, 4).reshape(3, 288, 768, 3).permute(0, 3, 1, 2).float()
        a = m(wide, tel.permute(0, 3, 1, 2).float()).float()
        b = m.forward_u8(rgbs, tel).float()
    assert (a - b).abs().max().item() < 1e-2, (a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", [(3, 72, 64, 64, 1, True), (2, 36, 32, 128, 2, True), (2, 36, 32, 128, 16, True), (1, 7, 64, 64, 1, False),
                                 (24, 72, 64, 64, 1, True), (96, 36, 32, 128, 4, True)])   # last two: several tiles per CTA (persistent loop)
def test_conv_pair_umma_vs_torch(cuda, cfg):
    """lavb_conv_pair_umma == relu(conv3x1) -> conv1x3 -> affine (+res) -> relu of erfnet.py:37-63, f16 operands, tol 1e-2.
    The caller folds the BatchNorm scale into the second conv's weights (in fp32, rounded once) and passes b2*s + t as shift."""
    n, h, w, c, dil, use_res = cfg
    g = torch.Generator().manual_seed(4)
    x = torch.randn(n, c, h, w, generator=g)
    w1 = torch.randn(c, c, 3, 1, generator=g) * (1.0 / (3 * c) ** 0.5)
    w2 = torch.randn(c, c, 1, 3, generator=g) * (1.0 / (3 * c) ** 0.5)
    b1, b2 = torch.randn(c, generator=g) * 0.1, torch.randn(c, generator=g) * 0.1
    s2, t2 = torch.rand(c, generator=g) + 0.5, torch.randn(c, generator=g) * 0.1
    bf = lambda t: t.to(ops.h16()).float()
    mid = bf(F.relu(F.conv2d(bf(x), bf(w1), b1, padding=(dil, 0), dilation=(dil, 1))))
    w2 = w2 * s2[:, None, None, None]                                                  # the fold: (conv + b) s + t = conv_{w s} + (b s + t)
    ref = F.conv2d(mid, bf(w2), b2 * s2 + t2, padding=(0, dil), dilation=(1, dil))
    if use_res:
        ref = ref + bf(x)
    ref = F.relu(ref).permute(0, 2, 3, 1)
    xd = x.permute(0, 2, 3, 1).contiguous().to(ops.h16()).cuda()
    w1u = w1[:, :, :, 0].permute(2, 0, 1).contiguous().to(ops.h16()).cuda()       # [tap][cout][cin]
    w2u = w2[:, :, 0, :].permute(2, 0, 1).contiguous().to(ops.h16()).cuda()
    out = ops.conv_pair_umma(xd, w1u, b1.cuda(), w2u, (b2 * s2 + t2).cuda(), dil, res=xd if use_res else None).float().cpu()
    err = (out - ref).abs().max().item() / ref.abs().max().item()
    assert err < 1e-2, err


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(3, 144, 128), (2, 20, 32), (1, 7, 16), (5, 33, 64)])
def test_erf_nb16_block_vs_torch(cuda, shape):
    """lavb_erf_nb16 == non_bottleneck_1d(16, dilated=1) in eval mode (lav/models/erfnet.py:37-63), h16 operands: ragged
    heights (tiles of 8 rows, halo rows above/below the image) and every supported width."""
    from lav_b200.erfnet import _NB1D, non_bottleneck_1d
    n, h, w = shape
    torch.manual_seed(5)
    blk = non_bottleneck_1d(16, 0.0, 1).eval()
    sd = synth.fill_state_dict_(blk.state_dict())
    blk.load_state_dict(sd)
    x = torch.randn(n, 16, h, w)
    with torch.no_grad():
        want = O._erf_nb1d(x.to(ops.h16()).float(), {k: v.clone() for k, v in sd.items()}, "", 1).permute(0, 2, 3, 1)
    plan = _NB1D(blk.to(cuda))
    assert plan.nb16 is not None
    got = ops.erf_nb16(x.permute(0, 2, 3, 1).contiguous().to(cuda).to(ops.h16()), *plan.nb16).float().cpu()
    err = (got - want).abs().max().item() / want.abs().max().item()
    assert err < 5e-3, err


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(3, 288, 256), (2, 18, 70), (1, 2, 2)])
def test_erf_stem_vs_torch(cuda, shape):
    """lavb_erf_stem == normalize + DownsamplerBlock(3, 16) (lav/models/rgb.py:41-45, erfnet.py:12-23) on uint8 frames, fp32
    output at 1e-5 (borders = zero padding in the NORMALISED domain, ragged tiles)."""
    n, h, w = shape
    m, sd = util.seg_model(cuda)
    stem = m.erfnet._build(cuda)[3]
    rgb = torch.randint(0, 256, (n, h, w, 3), generator=torch.Generator().manual_seed(7), dtype=torch.uint8)
    with torch.no_grad():
        x = (rgb.permute(0, 3, 1, 2).float() / 255. - .5) * 2
        want = O._erf_down(x, sd, "erfnet.encoder.initial_block.").permute(0, 2, 3, 1)
    got = ops.erf_stem(rgb.to(cuda), *stem, torch.float32).cpu()
    assert got.shape == want.shape == (n, h // 2, w // 2, 16)
    assert util.rel_err(got, want) < 1e-5
    got16 = ops.erf_stem(rgb.to(cuda), *stem, ops.h16()).float().cpu()
    assert util.rel_err(got16, want) < 1e-3


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(3, 144, 128), (2, 20, 36), (1, 2, 2), (5, 10, 128)])
def test_erf_down16_block_vs_torch(cuda, shape):
    """lavb_erf_down16 == DownsamplerBlock(16, 64) in eval mode (lav/models/erfnet.py:12-23): conv3x3 s2 p1 (48) || maxpool2x2
    (16) -> BN -> ReLU, h16 operands; ragged tiles, narrow images, the left / top zero padding."""
    from lav_b200.erfnet import DownsamplerBlock, _Down
    n, h, w = shape
    blk = DownsamplerBlock(16, 64).eval()
    sd = synth.fill_state_dict_(blk.state_dict())
    blk.load_state_dict(sd)
    x = torch.randn(n, 16, h, w, generator=torch.Generator().manual_seed(9))
    with torch.no_grad():
        want = O._erf_down(x.to(ops.h16()).float(), {k: v.clone() for k, v in sd.items()}, "").permute(0, 2, 3, 1)
    plan = _Down(blk.to(cuda))
    assert plan.down16 is not None
    got = ops.erf_down16(x.permute(0, 2, 3, 1).contiguous().to(cuda).to(ops.h16()), *plan.down16).float().cpu()
    assert got.shape == want.shape == (n, h // 2, w // 2, 64)
    err = (got - want).abs().max().item() / want.abs().max().item()
    assert err < 3e-3, err
