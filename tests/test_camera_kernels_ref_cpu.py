"""CPU: the fp64 statements of the camera kernels (tests/util.py: erf_stem_ref64, erf_down16_ref64, erf_nb16_ref64,
stem7x7s2_u8_ref64, maxpool3x3s2_ref64) pinned to the oracle modules they stand for, and to hand-worked per-pixel loops at
corners, the left and top padding and the seams between cameras.  tests/test_gpu_camera_kernels_contract.py holds the
kernels to these statements."""
import functools

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from lav_b200 import ops, synth
from oracle import lav_ref as O
from tests import util

MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]


def h16r(t):
    return t.to(torch.float16).to(t.dtype)


def within(got, want, tol):
    d = (got - want).abs()
    assert bool((d <= tol).all()), f"{int((d > tol).sum())} of {d.numel()} over; worst {float((d - tol).max()):.3g}"


# ----------------------------------------------------------------------------------------------------- statement vs model
def test_erf_stem_lut_is_the_reference_formula():
    """the kernel's LUT, (v / 255 - .5) * 2 with three fp32 roundings, is bit for bit rgb.py:41 in torch fp32"""
    assert torch.equal(util.erf_stem_lut(), ((torch.arange(256).float() / 255. - .5) * 2).double())


def _seg_stem():
    m, sd = util.seg_model()
    return m.erfnet._build(torch.device("cpu"))[3], sd


@pytest.mark.parametrize("out_dtype", [torch.float32, torch.float16])
def test_erf_stem_statement_is_the_initial_block(out_dtype):
    """erf_stem_ref64 == _erf_down(initial_block) on the normalised image: within the statement's bound plus the model's
    own fp32 rounding (its unfused BatchNorm)"""
    stem, sd = _seg_stem()
    rgb = torch.randint(0, 256, (2, 18, 70, 3), generator=torch.Generator().manual_seed(7), dtype=torch.uint8)
    rgb[0, 0, :, :] = 255
    rgb[1, :, 0, :] = 0
    want, bound = util.erf_stem_ref64(rgb, *stem, out_dtype)
    with torch.no_grad():
        x = (rgb.permute(0, 3, 1, 2).float() / 255. - .5) * 2
        model = O._erf_down(x, sd, "erfnet.encoder.initial_block.").permute(0, 2, 3, 1).double()
    assert want.shape == (2, 9, 35, 16)
    within(want, model, bound + 2.0 ** -20 * model.abs().max())


def test_erf_down16_statement_is_the_downsampler():
    """erf_down16_ref64 == _erf_down(DownsamplerBlock(16, 64)) on h16 input with h16-exact conv weights (so the kernel's
    weight rounding is the identity), within the bound plus the model's fp32 rounding"""
    from lav_b200.erfnet import DownsamplerBlock, _Down
    blk = DownsamplerBlock(16, 64).eval()
    sd = synth.fill_state_dict_(blk.state_dict())
    sd["conv.weight"] = h16r(sd["conv.weight"])
    blk.load_state_dict(sd)
    x = h16r(torch.randn(2, 16, 10, 22, generator=torch.Generator().manual_seed(9)))
    plan = _Down(blk)
    want, bound = util.erf_down16_ref64(x.permute(0, 2, 3, 1).half(), *plan.down16)
    with torch.no_grad():
        model = O._erf_down(x, {k: v.clone() for k, v in sd.items()}, "").permute(0, 2, 3, 1).double()
    within(want, model, bound + 2.0 ** -20 * model.abs().max())


def test_erf_nb16_statement_is_non_bottleneck_1d():
    """erf_nb16_ref64 == _erf_nb1d(non_bottleneck_1d(16, dilated 1)) on h16 input with h16-exact conv weights: the model
    keeps its intermediates in fp32, the statement rounds them to h16, which the bound's one-ulp terms cover"""
    from lav_b200.erfnet import _NB1D, non_bottleneck_1d
    blk = non_bottleneck_1d(16, 0.0, 1).eval()
    sd = synth.fill_state_dict_(blk.state_dict())
    for k in sd:
        if k.endswith(".weight") and k.startswith("conv"):
            sd[k] = h16r(sd[k])
    blk.load_state_dict(sd)
    x = h16r(torch.randn(2, 16, 11, 32, generator=torch.Generator().manual_seed(5)))
    want, bound = util.erf_nb16_ref64(x.permute(0, 2, 3, 1).half(), *_NB1D(blk).nb16)
    with torch.no_grad():
        model = O._erf_nb1d(x, {k: v.clone() for k, v in sd.items()}, "", 1).permute(0, 2, 3, 1).double()
    within(want, model, bound + 2.0 ** -20 * model.abs().max())


def _brake_stem(seed=3):
    g = torch.Generator().manual_seed(seed)
    sd = {"conv1.weight": torch.randn(64, 3, 7, 7, generator=g) * 0.1, "bn1.weight": torch.rand(64, generator=g) + 0.5,
          "bn1.bias": torch.randn(64, generator=g) * 0.1, "bn1.running_mean": torch.randn(64, generator=g) * 0.1,
          "bn1.running_var": torch.rand(64, generator=g) + 0.5}
    s = sd["bn1.weight"].double() / torch.sqrt(sd["bn1.running_var"].double() + 1e-5)          # heads.py's fold
    w = (sd["conv1.weight"].double() * s[:, None, None, None]).float()
    b = (sd["bn1.bias"].double() - sd["bn1.running_mean"].double() * s).float()
    return sd, ops.pack_stem_weights(w), b


def test_stem_u8_operand_against_the_reference_normalisation():
    """the staged operand fmaf(u8, na, nb) differs from the reference's fp32 (x / 255 - mean) / std: with the ImageNet
    constants it does so in 522 of the 768 (byte, channel) pairs, by at most 2^-21 (a few fp32 ulps at the operand's scale
    of ~2; each side makes three or four fp32 roundings of values below 4.5, 8 u (255 na + |nb|) < 3.1e-6 bounds it).
    Rounded to h16 the two operands are identical for every byte value."""
    m, s = np.asarray(MEAN, np.float32), np.asarray(STD, np.float32)
    na, nb = np.float32(1) / (np.float32(255) * s), -m / s
    f32 = (np.arange(256, dtype=np.float64)[:, None] * na.astype(np.float64) + nb.astype(np.float64)).astype(np.float32)
    ref = ((torch.arange(256).float()[:, None] / 255. - torch.tensor(MEAN)) / torch.tensor(STD)).numpy()
    d = np.abs(f32.astype(np.float64) - ref.astype(np.float64))
    assert int((d > 0).sum()) == 522 and float(d.max()) == 2.0 ** -21
    assert float(d.max()) <= 8 * 2.0 ** -24 * float((255 * na + np.abs(nb)).max())
    assert torch.equal(util.stem_u8_operand(MEAN, STD), torch.from_numpy(ref).half().double())
    assert torch.equal(util.stem_u8_operand(MEAN, STD), torch.from_numpy(f32).half().double())


@pytest.mark.parametrize("shape", [(1, 3, 20, 16), (2, 1, 9, 12)])
def test_stem_u8_statement_is_conv1_bn1_relu(shape):
    """stem7x7s2_u8_ref64 == resnet18_features' conv1 / bn1 / ReLU on (x / 255 - mean) / std of the side-by-side image:
    within the bound plus the h16 rounding of the folded weights and the operands, 2^-10 sum |x w|"""
    b, ncam, h, cw = shape
    sd, wk, bias = _brake_stem()
    img = torch.randint(0, 256, (b, ncam, h, cw, 3), generator=torch.Generator().manual_seed(4), dtype=torch.uint8)
    want, bound = util.stem7x7s2_u8_ref64(img, wk, bias, MEAN, STD)
    wide = img.permute(0, 2, 1, 3, 4).reshape(b, h, ncam * cw, 3).permute(0, 3, 1, 2).float()
    x = (wide / 255. - torch.tensor(MEAN)[None, :, None, None]) / torch.tensor(STD)[None, :, None, None]
    with torch.no_grad():
        model = O._cbr(x, sd, "conv1.", "bn1.", 2, 3).permute(0, 2, 3, 1).double()
    sa = F.conv2d(x.double().abs(), sd["conv1.weight"].double().abs(), stride=2, padding=3)
    s = (sd["bn1.weight"].double() / torch.sqrt(sd["bn1.running_var"].double() + 1e-5)).abs()
    slack = 2.0 ** -10 * (sa * s[None, :, None, None]).permute(0, 2, 3, 1)
    assert want.shape == model.shape
    within(want, model, bound + slack + 2.0 ** -20 * model.abs().max())


def test_maxpool_statement_is_max_pool2d():
    """maxpool3x3s2_ref64 == F.max_pool2d(3, 2, 1), NaN, +-inf and +-65504 included, except for the +-0 rule"""
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, 7, 9, 16, generator=g).half()
    flat = x.view(-1)
    idx = torch.randperm(flat.numel(), generator=g)
    flat[idx[:20]] = float("nan")
    flat[idx[20:30]] = float("inf")
    flat[idx[30:40]] = -float("inf")
    flat[idx[40:50]] = 65504
    flat[idx[50:60]] = -65504
    got = util.maxpool3x3s2_ref64(x)
    want = F.max_pool2d(x.double().permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
    nan = torch.isnan(want)
    assert bool(nan.any()) and torch.equal(torch.isnan(got), nan) and torch.equal(got[~nan], want[~nan])


def test_maxpool_statement_zero_rule():
    """-0 ranks below +0: a window holding -0 then +0 gives +0 where max_pool2d keeps the first, -0"""
    x = torch.full((1, 3, 3, 8), -1.0).half()
    x[0, 0, 0] = -0.0
    x[0, 1, 1] = 0.0
    got = util.maxpool3x3s2_ref64(x)
    torch_ = F.max_pool2d(x.double().permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
    assert not bool(torch.signbit(got[0, 0, 0]).any()) and bool(torch.signbit(torch_[0, 0, 0]).all())
    x[0, 1, 1] = -1.0
    assert bool(torch.signbit(util.maxpool3x3s2_ref64(x)[0, 0, 0]).all())       # -0 alone stays -0


# ----------------------------------------------------------------------------------------------------- hand-worked pixels
def test_erf_stem_statement_by_hand():
    """single output pixels by an explicit loop over the 3x3 window and the 2x2 pool: the corners, the top and left
    padding, and a pixel inside"""
    stem, _ = _seg_stem()
    w27, s, t = (np.asarray(v, np.float64) for v in stem)
    rgb = torch.randint(0, 256, (1, 10, 14, 3), generator=torch.Generator().manual_seed(8), dtype=torch.uint8)
    lut = util.erf_stem_lut().numpy()
    want, bound = util.erf_stem_ref64(rgb, *stem, torch.float32)
    for oy, ox in [(0, 0), (0, 6), (4, 0), (4, 6), (2, 3)]:
        o = np.zeros(16)
        for co in range(13):
            acc = 0.0
            for ky in range(3):
                for kx in range(3):
                    iy, ix = 2 * oy - 1 + ky, 2 * ox - 1 + kx
                    if 0 <= iy < 10 and 0 <= ix < 14:
                        for c in range(3):
                            acc += lut[rgb[0, iy, ix, c]] * w27[(ky * 3 + kx) * 3 + c, co]
            o[co] = max(acc * s[co] + t[co], 0.0)
        for c in range(3):
            m = max(lut[rgb[0, 2 * oy + dy, 2 * ox + dx, c]] for dy in (0, 1) for dx in (0, 1))
            o[13 + c] = max(m * s[13 + c] + t[13 + c], 0.0)
        assert np.all(np.abs(o - want[0, oy, ox].numpy()) <= 1e-12 * (1 + np.abs(o))), (oy, ox)
        assert float(bound[0, oy, ox].max()) > 0


def test_erf_down16_statement_by_hand():
    """single output pixels by an explicit loop: corners, top / left padding, and the pool's NaN rule (a NaN is skipped;
    four NaNs give -inf, 65504 after a negative scale)"""
    g = torch.Generator().manual_seed(11)
    x = torch.randn(1, 8, 10, 16, generator=g).half()
    x[0, 2:4, 4:6, 0] = float("nan")                 # pooled output (1, 2): all four NaN in channel 0
    x[0, 0, 0, 1] = float("nan")                     # pooled output (0, 0): one NaN in channel 1
    w9 = torch.randn(9, 16, 48, generator=g) * 0.2
    st = torch.stack([torch.randn(64, generator=g), torch.randn(64, generator=g) * 0.1], 1)
    st[48, 0] = -1.5
    want, _ = util.erf_down16_ref64(x, w9, st)
    W = w9.half().double().numpy()
    xs, S = x.double().numpy(), st.double().numpy()
    for oy, ox in [(0, 0), (0, 4), (3, 0), (3, 4), (1, 2)]:
        o = np.zeros(64)
        for co in range(48):
            acc = 0.0
            for ky in range(3):
                for kx in range(3):
                    iy, ix = 2 * oy - 1 + ky, 2 * ox - 1 + kx
                    if 0 <= iy < 8 and 0 <= ix < 10:
                        acc += float(np.dot(xs[0, iy, ix], W[ky * 3 + kx, :, co]))
            o[co] = acc * S[co, 0] + S[co, 1]
        for c in range(16):
            vals = [xs[0, 2 * oy + dy, 2 * ox + dx, c] for dy in (0, 1) for dx in (0, 1)]
            m = max([v for v in vals if not np.isnan(v)], default=-np.inf)
            o[48 + c] = m * S[48 + c, 0] + S[48 + c, 1]
        o = np.where(np.isnan(o), 0.0, np.maximum(o, 0.0))
        o = np.minimum(o, 65504).astype(np.float16).astype(np.float64)
        assert np.all(np.abs(want[0, oy, ox].numpy() - o) <= 2.0 ** -10 * np.abs(o) + 2.0 ** -24), (oy, ox)
    assert float(want[0, 1, 2, 48]) == 65504.0
    assert float(want[0, 0, 0, 49]) == float(np.float16(max(xs[0, 0, 1, 1], xs[0, 1, 0, 1], xs[0, 1, 1, 1]) * S[49, 0] + S[49, 1]).clip(0))


def test_erf_nb16_statement_by_hand():
    """single output pixels through the four stages by an explicit recursion with h16 intermediates and zero padding:
    corners, the first and last rows (the halo rows outside the image), and a pixel inside"""
    g = torch.Generator().manual_seed(12)
    H, W = 5, 16
    x = torch.randn(1, H, W, 16, generator=g).half()
    w4 = torch.randn(4, 3, 16, 16, generator=g) * 0.25
    st = torch.stack([torch.rand(4, 16, generator=g) + 0.5, torch.randn(4, 16, generator=g) * 0.1], 2)
    want, _ = util.erf_nb16_ref64(x, w4, st)
    Wt, S, xs = w4.half().double().numpy(), st.double().numpy(), x.double().numpy()[0]

    @functools.lru_cache(maxsize=None)
    def stage(k, y, x_):
        if not (0 <= y < H and 0 <= x_ < W):
            return np.zeros(16)
        if k < 0:
            return xs[y, x_]
        acc = np.zeros(16)
        for tap in range(3):
            yy, xx = (y + tap - 1, x_) if k % 2 == 0 else (y, x_ + tap - 1)
            acc += stage(k - 1, yy, xx) @ Wt[k, tap]
        v = acc * S[k, :, 0] + S[k, :, 1]
        if k == 3:
            v = v + xs[y, x_]
        return np.minimum(np.maximum(v, 0.0), 65504).astype(np.float16).astype(np.float64)

    for y, x_ in [(0, 0), (0, W - 1), (H - 1, 0), (H - 1, W - 1), (2, 7)]:
        o = stage(3, y, x_)
        assert np.all(np.abs(want[0, y, x_].numpy() - o) <= 2.0 ** -9 * np.abs(o) + 2.0 ** -23), (y, x_)


def test_stem_u8_statement_by_hand():
    """single output pixels by an explicit loop that reads the (B, ncam, H, cam_w, 3) tensor itself, camera by camera: the
    corners, the top / left padding and the output columns whose 7-wide window crosses each of the three seams"""
    _, wk, bias = _brake_stem(seed=6)
    ncam, H, cw = 4, 11, 8
    img = torch.randint(0, 256, (1, ncam, H, cw, 3), generator=torch.Generator().manual_seed(13), dtype=torch.uint8)
    for c in range(ncam):                                # every camera distinct: a wrong camera index cannot go unseen
        img[0, c, :, :, c % 3] = 40 * c + 10
    want, _ = util.stem7x7s2_u8_ref64(img, wk, bias, MEAN, STD)
    op = util.stem_u8_operand(MEAN, STD).numpy()
    Wt = util.stem_unpack_weights(wk).numpy()
    b = bias.double().numpy()
    ho, wo = (H - 1) // 2 + 1, (ncam * cw - 1) // 2 + 1
    cols = [0, wo - 1] + [(s * cw) // 2 + d for s in (1, 2, 3) for d in (-1, 0, 1)]
    for oy, ox in [(0, c) for c in cols] + [(ho - 1, c) for c in cols] + [(2, 5)]:
        acc = b.copy()
        for ky in range(7):
            for kx in range(7):
                iy, X = 2 * oy - 3 + ky, 2 * ox - 3 + kx
                if 0 <= iy < H and 0 <= X < ncam * cw:
                    px = img[0, X // cw, iy, X % cw]
                    for c in range(3):
                        acc += op[px[c], c] * Wt[:, c, ky, kx]
        o = np.minimum(np.maximum(acc, 0.0), 65504).astype(np.float16).astype(np.float64)
        assert np.all(np.abs(want[0, oy, ox].numpy() - o) <= 2.0 ** -10 * np.abs(o) + 2.0 ** -24), (oy, ox)


def test_maxpool_statement_by_hand():
    """every output pixel of odd and even maps by an explicit loop over the clipped 3x3 window"""
    g = torch.Generator().manual_seed(14)
    for h, w in [(1, 1), (2, 3), (5, 4), (7, 9)]:
        x = torch.randn(1, h, w, 8, generator=g).half()
        got = util.maxpool3x3s2_ref64(x).numpy()
        xs = x.double().numpy()[0]
        for oy in range((h - 1) // 2 + 1):
            for ox in range((w - 1) // 2 + 1):
                win = [xs[iy, ix] for iy in range(2 * oy - 1, 2 * oy + 2) for ix in range(2 * ox - 1, 2 * ox + 2)
                       if 0 <= iy < h and 0 <= ix < w]
                assert np.array_equal(got[0, oy, ox], np.max(win, 0)), (h, w, oy, ox)


# ----------------------------------------------------------------------------------------------------- nb16 bound strength
def _nb16_fp32(x, w4, st, mid=torch.float16, wdt=torch.float16, shift=None, scale=None):
    """an fp32 forward of the nb16 block, used as a stand-in kernel: weights rounded to wdt, each stage's output stored as
    mid; shift = (stage, channel, delta) and scale = (stage, factor) perturb the affine constants"""
    x0 = x.float().permute(0, 3, 1, 2)
    W, S = w4.to(wdt).float(), st.clone()
    if shift:
        S[shift[0], shift[1], 1] += shift[2]
    if scale:
        S[scale[0], :, 0] *= scale[1]
    v = x0
    for k in range(4):
        Wk = W[k].permute(2, 1, 0)
        Wk, pad = (Wk[..., None], (1, 0)) if k % 2 == 0 else (Wk[:, :, None, :], (0, 1))
        pre = F.conv2d(v, Wk, padding=pad) * S[k, :, 0][None, :, None, None] + S[k, :, 1][None, :, None, None]
        if k == 3:
            pre = pre + x0
        v = torch.relu(pre).clamp(max=65504).to(mid).float()
    return v.permute(0, 2, 3, 1).double()


def test_erf_nb16_bound_tells_h16_from_bf16():
    """erf_nb16_ref64's acceptance rule on the GPU test's operands (util.nb16_test_params): an fp32 forward that stores h16
    intermediates passes, and forwards that store bf16 intermediates, read bf16 weights, add 0.1 or 0.01 to one shift, or
    scale one stage's BatchNorm by 1.05 fail"""
    w4, st = util.nb16_test_params(15)
    x = torch.randn(2, 17, 128, 16, generator=torch.Generator().manual_seed(16)).half()
    want, bound = util.erf_nb16_ref64(x, w4, st)

    def over(got):
        return int((((got - want).abs() > bound) & (got != want)).sum())

    assert over(_nb16_fp32(x, w4, st)) == 0
    assert over(_nb16_fp32(x, w4, st, mid=torch.bfloat16)) > 1000
    assert over(_nb16_fp32(x, w4, st, wdt=torch.bfloat16)) > 100
    assert over(_nb16_fp32(x, w4, st, scale=(2, 1.05))) > 1000
    for c in range(16):
        assert over(_nb16_fp32(x, w4, st, shift=(1, c, 0.1))) > 1000, c
    for k in range(4):
        for c in (0, 7, 15):
            assert over(_nb16_fp32(x, w4, st, shift=(k, c, 0.01))) > 0, (k, c)
