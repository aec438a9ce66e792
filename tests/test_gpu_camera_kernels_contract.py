"""GPU: the camera kernels lavb_erf_stem, lavb_erf_down16, lavb_erf_nb16, lavb_stem7x7s2_u8 and lavb_maxpool3x3s2_nhwc
against their whole C-ABI contract (include/lav_b200.h), each output element held to the fp64 statement and per-element
bound of tests/util.py (erf_stem_ref64, erf_down16_ref64, erf_nb16_ref64, stem7x7s2_u8_ref64; maxpool3x3s2_ref64 is exact,
bit for bit).  The statements run on the GPU in float64.

The kernels are called through capi with outputs filled beforehand with a NaN canary bit pattern and one spare image past
the end: every element of the documented output must be written and the spare image must keep the canary bit for bit.  The
ops wrappers are checked to give the same bits.  Every rejection is confirmed to launch nothing (torch.profiler, with a
control launch in the same capture) and to write nothing.  Cases cover each kernel's tile edges (erf_stem 8 x 32 output tiles, erf_down16 4 rows x 64 columns,
erf_nb16 8 rows with +-2 halo rows, stem7x7s2_u8 8 rows x 128 columns and the seams between cameras), the product shapes,
batch independence and run-to-run bit equality.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from lav_b200 import capi, ops
from tests import util
from tests.util import INT, canary, is_canary, kernels

pytestmark = pytest.mark.gpu

MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
RATIO = {}          # kernel -> largest |got - want| / bound seen at the product shapes (printed with -s)


def lib():
    return capi.lib()


def h16():
    return ops.h16()


def gen(seed):
    return torch.Generator().manual_seed(seed)


def bits(t):
    return t.contiguous().view(INT[t.dtype])


def hold(full, n, want, bound, what, product=False):
    """full: the canary-filled output with one spare image; the first n images must all be written and within the bound
    of the statement, the spare untouched"""
    got = full[:n]
    assert not bool(is_canary(got).any()), f"{what}: {int(is_canary(got).sum())} outputs never written"
    assert bool(is_canary(full[n:]).all()), f"{what}: written past the end of the output"
    g = got.double()
    err = (g - want).abs()
    ok = (err <= bound) | (g == want)
    assert bool(ok.all()), (f"{what}: {int((~ok).sum())} of {ok.numel()} outside the bound; worst at "
                            f"{np.unravel_index(int(torch.argmax(torch.where(ok, 0., err - bound))), tuple(ok.shape))}")
    finite = torch.isfinite(want) & (bound > 0)
    r = float((err[finite] / bound[finite]).max()) if bool(finite.any()) else 0.0
    if product:
        RATIO[what] = max(RATIO.get(what, 0.0), r)
        print(f"\n{what}: largest error / bound = {r:.3g}")
    return r


def rejected(tmp_path, cases, outs):
    """cases: (call, cause) pairs, each returning the entry point's status.  Every call must fail with a message naming its
    cause; together they must launch nothing and leave every output canary.  The capture ends with one valid control launch
    (a 1-pixel max-pool), so that it holds kernel records: the rejected calls launched nothing when the control is the only
    kernel the profiler saw."""
    seen = []
    x = torch.zeros(1, 1, 1, 8, dtype=h16(), device="cuda")
    y = torch.empty_like(x)

    def run():
        seen.clear()
        for fn, cause in cases:
            code = fn()
            seen.append((code, cause, lib().lavb_last_error().decode()))
        assert c_pool(x, 1, 1, 1, 8, y) == 0

    launched = kernels(run, tmp_path)
    assert len(launched) == 1 and "maxpool3x3s2_kernel" in launched[0][0], launched
    assert len(seen) == len(cases)
    for code, cause, msg in seen:
        assert code != 0 and cause in msg, (cause, code, msg)
    for o in outs:
        assert bool(is_canary(o).all())


# ------------------------------------------------------------------------------------------------------------- erf_stem
def stem_params(seed, nan_cols=False):
    g = gen(seed)
    w27 = (torch.randn(27, 16, generator=g) * 0.3).numpy()
    w27[:, 13:] = np.nan if nan_cols else 0.0
    s = (torch.rand(16, generator=g) + 0.5).numpy()
    s[[2, 14]] *= -1                                       # a negative scale on a conv and a pooled channel
    t = (torch.randn(16, generator=g) * 0.1).numpy()
    return w27.astype(np.float32), s.astype(np.float32), t.astype(np.float32)


def c_erf_stem(rgb, n, h, w, p, out, dt):
    a, b, c = (np.ascontiguousarray(v, dtype=np.float32) for v in p)
    return lib().lavb_erf_stem(ops._ptr(rgb), n, h, w, a.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p),
                               c.ctypes.data_as(C.c_void_p), ops._ptr(out), ops._DT[dt], ops._stream())


def run_erf_stem(rgb, p, dt):
    n, h, w, _ = rgb.shape
    full = canary((n + 1, h // 2, w // 2, 16), dt, rgb.device)
    assert c_erf_stem(rgb, n, h, w, p, full, dt) == 0
    return full


STEM_SHAPES = [(1, 2, 2), (2, 16, 62), (2, 16, 64), (2, 16, 66), (1, 16, 126), (1, 16, 128), (1, 16, 130),
               (2, 14, 70), (2, 16, 70), (2, 18, 70), (96, 288, 256)]


@pytest.mark.parametrize("dt", ["f32", "h16"])
@pytest.mark.parametrize("shape", STEM_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_erf_stem(cuda, shape, dt):
    """output widths 1 / 31..33 / 63..65, heights 7..9 across the 8 x 32 tiles, and the product's 96 x 288 x 256"""
    dt = torch.float32 if dt == "f32" else h16()
    n, h, w = shape
    p = stem_params(1)
    rgb = torch.randint(0, 256, (n, h, w, 3), generator=gen(2), dtype=torch.uint8).to(cuda)
    full = run_erf_stem(rgb, p, dt)
    want, bound = util.erf_stem_ref64(rgb, *p, dt)
    hold(full, n, want, bound, f"erf_stem {dt}", product=shape[0] == 96)
    again = run_erf_stem(rgb, p, dt)
    assert torch.equal(bits(again), bits(full))                                   # run to run
    assert torch.equal(bits(ops.erf_stem(rgb, *p, dt)), bits(full[:n]))          # the wrapper


@pytest.mark.parametrize("dt", ["f32", "h16"])
def test_erf_stem_every_byte_and_nan_columns(cuda, dt):
    """an image holding all 256 byte values in every channel with 0 and 255 along its borders; weight columns 13..15 NaN,
    which the kernel must never read"""
    dt = torch.float32 if dt == "f32" else h16()
    g = gen(3)
    rgb = torch.stack([torch.randperm(32 * 48, generator=g) % 256 for _ in range(3)], 1).reshape(1, 32, 48, 3).to(torch.uint8)
    rgb[0, 0], rgb[0, -1], rgb[0, :, 0], rgb[0, :, -1] = 0, 255, 255, 0
    assert all(len(torch.unique(rgb[..., c])) == 256 for c in range(3))
    rgb = rgb.to(cuda)
    p = stem_params(4, nan_cols=True)
    full = run_erf_stem(rgb, p, dt)
    want, bound = util.erf_stem_ref64(rgb, *p, dt)
    hold(full, 1, want, bound, "erf_stem every byte")
    assert not bool(torch.isnan(full[:1].float()).any())


def erf_stem_rejections(cuda, tmp_path):
    p = stem_params(5)
    rgb = torch.randint(0, 256, (2, 18, 70, 3), generator=gen(6), dtype=torch.uint8).to(cuda)
    f32 = canary((3, 9, 35, 16), torch.float32, cuda)
    hh = canary((3, 9, 35, 16), h16(), cuda)
    flat = canary((2 * 9 * 35 * 16 + 4,), torch.float32, cuda)
    cases = [
        (lambda: c_erf_stem(rgb, 2, 17, 70, p, f32, torch.float32), "even"),
        (lambda: c_erf_stem(rgb, 2, 18, 69, p, f32, torch.float32), "even"),
        (lambda: c_erf_stem(rgb, 2, 0, 70, p, f32, torch.float32), "even"),
        (lambda: c_erf_stem(rgb, -1, 18, 70, p, f32, torch.float32), "even"),
        (lambda: lib().lavb_erf_stem(ops._ptr(rgb), 2, 18, 70, *(v.ctypes.data_as(C.c_void_p) for v in p), ops._ptr(f32), 99,
                                     ops._stream()), "dtype"),
        (lambda: c_erf_stem(rgb, 2 ** 30, 18, 70, p, f32, torch.float32), "2^31"),
        (lambda: c_erf_stem(None, 2, 18, 70, p, f32, torch.float32), "null"),
        (lambda: c_erf_stem(rgb, 2, 18, 70, p, None, torch.float32), "null"),
        (lambda: lib().lavb_erf_stem(ops._ptr(rgb), 2, 18, 70, None, *(v.ctypes.data_as(C.c_void_p) for v in p[1:]),
                                     ops._ptr(f32), capi.F32, ops._stream()), "null"),
        (lambda: c_erf_stem(rgb, 2, 18, 70, p, flat[1:], torch.float32), "aligned"),              # 4 bytes off 16
        (lambda: c_erf_stem(rgb, 2, 18, 70, p, hh.view(-1)[2:], h16()), "aligned"),                # 4 bytes off 8
        (lambda: c_erf_stem(rgb, 2, 18, 70, p, rgb, torch.float32), "overlap"),
    ]
    rejected(tmp_path, cases, [f32, hh, flat])
    assert c_erf_stem(rgb, 0, 18, 70, p, f32, torch.float32) == 0 and bool(is_canary(f32).all())
    with pytest.raises(capi.LavbError):
        ops.erf_stem(rgb, *p, torch.int32)


# ----------------------------------------------------------------------------------------------------------- erf_down16
def down_params(seed):
    g = gen(seed)
    w9 = torch.randn(9, 16, 48, generator=g) * 0.15
    s = torch.rand(64, generator=g) + 0.5
    s[torch.arange(64) % 3 == 0] *= -1                     # negative BatchNorm scales, pooled channels included
    st = torch.stack([s, torch.randn(64, generator=g) * 0.1], 1)
    return w9, st


def c_down16(x, out, n, h, w, w9, st):
    return lib().lavb_erf_down16(ops._ptr(x), ops._ptr(out), n, h, w, ops._ptr(w9), ops._ptr(st), ops._stream())


def run_down16(x, w9, st):
    n, h, w, _ = x.shape
    full = canary((n + 1, h // 2, w // 2, 64), h16(), x.device)
    assert c_down16(x, full, n, h, w, w9, st) == 0
    return full


@pytest.mark.parametrize("h", [2, 6, 8, 10, 144])
@pytest.mark.parametrize("w", [2, 4, 30, 32, 34, 126, 128])
def test_erf_down16(cuda, w, h):
    """widths around the 64-column tile (output 1..64 columns), heights around the 4-row tile"""
    w9, st = (t.to(cuda) for t in down_params(7))
    x = torch.randn(2, h, w, 16, generator=gen(8)).to(cuda).to(h16())
    full = run_down16(x, w9, st)
    want, bound = util.erf_down16_ref64(x, w9, st)
    hold(full, 2, want, bound, "erf_down16")
    assert torch.equal(bits(ops.erf_down16(x, w9, st)), bits(full[:2]))


def test_erf_down16_product(cuda):
    """the product's 96 x 144 x 128 x 16, run twice for bit equality"""
    w9, st = (t.to(cuda) for t in down_params(9))
    x = torch.randn(96, 144, 128, 16, generator=gen(10)).to(cuda).to(h16())
    full = run_down16(x, w9, st)
    want, bound = util.erf_down16_ref64(x, w9, st)
    hold(full, 96, want, bound, "erf_down16", product=True)
    assert torch.equal(bits(run_down16(x, w9, st)), bits(full))


def test_erf_down16_nan(cuda):
    """NaN rules: a conv channel whose window holds a NaN is 0; the pool skips a NaN; a window of four NaNs gives -inf,
    0 after a positive scale and 65504 after a negative one"""
    w9, st = (t.to(cuda) for t in down_params(11))
    x = torch.randn(1, 8, 12, 16, generator=gen(12)).to(h16())
    x[0, 2:4, 4:6, :] = float("nan")                       # output (1, 2): every channel's pool window all NaN
    x[0, 6, 9, 3] = float("nan")                           # output (3, 4): one NaN in channel 3's window
    x = x.to(cuda)
    full = run_down16(x, w9, st)
    want, bound = util.erf_down16_ref64(x, w9, st)
    hold(full, 1, want, bound, "erf_down16 nan")
    got = full[0].float().cpu()
    s = st[48:, 0].cpu()
    assert torch.equal(got[1, 2, 48:], torch.where(s < 0, torch.tensor(65504.), torch.tensor(0.)))
    assert not bool(torch.isnan(got).any())


def erf_down16_rejections(cuda, tmp_path):
    w9, st = (t.to(cuda) for t in down_params(13))
    x = torch.randn(2, 8, 32, 16, generator=gen(14)).to(cuda).to(h16())
    big = torch.zeros(2, 8, 130, 16, device=cuda, dtype=h16())
    out = canary((3, 4, 16, 64), h16(), cuda)
    flat = canary((2 * 4 * 16 * 64 + 8,), h16(), cuda)
    xf = x.view(-1)
    xs = torch.zeros(xf.numel() + 8, dtype=h16(), device=cuda)
    cases = [
        (lambda: c_down16(big, out, 2, 8, 130, w9, st), "width"),
        (lambda: c_down16(x, out, 2, 8, 31, w9, st), "even"),
        (lambda: c_down16(x, out, 2, 7, 32, w9, st), "even"),
        (lambda: c_down16(x, out, -1, 8, 32, w9, st), "even"),
        (lambda: c_down16(x, out, 2 ** 30, 18, 32, w9, st), "2^31"),
        (lambda: c_down16(None, out, 2, 8, 32, w9, st), "null"),
        (lambda: c_down16(x, None, 2, 8, 32, w9, st), "null"),
        (lambda: c_down16(x, out, 2, 8, 32, None, st), "null"),
        (lambda: c_down16(x, out, 2, 8, 32, w9, None), "null"),
        (lambda: c_down16(xs[4:], out, 2, 8, 32, w9, st), "aligned"),                              # 8 bytes off 16
        (lambda: c_down16(x, flat[4:], 2, 8, 32, w9, st), "aligned"),
        (lambda: c_down16(x, x, 2, 8, 32, w9, st), "overlap"),
        (lambda: c_down16(x, xf[8 * 32 * 16:], 2, 8, 32, w9, st), "overlap"),                      # out = image 1 of x
        (lambda: c_down16(x, out, 2, 8, 32, out.view(-1)[64:], st), "overlaps d_w9"),
        (lambda: c_down16(x, out, 2, 8, 32, w9, out.view(-1)[4 * 16 * 64:]), "overlaps d_w9 or d_st"),
    ]
    rejected(tmp_path, cases, [out, flat])
    assert c_down16(x, out, 0, 8, 32, w9, st) == 0 and bool(is_canary(out).all())
    with pytest.raises(capi.LavbError):
        ops.erf_down16(x, w9[:8], st)


# ------------------------------------------------------------------------------------------------------------- erf_nb16
def nb_params(seed):
    return util.nb16_test_params(seed)


def c_nb16(x, out, n, h, w, w4, st):
    return lib().lavb_erf_nb16(ops._ptr(x), ops._ptr(out), n, h, w, ops._ptr(w4), ops._ptr(st), ops._stream())


def run_nb16(x, w4, st):
    n, h, w, _ = x.shape
    full = canary((n + 1, h, w, 16), h16(), x.device)
    assert c_nb16(x, full, n, h, w, w4, st) == 0
    return full


@pytest.mark.parametrize("h", [1, 2, 7, 8, 9, 15, 16, 17, 144])
@pytest.mark.parametrize("w", [16, 32, 128, 144, 240, 256])
def test_erf_nb16(cuda, w, h):
    """heights around the 8-row tile and its +-2 halo rows above and below the image; every width class; inputs (the
    residual) of both signs"""
    w4, st = (t.to(cuda) for t in nb_params(15))
    x = torch.randn(2, h, w, 16, generator=gen(16)).to(cuda).to(h16())
    full = run_nb16(x, w4, st)
    want, bound = util.erf_nb16_ref64(x, w4, st)
    hold(full, 2, want, bound, "erf_nb16")
    assert torch.equal(bits(ops.erf_nb16(x, w4, st)), bits(full[:2]))


@pytest.mark.parametrize("weight_scale", [0.03, 0.2], ids=["tight", "wide_weights"])
def test_erf_nb16_product(cuda, weight_scale):
    """the product's 96 x 144 x 128 x 16, run twice for bit equality; with the tight test weights, and with weights of
    sum |w| about 8 per stage, whose bound is looser but whose values span more of the h16 range"""
    w4, st = (t.to(cuda) for t in util.nb16_test_params(17, weight_scale))
    x = torch.randn(96, 144, 128, 16, generator=gen(18)).to(cuda).to(h16())
    full = run_nb16(x, w4, st)
    want, bound = util.erf_nb16_ref64(x, w4, st)
    hold(full, 96, want, bound, f"erf_nb16 w*{weight_scale}", product=True)
    assert torch.equal(bits(run_nb16(x, w4, st)), bits(full))


def test_erf_nb16_nan(cuda):
    """a NaN input reaches ReLUs only (fmaxf(NaN, 0) = 0): no output is NaN, and the rest matches the statement"""
    w4, st = (t.to(cuda) for t in nb_params(19))
    x = torch.randn(1, 12, 32, 16, generator=gen(20)).to(h16())
    x[0, 5, 7, :] = float("nan")
    x[0, 0, 0, 3] = float("nan")
    x = x.to(cuda)
    full = run_nb16(x, w4, st)
    want, bound = util.erf_nb16_ref64(x, w4, st)
    hold(full, 1, want, bound, "erf_nb16 nan")
    assert not bool(torch.isnan(full[:1].float()).any())


def erf_nb16_rejections(cuda, tmp_path):
    w4, st = (t.to(cuda) for t in nb_params(21))
    x = torch.randn(2, 9, 32, 16, generator=gen(22)).to(cuda).to(h16())
    wide = torch.zeros(1, 2, 272, 16, device=cuda, dtype=h16())
    out = canary((3, 9, 32, 16), h16(), cuda)
    flat = canary((2 * 9 * 32 * 16 + 8,), h16(), cuda)
    xs = torch.zeros(x.numel() + 8, dtype=h16(), device=cuda)
    st_flat = torch.zeros(st.numel() + 1, device=cuda)
    cases = [
        (lambda: c_nb16(wide, out, 1, 2, 272, w4, st), "width"),
        (lambda: c_nb16(x, out, 2, 9, 8, w4, st), "width"),
        (lambda: c_nb16(x, out, 2, 9, 24, w4, st), "width"),
        (lambda: c_nb16(x, out, 2, 0, 32, w4, st), "width"),
        (lambda: c_nb16(x, out, -1, 9, 32, w4, st), "width"),
        (lambda: c_nb16(x, out, 2 ** 30, 9, 32, w4, st), "2^31"),
        (lambda: c_nb16(None, out, 2, 9, 32, w4, st), "null"),
        (lambda: c_nb16(x, None, 2, 9, 32, w4, st), "null"),
        (lambda: c_nb16(x, out, 2, 9, 32, None, st), "null"),
        (lambda: c_nb16(x, out, 2, 9, 32, w4, None), "null"),
        (lambda: c_nb16(xs[4:], out, 2, 9, 32, w4, st), "aligned"),
        (lambda: c_nb16(x, flat[4:], 2, 9, 32, w4, st), "aligned"),
        (lambda: c_nb16(x, out, 2, 9, 32, w4, st_flat[1:]), "aligned"),                             # 4 bytes off 8
        (lambda: c_nb16(x, x, 2, 9, 32, w4, st), "overlap"),
        (lambda: c_nb16(x, x.view(-1)[32 * 16:], 2, 9, 32, w4, st), "overlap"),                     # one row down
        (lambda: c_nb16(x, out, 2, 9, 32, out, st), "overlaps d_w4"),
        (lambda: c_nb16(x, out, 2, 9, 32, w4, out.view(-1)[2 * 9 * 32 * 16 - 8:]), "overlaps d_w4 or d_st"),
    ]
    rejected(tmp_path, cases, [out, flat])
    assert c_nb16(x, out, 0, 9, 32, w4, st) == 0 and bool(is_canary(out).all())
    with pytest.raises(TypeError):
        ops.erf_nb16(x, w4, st, out=out)                   # the wrapper takes no caller output


# ------------------------------------------------------------------------------------------------------------ stem u8
def stem_u8_params(seed, device):
    g = gen(seed)
    w = torch.randn(64, 3, 7, 7, generator=g) * 0.08
    bias = torch.randn(64, generator=g) * 0.1
    return ops.pack_stem_weights(w.to(device)), bias.to(device)


def c_stem_u8(img, b, ncam, h, cw, wk, bias, out, mean=MEAN, std=STD):
    m = (C.c_float * 3)(*mean) if mean is not None else None
    sd = (C.c_float * 3)(*std) if std is not None else None
    return lib().lavb_stem7x7s2_u8(ops._ptr(img), b, ncam, h, cw, ops._ptr(wk), ops._ptr(bias), m, sd, ops._ptr(out),
                                   ops._stream())


def distinct_cameras(b, ncam, h, cw, seed):
    """random frames with each camera shifted to its own range, so a wrong camera index or seam shows"""
    img = torch.randint(0, 128, (b, ncam, h, cw, 3), generator=gen(seed), dtype=torch.int32)
    img = img + torch.arange(ncam, dtype=torch.int32)[None, :, None, None, None] * 40
    return img.clamp(0, 255).to(torch.uint8)


def run_stem_u8(img, wk, bias):
    b, ncam, h, cw, _ = img.shape
    full = canary((b + 1, (h - 1) // 2 + 1, (ncam * cw - 1) // 2 + 1, 64), h16(), img.device)
    assert c_stem_u8(img, b, ncam, h, cw, wk, bias, full) == 0
    return full


# (ncam, cam_w, h): every camera count at the narrow widths; heights around the 8-row block; logical widths of 252, 256,
# 260, 512 and 516 pixels put the output's last column at 126, 128, 130, 256 and 258 (cam_w % 4 == 0 makes the output
# width even, so 127, 129 and 257 columns cannot occur); the product's wide and telephoto images
STEM_U8 = ([(c, w, 9) for c in (1, 2, 3, 4) for w in (8, 12)] + [(c, w, 8) for c in (1, 2, 3, 4) for w in (256, 480)]
           + [(1, 256, h) for h in (7, 9, 192, 288)] + [(3, 84, 16), (4, 64, 17), (1, 260, 15), (2, 256, 10), (3, 172, 11)])


@pytest.mark.parametrize("case", STEM_U8, ids=lambda c: "x".join(map(str, c)))
def test_stem7x7s2_u8(cuda, case):
    ncam, cw, h = case
    wk, bias = stem_u8_params(23, cuda)
    img = distinct_cameras(2, ncam, h, cw, 24).to(cuda)
    full = run_stem_u8(img, wk, bias)
    want, bound = util.stem7x7s2_u8_ref64(img, wk, bias, MEAN, STD)
    hold(full, 2, want, bound, "stem7x7s2_u8")
    assert torch.equal(bits(ops.stem7x7s2_u8(img, wk, bias, MEAN, STD)), bits(full[:2]))


@pytest.mark.parametrize("shape", [(32, 3, 288, 256), (32, 1, 192, 480)], ids=["wide", "telephoto"])
def test_stem7x7s2_u8_product(cuda, shape):
    wk, bias = stem_u8_params(25, cuda)
    img = distinct_cameras(*shape, 26).to(cuda)
    full = run_stem_u8(img, wk, bias)
    want, bound = util.stem7x7s2_u8_ref64(img, wk, bias, MEAN, STD)
    hold(full, shape[0], want, bound, "stem7x7s2_u8", product=True)
    assert torch.equal(bits(run_stem_u8(img, wk, bias)), bits(full))


def stem7x7s2_u8_rejections(cuda, tmp_path):
    wk, bias = stem_u8_params(27, cuda)
    img = distinct_cameras(2, 3, 16, 12, 28).to(cuda)
    out = canary((3, 8, 18, 64), h16(), cuda)
    flat = canary((2 * 8 * 18 * 64 + 8,), h16(), cuda)
    raw = torch.zeros(img.numel() + 4, dtype=torch.uint8, device=cuda)
    wflat = torch.zeros(wk.numel() + 2, dtype=h16(), device=cuda)
    cases = [
        (lambda: c_stem_u8(img, 2, 5, 16, 12, wk, bias, out), "shape"),
        (lambda: c_stem_u8(img, 2, 0, 16, 12, wk, bias, out), "shape"),
        (lambda: c_stem_u8(img, 2, 3, 6, 12, wk, bias, out), "shape"),
        (lambda: c_stem_u8(img, 2, 3, 16, 4, wk, bias, out), "shape"),
        (lambda: c_stem_u8(img, -1, 3, 16, 12, wk, bias, out), "shape"),
        (lambda: c_stem_u8(img, 2, 3, 16, 10, wk, bias, out), "multiple of 4"),
        (lambda: c_stem_u8(img, 2 ** 30, 3, 17, 12, wk, bias, out), "grid"),
        (lambda: c_stem_u8(img, 2, 4, 16, 2 ** 22, wk, bias, out), "grid"),
        (lambda: c_stem_u8(None, 2, 3, 16, 12, wk, bias, out), "null"),
        (lambda: c_stem_u8(img, 2, 3, 16, 12, None, bias, out), "null"),
        (lambda: c_stem_u8(img, 2, 3, 16, 12, wk, None, out), "null"),
        (lambda: c_stem_u8(img, 2, 3, 16, 12, wk, bias, None), "null"),
        (lambda: c_stem_u8(img, 2, 3, 16, 12, wk, bias, out, mean=None), "null"),
        (lambda: c_stem_u8(img, 2, 3, 16, 12, wk, bias, out, std=None), "null"),
        (lambda: c_stem_u8(raw[1:], 2, 3, 16, 12, wk, bias, out), "aligned"),
        (lambda: c_stem_u8(img, 2, 3, 16, 12, wflat[1:], bias, out), "aligned"),
        (lambda: c_stem_u8(img, 2, 3, 16, 12, wk, bias, flat[4:]), "aligned"),
        (lambda: c_stem_u8(img, 2, 3, 16, 12, wk, bias, img), "overlap"),
        (lambda: c_stem_u8(img, 2, 3, 16, 12, out.view(-1)[64:], bias, out), "overlaps d_w"),
        (lambda: c_stem_u8(img, 2, 3, 16, 12, wk, out.view(-1)[2 * 8 * 18 * 64 - 8:], out), "overlaps d_w or d_bias"),
        (lambda: c_stem_u8(img, 2, 3, 16, 12, wk, bias, out, std=[0.229, 0.0, 0.225]), "non-finite"),
        (lambda: c_stem_u8(img, 2, 3, 16, 12, wk, bias, out, std=[0.229, float("nan"), 0.225]), "non-finite"),
        (lambda: c_stem_u8(img, 2, 3, 16, 12, wk, bias, out, mean=[float("inf"), 0.456, 0.406]), "non-finite"),
    ]
    rejected(tmp_path, cases, [out, flat])
    assert c_stem_u8(img, 0, 3, 16, 12, wk, bias, out) == 0 and bool(is_canary(out).all())
    with pytest.raises(capi.LavbError):
        ops.stem7x7s2_u8(img, wk, bias[:32], MEAN, STD)


# --------------------------------------------------------------------------------------------------------------- maxpool
def c_pool(x, n, h, w, c, out):
    return lib().lavb_maxpool3x3s2_nhwc(ops._ptr(x), n, h, w, c, ops._ptr(out), ops._stream())


def run_pool(x):
    n, h, w, c = x.shape
    full = canary((n + 1, (h - 1) // 2 + 1, (w - 1) // 2 + 1, c), h16(), x.device)
    assert c_pool(x, n, h, w, c, full) == 0
    return full


def hold_pool(full, x, what):
    """bit for bit the statement; a NaN is the canonical 0x7FFF, except on a 1 x 1 map, whose single-pixel windows pass
    their pixel through bit for bit"""
    n = x.shape[0]
    assert not bool(is_canary(full[:n]).any()), f"{what}: outputs never written"
    assert bool(is_canary(full[n:]).all()), f"{what}: written past the end"
    want = util.maxpool3x3s2_ref64(x)
    got = bits(full[:n])
    nan = torch.isnan(want)
    assert torch.equal(got[~nan], bits(want.to(h16()))[~nan]), what
    if x.shape[1] == x.shape[2] == 1:
        assert torch.equal(got, bits(x)), what
    else:
        assert bool((got[nan] == 0x7FFF).all()), what


POOL = [(h, w, 8 * (1 + (h * w) % 3)) for h in range(1, 6) for w in range(1, 6)] + \
       [(7, 9, c) for c in (8, 16, 64, 72, 384)] + [(13, 6, 24), (6, 13, 40)]


@pytest.mark.parametrize("case", POOL, ids=lambda c: "x".join(map(str, c)))
def test_maxpool3x3s2(cuda, case):
    h, w, c = case
    x = torch.randn(3, h, w, c, generator=gen(29)).to(h16()).to(cuda)
    full = run_pool(x)
    hold_pool(full, x, f"maxpool {case}")
    assert torch.equal(bits(ops.maxpool3x3s2_nhwc(x)), bits(full[:3]))


def test_maxpool3x3s2_product(cuda):
    x = torch.randn(32, 144, 384, 64, generator=gen(30)).to(h16()).to(cuda)
    full = run_pool(x)
    hold_pool(full, x, "maxpool product")
    assert torch.equal(bits(run_pool(x)), bits(full))


def test_maxpool3x3s2_special_values(cuda):
    """+-inf, +-0, +-65504 and NaN at chosen window positions: a NaN on a pixel four windows share and one on the map's
    corner, seen by one window; -0 with +0 gives +0; -0 alone stays -0"""
    x = torch.full((2, 5, 5, 16), -3.0)
    x[0, 1, 1, 0] = float("nan")                           # in windows (0..1, 0..1)
    x[0, 0, 0, 1] = float("nan")                           # in window (0, 0) only
    x[0, 4, 4, 2] = float("inf")
    x[0, :, :, 3] = -float("inf")                          # a channel of -inf only
    x[0, 2, 3, 4] = 65504
    x[0, :, :, 5] = -65504
    x[0, :, :, 6] = -0.0
    x[0, 3, 3, 6] = 0.0                                    # +0 in windows (1, 1), (1, 2), (2, 1), (2, 2)
    x[0, :, :, 7] = -0.0                                   # -0 only
    x[1] = torch.randn(5, 5, 16, generator=gen(31))
    x[1, 1, 2, 8] = float("nan")
    x = x.to(h16()).to(cuda)
    full = run_pool(x)
    hold_pool(full, x, "maxpool special")
    got = full[0].float().cpu()
    nan0 = torch.zeros(3, 3, dtype=torch.bool)
    nan0[:2, :2] = True
    assert torch.equal(torch.isnan(got[:, :, 0]), nan0)
    assert bool(torch.isnan(got[0, 0, 1])) and not bool(torch.isnan(got[0, 1, 1]))
    assert float(got[2, 2, 2]) == float("inf") and bool((got[:, :, 3] == -float("inf")).all())
    assert bool((got[:, :, 5] == -65504).all()) and float(got[1, 1, 4]) == 65504
    s6 = torch.signbit(got[:, :, 6])
    assert not bool(s6[1:, 1:].any()) and bool(s6[0, 0]) and bool(torch.signbit(got[:, :, 7]).all())


def test_maxpool3x3s2_nan_single_pixel(cuda):
    """a 1 x 1 map: each window is its one pixel, copied with its NaN payload and sign; a 1 x 2 map's window of two
    pixels gives the canonical NaN"""
    x = torch.randn(2, 1, 1, 16, generator=gen(42)).to(h16())
    xb = x.view(torch.int16)
    xb[0, 0, 0, :4] = torch.tensor([0x7E01, 0x7FFF, -512, -255], dtype=torch.int16)       # 0x7E01, 0x7FFF, 0xFE00, 0xFF01
    x = x.to(cuda)
    full = run_pool(x)
    hold_pool(full, x, "maxpool 1x1 nan")
    assert torch.equal(bits(full[:2]), bits(x))
    y = torch.cat([x, x], 2).contiguous()
    full = run_pool(y)
    hold_pool(full, y, "maxpool 1x2 nan")
    assert bool((bits(full[0, 0, 0, :4]) == 0x7FFF).all())


def maxpool3x3s2_rejections(cuda, tmp_path):
    x = torch.randn(2, 7, 9, 64, generator=gen(32)).to(h16()).to(cuda)
    out = canary((3, 4, 5, 64), h16(), cuda)
    flat = canary((2 * 4 * 5 * 64 + 8,), h16(), cuda)
    xs = torch.zeros(x.numel() + 8, dtype=h16(), device=cuda)
    cases = [
        (lambda: c_pool(x, 2, 7, 9, 60, out), "bad shape"),
        (lambda: c_pool(x, 2, 7, 9, 0, out), "bad shape"),
        (lambda: c_pool(x, 2, 0, 9, 64, out), "bad shape"),
        (lambda: c_pool(x, -1, 7, 9, 64, out), "bad shape"),
        (lambda: c_pool(x, 2 ** 30, 7, 9, 384, out), "2^31"),
        (lambda: c_pool(None, 2, 7, 9, 64, out), "null"),
        (lambda: c_pool(x, 2, 7, 9, 64, None), "null"),
        (lambda: c_pool(xs[4:], 2, 7, 9, 64, out), "aligned"),
        (lambda: c_pool(x, 2, 7, 9, 64, flat[4:]), "aligned"),
        (lambda: c_pool(x, 2, 7, 9, 64, x), "overlap"),
        (lambda: c_pool(x, 2, 7, 9, 64, x.view(-1)[7 * 9 * 64:]), "overlap"),
    ]
    rejected(tmp_path, cases, [out, flat])
    assert c_pool(x, 0, 7, 9, 64, out) == 0 and bool(is_canary(out).all())
    with pytest.raises(capi.LavbError):
        ops.maxpool3x3s2_nhwc(x[..., :60].contiguous())


# ---------------------------------------------------------------------------------------------------- batch independence
def test_batch_independence(cuda):
    """image i of a batch equals image i run alone, bit for bit, for all five kernels"""
    rgb = torch.randint(0, 256, (3, 18, 70, 3), generator=gen(33), dtype=torch.uint8).to(cuda)
    p = stem_params(34)
    for dt in (torch.float32, h16()):
        full = run_erf_stem(rgb, p, dt)
        for i in range(3):
            assert torch.equal(bits(run_erf_stem(rgb[i:i + 1].contiguous(), p, dt)[0]), bits(full[i]))
    x16 = torch.randn(3, 10, 34, 16, generator=gen(35)).to(cuda).to(h16())
    w9, st = (t.to(cuda) for t in down_params(36))
    w4, st4 = (t.to(cuda) for t in nb_params(37))
    x32 = torch.randn(3, 17, 32, 16, generator=gen(38)).to(cuda).to(h16())
    dn, nb = run_down16(x16, w9, st), run_nb16(x32, w4, st4)
    for i in range(3):
        assert torch.equal(bits(run_down16(x16[i:i + 1].contiguous(), w9, st)[0]), bits(dn[i]))
        assert torch.equal(bits(run_nb16(x32[i:i + 1].contiguous(), w4, st4)[0]), bits(nb[i]))
    img = distinct_cameras(3, 3, 17, 12, 39).to(cuda)
    wk, bias = stem_u8_params(40, cuda)
    su = run_stem_u8(img, wk, bias)
    xp = torch.randn(3, 9, 11, 24, generator=gen(41)).to(h16()).to(cuda)
    pl = run_pool(xp)
    for i in range(3):
        assert torch.equal(bits(run_stem_u8(img[i:i + 1].contiguous(), wk, bias)[0]), bits(su[i]))
        assert torch.equal(bits(run_pool(xp[i:i + 1].contiguous())[0]), bits(pl[i]))


# ------------------------------------------------------------------------------------------------------------ rejections
def rejections_main(tmp_path):
    cuda = torch.device("cuda:0")
    for check in (erf_stem_rejections, erf_down16_rejections, erf_nb16_rejections, stem7x7s2_u8_rejections,
                  maxpool3x3s2_rejections):
        check(cuda, tmp_path)


def test_rejections(cuda, tmp_path):
    """every rejection of the five entry points, in a child process: torch.profiler is started there, so that this process's
    profiler is first started where the rest of the suite expects it (a profiler started earlier in a long session can lose
    the kernel records of later captures)"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = (f"import sys; sys.path.insert(0, {root!r}); from tests import test_gpu_camera_kernels_contract as t; "
            f"t.rejections_main({str(tmp_path)!r})")
    r = subprocess.run([sys.executable, *(["-s"] if sys.flags.no_user_site else []), "-c", code], cwd=root,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
