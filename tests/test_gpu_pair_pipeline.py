"""GPU: lavb_conv_pair_umma's tile pipeline: the residual tile arrives by TMA into the tile's output ring slot, epilogue 2
writes the result over it and one TMA store per 64 channels writes it out, clipping rows past the image.

Compared with the fp64 restatement of the pair (tests/test_gpu_h16_range.py: pair_ref) at its 1e-2 tolerance.  The output
lies inside a canary-filled buffer: no byte outside the tensor may change.  The cases cover tile counts around the grid size
(C = 128: one CTA per SM; C = 64: two), a partial last tile, a dilation of at least the tile height, both flags and a saturating
residual sum.
"""
import pytest
import torch

from lav_b200 import capi, ops
from tests.test_gpu_h16_range import H, pair_ref, q

pytestmark = pytest.mark.gpu

CANARY = 0x5A5A                  # an h16 bit pattern no output of these cases takes
PAD = 4096                       # canary elements on each side of the output


def ctas(c):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return 2 * sms if c == 64 else sms


def run_pair(n, h, w, c, dil, res, relu, seed, overflow=False):
    g = torch.Generator().manual_seed(seed)
    x = q(torch.randn(n, h, w, c, generator=g)).cuda()
    w1 = q(torch.randn(c, c, 3, generator=g) / (3 * c) ** 0.5).cuda()
    w2 = q(torch.randn(c, c, 3, generator=g) / (3 * c) ** 0.5).cuda()
    b1, t2 = (torch.randn(c, generator=g) * 0.1).cuda(), (torch.randn(c, generator=g) * 0.1).cuda()
    r = None
    if overflow:                 # conv + shift within +-0.7 * 65504, residual of 40000..65504 of either sign
        k2 = 0.7 * H / float(pair_ref(x, w1, b1, w2, t2, dil, None, False)[2].abs().max())
        w2, t2 = q(w2 * k2), t2 * k2
        r = torch.rand(n, h, w, c, generator=g) * (H - 40000) + 40000
        r = q(torch.where(torch.rand(n, h, w, c, generator=g) < 0.5, -r, r)).cuda()
    elif res:
        r = q(torch.randn(n, h, w, c, generator=g)).cuda()
    want, raw, _ = pair_ref(x, w1, b1, w2, t2, dil, r, relu)
    buf = torch.full((n * h * w * c + 2 * PAD,), CANARY, dtype=torch.int16, device="cuda")
    out = buf[PAD:PAD + n * h * w * c].view(torch.float16).view(n, h, w, c)
    ops.conv_pair_umma(x.half(), w1.permute(2, 0, 1).half().contiguous(), b1.float(), w2.permute(2, 0, 1).half().contiguous(),
                       t2.float(), dil, res=None if r is None else r.half(), post_relu=relu, out=out)
    torch.cuda.synchronize()
    assert bool((buf[:PAD] == CANARY).all()) and bool((buf[-PAD:] == CANARY).all()), "bytes outside the output were written"
    got = out.double()
    assert bool(torch.isfinite(got).all())
    return got, want, raw


def check(got, want, raw):
    over = raw.abs() > H * (1 + 1e-3)
    assert torch.equal(got[over], torch.sign(raw[over]) * H)
    rest = ~over
    err = float((got[rest] - want[rest]).abs().max() / want[rest].abs().max())
    assert err < 1e-2, err


def tiles_case(c, w, count):
    """(n, h) with exactly `count` tiles of 128 // w rows each"""
    th = 128 // w
    for n in range(1, count + 1):
        if count % n == 0 and (count // n) * th * w * c * n <= 16 << 20:
            return n, count // n * th
    raise AssertionError(count)


@pytest.mark.parametrize("c", [64, 128])
@pytest.mark.parametrize("which", ["fewer", "grid", "grid+1", "2 per CTA", "3 per CTA"])
def test_pair_tile_counts(cuda, c, which):
    """tile counts around the grid size: the persistent loop's first and last tiles, and CTAs with 1, 2 and 3 tiles"""
    k = ctas(c)
    count = {"fewer": k // 3, "grid": k, "grid+1": k + 1, "2 per CTA": 2 * k, "3 per CTA": 3 * k}[which]
    w = 128 if which == "grid+1" else 64
    n, h = tiles_case(c, w, count)
    check(*run_pair(n, h, w, c, 1, True, True, seed=count + c))


@pytest.mark.parametrize("c,h,w", [(128, 35, 32), (64, 71, 64), (64, 37, 32), (128, 3, 128)])
@pytest.mark.parametrize("res", [False, True])
def test_pair_partial_last_tile(cuda, c, h, w, res):
    """h not a multiple of the tile height: the store clips the rows past the image, the residual load zero-fills them"""
    check(*run_pair(3, h, w, c, 2, res, True, seed=h + w))


@pytest.mark.parametrize("dil", [4, 8, 16])
def test_pair_dilation_past_tile_height(cuda, dil):
    """dilation >= tile height at h = 36 (128 channels, 4-row tiles), as in the encoder's dilated blocks"""
    check(*run_pair(2, 36, 32, 128, dil, True, True, seed=dil))


@pytest.mark.parametrize("w", [32, 64, 128])
@pytest.mark.parametrize("c", [64, 128])
@pytest.mark.parametrize("res,relu", [(False, False), (False, True), (True, False), (True, True)])
def test_pair_one_image_flags(cuda, w, c, res, relu):
    """n = 1 at every supported width, with and without the residual and the final ReLU"""
    check(*run_pair(1, 9, w, c, 1, res, relu, seed=w + c))


@pytest.mark.parametrize("c", [64, 128])
@pytest.mark.parametrize("relu", [False, True])
def test_pair_residual_sum_saturates(cuda, c, relu):
    """the residual sum leaves the h16 range: the output saturates at +-65504 (on a partial last tile)"""
    got, want, raw = run_pair(2, 35, 32, c, 1, True, relu, seed=c, overflow=True)
    assert int((raw.abs() > H * (1 + 1e-3)).sum()) >= 0.05 * raw.numel()
    check(got, want, raw)


@pytest.mark.parametrize("alias", ["in", "res", "overlap"])
def test_pair_rejects_aliased_output(cuda, alias):
    """out overlapping in or res is rejected before anything is launched"""
    n, h, w, c = 2, 8, 64, 64
    buf = torch.randn(2 * n * h * w * c, device="cuda").half()
    x, r = buf[:n * h * w * c].view(n, h, w, c), buf[n * h * w * c:].view(n, h, w, c)
    out = {"in": x, "res": r, "overlap": buf[n * h * w * c // 2:n * h * w * c * 3 // 2].view(n, h, w, c)}[alias]
    before = buf.clone()
    w1 = torch.randn(3, c, c, device="cuda").half()
    b = torch.zeros(c, device="cuda")
    with pytest.raises(capi.LavbError, match="must not overlap"):
        ops.conv_pair_umma(x, w1, b, w1, b, 1, res=r, out=out)
    torch.cuda.synchronize()
    assert torch.equal(buf, before)
