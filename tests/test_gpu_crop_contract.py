"""GPU: the rotated crop (lavb_crop_bilinear, fp32 and h16) and its gather backward (lavb_crop_bilinear_bwd) against the
float64 reference of tests/util.py (crop_ref64 and its adjoint, pinned to a per-pixel loop by tests/test_crop_ref_cpu.py),
across the contract include/lav_b200.h states.

The crop is independent per channel, so the kernels run at full size and a channel subset is compared: channels 0-7, the
last 8 and a seeded few.  Every kernel output starts as NaN (the forward through the C ABI, the backward through ``out=``),
so an element the kernel fails to write shows.  Tolerances are per element, in units of the sums of the terms' magnitudes:
sum |w f| = crop_ref64(|f|) for the forward and sum |w g| = adjoint(|g|) for the backward.

Sample positions.  The kernel forms a sample position in fp32, the reference in fp64 from the same fp32 theta.  The fp32
position ix = (gx + 1) / 2 * (W - 1), gx = theta00 x + theta01 y + theta02 with |x|, |y| <= 1, takes about 6 roundings of
relative size 2^-24 on terms no larger than 1 + |theta0.|, so its error is below
    dx = 2^-21 (W - 1) / 2 (1 + |theta00| + |theta01| + |theta02|)   (8 units in the last place of the scale)
and likewise dy.  The bilinear interpolant of a map is Lipschitz in the position with, per axis, the largest difference of
neighbouring pixels around the sample (zeros off the map); sampling the 3 x 3 maximum of those differences with border
padding bounds it at every position, edges included.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from lav_b200 import capi, ops
from lav_b200.heads import crop_theta
from tests import util

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
NAN = float("nan")


# ------------------------------------------------------------------------------------------------------------- helpers
def nchw(x):
    return x.permute(0, 3, 1, 2)


def channels(c, seed=0):
    g = torch.Generator().manual_seed(seed)
    pick = set(range(min(8, c))) | set(range(max(0, c - 8), c)) | set(torch.randperm(c, generator=g)[:4].tolist())
    return torch.tensor(sorted(pick))


def cuda_gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def fwd(feats, fidx, theta, S):
    """lavb_crop_bilinear through the C ABI into an output filled with NaN; asserts that every element was written"""
    b, h, w, c = feats.shape
    k = theta.shape[0]
    fidx, theta = fidx.to(torch.int32).contiguous(), theta.float().contiguous()
    out = torch.full((k, S, S, c), NAN, dtype=feats.dtype, device=feats.device)
    capi.check(capi.lib().lavb_crop_bilinear(C.c_void_p(feats.data_ptr()), ops._DT[feats.dtype], b, h, w, c, C.c_void_p(fidx.data_ptr()),
                                             C.c_void_p(theta.data_ptr()), k, S, C.c_void_p(out.data_ptr()), ops._stream()),
               "lavb_crop_bilinear")
    assert not bool(out.isnan().any()), f"{int(out.isnan().sum())} crop elements not written"
    return out


def bwd(gout, fidx, theta, feat_shape):
    """ops.crop_bilinear_bwd into an ``out`` filled with NaN; asserts that every element was written"""
    out = torch.full(feat_shape, NAN, dtype=torch.float32, device=gout.device)
    got = ops.crop_bilinear_bwd(gout, fidx, theta, feat_shape, out=out)
    assert got.data_ptr() == out.data_ptr()
    assert not bool(out.isnan().any()), f"{int(out.isnan().sum())} gradient elements not written"
    return out


def pos_err(theta, H, W):
    """(dx, dy), each (K,1,1,1): bounds of the fp32 sample position's error in feature pixels (module docstring)"""
    t = theta.double().cpu().abs()
    dx = 2.0 ** -21 * (W - 1) / 2 * (1 + t[:, 0].sum(1))
    dy = 2.0 ** -21 * (H - 1) / 2 * (1 + t[:, 1].sum(1))
    return dx.view(-1, 1, 1, 1), dy.view(-1, 1, 1, 1)


def fwd_bound(fsub, fidx, theta, S, exact=False):
    """per-element bound of |kernel - crop_ref64| for an fp32 crop of fsub (B,c,H,W) float64.
    exact: every sample position and weight is exact in fp32, and four fmaf roundings, each at most 2^-24 of a partial sum
    no larger than sum |w f|, leave at most 2^-22 sum |w f|.  Otherwise the weights carry up to three more roundings (1 - ax
    for ix in (0, 1), the product) -> 2^-21 sum |w f|, plus the position errors times the interpolant's slopes."""
    mag = util.crop_ref64(fsub.abs(), fidx, theta, S)
    if exact:
        return 2.0 ** -22 * mag
    H, W = fsub.shape[-2:]
    fp = F.pad(fsub, (1, 1, 1, 1))
    lx = F.max_pool2d((fp[..., 1:] - fp[..., :-1]).abs(), 3, 1, 1)[..., 1:H + 1, :W]
    ly = F.max_pool2d((fp[..., 1:, :] - fp[..., :-1, :]).abs(), 3, 1, 1)[..., :H, 1:W + 1]
    dx, dy = pos_err(theta, H, W)
    return (dx * util.crop_ref64(lx, fidx, theta, S, "border") + dy * util.crop_ref64(ly, fidx, theta, S, "border")
            + 2.0 ** -21 * mag)


def bwd_bound(gsub, fidx, theta, feat_shape):
    """per-element bound of |kernel - adjoint| for the gradient of gsub (K,c,S,S) float64 on a (B,c,H,W) map.
    A feature pixel sums n terms w g in fp32 (one fmaf rounding each) with weights that carry up to three roundings:
    (n + 3) 2^-24 sum |w g|.  A position error moves each weight by at most dx + dy, also for a sample that crosses into a
    neighbouring cell (whose weight is then below dx + dy); the terms that can touch a pixel are those whose sample lies in
    the 4 x 4 pixels around it, so 2 (dx + dy) times the sum of their |g| bounds that part.  n is counted over the same 4 x 4."""
    B, c, H, W = feat_shape
    K, _, S, _ = gsub.shape
    grid = F.affine_grid(theta.double().cpu(), [K, c, S, S], align_corners=True)
    x0 = ((grid[..., 0] + 1) / 2 * (W - 1)).floor().clamp(-8, W + 8).long()
    y0 = ((grid[..., 1] + 1) / 2 * (H - 1)).floor().clamp(-8, H + 8).long()
    b = fidx.long().cpu().clamp(0, B - 1).view(K, 1, 1)
    vals = torch.cat([gsub.abs().permute(0, 2, 3, 1), torch.ones(K, S, S, 1, dtype=torch.float64)], -1).reshape(-1, c + 1)
    acc = torch.zeros(B * H * W, c + 1, dtype=torch.float64)
    for oy in range(-1, 3):
        for ox in range(-1, 3):
            x, y = x0 + ox, y0 + oy
            ok = ((x >= 0) & (x < W) & (y >= 0) & (y < H)).reshape(-1)
            acc.index_add_(0, ((b * H + y) * W + x).reshape(-1)[ok], vals[ok])
    acc = acc.view(B, H, W, c + 1).permute(0, 3, 1, 2)
    near, n = acc[:, :c], acc[:, c:]
    dx, dy = pos_err(theta, H, W)
    mag = util.crop_ref64_adjoint(gsub.abs(), fidx, theta, feat_shape)
    return (n + 3) * U * mag + 2 * float((dx + dy).max()) * near


def assert_within(got, want, bound, what):
    err = (got - want).abs()
    bad = err > bound
    assert not bool(bad.any()), (f"{what}: {int(bad.sum())} of {err.numel()} elements over the bound; worst excess "
                                 f"{float((err - bound).max()):.3e} (error {float(err[bad].max()):.3e})")


def dot64(a, b):
    """<a, b> in float64, a slab at a time"""
    return sum(float((a[i:i + 8].double() * b[i:i + 8].double()).sum()) for i in range(0, a.shape[0], 8))


def rot_theta(K, scale, seed, spread=0.3, dev=None):
    """K rotated crops: any heading, the given scale, centres within +-spread of the map's centre (normalised units)"""
    g = torch.Generator().manual_seed(seed)
    a = torch.rand(K, generator=g) * 2 * math.pi - math.pi
    t = (torch.rand(K, 2, generator=g) * 2 - 1) * spread
    c, s = torch.cos(a) * scale, torch.sin(a) * scale
    th = torch.stack([torch.stack([c, -s, t[:, 0]], -1), torch.stack([s, c, t[:, 1]], -1)], -2)
    return th if dev is None else th.to(dev)


def planner_theta(K, H, W, S, seed, dev, spread=12.0, off=True):
    """crop poses of the planners (heads.crop_theta, 2 px/m, y offset 0.75): any heading with +-20 deg of jitter; with ``off``
    the first four lie partly or fully off the map"""
    g = torch.Generator().manual_seed(seed)
    locs = torch.randn(K, 2, generator=g) * spread
    if off:
        locs[:4] += torch.tensor([[90.0, 0.0], [0.0, -85.0], [38.0, 38.0], [-42.0, 10.0]])[:K]
    oris = torch.rand(K, generator=g) * 2 * math.pi - math.pi + (torch.rand(K, generator=g) * 2 - 1) * math.radians(20)
    return crop_theta(locs, oris, H, W, 2.0, S, torch.tensor(0.0), torch.tensor(0.75)).to(dev)


def check_fwd(got, feats, fidx, theta, S, exact=False, seed=0):
    ch = channels(feats.shape[-1], seed)
    fsub = nchw(feats[..., ch.to(feats.device)]).double().cpu()
    want = util.crop_ref64(fsub, fidx, theta, S)
    assert_within(nchw(got[..., ch.to(got.device)]).double().cpu(), want, fwd_bound(fsub, fidx, theta, S, exact), "forward")


def run_case(B, H, W, C, S, fidx, theta, seed):
    """forward and backward of one case against the fp64 reference, plus the adjoint identity <fwd(f), g> = <f, bwd(g)> on
    the kernels' own outputs.  g = fwd(f) + noise keeps <fwd(f), g> of the order of |fwd(f)|^2, clear of cancellation.
    -> the kernel's gradient."""
    dev = theta.device
    f = torch.randn(B, H, W, C, device=dev, generator=cuda_gen(seed))
    out = fwd(f, fidx, theta, S)
    check_fwd(out, f, fidx, theta, S, seed=seed)
    g = out + torch.randn(out.shape, device=dev, generator=cuda_gen(seed + 1))
    gfeat = bwd(g, fidx, theta, (B, H, W, C))
    ch = channels(C, seed)
    gsub = nchw(g[..., ch.to(dev)]).double().cpu()
    want = util.crop_ref64_adjoint(gsub, fidx, theta, (B, len(ch), H, W))
    assert_within(nchw(gfeat[..., ch.to(dev)]).double().cpu(), want, bwd_bound(gsub, fidx, theta, (B, len(ch), H, W)), "backward")
    lhs, rhs = dot64(out, g), dot64(f, gfeat)
    assert abs(lhs - rhs) <= 1e-6 * abs(lhs), (lhs, rhs)
    return gfeat


# ------------------------------------------------------------------------------------------------------------- forward, fp32
def test_sample_positions_are_torch_linspace_bit_for_bit(cuda):
    """A 1 x 2 map holding 0 and 1 makes the crop output its own sample position: out = ax = ix.  With the identity theta
    the position is (x + 1) / 2 for x = torch.linspace(-1, 1, S) in fp32: start + step i for the first S // 2 points and
    end - step (S - 1 - i) after, each one fused multiply-add.  Pinned bit for bit (emulated exactly in float64) for both
    axes, at even and odd S."""
    feats = torch.zeros(1, 1, 2, 4, device=cuda)
    feats[0, 0, 1] = 1.0
    theta = torch.tensor([[[1.0, 0.0, 0.0], [0.0, 1.0, 0.0]], [[0.0, 1.0, 0.0], [1.0, 0.0, 0.0]]], device=cuda)
    for S in (2, 3, 95, 96, 97, 160, 255):
        step = np.float32(2) / np.float32(S - 1)
        i = np.arange(S, dtype=np.float64)
        lo = (i * np.float64(step) - 1.0).astype(np.float32)                  # exact in float64, one rounding: fmaf
        hi = (1.0 - (S - 1 - i) * np.float64(step)).astype(np.float32)
        x = np.where(np.arange(S) < S // 2, lo, hi)
        want = torch.from_numpy((x + np.float32(1)) * np.float32(0.5))
        got = fwd(feats, torch.zeros(2, dtype=torch.int32, device=cuda), theta, S).cpu()
        for ch in range(4):
            assert torch.equal(got[0, :, :, ch], want[None, :].expand(S, S)), S
            assert torch.equal(got[1, :, :, ch], want[:, None].expand(S, S)), S


def test_forward_exact_positions(cuda):
    """dyadic theta, S - 1, H - 1 and W - 1 powers of two: every sample position and weight is exact in fp32, so the only
    error is the four fmaf roundings (<= 2^-22 sum |w f|); an identity crop of a square map (S = H = W) is a bit-exact copy"""
    B, C, H, W, S = 2, 24, 17, 33, 17
    theta = torch.tensor([[[0.5, -0.25, 0.125], [0.25, 0.75, -0.375]], [[1.0, 0.0, 0.0], [0.0, 1.0, 0.0]],
                          [[-0.75, 0.5, 0.25], [0.5, 0.5, 0.5]], [[1.25, 0.0, -0.5], [0.0, -1.5, 0.25]],
                          [[0.0, 1.0, 0.0], [-1.0, 0.0, 0.0]], [[0.0625, 0.0, 0.96875], [0.0, 0.0625, -0.96875]]], device=cuda)
    fidx = torch.tensor([0, 1, 1, 0, 1, 0], dtype=torch.int32, device=cuda)
    feats = torch.randn(B, H, W, C, device=cuda, generator=cuda_gen(11))
    check_fwd(fwd(feats, fidx, theta, S), feats, fidx, theta, S, exact=True)
    sq = torch.randn(2, 33, 33, 40, device=cuda, generator=cuda_gen(12))
    eye = torch.tensor([[[1.0, 0.0, 0.0], [0.0, 1.0, 0.0]]] * 2, device=cuda)
    assert torch.equal(fwd(sq, torch.tensor([1, 0], dtype=torch.int32, device=cuda), eye, 33), sq[[1, 0]])


@pytest.mark.parametrize("size", ["inference", "training"])
def test_forward_planner_poses_full_size(cuda, size):
    """32 frames x 384 channels x 160 x 160, 96 x 96 crops at the planners' poses.  inference: 128 detected vehicles over the
    frames and one ego crop per frame in one call; training: 4 crops per frame, then the 32 jittered ego crops in a second call."""
    B, C, H, W, S = 32, 384, 160, 160, 96
    feats = torch.randn(B, H, W, C, device=cuda, generator=cuda_gen(21))
    if size == "inference":
        g = torch.Generator().manual_seed(22)
        fidx = torch.cat([torch.randint(0, B, (128,), generator=g), torch.arange(B)]).to(torch.int32).to(cuda)
        calls = [(fidx, planner_theta(160, H, W, S, 23, cuda))]
    else:
        g = torch.Generator().manual_seed(24)
        ego_locs = torch.cat([(torch.rand(B, 1, generator=g) * 2 - 1), torch.zeros(B, 1)], 1)      # lateral jitter, metres
        ego_oris = (torch.rand(B, generator=g) * 2 - 1) * math.radians(10)
        calls = [(torch.arange(B, dtype=torch.int32, device=cuda).repeat_interleave(4), planner_theta(128, H, W, S, 25, cuda)),
                 (torch.arange(B, dtype=torch.int32, device=cuda),
                  crop_theta(ego_locs, ego_oris, H, W, 2.0, S, torch.tensor(0.0), torch.tensor(0.75)).to(cuda))]
    for n, (fidx, theta) in enumerate(calls):
        check_fwd(fwd(feats, fidx, theta, S), feats, fidx, theta, S, seed=n)


@pytest.mark.parametrize("shape", [
    # (B, H, W, C, S)
    (3, 40, 48, 4, 24), (3, 40, 48, 8, 24), (3, 40, 48, 24, 24), (3, 40, 48, 40, 24), (3, 40, 48, 384, 24),
    (2, 40, 56, 8, 2), (2, 40, 56, 8, 3), (2, 40, 56, 8, 95), (2, 56, 40, 8, 96),
    (1, 40, 48, 16, 24), (1, 1, 37, 8, 24), (2, 29, 1, 8, 24), (1, 1, 1, 8, 5)])
def test_forward_shape_edges(cuda, shape):
    """channel counts with a half-used channel slice (C = 8 mod 16) and single 16-byte vectors, crops of 2, 3, 95 and 96,
    H != W, one frame, maps one pixel wide or high"""
    B, H, W, C, S = shape
    K = 9
    feats = torch.randn(B, H, W, C, device=cuda, generator=cuda_gen(31 + C + S))
    fidx = (torch.arange(K, device=cuda) % B).to(torch.int32)
    for theta in (planner_theta(K, H, W, S, 32, cuda, spread=6.0), rot_theta(K, 0.7, 33, dev=cuda)):
        check_fwd(fwd(feats, fidx, theta, S), feats, fidx, theta, S)


# ------------------------------------------------------------------------------------------------------------- forward, h16
def test_forward_h16_product_shape(cuda):
    """the 16-bit crop at the product's size is the fp32 crop of the same (h16-valued) map rounded once to nearest, bit for
    bit: both instantiations read the taps in the same fmaf order.  Against the fp64 reference on the h16-rounded map: the
    fp32 bound plus 2^-11 |ref| for the final rounding (2^-25 absolute below the normal range)."""
    h16 = ops.h16()
    B, C, H, W, S, K = 32, 384, 160, 160, 96, 160
    x16 = torch.randn(B, H, W, C, device=cuda, generator=cuda_gen(41)).to(h16)
    g = torch.Generator().manual_seed(42)
    fidx = torch.cat([torch.randint(0, B, (K - B,), generator=g), torch.arange(B)]).to(torch.int32).to(cuda)
    theta = planner_theta(K, H, W, S, 43, cuda)
    got16 = fwd(x16, fidx, theta, S)
    got32 = fwd(x16.float(), fidx, theta, S)
    assert torch.equal(got16, got32.to(h16))
    del got32
    ch = channels(C, 1)
    fsub = nchw(x16[..., ch.to(cuda)]).double().cpu()
    want = util.crop_ref64(fsub, fidx, theta, S)
    bound = 2.0 ** -11 * want.abs() + 2.0 ** -25 + (1 + 2.0 ** -11) * fwd_bound(fsub, fidx, theta, S)
    assert_within(nchw(got16[..., ch.to(cuda)]).double().cpu(), want, bound, "h16 forward")


# ------------------------------------------------------------------------------------------------------------- contract
@pytest.mark.parametrize("dtype", ["fp32", "h16"])
def test_frame_indices_are_clamped(cuda, dtype):
    dt = torch.float32 if dtype == "fp32" else ops.h16()
    feats = torch.randn(3, 20, 24, 16, device=cuda, generator=cuda_gen(51)).to(dt)
    theta = rot_theta(6, 0.8, 52, dev=cuda)
    raw = torch.tensor([-5, -1, 0, 2, 3, 1000], dtype=torch.int32, device=cuda)
    clamped = torch.tensor([0, 0, 0, 2, 2, 2], dtype=torch.int32, device=cuda)
    assert torch.equal(fwd(feats, raw, theta, 12), fwd(feats, clamped, theta, 12))
    if dtype == "fp32":
        g = torch.randn(6, 12, 12, 16, device=cuda, generator=cuda_gen(53))
        assert torch.equal(bwd(g, raw, theta, (3, 20, 24, 16)), bwd(g, clamped, theta, (3, 20, 24, 16)))


def test_zero_crops(cuda):
    """k = 0: the forward launches nothing and writes nothing; the backward writes a zero gradient everywhere"""
    feats = torch.randn(2, 8, 8, 8, device=cuda)
    out = torch.full((1, 4, 4, 8), NAN, device=cuda)
    none_i, none_t = torch.zeros(0, dtype=torch.int32, device=cuda), torch.zeros(0, 2, 3, device=cuda)
    capi.check(capi.lib().lavb_crop_bilinear(C.c_void_p(feats.data_ptr()), capi.F32, 2, 8, 8, 8, C.c_void_p(none_i.data_ptr()),
                                             C.c_void_p(none_t.data_ptr()), 0, 4, C.c_void_p(out.data_ptr()), ops._stream()),
               "lavb_crop_bilinear")
    torch.cuda.synchronize()
    assert bool(out.isnan().all())
    assert ops.crop_bilinear(feats, none_i, none_t, 4).shape == (0, 4, 4, 8)
    g = bwd(torch.zeros(0, 4, 4, 8, device=cuda), none_i, none_t, (2, 8, 8, 8))
    assert torch.equal(g, torch.zeros_like(g))


# ------------------------------------------------------------------------------------------------------------- backward
def test_backward_training_size(cuda):
    """32 frames x 384 channels x 160 x 160, 160 crops of 96 x 96: frame 0 holds 40 crops (two passes of the 32-crop list,
    four of them through clamped indices -3), frames 25-30 none (their gradient must be exactly 0), frame 31 is reached
    through clamped indices 99 as well as 31"""
    B, C, H, W, S = 32, 384, 160, 160, 96
    fidx = torch.tensor([0] * 36 + [-3] * 4 + [b for b in range(1, 25) for _ in range(4)] + [31] * 12 + [99] * 12, dtype=torch.int32)
    assert fidx.numel() == 160
    theta = planner_theta(160, H, W, S, 61, cuda, spread=10.0)
    gfeat = run_case(B, H, W, C, S, fidx.to(cuda), theta, 62)
    assert torch.equal(gfeat[25:31], torch.zeros_like(gfeat[25:31]))
    assert bool((gfeat[0] != 0).any()) and bool((gfeat[31] != 0).any())


@pytest.mark.parametrize("C", [4, 8, 380, 384, 388, 772])
def test_backward_channel_passes(cuda, C):
    """one, two and three passes of 96 float4 over the channels, the last one partly used"""
    B, H, W, S, K = 3, 40, 48, 24, 12
    fidx = (torch.arange(K, device=cuda) % B).to(torch.int32)
    run_case(B, H, W, C, S, fidx, planner_theta(K, H, W, S, 70 + C, cuda, spread=8.0), 71 + C)


@pytest.mark.parametrize("kind", ["upsample", "downsample2", "downsample3"])
def test_backward_candidate_batches(cuda, kind):
    """upsampling crops (scale 0.05, S = 96): one feature pixel gathers from hundreds of crop pixels, in batches of 32;
    downsampling crops (S = 2 or 3 spanning the map): a few widely spaced candidates"""
    B, H, W, C = 2, 24, 20, 8
    if kind == "upsample":
        S, theta = 96, rot_theta(6, 0.05, 81, spread=0.8, dev=cuda)
    else:
        S, theta = int(kind[-1]), rot_theta(6, 1.0, 82, spread=0.1, dev=cuda)
    run_case(B, H, W, C, S, torch.tensor([0, 1, 1, 0, 1, 0], dtype=torch.int32, device=cuda), theta, 83)


@pytest.mark.parametrize("kind", ["one_wide", "one_high", "rank1_theta"])
def test_backward_singular_maps(cuda, kind):
    """a map one pixel wide or high, or a rank-deficient theta, has no inverse sample position: every crop pixel is a candidate"""
    C, S = 8, 12
    if kind == "rank1_theta":
        B, H, W = 2, 40, 48
        theta = torch.tensor([[[0.5, 0.5, 0.1], [0.25, 0.25, -0.1]], [[0.6, -0.3, 0.0], [-0.4, 0.2, 0.05]],
                              [[0.7, 0.0, 0.2], [0.0, 0.0, 0.3]]], device=cuda)
    else:
        B, H, W = (2, 29, 1) if kind == "one_wide" else (2, 1, 37)
        theta = rot_theta(3, 0.6, 91, spread=0.2, dev=cuda)
    run_case(B, H, W, C, S, torch.tensor([0, 1, 0], dtype=torch.int32, device=cuda), theta, 92)


# ------------------------------------------------------------------------------------------------------------- arguments
def test_ops_reject_bad_arguments_before_launch(cuda):
    f = torch.randn(2, 10, 12, 8, device=cuda)
    fi = torch.tensor([0, 1, 1], dtype=torch.int32, device=cuda)
    th = rot_theta(3, 0.8, 101, dev=cuda)
    g = torch.randn(3, 6, 6, 8, device=cuda)
    misaligned = torch.randn(f.numel() + 4, device=cuda)[1:1 + f.numel()].view(f.shape)       # contiguous, 4 bytes off
    n0 = ops.launches()
    bad_fwd = [
        (f, fi[:2], th), (f, torch.cat([fi, fi]), th), (f, fi.view(3, 1), th), (f, fi.float(), th),   # frame_idx
        (f, fi, th.view(3, 6)), (f, fi, th[:, :, :2].contiguous()), (f, fi, th[:2]),                  # theta
        (f.permute(0, 2, 1, 3), fi, th), (f.double(), fi, th), (f[..., :6].contiguous(), fi, th),     # map
        (f.to(ops.h16())[..., :4].contiguous(), fi, th), (misaligned, fi, th), (f[0], fi, th),
    ]
    for args in bad_fwd:
        with pytest.raises(capi.LavbError):
            ops.crop_bilinear(*args, 6)
    shape = (2, 10, 12, 8)
    bad_bwd = [
        (g, fi[:2], th, shape), (g, fi, th[:2], shape), (g, fi, th.view(3, 6), shape),              # poses
        (g[..., :4].contiguous(), fi, th, shape), (g, fi, th, (2, 10, 12, 4)), (g, fi, th, (2, 10, 12)),  # channels / shape
        (g[:, :, :5].contiguous(), fi, th, shape), (g.transpose(1, 2), fi, th, shape), (g.double(), fi, th, shape),
    ]
    for args in bad_bwd:
        with pytest.raises(capi.LavbError):
            ops.crop_bilinear_bwd(*args)
    for out in (torch.empty(2, 10, 12, 4, device=cuda), torch.empty(2, 10, 12, 8, device=cuda).double(),
                torch.empty(2, 12, 10, 8, device=cuda).transpose(1, 2)):
        with pytest.raises(capi.LavbError):
            ops.crop_bilinear_bwd(g, fi, th, shape, out=out)
    assert ops.launches() == n0


def test_int64_frame_indices_match_int32(cuda):
    f = torch.randn(3, 16, 20, 12, device=cuda, generator=cuda_gen(111))
    th = rot_theta(5, 0.7, 112, dev=cuda)
    i64 = torch.tensor([2, -(2 ** 33), 1, 2 ** 33, 2 ** 32], dtype=torch.int64, device=cuda)
    i32 = torch.tensor([2, 0, 1, 2, 2], dtype=torch.int32, device=cuda)
    assert torch.equal(ops.crop_bilinear(f, i64, th, 10), ops.crop_bilinear(f, i32, th, 10))
    g = torch.randn(5, 10, 10, 12, device=cuda, generator=cuda_gen(113))
    assert torch.equal(ops.crop_bilinear_bwd(g, i64, th, f.shape), ops.crop_bilinear_bwd(g, i32, th, f.shape))
    x = f.requires_grad_(True)
    ops.CropBilinear.apply(x, i64, th, 10).backward(g)
    assert torch.equal(x.grad, ops.crop_bilinear_bwd(g, i32, th, f.shape))


def test_uniplanner_crop_feature_12_channels(cuda):
    """C = 12 (fp32, a multiple of 4 but not of 8) goes through the crop kernel in both grad modes and matches grid_sample"""
    import lav_b200.heads as Hd
    from tests.test_heads_cpu import uniplanner
    up = uniplanner()[0].to(cuda)
    g = torch.Generator().manual_seed(121)
    feats = torch.randn(2, 12, 40, 48, generator=g).to(cuda).contiguous(memory_format=torch.channels_last)
    locs, oris = (torch.randn(5, 2, generator=g) * 3).to(cuda), (torch.rand(5, generator=g) - 0.5).to(cuda)
    fr = torch.tensor([0, 1, 1, 0, 1], device=cuda)
    theta = crop_theta(locs, oris, 40, 48, 2, 24, up.offset_x, up.offset_y)
    want = F.grid_sample(feats[fr], F.affine_grid(theta, [5, 12, 24, 24], align_corners=True), align_corners=True)
    n0 = ops.launches()
    with torch.no_grad():
        got = up.crop_feature(feats, locs, oris, pixels_per_meter=2, crop_size=24, frame_idx=fr)
    assert ops.launches() == n0 + 1
    assert util.rel_err(got, want) < 1e-5
    grads = []
    for flag in (True, False):
        Hd.TRAIN_CROP_KERNEL = flag
        try:
            x = feats.detach().clone().requires_grad_(True)
            n0 = ops.launches()
            o = up.crop_feature(x, locs, oris, pixels_per_meter=2, crop_size=24, frame_idx=fr)
            o.square().sum().backward()
            assert ops.launches() == n0 + (2 if flag else 0)
            assert util.rel_err(o.detach(), want) < 1e-5
            grads.append(x.grad)
        finally:
            Hd.TRAIN_CROP_KERNEL = True
    assert util.rel_err(grads[0], grads[1]) < 1e-5
