"""The float64 reference of the rotated crop (tests/util.py: crop_ref64 and its adjoint) against a plain per-pixel loop.

The loop restates what the crop kernels compute, independently of torch: the sample of crop pixel (i, j) is
theta @ (x_i, y_j, 1) with x_i = -1 + 2 i / (S - 1) (affine_grid, align_corners=True), un-normalised to feature pixels
by (g + 1) / 2 * (W - 1); the four taps around it get the bilinear weights, and a tap off the map contributes nothing
(zero padding).  These cases pin align_corners and the zero padding at the places a sampler goes wrong: maps one pixel
wide or high, samples exactly on the last row or column, samples in (-1, 0) and (W - 1, W), crops entirely off the map,
and out-of-range frame indices.
"""
import math

import pytest
import torch

from tests import util


def loop_crop(feats, frame_idx, theta, S):
    """-> (out, abs_sum): the crop and the per-element sum |w f| of its terms, (K,C,S,S) float64, one pixel at a time"""
    B, C, H, W = feats.shape
    K = theta.shape[0]
    out = torch.zeros(K, C, S, S, dtype=torch.float64)
    mag = torch.zeros_like(out)
    f = feats.double()
    for k in range(K):
        b = min(max(int(frame_idx[k]), 0), B - 1)
        t = theta[k].double().tolist()
        for j in range(S):
            for i in range(S):
                for tap, w in _taps(t, i, j, S, H, W):
                    out[k, :, j, i] += w * f[b, :, tap[1], tap[0]]
                    mag[k, :, j, i] += w * f[b, :, tap[1], tap[0]].abs()
    return out, mag


def loop_adjoint(gout, frame_idx, theta, feat_shape):
    """the transpose of loop_crop: each crop pixel's gradient scattered to the taps it read, with the same weights"""
    B, C, H, W = feat_shape
    S = gout.shape[-1]
    g = torch.zeros(feat_shape, dtype=torch.float64)
    for k in range(theta.shape[0]):
        b = min(max(int(frame_idx[k]), 0), B - 1)
        t = theta[k].double().tolist()
        for j in range(S):
            for i in range(S):
                for tap, w in _taps(t, i, j, S, H, W):
                    g[b, :, tap[1], tap[0]] += w * gout[k, :, j, i].double()
    return g


def _taps(t, i, j, S, H, W):
    xb, yb = -1 + 2 * i / (S - 1), -1 + 2 * j / (S - 1)
    ix = (t[0][0] * xb + t[0][1] * yb + t[0][2] + 1) / 2 * (W - 1)
    iy = (t[1][0] * xb + t[1][1] * yb + t[1][2] + 1) / 2 * (H - 1)
    x0, y0 = math.floor(ix), math.floor(iy)
    ax, ay = ix - x0, iy - y0
    for dx, dy, w in ((0, 0, (1 - ax) * (1 - ay)), (1, 0, ax * (1 - ay)), (0, 1, (1 - ax) * ay), (1, 1, ax * ay)):
        x, y = x0 + dx, y0 + dy
        if 0 <= x < W and 0 <= y < H and w != 0:
            yield (x, y), w


def _rot(angle, scale, tx, ty):
    c, s = math.cos(angle) * scale, math.sin(angle) * scale
    return [[c, -s, tx], [s, c, ty]]


# (H, W, S, thetas): every theta row is (a00, a01, a02, a10, a11, a12) of one crop
CASES = {
    "1x1": (1, 1, 3, [_rot(0.3, 0.8, 0.1, -0.2), _rot(0, 1, 0, 0)]),
    "1x5": (1, 5, 2, [_rot(0.0, 1.0, 0.0, 0.0), _rot(1.1, 0.7, 0.3, 0.0), _rot(0, 0.5, 0.25, 0.9)]),
    "5x1": (5, 1, 3, [_rot(0.0, 1.0, 0.0, 0.0), _rot(-0.6, 1.3, 0.0, 0.4)]),
    # S = H = W, identity: samples exactly on every pixel, the last row and column included (zero weight on the taps past them)
    "identity": (4, 6, 3, [_rot(0, 1, 0, 0)]),
    "last_row_col": (5, 5, 3, [[[1.0, 0.0, 0.0], [0.0, 0.5, 0.5]], [[0.5, 0.0, 0.5], [0.0, 1.0, 0.0]]]),
    # samples in (-1, 0) and (W-1, W): shifted by a third of a pixel past either edge
    "past_edges": (4, 7, 3, [[[1.0, 0.0, -1.0 / 9], [0.0, 1.0, 1.0 / 9]], [[1.0, 0.0, 1.0 / 9], [0.0, 1.0, -1.0 / 9]],
                             [[1.1, 0.0, 0.0], [0.0, 1.2, 0.0]]]),
    "off_map": (4, 5, 3, [_rot(0.4, 0.5, 3.5, 0.0), _rot(0, 0.5, 0.0, -3.2), _rot(2.0, 0.3, -5.0, 5.0)]),
    "rotated": (6, 7, 3, [_rot(0.7, 0.6, 0.1, -0.3), _rot(-2.5, 0.9, -0.4, 0.2), _rot(3.1, 1.4, 0.0, 0.0)]),
}


@pytest.mark.parametrize("case", list(CASES))
def test_crop_ref64_matches_the_pixel_loop(case):
    H, W, S, thetas = CASES[case]
    g = torch.Generator().manual_seed(list(CASES).index(case))
    B, C = 3, 2
    theta = torch.tensor(thetas, dtype=torch.float64)
    K = theta.shape[0]
    frame_idx = torch.tensor([-4, 1, 9, 2][:K], dtype=torch.int32)        # clamped to 0, 1, 2, 2
    feats = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    want, want_mag = loop_crop(feats, frame_idx, theta, S)
    got = util.crop_ref64(feats, frame_idx, theta, S)
    assert got.dtype == torch.float64 and got.shape == (K, C, S, S)
    assert torch.allclose(got, want, rtol=0, atol=1e-12), (got - want).abs().max()
    # the error scale of the forward: crop_ref64(|f|) = sum |w f| of each element's terms
    assert torch.allclose(util.crop_ref64(feats.abs(), frame_idx, theta, S), want_mag, rtol=0, atol=1e-12)
    if case == "off_map":
        assert torch.equal(got, torch.zeros_like(got))
    gout = torch.randn(K, C, S, S, generator=g, dtype=torch.float64)
    want_g = loop_adjoint(gout, frame_idx, theta, feats.shape)
    got_g = util.crop_ref64_adjoint(gout, frame_idx, theta, feats.shape)
    assert torch.allclose(got_g, want_g, rtol=0, atol=1e-12), (got_g - want_g).abs().max()
    assert torch.allclose(util.crop_ref64_adjoint(gout.abs(), frame_idx, theta, feats.shape),
                          loop_adjoint(gout.abs(), frame_idx, theta, feats.shape), rtol=0, atol=1e-12)
    # the adjoint is the transpose: <crop(f), g> = <f, adjoint(g)>
    assert abs(float((got * gout).sum() - (feats * got_g).sum())) < 1e-12 * float((got.abs() * gout.abs()).sum() + 1)


def test_identity_crop_of_a_square_map_is_a_copy():
    """S = H = W with the identity theta samples every pixel exactly once, with weight 1"""
    g = torch.Generator().manual_seed(7)
    feats = torch.randn(2, 3, 5, 5, generator=g, dtype=torch.float64)
    theta = torch.tensor([_rot(0, 1, 0, 0)] * 2, dtype=torch.float64)
    got = util.crop_ref64(feats, torch.tensor([1, 0]), theta, 5)
    assert torch.equal(got, feats[[1, 0]])


def test_crop_ref64_adjoint_of_a_frame_no_crop_reads_is_zero():
    theta = torch.tensor([_rot(0.2, 0.5, 0.1, 0.1)] * 3, dtype=torch.float64)
    gout = torch.randn(3, 2, 4, 4, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    got = util.crop_ref64_adjoint(gout, torch.tensor([0, 2, 7]), theta, (4, 2, 6, 6))   # 7 is clamped to frame 3
    assert torch.equal(got[1], torch.zeros_like(got[1]))
    assert float(got[0].abs().sum()) > 0 and float(got[2].abs().sum()) > 0 and float(got[3].abs().sum()) > 0
