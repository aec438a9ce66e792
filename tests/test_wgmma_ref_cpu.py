"""CPU: the fp64 statements of the wgmma convolutions (tests/util.py: tap_conv64, wgmma_epilogue64, convT_assemble64,
d2s_scatter64, pair_ref64) against torch's float64 F.conv2d / F.conv_transpose2d, their NaN rule against a brute-force
receptive field, and the distance of each plausible wrong kernel (util.WGMMA_MUTANTS) from the statement at the inputs
tests/test_gpu_wgmma_contract.py uses: at least 100 times the GPU tolerance, so the GPU test would catch it."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests import util


def nhwc(t):
    return t.permute(0, 2, 3, 1)


def nchw(t):
    return t.permute(0, 3, 1, 2)


def close(a, b):
    return torch.allclose(a, b, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("k,pad,dil,stride", [(3, 1, 1, (1, 1)), (3, 1, 1, (2, 1)), (3, 1, 1, (1, 3)), (1, 0, 1, (8, 8)),
                                              (3, 1, 1, (8, 8)), (3, 2, 2, (1, 1)), (4, 1, 1, (2, 2)), ((3, 1), (1, 0), 1, (1, 1))])
def test_tap_conv_is_conv2d(k, pad, dil, stride):
    """the tap sum with Conv2d's tap list (dy = ky dil - pad) and the input stride as in_s is F.conv2d"""
    g = torch.Generator().manual_seed(1)
    kh, kw = (k, k) if isinstance(k, int) else k
    ph, pw = (pad, pad) if isinstance(pad, int) else pad
    x = torch.randn(2, 19, 29, 16, generator=g, dtype=torch.float64)
    wt = torch.randn(24, 16, kh, kw, generator=g, dtype=torch.float64)
    want = nhwc(F.conv2d(nchw(x), wt, None, stride, (ph, pw), dil))
    taps = [(ky * dil - ph, kx * dil - pw) for ky in range(kh) for kx in range(kw)]
    w = wt.permute(2, 3, 0, 1).reshape(kh * kw, 24, 16)
    got = util.tap_conv64(x, taps, w, stride, want.shape[1], want.shape[2])
    assert close(got, want)


def test_tap_conv_nan_is_the_receptive_field():
    """NaN exactly where some tap reads a NaN pixel (brute force over every output), the other outputs the conv of the
    finite values; an inf pixel gives +-inf by the weight's sign"""
    g = torch.Generator().manual_seed(2)
    x = torch.randn(1, 9, 11, 8, generator=g, dtype=torch.float64)
    x[0, 4, 5, 3] = math.nan
    x[0, 0, 10, 1] = math.inf
    w = torch.randn(9, 4, 8, generator=g, dtype=torch.float64)
    taps = util._taps(3, 1)
    for s in ((1, 1), (2, 1), (1, 3)):
        hog, wog = (9 - 1) // s[0] + 1, (11 - 1) // s[1] + 1
        got = util.tap_conv64(x, taps, w, s, hog, wog)
        for oy in range(hog):
            for ox in range(wog):
                reads = [(oy * s[0] + dy, ox * s[1] + dx) for dy, dx in taps]
                hit_nan = (4, 5) in reads
                t_inf = [t for t, r in enumerate(reads) if r == (0, 10)]
                if hit_nan:
                    assert bool(torch.isnan(got[0, oy, ox]).all())
                elif t_inf:
                    assert torch.equal(got[0, oy, ox], math.inf * torch.sign(w[t_inf[0], :, 1]))
                else:
                    assert bool(torch.isfinite(got[0, oy, ox]).all())


@pytest.mark.parametrize("name", list(util.UMMA_CONVT))
def test_convT_phases_are_conv_transpose2d(name):
    """the four phases with layers.py's tap lists, each placed on its lattice, are F.conv_transpose2d (then the epilogue)"""
    c = util.ConvTCase(name, **util.UMMA_CONVT[name])
    op = c.hout - (2 * c.h - 1)
    want = c.epi(nhwc(F.conv_transpose2d(nchw(c.x.double()), c.wt.double(), None, 2, 1, op)))
    assert close(c.want(), want)


@pytest.mark.parametrize("no", [2, 3, 8])
@pytest.mark.parametrize("hw,out_o", [((12, 14), (0, 0)), ((11, 13), (0, 0)), ((12, 14), (1, 1))])
def test_d2s_scatter_is_conv_transpose2d(no, hw, out_o):
    """the 2 x 2-tap GEMM of pack_d2s with the depth-to-space store is ConvTranspose2d(k3, s2, p1, op1) wherever its pixel
    lies inside hout x wout: the full 2h x 2w map, an odd one (each position clipped on its own), and a lattice shifted by
    out_o = (1, 1) that loses its last row and column"""
    g = torch.Generator().manual_seed(no)
    h, w = 6, 7
    x = torch.randn(2, h, w, 64, generator=g, dtype=torch.float64)
    wt = torch.randn(64, no, 3, 3, generator=g, dtype=torch.float64)
    full = nhwc(F.conv_transpose2d(nchw(x), wt, None, 2, 1, 1))              # (2, 2h, 2w, no)
    v = util.tap_conv64(x, [(0, 0), (0, 1), (1, 0), (1, 1)], util.pack_d2s(wt, no), (1, 1), h, w)
    hout, wout = hw
    got, written = util.d2s_scatter64(v, no, hout, wout, out_o)
    oy, ox = out_o
    exp_w = torch.zeros_like(written)
    exp_w[:, oy:, ox:] = True
    assert torch.equal(written, exp_w)
    assert close(got[:, oy:, ox:], full[:, :hout - oy, :wout - ox])


@pytest.mark.parametrize("dil,res,relu", [(1, True, True), (3, False, False), (31, True, False)])
def test_pair_is_two_conv2d(dil, res, relu):
    """the pair statement is relu(h16(conv3x1 + b1)) -> h16(conv1x3 + shift2) [+ res, h16] [relu] with F.conv2d; a NaN in
    the residual stays NaN without the ReLU and is 0 with it"""
    g = torch.Generator().manual_seed(dil)
    q = lambda t: t.half().double()                                           # noqa: E731
    x = q(torch.randn(2, 6, 32, 64, generator=g))
    w1, w2 = (q(torch.randn(3, 64, 64, generator=g) / 14) for _ in range(2))
    b1, t2 = torch.randn(64, generator=g) * 0.1, torch.randn(64, generator=g) * 0.1
    r = q(torch.randn(2, 6, 32, 64, generator=g)) if res else None
    if res:
        r[1, 2, 3, 4] = math.nan
    mid = util.fmax0(q(F.conv2d(nchw(x), w1.permute(1, 2, 0)[..., None], b1.double(), padding=(dil, 0), dilation=(dil, 1))))
    a = q(nhwc(F.conv2d(mid, w2.permute(1, 2, 0)[:, :, None, :], t2.double(), padding=(0, dil), dilation=(1, dil))))
    if res:
        a = q(a + r)
    want = util.fmax0(a) if relu else a
    got = util.pair_ref64(x, w1, b1, w2, t2, dil, r, relu)
    assert util.wgmma_err(got, want) == 0.0
    if res:
        assert bool(torch.isnan(got[1, 2, 3, 4])) != relu


def test_store_and_epilogue_rules():
    """h16 stores saturate and keep NaN; a ReLU turns NaN into 0, no ReLU keeps it; the folded bias is the same fp64 value"""
    a = torch.tensor([math.nan, 1e6, -1e6, -0.5, 2.0], dtype=torch.float64)
    assert util.wgmma_err(util.store64(a, "h16"), torch.tensor([math.nan, 65504, -65504, -0.5, 2.0], dtype=torch.float64)) == 0
    one = torch.ones(5)
    assert torch.isnan(util.wgmma_epilogue64(a, one, -one, one, None, False, False)[0])
    assert util.wgmma_epilogue64(a, one, -one, one, None, True, False)[0] == 1.0
    assert util.wgmma_epilogue64(a, one, -one, one, None, False, True)[0] == 0.0


@pytest.mark.parametrize("mutant", util.WGMMA_MUTANTS)
def test_mutants_are_far_from_the_statement(mutant):
    """each plausible wrong kernel lands at least 100 x the GPU test's tolerance from the statement at that test's inputs
    (inf: a NaN or infinity in the wrong place)"""
    kind, name = util.WGMMA_MUTANT_CASES[mutant]
    if kind == "convT":
        c = util.ConvTCase(name, **util.UMMA_CONVT[name])
        tol = util.WGMMA_TOL["f32"]
    else:
        c = util.UmmaCase(name, **util.UMMA_CASES[name])
        tol = util.WGMMA_TOL[c.out]
    want = c.want()
    assert util.wgmma_err(want, want) == 0.0
    err = util.wgmma_err(c.want(mutant), want)
    print(f"{mutant} at {name}: {err / tol:.3g} x the tolerance")
    assert err >= 100 * tol, (mutant, err)


@pytest.mark.parametrize("name", list(util.UMMA_CASES))
def test_umma_cases_are_well_posed(name):
    """every conv_umma case of the GPU test has a non-trivial statement: finite outputs that are not all zero, NaN / inf
    only where the case puts them, and the stored weight rows finite"""
    c = util.UmmaCase(name, **util.UMMA_CASES[name])
    want = c.want()
    fin = torch.isfinite(want)
    assert float(want[fin].abs().max()) > 0.1
    spec = util.UMMA_CASES[name]
    assert bool(torch.isnan(want).any()) == (spec.get("nan", False) and not spec.get("pre", True) and not spec.get("post", False)
                                              or spec.get("nan", False) and spec.get("sig", False))
    assert bool(torch.isfinite(c.w[:, :c.cout]).all())
