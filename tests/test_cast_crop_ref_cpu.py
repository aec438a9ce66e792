"""The fp64 statements of the cast GRU and the uint8 BEV crop (tests/util.py: cast_gru_ref, crop_u8_ref) pinned to torch's
own float64 modules, and the cast mutants shown to be far outside the tolerance tests/test_gpu_cast_crop_contract.py holds
the kernel to, at that test's inputs."""
import math

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from lav_b200.heads import crop_theta
from tests import util


# ------------------------------------------------------------------------------------------------------------------ cast GRU
def modules_f64(wih_t, whh_t, bih, bhh, wmlp, bmlp):
    """one float64 nn.GRU(512, 64) and nn.Linear(64, 2) per branch, loaded from the packed operands"""
    grus, mlps = [], []
    for c in range(wih_t.shape[0]):
        g = nn.GRU(512, 64, batch_first=True, dtype=torch.float64)
        m = nn.Linear(64, 2, dtype=torch.float64)
        with torch.no_grad():
            g.weight_ih_l0.copy_(wih_t[c].t())
            g.weight_hh_l0.copy_(whh_t[c].t())
            g.bias_ih_l0.copy_(bih[c])
            g.bias_hh_l0.copy_(bhh[c])
            m.weight.copy_(wmlp[c])
            m.bias.copy_(bmlp[c])
        grus.append(g)
        mlps.append(m)
    return grus, mlps


def modules_out(embd, grus, mlps, steps):
    u = embd.double()[:, None].expand(-1, steps, -1).contiguous()
    with torch.no_grad():
        return torch.stack([torch.cumsum(m(g(u)[0]), 1) for g, m in zip(grus, mlps)], 1)


@pytest.mark.parametrize("ncmd,steps,scale", [(1, 1, "product"), (6, 20, "product"), (7, 64, "product"), (3, 2, "saturating"),
                                              (7, 20, "saturating")])
def test_cast_ref_is_torch_gru_in_float64(ncmd, steps, scale):
    ops_ = util.cast_inputs(9, ncmd, scale, seed=ncmd * 100 + steps)
    want = modules_out(ops_[0], *modules_f64(*ops_[1:]), steps)
    got, mag = util.cast_gru_ref(*ops_, steps)
    assert got.shape == mag.shape == (9, ncmd, steps, 2)
    assert float((got - want).abs().max()) <= 1e-12 * float(want.abs().max())
    # mag bounds every output and grows with the steps
    assert bool((got.abs() <= mag * (1 + 1e-12)).all()) and bool((mag[:, :, 1:] >= mag[:, :, :-1]).all())


def test_cast_ref_planner_weights_match_the_module_path():
    """cast_planner_inputs packs the benchmarked planner's ego branches as heads._cast_branches does: the statement equals
    that planner's module path (heads._cast_branches with the kernel off) in float64"""
    import lav_b200.heads as Hd
    from bench import build_models  # noqa: F401  (the planner whose weights cast_planner_inputs restates)
    embd, *pack = util.cast_planner_inputs(5)
    (_, _, uni, _), _ = build_models()
    up = uni.double()
    with torch.no_grad():
        want = Hd._cast_branches(up, up.cast_grus_ego, up.cast_mlps_ego, embd.double(), up.num_plan)
    got, _ = util.cast_gru_ref(embd, *pack, up.num_plan)
    assert float((got - want).abs().max()) <= 1e-12 * float(want.abs().max())


def test_cast_saturating_scale_saturates_the_fp32_gates():
    """at the saturating scale most fp32 gates are exactly 0 or 1 (about 3 in 4; the kernel's sigmoid is 1 / (1 + expf(-v)), which
    is 0 only once expf overflows, below -88)"""
    embd, wih_t, _, bih, bhh, _, _ = util.cast_inputs(16, 7, "saturating", seed=1)
    gi = (torch.einsum("nk,ckg->cng", embd.double(), wih_t.double()) + bih[:, None].double() + bhh[:, None].double()).float()
    s = 1 / (1 + torch.exp(-gi[..., :128]))
    assert float(((s == 0) | (s == 1)).float().mean()) > 0.6


def test_cast_ref_nan_and_inf_rules():
    """a NaN embedding element makes every output of its row NaN; an infinite one saturates the gates and leaves the
    outputs finite (the header's rule), matching float64 nn.GRU; the other rows are untouched"""
    ops_ = list(util.cast_inputs(4, 3, "product", seed=5))
    clean, _ = util.cast_gru_ref(*ops_, 7)
    embd = ops_[0].clone()
    embd[1, 17] = math.nan
    embd[2, 300] = math.inf
    embd[3, 5] = -math.inf
    got, _ = util.cast_gru_ref(embd, *ops_[1:], 7)
    want = modules_out(embd, *modules_f64(*ops_[1:]), 7)
    assert bool(torch.isnan(got[1]).all())
    assert bool(torch.isfinite(got[2:]).all())
    assert torch.equal(got[0], clean[0])
    assert float((got[2:] - want[2:]).abs().max()) <= 1e-12 * float(want[2:].abs().max())


@pytest.mark.parametrize("case", list(util.CAST_MUTANT_CASES))
@pytest.mark.parametrize("mutant", util.CAST_MUTANTS)
def test_cast_mutants_are_far_outside_the_tolerance(case, mutant):
    """each mutant differs from the statement, in the GPU test's units (|d| / mag) and at that test's inputs (the first 16
    rows: rows are independent), by at least 100 x the tolerance the kernel is held to"""
    ops_, steps = util.cast_case(*util.CAST_MUTANT_CASES[case], rows=16)
    want, mag = util.cast_gru_ref(*ops_, steps)
    bad, _ = util.cast_gru_ref(*ops_, steps, mutant=mutant)
    err = util.cast_rel_err(bad, want, mag)
    assert err >= 100 * util.CAST_TOL, (case, mutant, err)


# ------------------------------------------------------------------------------------------------------------------ u8 crop
def poses(K, H, W, S, seed):
    g = torch.Generator().manual_seed(seed)
    locs = torch.randn(K, 2, generator=g) * 8
    oris = torch.rand(K, generator=g) * 2 * math.pi - math.pi
    return crop_theta(locs, oris, H, W, 2.0, S, torch.tensor(0.0), torch.tensor(0.75))


def grid_sample64(bev, fidx, gx, gy):
    B = bev.shape[0]
    return F.grid_sample(bev.double()[fidx.long().clamp(0, B - 1)], torch.stack([gx, gy], -1), mode="bilinear", padding_mode="zeros",
                         align_corners=True)


@pytest.mark.parametrize("S", [2, 3, 17, 32, 33, 97])
def test_crop_linspace_is_torch_linspace(S):
    assert np.array_equal(util.crop_linspace32(S), torch.linspace(-1, 1, S, dtype=torch.float32).numpy())


@pytest.mark.parametrize("shape", [(3, 2, 24, 40, 17), (1, 9, 40, 24, 33), (2, 1, 1, 37, 12), (2, 3, 29, 1, 12), (1, 1, 1, 1, 5)])
def test_crop_ref_is_grid_sample_in_float64(shape):
    """the statement's bilinear with zero padding equals F.grid_sample in float64 on the same grid (positions off the map,
    maps one pixel wide or high included), and with a grid of exact linspace values (S - 1 a power of two) it equals
    F.affine_grid + F.grid_sample outright"""
    B, C, H, W, S = shape
    g = torch.Generator().manual_seed(sum(shape))
    bev = (torch.rand(B, C, H, W, generator=g) * 256).to(torch.uint8)
    K = 7
    theta = poses(K, H, W, S, 3)
    theta[0] = torch.tensor([[1.0, 0, 0], [0, 1.0, 0]])
    theta[1] = torch.tensor([[1.0, 0, 3.0], [0, 1.0, 3.0]])                   # entirely off the map
    theta[2] = torch.tensor([[0.5, 0, 1e7], [0, 0.5, -1e7]])                  # positions past +-2^31 (0 on a 1-pixel axis)
    fidx = torch.tensor([0, 1, 2, -4, 9, 1, 0], dtype=torch.int32)
    got = util.crop_u8_ref(bev, fidx, theta, S)
    x = torch.from_numpy(util.crop_linspace32(S).astype(np.float64))
    t = theta.double()
    gx = t[:, 0, 0, None, None] * x[None, None] + t[:, 0, 1, None, None] * x[None, :, None] + t[:, 0, 2, None, None]
    gy = t[:, 1, 0, None, None] * x[None, None] + t[:, 1, 1, None, None] * x[None, :, None] + t[:, 1, 2, None, None]
    want = grid_sample64(bev, fidx, gx, gy)
    assert float((got - want).abs().max()) <= 1e-12 * 255
    if H > 1 or W > 1:
        assert float(got[1].abs().max()) == 0 and float(got[2].abs().max()) == 0
    grid = F.affine_grid(t, [K, C, S, S], align_corners=True)
    affine = grid_sample64(bev, fidx, grid[..., 0], grid[..., 1])
    # the fp32 grid values differ from exact linspace values by at most 2^-24, which moves a position by at most 2^-24 (|t.0|
    # + |t.1|) (n - 1) / 2 pixels and the output by 255 per pixel and axis; none of that when S - 1 is a power of two
    exact = (S - 1) & (S - 2) == 0
    tol = 1e-12 * 255 if exact else 255 * 2.0 ** -24 * t[:, :, :2].abs().sum((1, 2)) * max(H, W) + 1e-12 * 255
    assert bool(((got - affine).abs().amax((1, 2, 3)) <= tol).all())


def test_crop_ref_fp32_positions():
    """fp32=True restates the kernels' positions: within 8 fp32 units of the scale of the float64 positions (the bound
    tests/test_gpu_crop_contract.py derives), exact on dyadic poses, and NaN / inf where theta is"""
    H, W, S = 320, 288, 97
    theta = poses(40, H, W, S, 7)
    for exact in (False, True):
        ix32, iy32 = util.crop_positions(theta, S, H, W, fp32=True)
        ix, iy = util.crop_positions(theta, S, H, W)
        t = theta.double().abs()
        dx = 2.0 ** -21 * (W - 1) / 2 * (1 + t[:, 0].sum(1))
        dy = 2.0 ** -21 * (H - 1) / 2 * (1 + t[:, 1].sum(1))
        if exact:
            assert torch.equal(ix32, ix) and torch.equal(iy32, iy)
        else:
            assert bool(((ix32 - ix).abs() <= dx[:, None, None]).all()) and bool(((iy32 - iy).abs() <= dy[:, None, None]).all())
            assert bool((ix32 != ix).any())
        theta = torch.tensor([[[1.0, 0.0, 0.0], [0.0, 1.0, 0.0]], [[0.5, -0.25, 0.125], [0.25, 0.75, -0.5]]])
        H, W, S = 33, 17, 33
    bad = torch.tensor([[[math.nan, 0, 0], [0, 1.0, 0]], [[math.inf, 0, 0], [0, 1.0, 0]], [[1.0, 0, 0], [0, 1.0, -math.inf]]])
    ix, iy = util.crop_positions(bad, 5, 8, 8, fp32=True)
    assert bool(torch.isnan(ix[0]).all()) and bool(torch.isfinite(iy[0]).all())
    assert bool(torch.isnan(ix[1, :, 2]).all()) and bool(torch.isinf(ix[1, :, 0]).all())          # inf * 0 = NaN at x = 0
    out = util.crop_u8_ref(torch.full((1, 2, 8, 8), 9, dtype=torch.uint8), torch.zeros(3, dtype=torch.int32), bad, 5, True)
    assert bool(torch.isnan(out[0]).all()) and bool(torch.isnan(out[1, :, :, 2]).all())
    assert float(out[1, :, :, 0].abs().max()) == 0 and float(out[2].abs().max()) == 0
