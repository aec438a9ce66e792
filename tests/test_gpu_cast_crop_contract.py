"""GPU: the planners' cast GRU (lavb_cast_gru) and the uint8 BEV crop (lavb_crop_bilinear_u8) against their whole C-ABI
contract (include/lav_b200.h) and the fp64 statements of tests/util.py (cast_gru_ref, crop_u8_ref; pinned to torch's float64
nn.GRU and F.affine_grid + F.grid_sample by tests/test_cast_crop_ref_cpu.py).

Outputs start as a canary bit pattern (a NaN no kernel writes) in a buffer with spare rows or crops before and after the
slice the call owns; every element of the slice must be written and every element outside it must keep the canary, bit for
bit.

Cast GRU.  The error of an output is measured in units of cast_gru_ref's mag: the cumsum over the steps so far of
|b_mlp| + sum_j |W_mlp,j| |h_j|, i.e. against that step's own waypoint terms rather than the largest waypoint, so an error at
an early, small step shows.  The kernel's fp32 arithmetic (two fmaf chains of 512 and 64 terms, expf / tanhf within 2 ulp,
the recurrence over up to 64 steps) measured, in these units, at most 5.6e-7 at the product scale, 2.9e-7 on the frame
path and 9.5e-6 at the saturating scale, whose gates that do not saturate sum 512 inputs of size ~150 with fp32 roundings to
match (an H100 80GB HBM3 at its 700 W power limit).  util.CAST_TOL = 4e-5 leaves a margin of 4x over the largest.  The
mutants of util.CAST_MUTANTS (b_hn outside the reset gate, r and z swapped, h' = (1 - z) h + z n, the cumsum one step off,
two branches' weights swapped) are at least 0.037 away at this test's inputs, more than 100 x CAST_TOL
(tests/test_cast_crop_ref_cpu.py).

u8 crop.  Every case is compared bit for bit with lavb_crop_bilinear (fp32) on the float copy of the map, NaN patterns
included, and each crop with a finite theta is held within 1e-6 * 255 of crop_u8_ref on the kernels' own fp32 sample
positions (the header states them bit for bit): what is left is the weights' and the four fmaf roundings, below 2^-21 * 255.
A flat 1e-6 * 255 against float64 positions would not hold: an fp32 position is off by up to 2^-21 (w - 1) / 2 (1 +
sum |theta|) pixels, and a 0..255 map changes by up to 255 per pixel.  Crops with a non-finite theta follow the header's
rule (a NaN coordinate: NaN in every channel; an infinite one: 0), which crop_u8_ref states as well.
"""
import ctypes as C
import math

import pytest
import torch

from lav_b200 import capi, ops
from lav_b200.heads import crop_theta
from tests import util
from tests.util import canary, is_canary

pytestmark = pytest.mark.gpu

NAN, INF = math.nan, math.inf
CAST_WORST = {}           # case -> measured error / mag (printed with -s)


def bits(t):
    return t.contiguous().view(torch.int32)


def P(t, off=0):
    """the address of tensor t plus off bytes as a C pointer (None: NULL)"""
    return C.c_void_p(0 if t is None else t.data_ptr() + off)


def rejected(cases):
    """cases: (call, cause) pairs, each returning an entry point's status: every call must be refused with a message naming
    its cause"""
    for fn, cause in cases:
        code = fn()
        msg = capi.lib().lavb_last_error().decode() if code else ""
        assert code != 0 and cause in msg, (cause, code, msg)


# ------------------------------------------------------------------------------------------------------------------ cast GRU
def run_cast(operands, steps, dev, before=1, after=2):
    """ops.cast_gru into rows [before, before + n) of a canary buffer -> the output view; asserts that every row of the view
    and nothing else was written"""
    embd, *w = (t.to(dev) for t in operands)
    n, ncmd = embd.shape[0], w[0].shape[0]
    full = canary((before + n + after, ncmd, steps, 2), torch.float32, dev)
    out = full[before:before + n]
    got = ops.cast_gru(embd, *w, steps, out=out)
    assert got.data_ptr() == out.data_ptr()
    torch.cuda.synchronize()
    assert not bool(is_canary(out).any()), f"{int(is_canary(out).sum())} outputs never written"
    assert bool(is_canary(full[:before]).all()) and bool(is_canary(full[before + n:]).all()), "written outside rows 0..n-1"
    return out


def hold_cast(got, operands, steps, what):
    want, mag = util.cast_gru_ref(*(t.to(got.device) for t in operands), steps)
    err = util.cast_rel_err(got, want, mag)
    CAST_WORST[what] = err
    print(f"\ncast {what}: max |kernel - fp64| / mag = {err:.3g} (worst so far {max(CAST_WORST.values()):.3g})")
    assert err <= util.CAST_TOL, (what, err)
    return want


@pytest.mark.parametrize("steps", [1, 2, 20, 64])
@pytest.mark.parametrize("ncmd", [1, 6, 7])
@pytest.mark.parametrize("n", [1, 15, 16, 17, 37, 4099])
def test_cast_product_scale(cuda, n, ncmd, steps):
    """one sequence, a block less one, exactly one block, one past it, a partly full third block and 257 blocks; one branch,
    the planners' six and seven; one step up to 64; distinct weights per branch with N(0, 1) biases"""
    operands, steps = util.cast_case(n, ncmd, steps, "product")
    hold_cast(run_cast(operands, steps, cuda), operands, steps, f"product n{n} c{ncmd} t{steps}")


@pytest.mark.parametrize("n,ncmd,steps", [(37, 7, 20), (17, 6, 64), (4099, 7, 2)])
def test_cast_saturating_scale(cuda, n, ncmd, steps):
    """embeddings large enough that most gates round to exactly 0 or 1 in fp32 (tests/test_cast_crop_ref_cpu.py)"""
    operands, steps = util.cast_case(n, ncmd, steps, "saturating")
    hold_cast(run_cast(operands, steps, cuda), operands, steps, f"saturating n{n} c{ncmd} t{steps}")


def test_cast_frame_path(cuda):
    """the frame path at the benchmark's batch: 128 rows (2 pipelines x (32 egos + 96 detected vehicles)), the benchmarked
    UniPlanner's six ego branches with synth.fill_state_dict_ weights, num_plan = 20 steps; ops.cast_gru's own output equals
    the canary run bit for bit"""
    operands, steps = util.cast_case(*util.CAST_MUTANT_CASES["frame_path"])
    got = run_cast(operands, steps, cuda)
    hold_cast(got, operands, steps, "frame path")
    assert torch.equal(bits(ops.cast_gru(*(t.to(cuda) for t in operands), steps)), bits(got))


def test_cast_nan_inf_rows(cuda):
    """row 20 (second block) holds a NaN and an inf: every output of it is NaN.  Row 3 holds +inf and row 35 (the partly
    full last block) -inf: their gates saturate and their outputs stay finite, within the tolerance of the statement.  Every
    other row, the other 15 rows of each touched block included, is bit-identical to the run without them."""
    operands, steps = util.cast_case(37, 6, 20, "product")
    clean = run_cast(operands, steps, cuda)
    embd = operands[0].clone()
    embd[20, 7], embd[20, 400] = NAN, INF
    embd[3, 100] = INF
    embd[35, 511] = -INF
    got = run_cast((embd, *operands[1:]), steps, cuda)
    assert bool(torch.isnan(got[20]).all())
    others = [r for r in range(37) if r not in (3, 20, 35)]
    assert torch.equal(bits(got[others]), bits(clean[others]))
    assert bool(torch.isfinite(got[[3, 35]]).all())
    want, mag = util.cast_gru_ref(embd.to(cuda), *(t.to(cuda) for t in operands[1:]), steps)
    assert bool(torch.isnan(want[20]).all())
    err = util.cast_rel_err(got[[3, 35]], want[[3, 35]], mag[[3, 35]])
    assert err <= util.CAST_TOL, err


def test_cast_zero_rows(cuda):
    operands, steps = util.cast_case(1, 6, 20, "product")
    w = [t.to(cuda) for t in operands[1:]]
    full = canary((2, 6, 20, 2), torch.float32, cuda)
    empty = torch.zeros(0, 512, device=cuda)
    assert ops.cast_gru(empty, *w, steps, out=full[:0]).shape == (0, 6, 20, 2)
    assert capi.lib().lavb_cast_gru(P(empty), 0, *(P(t) for t in w), 6, steps, P(full), ops._stream()) == 0
    torch.cuda.synchronize()
    assert bool(is_canary(full).all())


def test_cast_rejections(cuda):
    """each refused call returns nonzero, names its cause and leaves the output's canary intact"""
    operands, steps = util.cast_case(5, 2, 4, "product")
    embd, *w = (t.to(cuda) for t in operands)
    full = canary((5, 2, steps, 2), torch.float32, cuda)
    spare = canary((5 * 2 * steps * 2 + 1,), torch.float32, cuda)
    lib = capi.lib()

    def call(e=embd, n=5, ws=None, ncmd=2, t=steps, out=full, e_off=0, out_off=0, w_off=(0,) * 6):
        ws = w if ws is None else ws
        return lib.lavb_cast_gru(P(e, e_off), n, *(P(x, o) for x, o in zip(ws, w_off)), ncmd, t, P(out, out_off), ops._stream())

    cases = [(lambda: call(n=-1), "bad shape"), (lambda: call(ncmd=0), "bad shape"), (lambda: call(ncmd=65536), "bad shape"),
             (lambda: call(t=0), "bad shape"), (lambda: call(e=None), "null"), (lambda: call(out=None), "null"),
             (lambda: call(e_off=2), "aligned"), (lambda: call(out=spare, out_off=2), "aligned"), (lambda: call(out=embd), "overlap"),
             (lambda: call(e=spare, out=spare, e_off=4 * 8), "overlap")]
    for a in range(6):
        cases += [(lambda a=a: call(ws=[None if b == a else x for b, x in enumerate(w)]), "null"),
                  (lambda a=a: call(w_off=tuple(2 if b == a else 0 for b in range(6))), "aligned"),
                  (lambda a=a: call(out=w[a]), "overlap")]                   # the output over the input's own bytes
    rejected(cases)
    torch.cuda.synchronize()
    assert bool(is_canary(full).all()) and bool(is_canary(spare).all())
    assert all(torch.equal(x, o.to(cuda)) for x, o in zip((embd, *w), operands))


# ------------------------------------------------------------------------------------------------------------------ u8 crop
SPECIAL = {        # theta rows of the first crops of a batch, by what they exercise
    "identity": [[1.0, 0.0, 0.0], [0.0, 1.0, 0.0]],
    "corner_w0_hmax": [[0.0, 0.0, -1.0], [0.0, 0.0, 1.0]],          # every sample exactly on pixel (0, h - 1)
    "corner_wmax_h0": [[0.0, 0.0, 1.0], [0.0, 0.0, -1.0]],          # ... on (w - 1, 0): the +1 taps lie off the map
    "centre": [[0.0, 0.0, 0.0], [0.0, 0.0, 0.0]],                    # (w - 1) / 2, (h - 1) / 2: a pixel or a half-pixel edge
    "half_scale_edges": [[0.5, 0.0, -0.5], [0.0, 0.5, 0.5]],
    "off_map": [[1.0, 0.0, 3.0], [0.0, 1.0, -3.0]],
    "past_2^31": [[0.5, 0.0, 3e7], [0.0, 0.5, -3e7]],
    "nan": [[NAN, 0.0, 0.0], [0.0, 1.0, 0.0]],
    "nan_y_x_off_map": [[1.0, 0.0, 1e9], [NAN, 0.0, 0.0]],         # NaN in one coordinate, the other far off the map
    "inf_scale": [[INF, 0.0, 0.0], [0.0, 1.0, 0.0]],                # +-inf, and inf * 0 = NaN where x_i is 0
    "minus_inf_shift": [[1.0, 0.0, 0.0], [0.0, 1.0, -INF]],
    "inf_both": [[0.0, -INF, 0.0], [INF, 0.0, 0.0]],
}
FINITE = ("identity", "corner_w0_hmax", "corner_wmax_h0", "centre", "half_scale_edges", "off_map", "past_2^31")


def bev_poses(K, H, W, S, seed):
    """crop poses of BEVPlanner.forward as train_bev builds them (heads.crop_theta, 2 px/m, y offset 0.75): vehicles up to
    ~25 m away, any heading, with the +-20 degree heading and +-1.5 m lateral jitter"""
    g = torch.Generator().manual_seed(seed)
    locs = torch.randn(K, 2, generator=g) * 12
    locs[:, 0] += (torch.rand(K, generator=g) * 2 - 1) * 1.5
    oris = torch.rand(K, generator=g) * 2 * math.pi - math.pi + (torch.rand(K, generator=g) * 2 - 1) * math.radians(20)
    return crop_theta(locs, oris, H, W, 2.0, S, torch.tensor(0.0), torch.tensor(0.75))


def u8_map(b, c, h, w, values, seed):
    g = torch.Generator().manual_seed(seed)
    if values == "binary":                                     # as bev_targets writes them
        return (torch.rand(b, c, h, w, generator=g) > 0.6).to(torch.uint8)
    m = torch.randint(0, 256, (b, c, h, w), generator=g, dtype=torch.uint8)
    m.view(-1)[:4] = torch.tensor([0, 255, 255, 0], dtype=torch.uint8)
    return m


def batch(K, b, h, w, S, seed):
    """K crop poses, the special ones first (as many as fit), then BEVPlanner poses; frame indices from -3 to b + 2 (the
    out-of-range ones are clamped) -> frame_idx, theta, names of the special crops in order"""
    names = list(SPECIAL)[:K]
    theta = bev_poses(K, h, w, S, seed)
    theta[:len(names)] = torch.tensor([SPECIAL[n] for n in names])
    g = torch.Generator().manual_seed(seed + 1)
    fidx = torch.randint(-3, b + 3, (K,), generator=g, dtype=torch.int32)
    return fidx, theta, names


def run_u8(bev, fidx, theta, S):
    """ops.crop_bilinear_u8 into crops [1, k + 1) of a canary buffer -> the output view; asserts every element of the view and
    nothing else was written"""
    k, c = theta.shape[0], bev.shape[1]
    full = canary((k + 2, c, S, S), torch.float32, bev.device)
    out = full[1:k + 1]
    got = ops.crop_bilinear_u8(bev, fidx, theta, S, out=out)
    assert got.data_ptr() == out.data_ptr()
    torch.cuda.synchronize()
    assert not bool(is_canary(out).any()), f"{int(is_canary(out).sum())} crop elements never written"
    assert bool(is_canary(full[0]).all()) and bool(is_canary(full[k + 1]).all()), "written outside the k crops"
    return out


def fp32_crop(bev, fidx, theta, S):
    """lavb_crop_bilinear (fp32) on the float copy of the map, NHWC with the channels zero-padded to a multiple of 4 -> NCHW"""
    b, c, h, w = bev.shape
    feats = torch.zeros(b, h, w, (c + 3) // 4 * 4, device=bev.device)
    feats[..., :c] = bev.permute(0, 2, 3, 1).float()
    return ops.crop_bilinear(feats, fidx, theta, S)[..., :c].permute(0, 3, 1, 2)


def check_u8(bev_cpu, fidx, theta, S, dev, names=()):
    bev = bev_cpu.to(dev)
    fidx, theta = fidx.to(dev), theta.to(dev)
    got = run_u8(bev, fidx, theta, S)
    assert torch.equal(bits(got), bits(fp32_crop(bev, fidx, theta, S))), "not bit-identical to the fp32 crop"
    want = util.crop_u8_ref(bev, fidx, theta, S, fp32_positions=True)
    # a crop with a finite theta is never NaN; elsewhere NaN exactly where a coordinate is NaN (the header's rule)
    assert not bool(torch.isnan(got[torch.isfinite(theta).flatten(1).all(1)]).any())
    assert torch.equal(torch.isnan(got), torch.isnan(want))
    fine = ~torch.isnan(want)
    err = float((got.double()[fine] - want[fine]).abs().max()) if bool(fine.any()) else 0.0
    assert err <= 1e-6 * 255, err
    for k, name in enumerate(names):
        if name in ("off_map", "past_2^31", "minus_inf_shift") and bev.shape[2] > 1 and bev.shape[3] > 1:
            assert float(got[k].abs().max()) == 0, name
        if name in ("nan", "nan_y_x_off_map"):
            assert bool(torch.isnan(got[k]).all()), name
    return got


MAPS = {"b1_c1": (1, 1, 40, 56), "b3_c2": (3, 2, 56, 40), "b3_c9_one_wide": (3, 9, 37, 1), "b1_c12_one_high": (1, 12, 1, 29),
        "b3_c12": (3, 12, 33, 48)}


@pytest.mark.parametrize("values", ["binary", "full"])
@pytest.mark.parametrize("S", [2, 3, 31, 32, 33, 96, 97])
@pytest.mark.parametrize("shape", list(MAPS))
def test_u8_crop_contract(cuda, shape, S, values):
    """300 crops: every special pose of SPECIAL, then BEVPlanner poses; crops at and around the kernel's 32 x 8 block edges;
    one channel up to 12; h != w; maps one pixel wide or high"""
    b, c, h, w = MAPS[shape]
    seed = sum(MAPS[shape]) * 100 + S
    fidx, theta, names = batch(300, b, h, w, S, seed)
    check_u8(u8_map(b, c, h, w, values, seed), fidx, theta, S, cuda, names)


@pytest.mark.parametrize("S", [2, 33, 97])
def test_u8_crop_single(cuda, S):
    """k = 1 for each map and each special pose, with a frame index past the last frame"""
    for shape, (b, c, h, w) in MAPS.items():
        bev = u8_map(b, c, h, w, "full", S)
        for name, th in SPECIAL.items():
            check_u8(bev, torch.tensor([b + 5], dtype=torch.int32), torch.tensor([th]), S, cuda, [name])


def test_u8_crop_bev_planner_product_shape(cuda):
    """BEVPlanner's training crop: 4 frames of the 9-channel 320 x 320 0/1 BEV, 192 x 192 crops (2 x crop_size 96) at 300
    poses of vehicles ahead and egos"""
    b, c, h, w, S, K = 4, 9, 320, 320, 192, 300
    fidx = torch.randint(0, b, (K,), generator=torch.Generator().manual_seed(77), dtype=torch.int32)
    check_u8(u8_map(b, c, h, w, "binary", 78), fidx, bev_poses(K, h, w, S, 79), S, cuda)


def test_u8_crop_int64_frame_indices_are_clamped(cuda):
    """ops.crop_bilinear_u8 clamps int64 frame indices before narrowing them, as the kernels clamp int32 ones (2^32 once
    wrapped to frame 0)"""
    bev = u8_map(3, 2, 20, 24, "full", 5).to(cuda)
    theta = bev_poses(5, 20, 24, 8, 6).to(cuda)
    i64 = torch.tensor([2, -(2 ** 33), 1, 2 ** 33, 2 ** 32], dtype=torch.int64, device=cuda)
    i32 = torch.tensor([2, 0, 1, 2, 2], dtype=torch.int32, device=cuda)
    assert torch.equal(ops.crop_bilinear_u8(bev, i64, theta, 8), ops.crop_bilinear_u8(bev, i32, theta, 8))


def test_u8_crop_rejections(cuda):
    """each refused call returns nonzero, names its cause and leaves the output's canary intact; k = 0 writes nothing"""
    b, c, h, w, k, S = 2, 3, 10, 12, 4, 6
    bev = u8_map(b, c, h, w, "full", 9).to(cuda)
    fidx, theta, _ = batch(k, b, h, w, S, 10)
    fidx, theta = fidx.to(cuda), theta.to(cuda).contiguous()
    full = canary((k, c, S, S), torch.float32, cuda)
    spare = canary((k * c * S * S + 64,), torch.float32, cuda)
    lib = capi.lib()

    def call(m=bev, bb=b, cc=c, hh=h, ww=w, fi=fidx, th=theta, kk=k, s=S, out=full, fi_off=0, th_off=0, out_off=0):
        return lib.lavb_crop_bilinear_u8(P(m), bb, cc, hh, ww, P(fi, fi_off), P(th, th_off), kk, s, P(out, out_off), ops._stream())

    cases = [(lambda: call(cc=0), "channel"), (lambda: call(s=1), "crop size"), (lambda: call(s=65536), "crop size"),
             (lambda: call(bb=0), "empty map"), (lambda: call(hh=0), "empty map"), (lambda: call(kk=-1), "negative"),
             (lambda: call(kk=65536), "65535"), (lambda: call(m=None), "null"), (lambda: call(fi=None), "null"),
             (lambda: call(th=None), "null"), (lambda: call(out=None), "null"), (lambda: call(fi_off=2), "aligned"),
             (lambda: call(th_off=2), "aligned"), (lambda: call(out=spare, out_off=2), "aligned"), (lambda: call(out=bev), "overlap"),
             (lambda: call(out=fidx), "overlap"), (lambda: call(out=theta), "overlap"),
             (lambda: call(fi=spare, out=spare, fi_off=4 * 16), "overlap"),
             (lambda: lib.lavb_crop_bilinear(P(bev), capi.F32, b, h, w, 4, P(fidx), P(theta), k, 65536, P(full), ops._stream()),
              "bad crop size")]
    rejected(cases)
    assert call(kk=0) == 0
    torch.cuda.synchronize()
    assert bool(is_canary(full).all()) and bool(is_canary(spare).all())
