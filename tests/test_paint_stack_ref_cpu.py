"""The fp32 statements of the painting and stacking kernels (tests/util.py) tied to exact arithmetic and to the oracle: fma32
against exact rationals, the projection on hand-worked points, the statements against oracle.lav_ref's torch restatements,
and lavb_lidar_batch's statement against the composition its header names."""
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

from lav_b200 import ops, synth
from lav_b200 import point_painting as PP
from oracle import lav_ref as O
from tests import util
from tests.util import F32

pytestmark = pytest.mark.filterwarnings("ignore::RuntimeWarning")


def exact_f32(fr):
    """a rational rounded to fp32, round half to even, by integer arithmetic (no intermediate binary64 rounding)"""
    if fr == 0:
        return 0.0
    sign, q = (-1 if fr < 0 else 1), abs(fr)
    e = q.numerator.bit_length() - q.denominator.bit_length()
    if Fraction(2) ** e > q:
        e -= 1
    e = max(e, -126)
    m = q / Fraction(2) ** (e - 23)
    n = m.numerator // m.denominator
    rem = m - n
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and n % 2 == 1):
        n += 1
    with np.errstate(over="ignore"):
        return float(np.float32(sign * math.ldexp(n, e - 23)))


def double_rounding_triples():
    """a*b + c one 2^-70-relative step off an fp32 midpoint: binary64 rounds onto the midpoint, and ties-to-even then picks the
    wrong fp32 neighbour"""
    a = 1 + 2.0 ** -23
    b = (1 - 2.0 ** -23) * 2.0 ** -24
    out = []
    for k in (-20, 0, 7, 40):
        s = 2.0 ** k
        out += [(a, b * s, (1 + 2.0 ** -23) * s), (a, -b * s, (1 + 2.0 ** -23) * s), (-a, b * s, -(1 + 2.0 ** -23) * s)]
    return np.array(out, dtype=F32)


def test_fma32_is_correctly_rounded():
    hand = double_rounding_triples()
    g = np.random.default_rng(3)
    n = 300_000
    mant = g.uniform(1, 2, (n, 3)).astype(F32) * np.where(g.random((n, 3)) < 0.5, F32(-1), F32(1))
    ex = g.integers(-30, 30, (n, 3))
    rnd = (mant * np.exp2(ex).astype(F32)).astype(F32)
    near = rnd.copy()                                # c close to -a*b: cancellation, the hard half of fma
    near[: n // 2, 2] = (-(near[: n // 2, 0].astype(np.float64) * near[: n // 2, 1])).astype(F32) * F32(1 + 2 ** -20)
    for trip in (hand, near):
        got = util.fma32(trip[:, 0], trip[:, 1], trip[:, 2])
        want = np.array([exact_f32(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))) for a, b, c in trip], F32)
        assert np.array_equal(got, want), np.flatnonzero(got != want)[:10]
    plain = (hand[:, 0].astype(np.float64) * hand[:, 1] + hand[:, 2]).astype(F32)
    assert (plain != util.fma32(hand[:, 0], hand[:, 1], hand[:, 2])).all(), "the hand-picked triples must double-round"


# -------------------------------------------------------------------------------------------------------- projection
def unit_cams(shift=(0.0, 0.0)):
    """lidar_to_world = world_to_cam = I, K = [[1, 0, su], [0, 1, sv], [0, 0, 1]]: q = (y + su x, -z + sv x, x)"""
    K = np.array([[1, 0, shift[0]], [0, 1, shift[1]], [0, 0, 1]], np.float32)
    return np.concatenate([K.ravel(), np.eye(4, dtype=np.float32).ravel(), np.eye(4, dtype=np.float32).ravel()])[None]


H, W = 5, 7


def test_project_hit32_hand_worked():
    """x = 1024 absorbs the 1e-5 (den = 1024 exactly), so u = trunc(y / 1024), v = trunc(-z / 1024) are exact"""
    cams = unit_cams()
    pts = np.array([
        [1024, 0, 0, 0, 0],                     # pixel (0, 0)
        [1024, 1024 * W - 1, -(1024 * H - 1), W - 1, H - 1],   # last pixel: u = W - 2^-10 -> W - 1
        [1024, 1024 * W, 0, -1, 0],              # u == W: outside
        [1024, 0, -1024 * H, -1, 0],             # v == H: outside
        [1024, -1, 1, 0, 0],                    # u = trunc(-2^-10) = 0, v likewise: toward zero, seen
        [1024, -1024, 0, -1, 0],                 # u = -1: outside
        [-0.5, 0, 0, 0, 0],                      # q2 in (-1, 0) truncates to 0: in front
        [-1, 0, 0, -1, 0],                       # q2 = -1: behind
        [2.0 ** 62, 0, 0, 0, 0],                 # q2 < 2^63: truncates, seen
        [2.0 ** 63, 0, 0, -1, 0],                # q2 = 2^63 -> INT64_MIN: never a hit
        [np.inf, 0, 0, -1, 0], [np.nan, 0, 0, -1, 0], [1024, np.nan, 0, -1, 0], [1024, 0, np.inf, -1, 0],
        [1e30, 1e30, 1e30, -1, 0],
    ], np.float64)
    cam, u, v = util.project_hit32(cams, pts[:, 0], pts[:, 1], pts[:, 2], H, W)
    exp_u = pts[:, 3].astype(np.int64)
    assert np.array_equal(cam, np.where(exp_u >= 0, 0, -1))
    seen = cam >= 0
    assert np.array_equal(u[seen], exp_u[seen]) and np.array_equal(v[seen], pts[seen, 4].astype(np.int64))
    # two cameras that both see a point: the later one wins, with its own pixel
    two = np.concatenate([unit_cams(), unit_cams((2.0, 1.0))])
    cam, u, v = util.project_hit32(two, np.float32([1024]), np.float32([0]), np.float32([0]), H, W)
    assert (int(cam[0]), int(u[0]), int(v[0])) == (1, 2, 1)
    # the oracle's torch twin agrees on every hand-worked point (its values are exact here)
    sem = torch.arange(H * W, dtype=torch.float32).view(1, 1, H, W) + 1
    conv = (two[0, :9].reshape(3, 3), two[0, 9:25].reshape(4, 4), two[0, 25:].reshape(4, 4))
    want = O.point_painting_f32(torch.from_numpy(pts[:, :3].astype(np.float32)), sem, [conv])[:, 0].numpy()
    got = util.paint32(pts[:, :3], sem.numpy(), unit_cams(), 0, H, W)[0][:, 0]
    assert np.array_equal(got, want)


# ---------------------------------------------------------------------------------------------- against the oracle
def test_paint32_matches_oracle():
    from tests.test_gpu_paint_pillar import _flip_ok
    lidar, sem5, _ = util.paint_inputs()
    convs_o = O.default_converters()
    cams = np.stack([c.packed() for c in PP.make_converters()])
    sem4 = O.suppress_background(sem5)
    got, _, _ = util.paint32(lidar.numpy(), sem4.numpy(), cams, 0, 288, 256)
    want = O.point_painting_f32(lidar, sem4, convs_o).numpy()
    bad = np.flatnonzero((got != want).any(1))
    print(f"paint32 vs oracle: {len(bad)} of {len(lidar)} rows differ, all at a pixel border")
    assert len(bad) <= max(2, len(lidar) // 5000) and _flip_ok(lidar, convs_o, torch.from_numpy(bad))
    fused, _, _ = util.paint32(lidar.numpy(), sem5.numpy(), cams, 1, 288, 256)
    wantf = O.forward_paint(lidar, sem5, convs_o)[:, 4:].numpy()
    badf = np.flatnonzero((fused != wantf).any(1))
    assert set(badf.tolist()) <= set(bad.tolist())
    # mode 2: the oracle's torch softmax lies within the statement's bound on the rows both paint alike
    logits = torch.randn(3, 5, 288, 256, generator=synth._gen(5, "logits"))
    w2, b2, nan = util.paint32(lidar.numpy(), logits.numpy(), cams, 2, 288, 256)
    o2 = O.forward_paint(lidar, torch.softmax(logits, 1), convs_o)[:, 4:].numpy().astype(np.float64)
    ok = np.ones(len(lidar), bool)
    ok[bad] = False
    assert not nan.any() and (np.abs(o2 - w2)[ok] <= b2[ok] + 2.0 ** -24 * np.abs(w2[ok])).all()


def test_roof_and_stack_match_oracle():
    from tests.test_gpu_paint_pillar import _roof_sweep
    pts = _roof_sweep(5000, "rfcpu")
    keep = util.roof_keep32(pts.numpy())
    want = O.preprocess(pts).numpy()
    assert np.array_equal(np.nan_to_num(pts.numpy()[keep], nan=-7), np.nan_to_num(want, nan=-7))
    sweeps = [synth.painted_sweep(3000, tag=f"s{i}") for i in range(3)]
    loc, ori = synth.ego_motion(3, tag="stk")
    want = O.stack_lidar(sweeps, loc, ori).numpy()
    got = []
    for i, s in enumerate(sweeps):
        d = ori[i] - ori[0]
        R = np.array([[math.cos(d), math.sin(d), 0], [-math.sin(d), math.cos(d), 0], [0, 0, 1]])
        c0, s0 = math.cos(ori[0]), math.sin(ori[0])
        dl = (loc[i] - loc[0]) @ np.array([[c0, -s0], [s0, c0]])
        got.append(util.stack32(s.numpy(), R, dl[0], dl[1], i, 3))
    got = np.concatenate(got)
    diff = np.flatnonzero((got.view(np.int32) != want.view(np.int32)).any(1))
    print(f"stack32 vs oracle: {len(diff)} of {len(got)} rows differ")
    assert len(diff) == 0, diff[:10]


def test_move_point32_signed_zeros():
    """x' and y' take a real add (a -0 becomes +0); z' has no add, so a -0 z' survives"""
    R = np.eye(3, dtype=F32)
    nx, ny, nz = util.move_point32(R, 0.0, 0.0, F32([-0.0, -1]), F32([-0.0, -1]), F32([-0.0, -0.0]))
    assert not np.signbit(nx[0]) and not np.signbit(ny[0])
    assert np.signbit(nz).all()


def test_lidar_batch32_is_the_staged_composition():
    """lavb_lidar_batch = roof filter (on the row table) -> stack_sweep(R_aug) -> paint mode 0 on a ones map -> multiply ->
    stack_sweep(R_mv, dx, dy, one-hot), row by row, as include/lav_b200.h says"""
    g = np.random.default_rng(11)
    c, T, Hc, Wc = 4, 3, 288, 256
    cams = np.stack([cv.packed() for cv in PP.make_converters()])
    sizes = [700, 0, 500, 300]
    raw = np.concatenate([np.concatenate([synth.lidar_sweep(n, tag=f"lb{k}").numpy() if n else np.zeros((0, 4), F32),
                                          g.standard_normal((n, c)).astype(F32)], 1) for k, n in enumerate(sizes)])
    raw[:5, :3] = [[-1, 0, -1.2], [-0.0, -0.0, -0.0], [np.nan, 1, 1], [1e30, 0, 0], [5, -0.0, -0.0]]
    sw = np.zeros(len(sizes), ops.LIDAR_SWEEP_DTYPE)
    r0 = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    for s in range(len(sizes)):
        a, d = g.uniform(-0.3, 0.3, 2)
        sw[s] = (np.array([[math.cos(a), math.sin(a), 0], [-math.sin(a), math.cos(a), 0], [0, 0, 1]]).ravel(),
                 np.array([[math.cos(d), math.sin(d), 0], [-math.sin(d), math.cos(d), 0], [0, 0, 1]]).ravel(),
                 *g.uniform(-3, 3, 2), s % (T + 1), r0[s])
    rows = np.flatnonzero(util.roof_keep32(raw))
    rows = np.concatenate([g.permutation(rows), [-1, len(raw), -5]]).astype(np.int32)
    got = util.lidar_batch32(raw, rows, sw, cams, Hc, Wc, T)
    ones = np.ones((3, 1, Hc, Wc), F32)
    for r, src in enumerate(rows):
        if not 0 <= src < len(raw):
            assert not got[r].any()
            continue
        s = np.searchsorted(r0, src, side="right") - 1
        rot = util.stack32(raw[src:src + 1], sw[s]["R_aug"], 0.0, 0.0, 0, 0)
        vis, _, _ = util.paint32(rot, ones, cams, 0, Hc, Wc)
        rot[:, 4:] = (rot[:, 4:] * vis).astype(F32)
        want = util.stack32(rot, sw[s]["R_mv"], sw[s]["dx"], sw[s]["dy"], int(sw[s]["time_idx"]), T)
        assert np.array_equal(got[r].view(np.int32), want[0].view(np.int32)), r
