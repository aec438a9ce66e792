"""The painting, sweep stacking, roof filter and LiDAR batch kernels against their C-ABI contract (include/lav_b200.h): every
output bit for bit against the fp32 statements of tests/util.py, except the softmax outputs, which must lie within the
statement's bound.  Every output starts as a canary with a spare row and frame past the end, so an element written that the
contract leaves alone, or one never written, fails the test."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from lav_b200 import capi, ops, synth
from lav_b200 import point_painting as PP
from tests import util
from tests.util import F32, canary, is_canary, kernels

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore::RuntimeWarning")]

RATIO = {}            # largest |got - want| / bound of the softmax outputs, per case (printed with -s)
NAN32 = 0x7FC00000


def lib():
    return capi.lib()


def gen(seed):
    return torch.Generator().manual_seed(seed)


def bits(t):
    t = t.cpu().contiguous() if torch.is_tensor(t) else torch.from_numpy(np.ascontiguousarray(t))
    return t.view(torch.int32)


def hold_values(got, want, what):
    """bit for bit, except that a NaN the kernel computes only has to be a NaN: the GPU's arithmetic returns its canonical
    NaN where numpy passes the operand's payload on"""
    g, w = got.cpu().contiguous().numpy(), np.ascontiguousarray(want, dtype=F32)
    wn = np.isnan(w)
    assert np.array_equal(np.isnan(g), wn), f"{what}: NaN pattern"
    assert np.array_equal(g.view(np.int32)[~wn], w.view(np.int32)[~wn]), f"{what}: values"


def cams_for(H, W, ncam=3):
    """the agent's cameras for an H x W image; a 4th camera repeats the first with its image shifted, so every point the
    first sees is seen twice (the later camera must win)"""
    cams = np.stack([c.packed() for c in PP.make_converters(rgb_h=H, rgb_w=W)])
    if ncam == 4:
        c4 = cams[0].copy()
        c4[2] += 1.5                       # K[0][2]: u shifted by 1.5 * q2
        cams = np.concatenate([cams, c4[None]])
    return np.ascontiguousarray(cams[:ncam], dtype=F32)


SPECIAL = [(math.nan, 5, 1), (5, math.nan, 1), (5, 1, math.nan), (math.inf, 0, 0), (-math.inf, 0, 0), (5, math.inf, 1),
           (5, 1, -math.inf), (1e30, 1e30, 1e30), (-1e30, 0, 0), (5, 1e30, 0), (0, 0, 0), (-0.0, -0.0, -0.0), (5, 0, -0.0),
           (-5, 0, 0)]


def points(F, n, seed, spread=40.0):
    """(F, n, 4) fp32: LiDAR-like points around the car, the special values of SPECIAL in the first rows of frame 0"""
    g = gen(seed)
    p = torch.cat([(torch.rand(F, n, 3, generator=g) - 0.5) * 2 * spread, torch.rand(F, n, 1, generator=g)], 2)
    p[..., 2] = p[..., 2] * 0.1 - 1.0
    k = min(n, len(SPECIAL))
    p[0, :k, :3] = torch.tensor(SPECIAL[:k], dtype=torch.float32)
    return p.contiguous()


def point_view(p, ps, misalign, dev, gap=0):
    """p (F, n, 4) -> a (F, n, ps) view whose leading 4 columns are p's (columns >= 4 random); misalign shifts the view by one
    float, gap leaves that many floats between frames (frame stride n * ps + gap)"""
    F, n, _ = p.shape
    full = torch.rand(F, n, max(ps, 4), generator=gen(ps))
    full[..., :4] = p
    fs = n * ps + gap
    flat = torch.zeros(F * fs + 8, device=dev)
    off = 1 if misalign else 0
    v = flat[off:off + F * fs].view(F, fs)[:, :n * ps].view(F, n, ps)
    v.copy_(full[..., :ps].to(dev))
    return v


def c_paint_batched(pts, ps, pts_fs, F, n, sem, mode, cams, out, out_stride, out_fs, col0, copy, ncam=None):
    """lavb_paint_batched on a logical (F, ncam, C, H, W) sem view of any strides; -> status"""
    _, nc, Cc, H, W = sem.shape
    s = sem.stride()
    cams = np.ascontiguousarray(cams, dtype=F32)
    return lib().lavb_paint_batched(ops._ptr(pts), F, n, ps, pts_fs, ops._ptr(sem), ncam or nc, Cc, H, W, s[0], s[1], s[2], s[3],
                                    s[4], ops._hptr(cams), mode, ops._ptr(out), out_stride, out_fs, col0, copy, ops._stream())


def hold_rows(full, F, n, pts, copy, col0, want, bound, nan, what, copied=False):
    """full (F + 1, n + 1, S) canary-filled output; rows [0, n) of frames [0, F) hold the copied columns bit for bit, the painted
    channels against (want, bound, nan) of the statement, every other element canary"""
    c_out = want.shape[-1]
    full = full.cpu()
    S = full.shape[-1]
    assert bool(is_canary(full[F:]).all()) and bool(is_canary(full[:, n:]).all()), f"{what}: written past the end"
    got = full[:F, :n]
    assert torch.equal(bits(got[..., :copy]), bits(pts[..., :copy].cpu())), f"{what}: copied columns"
    assert bool(is_canary(got[..., copy:col0]).all()) and bool(is_canary(got[..., col0 + c_out:]).all()), f"{what}: gap / tail written"
    g = got[..., col0:col0 + c_out].numpy()
    assert S >= col0 + c_out and not bool(is_canary(got[..., col0:col0 + c_out]).any()), f"{what}: painted channels not written"
    if copied:                            # mode 0: the map's bits, NaN payloads included
        assert np.array_equal(g.view(np.int32), want.astype(F32).view(np.int32)), f"{what}: values"
        return
    if bound is None:
        wn = np.isnan(want)
        assert np.array_equal(np.isnan(g), wn), f"{what}: NaN pattern"
        assert np.array_equal(g.view(np.int32)[~wn], want.astype(F32).view(np.int32)[~wn]), f"{what}: values"
        return
    assert np.array_equal(np.isnan(g).all(-1), nan) and not np.isnan(g[~nan]).any(), f"{what}: NaN rule"
    g, w, b = g[~nan].astype(np.float64), want[~nan], bound[~nan]
    err = np.abs(g - w)
    ok = (err <= b) | (g == w)
    assert ok.all(), f"{what}: {int((~ok).sum())} outside the bound, worst {float((err - b).max())}"
    live = b > 0
    RATIO[what] = float((err[live] / b[live]).max()) if live.any() else 0.0


def sem_view(F, ncam, Cc, H, W, layout, seed, dev, special=False):
    """a logical (F, ncam, C, H, W) fp32 view in the given storage layout"""
    g = gen(seed)
    if layout == "nchw":
        s = torch.randn(F, ncam, Cc, H, W, generator=g)
    elif layout == "cl":
        s = torch.randn(F, ncam, H, W, Cc, generator=g)
    elif layout == "slice":
        s = torch.randn(F, ncam, Cc + 3, H, W, generator=g)
    elif layout == "expand":
        s = torch.randn(F, 1, Cc, H, W, generator=g)
    else:                                 # "hw_t": H and W transposed in storage
        s = torch.randn(F, ncam, Cc, W, H, generator=g)
    if special:                           # NaN, +-inf, +-1e30 and -0 at a tenth of the stored values
        flat = s.view(-1)
        pick = torch.randperm(flat.numel(), generator=g)[:max(1, flat.numel() // 10)]
        vals = torch.tensor([math.nan, math.inf, -math.inf, 1e30, -1e30, -0.0])
        flat[pick] = vals[torch.arange(len(pick)) % len(vals)]
    s = s.to(dev)
    if layout == "cl":
        return s.permute(0, 1, 4, 2, 3)
    if layout == "slice":
        return s[:, :, 2:2 + Cc]
    if layout == "expand":
        return s.expand(F, ncam, Cc, H, W)
    if layout == "hw_t":
        return s.transpose(3, 4)
    return s


def run_paint(dev, F, n, ps, misalign, sem, mode, cams, copy, col0, out_misalign=False, sem_fs0=False, S=None, pts_gap=0,
              out_gap=0):
    """lavb_paint_batched into a canary output (F + 1, n + 1, S), one float off when out_misalign, with out_gap floats between
    its frames (which must stay canary) -> (output, points, statement)"""
    p = points(F, n, 17 + n + ps)
    pv = point_view(p, ps, misalign, dev, pts_gap)
    _, ncam, Cc, H, W = sem.shape
    c_out = Cc if mode == 0 else Cc - 1
    off = 1 if out_misalign else 0
    S = S or col0 + c_out + 1 + off
    ofs = (n + 1) * S + out_gap
    flat = canary(((F + 1) * ofs + 4,), torch.float32, dev)
    frames = flat[off:off + (F + 1) * ofs].view(F + 1, ofs)
    full = frames[:, :(n + 1) * S].view(F + 1, n + 1, S)
    assert c_paint_batched(pv, ps, pv.stride(0), F, n, sem, mode, cams, full, S, ofs, col0, copy) == 0, \
        lib().lavb_last_error().decode()
    assert bool(is_canary(frames[:, (n + 1) * S:]).all()), "written between the output frames"
    pc = pv.cpu().numpy()
    if sem_fs0:
        return (full, pv, *util.paint32(pc, sem[0].cpu().numpy(), cams, mode, H, W))
    sc = sem.cpu().numpy()
    res = [util.paint32(pc[f], sc[f], cams, mode, H, W) for f in range(F)]
    want = np.stack([r[0] for r in res])
    bound = None if res[0][1] is None else np.stack([r[1] for r in res])
    nan = None if res[0][2] is None else np.stack([r[2] for r in res])
    return full, pv, want, bound, nan


# --------------------------------------------------------------------------------------------------------- painting
LAYOUTS = ["nchw", "cl", "slice", "expand", "hw_t"]
MODES = [(m, c) for m in (0, 1, 2) for c in ((1 if m == 0 else 2), 5, 8)]


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("mode,c_in", MODES, ids=lambda v: str(v))
def test_paint_modes_layouts(cuda, mode, c_in, layout):
    k = MODES.index((mode, c_in)) + LAYOUTS.index(layout)
    ps = (3, 4, 5, 11)[k % 4]
    copy = min(ps, (0, 1, 3, 4, 2)[k % 5])
    col0 = copy + (k % 3)
    H, W = ((7, 5), (37, 29), (1, 1))[k % 3]
    cams = cams_for(H, W, 3)
    sem = sem_view(3, 3, c_in, H, W, layout, 100 + k, cuda, special=(k % 2 == 0))
    full, pv, want, bound, nan = run_paint(cuda, 3, 257, ps, k % 2 == 1, sem, mode, cams, copy, col0, out_misalign=(k % 3 == 1))
    hold_rows(full, 3, 257, pv, copy, col0, want, bound, nan, f"paint m{mode} c{c_in} {layout}", copied=(mode == 0))


@pytest.mark.parametrize("n", [1, 255, 256, 257])
@pytest.mark.parametrize("ncam", [1, 2, 4])
def test_paint_sizes_and_cameras(cuda, n, ncam):
    """288 x 256 images, pt_stride 4 with 4 copied columns (the vector path) and the other camera counts; 4 cameras make every
    point the first camera sees a point two cameras see"""
    cams = cams_for(288, 256, ncam)
    sem = sem_view(2, ncam, 5, 288, 256, "cl", n + ncam, cuda)
    full, pv, want, bound, nan = run_paint(cuda, 2, n, 4, False, sem, 2, cams, 4, 4)
    hold_rows(full, 2, n, pv, 4, 4, want, bound, nan, f"paint n{n} ncam{ncam}")


def test_paint_product_shape(cuda):
    """the agent's painting: 40 000 points x 8 frames, logits channels-last, rows of 8 floats, copy 4 then 4 channels (mode 2):
    the vector load and store the agent takes"""
    cams = cams_for(288, 256)
    sem = sem_view(8, 3, 5, 288, 256, "cl", 7, cuda)
    full, pv, want, bound, nan = run_paint(cuda, 8, 40000, 4, False, sem, 2, cams, 4, 4, S=8)
    hold_rows(full, 8, 40000, pv, 4, 4, want, bound, nan, "paint product")
    print("paint product: largest softmax error / bound", RATIO["paint product"])


@pytest.mark.parametrize("case", ["aligned", "out_view_misaligned", "pts_frame_gap", "out_frame_gap"])
def test_paint_vector_path_layouts(cuda, case):
    """pt_stride 4, 4 copied columns, out_col0 4 and rows of 12 floats: aligned, the vector load and store apply; an output view
    one float off (buf[:, 1:] of an (n, 13) buffer), or frames of points or of output one float apart, must take the
    per-element path for the rows it cannot vectorise and give the same values"""
    cams = cams_for(37, 29)
    sem = sem_view(3, 3, 5, 37, 29, "cl", 60, cuda)
    kw = dict(aligned={}, out_view_misaligned=dict(out_misalign=True), pts_frame_gap=dict(pts_gap=1), out_frame_gap=dict(out_gap=1))
    full, pv, want, bound, nan = run_paint(cuda, 3, 300, 4, False, sem, 2, cams, 4, 4, S=12, **kw[case])
    hold_rows(full, 3, 300, pv, 4, 4, want, bound, nan, f"paint vector {case}")


@pytest.mark.parametrize("frames", [1, 3, 64, 65535])
def test_paint_frames(cuda, frames):
    """the frame index reaches every frame: 65535 frames of 2 points; the semantic maps of all frames share one (s_frame 0)"""
    n = 2 if frames > 64 else 33
    cams = cams_for(7, 5)
    sem = sem_view(1, 3, 3, 7, 5, "nchw", frames, cuda).expand(frames, 3, 3, 7, 5)
    full, pv, want, bound, nan = run_paint(cuda, frames, n, 4, False, sem, 1, cams, 4, 4, sem_fs0=True)
    hold_rows(full, frames, n, pv, 4, 4, want, bound, nan, f"paint frames {frames}")


def test_paint_logit_rules(cuda):
    """mode 2 on hand-set logits at every pixel of a 1 x 1 image: a NaN or +inf logit, or all -inf, make every painted channel
    NaN; a -inf logit among finite ones is an exact 0 probability; a point no camera sees gets exact zeros"""
    rows = torch.tensor([[0.0, 1, 2, 3], [math.nan, 1, 2, 3], [0, 1, math.inf, 3], [-math.inf] * 4, [0, -math.inf, 2, 3],
                         [1e30, -1e30, 0, 0], [-0.0, 0.0, -0.0, 0.0], [0, 1, math.nan, math.nan]])
    cams = cams_for(1, 1)
    pv = points(1, 128, 5).to(cuda)
    seen = torch.from_numpy(util.project_hit32(cams, *pv[0, :, :3].cpu().numpy().T, 1, 1)[0] >= 0)
    assert bool(seen.any()) and not bool(seen.all())
    for r in rows:
        sem = r.view(1, 1, 4, 1, 1).expand(1, 3, 4, 1, 1).to(cuda)
        full = canary((2, 129, 8), torch.float32, cuda)
        assert c_paint_batched(pv, 4, 128 * 4, 1, 128, sem, 2, cams, full, 8, 129 * 8, 4, 4) == 0
        want, bound, nan = util.paint32(pv[0].cpu().numpy(), sem[0].cpu().numpy(), cams, 2, 1, 1)
        hold_rows(full, 1, 128, pv, 4, 4, want[None], bound[None], nan[None], f"logits {r.tolist()}")
        got = full[0, :128, 4:7].cpu()
        assert torch.equal(bits(got[~seen]), torch.zeros(int((~seen).sum()), 3, dtype=torch.int32))
        expect_nan = bool(torch.isnan(r).any() or (r == math.inf).any() or (r == -math.inf).all())
        assert bool(torch.isnan(got[seen]).all()) == expect_nan and (expect_nan or not bool(torch.isnan(got).any()))


# ------------------------------------------------------------------------------------------------- painting from features
def run_deconv(dev, F, n, dtype, Cc, H, W, seed, ncam=3, nan_feat=False, copy=4, col0=4, S=None):
    g = gen(seed)
    cams = cams_for(H, W, ncam)
    feat = torch.randn(F * ncam, H // 2, W // 2, 16, generator=g) * 0.5
    if nan_feat:
        feat.view(-1, 16)[torch.randperm(feat.numel() // 16, generator=g)[:feat.numel() // 160], 3] = math.nan
    feat = feat.to(dtype).to(dev)
    table = ops.pack_deconv2x2(torch.randn(16, Cc, 2, 2, generator=g) * 0.4, torch.randn(Cc, generator=g)).to(dev)
    p = points(F, n, seed + 1).to(dev)
    S = S or col0 + Cc - 1 + 1
    full = canary((F + 1, n + 1, S), torch.float32, dev)
    code = lib().lavb_paint_deconv_batched(ops._ptr(p), F, n, 4, n * 4, ops._ptr(feat), ops._DT[dtype], ncam, Cc, H, W,
                                           ops._ptr(table), ops._hptr(cams), ops._ptr(full), S, (n + 1) * S, col0, copy, ops._stream())
    assert code == 0, lib().lavb_last_error().decode()
    want, bound, nan = util.paint_deconv32(p.cpu().numpy(), feat.float().cpu().numpy(), table.cpu().numpy(), cams, Cc, H, W)
    return full, p, want, bound, nan


@pytest.mark.parametrize("c_cls", [2, 5, 8])
@pytest.mark.parametrize("dtype", ["f32", "h16"])
def test_paint_deconv(cuda, dtype, c_cls):
    dt = torch.float32 if dtype == "f32" else ops.h16()
    full, p, want, bound, nan = run_deconv(cuda, 3, 3000, dt, c_cls, 36, 30, 40 + c_cls, nan_feat=True)
    hold_rows(full, 3, 3000, p, 4, 4, want, bound, nan, f"deconv {dtype} c{c_cls}")
    assert nan.any() and (~nan).any()


def test_paint_deconv_product_shape(cuda):
    """the agent's shape: rows of 8 floats (4 copied, 4 painted), the vector load and store it takes"""
    full, p, want, bound, nan = run_deconv(cuda, 4, 40000, ops.h16(), 5, 288, 256, 9, S=8)
    hold_rows(full, 4, 40000, p, 4, 4, want, bound, nan, "deconv product")
    print("deconv product: largest softmax error / bound", RATIO["deconv product"])


def test_batch_independence_and_repeat(cuda):
    """no atomics: a frame alone equals the frame in a batch, and two runs give the same bits"""
    a = run_deconv(cuda, 3, 2000, ops.h16(), 5, 36, 30, 70)
    b = run_deconv(cuda, 3, 2000, ops.h16(), 5, 36, 30, 70)
    assert torch.equal(bits(a[0]), bits(b[0]))
    p, full = a[1], a[0]
    cams = cams_for(36, 30)
    sem = sem_view(3, 3, 5, 36, 30, "cl", 71, cuda)
    outs = []
    for f in (None, 0, 1, 2):
        F = 3 if f is None else 1
        pf = p if f is None else p[f:f + 1].contiguous()
        sf = sem if f is None else sem[f:f + 1]
        o = canary((F, 2000, 8), torch.float32, cuda)
        assert c_paint_batched(pf, 4, 2000 * 4, F, 2000, sf, 2, cams, o, 8, 2000 * 8, 4, 4) == 0
        outs.append(o)
    for f in range(3):
        assert torch.equal(bits(outs[0][f]), bits(outs[1 + f][0]))


# ------------------------------------------------------------------------------------------------------------ stacking
def roof_rows(n, cols, seed):
    """rows with every face of the roof box exactly on its fp32 bound and one ulp inside, -0 coordinates, NaN, the rest random
    around the box"""
    g = np.random.default_rng(seed)
    r = np.empty((n, cols), F32)
    r[:, :3] = g.uniform([-3, -1, -1.7], [0.5, 1, -0.8], (n, 3)).astype(F32)
    r[:, 3:] = g.standard_normal((n, cols - 3)).astype(F32)
    x0, x1, y0, y1, z0, z1 = util.ROOF
    mid = [F32(-1.2), F32(0), F32(-1.25)]
    faces = []
    for ax, (lo, hi) in enumerate(((x0, x1), (y0, y1), (z0, z1))):
        for v in (lo, hi, np.nextafter(lo, hi), np.nextafter(hi, lo)):
            q = list(mid)
            q[ax] = v
            faces.append(q)
    faces += [[-1.2, -0.0, -1.25], [-0.0, -0.0, -0.0], [math.nan, 0, -1.25], [-1.2, math.nan, -1.25]]
    k = min(n, len(faces))
    r[:k, :3] = np.array(faces[:k], F32)
    return r


def rot(a):
    c, s = math.cos(a), math.sin(a)
    return np.array([[c, s, 0], [-s, c, 0], [0, 0, 1]], F32)


@pytest.mark.parametrize("n_time", [0, 1, 3])
@pytest.mark.parametrize("src_cols", [3, 4, 8, 13])
def test_stack_sweep(cuda, src_cols, n_time):
    n = 513
    src = roof_rows(n, src_cols, src_cols * 10 + n_time)
    for roof, (dx, dy), R in ((0, (-0.0, -0.0), np.eye(3, dtype=F32)), (1, (1.5, -2.25), rot(0.3))):
        d = torch.from_numpy(src).to(cuda)
        full = canary((n + 1, src_cols + n_time), torch.float32, cuda)
        ti = max(n_time - 1, 0)
        assert lib().lavb_stack_sweep(ops._ptr(d), n, src_cols, ops._hptr(np.ascontiguousarray(R)), dx, dy, ti, n_time, roof,
                                      ops._ptr(full), ops._stream()) == 0
        want = util.stack32(src, R, dx, dy, ti, n_time, roof=bool(roof))
        hold_values(full[:n], want, f"stack roof {roof}")
        assert bool(is_canary(full[n:]).all())


def job_table(jobs):
    t = np.zeros(len(jobs), ops.STACK_JOB_DTYPE)
    for k, (src, dst, n, ti, R, dx, dy) in enumerate(jobs):
        t[k] = (src, dst, n, ti, R.ravel(), dx, dy, 0)
    return torch.from_numpy(t.view(np.uint8)).to("cuda")


STACK_CASES = [(3, 0), (3, 3), (4, 1), (8, 3), (8, 0), (13, 3), (8, 8), (13, 0)]


@pytest.mark.parametrize("src_cols,n_time", STACK_CASES)
def test_stack_jobs(cuda, src_cols, n_time):
    """jobs of n around multiples of 256, n = 0 and longer than max_n, a time_idx out of range, a src of 8 columns not 16-byte
    aligned; each job's output with a spare canary row after it"""
    ns = [0, 1, 255, 256, 257, 511, 700, 1300]
    max_n = 600
    dc = src_cols + n_time
    srcs, outs, jobs, wants = [], [], [], []
    for k, n in enumerate(ns):
        s = roof_rows(max(n, 1), src_cols, 300 + k)[:n]
        buf = torch.zeros(n * src_cols + 4, device=cuda)
        off = 1 if k == 2 else 0
        buf[off:off + n * src_cols] = torch.from_numpy(s.ravel()).to(cuda)
        o = canary(((n + 1) * dc,), torch.float32, cuda)
        R, dx, dy = rot(0.1 * k), F32(0.5 * k - 1), F32(-0.0 if k % 2 else 0.25 * k)
        ti = 7 if k == 4 else k % max(n_time, 1)
        jobs.append((buf.data_ptr() + 4 * off, o.data_ptr(), n, ti, R, dx, dy))
        srcs.append(buf)
        outs.append(o)
        wants.append(util.stack32(s, R, dx, dy, ti, n_time, roof=True))
    table = job_table(jobs)
    assert lib().lavb_stack_jobs(ops._ptr(table), len(jobs), max_n, src_cols, n_time, 1, ops._stream()) == 0
    for n, o, w in zip(ns, outs, wants):
        hold_values(o[:n * dc], w.ravel(), f"job of {n} rows")
        assert bool(is_canary(o[n * dc:]).all()), n


def test_stack_jobs_product_shape_and_graph(cuda):
    """192 jobs x 40 000 rows (B = 64 agents x T = 3 sweeps of 8 columns, the agent's shape); then the graph promise: one
    captured call replays the rewritten table (new R, n and source slot) and matches the statement of the new table"""
    B, T, N = 64, 3, 40000
    srcs = [roof_rows(N, 8, 500 + t) for t in range(T + 1)]
    src_d = torch.from_numpy(np.stack(srcs)).to(cuda)
    out = canary((B * T * N + 1, 8 + T), torch.float32, cuda)

    def table(rs, ns, slots):
        jobs = []
        for b in range(B):
            for t in range(T):
                jobs.append((src_d[slots[t]].data_ptr(), out[(b * T + t) * N].data_ptr(), ns[t], t, rs[t], F32(t), F32(-t)))
        return job_table(jobs)

    def check(rs, ns, slots):
        want = [util.stack32(srcs[slots[t]][:ns[t]], rs[t], F32(t), F32(-t), t, T, roof=True) for t in range(T)]
        o = out[:-1].view(B, T, N, 8 + T).cpu()
        for t in range(T):
            hold_values(o[:, t, :ns[t]], np.broadcast_to(want[t], (B, *want[t].shape)), f"sweep {t}")
        assert bool(is_canary(out[-1]).all())

    rs = [rot(0.2 * t) for t in range(T)]
    d_jobs = table(rs, [N] * T, [0, 1, 2])
    ops.stack_jobs(d_jobs, B * T, N, 8, T, roof_filter=True)
    check(rs, [N] * T, [0, 1, 2])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        ops.stack_jobs(d_jobs, B * T, N, 8, T, roof_filter=True)
    torch.cuda.current_stream().wait_stream(s)
    rs2, ns2 = [rot(-0.4 + t) for t in range(T)], [N, N - 257, 1000]
    d_jobs.copy_(table(rs2, ns2, [3, 0, 2]))
    g.replay()
    torch.cuda.synchronize()
    check(rs2, ns2, [3, 0, 2])


# --------------------------------------------------------------------------------------------------------- roof filter
@pytest.mark.parametrize("cols", [3, 4, 17])
@pytest.mark.parametrize("n", [0, 1, 1023, 1024, 1025, 40000])
def test_roof_filter(cuda, n, cols):
    """3 frames with gaps between them in both buffers; pad_nan on and off; counts NULL once"""
    F = 3
    sfs, dfs = n * cols + 5, n * cols + 7
    src = torch.zeros(F * sfs + 8, device=cuda)
    rows = [roof_rows(max(n, 1), cols, 900 + f + n)[:n] for f in range(F)]
    if n > 40:
        rows[1][:: 3, :3] = [-1.2, 0, -1.25]          # a third of frame 1 inside the box
    for f in range(F):
        src[f * sfs:f * sfs + n * cols] = torch.from_numpy(rows[f].ravel()).to(cuda)
    for pad in (0, 1):
        dst = canary((F * dfs + 8,), torch.float32, cuda)
        cnt = canary((F + 1,), torch.float32, cuda).view(torch.int32)
        cptr = ops._ptr(cnt) if pad or n != 1024 else ops._ptr(None)
        assert lib().lavb_roof_filter(ops._ptr(src), F, n, cols, sfs, ops._ptr(dst), dfs, cptr, pad, ops._stream()) == 0
        d = dst.cpu()
        for f in range(F):
            keep = util.roof_keep32(rows[f]) if n else np.zeros(0, bool)
            k = int(keep.sum())
            if cptr.value:
                assert int(cnt[f]) == k
            fr = d[f * dfs:f * dfs + n * cols]
            assert torch.equal(bits(fr[:k * cols]), bits(rows[f][keep].ravel()))
            tail = bits(fr[k * cols:])
            assert bool((tail == NAN32).all()) if pad else bool(is_canary(fr[k * cols:]).all())
            assert bool(is_canary(d[f * dfs + n * cols:(f + 1) * dfs]).all())      # the gap after each frame
        assert bool(is_canary(d[F * dfs:]).all())
        assert cptr.value or bool(is_canary(cnt.view(torch.float32)).all())
        assert not cptr.value or bool(is_canary(cnt[F:].view(torch.float32)).all())


# --------------------------------------------------------------------------------------------------------- lidar batch
def lidar_inputs(sizes, c, T, seed, first_row0=10):
    g = np.random.default_rng(seed)
    n_raw = first_row0 + sum(sizes)
    raw = np.concatenate([points(1, n_raw, seed)[0].numpy(), g.standard_normal((n_raw, c)).astype(F32)], 1)
    raw[first_row0:first_row0 + 40, :3] = roof_rows(40, 3, seed)[:, :3]
    sw = np.zeros(len(sizes), ops.LIDAR_SWEEP_DTYPE)
    r0 = first_row0 + np.concatenate([[0], np.cumsum(sizes)[:-1]])
    for s in range(len(sizes)):
        sw[s] = (rot(g.uniform(-0.3, 0.3)).ravel(), rot(g.uniform(-0.3, 0.3)).ravel(), *g.uniform(-3, 3, 2).astype(F32),
                 s % (T + 1), r0[s])
    return raw, sw


@pytest.mark.parametrize("c", [0, 4, 7])
def test_lidar_batch(cuda, c):
    """rows of -1, past n_raw and before the first row0; sweeps of 0 rows; a time_idx of n_time (no one-hot)"""
    T = 3
    raw, sw = lidar_inputs([300, 0, 700, 0, 257], c, T, 60 + c)
    n_raw = len(raw)
    g = np.random.default_rng(c)
    rows = np.concatenate([g.permutation(n_raw), [-1, n_raw, n_raw + 5, 0, 9, -7]]).astype(np.int32)
    cams = cams_for(288, 256)
    d_raw, d_rows = torch.from_numpy(raw).to(cuda), torch.from_numpy(rows).to(cuda)
    d_sw = torch.from_numpy(sw.view(np.uint8)).to(cuda)
    dc = 4 + c + T
    full = canary((len(rows) + 1, dc), torch.float32, cuda)
    assert lib().lavb_lidar_batch(ops._ptr(d_raw), n_raw, c, ops._ptr(d_rows), len(rows), ops._ptr(d_sw), len(sw), ops._hptr(cams), 3,
                                  288, 256, T, ops._ptr(full), ops._stream()) == 0
    want = util.lidar_batch32(raw, rows, sw, cams, 288, 256, T)
    hold_values(full[:-1], want, f"lidar_batch c {c}")
    assert bool(is_canary(full[-1]).all())
    assert not want[rows < 10].any()


def test_lidar_batch_training_shape(cuda):
    """32 samples x 120 000 rows over 3 sweeps of 40 000 raw rows each (the statement is taken per raw row once)"""
    T, c = 3, 4
    raw, sw = lidar_inputs([40000] * 3, c, T, 77, first_row0=0)
    n_raw = len(raw)
    g = torch.Generator().manual_seed(3)
    rows = torch.stack([torch.randperm(n_raw, generator=g) for _ in range(32)]).to(torch.int32)
    rows[5, -1000:] = -1
    cams = cams_for(288, 256)
    out = ops.lidar_batch(torch.from_numpy(raw).to(cuda), rows.to(cuda), torch.from_numpy(sw.view(np.uint8)).to(cuda), cams,
                          (288, 256), T)
    per_raw = util.lidar_batch32(raw, np.arange(n_raw), sw, cams, 288, 256, T)
    r = rows.numpy()
    want = np.where((r >= 0)[..., None], per_raw[np.clip(r, 0, None)], F32(0))
    hold_values(out, want, "lidar_batch training shape")


# ------------------------------------------------------------------------------------------------------------ rejections
def rejections_main(tmp_path):
    cuda = torch.device("cuda:0")
    H, W = 8, 6
    cams = cams_for(H, W)
    null = C.c_void_p(0)
    pts = torch.zeros(64 * 4 + 8, device=cuda)
    sem = torch.zeros(3, 5, H, W, device=cuda)
    out = canary((64 * 8 + 8,), torch.float32, cuda)
    feat = torch.zeros(3 * (H // 2) * (W // 2) * 16 + 8, device=cuda)
    table = torch.zeros(520, device=cuda)
    st = ops._stream()
    hc = ops._hptr(cams)
    R = np.eye(3, dtype=F32)
    sweep = torch.zeros(100 * 4 + 8, device=cuda)
    dst = canary((100 * 7 + 8,), torch.float32, cuda)
    jobs = torch.zeros(72 * 2 + 8, dtype=torch.uint8, device=cuda)
    raw = torch.zeros(100 * 4 + 8, device=cuda)
    rows = torch.zeros(10, dtype=torch.int32, device=cuda)
    sw = torch.zeros(88 + 8, dtype=torch.uint8, device=cuda)
    P = ops._ptr

    def off(t, b):
        return C.c_void_p(t.data_ptr() + b)

    def paint(p=P(pts), s=P(sem), o=P(out), h=hc, n=64, frames=1):
        return lib().lavb_paint_batched(p, frames, n, 4, 256, s, 3, 5, H, W, 0, 5 * H * W, H * W, W, 1, h, 2, o, 8, 512, 4, 4, st)

    def deconv(p=P(pts), f=P(feat), d=P(table), h=hc, o=P(out), dt=capi.F32):
        return lib().lavb_paint_deconv_batched(p, 1, 64, 4, 256, f, dt, 3, 5, H, W, d, h, o, 8, 512, 4, 4, st)

    def stack(s=P(sweep), h=ops._hptr(R), d=P(dst)):
        return lib().lavb_stack_sweep(s, 100, 4, h, 0.0, 0.0, 0, 3, 0, d, st)

    def roof(s=P(sweep), d=P(dst), frames=1, sfs=400, dfs=400, n=100):
        return lib().lavb_roof_filter(s, frames, n, 4, sfs, d, dfs, null, 1, st)

    def sjobs(j=P(jobs), max_n=100):
        return lib().lavb_stack_jobs(j, 2, max_n, 8, 3, 0, st)

    def lb(r=P(raw), o=P(out), s=P(sw), n_rows=10):
        return lib().lavb_lidar_batch(r, 100, 0, P(rows), n_rows, s, 1, hc, 3, H, W, 3, o, st)

    cases = [
        (lambda: paint(p=null), "null"), (lambda: paint(s=null), "null"), (lambda: paint(o=null), "null"),
        (lambda: paint(h=null), "null"), (lambda: paint(p=off(pts, 2)), "aligned"), (lambda: paint(o=off(out, 2)), "aligned"),
        (lambda: paint(s=off(sem, 1)), "aligned"), (lambda: paint(frames=65536), "frames"),
        (lambda: deconv(p=null), "null"), (lambda: deconv(f=null), "null"), (lambda: deconv(d=null), "null"),
        (lambda: deconv(h=null), "null"), (lambda: deconv(f=off(feat, 8)), "aligned"),
        (lambda: deconv(f=off(feat, 4), dt=ops._DT[ops.h16()]), "aligned"), (lambda: deconv(d=off(table, 2)), "aligned"),
        (lambda: deconv(dt=7), "dtype"),
        (lambda: stack(s=null), "null"), (lambda: stack(h=null), "null"), (lambda: stack(d=null), "null"),
        (lambda: stack(d=P(sweep)), "overlaps"), (lambda: stack(d=off(sweep, 4 * 399)), "overlaps"),
        (lambda: stack(s=off(sweep, 2)), "aligned"),
        (lambda: roof(d=P(sweep)), "overlaps"), (lambda: roof(d=off(sweep, 4 * 50)), "overlaps"),
        (lambda: roof(s=null), "null"), (lambda: roof(d=off(dst, 2)), "aligned"),
        (lambda: roof(frames=2, n=50, dfs=100), "overlap"), (lambda: roof(sfs=-1), "bad arguments"),
        (lambda: sjobs(max_n=-1), "bad arguments"), (lambda: sjobs(j=null), "8-byte"), (lambda: sjobs(j=off(jobs, 4)), "8-byte"),
        (lambda: lb(r=off(raw, 2)), "aligned"), (lambda: lb(s=off(sw, 2)), "aligned"), (lambda: lb(o=off(out, 2)), "aligned"),
        (lambda: lb(n_rows=256 * 2 ** 31), "2^31"),
    ]
    seen = []
    ctl_src = torch.zeros(4, 3, device=cuda)
    ctl_dst = torch.empty(4, 3, device=cuda)

    def run():
        seen.clear()
        for fn, cause in cases:
            seen.append((fn(), cause, lib().lavb_last_error().decode()))
        assert lib().lavb_stack_sweep(P(ctl_src), 4, 3, ops._hptr(R), 0.0, 0.0, 0, 0, 0, P(ctl_dst), st) == 0

    launched = kernels(run, tmp_path)
    assert len(launched) == 1 and "stack_kernel" in launched[0][0], launched
    for code, cause, msg in seen:
        assert code != 0 and cause in msg, (cause, code, msg)
    for o in (out, dst):
        assert bool(is_canary(o).all())
    # the zero-size calls are no-ops that need no pointers
    assert lib().lavb_paint_batched(null, 0, 64, 4, 256, null, 3, 5, H, W, 0, 1, 1, 1, 1, null, 2, null, 8, 512, 4, 4, st) == 0
    assert lib().lavb_stack_jobs(null, 2, 0, 8, 3, 0, st) == 0


def test_rejections(cuda, tmp_path):
    """every rejection, in a child process (torch.profiler is started there, as in test_gpu_camera_kernels_contract)"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = (f"import sys; sys.path.insert(0, {root!r}); from tests import test_gpu_paint_stack_contract as t; "
            f"t.rejections_main({str(tmp_path)!r})")
    r = subprocess.run([sys.executable, *(["-s"] if sys.flags.no_user_site else []), "-c", code], cwd=root,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
