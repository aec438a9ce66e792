"""GPU: lavb_det_peaks (ops.det_peaks) against the statement of its whole packed output in tests/test_det_decode_cpu.py, bit for
bit, on scores torch.sigmoid computes on the device: tiny maps, partial 32-pixel tiles, up to 8 classes, max_det 1 / 15 / 64,
min_score 0.1 / 0.2 / 0.5; blobs with fewer peaks than max_det, noise, 6400 strict maxima, tied plateaus, a saturated plateau
of more candidates than the kernel lists, NaN / inf logits and an empty map.  Also: the threshold boundary, repeated calls, a
frame decoded alone, the statement's detections against oracle.lav_ref.det_inference, bit 4 of lavb_eval_batch on the host
filter's boundary cases, and the rejected arguments."""
import ctypes as C

import numpy as np
import pytest
import torch

from lav_b200 import capi, ops
from lav_b200.model_inference import InferModel, peak_filter
from tests import test_det_decode_cpu as D

pytestmark = pytest.mark.gpu

SHAPES = [(1, 1, 1, 2), (2, 7, 7, 2), (3, 31, 45, 1), (2, 33, 97, 3), (1, 321, 319, 8), (3, 320, 320, 2), (64, 320, 320, 2)]
MAPS = ["blobs", "noise", "lattice", "plateaus", "saturated", "nonfinite", "below"]
SPECIAL = [16.7, -16.7, 88.0, -88.0, 104.0, -104.0, float("inf"), float("-inf"), float("nan")]


def logits_of(kind, shape, seed):
    """(B, H, W, ncls) fp32 logits on the CPU."""
    B, H, W, ncls = shape
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    if kind == "blobs":                                 # class c of frame b: (b + c) % 4 blobs, fewer than max_det >= 15
        out = torch.full(shape, -6.0)
        for b in range(B):
            for c in range(ncls):
                for _ in range((b + c) % 4):
                    cx, cy = float(torch.rand(1, generator=g)) * W, float(torch.rand(1, generator=g)) * H
                    amp = 5.0 + float(torch.rand(1, generator=g)) * 8
                    out[b, :, :, c] = torch.maximum(out[b, :, :, c], -6 + amp * torch.exp(-((xx - cx) ** 2 + (yy - cy) ** 2) / 8.0))
        return out
    if kind == "noise":
        return torch.randn(shape, generator=g) * 1.5 - 0.5
    if kind == "lattice":                               # a strict maximum every 4 px (6400 on 320 x 320), all scores distinct
        out = torch.full(shape, -10.0)
        on = (yy % 4 == 0) & (xx % 4 == 0)
        n = int(on.sum())
        for b in range(B):
            for c in range(ncls):
                out[b, :, :, c][on] = -2.5 + 5.0 * torch.randperm(n, generator=g).float() / max(n, 1)
        return out
    if kind == "plateaus":                              # 2 to 4 pixels of one value inside a 3 x 3 square, every 8 px
        out = torch.full(shape, -10.0)
        ny, nx = (H + 7) // 8, (W + 7) // 8
        rank = torch.rand(B, ny, nx, ncls, 9, generator=g).argsort(-1).argsort(-1)
        k = torch.randint(2, 5, (B, ny, nx, ncls, 1), generator=g)
        v = torch.randn(B, ny, nx, ncls, generator=g) * 2
        bi, yi, xi, ci, cell = (rank < k).nonzero(as_tuple=True)
        out[bi, (yi * 8 + cell // 3).clamp(max=H - 1), (xi * 8 + cell % 3).clamp(max=W - 1), ci] = v[bi, yi, xi, ci]
        return out
    if kind == "saturated":                             # class 0: logit 30 (score exactly 1.0) on up to 100 x 100 pixels
        out = torch.randn(shape, generator=g) * 1.5 - 0.5
        out[:, 20:120, 10:110, 0] = 30.0
        return out
    if kind == "nonfinite":
        out = torch.randn(shape, generator=g) * 1.5
        flat = out.view(-1)
        idx = torch.randperm(flat.numel(), generator=g)[:max(len(SPECIAL), flat.numel() // 4000)]   # ~3 NaN per 320 x 320
        flat[idx] = torch.tensor(SPECIAL)[torch.arange(len(idx)) % len(SPECIAL)]
        return out
    assert kind == "below"
    return torch.full(shape, -1.5) - torch.rand(shape, generator=g)      # sigmoid < 0.19


def maps_of(kind, shape, seed):
    B, H, W, _ = shape
    g = torch.Generator().manual_seed(seed + 1)
    return logits_of(kind, shape, seed), torch.randn(B, H, W, 2, generator=g), torch.randn(B, H, W, 2, generator=g)


def same(a, b):
    """bit for bit, NaN matching NaN."""
    a, b = a.cpu(), b.cpu()
    if a.shape != b.shape or not torch.equal(a.isnan(), b.isnan()):
        return False
    keep = ~a.isnan()
    return torch.equal(a[keep].view(torch.int32), b[keep].view(torch.int32))


def run(cuda, logit, box, ori, min_score, max_det):
    return ops.det_peaks(logit.to(cuda).contiguous(), box.to(cuda), ori.to(cuda), min_score=min_score, max_det=max_det)


def statement(cuda, logit, box, ori, min_score, max_det):
    return D.peaks_statement(torch.sigmoid(logit.to(cuda)).cpu(), box, ori, min_score, max_det)


CASES = [(shape, kind, (1, 15, 64)[(i + j) % 3], (0.1, 0.2, 0.5)[(i + 2 * j) % 3])
         for i, shape in enumerate(SHAPES) for j, kind in enumerate(MAPS)]


@pytest.mark.parametrize("shape,kind,max_det,min_score", CASES, ids=[f"{'x'.join(map(str, s))}-{k}-k{m}-t{t}" for s, k, m, t in CASES])
def test_det_peaks_equals_the_statement(cuda, shape, kind, max_det, min_score):
    """The whole packed tensor bit for bit; a second call identical; each of (up to) three frames decoded alone identical."""
    seed = sum(shape) * 7 + MAPS.index(kind)
    logit, box, ori = maps_of(kind, shape, seed)
    want = statement(cuda, logit, box, ori, min_score, max_det)
    got = run(cuda, logit, box, ori, min_score, max_det)
    assert same(got, want), (np.argwhere(~(got.cpu() == want) & ~(got.cpu().isnan() & want.isnan())).T[:, :8])
    assert same(run(cuda, logit, box, ori, min_score, max_det), got)
    B = shape[0]
    for b in sorted({0, B // 2, B - 1}):
        assert same(run(cuda, logit[b:b + 1], box[b:b + 1], ori[b:b + 1], min_score, max_det), got[b:b + 1])
    if kind == "blobs":                                 # padding: some (frame, class) have no peak at all
        pad = want[:, 0] == -1e5
        assert pad.any() and bool((want.permute(0, 2, 1)[pad][:, :6] == torch.tensor(D.PAD)).all())
    if kind == "saturated" and shape[1] * shape[2] > 8192:
        assert bool((want[:, 0, :max_det] == 1.0).all())            # the plateau's first pixels in flat order


@pytest.mark.parametrize("shape,kind,min_score", [(SHAPES[5], "blobs", 0.2), (SHAPES[5], "noise", 0.1), (SHAPES[5], "nonfinite", 0.2),
                                                   (SHAPES[5], "saturated", 0.5), (SHAPES[6], "noise", 0.2)])
def test_statement_detections_equal_det_inference(cuda, shape, kind, min_score):
    """What the host filter keeps of the statement's first 15 columns is the reference's det_inference on the same device
    scores, as sets per (frame, class); where the 15th and 16th candidates tie, only the peaks ranked above the tied score are
    compared (torch.topk's order among equal values is unspecified)."""
    logit, box, ori = maps_of(kind, shape, 11)
    s = torch.sigmoid(logit.to(cuda)).cpu()
    packed = D.peaks_statement(s, box, ori, min_score, 16)
    mine = InferModel.decode_packed(D.STUB, packed[:, :, [j for c in range(2) for j in range(16 * c, 16 * c + 15)]], 2, min_score)
    ref = D.reference_dets(s, box, ori, min_score)
    compared = 0
    for b in range(shape[0]):
        for c in range(2):
            col = packed[b, 0, 16 * c:16 * c + 16]
            if col[14] == col[15] and col[14] > -1e5:
                keep = lambda dets: {d for d in dets if float(s[b, d[1], d[0], c]) > float(col[14])}
                assert keep(mine[b][c]) == keep(ref[b][c]), (b, c)
            else:
                assert set(mine[b][c]) == set(ref[b][c]), (b, c)
                compared += len(ref[b][c])
    assert compared > 0


def boundary_logits(cuda, p):
    """fp32 logits within 4096 steps of log(p / (1 - p)) whose device torch.sigmoid is float32(p), and the nearest three below
    and above it."""
    x0 = np.float32(np.log(p / (1 - p)))
    h = max(float(np.spacing(x0)), 2.0 ** -30)                     # around 0, denormal steps would never leave sigmoid = 0.5
    xs = np.unique((float(x0) + np.arange(-4096, 4097) * h).astype(np.float32))
    sv = torch.sigmoid(torch.from_numpy(xs).to(cuda)).cpu().numpy()
    t = np.float32(p)
    return xs[sv == t], xs[sv < t][-3:], xs[sv > t][:3]


@pytest.mark.parametrize("min_score", [0.1, 0.2, 0.5])
def test_threshold_boundary(cuda, min_score):
    """Scores exactly float32(min_score) are not candidates; the nearest scores above are, and below are not."""
    at, below, above = boundary_logits(cuda, min_score)
    assert len(below) == len(above) == 3
    if min_score == 0.5:
        assert 0.0 in at.tolist()                                   # sigmoid(0) = 1 / 2 exactly
    if min_score != 0.1:                                            # at 0.1 a logit step moves the score by ~3 ulps
        assert len(at) > 0
    vals = np.concatenate([at[:8], below, above]).astype(np.float32)
    logit = torch.full((1, 64, 64, 2), -20.0)
    for i, v in enumerate(vals):
        logit[0, 4 + 8 * (i // 7), 4 + 8 * (i % 7), i % 2] = float(v)
    box, ori = torch.randn(1, 64, 64, 2), torch.randn(1, 64, 64, 2)
    got = run(cuda, logit, box, ori, min_score, 32)
    assert same(got, statement(cuda, logit, box, ori, min_score, 32))
    scores = got[0, 0].cpu()
    assert int((scores > -1e5).sum()) == len(above)
    assert bool((scores[scores > -1e5] > np.float32(min_score)).all())


def test_scores_are_torch_sigmoid_on_the_device(cuda):
    """One-pixel maps with min_score -1 emit every pixel: each score is the device torch.sigmoid of its logit, bit for bit, over
    the whole range, where fp32 sigmoid saturates to 1 (16.7, 88, 104, inf), turns denormal (-88) or 0 (-104, -inf), and NaN."""
    g = torch.Generator().manual_seed(0)
    vals = torch.cat([torch.tensor(SPECIAL + [16.6, 16.8, 87.3, -87.3, -103.0, 0.0, -0.0]), torch.linspace(-110, 110, 4001),
                      torch.randn(4000, generator=g) * 8])
    n = len(vals)
    logit = vals.view(n, 1, 1, 1)
    box, ori = torch.randn(n, 1, 1, 2, generator=g), torch.randn(n, 1, 1, 2, generator=g)
    got = run(cuda, logit, box, ori, -1.0, 1)
    assert same(got[:, 0, 0], torch.sigmoid(logit.to(cuda)).view(-1))
    assert same(got, statement(cuda, logit, box, ori, -1.0, 1))
    assert bool((got[:, 0, 0] == 0).any()) and bool(((got[:, 0, 0] > 0) & (got[:, 0, 0] < 1.2e-38)).any())


def test_eval_batch_survivors_equal_peak_filter(cuda):
    """Bit 4 of lavb_eval_batch's flags is peak_filter's keep on the host filter's boundary cases (fp32 score threshold, size
    threshold, window edges, NaN score, padding) and on the kernel's own output."""
    packed = np.concatenate([D.packed_of(D.FRAMES), D.packed_of([[(c, v, 60 + 10 * i, 200 + 20 * c, 1, 1) for c in range(2)
                                                                  for i, v in enumerate([D.S2, D.S2_UP, D.S2_DOWN, float("nan"), -1e5])]])])
    logit, box, ori = maps_of("noise", (4, 320, 320, 2), 5)
    packed = np.concatenate([packed, run(cuda, logit, box * 0.5, ori, 0.2, 15).cpu().numpy()])
    B = len(packed)
    seg = torch.zeros((B, 320, 320, 3), device=cuda)
    gt = torch.zeros((B, 3, 320, 320), dtype=torch.uint8, device=cuda)
    plan, ego = torch.zeros((B, 20, 2), device=cuda), torch.zeros((B, 21, 2), device=cuda)
    actors = torch.zeros((0, 6), device=cuda)
    v = ops.eval_views(ops.eval_batch(seg, gt, torch.from_numpy(packed).to(cuda), actors, np.zeros(B + 1, np.int32), plan, ego).cpu(),
                       B, 30)
    keep, *_ = peak_filter(packed, D.PPM)
    assert np.array_equal((v["flags"].numpy() & 16) != 0, keep)
    assert keep[:4].sum() == sum(len(k) for k in D.KEPT) and keep[5:].any()


def test_det_peaks_rejects_bad_arguments_with_lavb_error_and_writes_nothing(cuda):
    """Rejected calls (checked on the host, before any launch) return non-zero and leave the output as it was; batch = 0
    succeeds and writes nothing."""
    lib = capi.lib()
    big = (1, 4097, 4096, 1)                                        # h * w > 2^24; the buffers are large enough either way
    center = torch.full(big, -5.0, device=cuda)
    box = torch.zeros(big[:3] + (2,), device=cuda)
    ori = torch.zeros_like(box)
    packed = torch.full((4, 7, 8 * 65), 123.0, device=cuda)
    ws = torch.zeros(lib.lavb_det_peaks_workspace_bytes(4, 9), dtype=torch.uint8, device=cuda)
    p = lambda t: C.c_void_p(t.data_ptr())
    bad = [dict(ncls=0), dict(ncls=9), dict(max_det=0), dict(max_det=65), dict(h=0), dict(w=0), dict(h=0, w=0), dict(batch=-1),
           dict(h=4097, w=4096)]
    for kw in bad:
        a = dict(batch=1, h=16, w=16, ncls=1, max_det=15)
        a.update(kw)
        rc = lib.lavb_det_peaks(p(center), p(box), p(ori), a["batch"], a["h"], a["w"], a["ncls"], 0.2, a["max_det"], p(packed),
                                p(ws), C.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc != 0, kw
    assert lib.lavb_det_peaks(p(center), p(box), p(ori), 0, 16, 16, 2, 0.2, 15, p(packed), p(ws),
                              C.c_void_p(torch.cuda.current_stream().cuda_stream)) == 0
    torch.cuda.synchronize()
    assert bool((packed == 123.0).all())
    ok = ops.det_peaks(center[:, :16, :16].contiguous(), box[:, :16, :16].contiguous(), ori[:, :16, :16].contiguous())
    assert ok.shape == (1, 7, 15)
    for b, o in ((box[:, :16, :15].contiguous(), ori[:, :16, :16].contiguous()),
                 (box[:, :16, :16].contiguous(), torch.zeros((1, 16, 16, 3), device=cuda))):
        with pytest.raises(capi.LavbError):
            ops.det_peaks(center[:, :16, :16].contiguous(), b, o)
