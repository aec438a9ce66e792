"""CPU: the detection decode's contract.  The statement of lavb_det_peaks' whole packed output (sigmoid scores -> 7x7 NMS ->
candidates -> ranked columns -> padding), checked against the reference's extract_peak / det_inference; and the host filter
(model_inference.peak_filter, InferModel.decode_packed) against the reference's per-peak loop at its boundaries: the fp32
score threshold, the class-1 size threshold, the ego window's edges and a NaN score."""
import numpy as np
import torch
import torch.nn.functional as F

from lav_b200.model_inference import InferModel, peak_filter, score_kept
from oracle import lav_ref as O

PPM = 4
STUB = type("S", (), {"pixels_per_meter": PPM})()
PAD = (-1e5, 0.0, 0.0, 0.0, 0.0, 0.0)           # a column past the last candidate, then W


# ---------------------------------------------------------------------------------------------------- the statement
def peaks_statement(s, box, ori, min_score=0.2, max_det=15):
    """lavb_det_peaks on scores s (B, H, W, ncls) fp32 (torch.sigmoid of the logits), box / ori (B, H, W, 2) fp32
    -> packed (B, 7, ncls * max_det).  A candidate is a pixel whose 7x7 window maximum (max_pool2d: -inf padding, NaN
    propagating) is not larger than it, with s > float32(min_score) in fp32, or a NaN pixel.  Candidates rank NaN first, then
    by descending s, ties to the lower flat index; the max_det first fill the columns, the rest is padding."""
    B, H, W, ncls = s.shape
    plane = s.permute(0, 3, 1, 2).reshape(B * ncls, 1, H, W).float()
    peak = ~(F.max_pool2d(plane, 7, 1, 3) > plane)
    flat = plane.reshape(B * ncls, H * W)
    cand = (peak.reshape(B * ncls, H * W) & (flat > torch.tensor(min_score, dtype=torch.float32))) | flat.isnan()
    rank = torch.where(flat.isnan(), torch.full_like(flat, 2.0), flat)           # scores are in [0, 1]: NaN ranks first
    rank = torch.where(cand, rank, torch.full_like(flat, -1.0))
    order = torch.sort(rank, dim=1, descending=True, stable=True).indices[:, :max_det]   # stable: ties keep the flat order
    n = torch.minimum(cand.sum(1), torch.tensor(max_det))
    packed = torch.empty((B, ncls, 7, max_det), dtype=torch.float32)
    packed[:, :, :6] = torch.tensor(PAD).view(1, 1, 6, 1)
    packed[:, :, 6] = float(W)
    maps = torch.cat([box, ori], 3).reshape(B, H * W, 4)
    for m in range(B * ncls):
        b, c, k = m // ncls, m % ncls, int(n[m])
        loc = order[m, :k]
        packed[b, c, 0, :k] = flat[m, loc]
        packed[b, c, 1, :k] = loc.float()
        packed[b, c, 2:6, :k] = maps[b, loc].T
    return packed.permute(0, 2, 1, 3).reshape(B, 7, ncls * max_det)


def reference_dets(s, box, ori, min_score=0.2):
    """oracle.lav_ref.det_inference per frame on NHWC maps (its extract_peak keeps 15 peaks)."""
    return [O.det_inference(s[b].permute(2, 0, 1), box[b].permute(2, 0, 1), ori[b].permute(2, 0, 1), PPM, min_score)
            for b in range(s.shape[0])]


def f32(v):
    return float(np.float32(v))


def step(v, n):
    """the float32 n steps from float32(v)."""
    x = np.float32(v)
    for _ in range(abs(n)):
        x = np.nextafter(x, np.float32(np.inf if n > 0 else -np.inf))
    return float(x)


def test_statement_equals_the_reference_on_distinct_scores():
    """Distinct scores: the statement's columns that pass the host filter are det_inference's detections, in its order."""
    g = torch.Generator().manual_seed(3)
    B, H, W = 2, 320, 320
    logit = torch.randn(B, H, W, 2, generator=g) * 2 - 1
    logit[0, :, :, 1] = -9.0                                            # a class with nothing above the threshold
    s = torch.sigmoid(logit)
    box, ori = torch.rand(B, H, W, 2, generator=g) * 3, torch.randn(B, H, W, 2, generator=g)
    for ms in (0.1, 0.2, 0.5):
        packed = peaks_statement(s, box, ori, ms, 15)
        want = reference_dets(s, box, ori, ms)
        assert InferModel.decode_packed(STUB, packed, 2, ms) == want
        assert sum(len(d) for w in want for d in w) >= 5


def test_statement_on_plateaus_nan_and_padding():
    """Known answers: tied pixels inside one window all count, in flat order; a NaN is a candidate ranked first and keeps
    its neighbours from being suppressed; the columns past the last candidate are padding."""
    H, W = 12, 20
    s = torch.full((1, H, W, 1), 0.05)
    s[0, 2, 3, 0] = s[0, 3, 4, 0] = s[0, 2, 5, 0] = 0.7                 # three tied pixels in one window
    s[0, 3, 2, 0] = 0.6                                                 # suppressed by them
    s[0, 9, 15, 0] = float("nan")
    s[0, 9, 13, 0], s[0, 8, 16, 0] = 0.3, 0.9                           # 0.3 beside the larger 0.9, but a NaN shares both windows
    box, ori = torch.arange(H * W * 2.).view(1, H, W, 2), -torch.arange(H * W * 2.).view(1, H, W, 2)
    p = peaks_statement(s, box, ori, 0.2, 7)
    locs = [9 * W + 15, 8 * W + 16, 2 * W + 3, 2 * W + 5, 3 * W + 4, 9 * W + 13]
    assert torch.isnan(p[0, 0, 0]) and p[0, 0, 1:6].tolist() == [f32(0.9), f32(0.7), f32(0.7), f32(0.7), f32(0.3)]
    assert p[0, 1, :6].tolist() == locs
    assert p[0, 2, :6].tolist() == [2.0 * i for i in locs] and p[0, 5, :6].tolist() == [-(2.0 * i + 1) for i in locs]
    assert p[0, :6, 6].tolist() == list(PAD) and p[0, 6].tolist() == [W] * 7
    # without the NaN, 0.9 suppresses 0.3 and the NaN pixel's own value (0.05) is below the threshold
    s[0, 9, 15, 0] = 0.05
    p = peaks_statement(s, box, ori, 0.2, 7)
    assert p[0, 1, :4].tolist() == locs[1:5] and p[0, 0, 4:].tolist() == [-1e5] * 3


def test_statement_threshold_is_fp32():
    s = torch.full((1, 30, 30, 1), 0.0)
    vals = [step(0.2, -1), f32(0.2), step(0.2, 1)]
    for i, v in enumerate(vals):
        s[0, 5, 5 + 8 * i, 0] = v
    p = peaks_statement(s, torch.zeros(1, 30, 30, 2), torch.zeros(1, 30, 30, 2), 0.2, 3)
    assert p[0, 0].tolist() == [vals[2], -1e5, -1e5]


# ---------------------------------------------------------------------------------------------------- the host filter
def reference_loop(packed, ppm=PPM, min_score=0.2, ncls=2):
    """det_inference's per-peak loop (model_inference.py:98-121, oracle.lav_ref.det_inference) over packed columns: each
    score a 0-d fp32 tensor compared with the Python float, the box and orientation read as Python floats."""
    packed = np.asarray(packed, np.float32)
    W, nd = int(packed[0, 6, 0]), packed.shape[2] // ncls
    out = []
    for b in range(packed.shape[0]):
        dets = []
        for i in range(ncls):
            det = []
            for j in range(i * nd, (i + 1) * nd):
                s = torch.tensor(packed[b, 0, j])
                if not s > min_score:
                    continue
                loc = int(packed[b, 1, j])
                x, y = loc % W, loc // W
                w, h = float(packed[b, 2, j]), float(packed[b, 3, j])
                cos, sin = float(packed[b, 4, j]), float(packed[b, 5, j])
                if i == 1 and max(w, h) < 0.1 * ppm:
                    continue
                dist = np.linalg.norm([x - 160, y - 280])
                if dist <= 2 or dist >= 30 * ppm:
                    continue
                det.append((x, y, w, h, cos, sin))
            dets.append(det)
        out.append(dets)
    return out


# peaks (class, score, x, y, w, h) of four frames, each isolated in its 7x7 window and in descending score per class
S2, S2_UP, S2_DOWN, S4, S4_UP, S4_DOWN = f32(0.2), step(0.2, 1), step(0.2, -1), f32(0.4), step(0.4, 1), step(0.4, -1)
FRAMES = [
    [(0, 0.9, 100, 200, 1, 1), (0, S2_UP, 110, 200, 1, 1), (0, S2, 120, 200, 1, 1), (0, S2_DOWN, 130, 200, 1, 1),
     (1, 0.9, 100, 220, 1, 1), (1, S2_UP, 110, 220, 1, 1), (1, S2, 120, 220, 1, 1), (1, S2_DOWN, 130, 220, 1, 1)],
    [(0, 0.6, 100, 240, 0.01, 0.02),                                                          # class 0: no size filter
     (1, 0.9, 100, 200, S4, 0.1), (1, 0.8, 110, 200, 0.1, S4), (1, 0.7, 120, 200, S4_DOWN, S4_DOWN),
     (1, 0.6, 130, 200, S4_UP, 0.0), (1, 0.5, 140, 200, S4_DOWN, 0.0), (1, 0.4, 150, 200, 0.0, S4_UP)],
    [(0, 0.9, 160, 282, 1, 1), (0, 0.8, 160, 270, 1, 1), (0, 0.7, 88, 184, 1, 1), (0, 0.6, 256, 208, 1, 1),  # d = 2, 10, 120, 120
     (1, 0.9, 162, 280, 1, 1), (1, 0.7, 88, 185, 1, 1), (1, 0.6, 158, 279, 1, 1)],                      # d = 2, 119.2, 2.24
    [(0, float("nan"), 100, 200, 1, 1), (0, 0.5, 120, 200, 1, 1), (0, 0.4, 163, 280, 1, 1),                 # d = 3
     (1, float("nan"), 100, 220, 1, 1), (1, float("nan"), 120, 220, 1, 1), (1, 0.3, 140, 220, 1, 1)],
]
KEPT = [  # (class, x, y) det_inference keeps, in order
    [(0, 100, 200), (0, 110, 200), (1, 100, 220), (1, 110, 220)],
    [(0, 100, 240), (1, 100, 200), (1, 110, 200), (1, 130, 200), (1, 150, 200)],
    [(0, 160, 270), (1, 88, 185), (1, 158, 279)],
    [(0, 120, 200), (0, 163, 280), (1, 140, 220)],
]


def packed_of(frames, n_det=15, w=320):
    """frames of peaks -> (B, 7, 2 * n_det), the unused columns padded as lavb_det_peaks pads them."""
    p = np.zeros((len(frames), 7, 2 * n_det), np.float32)
    p[:, :6] = np.array(PAD, np.float32)[:, None]
    p[:, 6] = w
    for b, peaks in enumerate(frames):
        used = [0, 0]
        for c, s, x, y, bw, bh in peaks:
            p[b, :6, c * n_det + used[c]] = (s, y * w + x, bw, bh, 0.25 * x, -0.5 * y)
            used[c] += 1
    return p


def maps_of(frames, h=320, w=320):
    """the same peaks as maps: heat (B, 2, h, w) already sigmoided, 0 elsewhere; size / orientation (B, 2, h, w)."""
    heat, size, ori = torch.zeros(len(frames), 2, h, w), torch.zeros(len(frames), 2, h, w), torch.zeros(len(frames), 2, h, w)
    for b, peaks in enumerate(frames):
        for c, s, x, y, bw, bh in peaks:
            heat[b, c, y, x] = s
            size[b, :, y, x] = torch.tensor([bw, bh])
            ori[b, :, y, x] = torch.tensor([0.25 * x, -0.5 * y])
    return heat, size, ori


def test_host_filter_equals_the_reference_loop_at_its_boundaries():
    packed = packed_of(FRAMES)
    got = InferModel.decode_packed(STUB, torch.from_numpy(packed))
    assert got == reference_loop(packed)
    assert [[(c, x, y) for c in range(2) for x, y, *_ in d[c]] for d in got] == KEPT
    keep, x, y, cls = peak_filter(packed, PPM)
    assert [[(int(cls[j]), int(x[b, j]), int(y[b, j])) for j in np.nonzero(keep[b])[0]] for b in range(len(FRAMES))] == KEPT
    assert not keep[:, 14].any() and not keep[:, 29].any()                  # padding never survives


def test_host_filter_through_maps_equals_det_inference():
    """The same peaks drawn as maps: pack_peaks -> decode_packed is det_inference on them, and so is the decode of the
    hand-built packed array."""
    heat, size, ori = maps_of(FRAMES)
    want = [O.det_inference(heat[b], size[b], ori[b], PPM) for b in range(len(FRAMES))]
    assert InferModel.decode_packed(STUB, InferModel.pack_peaks(heat, size, ori)) == want
    assert InferModel.decode_packed(STUB, torch.from_numpy(packed_of(FRAMES))) == want


def test_score_threshold_is_compared_in_fp32():
    for ms in (0.1, 0.2, 0.5, 0.3):
        v = [step(ms, -1), f32(ms), step(ms, 1), float("nan"), -1e5]
        assert score_kept(np.array(v, np.float32), ms).tolist() == [False, False, True, False, False]
        assert score_kept(v, ms).tolist() == [bool(torch.tensor(np.float32(s)) > ms) for s in v]
