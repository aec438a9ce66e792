"""Shared builders for the tests: seeded weights (identical in the pin script) and inputs."""
import itertools
import json
import math
import os

import numpy as np
import torch

from lav_b200 import synth

GRID = dict(min_x=-10, max_x=70, min_y=-40, max_y=40)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def lidar_model(device=None):
    from lav_b200.lidar import LiDARModel
    m = LiDARModel(num_input=16, num_features=[64, 64], backbone="cnn", pixels_per_meter=4, **GRID).eval()
    sd = synth.fill_state_dict_(m.state_dict())
    m.load_state_dict(sd)
    if device is not None:
        m = m.to(device)
    return m, {k: v.clone() for k, v in sd.items()}


def seg_model(device=None, real=False):
    from lav_b200.rgb import RGBSegmentationModel
    m = RGBSegmentationModel([4, 6, 7, 10]).eval()
    if real:
        sd = torch.load(os.path.join(ROOT, "oracle", "_ref", "seg_1.state_dict.pt"), map_location="cpu")
    else:
        sd = synth.fill_state_dict_(m.state_dict())
    m.load_state_dict(sd)
    if device is not None:
        m = m.to(device)
    return m, {k: v.clone() for k, v in sd.items()}


def have_real_seg():
    return os.path.exists(os.path.join(ROOT, "oracle", "_ref", "seg_1.state_dict.pt"))


def pillar_clouds():
    return [synth.stacked_lidar(2000, tag="pp0"), synth.stacked_lidar(1500, tag="pp1")]


def paint_inputs():
    gold = np.load(os.path.join(ROOT, "tests", "golden", "paint.npz"))
    lidar = torch.cat([synth.lidar_sweep(8192, tag="paint"), torch.from_numpy(gold["edge"])]).contiguous()
    return lidar, synth.sem_probs(tag="paint"), gold


def rel_err(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def crop_ref64(feats_nchw, frame_idx, theta, S, padding="zeros"):
    """lavb_crop_bilinear in float64: frame indices clamped to [0, B) as the kernel clamps them, then
    F.affine_grid(theta, align_corners=True) + F.grid_sample(bilinear, align_corners=True).  feats (B,C,H,W), frame_idx (K,),
    theta (K,2,3) -> (K,C,S,S) float64.  The bilinear weights are >= 0, so crop_ref64(|f|) is the per-element sum |w f| of
    the forward.  ``padding`` other than the kernel's "zeros" is for error bounds (tests/test_gpu_crop_contract.py)."""
    import torch.nn.functional as F
    B, C = feats_nchw.shape[:2]
    fi = frame_idx.long().cpu().clamp(0, B - 1)
    grid = F.affine_grid(theta.double().cpu(), [theta.shape[0], C, S, S], align_corners=True)
    return F.grid_sample(feats_nchw.double().cpu()[fi], grid, mode="bilinear", padding_mode=padding, align_corners=True)


def crop_ref64_adjoint(gout_nchw, frame_idx, theta, feat_shape):
    """the adjoint of crop_ref64 (the crop's gradient with respect to the (B,C,H,W) map) by float64 autograd through the same
    call: gout (K,C,S,S) -> (B,C,H,W) float64.  Applied to |gout| it gives the per-element sum |w g| of the backward."""
    f = torch.zeros(feat_shape, dtype=torch.float64, requires_grad=True)
    out = crop_ref64(f, frame_idx, theta, gout_nchw.shape[-1])
    return torch.autograd.grad(out, f, gout_nchw.double().cpu())[0]


def seg_logit_err(got_prob, ref_feats, sd):
    """error of the seg head measured BEFORE its sigmoid, as a fraction of the logit scale: the reference module returns
    sigmoid(logits) with logits of O(30-90) on seeded weights, so a probability-space max-norm would measure the sigmoid's slope.
    ref_feats: oracle features (B,384,h,w); got_prob: our sigmoid output (B,3,H,W).  Compared where our sigmoid is invertible
    (|reference logit| < 10), normalised by max |reference logit|."""
    from oracle import lav_ref as O
    with torch.no_grad():
        ref_logit = O.head(sd, ref_feats, "seg_head.", sigmoid=False)
    got_logit = torch.logit(got_prob.double().cpu().clamp(1e-9, 1 - 1e-9))
    live = ref_logit.abs() < 10
    assert float(live.float().mean()) > 0.05
    return float((got_logit - ref_logit.double())[live].abs().max() / ref_logit.abs().max())


# ----------------------------------------------------------------------------------------------------- pillar encoders
U32, U16 = 2.0 ** -24, 2.0 ** -11          # unit roundoff of fp32 and of IEEE half


def gamma(n, u=U32):
    return n * u / (1 - n * u)


def round_h16(x):
    """x -> the nearest IEEE half value (ties to even), saturating at +-65504 as cvt.rn.satfinite does; NaN stays NaN."""
    return x.float().clamp(-65504, 65504).half().to(x.dtype)


def _relu(v):
    return torch.where(v > 0, v, torch.zeros((), dtype=v.dtype, device=v.device))        # NaN -> 0, as fmaxf(v, 0)


def pillar_locate(x, y, grid):
    """The encoders' grid location, bit for bit: the half-open window test on the raw fp32 x, y, then
    xi = trunc(fp32(fp32(x - min_x) * ppm)), yi likewise.  -> keep (bool), xi, yi (int64; meaningless where not kept)."""
    mn_x, mx_x, mn_y, mx_y, ppm = (torch.tensor(np.float32(v), device=x.device) for v in grid[:5])
    keep = (x >= mn_x) & (x < mx_x) & (y >= mn_y) & (y < mx_y)
    xs, ys = torch.where(keep, x, mn_x), torch.where(keep, y, mn_y)
    return keep, ((xs - mn_x) * ppm).long(), ((ys - mn_y) * ppm).long()


def pillar_origins(grid):
    """fp32(fp32(i / ppm) + min) for i = 0 .. max(nx, ny), per axis, as float64: the kernels' cell-origin terms."""
    mn_x, _, mn_y, _, ppm, nx, ny = grid
    i = np.arange(max(nx, ny) + 1, dtype=np.float32)
    q = i / np.float32(ppm)
    return (torch.from_numpy((q + np.float32(mn_x)).astype(np.float64)), torch.from_numpy((q + np.float32(mn_y)).astype(np.float64)))


def pillar_forward_ref64(pts, starts, counts, grid, w1, s1, t1, w2, s2, t2, mode, parts="all"):
    """lavb_pillar_forward (mode "fp32") and lavb_pillar_forward_sorted (mode "sorted": fp32 canvas, "sorted_h16": h16 canvas)
    stated in float64, on pts' device.  pts: 2-D fp32 rows (>= 11 columns used); cloud b = rows [starts[b], +counts[b]).
    -> (canvas (B, ny, nx, 64) float64, bound (B, ny, nx, 64) float64): every correct encoder output c satisfies
    |c - canvas| <= bound element-wise, for finite inputs whose fp32 sums stay finite.

    The statement:
      * grid location in fp32, bit-exact (pillar_locate); a pillar is (b, xi, yi) before any clamp; its cell is
        row = clamp(ny-1-xi, 0, ny-1), col = clamp(yi, 0, nx-1);
      * decorated row [pt(11) | xyz - centroid | x - ox(yi) | y - oy(xi)] with the exact centroid in fp64 and the fp32
        cell origins of pillar_origins;
      * the MLP in fp64 on the operands as each encoder reads them: fp32 weights, except that "sorted" layer 2 reads w2 and
        the hidden activations (after affine and ReLU) rounded to half (saturating); ReLU maps NaN to 0;
      * each cell takes the per-channel max over the rows of ALL pillars that clamp onto it (0 for an empty cell).  This is
        the header's rule; oracle/lav_ref.pillar_net assigns one pillar's max per cell (indexed assignment, last write wins);
      * "sorted_h16" rounds the cell value to half once, saturating.

    The bound, an fp64 pass of absolute values through the same MLP (u = 2^-24, u_h = 2^-11, gamma_n = n u / (1 - n u)):
      * centroid: the sums are float atomics in any order, so per pillar of n points and axis the kernel's centroid is
        within gamma_(n+1) sum|x_i| / n of the exact mean (summation, division); the subtraction adds u |f|;
      * cell-origin columns: u |f| (one fp32 subtraction; the origin itself is exact);
      * layer 1, "fp32": a 16-term fp32 FMA chain, gamma_16 sum_k |f_k w_k|; "sorted": f and w are split into half hi + lo
        (|x - hi - lo| <= 2^-22 |x| + 2^-25 absolute, from half subnormals) and lo*lo is dropped, 3 * 2^-22 |f||w| +
        2^-24 (|f| + |w|) per product, and the three MMAs accumulate in fp32 on the tensor cores, which is not IEEE
        round-to-nearest: bounded generously by 2^-16 sum |f_k w_k| (16x gamma_16);
      * each affine is one fmaf: |s| times the propagated error plus u (|s a| + |t|); ReLU and max are 1-Lipschitz;
      * "sorted" hidden activations: the kernel rounds its own fp32 value to half, so the two roundings can land one half
        ulp apart at a tie: + 2^-10 (|h| + e) + 2^-24 on each hidden value.  w2 is read rounded to half by both, exactly;
      * layer 2: the propagated error sum_k e_k |w2_jk| plus gamma_64 sum_k |h_k w2_jk| ("fp32", a 64-term FMA chain) or
        2^-16 sum_k |h_k w2_jk| ("sorted", tensor-core accumulation as above);
        * "sorted_h16": one final half rounding, 2^-10 (|c| + e) + 2^-24.
    A row whose decorated values hold a NaN is exactly relu(t2) in both the statement and the encoders: its bound is u |t2|.
    parts="centroid" bounds instead the difference between two calls on the same input, which differ only in the order of
    the centroid sums: 0 on the rows of pillars of 1 or 2 points (their fp32 sums do not depend on the order, so those rows
    are bit-identical), twice the row bound on the others, and the final half rounding only where that is not 0.
    """
    assert mode in ("fp32", "sorted", "sorted_h16") and parts in ("all", "centroid")
    dev = pts.device
    mn_x, mx_x, mn_y, mx_y, ppm, nx, ny = grid
    B = len(counts)
    rows = torch.cat([torch.arange(int(s), int(s) + int(c), dtype=torch.int64) for s, c in zip(starts, counts)] +
                     [torch.zeros(0, dtype=torch.int64)]).to(dev)
    bidx = torch.cat([torch.full((int(c),), b, dtype=torch.int64) for b, c in enumerate(counts)] +
                     [torch.zeros(0, dtype=torch.int64)]).to(dev)
    p = pts[rows, :11]
    keep, xi, yi = pillar_locate(p[:, 0], p[:, 1], grid)
    p, xi, yi, bidx = p[keep], xi[keep], yi[keep], bidx[keep]
    canvas = torch.zeros((B * ny * nx, 64), dtype=torch.float64, device=dev)
    bound = torch.zeros_like(canvas)
    occupied = torch.zeros((B * ny * nx, 1), dtype=torch.bool, device=dev)
    if len(p) > 0:
        key = (bidx * (nx + 1) + xi) * (ny + 1) + yi
        _, inv = torch.unique(key, return_inverse=True)
        npil = int(inv.max()) + 1
        p64 = p.double()
        xyz = p64[:, :3]
        n = torch.zeros(npil, dtype=torch.float64, device=dev).index_add_(0, inv, torch.ones_like(xyz[:, 0]))[:, None]
        mean = torch.zeros((npil, 3), dtype=torch.float64, device=dev).index_add_(0, inv, xyz) / n
        absmean = torch.zeros((npil, 3), dtype=torch.float64, device=dev).index_add_(0, inv, xyz.abs()) / n
        ox, oy = (o.to(dev) for o in pillar_origins(grid))
        f = torch.cat([p64, xyz - mean[inv], p64[:, :1] - ox[yi][:, None], p64[:, 1:2] - oy[xi][:, None]], 1)
        e = torch.zeros_like(f)
        e[:, 11:14] = gamma(n + 1)[inv] * absmean[inv]
        e[:, 11:] += U32 * f[:, 11:].abs()
        nan_row = torch.isnan(f).any(1, keepdim=True)          # every hidden unit NaN -> 0: the row is exactly relu(t2)
        e = torch.where(nan_row, torch.zeros_like(e), e)
        sorted_ = mode != "fp32"
        W1, S1, T1, S2, T2 = (t.double().to(dev) for t in (w1, s1, t1, s2, t2))
        W2 = round_h16(w2.double()).to(dev) if sorted_ else w2.double().to(dev)
        a = f @ W1.T
        sa = f.abs() @ W1.abs().T
        ea = e @ W1.abs().T
        if sorted_:
            ea += (3 * 2.0 ** -22 + 2.0 ** -16) * 1.01 * (sa + ea) + 2.0 ** -24 * (f.abs().sum(1, keepdim=True) + W1.abs().sum(1))
        else:
            ea += gamma(16) * (sa + ea)
        h = _relu(a * S1 + T1)
        eh = S1.abs() * ea + U32 * (S1.abs() * a.abs() + T1.abs())
        if sorted_:
            eh = eh + 2.0 ** -10 * (h.abs() + eh) + 2.0 ** -24
            h = round_h16(h)
        eh = torch.where(nan_row, torch.zeros_like(eh), eh)
        o = h @ W2.T
        so = h.abs() @ W2.abs().T
        eo = eh @ W2.abs().T
        eo += (2.0 ** -16 * 1.01 if sorted_ else gamma(64)) * (so + eo)
        out = _relu(o * S2 + T2)
        e2 = S2.abs() * eo + U32 * (S2.abs() * o.abs() + T2.abs())
        if parts == "centroid":       # sums of 1 or 2 points do not depend on the order: those rows are bit-identical
            e2 = torch.where(n[inv] >= 3, 2 * e2, torch.zeros_like(e2))
        row = (ny - 1 - xi).clamp(0, ny - 1)
        col = yi.clamp(0, nx - 1)
        cell = (bidx * ny + row) * nx + col
        idx = cell[:, None].expand(-1, 64)
        canvas.scatter_reduce_(0, idx, out, "amax", include_self=True)
        bound.scatter_reduce_(0, idx, e2, "amax", include_self=True)
        occupied[cell] = True
    if mode == "sorted_h16":               # empty cells are written as exact zeros
        flip = 2.0 ** -10 * (canvas.abs() + bound) + 2.0 ** -24
        bound = bound + torch.where(occupied & ((bound > 0) | (parts == "all")), flip, torch.zeros_like(bound))
        canvas = round_h16(canvas)
    return canvas.view(B, ny, nx, 64), bound.view(B, ny, nx, 64)


# ----------------------------------------------------------------------------------------------------- output canaries
CANARY = {torch.float32: 0x7FC0DEAD, torch.float16: 0x7E5A, torch.bfloat16: 0x7FDA}    # NaN bit patterns no kernel writes
INT = {torch.float32: torch.int32, torch.float16: torch.int16, torch.bfloat16: torch.int16}
_TRACES = itertools.count()


def canary(shape, dtype, device):
    t = torch.empty(shape, dtype=dtype, device=device)
    t.view(INT[dtype]).fill_(CANARY[dtype])
    return t


def is_canary(t):
    return t.contiguous().view(INT[t.dtype]) == CANARY[t.dtype]


def kernels(fn, tmp_path, tries=5):
    """run fn under torch.profiler; the (name, grid) of every kernel it launched, in launch order.  Every call traced here
    is idempotent (same outputs, same elements written), so fn may be traced more than once.  The profiler's kernel
    records can be missing from a short capture and arrive in a later one, so the kernel records of all captures are pooled
    by correlation id, and the first capture in which every kernel launch has its kernel record is the answer."""
    from torch.profiler import ProfilerActivity, profile
    records, captures = {}, []
    for _ in range(tries):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        path = os.path.join(str(tmp_path), f"trace{next(_TRACES)}.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
        os.remove(path)
        captures.append([e["args"]["correlation"] for e in events
                         if e.get("cat") in ("cuda_runtime", "cuda_driver") and "Launch" in e.get("name", "")
                         and "correlation" in e.get("args", {})])
        records.update({e["args"]["correlation"]: (e["name"], e["args"].get("grid")) for e in events
                        if e.get("cat") == "kernel" and "correlation" in e.get("args", {})})
        for launches in captures:
            if launches and all(c in records for c in launches):
                return [records[c] for c in launches]
    return []


# ----------------------------------------------------------------------------------------------------- camera kernels
# fp64 statements of lavb_erf_stem, lavb_erf_down16, lavb_erf_nb16, lavb_stem7x7s2_u8 and lavb_maxpool3x3s2_nhwc
# (include/lav_b200.h), on the operands as each kernel reads them.  Each returns (expected, bound) as float64 NHWC on the
# input's device: every correct kernel output c satisfies |c - expected| <= bound element-wise (bound 0 = bit-exact value).
U_MMA = 2.0 ** -23          # fp32 accumulation on the tensor cores: mma.sync is not guaranteed to round to nearest


def _store_h16(v, e):
    """the final saturating h16 store of a value known within e: both the kernel and the statement round their own value,
    so they can land one h16 ulp apart, 2^-10 (|v| + e) for normal values and 2^-24 (the subnormal spacing) below.  A
    non-finite v (an exact -inf / +inf of the pool branch) is stored exactly."""
    fin = torch.isfinite(v)
    e = torch.where(fin, e + 2.0 ** -10 * (v.abs() + e) + 2.0 ** -24, torch.zeros_like(e))
    return round_h16(v), e


def _store_h16_interval(v, e):
    """the same store, bounded exactly: the kernel's fp32 value lies in [v - e, v + e] and rounding is monotonic, so its h16
    value lies between the roundings of the two ends.  Where both ends round to round_h16(v) the kernel's stored value IS
    the statement's, bit for bit (bound 0); elsewhere the bound is the distance to the farther end's rounding."""
    r = round_h16(v)
    b = torch.maximum(round_h16(v + e) - r, r - round_h16(v - e))
    return r, torch.where(torch.isfinite(v), b, torch.zeros_like(b))


def _affine(a, ea, s, t):
    """relu(fmaf(a, s, t)) for a known within ea: |s| ea from the input, one fp32 rounding of the result.  A NaN (from a NaN
    operand) comes out as exactly 0 with bound 0, as fmaxf(NaN, 0) = 0."""
    v = a * s + t
    e = s.abs() * ea + U32 * (s.abs() * (a.abs() + ea) + t.abs())
    nan = torch.isnan(v)
    return _relu(v), torch.where(nan | ~torch.isfinite(e), torch.zeros_like(e), e)


def erf_stem_lut():
    """(v / 255 - .5) * 2 in fp32 for the 256 byte values, three roundings (rgb.py:41) -> float64 (256,).  numpy's fp32
    division, subtraction and product round to nearest, as the kernel's __fdiv_rn and fp32 ops do."""
    v = np.arange(256, dtype=np.float32)
    return torch.from_numpy(((v / np.float32(255) - np.float32(0.5)) * np.float32(2)).astype(np.float64))


def erf_stem_ref64(rgb_u8, w27, scale, shift, out_dtype):
    """lavb_erf_stem in float64.  rgb_u8 (N, H, W, 3) uint8; w27 (27, 16) [(ky*3+kx)*3+c][co] (only co < 13 read);
    scale / shift (16,); out_dtype float32 or the 16-bit type -> (N, H/2, W/2, 16) float64 expected and bound.

    The statement: x = erf_stem_lut()[rgb] (bit for bit the kernel's normalised image); channels 0..12 = relu(fmaf(conv3x3
    s2 p1 (x, w), s, t)) with zero padding in the normalised domain; channels 13..15 = relu(fmaf(maxpool2x2(x), s, t)).
    The bound (u = 2^-24, gamma_n = n u / (1 - n u)):
      * conv: the kernel's 27-term fp32 fmaf chain, gamma_27 sum |x w| (the exact fp64 sum of fp32 products adds < 2^-50
        sum |x w|, inside gamma_28, which is used);
      * pool: the max of four fp32 values is exact;
      * fmaf(a, s, t): |s| times the propagated error plus u (|s| (|a| + e) + |t|); ReLU is 1-Lipschitz;
      * h16 output: the final rounding (_store_h16)."""
    import torch.nn.functional as F
    dev = rgb_u8.device
    x = erf_stem_lut().to(dev)[rgb_u8.long()].permute(0, 3, 1, 2)
    w = torch.as_tensor(np.asarray(w27, dtype=np.float32)).double().to(dev)
    s = torch.as_tensor(np.asarray(scale, dtype=np.float32)).double().to(dev)[None, :, None, None]
    t = torch.as_tensor(np.asarray(shift, dtype=np.float32)).double().to(dev)[None, :, None, None]
    W = w[:, :13].reshape(3, 3, 3, 13).permute(3, 2, 0, 1)                 # [co][c][ky][kx]
    a = F.conv2d(x, W, stride=2, padding=1)
    ea = gamma(28) * F.conv2d(x.abs(), W.abs(), stride=2, padding=1)
    vc, ec = _affine(a, ea, s[:, :13], t[:, :13])
    m = F.max_pool2d(x, 2, 2)
    vp, ep = _affine(m, torch.zeros_like(m), s[:, 13:], t[:, 13:])
    v, e = torch.cat([vc, vp], 1).permute(0, 2, 3, 1), torch.cat([ec, ep], 1).permute(0, 2, 3, 1)
    if out_dtype != torch.float32:
        v, e = _store_h16(v, e)
    return v.contiguous(), e.contiguous()


def erf_down16_ref64(x_h16, w9, st):
    """lavb_erf_down16 in float64.  x_h16 (N, H, W, 16) 16-bit; w9 (9, 16, 48) fp32 [ky*3+kx][cin][cout]; st (64, 2) fp32
    (scale, shift) -> (N, H/2, W/2, 64) float64 expected and bound.

    The statement: channels 0..47 = relu(fmaf(conv3x3 s2 p1 (x, h16(w9)), s, t)); channels 48..63 = relu(fmaf(m, s, t)) with
    m the max of the 2x2 window that skips NaN and starts from -inf (so four NaNs give -inf); h16 store.
    The bound: the 144 products are exact in fp32 and summed on the tensor cores, bounded as gamma_144 with u = 2^-23 per
    add (U_MMA) on sum |x w|; the pool's max is exact; then _affine and _store_h16.  A conv channel whose window holds a NaN
    is exactly 0 (fmaxf(NaN, 0)), bound 0."""
    import torch.nn.functional as F
    x = x_h16.double().permute(0, 3, 1, 2)
    W = round_h16(w9.double()).to(x.device).reshape(3, 3, 16, 48).permute(3, 2, 0, 1)
    s, t = (st[:, i].double().to(x.device)[None, :, None, None] for i in (0, 1))
    a = F.conv2d(x, W, stride=2, padding=1)
    ea = gamma(144, U_MMA) * F.conv2d(x.abs(), W.abs(), stride=2, padding=1)
    vc, ec = _affine(a, ea, s[:, :48], t[:, :48])
    m = F.max_pool2d(torch.where(torch.isnan(x), torch.full_like(x, -math.inf), x), 2, 2)
    vp, ep = _affine(m, torch.zeros_like(m), s[:, 48:], t[:, 48:])
    v, e = torch.cat([vc, vp], 1).permute(0, 2, 3, 1), torch.cat([ec, ep], 1).permute(0, 2, 3, 1)
    return tuple(r.contiguous() for r in _store_h16(v, e))


def erf_nb16_ref64(x_h16, w4, st):
    """lavb_erf_nb16 in float64.  x_h16 (N, H, W, 16) 16-bit; w4 (4, 3, 16, 16) fp32 [conv][tap][cin][cout]; st (4, 16, 2)
    fp32 (scale, shift) -> (N, H, W, 16) float64 expected and bound.

    The statement: four stages, 3x1 / 1x3 / 3x1 / 1x3 with zero padding, each relu(fmaf(conv(in, h16(w)), s, t)) [+ x before
    the last ReLU, one fp32 add] stored as h16 for the next stage.
    The bound carries each stage's error e_in into the next: sum |w| e_in through the conv, plus the tensor-core sum of 48
    products, gamma_48 (u = 2^-23) on sum |w| (|in| + e_in); then _affine; the residual add rounds once more, u (|v| + e);
    ReLU is 1-Lipschitz.  Each h16 store is bounded exactly by _store_h16_interval: the fp32 error before a store is far
    below an h16 ulp, so almost every intermediate is bit-exact (bound 0) and only values within that error of a rounding
    boundary carry a one-ulp bound into the next stage, which amplifies it by its sum |w| |s|.  A NaN that reaches a ReLU
    gives exactly 0 (bound 0) in both."""
    import torch.nn.functional as F
    x = x_h16.double().permute(0, 3, 1, 2)
    W = round_h16(w4.double()).to(x.device)
    S = st.double().to(x.device)
    v, e = x, torch.zeros_like(x)
    for k in range(4):
        Wk = W[k].permute(2, 1, 0)                                              # [cout][cin][tap]
        Wk, pad = (Wk[..., None], (1, 0)) if k % 2 == 0 else (Wk[:, :, None, :], (0, 1))
        a = F.conv2d(v, Wk, padding=pad)
        ep = F.conv2d(e, Wk.abs(), padding=pad)
        ea = ep + gamma(48, U_MMA) * (F.conv2d(v.abs(), Wk.abs(), padding=pad) + ep)
        s, t = S[k, :, 0][None, :, None, None], S[k, :, 1][None, :, None, None]
        pre = a * s + t
        epre = s.abs() * ea + U32 * (s.abs() * (a.abs() + ea) + t.abs())
        if k == 3:
            pre = pre + x
            epre = epre + U32 * (pre.abs() + epre)
        nan = torch.isnan(pre)
        v = _relu(pre)
        e = torch.where(nan | ~torch.isfinite(epre), torch.zeros_like(epre), epre)
        v, e = _store_h16_interval(v, e)
    return v.permute(0, 2, 3, 1).contiguous(), e.permute(0, 2, 3, 1).contiguous()


def nb16_test_params(seed, weight_scale=0.03):
    """seeded erf_nb16 operands for the tests: w4 (4, 3, 16, 16) randn * weight_scale and st (4, 16, 2) fp32.  The default
    scale keeps sum |w| |s| of every stage below 2, so a one-ulp h16 difference is not amplified into a bound as large as the
    values: the statement's bound then tells an h16 kernel from a bf16 one (tests/test_camera_kernels_ref_cpu.py).  The
    scales of the two convs without BatchNorm are 1; the shifts of stages 1..3 are positive, so every channel is alive
    after their ReLUs; the last shift takes both signs."""
    g = torch.Generator().manual_seed(seed)
    w4 = torch.randn(4, 3, 16, 16, generator=g) * weight_scale
    s = torch.rand(4, 16, generator=g) + 0.5
    s[0], s[2] = 1.0, 1.0
    t = torch.randn(4, 16, generator=g) * 0.2
    t[:3] = t[:3].abs() + 0.05
    return w4, torch.stack([s, t], 2)


def stem_u8_operand(mean, std):
    """the staged operand of lavb_stem7x7s2_u8 for every byte value and channel, bit for bit -> (256, 3) float64 of h16
    values: na = 1.f / (255.f * std), nb = -mean / std in fp32 as the host computes them; fmaf(u8, na, nb), whose fp64
    product and sum are exact here (at most 40 significant bits), rounded once to fp32; then rounded to h16."""
    m, s = np.asarray(mean, dtype=np.float32), np.asarray(std, dtype=np.float32)
    na = np.float32(1) / (np.float32(255) * s)
    nb = -m / s
    u = np.arange(256, dtype=np.float64)[:, None]
    f32 = (u * na.astype(np.float64) + nb.astype(np.float64)).astype(np.float32)
    return torch.from_numpy(f32).half().double()


def stem_unpack_weights(w_h16):
    """(64, 160) in the stem kernel's K order k = ky*22 + kx*3 + c -> (64, 3, 7, 7) float64; slot 21 of each window row and
    k >= 154 are zero by the header's contract and are not part of the statement."""
    return w_h16.double()[:, :154].reshape(64, 7, 22)[:, :, :21].reshape(64, 7, 7, 3).permute(0, 3, 1, 2)


def stem7x7s2_u8_ref64(img_u8, w_h16, bias, mean, std):
    """lavb_stem7x7s2_u8 in float64.  img_u8 (B, ncam, H, cam_w, 3) uint8; w_h16 (64, 160) 16-bit from pack_stem_weights;
    bias (64,) fp32 -> (B, (H-1)//2+1, (ncam*cam_w-1)//2+1, 64) float64 expected and bound.

    The statement: the side-by-side image of the cameras, each byte replaced by stem_u8_operand (zero padding in the
    normalised domain), conv 7x7 s2 p3 with the h16 weights (exact products), + bias, ReLU, h16 store.
    The bound: the 147 live products (154 slots) are summed in fp32 on the tensor cores over 10 k-steps of 16, bounded as
    gamma_160 with u = 2^-23 per add on sum |x w|; the bias add rounds once, u (|a| + e + |b|); then _store_h16."""
    import torch.nn.functional as F
    B, ncam, H, cw, _ = img_u8.shape
    dev = img_u8.device
    op = stem_u8_operand(mean, std).to(dev)
    wide = img_u8.permute(0, 2, 1, 3, 4).reshape(B, H, ncam * cw, 3).long()
    x = torch.stack([op[wide[..., c], c] for c in range(3)], 1)
    W = stem_unpack_weights(w_h16).to(dev)
    b = bias.double().to(dev)[None, :, None, None]
    a = F.conv2d(x, W, stride=2, padding=3)
    ea = gamma(160, U_MMA) * F.conv2d(x.abs(), W.abs(), stride=2, padding=3)
    v = a + b
    e = ea + U32 * (a.abs() + ea + b.abs())
    v, e = _store_h16(_relu(v).permute(0, 2, 3, 1), e.permute(0, 2, 3, 1))
    return v.contiguous(), e.contiguous()


def maxpool3x3s2_ref64(x_h16):
    """lavb_maxpool3x3s2_nhwc in float64, exact: (N, H, W, C) 16-bit -> (N, (H-1)//2+1, (W-1)//2+1, C) float64.  Pixels off
    the map are skipped, a NaN anywhere in the window gives NaN (MaxPool2d's rule), and -0 ranks below +0 (the header's
    rule; MaxPool2d would keep whichever zero comes first)."""
    import torch.nn.functional as F
    x = x_h16.double().permute(0, 3, 1, 2)
    neg0 = (x == 0) & torch.signbit(x)
    tiny = -1e-300                                  # -0 -> a value between every negative h16 (<= -2^-24) and +0
    m = F.max_pool2d(torch.where(neg0, torch.full_like(x, tiny), x), 3, 2, 1)
    m = torch.where(m == tiny, torch.full_like(m, -0.0), m)
    return m.permute(0, 2, 3, 1).contiguous()


# ----------------------------------------------------------------------------------------------------- painting and stacking
# Bit-exact fp32 statements of lavb_paint / _batched / lavb_paint_deconv_batched, lavb_stack_sweep / lavb_stack_jobs,
# lavb_roof_filter and lavb_lidar_batch (include/lav_b200.h), in numpy.  numpy's fp32 +, -, *, / round to nearest as the
# kernels' __fadd_rn, __fsub_rn, __fmul_rn, __fdiv_rn do; fma32 is a correctly rounded fmaf.  The one operation that is not
# correctly rounded, expf, is bounded instead (paint_softmax32).
F32 = np.float32
INT64_MIN = np.int64(-2 ** 63)


def fma32(a, b, c):
    """fmaf(a, b, c) element-wise, correctly rounded: a*b is exact in fp64 (48 significant bits); s = a*b + c rounded to fp64
    with its exact error from TwoSum; where the error is nonzero s is moved to the odd fp64 neighbour of the exact sum (round to
    odd, 53 >= 24 + 2 bits), so the final fp64 -> fp32 rounding cannot double-round."""
    a, b, c = (np.asarray(v, dtype=F32) for v in (a, b, c))
    with np.errstate(all="ignore"):
        p = a.astype(np.float64) * b.astype(np.float64)
        c64 = c.astype(np.float64)
        s = p + c64
        bb = s - p
        err = (p - (s - bb)) + (c64 - bb)
        fix = np.isfinite(s) & (err != 0) & ((s.view(np.int64) & 1) == 0)
        s = np.where(fix, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
        return s.astype(F32)


def trunc_i64(v):
    """cvttss2si as project_hit.cuh restates it: toward zero, NaN / +-inf / |v| >= 2^63 -> INT64_MIN"""
    v = np.asarray(v, dtype=F32)
    ok = np.abs(v) < F32(2.0 ** 63)
    with np.errstate(all="ignore"):
        return np.where(ok, np.where(ok, v, 0).astype(np.int64), INT64_MIN)


def _dot(r, xs):
    acc = (F32(r[0]) * xs[0]).astype(F32)
    for k in range(1, len(xs)):
        acc = fma32(F32(r[k]), xs[k], acc)
    return acc


def project_hit32(cams, x, y, z, H, W):
    """project_hit.cuh: -> (camera (int64, -1 = unseen), u, v) for fp32 points; the last camera whose truncated pixel lies in
    the W x H image wins."""
    cams = np.asarray(cams, dtype=F32)
    x, y, z = (np.asarray(t, dtype=F32) for t in (x, y, z))
    one = np.ones_like(x)
    cam, hu, hv = np.full(x.shape, -1, np.int64), np.zeros(x.shape, np.int64), np.zeros(x.shape, np.int64)
    with np.errstate(all="ignore"):
        for c in range(len(cams)):
            K, L, Wc = cams[c, :9], cams[c, 9:25], cams[c, 25:41]
            w = [_dot(L[4 * i:4 * i + 4], (x, y, z, one)) for i in range(4)]
            c0, c1, c2 = (_dot(Wc[4 * i:4 * i + 4], w) for i in range(3))
            a = (c1, -c2, c0)
            q0, q1, q2 = (_dot(K[3 * i:3 * i + 3], a) for i in range(3))
            den = (F32(1e-5) + q2).astype(F32)
            u, v, zi = trunc_i64((q0 / den).astype(F32)), trunc_i64((q1 / den).astype(F32)), trunc_i64(q2)
            hit = (zi >= 0) & (u >= 0) & (u < W) & (v >= 0) & (v < H)
            cam, hu, hv = np.where(hit, c, cam), np.where(hit, u, hu), np.where(hit, v, hv)
    return cam, hu, hv


def paint_softmax32(x):
    """lavb_paint mode 2's softmax and suppression on fp32 logits x (..., C) -> (want (..., C-1) float64, bound float64, nan
    (...,) bool: every painted channel NaN).

    Bit-exact parts: mx = fmaxf over the classes in order (NaN skipped), d_k = fp32(x_k - mx).  E_k = exp(d_k) in fp64; the
    statement is want_k = P_k (1 - P_0), P_k = E_k / S, S = sum E_k.  The bound (u = 2^-24, gamma_n = n u / (1 - n u)):
      * expf is within 2 ulp (CUDA C Programming Guide, full range): |e_k - E_k| <= dl_k = 2^-22 E_k + 2^-148 (the ulp of a
        value is at most 2^-23 of it, or the subnormal spacing 2^-149);
      * the sequential fp32 sum of C terms: |s - S| <= dS = sum dl_k + gamma_(C-1) sum (E_k + dl_k); S >= 1 (the max's term is
        expf(0) = 1 exactly), so S - dS > 0 here;
      * p_k = fp32(e_k / s): |e_k / s - P_k| <= (dl_k S + E_k dS) / (S (S - dS)) = r_k, plus the rounding u (P_k + r_k): eta_k;
      * bg = fp32(1 - p_0): 1 - P_0 cancels, so its error is absolute: ebg = eta_0 + u (B + eta_0), B = 1 - P_0;
      * o_k = fp32(p_k bg): |p_k bg - P_k B| <= eta_k (B + ebg) + P_k ebg, plus u times the magnitude.
    The bound is on the absolute error of each output, with a 2^-40 relative margin for the fp64 evaluation of the statement.
    NaN rule: any NaN or +inf logit, or all logits -inf, makes every output NaN (the sum is NaN)."""
    x = np.asarray(x, dtype=F32)
    C = x.shape[-1]
    with np.errstate(all="ignore"):
        mx = x[..., 0]
        for k in range(1, C):
            mx = np.fmax(mx, x[..., k])
        d = (x - mx[..., None]).astype(F32)
        nan = np.isnan(d).any(-1)
        E = np.exp(d.astype(np.float64))
        dl = 2.0 ** -22 * E + 2.0 ** -148
        S = E.sum(-1, keepdims=True)
        dS = dl.sum(-1, keepdims=True) + gamma(C - 1) * (E + dl).sum(-1, keepdims=True)
        P = E / S
        r = (dl * S + E * dS) / (S * (S - dS))
        eta = r + U32 * (P + r)
        B = 1.0 - P[..., :1]
        ebg = eta[..., :1] + U32 * (B + eta[..., :1])
        want = P[..., 1:] * B
        e = eta[..., 1:] * (B + ebg) + P[..., 1:] * ebg
        bound = (e + U32 * (want + e)) * (1 + 2.0 ** -40)
    want = np.where(nan[..., None], np.nan, want)
    return want, np.where(nan[..., None], 0.0, bound), nan


def paint32(pts, sem, cams, mode, H, W):
    """the painted channels of lavb_paint for fp32 points pts (..., >=3) and one frame's semantic maps sem (ncam, C, H, W) as a
    numpy array (any strides) -> (want (..., c_out), bound or None, nan (...,) or None): mode 0 / 1 are bit-exact fp32 (bound
    None), mode 2 is paint_softmax32's statement.  Unseen points are exact zeros."""
    pts = np.asarray(pts, dtype=F32)
    cam, u, v = project_hit32(cams, pts[..., 0], pts[..., 1], pts[..., 2], H, W)
    seen = cam >= 0
    g = np.asarray(sem, dtype=F32)[np.where(seen, cam, 0), :, np.where(seen, v, 0), np.where(seen, u, 0)]   # (..., C)
    return _paint_values(g, seen, mode)


def _paint_values(g, seen, mode):
    C = g.shape[-1]
    c_out = C if mode == 0 else C - 1
    if mode == 0:
        return np.where(seen[..., None], g, F32(0)), None, None
    if mode == 1:
        with np.errstate(all="ignore"):
            bg = (F32(1) - g[..., 0]).astype(F32)
            want = (g[..., 1:] * bg[..., None]).astype(F32)
        return np.where(seen[..., None], want, F32(0)), None, None
    want, bound, nan = paint_softmax32(g)
    return np.where(seen[..., None], want, 0.0), np.where(seen[..., None], bound, 0.0), nan & seen


def deconv_logits32(fv, table, pv, pu, C):
    """deconv_logits.cuh: fv (..., 16) fp32 (h16 features widened exactly), table the 520-float pack_deconv2x2 table,
    phases pv, pu (...) -> logits (..., C) fp32, bias then fmaf over the 16 channels in order"""
    t = np.asarray(table, dtype=F32)
    w, bias = t[:512].reshape(2, 2, 16, 8), t[512:]
    out = []
    for k in range(C):
        acc = np.broadcast_to(bias[k], fv.shape[:-1]).astype(F32)
        for c in range(16):
            acc = fma32(fv[..., c], w[pv, pu, c, k], acc)
        out.append(acc)
    return np.stack(out, -1)


def paint_deconv32(pts, feat, table, cams, C, H, W):
    """lavb_paint_deconv_batched's painted channels: pts (F, N, >=3) fp32, feat (F * ncam, H/2, W/2, 16) as float32 (the h16
    features widened) -> as paint32 mode 2"""
    pts = np.asarray(pts, dtype=F32)
    ncam = len(cams)
    cam, u, v = project_hit32(cams, pts[..., 0], pts[..., 1], pts[..., 2], H, W)
    seen = cam >= 0
    f = np.arange(pts.shape[0])[:, None] * ncam + np.where(seen, cam, 0)
    vv, uu = np.where(seen, v, 0), np.where(seen, u, 0)
    fv = np.asarray(feat, dtype=F32)[f, vv >> 1, uu >> 1]
    g = deconv_logits32(fv, table, vv & 1, uu & 1, C)
    return _paint_values(g, seen, 2)


def move_point32(R, dx, dy, x, y, z):
    """paint.cu move_point: [x y z] @ R as k-sequential fmaf chains, then x + dx, y + dy as fp32 adds (z has no add)"""
    R = np.asarray(R, dtype=F32).ravel()
    with np.errstate(all="ignore"):
        nx = (fma32(z, R[6], fma32(y, R[3], (x * R[0]).astype(F32))) + F32(dx)).astype(F32)
        ny = (fma32(z, R[7], fma32(y, R[4], (x * R[1]).astype(F32))) + F32(dy)).astype(F32)
        nz = fma32(z, R[8], fma32(y, R[5], (x * R[2]).astype(F32)))
    return nx, ny, nz


ROOF = tuple(F32(v) for v in (-2.4, 0, -0.8, 0.8, -1.5, -1))


def roof_keep32(rows):
    """lavb_roof_filter's keep predicate on (n, >=3) fp32 rows: not strictly inside the box (a NaN coordinate keeps the row)"""
    x, y, z = (np.asarray(rows, dtype=F32)[:, k] for k in range(3))
    x0, x1, y0, y1, z0, z1 = ROOF
    return ~((x > x0) & (x < x1) & (y > y0) & (y < y1) & (z > z0) & (z < z1))


def stack32(src, R, dx, dy, time_idx, n_time, roof=False):
    """lavb_stack_sweep's rows: src (n, cols) fp32 -> (n, cols + n_time) fp32"""
    src = np.asarray(src, dtype=F32)
    out = np.zeros((src.shape[0], src.shape[1] + n_time), F32)
    nx, ny, nz = move_point32(R, dx, dy, src[:, 0], src[:, 1], src[:, 2])
    if roof:
        nx = np.where(roof_keep32(src), nx, np.array([0x7FC00000], np.uint32).view(F32)[0])
    out[:, 0], out[:, 1], out[:, 2] = nx, ny, nz
    out[:, 3:src.shape[1]] = src[:, 3:]
    if 0 <= time_idx < n_time:
        out[:, src.shape[1] + time_idx] = 1
    return out


def lidar_batch32(raw, rows, sweeps, cams, H, W, n_time):
    """lavb_lidar_batch: raw (n_raw, 4 + c) fp32, rows (n_rows,) int, sweeps LIDAR_SWEEP_DTYPE records sorted by row0 ->
    (n_rows, 4 + c + n_time) fp32"""
    raw = np.asarray(raw, dtype=F32)
    rows = np.asarray(rows, dtype=np.int64).ravel()
    cols = raw.shape[1]
    out = np.zeros((len(rows), cols + n_time), F32)
    valid = (rows >= 0) & (rows < len(raw))
    s = np.searchsorted(sweeps["row0"].astype(np.int64), np.where(valid, rows, 0), side="right") - 1 if len(sweeps) else \
        np.full(len(rows), -1)
    live = valid & (s >= 0)
    for k in np.unique(s[live]):
        m = live & (s == k)
        sw = sweeps[k]
        p = raw[rows[m]]
        ax, ay, az = move_point32(sw["R_aug"], 0.0, 0.0, p[:, 0], p[:, 1], p[:, 2])
        vis = (project_hit32(cams, ax, ay, az, H, W)[0] >= 0).astype(F32)
        o = out[m]
        o[:, 0], o[:, 1], o[:, 2] = move_point32(sw["R_mv"], sw["dx"], sw["dy"], ax, ay, az)
        o[:, 3] = p[:, 3]
        with np.errstate(all="ignore"):
            o[:, 4:cols] = (p[:, 4:] * vis[:, None]).astype(F32)
        if 0 <= sw["time_idx"] < n_time:
            o[:, cols + sw["time_idx"]] = 1
        out[m] = o
    return out


# ----------------------------------------------------------------------------------------------------- cast GRU and u8 crop
# fp64 statements of lavb_cast_gru and lavb_crop_bilinear_u8 (include/lav_b200.h), pinned to torch's float64 nn.GRU and
# F.affine_grid + F.grid_sample by tests/test_cast_crop_ref_cpu.py and held against the kernels by
# tests/test_gpu_cast_crop_contract.py.
CAST_MUTANTS = ("bhn_outside_r", "r_z_swapped", "h_update_swapped", "cumsum_shifted", "branches_swapped")
# largest |kernel - cast_gru_ref| / mag allowed on the H100, mag being cast_gru_ref's per-element magnitude
# (tests/test_gpu_cast_crop_contract.py states the measured value and the margin)
CAST_TOL = 4e-5


def cast_gru_ref(embd, wih_t, whh_t, bih, bhh, wmlp, bmlp, steps, mutant=None):
    """lavb_cast_gru in float64 on embd's device, from the packed operands the kernel reads (embd (n, 512), wih_t (ncmd, 512,
    192), whh_t (ncmd, 64, 192), bih / bhh (ncmd, 192), wmlp (ncmd, 2, 64), bmlp (ncmd, 2)) -> (out, mag), both
    (n, ncmd, steps, 2) float64.

    out: nn.GRU(512, 64) over the embedding repeated ``steps`` times from h = 0 (gate order r, z, n; n = tanh(gi_n +
    r (W_hn h + b_hn)); h' = (1 - z) n + z h), then Linear(64, 2) and the inclusive cumsum over the steps.
    mag: the cumsum of |b_mlp| + sum_j |W_mlp,j| |h'_j| over the same steps, the size of the terms that make up each output:
    an error measured in units of mag is measured against that step's own waypoint, not the largest one.
    mutant: one of CAST_MUTANTS states a plausible wrong kernel instead: b_hn added outside the reset gate, the r and z
    columns swapped, h' = (1 - z) h + z n, the cumsum shifted by one step (exclusive), or branches 0 and 1 swapped."""
    assert mutant is None or mutant in CAST_MUTANTS
    dev = embd.device
    x = embd.double()
    wi, wh, bi, bh, wm, bm = (t.to(dev).double() for t in (wih_t, whh_t, bih, bhh, wmlp, bmlp))
    if mutant == "branches_swapped":
        perm = torch.arange(wi.shape[0], device=dev)
        perm[[0, 1]] = perm[[1, 0]]
        wi, wh, bi, bh, wm, bm = (t[perm] for t in (wi, wh, bi, bh, wm, bm))
    ncmd, n = wi.shape[0], x.shape[0]
    gi = torch.einsum("nk,ckg->cng", x, wi) + bi[:, None]                  # (ncmd, n, 192)
    h = torch.zeros((ncmd, n, 64), dtype=torch.float64, device=dev)
    loc, mg = torch.zeros((ncmd, n, 2), dtype=torch.float64, device=dev), torch.zeros((ncmd, n, 2), dtype=torch.float64, device=dev)
    outs, mags = [], []
    for _ in range(steps):
        ghw = torch.bmm(h, wh)                                                 # W_hh h, (ncmd, n, 192)
        gh = ghw + bh[:, None]
        r = torch.sigmoid(gi[..., :64] + gh[..., :64])
        z = torch.sigmoid(gi[..., 64:128] + gh[..., 64:128])
        if mutant == "r_z_swapped":
            r, z = z, r
        if mutant == "bhn_outside_r":
            nn_ = torch.tanh(gi[..., 128:] + r * ghw[..., 128:] + bh[:, None, 128:])
        else:
            nn_ = torch.tanh(gi[..., 128:] + r * gh[..., 128:])
        h = (1 - z) * h + z * nn_ if mutant == "h_update_swapped" else (1 - z) * nn_ + z * h
        loc = loc + torch.einsum("cnj,coj->cno", h, wm) + bm[:, None]
        mg = mg + torch.einsum("cnj,coj->cno", h.abs(), wm.abs()) + bm.abs()[:, None]
        outs.append(loc)
        mags.append(mg)
    out, mag = torch.stack(outs, 2).permute(1, 0, 2, 3), torch.stack(mags, 2).permute(1, 0, 2, 3)
    if mutant == "cumsum_shifted":
        out = torch.cat([torch.zeros_like(out[:, :, :1]), out[:, :, :-1]], 2)
    return out.contiguous(), mag.contiguous()


def cast_rel_err(got, want, mag):
    """max over the elements where want is finite of |got - want| / mag (cast_gru_ref's units); inf if got is not finite there"""
    fin = torch.isfinite(want)
    if not bool(fin.any()):
        return 0.0
    g, w, m = got.double().to(want.device)[fin], want[fin], mag[fin]
    if not bool(torch.isfinite(g).all()):
        return math.inf
    return float(((g - w).abs() / m).max())


def cast_inputs(n, ncmd, scale="product", seed=0):
    """seeded fp32 CPU operands of lavb_cast_gru, packed as the kernel reads them: (embd, wih_t, whh_t, bih, bhh, wmlp, bmlp).
    Every branch has its own weights; the biases are N(0, 1), eight times nn.GRU's default init, so that where a bias enters
    the gate formula shows in the output.  scale "product": non-negative embeddings of the embedder's ReLU + average-pool
    output, about 0.5 on average; "saturating": N(0, 150) embeddings, whose input projections reach +-100 and beyond, so that
    most gates round to exactly 0 or 1 in fp32 (expf(100) overflows; tanhf(17) is 1)."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(s, generator=g)                                 # noqa: E731
    embd = r(n, 512).abs() * 0.6 if scale == "product" else r(n, 512) * 150.0
    wih = r(ncmd, 192, 512) / 512 ** 0.5
    whh = r(ncmd, 192, 64) / 64 ** 0.5
    bih, bhh = r(ncmd, 192), r(ncmd, 192)
    wmlp, bmlp = r(ncmd, 2, 64) / 8, r(ncmd, 2)
    return (embd.contiguous(), wih.transpose(1, 2).contiguous(), whh.transpose(1, 2).contiguous(), bih, bhh, wmlp.contiguous(), bmlp)


def cast_planner_inputs(n, seed=0):
    """the ego cast branches of the benchmarked UniPlanner (6 x GRU(512, 64) + Linear(64, 2)) with synth.fill_state_dict_
    weights, packed as heads._cast_branches packs them, and n product-scale embeddings -> as cast_inputs"""
    import torch.nn as nn

    class Branches(nn.Module):                         # the state_dict keys of UniPlanner's ego branches
        def __init__(self):
            super().__init__()
            self.cast_grus_ego = nn.ModuleList([nn.GRU(512, 64, batch_first=True) for _ in range(6)])
            self.cast_mlps_ego = nn.ModuleList([nn.Linear(64, 2) for _ in range(6)])

    m = Branches()
    m.load_state_dict(synth.fill_state_dict_(m.state_dict()))
    grus, mlps = m.cast_grus_ego, m.cast_mlps_ego
    with torch.no_grad():
        pack = (torch.stack([q.weight_ih_l0.t() for q in grus]).contiguous(), torch.stack([q.weight_hh_l0.t() for q in grus]).contiguous(),
                torch.stack([q.bias_ih_l0 for q in grus]).contiguous(), torch.stack([q.bias_hh_l0 for q in grus]).contiguous(),
                torch.stack([q.weight for q in mlps]).contiguous(), torch.stack([q.bias for q in mlps]).contiguous())
    return (cast_inputs(n, 1, "product", seed)[0], *pack)


def crop_linspace32(S):
    """torch.linspace(-1, 1, S) in fp32 as the crop kernels form it (start + step i for i < S // 2, end - step (S - 1 - i)
    after, one fmaf each: i * step is exact in float64, so one rounding to fp32 is the fmaf) -> float32 numpy (S,)"""
    step = np.float32(2) / np.float32(S - 1)
    i = np.arange(S, dtype=np.float64)
    lo = (i * np.float64(step) - 1.0).astype(np.float32)
    hi = (1.0 - (S - 1 - i) * np.float64(step)).astype(np.float32)
    return np.where(np.arange(S) < S // 2, lo, hi)


def crop_positions(theta, S, H, W, fp32=False):
    """sample positions of the crops of theta (K, 2, 3) on an H x W map -> (ix, iy), each (K, S, S) float64 CPU, [k, j, i].
    fp32=False: the affine map in float64 from the fp32 grid values x_i, y_j (crop_linspace32) and the fp32 theta.
    fp32=True: the kernels' own fp32 positions, bit for bit: gx = fmaf(t00, x_i, fmaf(t01, y_j, t02)), ix = (gx + 1) * 0.5 *
    (W - 1), each operation rounded to fp32 (fma32 is a correctly rounded fmaf)."""
    lin = crop_linspace32(S)
    if fp32:
        t = theta.detach().float().cpu().numpy()
        X, Y = lin[None, None, :], lin[None, :, None]
        out = []
        for row, n in ((0, W), (1, H)):
            g = fma32(t[:, row, 0, None, None], X, fma32(t[:, row, 1, None, None], Y, t[:, row, 2, None, None]))
            with np.errstate(all="ignore"):
                out.append(torch.from_numpy((((g + F32(1)) * F32(0.5)) * F32(n - 1)).astype(np.float64)))
        return out[0], out[1]
    t = theta.detach().float().cpu().double()
    x = torch.from_numpy(lin.astype(np.float64))
    X, Y = x[None, None, :], x[None, :, None]
    gx = t[:, 0, 0, None, None] * X + t[:, 0, 1, None, None] * Y + t[:, 0, 2, None, None]
    gy = t[:, 1, 0, None, None] * X + t[:, 1, 1, None, None] * Y + t[:, 1, 2, None, None]
    return (gx + 1) / 2 * (W - 1), (gy + 1) / 2 * (H - 1)


def crop_u8_ref(bev_u8, frame_idx, theta, S, fp32_positions=False):
    """lavb_crop_bilinear_u8 in float64 on bev_u8's device: bev_u8 (B, C, H, W) uint8, frame_idx (K,) clamped to [0, B),
    theta (K, 2, 3) -> (K, C, S, S) float64.  Bilinear with zero padding at crop_positions(theta, S, H, W, fp32_positions):
    taps floor(ix) + {0, 1}, floor(iy) + {0, 1} with weights (1 - ax)(1 - ay), ax (1 - ay), (1 - ax) ay, ax ay; a tap off
    the map adds nothing.  The header's rule for non-finite positions: a NaN coordinate gives NaN in every channel; an
    infinite one reads no tap (0)."""
    B, C, H, W = bev_u8.shape
    dev = bev_u8.device
    fi = frame_idx.long().to(dev).clamp(0, B - 1)
    ix, iy = (p.to(dev) for p in crop_positions(theta, S, H, W, fp32_positions))
    x0, y0 = ix.floor(), iy.floor()
    ax, ay = ix - x0, iy - y0
    flat = bev_u8.reshape(-1)
    chan = (torch.arange(C, device=dev) * (H * W))[None, :, None, None]
    out = torch.zeros((fi.numel(), C, S, S), dtype=torch.float64, device=dev)
    for dy, dx, wgt in ((0, 0, (1 - ax) * (1 - ay)), (0, 1, ax * (1 - ay)), (1, 0, (1 - ax) * ay), (1, 1, ax * ay)):
        x, y = x0 + dx, y0 + dy
        ok = (x >= 0) & (x < W) & (y >= 0) & (y < H)
        base = fi[:, None, None] * (C * H * W) + torch.where(ok, y, 0).long() * W + torch.where(ok, x, 0).long()
        out += torch.where(ok, wgt, 0.0)[:, None] * flat[base[:, None] + chan].double()
    nan = (torch.isnan(ix) | torch.isnan(iy))[:, None].expand_as(out)
    return torch.where(nan, torch.full_like(out, math.nan), out)


def cast_case(n, ncmd, steps, scale, rows=None):
    """the operands of one case of tests/test_gpu_cast_crop_contract.py, seeded by the case itself -> (operands, steps).
    scale "product" / "saturating": cast_inputs; "planner": cast_planner_inputs (ncmd must be 6).  rows: keep only the first
    rows embeddings (the cases' rows are independent, so these are still the GPU test's inputs)."""
    seed = n * 1000 + ncmd * 100 + steps + {"product": 0, "saturating": 1, "planner": 2}[scale]
    if scale == "planner":
        assert ncmd == 6
        ops_ = cast_planner_inputs(n, seed)
    else:
        ops_ = cast_inputs(n, ncmd, scale, seed)
    if rows is not None:
        ops_ = (ops_[0][:rows].contiguous(), *ops_[1:])
    return ops_, steps


# (n, ncmd, steps, scale) cases of the GPU test at which the CPU test shows every mutant far outside CAST_TOL; the last is the
# frame path at the benchmark's batch: 2 pipelines x 32 agents, 3 detected vehicles each -> 96 + 32 rows, 20 steps
CAST_MUTANT_CASES = {"product": (37, 7, 20, "product"), "saturating": (37, 7, 20, "saturating"), "frame_path": (128, 6, 20, "planner")}


# ----------------------------------------------------------------------------------------------------- wgmma convolutions
# fp64 statements of lavb_conv_umma, lavb_conv3x3_umma, lavb_conv7x7s2_umma and lavb_conv_pair_umma (include/lav_b200.h) on
# the operands as the kernels read them, tied to F.conv2d / F.conv_transpose2d by tests/test_wgmma_ref_cpu.py and held against
# the kernels by tests/test_gpu_wgmma_contract.py.  The tolerances are max-norm errors as a fraction of the output scale (the
# largest finite |expected|), bounds the kernels must meet: fp32 output, h16 output, the pair (two h16 roundings and a packed
# h16 residual add).
WGMMA_TOL = {"f32": 2e-5, "h16": 1e-3, "pair": 1e-2}
WGMMA_MUTANTS = ("k_chunk_dropped", "tap_shifted", "phase_out_o_swapped", "bias_after_pre_relu", "res_slice_off8", "nan_to_neg_inf")


def fmax0(a):
    """fmaxf(a, 0.f): a NaN comes out as 0 (torch.relu would keep it)"""
    return torch.where(torch.isnan(a), torch.zeros_like(a), a.clamp_min(0))


def tap_conv64(x, taps, w, in_s, hog, wog, mutant=None):
    """the tap sum of the wgmma convolutions in float64: x (n, H, W, cin) (the channel slice the kernel reads), taps [(dy, dx)],
    w (ntaps, cout, cin), in_s (sy, sx) -> (n, hog, wog, cout) with
    acc[n, oy, ox, co] = sum_t sum_ci x[n, oy*sy + dy_t, ox*sx + dx_t, ci] w[t, co, ci]   (zero outside the input).
    NaN rule: an output whose receptive field (the pixels its taps read) holds a NaN is NaN, whatever the weights; that set is
    computed from the NaN mask apart from the sum, so that the fp64 algorithm cannot spread a NaN.  Infinities enter the
    sum as they are (one infinite pixel reaches an output through one tap, so the sum is +-inf, never inf - inf).
    mutant "k_chunk_dropped": the last 64-channel chunk of every tap left out; "tap_shifted": tap 0 reads one pixel to the
    right."""
    n, H, W, cin = x.shape
    sy, sx = in_s
    dev = x.device
    nan_px = torch.isnan(x).any(-1)
    xz = torch.where(torch.isnan(x), torch.zeros_like(x), x)
    if mutant == "k_chunk_dropped":
        xz = xz.clone()
        xz[..., cin - 64:] = 0
    acc = torch.zeros((n, hog, wog, w.shape[1]), dtype=torch.float64, device=dev)
    hit = torch.zeros((n, hog, wog), dtype=torch.bool, device=dev)
    for t, (dy, dx) in enumerate(taps):
        if mutant == "tap_shifted" and t == 0:
            dx += 1
        ry = torch.arange(hog, device=dev) * sy + dy
        rx = torch.arange(wog, device=dev) * sx + dx
        oky, okx = (ry >= 0) & (ry < H), (rx >= 0) & (rx < W)
        ok = oky[:, None] & okx[None, :]
        g = xz[:, ry.clamp(0, H - 1)][:, :, rx.clamp(0, W - 1)]
        g = torch.where(ok[None, :, :, None], g, torch.zeros_like(g))
        acc += torch.einsum("nhwc,oc->nhwo", g, w[t].double().to(dev))
        hit |= nan_px[:, ry.clamp(0, H - 1)][:, :, rx.clamp(0, W - 1)] & ok[None]
    return torch.where(hit[..., None], torch.full_like(acc, math.nan), acc)


def wgmma_epilogue64(a, bias=None, scale=None, shift=None, res=None, pre=False, post=False, sig=False, mutant=None):
    """the epilogue of lavb_conv_umma / lavb_conv3x3_umma in float64: a += bias; pre: fmax0; a * scale + shift; a += res; post:
    fmax0; sigmoid.  A missing operand skips its step.  mutant "bias_after_pre_relu": fmax0(a) + bias; "nan_to_neg_inf": each
    ReLU that is off is fmaxf(a, -inf), which turns a NaN into -inf (the rule before it was fixed)."""
    ninf = torch.full_like(a, -math.inf)
    if mutant == "nan_to_neg_inf" and not pre:
        a = torch.where(torch.isnan(a), ninf, a)
    if bias is not None and mutant != "bias_after_pre_relu":
        a = a + bias.double().to(a.device)
    if pre:
        a = fmax0(a)
    if bias is not None and mutant == "bias_after_pre_relu":
        a = a + bias.double().to(a.device)
    if scale is not None:
        a = a * scale.double().to(a.device) + shift.double().to(a.device)
    if res is not None:
        a = a + res.double().to(a.device)
    if mutant == "nan_to_neg_inf" and not post:
        a = torch.where(torch.isnan(a), ninf, a)
    if post:
        a = fmax0(a)
    if sig:
        a = torch.sigmoid(a)
    return a


def store64(v, out):
    """the output store: "f32" keeps the value (fp32 NaN / inf as they are); "h16" saturates at +-65504 and keeps NaN.  The
    statement is not rounded further: the tolerances cover the roundings."""
    return v.clamp(-65504, 65504) if out == "h16" else v


def convT_phases(wt, k=3, s=2, p=1):
    """ConvTranspose2d(k, stride s, padding p) with weight wt (cin, cout, k, k) as s * s output phases, the way
    lav_b200/layers.py issues it: [(out_o, taps, w (ntaps, cout, cin))], phase (py, px) writing pixels (s oy + py, s ox + px)"""
    phases = []
    for py in range(s):
        for px in range(s):
            taps, blocks = [], []
            for ky in range(k):
                if (py + p - ky) % s:
                    continue
                for kx in range(k):
                    if (px + p - kx) % s:
                        continue
                    taps.append(((py + p - ky) // s, (px + p - kx) // s))
                    blocks.append(wt[:, :, ky, kx].t())
            phases.append(((py, px), taps, torch.stack(blocks)))
    return phases


def convT_assemble64(x, phases, hout, wout, epi, mutant=None):
    """every phase's tap sum and epilogue placed on its lattice of an (n, hout, wout, cout) float64 map (the pixels of
    hout x wout that the phase's lattice reaches; a phase is called on the input's h x w grid).  mutant
    "phase_out_o_swapped": phases (0, 1) and (1, 0) write each other's lattice."""
    n, h, w, _ = x.shape
    out = torch.zeros((n, hout, wout, phases[0][2].shape[1]), dtype=torch.float64, device=x.device)
    for (py, px), taps, wp in phases:
        if mutant == "phase_out_o_swapped" and (py, px) in ((0, 1), (1, 0)):
            py, px = px, py
        v = epi(tap_conv64(x, taps, wp, (1, 1), h, w))
        ly, lx = len(range(py, hout, 2)), len(range(px, wout, 2))
        out[:, py::2, px::2] = v[:, :ly, :lx]
    return out


def d2s_scatter64(v, no, hout, wout, out_o=(0, 0)):
    """the depth-to-space store: v (n, hog, wog, 32) columns q = pos * no + k -> pixel (2 gy + oy0 + pos // 2, 2 gx + ox0 +
    pos % 2), channel k, each position clipped to hout x wout -> (values, written mask), both (n, hout, wout, no)"""
    n, hog, wog, _ = v.shape
    out = torch.zeros((n, hout, wout, no), dtype=torch.float64, device=v.device)
    written = torch.zeros(out.shape, dtype=torch.bool, device=v.device)
    for pos in range(4):
        y0, x0 = out_o[0] + pos // 2, out_o[1] + pos % 2
        ys, xs = list(range(y0, hout, 2))[:hog], list(range(x0, wout, 2))[:wog]
        if ys and xs:
            blk = v[:, :len(ys), :len(xs), pos * no:(pos + 1) * no]
            out[:, y0:y0 + 2 * len(ys):2, x0:x0 + 2 * len(xs):2] = blk
            written[:, y0:y0 + 2 * len(ys):2, x0:x0 + 2 * len(xs):2] = True
    return out, written


def pair_ref64(x, w1, b1, w2, t2, dil, res=None, relu=True, h16=torch.float16):
    """lavb_conv_pair_umma in float64: x (n, h, w, c) 16-bit values, w1 / w2 (3, c, c) [tap][cout][cin] -> (n, h, w, c).
    mid = fmax0(h16(conv3x1_dil(x) + b1)); a = h16(conv1x3_dil(mid) + shift2); with a residual h16(a + res) saturating;
    relu: fmax0.  The NaN rule is tap_conv64's, and every ReLU turns a NaN into 0."""
    rnd = lambda v: v.clamp(-65504, 65504).to(h16).double() if h16 == torch.float16 else v.to(h16).double()  # noqa: E731
    a = tap_conv64(x, [((t - 1) * dil, 0) for t in range(3)], w1, (1, 1), x.shape[1], x.shape[2])
    mid = fmax0(rnd(a + b1.double().to(x.device)))
    a = rnd(tap_conv64(mid, [(0, (t - 1) * dil) for t in range(3)], w2, (1, 1), x.shape[1], x.shape[2]) + t2.double().to(x.device))
    if res is not None:
        a = rnd(a + res.double())
    return fmax0(a) if relu else a


def wgmma_err(got, want):
    """max |got - want| over the finite expected values as a fraction of their largest magnitude, after the NaN pattern,
    every infinite expected value and every saturated h16 one (+-65504) are matched exactly (inf when they are not)"""
    g, w = got.double().to(want.device), want
    if not torch.equal(torch.isnan(g), torch.isnan(w)):
        return math.inf
    inf = torch.isinf(w) | (w.abs() == 65504)          # infinities, and h16 stores the statement saturates: exact
    if not torch.equal(g[inf], w[inf]):
        return math.inf
    fin = ~inf & ~torch.isnan(w)
    if not bool(fin.any()):
        return 0.0
    if not bool(torch.isfinite(g[fin]).all()):
        return math.inf
    return float((g - w)[fin].abs().max() / (w[fin].abs().max() or 1.0))


def _taps(k, pad, dil=1):
    kh, kw = (k, k) if isinstance(k, int) else k
    ph, pw = (pad, pad) if isinstance(pad, int) else pad
    return [(ky * dil - ph, kx * dil - pw) for ky in range(kh) for kx in range(kw)]


# lavb_conv_umma cases of tests/test_gpu_wgmma_contract.py (one call each; the transposed phases are UMMA_CONVT).  Defaults:
# n 2, 13 x 21 input, cin 64 -> cout 64, 3 x 3 taps with padding 1, stride 1, bias + affine, pre-ReLU, fp32 output.
UMMA_CASES = {
    # input strides the product does not use: asymmetric, and the entry's maximum 8 (a 1 x 1 and a 3 x 3 tap set)
    "in_s21": dict(in_s=(2, 1), hin=17, win=19, cin=128, out="h16"),
    "in_s13": dict(in_s=(1, 3), hin=11, win=40, res=True, post=True),
    "in_s8_1x1": dict(in_s=(8, 8), k=1, pad=0, hin=41, win=70, cout=96),
    "in_s8_3x3": dict(in_s=(8, 8), hin=35, win=131, cin=128, cout=32, out="h16", res=True),
    # weight rows past cout (cout_mma = 32, 32, 64, 256) hold NaN, which must never reach a stored channel
    "pad_rows_cout8": dict(cout=8, pad_nan=True),
    "pad_rows_cout16": dict(cout=16, pad_nan=True, out="h16", pre=False, post=True),
    "pad_rows_cout40": dict(cout=40, pad_nan=True, out_cs=56, out_off=8),
    "pad_rows_cout248": dict(cout=248, pad_nan=True, cin=128, out="h16"),
    # a residual slice (the mutant reads it 8 channels further on) and the sigmoid
    "res_slice": dict(cout=96, res=True, res_cs=120, res_off=16, post=True, out="h16"),
    "sigmoid": dict(cout=32, pre=False, sig=True),
    # one NaN pixel and one +-inf pixel, without / with the ReLUs, both outputs; a negative scale on some channels
    "nan_plain_f32": dict(nan=True, pre=False, neg_scale=True),
    "nan_plain_h16": dict(nan=True, pre=False, neg_scale=True, out="h16", res=True),
    "nan_pre": dict(nan=True, neg_scale=True),
    "nan_post": dict(nan=True, pre=False, post=True, res=True, out="h16"),
    "inf_plain_h16": dict(inf=True, pre=False, out="h16"),
    "inf_pre_post": dict(inf=True, post=True, neg_scale=True),
    "nan_inf_sigmoid": dict(nan=True, inf=True, pre=False, sig=True, cout=32),
}


class UmmaCase:
    """the seeded CPU operands of one lavb_conv_umma call, h16 values as the kernel reads them (float32 tensors holding
    16-bit values of the type ``h16``), and its statement"""

    def __init__(self, name, h16=torch.float16, n=2, hin=13, win=21, cin=64, cout=64, k=3, pad=1, in_s=(1, 1), in_cs=None, in_off=0,
                 out_cs=None, out_off=0, res=False, res_cs=None, res_off=0, bias=True, affine=True, neg_scale=False, pre=True,
                 post=False, sig=False, out="f32", nan=False, inf=False, pad_nan=False):
        g = synth._gen(57, f"umma:{name}")
        self.name, self.n, self.cin, self.cout, self.in_s, self.out = name, n, cin, cout, in_s, out
        self.in_off, self.out_off, self.res_off = in_off, out_off, res_off
        self.in_cs, self.out_cs, self.res_cs = in_cs or cin, out_cs or cout, res_cs or cout
        self.pre, self.post, self.sig = pre, post, sig
        self.taps = _taps(k, pad)
        kh = kw = k
        self.hog = (hin + 2 * pad - kh) // in_s[0] + 1
        self.wog = (win + 2 * pad - kw) // in_s[1] + 1
        rnd = lambda t: t.to(h16).float()                                      # noqa: E731
        x = torch.randn(n, hin, win, self.in_cs, generator=g)
        if nan:
            x[1, hin // 2, win // 3, in_off + 5] = math.nan
        if inf:
            x[0, 1, win - 2, in_off + 7] = math.inf
            x[1, hin - 1, 2, in_off + 60] = -math.inf
        self.x = rnd(x)
        cm = (cout + 31) // 32 * 32
        w = torch.full((len(self.taps), cm, cin), math.nan if pad_nan else 0.0)
        w[:, :cout] = torch.randn(len(self.taps), cout, cin, generator=g) / (cin * len(self.taps)) ** 0.5
        self.w = rnd(w)
        self.bias = torch.randn(cout, generator=g) if bias else None
        self.scale = torch.rand(cout, generator=g) + 0.5 if affine else None
        if affine and neg_scale:
            self.scale[::3] *= -1
        self.shift = torch.randn(cout, generator=g) if affine else None
        self.res = rnd(torch.randn(n, self.hog, self.wog, self.res_cs, generator=g)) if res else None

    def want(self, mutant=None):
        """(n, hog, wog, cout) float64: the statement on the output lattice (out_s 1 here: the whole hog x wog map)"""
        a = tap_conv64(self.x[..., self.in_off:self.in_off + self.cin].double(), self.taps, self.w[:, :self.cout], self.in_s,
                       self.hog, self.wog, mutant)
        ro = self.res_off + (8 if mutant == "res_slice_off8" else 0)
        r = None if self.res is None else self.res[..., ro:ro + self.cout]
        v = wgmma_epilogue64(a, self.bias, self.scale, self.shift, r, self.pre, self.post, self.sig, mutant)
        return store64(v, self.out)


# the two UpsamplerBlocks of ERFNet's decoder at the agent's 288 x 256 frames (ConvTranspose2d(k3, s2, p1, op1) + BatchNorm +
# ReLU: bias, affine and post-ReLU), and the 64 -> 16 one on an odd output (output_padding 0: hout = 2h - 1, wout = 2w - 1),
# where the odd phases' last row / column falls outside the map
UMMA_CONVT = {"erf_up128_64": dict(cin=128, cout=64, h=36, w=32, op=1), "erf_up64_16": dict(cin=64, cout=16, h=72, w=64, op=1),
              "erf_up64_16_odd": dict(cin=64, cout=16, h=9, w=13, op=0)}


class ConvTCase:
    """the seeded CPU operands of one transposed convolution run as four lavb_conv_umma phase calls"""

    def __init__(self, name, h16=torch.float16, cin=64, cout=16, h=9, w=13, op=1, n=2):
        g = synth._gen(58, f"convT:{name}")
        rnd = lambda t: t.to(h16).float()                                      # noqa: E731
        self.n, self.cin, self.cout, self.h, self.w = n, cin, cout, h, w
        self.hout, self.wout = 2 * h - 1 + op, 2 * w - 1 + op
        self.x = rnd(torch.randn(n, h, w, cin, generator=g))
        self.wt = rnd(torch.randn(cin, cout, 3, 3, generator=g) / (cin * 2.25) ** 0.5)
        self.bias = torch.randn(cout, generator=g)
        self.scale, self.shift = torch.rand(cout, generator=g) + 0.5, torch.randn(cout, generator=g)
        self.phases = convT_phases(self.wt)

    def epi(self, a, mutant=None):
        return wgmma_epilogue64(a, self.bias, self.scale, self.shift, None, False, True, False, mutant)

    def want(self, mutant=None):
        """(n, hout, wout, cout) float64, fp32 output"""
        return convT_assemble64(self.x.double(), self.phases, self.hout, self.wout, lambda a: self.epi(a, mutant), mutant)


# the mutant each statement must tell apart, and the case it is shown at (the GPU test's inputs)
WGMMA_MUTANT_CASES = {"k_chunk_dropped": ("umma", "in_s21"), "tap_shifted": ("umma", "pad_rows_cout40"),
                      "phase_out_o_swapped": ("convT", "erf_up64_16_odd"), "bias_after_pre_relu": ("umma", "in_s13"),
                      "res_slice_off8": ("umma", "res_slice"), "nan_to_neg_inf": ("umma", "nan_plain_h16")}


def pack_d2s(wt, no):
    """ConvTranspose2d(cin, no, 3, stride 2, padding 1, output_padding 1) weight (cin, no, 3, 3) -> the 2 x 2-tap GEMM operand
    [tap = dy*2 + dx][column = pos*no + k][cin] of lavb_conv_umma's depth-to-space epilogue (taps (0,0), (0,1), (1,0), (1,1)),
    zero in the columns past 4 no"""
    wu = torch.zeros((4, 32, wt.shape[0]), dtype=wt.dtype, device=wt.device)
    opts = {0: [(0, 1)], 1: [(0, 2), (1, 0)]}
    for pa in (0, 1):
        for pb in (0, 1):
            for dy, ky in opts[pa]:
                for dx, kx in opts[pb]:
                    wu[dy * 2 + dx, (pa * 2 + pb) * no:(pa * 2 + pb + 1) * no] = wt[:, :, ky, kx].t()
    return wu
