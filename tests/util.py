"""Shared builders for the tests: seeded weights (identical in the pin script) and inputs."""
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
