"""Torch-tensor front ends of the C-ABI kernels (device pointers + current stream in, tensors out).

PyTorch is plumbing here: allocation, streams, views.  Every function launches hand-written
sm_90a kernels through lav_b200.capi; nothing falls back to torch math.
"""
import ctypes as C
import math

import numpy as np
import torch

from . import capi
from .capi import BF16, F16, F32, ConvDesc, check, lib

_DT = {torch.float32: F32, torch.bfloat16: BF16, torch.float16: F16}


def h16():
    """torch dtype of the library's 16-bit storage type: float16 (fp32 accumulation, saturating stores) unless the library was
    built with -DLAVB_H16_BF16."""
    return torch.float16 if capi.h16_code() == F16 else torch.bfloat16



def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise capi.LavbError("lav_b200 kernels need CUDA tensors (there is no CPU fallback)")


def _require(ok, msg):
    """argument checks that protect memory: a LavbError, never an assert (python -O strips asserts)."""
    if not ok:
        raise capi.LavbError(msg)


def launches():
    """number of kernel launches issued through this module (bench.py reports it)."""
    return _COUNT[0]


_COUNT = [0]
PROFILE = None     # bench.py sets this to a list to collect (kind, work, start_event, end_event) per launch


def _prof_begin():
    if PROFILE is None:
        return None
    e = torch.cuda.Event(enable_timing=True)
    e.record()
    return e


def _prof_end(kind, work, e0):
    if e0 is not None:
        e1 = torch.cuda.Event(enable_timing=True)
        e1.record()
        PROFILE.append((kind, work, e0, e1))


# ----------------------------------------------------------------------------- painting
def paint(points, sem, cams, mode, copy_cols=0, out=None, out_col0=None):
    """points (N,>=3) fp32; sem (ncam,C,H,W)-shaped tensor with ANY strides (NCHW or channels-last);
    cams (ncam,41) float32 numpy (K|lidar_to_world|world_to_cam).  See lavb_paint in include/lav_b200.h."""
    _need_cuda(points, sem)
    assert points.dtype == torch.float32 and sem.dtype == torch.float32 and points.dim() == 2
    assert points.stride(1) == 1
    ncam, c_in, h, w = sem.shape
    c_out = c_in if mode == 0 else c_in - 1
    n = points.shape[0]
    if out_col0 is None:
        out_col0 = copy_cols
    if out is None:
        out = torch.empty((n, out_col0 + c_out), dtype=torch.float32, device=points.device)
    assert out.stride(1) == 1
    cams = np.ascontiguousarray(cams, dtype=np.float32)
    assert cams.shape == (ncam, 41)
    s = sem.stride()
    check(lib().lavb_paint(_ptr(points), n, points.stride(0), _ptr(sem), ncam, c_in, h, w, s[0], s[1], s[2], s[3],
                           cams.ctypes.data_as(C.c_void_p), mode, _ptr(out), out.stride(0), out_col0, copy_cols, _stream()),
          "lavb_paint")
    _COUNT[0] += 1
    return out


def stack_sweep(src, R, dx, dy, time_idx, n_time, dst, roof_filter=False):
    """dst (n, src_cols+n_time) <- [src[:, :3] @ R + (dx,dy,0) | src[:,3:] | one_hot(time_idx)]"""
    _need_cuda(src, dst)
    assert src.is_contiguous() and dst.is_contiguous() and dst.shape == (src.shape[0], src.shape[1] + n_time)
    R = np.ascontiguousarray(R, dtype=np.float32)
    check(lib().lavb_stack_sweep(_ptr(src), src.shape[0], src.shape[1], R.ctypes.data_as(C.c_void_p), float(dx), float(dy),
                                 time_idx, n_time, int(roof_filter), _ptr(dst), _stream()), "lavb_stack_sweep")
    _COUNT[0] += 1
    return dst


def roof_filter(sweeps, pad_nan=False, out=None):
    """LAVAgent.preprocess (lav_agent.py:448-457) on the device, order preserving.  sweeps: (n, cols) or (F, n, cols) fp32
    contiguous -> (out like sweeps with the kept rows first, counts (F,) int32).  pad_nan fills rows past the count with NaN."""
    _need_cuda(sweeps)
    assert sweeps.dtype == torch.float32 and sweeps.is_contiguous() and sweeps.dim() in (2, 3)
    x = sweeps if sweeps.dim() == 3 else sweeps[None]
    f, n, cols = x.shape
    if out is None:
        out = torch.empty_like(x)
    assert out.is_contiguous() and out.shape == x.shape and out.data_ptr() != x.data_ptr()
    counts = torch.empty((f,), dtype=torch.int32, device=x.device)
    check(lib().lavb_roof_filter(_ptr(x), f, n, cols, n * cols, _ptr(out), n * cols, _ptr(counts), int(pad_nan), _stream()),
          "lavb_roof_filter")
    _COUNT[0] += 1
    return (out if sweeps.dim() == 3 else out[0]), counts


# ----------------------------------------------------------------------------- pillars
def _workspace(device, nbytes):
    """scratch for one call.  Deliberately NOT cached globally: under CUDA-graph capture the buffer must belong to the
    capturing graph's private pool (two pipelines replaying on different streams must never share scratch); the
    caching allocator makes the eager-mode cost negligible."""
    return torch.empty(int(nbytes), dtype=torch.uint8, device=device)


def _clouds(starts, counts, pts, what):
    """host arrays of the cloud table; raises LavbError when a cloud reaches past the last row of pts (the kernels read
    rows start .. start + count - 1 without a bound)."""
    b = len(counts)
    starts, counts = [int(s) for s in starts], [int(c) for c in counts]
    if len(starts) != b:
        raise capi.LavbError(f"{what}: {len(starts)} starts for {b} counts")
    for i, (s, c) in enumerate(zip(starts, counts)):
        if c > 0 and s + c > pts.shape[0]:
            raise capi.LavbError(f"{what}: cloud {i} = rows [{s}, {s + c}) lies past the {pts.shape[0]} rows of pts")
    st = (C.c_longlong * b)(*starts)
    ct = (C.c_int * b)(*counts)
    return b, st, ct


def _check_point_mlp(what, pts, w1, s1, t1, w2, s2, t2):
    """the encoders are built for the v2 point MLP only: w1 (64, 16), w2 (64, 64), s / t (64,), contiguous fp32 on pts' device,
    and rows of pts at least 11 floats wide."""
    for name, t, shape in (("w1", w1, (64, 16)), ("s1", s1, (64,)), ("t1", t1, (64,)), ("w2", w2, (64, 64)), ("s2", s2, (64,)),
                           ("t2", t2, (64,))):
        if (not torch.is_tensor(t) or tuple(t.shape) != shape or t.dtype != torch.float32 or not t.is_contiguous()
                or t.device != pts.device):
            got = f"{t.dtype} {tuple(t.shape)}" if torch.is_tensor(t) else type(t).__name__
            raise capi.LavbError(f"{what}: {name} must be a contiguous fp32 {shape} tensor on {pts.device}, got {got}")
    if pts.shape[1] < 11:
        raise capi.LavbError(f"{what}: point rows must hold at least 11 floats, got {pts.shape[1]}")


def pillar_forward(pts, starts, counts, grid, w1, s1, t1, w2, s2, t2):
    """pts: 2-D fp32 row buffer (rows of >= D floats); cloud b = rows [starts[b], starts[b]+counts[b]).
    Returns the NHWC canvas (B, ny, nx, H2) fp32."""
    _need_cuda(pts, w1, w2)
    assert pts.dtype == torch.float32 and pts.dim() == 2 and pts.stride(1) == 1
    _check_point_mlp("pillar_forward", pts, w1, s1, t1, w2, s2, t2)
    min_x, max_x, min_y, max_y, ppm, nx, ny = grid
    d = w1.shape[1] - 5
    b, st, ct = _clouds(starts, counts, pts, "pillar_forward")
    canvas = torch.empty((b, ny, nx, w2.shape[0]), dtype=torch.float32, device=pts.device)
    ws = _workspace(pts.device, lib().lavb_pillar_workspace_bytes(b, nx, ny))
    e0 = _prof_begin()
    check(lib().lavb_pillar_forward(_ptr(pts), pts.stride(0), d, st, ct, b, min_x, max_x, min_y, max_y, ppm, nx, ny,
                                    _ptr(w1), _ptr(s1), _ptr(t1), w1.shape[0], _ptr(w2), _ptr(s2), _ptr(t2), w2.shape[0],
                                    _ptr(canvas), F32, _ptr(ws), _stream()), "lavb_pillar_forward")
    # algorithmic bytes (SURVEY 8d): read P x D fp32 points once + write the canvas once
    _prof_end("pillar", float(sum(int(c) for c in counts)) * d * 4 + canvas.numel() * 4, e0)
    _COUNT[0] += 4
    return canvas


def pillar_decorate(pts, starts, counts, grid, d):
    """training stage 0: returns (feat (M,d+5) fp32, cell (M,) int32), rows in input order (clouds in batch order)."""
    _need_cuda(pts)
    assert pts.dtype == torch.float32 and pts.dim() == 2 and pts.stride(1) == 1
    min_x, max_x, min_y, max_y, ppm, nx, ny = grid
    b, st, ct = _clouds(starts, counts, pts, "pillar_decorate")
    ws = _workspace(pts.device, lib().lavb_pillar_workspace_bytes(b, nx, ny))
    total = int(sum(int(c) for c in counts))
    feat = torch.empty((total, d + 5), dtype=torch.float32, device=pts.device)
    cell = torch.empty((total,), dtype=torch.int32, device=pts.device)
    m = C.c_int(0)
    check(lib().lavb_pillar_decorate(_ptr(pts), pts.stride(0), d, st, ct, b, min_x, max_x, min_y, max_y, ppm, nx, ny,
                                     _ptr(feat), _ptr(cell), C.byref(m), _ptr(ws), _stream()), "lavb_pillar_decorate")
    _COUNT[0] += 4
    return feat[:m.value], cell[:m.value]


def pillar_scatter_max(h, cell, n_cells, want_argmax=True):
    """training stage 1: h (M,C) fp32 >= 0, cell (M,) int32 in [0, n_cells) -> (canvas (n_cells,C) fp32, arg (n_cells,C) int32
    or None).  See lavb_pillar_scatter_max in include/lav_b200.h for the tie rule and the empty-cell values."""
    _need_cuda(h, cell)
    assert h.dtype == torch.float32 and h.dim() == 2, "h must be (M, C) fp32"
    assert cell.dtype == torch.int32 and cell.shape == (h.shape[0],) and cell.is_contiguous(), "cell must be (M,) int32"
    assert cell.device == h.device and int(n_cells) >= 0
    h = h.contiguous()
    m, c = h.shape
    canvas = torch.empty((n_cells, c), dtype=torch.float32, device=h.device)
    arg = torch.empty((n_cells, c), dtype=torch.int32, device=h.device) if want_argmax else None
    check(lib().lavb_pillar_scatter_max(_ptr(h), _ptr(cell), m, c, n_cells, _ptr(canvas), _ptr(arg), _stream()),
          "lavb_pillar_scatter_max")
    _COUNT[0] += 2
    return canvas, arg


def pillar_scatter_max_bwd(gcanvas, arg, cell, m):
    """gh (m,C) fp32: gh[r, c] = gcanvas[cell[r], c] where arg[cell[r], c] == r, else 0.  gcanvas may have any strides."""
    _need_cuda(gcanvas, arg, cell)
    assert gcanvas.dtype == torch.float32 and gcanvas.dim() == 2, "gcanvas must be (n_cells, C) fp32"
    assert arg.dtype == torch.int32 and arg.shape == gcanvas.shape and arg.is_contiguous(), "arg must be (n_cells, C) int32"
    assert cell.dtype == torch.int32 and cell.shape == (m,) and cell.is_contiguous(), "cell must be (m,) int32"
    assert gcanvas.device == arg.device == cell.device
    gcanvas = gcanvas.contiguous()
    c = gcanvas.shape[-1]
    gh = torch.empty((m, c), dtype=torch.float32, device=gcanvas.device)
    check(lib().lavb_pillar_scatter_max_bwd(_ptr(gcanvas), _ptr(arg), _ptr(cell), m, c, _ptr(gh), _stream()),
          "lavb_pillar_scatter_max_bwd")
    _COUNT[0] += 1
    return gh


# ----------------------------------------------------------------------------- convolution
def conv_taps(x, cin, in_coff, out, cout, out_coff, hog, wog, in_s, out_s, out_o, taps, w, bias=None, scale=None, shift=None,
              res=None, res_coff=0, pre_relu=False, post_relu=False, sigmoid=False, umma=False, d2s_nout=0):
    """x, out, res: contiguous NHWC buffers (N,H,W,Ctot).  taps: list of (dy,dx).
    umma=False: CUDA-core kernel, w (ntaps,cin,cout_pad16) fp32.
    umma=True : wgmma kernel, x f16, w (ntaps,cout,cin) f16."""
    _need_cuda(x, out, w)
    assert x.is_contiguous() and out.is_contiguous() and w.is_contiguous()
    d = ConvDesc()
    d.inp, d.in_dtype = x.data_ptr(), _DT[x.dtype]
    d.n, d.hin, d.win, d.in_cstride = x.shape
    d.cin, d.in_coff = cin, in_coff
    d.out, d.out_dtype = out.data_ptr(), _DT[out.dtype]
    assert out.shape[0] == x.shape[0]
    _, d.hout, d.wout, d.out_cstride = out.shape
    d.cout, d.out_coff = cout, out_coff
    d.d2s_nout = d2s_nout
    if d2s_nout:
        assert umma and out.dtype == torch.float32 and out.shape[3] == d2s_nout and cout == 32 and 4 * d2s_nout <= 32
        d.out_cstride, d.out_coff = 32, 0        # (validated as a 32-column GEMM; addressing is done by the d2s epilogue)
    d.hog, d.wog = hog, wog
    d.in_sy, d.in_sx = in_s
    d.out_sy, d.out_sx = out_s
    d.out_oy, d.out_ox = out_o
    d.ntaps = len(taps)
    if umma:
        assert w.dtype == h16() and tuple(w.shape) == (len(taps), (cout + 31) // 32 * 32, cin) and x.dtype == h16()
    else:
        assert w.dtype == torch.float32 and tuple(w.shape) == (len(taps), cin, (cout + 15) // 16 * 16)
    for i, (dy, dx) in enumerate(taps):
        d.dy[i], d.dx[i] = dy, dx
    d.w = w.data_ptr()
    d.bias = bias.data_ptr() if bias is not None else None
    d.scale = scale.data_ptr() if scale is not None else None
    d.shift = shift.data_ptr() if shift is not None else None
    if res is not None:
        assert res.is_contiguous() and res.shape[:3] == out.shape[:3]
        d.res, d.res_dtype, d.res_cstride, d.res_coff = res.data_ptr(), _DT[res.dtype], res.shape[3], res_coff
    d.pre_relu, d.post_relu, d.sigmoid = int(pre_relu), int(post_relu), int(sigmoid)
    if umma:
        e0 = _prof_begin()
        check(lib().lavb_conv_umma(C.byref(d), _stream()), "lavb_conv_umma")
        _prof_end(f"umma:{cin}->{cout}x{len(taps)}taps@{hog}x{wog}", 2.0 * x.shape[0] * hog * wog * cout * cin * len(taps), e0)
    else:
        check(lib().lavb_conv_taps(C.byref(d), _stream()), "lavb_conv_taps")
    _COUNT[0] += 1
    return out


def pool2_affine_relu(x, c, in_coff, scale, shift, out, out_coff):
    _need_cuda(x, out)
    n, h, w, cs = x.shape
    check(lib().lavb_pool2_affine_relu(_ptr(x), _DT[x.dtype], n, h, w, c, cs, in_coff, _ptr(scale), _ptr(shift), _ptr(out),
                                       out.shape[3], out_coff, _stream()), "lavb_pool2_affine_relu")
    _COUNT[0] += 1
    return out


def rgb_normalize(rgb, out_dtype=torch.float32):
    """uint8 (N,H,W,3) or float (N,3,H,W) in 0..255 -> NHWC4 normalised ((x/255-.5)*2, 4th channel 0)."""
    _need_cuda(rgb)
    if rgb.dtype == torch.uint8:
        assert rgb.dim() == 4 and rgb.shape[3] == 3
        n, h, w, _ = rgb.shape
        u8 = 1
        rgb = rgb.contiguous()
    else:
        assert rgb.dim() == 4 and rgb.shape[1] == 3
        n, _, h, w = rgb.shape
        u8 = 0
        rgb = rgb.float().contiguous()
    out = torch.empty((n, h, w, 4), dtype=out_dtype, device=rgb.device)
    check(lib().lavb_rgb_normalize(_ptr(rgb), u8, n, h, w, _ptr(out), _DT[out_dtype], _stream()), "lavb_rgb_normalize")
    _COUNT[0] += 1
    return out


def convert(src, dtype):
    _need_cuda(src)
    src = src.contiguous()
    if src.dtype == dtype:
        return src
    dst = torch.empty(src.shape, dtype=dtype, device=src.device)
    check(lib().lavb_convert(_ptr(src), _DT[src.dtype], _ptr(dst), _DT[dtype], src.numel(), _stream()), "lavb_convert")
    _COUNT[0] += 1
    return dst


def crop_supported(feats_nhwc):
    """True when lavb_crop_bilinear takes this (B,H,W,C) map as it is: contiguous and 16-byte aligned, fp32 with C a multiple
    of 4 or the 16-bit type with C a multiple of 8 (a thread moves 16 bytes of channels)."""
    vec = {torch.float32: 4, h16(): 8}.get(feats_nhwc.dtype)
    return (vec is not None and feats_nhwc.dim() == 4 and feats_nhwc.is_contiguous() and feats_nhwc.data_ptr() % 16 == 0
            and feats_nhwc.shape[3] > 0 and feats_nhwc.shape[3] % vec == 0)


def _crop_poses(what, frame_idx, theta, b):
    """the K crop poses as the kernels read them: frame_idx (K,) of any integer type -> int32 (values clamped to [0, B) first,
    as the kernels clamp, so an int64 index past the int32 range still means the last frame), theta (K,2,3) -> fp32; both
    contiguous.  Raises LavbError when they do not describe the same K crops."""
    if theta.dim() != 3 or tuple(theta.shape[1:]) != (2, 3):
        raise capi.LavbError(f"{what}: theta must be (K, 2, 3), got {tuple(theta.shape)}")
    k = theta.shape[0]
    if frame_idx.dim() != 1 or frame_idx.numel() != k:
        raise capi.LavbError(f"{what}: frame_idx {tuple(frame_idx.shape)} does not hold one frame per crop (K = {k})")
    if frame_idx.dtype.is_floating_point or frame_idx.dtype.is_complex or frame_idx.dtype == torch.bool:
        raise capi.LavbError(f"{what}: frame_idx must be an integer tensor, got {frame_idx.dtype}")
    if frame_idx.dtype != torch.int32:
        frame_idx = frame_idx.clamp(0, b - 1).to(torch.int32)
    return k, frame_idx.contiguous(), theta.float().contiguous()


def crop_bilinear(feats_nhwc, frame_idx, theta, crop_size):
    """feats_nhwc (B,H,W,C) contiguous fp32 (C % 4 == 0) or h16 (C % 8 == 0); frame_idx (K,) integer; theta (K,2,3) ->
    (K,crop,crop,C) in the feature dtype.  Frame indices outside [0, B) are clamped to the nearest frame."""
    _need_cuda(feats_nhwc, frame_idx, theta)
    if not crop_supported(feats_nhwc):
        raise capi.LavbError(f"crop_bilinear: need a contiguous, 16-byte aligned (B,H,W,C) map, fp32 with C % 4 == 0 or "
                             f"{h16()} with C % 8 == 0; got {feats_nhwc.dtype} {tuple(feats_nhwc.shape)}")
    b, h, w, c = feats_nhwc.shape
    k, frame_idx, theta = _crop_poses("crop_bilinear", frame_idx, theta, b)
    out = torch.empty((k, crop_size, crop_size, c), dtype=feats_nhwc.dtype, device=feats_nhwc.device)
    check(lib().lavb_crop_bilinear(_ptr(feats_nhwc), _DT[feats_nhwc.dtype], b, h, w, c, _ptr(frame_idx), _ptr(theta), k, crop_size,
                                   _ptr(out), _stream()), "lavb_crop_bilinear")
    _COUNT[0] += 1
    return out


def crop_bilinear_u8(bev_u8, frame_idx, theta, crop_size, out=None):
    """bev_u8 (B,C,H,W) contiguous uint8; frame_idx (K,) int32; theta (K,2,3) fp32 -> fp32 NCHW (K,C,crop,crop): the crops of
    crop_bilinear read straight from a uint8 planar map (bit-identical to crop_bilinear on its float copy).  Frame indices
    outside [0, B) are clamped to the nearest frame.  ``out`` (K,C,crop,crop) fp32 contiguous is written in full if given."""
    _need_cuda(bev_u8, frame_idx, theta)
    if bev_u8.dtype != torch.uint8 or bev_u8.dim() != 4:
        raise capi.LavbError(f"crop_bilinear_u8: need a 4-d uint8 map, got {bev_u8.dtype} {tuple(bev_u8.shape)}")
    if not bev_u8.is_contiguous():
        raise capi.LavbError("crop_bilinear_u8: the map must be contiguous (B,C,H,W)")
    b, c, h, w = bev_u8.shape
    k = theta.shape[0]
    if tuple(theta.shape) != (k, 2, 3) or frame_idx.numel() != k:
        raise capi.LavbError(f"crop_bilinear_u8: theta {tuple(theta.shape)} / frame_idx {tuple(frame_idx.shape)} do not describe K crops")
    theta = theta.float().contiguous()
    frame_idx = frame_idx.to(torch.int32).contiguous()
    if out is None:
        out = torch.empty((k, c, crop_size, crop_size), dtype=torch.float32, device=bev_u8.device)
    elif tuple(out.shape) != (k, c, crop_size, crop_size) or out.dtype != torch.float32 or not out.is_contiguous():
        raise capi.LavbError(f"crop_bilinear_u8: out must be a contiguous fp32 ({k}, {c}, {crop_size}, {crop_size}) tensor")
    check(lib().lavb_crop_bilinear_u8(_ptr(bev_u8), b, c, h, w, _ptr(frame_idx), _ptr(theta), k, crop_size, _ptr(out), _stream()),
          "lavb_crop_bilinear_u8")
    _COUNT[0] += 1
    return out


def crop_bilinear_bwd(gout_nhwc, frame_idx, theta, feat_shape, out=None):
    """gout_nhwc (K,crop,crop,C) fp32 contiguous -> gradient of crop_bilinear w.r.t. the (B,H,W,C) fp32 feature map.
    ``out`` (B,H,W,C) fp32 contiguous is written in full if given (zeros for every frame no crop samples)."""
    _need_cuda(gout_nhwc, frame_idx, theta)
    if len(feat_shape) != 4:
        raise capi.LavbError(f"crop_bilinear_bwd: feat_shape must be (B, H, W, C), got {tuple(feat_shape)}")
    b, h, w, c = (int(v) for v in feat_shape)
    if gout_nhwc.dtype != torch.float32 or gout_nhwc.dim() != 4 or not gout_nhwc.is_contiguous() or gout_nhwc.data_ptr() % 16:
        raise capi.LavbError(f"crop_bilinear_bwd: gout must be a contiguous, 16-byte aligned fp32 (K, crop, crop, C) tensor, "
                             f"got {gout_nhwc.dtype} {tuple(gout_nhwc.shape)}")
    k, frame_idx, theta = _crop_poses("crop_bilinear_bwd", frame_idx, theta, b)
    crop = gout_nhwc.shape[1]
    if tuple(gout_nhwc.shape) != (k, crop, crop, c):
        raise capi.LavbError(f"crop_bilinear_bwd: gout {tuple(gout_nhwc.shape)} does not match {k} square crops of the "
                             f"{c}-channel map {tuple(feat_shape)}")
    if out is None:
        gfeat = torch.empty((b, h, w, c), dtype=torch.float32, device=gout_nhwc.device)
    elif tuple(out.shape) != (b, h, w, c) or out.dtype != torch.float32 or not out.is_contiguous() or out.device != gout_nhwc.device:
        raise capi.LavbError(f"crop_bilinear_bwd: out must be a contiguous fp32 ({b}, {h}, {w}, {c}) tensor on {gout_nhwc.device}")
    else:
        gfeat = out
    check(lib().lavb_crop_bilinear_bwd(_ptr(gout_nhwc), b, h, w, c, _ptr(frame_idx), _ptr(theta), k, crop, _ptr(gfeat), _stream()),
          "lavb_crop_bilinear_bwd")
    _COUNT[0] += 1
    return gfeat


class CropBilinear(torch.autograd.Function):
    """crop_bilinear with its hand-written backward (gradient to the feature map only: the crop poses are data)."""

    @staticmethod
    def forward(ctx, feats_nhwc, frame_idx, theta, crop_size):
        _need_cuda(frame_idx, theta)
        _, frame_idx, theta = _crop_poses("CropBilinear", frame_idx, theta.detach(), feats_nhwc.shape[0])
        ctx.save_for_backward(frame_idx, theta)
        ctx.feat_shape = tuple(feats_nhwc.shape)
        return crop_bilinear(feats_nhwc, frame_idx, theta, crop_size)

    @staticmethod
    def backward(ctx, gout):
        frame_idx, theta = ctx.saved_tensors
        return crop_bilinear_bwd(gout.contiguous(), frame_idx, theta, ctx.feat_shape), None, None, None


def deconv3x3s2_small(x, groups, cin_g, w, bias, n_outs, sigmoids):
    """x NHWC (N,H,W,Ctot); w fp32 (G,cin_g,9,4); bias (G,4) -> list of fp32 NHWC (N,2H,2W,n_out[g])."""
    _need_cuda(x, w, bias)
    assert x.is_contiguous() and w.is_contiguous() and bias.is_contiguous()
    n, h, wd, cs = x.shape
    outs = [torch.empty((n, 2 * h, 2 * wd, no), dtype=torch.float32, device=x.device) for no in n_outs]
    ptrs = (C.c_void_p * groups)(*[o.data_ptr() for o in outs])
    no = (C.c_int * groups)(*n_outs)
    sg = (C.c_int * groups)(*[int(s) for s in sigmoids])
    check(lib().lavb_deconv3x3s2_small(_ptr(x), _DT[x.dtype], n, h, wd, cs, groups, cin_g, _ptr(w), _ptr(bias), no, sg, ptrs,
                                       _stream()), "lavb_deconv3x3s2_small")
    _COUNT[0] += 1
    return outs


def paint_batched(points, sem, cams, mode, copy_cols, out):
    """points (F,N,>=3) fp32 contiguous; sem logical (F,ncam,C,H,W) any strides; out (F,N,copy_cols+c_out) contiguous."""
    _need_cuda(points, sem, out)
    assert points.is_contiguous() and out.is_contiguous() and points.dtype == torch.float32 and sem.dtype == torch.float32
    f, n, ps = points.shape
    _, ncam, c_in, h, w = sem.shape
    cams = np.ascontiguousarray(cams, dtype=np.float32)
    s = sem.stride()
    check(lib().lavb_paint_batched(_ptr(points), f, n, ps, n * ps, _ptr(sem), ncam, c_in, h, w, s[0], s[1], s[2], s[3], s[4],
                                   cams.ctypes.data_as(C.c_void_p), mode, _ptr(out), out.shape[2], n * out.shape[2], copy_cols,
                                   copy_cols, _stream()), "lavb_paint_batched")
    _COUNT[0] += 1
    return out


def pack_deconv2x2(weight, bias):
    """ConvTranspose2d(16, C, 2, stride=2) parameters (weight (16,C,2,2), bias (C,)) -> the 520-float table
    lavb_paint_deconv_batched reads: w[v%2][u%2][c_in][8] | bias[8]."""
    cin, c, kh, kw = weight.shape
    assert cin == 16 and kh == 2 and kw == 2 and c <= 8
    w = torch.zeros((2, 2, 16, 8), dtype=torch.float32, device=weight.device)
    w[:, :, :, :c] = weight.detach().float().permute(2, 3, 0, 1)
    b = torch.zeros((8,), dtype=torch.float32, device=weight.device)
    b[:c] = bias.detach().float()
    return torch.cat([w.reshape(-1), b]).contiguous()


def paint_deconv_batched(points, feat, n_classes, deconv, cams, copy_cols, out, image_hw):
    """points (F,N,>=3) fp32; feat NHWC (F*ncam, H/2, W/2, 16) fp32 / h16 = ERFNet decoder output before output_conv;
    deconv = pack_deconv2x2(...); out (F,N,copy_cols + n_classes-1)."""
    _need_cuda(points, feat, out, deconv)
    assert points.is_contiguous() and out.is_contiguous() and feat.is_contiguous() and points.dtype == torch.float32
    f, n, ps = points.shape
    h, w = image_hw
    cams = np.ascontiguousarray(cams, dtype=np.float32)
    ncam = cams.shape[0]
    assert feat.shape == (f * ncam, h // 2, w // 2, 16) and deconv.numel() == 520
    check(lib().lavb_paint_deconv_batched(_ptr(points), f, n, ps, n * ps, _ptr(feat), _DT[feat.dtype], ncam, n_classes, h, w,
                                          _ptr(deconv), cams.ctypes.data_as(C.c_void_p), _ptr(out), out.shape[2], n * out.shape[2],
                                          copy_cols, copy_cols, _stream()), "lavb_paint_deconv_batched")
    _COUNT[0] += 1
    return out


def sem_class_table(seg_channels):
    """filter_sem(sem, seg_channels) (lav/utils/__init__.py:3-8) as a lookup table: uint8 (256,) = the class of each CARLA tag, in
    that loop's order: an unlisted tag is class 0 and a later duplicate of a tag wins."""
    lut = np.zeros(256, np.uint8)
    for i, tag in enumerate(seg_channels):
        lut[int(tag)] = i + 1
    return lut


def seg_confusion(feat, table, labels, lut, n_classes, out=None):
    """Per-image confusion counts of ERFNet's class map in one launch (see lavb_seg_confusion in include/lav_b200.h).  feat NHWC
    (N, H/2, W/2, 16) fp32 / h16 = the input of output_conv (forward_features_nhwc); table = pack_deconv2x2 of output_conv; labels
    (N, H, W) uint8 = the recorded tags; lut = sem_class_table(seg_channels) on the host.  -> int32 (N, C*C + 1) = confusion[gt][pred]
    flattened, then the invalid (NaN-logit) pixels (written into ``out`` when given)."""
    _need_cuda(feat, table, labels)
    if feat.dtype not in (torch.float32, h16()) or feat.dim() != 4 or feat.shape[3] != 16 or not feat.is_contiguous():
        raise capi.LavbError(f"seg_confusion: feat must be a contiguous (N, H/2, W/2, 16) fp32 or {h16()} tensor, got {feat.dtype} "
                             f"{tuple(feat.shape)}")
    n, hh, wh, _ = feat.shape
    if labels.dtype != torch.uint8 or tuple(labels.shape) != (n, 2 * hh, 2 * wh) or not labels.is_contiguous():
        raise capi.LavbError(f"seg_confusion: labels must be a contiguous ({n}, {2 * hh}, {2 * wh}) uint8 tensor, got {labels.dtype} "
                             f"{tuple(labels.shape)}")
    if table.dtype != torch.float32 or table.numel() != 520 or not table.is_contiguous():
        raise capi.LavbError("seg_confusion: table must be the 520-float pack_deconv2x2 table")
    lut = np.ascontiguousarray(lut)
    if lut.dtype != np.uint8 or lut.shape != (256,):
        raise capi.LavbError(f"seg_confusion: lut must be a host (256,) uint8 array, got {lut.dtype} {lut.shape}")
    if len({feat.device, table.device, labels.device}) != 1:
        raise capi.LavbError("seg_confusion: the inputs must be on one device")
    c = int(n_classes)
    if out is None:
        out = torch.empty((n, c * c + 1), dtype=torch.int32, device=feat.device)
    elif out.dtype != torch.int32 or tuple(out.shape) != (n, c * c + 1) or not out.is_contiguous() or out.device != feat.device:
        raise capi.LavbError(f"seg_confusion: out must be a contiguous ({n}, {c * c + 1}) int32 tensor on {feat.device}")
    check(lib().lavb_seg_confusion(_ptr(feat), _DT[feat.dtype], _ptr(table), _ptr(labels), lut.ctypes.data_as(C.c_void_p), n, c,
                                   2 * hh, 2 * wh, _ptr(out), _stream()), "lavb_seg_confusion")
    _COUNT[0] += n > 0
    return out


PAINT_COUNTERS = ("points", "nan", "roof", "in_window", "not_visible", "not_visible_in_window", "invalid", "stored_invalid")
PAINT_RANGES_M = (10.0, 20.0, 40.0)      # the range bins' edges (horizontal distance), the last bin open


def paint_confusion_ints(ncam, n_classes, online, stored):
    """length of one frame's lavb_paint_confusion row."""
    per_src = ncam * (len(PAINT_RANGES_M) + 1) * 2 * n_classes * n_classes
    return len(PAINT_COUNTERS) + (int(online) + int(stored)) * per_src + (ncam * n_classes * n_classes if online and stored else 0)


def paint_confusion_views(counts, ncam, n_classes, online, stored):
    """views of paint_confusion rows (F, L) (torch or numpy): counters (F, 8) in PAINT_COUNTERS order, "online" / "stored"
    (F, ncam, 4, 2, C, C) = [camera][range bin][in window][recorded][predicted] for each scored source, and with both
    "agreement" (F, ncam, C, C) = [camera][online][stored]."""
    c, nr = n_classes, len(PAINT_RANGES_M) + 1
    per_src = ncam * nr * 2 * c * c
    views = dict(counters=counts[:, :len(PAINT_COUNTERS)])
    o = len(PAINT_COUNTERS)
    for name, on in (("online", online), ("stored", stored)):
        if on:
            views[name] = counts[:, o:o + per_src].reshape(-1, ncam, nr, 2, c, c)
            o += per_src
    if online and stored:
        views["agreement"] = counts[:, o:o + ncam * c * c].reshape(-1, ncam, c, c)
    return views


def paint_confusion(points, tags, lut, cams, window, n_classes, feat=None, table=None, stored=None, meta=None, out=None):
    """Per-frame confusion counts of the point painting against the recorded semantic cameras in one launch (see
    lavb_paint_confusion in include/lav_b200.h).  points (F, N, 4) fp32 = the NaN-padded sweeps; tags (F * ncam, H, W) uint8 =
    the recorded sem images; lut = sem_class_table(seg_channels) on the host; cams = the packed converters (ncam, 41); window =
    (min_x, max_x, min_y, max_y) of the pillar grid; feat NHWC (F * ncam, H/2, W/2, 16) fp32 / h16 with table = pack_deconv2x2
    (the online source) and / or stored (F, N, C - 1) fp32 = lidar_sem rows; meta (F, 2) int32 = (rows, stored scored) per frame
    or None.  -> int32 (F, paint_confusion_ints(...)) (written into ``out`` when given); paint_confusion_views splits it."""
    _need_cuda(points, tags, feat, table, stored, meta)
    c = int(n_classes)
    if points.dtype != torch.float32 or points.dim() != 3 or points.shape[2] != 4 or not points.is_contiguous():
        raise capi.LavbError(f"paint_confusion: points must be a contiguous (F, N, 4) fp32 tensor, got {points.dtype} "
                             f"{tuple(points.shape)}")
    f, n, _ = points.shape
    cams = np.ascontiguousarray(cams, dtype=np.float32)
    if cams.ndim != 2 or cams.shape[1] != 41 or not 1 <= cams.shape[0] <= 4:
        raise capi.LavbError(f"paint_confusion: cams must be (ncam, 41) with 1 <= ncam <= 4, got {cams.shape}")
    ncam = cams.shape[0]
    if tags.dtype != torch.uint8 or tags.dim() != 3 or tags.shape[0] != f * ncam or not tags.is_contiguous():
        raise capi.LavbError(f"paint_confusion: tags must be a contiguous ({f * ncam}, H, W) uint8 tensor, got {tags.dtype} "
                             f"{tuple(tags.shape)}")
    h, w = tags.shape[1:]
    if feat is None and stored is None:
        raise capi.LavbError("paint_confusion: give feat (the online painting), stored (lidar_sem rows) or both")
    if feat is not None:
        if feat.dtype not in (torch.float32, h16()) or tuple(feat.shape) != (f * ncam, h // 2, w // 2, 16) or not feat.is_contiguous():
            raise capi.LavbError(f"paint_confusion: feat must be a contiguous ({f * ncam}, {h // 2}, {w // 2}, 16) fp32 or {h16()} "
                                 f"tensor, got {feat.dtype} {tuple(feat.shape)}")
        if table is None or table.dtype != torch.float32 or table.numel() != 520 or not table.is_contiguous():
            raise capi.LavbError("paint_confusion: table must be the 520-float pack_deconv2x2 table")
    if stored is not None and (stored.dtype != torch.float32 or tuple(stored.shape) != (f, n, c - 1) or not stored.is_contiguous()):
        raise capi.LavbError(f"paint_confusion: stored must be a contiguous ({f}, {n}, {c - 1}) fp32 tensor, got {stored.dtype} "
                             f"{tuple(stored.shape)}")
    if meta is not None and (meta.dtype != torch.int32 or tuple(meta.shape) != (f, 2) or not meta.is_contiguous()):
        raise capi.LavbError(f"paint_confusion: meta must be a contiguous ({f}, 2) int32 tensor")
    lut = np.ascontiguousarray(lut)
    if lut.dtype != np.uint8 or lut.shape != (256,) or int(lut.max()) >= c:
        raise capi.LavbError(f"paint_confusion: lut must be a host (256,) uint8 array of classes below {c}, got {lut.dtype} "
                             f"{lut.shape}")
    if len({t.device for t in (points, tags, feat, table, stored, meta) if t is not None}) != 1:
        raise capi.LavbError("paint_confusion: the inputs must be on one device")
    ints = lib().lavb_paint_confusion_ints(ncam, c, feat is not None, stored is not None)
    if ints < 0:
        raise capi.LavbError(f"paint_confusion: {c} classes outside 2..8")
    if out is None:
        out = torch.empty((f, ints), dtype=torch.int32, device=points.device)
    elif out.dtype != torch.int32 or tuple(out.shape) != (f, ints) or not out.is_contiguous() or out.device != points.device:
        raise capi.LavbError(f"paint_confusion: out must be a contiguous ({f}, {ints}) int32 tensor on {points.device}")
    if n == 0:              # empty sweeps: every count is 0 (and an empty stored buffer has no device pointer to pass)
        return out.zero_()
    min_x, max_x, min_y, max_y = (float(v) for v in window)
    check(lib().lavb_paint_confusion(_ptr(points), f, n, _ptr(meta), _ptr(feat), _DT[feat.dtype] if feat is not None else F32,
                                     _ptr(table), _ptr(tags), lut.ctypes.data_as(C.c_void_p), _ptr(stored),
                                     cams.ctypes.data_as(C.c_void_p), ncam, c, h, w, min_x, max_x, min_y, max_y, _ptr(out),
                                     _stream()), "lavb_paint_confusion")
    _COUNT[0] += f > 0
    return out


STACK_JOB_DTYPE = np.dtype([("src", np.uint64), ("dst", np.uint64), ("n", np.int32), ("time_idx", np.int32), ("R", np.float32, 9),
                            ("dx", np.float32), ("dy", np.float32), ("pad", np.int32)])
assert STACK_JOB_DTYPE.itemsize == 72


def stack_jobs(d_jobs, n_jobs, max_n, src_cols, n_time, roof_filter=False):
    """d_jobs: uint8 device tensor holding n_jobs STACK_JOB_DTYPE records."""
    _need_cuda(d_jobs)
    check(lib().lavb_stack_jobs(_ptr(d_jobs), n_jobs, max_n, src_cols, n_time, int(roof_filter), _stream()), "lavb_stack_jobs")
    _COUNT[0] += 1


# ----------------------------------------------------------------------------- temporal BEV targets
BEV_JOB_DTYPE = np.dtype([("src", np.int64), ("dst", np.int64), ("m1", np.float64, 6), ("m2", np.float64, 6), ("dx", np.int32),
                          ("dy", np.int32), ("pad", np.int32, 2)])
assert BEV_JOB_DTYPE.itemsize == 128
BEV_MARGIN = 32                  # TemporalLiDARPaintedDataset.margin (lidar_painted_dataset.py:19)


def _inverse_rotation(angle_deg, center):
    """inverse of cv2.getRotationMatrix2D(center, angle, 1.0), computed as cv::warpAffine inverts it (same operation order, so
    the same fp64 roundings; math.cos / math.sin are the C library's, as OpenCV's)."""
    a = angle_deg * (math.pi / 180)
    c, s = math.cos(a), math.sin(a)
    cx, cy = center
    m = ((c, s, (1 - c) * cx - s * cy), (-s, c, s * cx + (1 - c) * cy))
    det = m[0][0] * m[1][1] - m[0][1] * m[1][0]
    d = 1.0 / det if det != 0 else 0.0
    a11, a22, a12, a21 = m[1][1] * d, m[0][0] * d, -m[0][1] * d, -m[1][0] * d
    return (a11, a12, -a11 * m[0][2] - a12 * m[1][2], a21, a22, -a21 * m[0][2] - a22 * m[1][2])


def bev_jobs(rows, center=(160, 280)):
    """rows of (src plane or -1, dst plane, first angle (deg), second angle (deg), dx, dy) -> BEV_JOB_DTYPE records for
    bev_targets: each output plane is rotate(src, angle1) -> shift by (dx rows, dy columns) -> rotate(., angle2) -> > 0."""
    jobs = np.zeros(len(rows), BEV_JOB_DTYPE)
    for k, (src, dst, a1, a2, dx, dy) in enumerate(rows):
        jobs[k] = (src, dst, _inverse_rotation(a1, center), _inverse_rotation(a2, center), dx, dy, (0, 0))
    return jobs


def bev_targets(src_planes, jobs, out=None):
    """The temporal BEV target planes (load_bev_channels, temporal_lidar_painted_dataset.py:182-198) in one launch.
    src_planes (P, h, w) uint8 CUDA; jobs: BEV_JOB_DTYPE records (see bev_jobs); out: uint8 CUDA tensor of (..., h, w) planes
    (default (max dst + 1, h, w)).  Every plane a job names is overwritten with 0/1; a missing source (src < 0) gives zeros.
    Raises LavbError for a shift beyond the 32-pixel margin, where the reference's crop fails."""
    _need_cuda(src_planes)
    assert src_planes.dtype == torch.uint8 and src_planes.dim() == 3 and src_planes.is_contiguous()
    jobs = np.ascontiguousarray(jobs, dtype=BEV_JOB_DTYPE)
    P, h, w = src_planes.shape
    if len(jobs) and (np.abs(jobs["dx"]).max() > BEV_MARGIN or np.abs(jobs["dy"]).max() > BEV_MARGIN):
        raise capi.LavbError(f"bev_targets: shift beyond the {BEV_MARGIN}-pixel margin "
                             f"(dx {jobs['dx'].tolist()}, dy {jobs['dy'].tolist()})")
    if out is None:
        out = torch.empty((int(jobs["dst"].max()) + 1 if len(jobs) else 0, h, w), dtype=torch.uint8, device=src_planes.device)
    _need_cuda(out)
    assert out.dtype == torch.uint8 and out.is_contiguous() and tuple(out.shape[-2:]) == (h, w)
    n_out = out.numel() // (h * w)
    if len(jobs) and (jobs["src"].max() >= P or jobs["dst"].min() < 0 or jobs["dst"].max() >= n_out):
        raise capi.LavbError(f"bev_targets: job plane index out of range ({P} source planes, {n_out} output planes)")
    if len(jobs) == 0:
        return out
    d_jobs = _to_device(jobs.view(np.uint8), src_planes.device)
    check(lib().lavb_bev_targets(_ptr(d_jobs), len(jobs), _ptr(src_planes), _ptr(out), h, w, _stream()), "lavb_bev_targets")
    _COUNT[0] += 1
    return out


PNG_JOB_DTYPE = np.dtype([("off", np.int64), ("len", np.int64), ("dst", np.int32), ("h", np.int32), ("w", np.int32),
                          ("pad", np.int32)])
assert PNG_JOB_DTYPE.itemsize == 32


def png_decode_gray8(src, jobs, out, status=None):
    """8-bit grayscale PNG images -> uint8 planes in one launch (see lavb_png_decode_gray8 in include/lav_b200.h), as
    cv2.imdecode(..., IMREAD_GRAYSCALE).  src: 1-D uint8 CUDA tensor of the images' zlib streams (their IDAT payloads,
    concatenated); jobs: PNG_JOB_DTYPE records (off, len, dst, h, w); out: contiguous (P, h, w) uint8 CUDA tensor, every job's (h, w)
    equal to its planes'.  -> status (n_jobs,) int32 on the device, 0 where the image decoded; a nonzero entry marks a malformed
    stream whose plane holds garbage.  The other planes of out are not written."""
    _need_cuda(src, out, status)
    if src.dtype != torch.uint8 or src.dim() != 1 or not src.is_contiguous():
        raise capi.LavbError(f"png_decode_gray8: src must be a contiguous 1-D uint8 tensor, got {src.dtype} {tuple(src.shape)}")
    if out.dtype != torch.uint8 or out.dim() != 3 or not out.is_contiguous() or out.device != src.device:
        raise capi.LavbError(f"png_decode_gray8: out must be a contiguous (P, h, w) uint8 tensor on {src.device}")
    jobs = np.ascontiguousarray(jobs, dtype=PNG_JOB_DTYPE)
    P, h, w = out.shape
    if not (0 < h <= 4096 and 0 < w <= 4096):
        raise capi.LavbError(f"png_decode_gray8: plane size {h}x{w} outside 1..4096")
    if len(jobs) and ((jobs["h"] != h).any() or (jobs["w"] != w).any()):
        raise capi.LavbError(f"png_decode_gray8: a job's size differs from the {h}x{w} planes")
    if len(jobs) and ((jobs["dst"] < 0).any() or (jobs["dst"] >= P).any() or len(np.unique(jobs["dst"])) != len(jobs)):
        raise capi.LavbError(f"png_decode_gray8: job planes must be distinct and in 0..{P - 1}")
    if len(jobs) and ((jobs["off"] < 0).any() or (jobs["len"] < 0).any() or (jobs["off"] + jobs["len"] > src.numel()).any()):
        raise capi.LavbError(f"png_decode_gray8: a job's stream lies outside the {src.numel()}-byte source")
    if status is None:
        status = torch.empty(len(jobs), dtype=torch.int32, device=src.device)
    elif status.dtype != torch.int32 or status.numel() != len(jobs) or not status.is_contiguous() or status.device != src.device:
        raise capi.LavbError(f"png_decode_gray8: status must be a contiguous ({len(jobs)},) int32 tensor on {src.device}")
    if len(jobs) == 0:
        return status
    d_jobs = _to_device(jobs.view(np.uint8), src.device)
    check(lib().lavb_png_decode_gray8(_ptr(src), src.numel(), _ptr(d_jobs), len(jobs), _ptr(out), P, h, w, _ptr(status), _stream()),
          "lavb_png_decode_gray8")
    _COUNT[0] += 1
    return status


def _to_device(a, device):
    """host array -> device tensor through pinned staging, without a host synchronisation (the pinned block is not reused
    before the copy has run: the caching host allocator records the copy's stream)."""
    return torch.from_numpy(np.ascontiguousarray(a)).pin_memory().to(device, non_blocking=True)


# ----------------------------------------------------------------------------- training batches
LIDAR_SWEEP_DTYPE = np.dtype([("R_aug", np.float32, 9), ("R_mv", np.float32, 9), ("dx", np.float32), ("dy", np.float32),
                              ("time_idx", np.int32), ("row0", np.int32)])
assert LIDAR_SWEEP_DTYPE.itemsize == 88


def lidar_batch(raw, rows, sweeps, cams, image_hw, n_time, out=None):
    """The LiDAR input of a training batch in one launch (see lavb_lidar_batch in include/lav_b200.h).  raw (N, 4+C) fp32: every
    sweep's rows [xyzr | painted]; rows (B, P) int32: the raw row of each output row, -1 for a zero row; sweeps: uint8 CUDA tensor
    of LIDAR_SWEEP_DTYPE records sorted by row0; cams (ncam, 41) float32 numpy; image_hw = the camera image size.
    -> (B, P, 4+C+n_time) fp32, bit-identical to GpuLidarStacker on each sample for the same shuffle."""
    _need_cuda(raw, rows, sweeps)
    if raw.dtype != torch.float32 or raw.dim() != 2 or not raw.is_contiguous() or raw.shape[1] < 4:
        raise capi.LavbError(f"lidar_batch: raw must be a contiguous (N, 4+C) fp32 tensor, got {raw.dtype} {tuple(raw.shape)}")
    if rows.dtype != torch.int32 or rows.dim() != 2 or not rows.is_contiguous():
        raise capi.LavbError(f"lidar_batch: rows must be a contiguous (B, P) int32 tensor, got {rows.dtype} {tuple(rows.shape)}")
    if sweeps.dtype != torch.uint8 or not sweeps.is_contiguous() or sweeps.numel() % LIDAR_SWEEP_DTYPE.itemsize:
        raise capi.LavbError("lidar_batch: sweeps must be a contiguous uint8 tensor of 88-byte LIDAR_SWEEP_DTYPE records")
    if not raw.device == rows.device == sweeps.device:
        raise capi.LavbError("lidar_batch: raw, rows and sweeps must be on one device")
    cams = np.ascontiguousarray(cams, dtype=np.float32)
    if cams.ndim != 2 or cams.shape[1] != 41:
        raise capi.LavbError(f"lidar_batch: cams must be (ncam, 41), got {cams.shape}")
    b, p = rows.shape
    c = raw.shape[1] - 4
    if out is None:
        out = torch.empty((b, p, 4 + c + n_time), dtype=torch.float32, device=raw.device)
    elif out.dtype != torch.float32 or tuple(out.shape) != (b, p, 4 + c + n_time) or not out.is_contiguous() \
            or out.device != raw.device:
        raise capi.LavbError(f"lidar_batch: out must be a contiguous fp32 ({b}, {p}, {4 + c + n_time}) tensor on {raw.device}")
    check(lib().lavb_lidar_batch(_ptr(raw), raw.shape[0], c, _ptr(rows), b * p, _ptr(sweeps),
                                 sweeps.numel() // LIDAR_SWEEP_DTYPE.itemsize, cams.ctypes.data_as(C.c_void_p), cams.shape[0],
                                 image_hw[0], image_hw[1], n_time, _ptr(out), _stream()), "lavb_lidar_batch")
    _COUNT[0] += 1
    return out


def det_grid(min_x=-10, max_x=70, min_y=-40, max_y=40, pixels_per_meter=4, radius=1):
    """(h, w, scalars) of the heat-map grid, each scalar computed as detections_to_heatmap's torch ops see it."""
    h, w = (max_y - min_y) * pixels_per_meter, (max_x - min_x) * pixels_per_meter
    inv_r = float(np.float32(1) / np.float32(radius))                  # torch divides by a scalar as a multiply by its reciprocal
    return int(h), int(w), (pixels_per_meter, (max_y - min_y) * pixels_per_meter / 2, h, min_x * pixels_per_meter, inv_r)


def det_heatmaps(actors, offsets, grid=None, out=None):
    """Heat, size and orientation maps of a batch in one launch (see lavb_det_heatmaps in include/lav_b200.h).  actors (A, 6)
    fp32 rows [x, y, ori, bx, by, typ]; offsets (B+1,) int32: sample i owns actors[offsets[i]:offsets[i+1]]; grid: the
    keyword arguments of det_grid.  -> (heat, size, orim), each (B, 2, h, w) fp32, bit-identical to detections_to_heatmap."""
    _need_cuda(actors, offsets)
    if actors.dtype != torch.float32 or actors.dim() != 2 or actors.shape[1] != 6 or not actors.is_contiguous():
        raise capi.LavbError(f"det_heatmaps: actors must be a contiguous (A, 6) fp32 tensor, got {actors.dtype} {tuple(actors.shape)}")
    if offsets.dtype != torch.int32 or offsets.dim() != 1 or offsets.numel() < 1 or not offsets.is_contiguous():
        raise capi.LavbError(f"det_heatmaps: offsets must be a contiguous (B+1,) int32 tensor, got {offsets.dtype} "
                             f"{tuple(offsets.shape)}")
    if actors.device != offsets.device:
        raise capi.LavbError("det_heatmaps: actors and offsets must be on one device")
    h, w, (ppm, cx0, cy0, cy1, inv_r) = det_grid(**(grid or {}))
    b = offsets.numel() - 1
    if out is None:
        out = tuple(torch.empty((b, 2, h, w), dtype=torch.float32, device=actors.device) for _ in range(3))
    elif any(t.dtype != torch.float32 or tuple(t.shape) != (b, 2, h, w) or not t.is_contiguous() or t.device != actors.device
             for t in out):
        raise capi.LavbError(f"det_heatmaps: out must be three contiguous fp32 ({b}, 2, {h}, {w}) tensors on {actors.device}")
    heat, size, orim = out
    check(lib().lavb_det_heatmaps(_ptr(actors), _ptr(offsets), b, h, w, ppm, cx0, cy0, cy1, inv_r, _ptr(heat), _ptr(size),
                                  _ptr(orim), _stream()), "lavb_det_heatmaps")
    _COUNT[0] += 1
    return heat, size, orim


def _eval_layout(b, ncols):
    """(name, dtype, shape, byte offset) of the parts of eval_batch's result buffer, 8-byte parts first, and its size."""
    parts = [("iou", torch.int64, (b, 3, 2)), ("plan_err", torch.float64, (b, 2)), ("ngt", torch.int32, (b, 2)),
             ("score", torch.float32, (b, ncols)), ("flags", torch.int32, (b, ncols))]
    out, pos = [], 0
    for name, dt, shape in parts:
        out.append((name, dt, shape, pos))
        pos += int(np.prod(shape)) * torch.empty((), dtype=dt).element_size()
    return out, pos


def eval_views(buf, b, ncols):
    """the named parts of an eval_batch result buffer (on the device or a host copy of it): iou (b,3,2) int64 = per BEV channel
    (intersection, union); plan_err (b,2) fp64 = (ADE, FDE); ngt (b,2) int32 = actors per class in the window; score / flags
    (b, ncols) = the packed scores and, per column, bit 4 for a surviving peak and bit k for a match at EVAL_THRESHOLDS_M[k]."""
    layout, _ = _eval_layout(b, ncols)
    return {name: buf[pos:pos + int(np.prod(shape)) * torch.empty((), dtype=dt).element_size()].view(dt).view(shape)
            for name, dt, shape, pos in layout}


EVAL_THRESHOLDS_M = (0.5, 1.0, 2.0, 4.0)      # centre-distance thresholds of the detection matching (evaluate.cu)


def eval_batch(seg, gt, packed, actors, offsets, plan, ego_locs, grid=None, min_score=0.2, out=None):
    """The scores of one evaluation batch in one launch (see lavb_eval_batch in include/lav_b200.h).  seg (B,H,W,3) NHWC sigmoid
    probabilities, fp32 or h16; gt (B,P>=3,H,W) uint8; packed (B,7,2*n_det) fp32 from det_peaks; actors (A,6) fp32 (the
    det_heatmaps table, on the device); offsets (B+1,) int32 on the HOST; plan (B,T,2) and ego_locs (B,T+1,2) fp32; grid: the
    keyword arguments of det_grid.  -> the uint8 result buffer (written into ``out`` when given), to be read through eval_views,
    usually after one copy to the host."""
    _need_cuda(seg, gt, packed, actors, plan, ego_locs)
    if seg.dim() != 4 or seg.shape[3] != 3 or seg.dtype not in (torch.float32, h16()) or not seg.is_contiguous():
        raise capi.LavbError(f"eval_batch: seg must be a contiguous (B,H,W,3) fp32 or {h16()} tensor, got {seg.dtype} {tuple(seg.shape)}")
    b, h, w, _ = seg.shape
    if gt.dtype != torch.uint8 or gt.dim() != 4 or gt.shape[0] != b or tuple(gt.shape[2:]) != (h, w) or not gt.is_contiguous():
        raise capi.LavbError(f"eval_batch: gt must be a contiguous ({b}, P, {h}, {w}) uint8 tensor, got {gt.dtype} {tuple(gt.shape)}")
    if packed.dtype != torch.float32 or packed.dim() != 3 or packed.shape[:2] != (b, 7) or packed.shape[2] % 2 \
            or not packed.is_contiguous():
        raise capi.LavbError(f"eval_batch: packed must be a contiguous ({b}, 7, 2*n_det) fp32 tensor, got {tuple(packed.shape)}")
    if actors.dtype != torch.float32 or actors.dim() != 2 or actors.shape[1] != 6 or not actors.is_contiguous():
        raise capi.LavbError(f"eval_batch: actors must be a contiguous (A, 6) fp32 tensor, got {actors.dtype} {tuple(actors.shape)}")
    offsets = np.ascontiguousarray(offsets.numpy() if torch.is_tensor(offsets) else offsets)
    if offsets.dtype != np.int32 or offsets.shape != (b + 1,):
        raise capi.LavbError(f"eval_batch: offsets must be a host ({b + 1},) int32 array, got {offsets.dtype} {offsets.shape}")
    t = plan.shape[1] if plan.dim() == 3 else -1
    if plan.dtype != torch.float32 or tuple(plan.shape) != (b, t, 2) or not plan.is_contiguous() or ego_locs.dtype != torch.float32 \
            or tuple(ego_locs.shape) != (b, t + 1, 2) or not ego_locs.is_contiguous():
        raise capi.LavbError(f"eval_batch: plan ({b}, T, 2) and ego_locs ({b}, T+1, 2) must be contiguous fp32, got "
                             f"{plan.dtype} {tuple(plan.shape)} / {ego_locs.dtype} {tuple(ego_locs.shape)}")
    if len({seg.device, gt.device, packed.device, actors.device, plan.device, ego_locs.device}) != 1:
        raise capi.LavbError("eval_batch: the inputs must be on one device")
    ncols = packed.shape[2]
    _, nbytes = _eval_layout(b, ncols)
    if out is None:
        out = torch.empty((nbytes,), dtype=torch.uint8, device=seg.device)
    elif out.dtype != torch.uint8 or tuple(out.shape) != (nbytes,) or out.device != seg.device:
        raise capi.LavbError(f"eval_batch: out must be a ({nbytes},) uint8 tensor on {seg.device}")
    v = eval_views(out, b, ncols)
    _, _, (ppm, cx0, cy0, cy1, _) = det_grid(**(grid or {}))
    check(lib().lavb_eval_batch(_ptr(seg), _DT[seg.dtype], _ptr(gt), gt.shape[1], b, h, w, _ptr(packed), ncols // 2, _ptr(actors),
                                actors.shape[0], offsets.ctypes.data_as(C.c_void_p), ppm, cx0, cy0, cy1, float(min_score), _ptr(plan),
                                _ptr(ego_locs), t, _ptr(v["iou"]), _ptr(v["ngt"]), _ptr(v["score"]), _ptr(v["flags"]),
                                _ptr(v["plan_err"]), _stream()), "lavb_eval_batch")
    _COUNT[0] += -(-b // 256)
    return out


def forecast_views(buf, k):
    """the named parts of a forecast_eval result buffer (on the device or a host copy of it): err (k,6) fp64 = (min ADE, min FDE,
    top-branch ADE, top-branch FDE, ADE and FDE under the recorded command or NaN); branch (k,2) int32 = (argmin-ADE branch, top
    branch)."""
    return dict(err=buf[:k * 48].view(torch.float64).view(k, 6), branch=buf[k * 48:k * 56].view(torch.int32).view(k, 2))


def forecast_eval(cast, score, target, cmd, out=None):
    """The forecast scores of k rows in one launch (see lavb_forecast_eval in include/lav_b200.h).  cast (k,C,T,2), score (k,C)
    and target (k,T,2) fp32; cmd (k,) int32, -1 where the row has no recorded command.  -> the uint8 result buffer (written into
    ``out`` when given), to be read through forecast_views, usually after one copy to the host."""
    _need_cuda(cast, score, target, cmd)
    if cast.dtype != torch.float32 or cast.dim() != 4 or cast.shape[3] != 2 or not cast.is_contiguous():
        raise capi.LavbError(f"forecast_eval: cast must be a contiguous (k, C, T, 2) fp32 tensor, got {cast.dtype} {tuple(cast.shape)}")
    k, c, t, _ = cast.shape
    if score.dtype != torch.float32 or tuple(score.shape) != (k, c) or not score.is_contiguous():
        raise capi.LavbError(f"forecast_eval: score must be a contiguous ({k}, {c}) fp32 tensor, got {score.dtype} {tuple(score.shape)}")
    if target.dtype != torch.float32 or tuple(target.shape) != (k, t, 2) or not target.is_contiguous():
        raise capi.LavbError(f"forecast_eval: target must be a contiguous ({k}, {t}, 2) fp32 tensor, got {target.dtype} "
                             f"{tuple(target.shape)}")
    if cmd.dtype != torch.int32 or tuple(cmd.shape) != (k,) or not cmd.is_contiguous():
        raise capi.LavbError(f"forecast_eval: cmd must be a contiguous ({k},) int32 tensor, got {cmd.dtype} {tuple(cmd.shape)}")
    if len({cast.device, score.device, target.device, cmd.device}) != 1:
        raise capi.LavbError("forecast_eval: the inputs must be on one device")
    if out is None:
        out = torch.empty((k * 56,), dtype=torch.uint8, device=cast.device)
    elif out.dtype != torch.uint8 or tuple(out.shape) != (k * 56,) or out.device != cast.device:
        raise capi.LavbError(f"forecast_eval: out must be a ({k * 56},) uint8 tensor on {cast.device}")
    v = forecast_views(out, k)
    check(lib().lavb_forecast_eval(_ptr(cast), _ptr(score), _ptr(target), _ptr(cmd), k, c, t, _ptr(v["err"]), _ptr(v["branch"]),
                                   _stream()), "lavb_forecast_eval")
    _COUNT[0] += k > 0
    return out


DET_MATCH_M = 2.0       # centre-distance radius of the detected-forecast match (det_forecast.cu)


def _det_match_layout(b, k, t):
    """(name, dtype, shape, byte offset) of the parts of det_forecast_match's result buffer and its size: forecast_eval's result
    of the k rows first (err, branch: its ``out`` is buf[:56 * k]), then the match's."""
    parts = [("err", torch.float64, (k, 6)), ("branch", torch.int32, (k, 2)), ("dist", torch.float64, (k,)),
             ("target", torch.float32, (k, t, 2)), ("actor", torch.int32, (k,)), ("flag", torch.int32, (k,)),
             ("ngt", torch.int32, (b, 2))]
    out, pos = [], 0
    for name, dt, shape in parts:
        out.append((name, dt, shape, pos))
        pos += int(np.prod(shape)) * torch.empty((), dtype=dt).element_size()
    return out, pos


def det_match_views(buf, b, k, t):
    """the named parts of a det_forecast_match result buffer of b samples, k rows and t steps (on the device or a host copy):
    err (k,6) fp64 / branch (k,2) int32 = forecast_views of the rows, once forecast_eval has written buf[:56 * k]; dist (k,) fp64 =
    match distance in metres, NaN when unmatched; target (k,t,2) fp32 = the matched track's future in the ego frame, NaN unless
    matched to a tracked actor; actor (k,) int32 = the actor row within its sample, or -1; flag (k,) int32 = bit 0 matched, bit 1
    matched to a tracked actor; ngt (b,2) int32 = vehicles in the window with and without a track."""
    layout, _ = _det_match_layout(b, k, t)
    return {name: buf[pos:pos + int(np.prod(shape)) * torch.empty((), dtype=dt).element_size()].view(dt).view(shape)
            for name, dt, shape, pos in layout}


def det_forecast_match(packed, actors, offsets, row_offsets, cols, num_objs, locs, ego_locs, grid=None, match_m=DET_MATCH_M,
                       out=None):
    """The match of one batch's forecast rows to the recorded actors in one launch (see lavb_det_forecast_match in
    include/lav_b200.h).  packed (B,7,2*n_det) fp32 from det_peaks; actors (A,6) fp32 on the device and offsets (B+1,) int32 on the
    HOST (eval_batch's actor table); row_offsets (B+1,) and cols (K,) int32 on the HOST = each sample's rows and their packed
    columns; num_objs (B,) on the HOST = the recorded tracks; locs (B,max_objs,T+1,2) and ego_locs (B,T+1,2) fp32 = the labels;
    grid: the keyword arguments of det_grid.  -> the uint8 result buffer (written into ``out`` when given), read through
    det_match_views; forecast_eval(..., out=buf[:56 * K]) puts the rows' scores in the same buffer."""
    _need_cuda(packed, actors, locs, ego_locs)
    if packed.dtype != torch.float32 or packed.dim() != 3 or packed.shape[1] != 7 or packed.shape[2] % 2 or not packed.is_contiguous():
        raise capi.LavbError(f"det_forecast_match: packed must be a contiguous (B, 7, 2*n_det) fp32 tensor, got {packed.dtype} "
                             f"{tuple(packed.shape)}")
    b = packed.shape[0]
    if actors.dtype != torch.float32 or actors.dim() != 2 or actors.shape[1] != 6 or not actors.is_contiguous():
        raise capi.LavbError(f"det_forecast_match: actors must be a contiguous (A, 6) fp32 tensor, got {actors.dtype} "
                             f"{tuple(actors.shape)}")
    host = lambda a: np.ascontiguousarray(a.numpy() if torch.is_tensor(a) else a)
    offsets, row_offsets, cols, num_objs = host(offsets), host(row_offsets), host(cols), host(num_objs).astype(np.int32)
    for name, a, shape in (("offsets", offsets, (b + 1,)), ("row_offsets", row_offsets, (b + 1,)), ("num_objs", num_objs, (b,))):
        if a.dtype != np.int32 or a.shape != shape:
            raise capi.LavbError(f"det_forecast_match: {name} must be a host {shape} int32 array, got {a.dtype} {a.shape}")
    k = int(row_offsets[-1])
    if cols.dtype != np.int32 or cols.shape != (k,):
        raise capi.LavbError(f"det_forecast_match: cols must be a host ({k},) int32 array, got {cols.dtype} {cols.shape}")
    if locs.dtype != torch.float32 or locs.dim() != 4 or locs.shape[0] != b or locs.shape[3] != 2 or not locs.is_contiguous():
        raise capi.LavbError(f"det_forecast_match: locs must be a contiguous ({b}, max_objs, T+1, 2) fp32 tensor, got {locs.dtype} "
                             f"{tuple(locs.shape)}")
    t = locs.shape[2] - 1
    if ego_locs.dtype != torch.float32 or tuple(ego_locs.shape) != (b, t + 1, 2) or not ego_locs.is_contiguous():
        raise capi.LavbError(f"det_forecast_match: ego_locs must be a contiguous ({b}, {t + 1}, 2) fp32 tensor, got {ego_locs.dtype} "
                             f"{tuple(ego_locs.shape)}")
    if len({packed.device, actors.device, locs.device, ego_locs.device}) != 1:
        raise capi.LavbError("det_forecast_match: the inputs must be on one device")
    _, nbytes = _det_match_layout(b, k, t)
    if out is None:
        out = torch.empty((nbytes,), dtype=torch.uint8, device=packed.device)
    elif out.dtype != torch.uint8 or tuple(out.shape) != (nbytes,) or out.device != packed.device:
        raise capi.LavbError(f"det_forecast_match: out must be a ({nbytes},) uint8 tensor on {packed.device}")
    v = det_match_views(out, b, k, t)
    h, w, (ppm, cx0, cy0, cy1, _) = det_grid(**(grid or {}))
    ip = lambda a: a.ctypes.data_as(C.c_void_p)
    check(lib().lavb_det_forecast_match(_ptr(packed), b, w, packed.shape[2] // 2, _ptr(actors), actors.shape[0], ip(offsets),
                                        ip(row_offsets), ip(cols), ip(num_objs), _ptr(locs), _ptr(ego_locs), locs.shape[1], t, ppm,
                                        cx0, cy0, cy1, float(match_m), _ptr(v["actor"]), _ptr(v["flag"]), _ptr(v["dist"]),
                                        _ptr(v["target"]), _ptr(v["ngt"]), _stream()), "lavb_det_forecast_match")
    _COUNT[0] += -(-b // 128)
    return out


# one (actor, step) record of plan_safety's actor table (lavb_plan_safety in include/lav_b200.h)
PLAN_SAFETY_ACTOR_DTYPE = np.dtype([("x", np.float64), ("y", np.float64), ("cos", np.float64), ("sin", np.float64),
                                    ("e1", np.float64), ("e2", np.float64), ("typ", np.int32), ("present", np.int32)])
assert PLAN_SAFETY_ACTOR_DTYPE.itemsize == 56
PLAN_SAFETY_FIELDS = ("veh_step", "veh_row", "ped_step", "ped_row", "off_road_step", "off_map_steps", "invalid_steps", "first_step")


def plan_safety_views(res):
    """the named columns of a plan_safety result (B, n, 8) int32 (on the device or a host copy), each (B, n): veh_step / veh_row
    = the first step (1..T) whose ego box overlaps a vehicle and that vehicle's actor row, ped_step / ped_row the same for
    pedestrians, off_road_step = the first step with a corner on a 0 pixel of the road plane, off_map_steps / invalid_steps =
    step counts, first_step = the first collision of either class; -1 for none."""
    return {name: res[..., i] for i, name in enumerate(PLAN_SAFETY_FIELDS)}


def plan_safety(traj, actors, offsets, ego_ext, bev, grid=None, out=None):
    """Collisions and road departures of n ego trajectories per sample in one launch (see lavb_plan_safety in include/lav_b200.h).
    traj (B,n,T,2) fp32 in the label frame; actors = PLAN_SAFETY_ACTOR_DTYPE records of every actor row and step as a 1-D uint8
    tensor on the device, sample i owning rows [offsets[i], offsets[i+1]) (offsets (B+1,) int32 on the HOST), row a's step s at
    record a * T + s - 1; ego_ext (B,2) fp64 = the ego's half extents; bev (B,P,H,W) uint8, plane 0 the road; grid: the keyword
    arguments of det_grid.  -> (B,n,8) int32, read through plan_safety_views (written into ``out`` when given)."""
    _need_cuda(traj, actors, ego_ext, bev)
    if traj.dtype != torch.float32 or traj.dim() != 4 or traj.shape[3] != 2 or not traj.is_contiguous():
        raise capi.LavbError(f"plan_safety: traj must be a contiguous (B, n, T, 2) fp32 tensor, got {traj.dtype} {tuple(traj.shape)}")
    b, n, t, _ = traj.shape
    offsets = np.ascontiguousarray(offsets.numpy() if torch.is_tensor(offsets) else offsets)
    if offsets.dtype != np.int32 or offsets.shape != (b + 1,):
        raise capi.LavbError(f"plan_safety: offsets must be a host ({b + 1},) int32 array, got {offsets.dtype} {offsets.shape}")
    rec = PLAN_SAFETY_ACTOR_DTYPE.itemsize
    if actors.dtype != torch.uint8 or actors.dim() != 1 or actors.numel() % (rec * t) or not actors.is_contiguous():
        raise capi.LavbError(f"plan_safety: actors must be a contiguous 1-D uint8 tensor of {rec}-byte records, {t} per actor row, "
                             f"got {actors.dtype} {tuple(actors.shape)}")
    if ego_ext.dtype != torch.float64 or tuple(ego_ext.shape) != (b, 2) or not ego_ext.is_contiguous():
        raise capi.LavbError(f"plan_safety: ego_ext must be a contiguous ({b}, 2) fp64 tensor, got {ego_ext.dtype} {tuple(ego_ext.shape)}")
    if bev.dtype != torch.uint8 or bev.dim() != 4 or bev.shape[0] != b or not bev.is_contiguous():
        raise capi.LavbError(f"plan_safety: bev must be a contiguous ({b}, P, H, W) uint8 tensor, got {bev.dtype} {tuple(bev.shape)}")
    if len({traj.device, actors.device, ego_ext.device, bev.device}) != 1:
        raise capi.LavbError("plan_safety: the inputs must be on one device")
    if out is None:
        out = torch.empty((b, n, 8), dtype=torch.int32, device=traj.device)
    elif out.dtype != torch.int32 or tuple(out.shape) != (b, n, 8) or not out.is_contiguous() or out.device != traj.device:
        raise capi.LavbError(f"plan_safety: out must be a contiguous ({b}, {n}, 8) int32 tensor on {traj.device}")
    _, _, h, w = bev.shape
    _, _, (ppm, cx0, cy0, cy1, _) = det_grid(**(grid or {}))
    check(lib().lavb_plan_safety(_ptr(traj), b, n, t, _ptr(actors), actors.numel() // (rec * t), offsets.ctypes.data_as(C.c_void_p),
                                 _ptr(ego_ext), _ptr(bev), bev[0].numel() if b else h * w, h, w, ppm, cx0, cy0, cy1, _ptr(out),
                                 _stream()), "lavb_plan_safety")
    _COUNT[0] += -(-b // 512)
    return out


def agent_control_state_bytes(turn_n, speed_n):
    """bytes of one agent's controller state (lavb_agent_control_state_bytes); all-zero bytes are a new route."""
    n = int(lib().lavb_agent_control_state_bytes(int(turn_n), int(speed_n)))
    if n == 0:
        raise capi.LavbError(f"agent_control: PID windows {turn_n}, {speed_n} outside 1..64")
    return n


def agent_control_state_views(state, turn_n, speed_n):
    """the named fields of a HOST copy of agent_control's state (a uint8 array of B records): stop (B,) and creep (B,) int32,
    turn (B, turn_n) and speed (B, speed_n) fp64 = the PID windows, oldest value first."""
    rec = np.dtype([("stop", np.int32), ("creep", np.int32), ("turn_head", np.int32), ("speed_head", np.int32),
                    ("turn", np.float64, (turn_n,)), ("speed", np.float64, (speed_n,))])
    s = np.ascontiguousarray(state).view(rec)
    roll = lambda w, h: np.take_along_axis(w, (h[:, None] + np.arange(w.shape[1])[None]) % w.shape[1], axis=1)
    return dict(stop=s["stop"].copy(), creep=s["creep"].copy(), turn=roll(s["turn"], s["turn_head"]),
                speed=roll(s["speed"], s["speed_head"]))


def agent_control(plan, cast, other_locs, other_cmds, offsets, pred_bra, speed, cmds, config, state, control=None, flags=None):
    """The agent's controls for B agents in one launch (see lavb_agent_control in include/lav_b200.h): plan / cast (B,T,2) fp32 =
    ego plan and ego cast under the command; other_locs (K,C,T,2) / other_cmds (K,C) fp32 = the forecast rows of all agents,
    agent i owning rows [offsets[i], offsets[i+1]) (offsets (B+1,) int32 on the HOST); pred_bra, speed (B,) fp32; cmds (B,)
    int32 on the HOST, or a (B,) int32 CUDA tensor (lavb_agent_control_dcmd: an agent whose command is outside 0..C-1 gets NaN
    controls and LAVB_CTL_BAD_CMD); config a capi.ControlConfig; state the agents' controller state, a contiguous uint8 device tensor of
    B * agent_control_state_bytes(config.turn_n, config.speed_n) bytes, updated in place.
    -> (control (B,3) fp32 = steer, throttle, brake; flags (B,) int32 of LAVB_CTL_* bits), written into ``control`` / ``flags``
    when given."""
    _need_cuda(plan, cast, other_locs, other_cmds, pred_bra, speed, state)
    f32 = lambda x, shape: x.dtype == torch.float32 and tuple(x.shape) == shape and x.is_contiguous()
    if plan.dtype != torch.float32 or plan.dim() != 3 or plan.shape[2] != 2 or not plan.is_contiguous():
        raise capi.LavbError(f"agent_control: plan must be a contiguous (B, T, 2) fp32 tensor, got {plan.dtype} {tuple(plan.shape)}")
    b, t, _ = plan.shape
    if not f32(cast, (b, t, 2)):
        raise capi.LavbError(f"agent_control: cast must be a contiguous ({b}, {t}, 2) fp32 tensor, got {cast.dtype} {tuple(cast.shape)}")
    if other_locs.dim() != 4 or not f32(other_locs, (other_locs.shape[0], other_locs.shape[1], t, 2)):
        raise capi.LavbError(f"agent_control: other_locs must be a contiguous (K, C, {t}, 2) fp32 tensor, got {other_locs.dtype} "
                             f"{tuple(other_locs.shape)}")
    k, c = other_locs.shape[:2]
    if not f32(other_cmds, (k, c)):
        raise capi.LavbError(f"agent_control: other_cmds must be a contiguous ({k}, {c}) fp32 tensor, got {other_cmds.dtype} "
                             f"{tuple(other_cmds.shape)}")
    if not f32(pred_bra, (b,)) or not f32(speed, (b,)):
        raise capi.LavbError(f"agent_control: pred_bra and speed must be contiguous ({b},) fp32 tensors, got "
                             f"{tuple(pred_bra.shape)} and {tuple(speed.shape)}")
    offsets = np.ascontiguousarray(offsets.numpy() if torch.is_tensor(offsets) else offsets)
    if offsets.dtype != np.int32 or offsets.shape != (b + 1,):
        raise capi.LavbError(f"agent_control: offsets must be a host ({b + 1},) int32 array, got {offsets.dtype} {offsets.shape}")
    dcmd = torch.is_tensor(cmds) and cmds.is_cuda
    if dcmd:
        if cmds.dtype != torch.int32 or tuple(cmds.shape) != (b,) or not cmds.is_contiguous() or cmds.device != plan.device:
            raise capi.LavbError(f"agent_control: device cmds must be a contiguous ({b},) int32 tensor on {plan.device}, got "
                                 f"{cmds.dtype} {tuple(cmds.shape)} on {cmds.device}")
    else:
        cmds = np.ascontiguousarray(cmds.numpy() if torch.is_tensor(cmds) else cmds)
        if cmds.dtype != np.int32 or cmds.shape != (b,):
            raise capi.LavbError(f"agent_control: cmds must be a host ({b},) int32 array, got {cmds.dtype} {cmds.shape}")
    if not isinstance(config, capi.ControlConfig):
        raise capi.LavbError("agent_control: config must be a capi.ControlConfig")
    nbytes = b * agent_control_state_bytes(config.turn_n, config.speed_n)
    if state.dtype != torch.uint8 or tuple(state.shape) != (nbytes,) or not state.is_contiguous():
        raise capi.LavbError(f"agent_control: state must be a contiguous ({nbytes},) uint8 tensor, got {state.dtype} {tuple(state.shape)}")
    dev = plan.device
    if len({dev, cast.device, other_locs.device, other_cmds.device, pred_bra.device, speed.device, state.device}) != 1:
        raise capi.LavbError("agent_control: the inputs must be on one device")
    if control is None:
        control = torch.empty((b, 3), dtype=torch.float32, device=dev)
    elif not f32(control, (b, 3)) or control.device != dev:
        raise capi.LavbError(f"agent_control: control must be a contiguous ({b}, 3) fp32 tensor on {dev}")
    if flags is None:
        flags = torch.empty((b,), dtype=torch.int32, device=dev)
    elif flags.dtype != torch.int32 or tuple(flags.shape) != (b,) or not flags.is_contiguous() or flags.device != dev:
        raise capi.LavbError(f"agent_control: flags must be a contiguous ({b},) int32 tensor on {dev}")
    ip = lambda a: a.ctypes.data_as(C.c_void_p)
    if dcmd:
        check(lib().lavb_agent_control_dcmd(_ptr(plan), _ptr(cast), b, t, c, _ptr(other_locs), _ptr(other_cmds), k, ip(offsets),
                                            _ptr(pred_bra), _ptr(speed), _ptr(cmds), C.byref(config), _ptr(state), _ptr(control),
                                            _ptr(flags), _stream()), "lavb_agent_control_dcmd")
    else:
        check(lib().lavb_agent_control(_ptr(plan), _ptr(cast), b, t, c, _ptr(other_locs), _ptr(other_cmds), k, ip(offsets),
                                       _ptr(pred_bra), _ptr(speed), ip(cmds), C.byref(config), _ptr(state), _ptr(control),
                                       _ptr(flags), _stream()), "lavb_agent_control")
    _COUNT[0] += -(-b // 512)
    return control, flags


NAV_STATE_DTYPE = np.dtype([("ekf_x", np.float64, (3,)), ("ekf_p", np.float64, (3,)), ("wp_x", np.float64), ("wp_y", np.float64),
                            ("rp_x", np.float64), ("rp_y", np.float64), ("route_scale", np.float64), ("ekf_scale", np.float64),
                            ("frames", np.int32), ("wp_idx", np.int32), ("wp_cmd", np.int32), ("rp_idx", np.int32),
                            ("lane_counter", np.int32), ("lane_changed", np.int32), ("pad", np.int32, (2,))])
assert NAV_STATE_DTYPE.itemsize == 128         # lavb_nav_state of include/lav_b200.h


def agent_nav_state_bytes():
    """bytes of one agent's lavb_nav_state record (lavb_agent_nav_state_bytes)."""
    n = int(lib().lavb_agent_nav_state_bytes())
    if n != NAV_STATE_DTYPE.itemsize:
        raise capi.LavbError(f"agent_nav: the library's state record has {n} bytes, NAV_STATE_DTYPE {NAV_STATE_DTYPE.itemsize}")
    return n


def _f64_rows(x, b, cols, what):
    shape = (b, cols) if cols else (b,)
    if x.dtype != torch.float64 or tuple(x.shape) != shape or not x.is_contiguous():
        raise capi.LavbError(f"{what} must be a contiguous {shape} fp64 tensor, got {x.dtype} {tuple(x.shape)}")


def agent_nav_front(nodes, node_cmd, route, gnss, compass, state, cmds=None, nxps=None, poses=None, flags=None):
    """The front of B agents' tick in one launch (lavb_agent_nav_front in include/lav_b200.h): nodes (M, 2) fp64 and node_cmd (M,)
    int32 = every route's nodes; route (B, 2) int32 = (start, count) per agent; gnss (B, 2) fp64 = lat, lon; compass (B,) fp64,
    raw; state B lavb_nav_state records (uint8, updated in place).  -> (cmds (B,) int32, nxps (B, 2) fp32, poses (B, 3) fp64,
    flags (B,) int32 of LAVB_NAV_* bits), written into the given tensors when given."""
    _need_cuda(nodes, node_cmd, route, gnss, compass, state)
    if route.dtype != torch.int32 or route.dim() != 2 or route.shape[1] != 2 or not route.is_contiguous():
        raise capi.LavbError(f"agent_nav_front: route must be a contiguous (B, 2) int32 tensor, got {route.dtype} {tuple(route.shape)}")
    b = route.shape[0]
    if nodes.dtype != torch.float64 or nodes.dim() != 2 or nodes.shape[1] != 2 or not nodes.is_contiguous():
        raise capi.LavbError(f"agent_nav_front: nodes must be a contiguous (M, 2) fp64 tensor, got {nodes.dtype} {tuple(nodes.shape)}")
    m = nodes.shape[0]
    if node_cmd.dtype != torch.int32 or tuple(node_cmd.shape) != (m,) or not node_cmd.is_contiguous():
        raise capi.LavbError(f"agent_nav_front: node_cmd must be a contiguous ({m},) int32 tensor, got {node_cmd.dtype} "
                             f"{tuple(node_cmd.shape)}")
    _f64_rows(gnss, b, 2, "agent_nav_front: gnss")
    _f64_rows(compass, b, 0, "agent_nav_front: compass")
    nbytes = b * agent_nav_state_bytes()
    if state.dtype != torch.uint8 or tuple(state.shape) != (nbytes,) or not state.is_contiguous():
        raise capi.LavbError(f"agent_nav_front: state must be a contiguous ({nbytes},) uint8 tensor, got {state.dtype} "
                             f"{tuple(state.shape)}")
    dev = route.device
    if len({dev, nodes.device, node_cmd.device, gnss.device, compass.device, state.device}) != 1:
        raise capi.LavbError("agent_nav_front: the inputs must be on one device")

    def out(x, shape, dt, name):
        if x is None:
            return torch.empty(shape, dtype=dt, device=dev)
        if x.dtype != dt or tuple(x.shape) != shape or not x.is_contiguous() or x.device != dev:
            raise capi.LavbError(f"agent_nav_front: {name} must be a contiguous {shape} {dt} tensor on {dev}")
        return x
    cmds, nxps = out(cmds, (b,), torch.int32, "cmds"), out(nxps, (b, 2), torch.float32, "nxps")
    poses, flags = out(poses, (b, 3), torch.float64, "poses"), out(flags, (b,), torch.int32, "flags")
    check(lib().lavb_agent_nav_front(b, _ptr(nodes), _ptr(node_cmd), m, _ptr(route), _ptr(gnss), _ptr(compass), _ptr(state),
                                     _ptr(cmds), _ptr(nxps), _ptr(poses), _ptr(flags), _stream()), "lavb_agent_nav_front")
    _COUNT[0] += 1 if b else 0
    return cmds, nxps, poses, flags


def agent_nav_update(control, speed, gnss, compass, state):
    """EKF.step of B agents after the controls (lavb_agent_nav_update): control (B, 3) fp32 = agent_control's output (steer in
    column 0); speed (B,) fp64 m/s; gnss (B, 2) fp64; compass (B,) fp64, raw; state as in agent_nav_front, updated in place."""
    _need_cuda(control, speed, gnss, compass, state)
    b = state.numel() // agent_nav_state_bytes()
    if control.dtype != torch.float32 or tuple(control.shape) != (b, 3) or not control.is_contiguous():
        raise capi.LavbError(f"agent_nav_update: control must be a contiguous ({b}, 3) fp32 tensor, got {control.dtype} "
                             f"{tuple(control.shape)}")
    _f64_rows(speed, b, 0, "agent_nav_update: speed")
    _f64_rows(gnss, b, 2, "agent_nav_update: gnss")
    _f64_rows(compass, b, 0, "agent_nav_update: compass")
    if state.dtype != torch.uint8 or state.numel() != b * agent_nav_state_bytes() or not state.is_contiguous():
        raise capi.LavbError("agent_nav_update: state must be a contiguous uint8 tensor of whole lavb_nav_state records")
    if len({control.device, speed.device, gnss.device, compass.device, state.device}) != 1:
        raise capi.LavbError("agent_nav_update: the inputs must be on one device")
    check(lib().lavb_agent_nav_update(b, _ptr(control), _ptr(speed), _ptr(gnss), _ptr(compass), _ptr(state), _stream()),
          "lavb_agent_nav_update")
    _COUNT[0] += 1 if b else 0


def stack_job_poses(d_jobs, b, t, gap, keep, tick, ring_pose, poses=None):
    """the R / dx / dy fields of stack_jobs' table from the device pose ring (lavb_stack_job_poses): d_jobs the uint8 table of
    b * t STACK_JOB_DTYPE records; ring_pose (b, keep, 3) fp64, ``poses`` (b, 3) fp64 written to slot tick % keep first."""
    _need_cuda(d_jobs, ring_pose, poses)
    if d_jobs.dtype != torch.uint8 or d_jobs.numel() != b * t * STACK_JOB_DTYPE.itemsize or not d_jobs.is_contiguous():
        raise capi.LavbError(f"stack_job_poses: jobs must hold {b} x {t} contiguous records")
    if ring_pose.dtype != torch.float64 or tuple(ring_pose.shape) != (b, keep, 3) or not ring_pose.is_contiguous():
        raise capi.LavbError(f"stack_job_poses: ring_pose must be a contiguous ({b}, {keep}, 3) fp64 tensor")
    if poses is not None:
        _f64_rows(poses, b, 3, "stack_job_poses: poses")
    check(lib().lavb_stack_job_poses(_ptr(d_jobs), b, t, gap, keep, int(tick), _ptr(ring_pose), _ptr(poses), _stream()),
          "lavb_stack_job_poses")
    _COUNT[0] += 1 if b else 0


PILLAR_ENCODER ="sorted"    # name of the 16-bit pipeline's pillar encoder, reported by bench.py; it selects nothing


def pillar_forward_sorted(pts, starts, counts, grid, w1, s1, t1, w2, s2, t2, canvas16=False):
    """tensor-core pillar encoder of the 16-bit pipeline: counting sort by canvas cell + persistent mma.sync encoder
    (lavb_pillar_forward_sorted).  Returns the NHWC canvas: fp32 (B,ny,nx,H2); with canvas16, h16 (B,ny,nx,H2), saturating —
    what the 16-bit pipeline feeds the backbone."""
    _need_cuda(pts, w1, w2)
    assert pts.dtype == torch.float32 and pts.dim() == 2 and pts.stride(1) == 1
    _check_point_mlp("pillar_forward_sorted", pts, w1, s1, t1, w2, s2, t2)
    min_x, max_x, min_y, max_y, ppm, nx, ny = grid
    d = w1.shape[1] - 5
    b, st, ct = _clouds(starts, counts, pts, "pillar_forward_sorted")
    total = int(sum(int(c) for c in counts))
    h2 = w2.shape[0]
    canvas = torch.empty((b, ny, nx, h2), dtype=h16() if canvas16 else torch.float32, device=pts.device)
    ws = _workspace(pts.device, lib().lavb_pillar_sorted_workspace_bytes(b, nx, ny, total))
    e0 = _prof_begin()
    check(lib().lavb_pillar_forward_sorted(_ptr(pts), pts.stride(0), d, st, ct, b, min_x, max_x, min_y, max_y, ppm, nx, ny,
                                           _ptr(w1), _ptr(s1), _ptr(t1), w1.shape[0], _ptr(w2), _ptr(s2), _ptr(t2), h2,
                                           _ptr(canvas), 2 if canvas16 else 0, _ptr(ws), _stream()), "lavb_pillar_forward_sorted")
    _prof_end("pillar", float(total) * d * 4 + float(b) * ny * nx * h2 * (2 if canvas16 else 4), e0)
    _COUNT[0] += 6
    return canvas


def det_peaks(center, box, ori, min_score=0.2, max_det=15):
    """center (LOGITS) fp32 NHWC (B,H,W,ncls), box, ori: fp32 NHWC (B,H,W,2), all contiguous -> packed (B,7,ncls*max_det)
    (see lavb_det_peaks)."""
    _need_cuda(center, box, ori)
    assert center.dim() == 4 and all(t.is_contiguous() and t.dtype == torch.float32 for t in (center, box, ori))
    b, h, w, ncls = center.shape
    assert tuple(box.shape) == tuple(ori.shape) == (b, h, w, 2), "det_peaks: box and ori must be (B, H, W, 2)"
    packed = torch.empty((b, 7, ncls * max_det), dtype=torch.float32, device=center.device)
    ws = _workspace(center.device, lib().lavb_det_peaks_workspace_bytes(b, ncls))
    check(lib().lavb_det_peaks(_ptr(center), _ptr(box), _ptr(ori), b, h, w, ncls, min_score, max_det, _ptr(packed), _ptr(ws), _stream()),
          "lavb_det_peaks")
    _COUNT[0] += 2
    return packed


def stem7x7s2_u8(img_u8, w_h16, bias, mean, std):
    """img_u8 (B, ncam, H, cam_w, 3) uint8 contiguous; w_h16 (64,160) packed by pack_stem_weights; bias (64,)
    -> f16 NHWC (B, H/2, ncam*cam_w/2, 64)."""
    _need_cuda(img_u8, w_h16, bias)
    _require(img_u8.dtype == torch.uint8 and img_u8.is_contiguous() and img_u8.dim() == 5 and img_u8.shape[4] == 3,
             "stem7x7s2_u8: img_u8 must be a contiguous uint8 (B, ncam, H, cam_w, 3) tensor")
    _require(w_h16.dtype == h16() and tuple(w_h16.shape) == (64, 160) and w_h16.is_contiguous(),
             "stem7x7s2_u8: w_h16 must be the contiguous (64, 160) 16-bit packing of pack_stem_weights")
    _require(bias.dtype == torch.float32 and tuple(bias.shape) == (64,) and bias.is_contiguous(),
             "stem7x7s2_u8: bias must be a contiguous fp32 (64,) tensor")
    _require(len(mean) == 3 and len(std) == 3, "stem7x7s2_u8: mean and std hold 3 values")
    b, ncam, h, cw, _ = img_u8.shape
    out = torch.empty((b, (h - 1) // 2 + 1, (ncam * cw - 1) // 2 + 1, 64), dtype=h16(), device=img_u8.device)
    m = (C.c_float * 3)(*[float(v) for v in mean])
    sd = (C.c_float * 3)(*[float(v) for v in std])
    check(lib().lavb_stem7x7s2_u8(_ptr(img_u8), b, ncam, h, cw, _ptr(w_h16), _ptr(bias), m, sd, _ptr(out), _stream()),
          "lavb_stem7x7s2_u8")
    _COUNT[0] += 1
    return out


def pack_stem_weights(w):
    """(64, 3, 7, 7) conv weights -> (64, 160) f16 in the stem kernel's K order k = ky*22 + kx*3 + c (zero elsewhere)."""
    wk = torch.zeros((64, 7, 22), dtype=torch.float32, device=w.device)
    wk[:, :, :21] = w.float().permute(0, 2, 3, 1).reshape(64, 7, 21)
    out = torch.zeros((64, 160), dtype=torch.float32, device=w.device)
    out[:, :154] = wk.reshape(64, 154)
    return out.to(h16()).contiguous()


def conv7x7s2_umma(x, w_packed, bias, out=None):
    """relu(conv 7x7 / stride 2 / pad 3 + bias) to 64 channels: x contiguous f16 NHWC (n, h, w, cin), cin % 64 == 0;
    w_packed (49, 64, cin) f16 from pack_conv7x7s2_weights; bias fp32 (64,) -> f16 NHWC (n, (h-1)//2+1, (w-1)//2+1, 64),
    written into `out` when given (contiguous, that shape)."""
    _need_cuda(x, w_packed, bias)
    assert x.dtype == h16() and x.is_contiguous() and x.dim() == 4
    n, h, w, cin = x.shape
    assert cin % 64 == 0 and h >= 7 and w >= 7, x.shape
    assert w_packed.dtype == h16() and w_packed.is_contiguous() and tuple(w_packed.shape) == (49, 64, cin)
    assert bias.dtype == torch.float32 and bias.is_contiguous() and bias.numel() == 64
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    if out is None:
        out = torch.empty((n, ho, wo, 64), dtype=h16(), device=x.device)
    assert out.dtype == h16() and out.is_contiguous() and tuple(out.shape) == (n, ho, wo, 64)
    e0 = _prof_begin()
    check(lib().lavb_conv7x7s2_umma(_ptr(x), n, h, w, cin, _ptr(w_packed), _ptr(bias), _ptr(out), _stream()),
          "lavb_conv7x7s2_umma")
    _prof_end(f"stem7x7s2:{cin}->64@{h}x{w}", 2.0 * n * ho * wo * 64 * cin * 49, e0)
    _COUNT[0] += 1
    return out


def conv3x3_umma(x, w, cout, stride, bias=None, scale=None, shift=None, pre_relu=False, out=None):
    """3x3 / pad 1 / stride 1 or 2 convolution with output channels in M (lavb_conv3x3_umma): x contiguous f16 NHWC (n, h, w, cin),
    cin in (64, 128, 384); w (9, cout, cin) f16, the conv_umma packing; cout in (64, 128, 256); bias / scale / shift fp32 (cout,)
    or None -> f16 NHWC (n, (h-1)//s+1, (w-1)//s+1, cout) = [relu](conv + bias) * scale + shift, written into `out` when given."""
    _need_cuda(x, w)
    assert x.dtype == h16() and x.is_contiguous() and x.dim() == 4
    n, h, wd, cin = x.shape
    assert w.dtype == h16() and w.is_contiguous() and tuple(w.shape) == (9, cout, cin), (tuple(w.shape), cout, cin)
    for v in (bias, scale, shift):
        assert v is None or (v.dtype == torch.float32 and v.is_contiguous() and v.numel() == cout)
    ho, wo = (h - 1) // stride + 1, (wd - 1) // stride + 1
    if out is None:
        out = torch.empty((n, ho, wo, cout), dtype=h16(), device=x.device)
    assert out.dtype == h16() and out.is_contiguous() and tuple(out.shape) == (n, ho, wo, cout)
    e0 = _prof_begin()
    check(lib().lavb_conv3x3_umma(_ptr(x), n, h, wd, cin, stride, _ptr(w), cout, _ptr(bias), _ptr(scale), _ptr(shift),
                                  int(pre_relu), _ptr(out), _stream()), "lavb_conv3x3_umma")
    # the label format of conv_taps' wgmma launches, so that bench.py's conv roofline keeps covering the same layers
    _prof_end(f"umma:{cin}->{cout}x9taps@{ho}x{wo}", 2.0 * n * ho * wo * cout * cin * 9, e0)
    _COUNT[0] += 1
    return out


def pack_conv7x7s2_weights(w):
    """(64, cin, 7, 7) conv weights -> (49, 64, cin) f16 [tap = ky*7 + kx][cout][cin], the layout conv7x7s2_umma reads."""
    assert w.dim() == 4 and tuple(w.shape[2:]) == (7, 7) and w.shape[0] == 64
    return w.permute(2, 3, 0, 1).reshape(49, 64, w.shape[1]).to(h16()).contiguous()


def maxpool3x3s2_nhwc(x):
    """MaxPool2d(3, 2, 1) on a contiguous f16 NHWC tensor."""
    _need_cuda(x)
    _require(x.dtype == h16() and x.is_contiguous() and x.dim() == 4 and x.shape[3] % 8 == 0,
             "maxpool3x3s2_nhwc: x must be a contiguous 16-bit NHWC tensor with channels a multiple of 8")
    n, h, w, c = x.shape
    out = torch.empty((n, (h - 1) // 2 + 1, (w - 1) // 2 + 1, c), dtype=h16(), device=x.device)
    check(lib().lavb_maxpool3x3s2_nhwc(_ptr(x), n, h, w, c, _ptr(out), _stream()), "lavb_maxpool3x3s2_nhwc")
    _COUNT[0] += 1
    return out


def conv_pair_umma(x, w1, bias1, w2, shift2, dil, res=None, post_relu=True, out=None):
    """fused pair: mid = relu(conv3x1_dil(x) + bias1); out = [relu](conv1x3_dil(mid) + shift2 [+ res]).  A BatchNorm affine after
    the second conv is folded by the caller: w2 <- w2 * s (per output channel), shift2 <- b2 * s + t.
    x / res: contiguous f16 NHWC (n, h, w, c), c in {64, 128}, w in {32, 64, 128}; w1 / w2: (3, c, c) f16 [tap][cout][cin];
    bias1 / shift2: fp32 (c,).  The result goes to `out` when given (contiguous, the shape of x)."""
    from .capi import ConvPairDesc
    _need_cuda(x, w1, w2, bias1, shift2)
    n, h, w, c = x.shape
    assert x.dtype == h16() and x.is_contiguous() and w1.is_contiguous() and w2.is_contiguous()
    assert tuple(w1.shape) == (3, c, c) and tuple(w2.shape) == (3, c, c) and w1.dtype == w2.dtype == h16()
    assert bias1.dtype == shift2.dtype == torch.float32 and bias1.numel() == shift2.numel() == c
    if out is None:
        out = torch.empty_like(x)
    assert out.dtype == h16() and out.is_contiguous() and out.shape == x.shape
    d = ConvPairDesc()
    d.inp, d.out = x.data_ptr(), out.data_ptr()
    d.n, d.h, d.w, d.c, d.dil, d.post_relu = n, h, w, c, int(dil), int(post_relu)
    d.w1, d.bias1 = w1.data_ptr(), bias1.data_ptr()
    d.w2, d.shift2 = w2.data_ptr(), shift2.data_ptr()
    if res is not None:
        assert res.is_contiguous() and res.shape == x.shape and res.dtype == h16()
        d.res = res.data_ptr()
    e0 = _prof_begin()
    check(lib().lavb_conv_pair_umma(C.byref(d), _stream()), "lavb_conv_pair_umma")
    _prof_end(f"umma_pair:{c}x{h}x{w}", 2.0 * n * h * w * c * c * 6, e0)
    _COUNT[0] += 1
    return out


def erf_stem(rgb_u8, w27, scale, shift, out_dtype):
    """fused normalize + ERFNet initial block: rgb_u8 (N,H,W,3) uint8 -> NHWC (N,H/2,W/2,16).  w27 (27,16), scale/shift (16,)
    are HOST float32 numpy arrays (kernel parameters)."""
    _need_cuda(rgb_u8)
    _require(rgb_u8.dtype == torch.uint8 and rgb_u8.is_contiguous() and rgb_u8.dim() == 4 and rgb_u8.shape[3] == 3,
             "erf_stem: rgb_u8 must be a contiguous uint8 (N, H, W, 3) tensor")
    _require(out_dtype in (torch.float32, h16()), f"erf_stem: out_dtype must be float32 or {h16()}, got {out_dtype}")
    n, h, w, _ = rgb_u8.shape
    a, b, c = (np.ascontiguousarray(t, dtype=np.float32) for t in (w27, scale, shift))
    _require(a.shape == (27, 16) and b.shape == (16,) and c.shape == (16,), "erf_stem: w27 must be (27, 16), scale and shift (16,)")
    out = torch.empty((n, h // 2, w // 2, 16), dtype=out_dtype, device=rgb_u8.device)
    check(lib().lavb_erf_stem(_ptr(rgb_u8), n, h, w, a.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), c.ctypes.data_as(C.c_void_p),
                              _ptr(out), _DT[out_dtype], _stream()), "lavb_erf_stem")
    _COUNT[0] += 1
    return out


def erf_down16(x, w9, st):
    """fused DownsamplerBlock(16, 64): x h16 NHWC (n,h,w,16) -> (n,h/2,w/2,64) (lavb_erf_down16)."""
    _need_cuda(x, w9, st)
    _require(x.dtype == h16() and x.is_contiguous() and x.dim() == 4 and x.shape[3] == 16,
             "erf_down16: x must be a contiguous 16-bit NHWC tensor of 16 channels")
    _require(w9.dtype == torch.float32 and tuple(w9.shape) == (9, 16, 48) and w9.is_contiguous(),
             "erf_down16: w9 must be a contiguous fp32 (9, 16, 48) tensor")
    _require(st.dtype == torch.float32 and tuple(st.shape) == (64, 2) and st.is_contiguous(),
             "erf_down16: st must be a contiguous fp32 (64, 2) tensor")
    n, h, w, _ = x.shape
    out = torch.empty((n, h // 2, w // 2, 64), dtype=x.dtype, device=x.device)
    check(lib().lavb_erf_down16(_ptr(x), _ptr(out), n, h, w, _ptr(w9), _ptr(st), _stream()), "lavb_erf_down16")
    _COUNT[0] += 1
    return out


def erf_nb16(x, w4, st):
    """fused non_bottleneck_1d(16, dilation 1) block: x h16 NHWC (n,h,w,16) -> same shape (lavb_erf_nb16)."""
    _need_cuda(x, w4, st)
    _require(x.dtype == h16() and x.is_contiguous() and x.dim() == 4 and x.shape[3] == 16,
             "erf_nb16: x must be a contiguous 16-bit NHWC tensor of 16 channels")
    _require(w4.dtype == torch.float32 and tuple(w4.shape) == (4, 3, 16, 16) and w4.is_contiguous(),
             "erf_nb16: w4 must be a contiguous fp32 (4, 3, 16, 16) tensor")
    _require(st.dtype == torch.float32 and tuple(st.shape) == (4, 16, 2) and st.is_contiguous(),
             "erf_nb16: st must be a contiguous fp32 (4, 16, 2) tensor")
    n, h, w, _ = x.shape
    out = torch.empty_like(x)
    check(lib().lavb_erf_nb16(_ptr(x), _ptr(out), n, h, w, _ptr(w4), _ptr(st), _stream()), "lavb_erf_nb16")
    _COUNT[0] += 1
    return out


def cast_gru(embd, wih_t, whh_t, bih, bhh, wmlp, bmlp, steps):
    """the 6 cast branches in one launch (csrc/cast_gru.cu).  embd (N, 512) fp32; wih_t (ncmd, 512, 192), whh_t (ncmd, 64, 192) the
    TRANSPOSED GRU weights; bih / bhh (ncmd, 192); wmlp (ncmd, 2, 64); bmlp (ncmd, 2) -> (N, ncmd, steps, 2) fp32 cumulative waypoints."""
    _need_cuda(embd, wih_t, whh_t)
    n, ncmd = embd.shape[0], wih_t.shape[0]
    assert tuple(embd.shape) == (n, 512) and tuple(wih_t.shape) == (ncmd, 512, 192) and tuple(whh_t.shape) == (ncmd, 64, 192)
    assert tuple(bih.shape) == tuple(bhh.shape) == (ncmd, 192) and tuple(wmlp.shape) == (ncmd, 2, 64) and tuple(bmlp.shape) == (ncmd, 2)
    for t in (embd, wih_t, whh_t, bih, bhh, wmlp, bmlp):
        assert t.dtype == torch.float32 and t.is_contiguous()
    out = torch.empty((n, ncmd, steps, 2), dtype=torch.float32, device=embd.device)
    check(lib().lavb_cast_gru(_ptr(embd), n, _ptr(wih_t), _ptr(whh_t), _ptr(bih), _ptr(bhh), _ptr(wmlp), _ptr(bmlp), ncmd, steps,
                              _ptr(out), _stream()), "lavb_cast_gru")
    _COUNT[0] += 1
    return out


def agent_view_scratch_bytes(b):
    """bytes of agent_view's scratch for b agents (lavb_agent_view_scratch_bytes)."""
    return int(lib().lavb_agent_view_scratch_bytes(int(b)))


def agent_view(rgbs, tels, points, bev, plan, cast, cmds, other_locs, other_cmds, offsets, boxes, box_offsets, target, config,
               scratch=None, out=None):
    """The agents' debug frames, visualize's canvas before its text, in one memset and four launches (see lavb_agent_view in
    include/lav_b200.h): rgbs (B, 3, 288, 256, 3) / tels (B, 192, 480, 3) uint8; points (B, P, S) fp32 rows with x, y first (NaN
    rows are padding); bev (B, C, 320, 320) fp32 or 16-bit logits, any strides; plan / cast (B, T, 2) fp32; cmds (B,) int32;
    other_locs (K, M, T, 2) / other_cmds (K, M) fp32 the forecast rows, agent i owning rows [offsets[i], offsets[i+1]) (offsets
    (B+1,) int32 on the HOST); boxes (NB, 6) fp64 on the HOST, (x, y, w, h, cos, sin) in BEV pixels, agent i owning rows
    [box_offsets[i], box_offsets[i+1]); target (B, 2) fp32; config a capi.ViewConfig; scratch a uint8 device tensor of at least
    agent_view_scratch_bytes(B) bytes.  -> out (B, 160, 1146, 3) uint8, written into ``out`` when given."""
    _need_cuda(rgbs, tels, points, bev, plan, cast, cmds, other_locs, other_cmds, target, scratch, out)
    f32 = lambda x, shape: x.dtype == torch.float32 and tuple(x.shape) == shape and x.is_contiguous()
    if rgbs.dtype != torch.uint8 or rgbs.dim() != 5 or tuple(rgbs.shape[1:]) != (3, 288, 256, 3) or not rgbs.is_contiguous():
        raise capi.LavbError(f"agent_view: rgbs must be a contiguous (B, 3, 288, 256, 3) uint8 tensor, got {rgbs.dtype} {tuple(rgbs.shape)}")
    b = rgbs.shape[0]
    if tels.dtype != torch.uint8 or tuple(tels.shape) != (b, 192, 480, 3) or not tels.is_contiguous():
        raise capi.LavbError(f"agent_view: tels must be a contiguous ({b}, 192, 480, 3) uint8 tensor, got {tels.dtype} {tuple(tels.shape)}")
    if points.dtype != torch.float32 or points.dim() != 3 or points.shape[0] != b or points.shape[2] < 2 or not points.is_contiguous():
        raise capi.LavbError(f"agent_view: points must be a contiguous ({b}, P, >= 2) fp32 tensor, got {points.dtype} {tuple(points.shape)}")
    if bev.dtype not in (torch.float32, h16()) or bev.dim() != 4 or bev.shape[0] != b or tuple(bev.shape[2:]) != (320, 320):
        raise capi.LavbError(f"agent_view: bev must be ({b}, C, 320, 320) fp32 or {h16()} logits, got {bev.dtype} {tuple(bev.shape)}")
    if plan.dtype != torch.float32 or plan.dim() != 3 or plan.shape[0] != b or plan.shape[2] != 2 or not plan.is_contiguous():
        raise capi.LavbError(f"agent_view: plan must be a contiguous ({b}, T, 2) fp32 tensor, got {plan.dtype} {tuple(plan.shape)}")
    t = plan.shape[1]
    if not f32(cast, (b, t, 2)) or not f32(target, (b, 2)):
        raise capi.LavbError(f"agent_view: cast ({b}, {t}, 2) and target ({b}, 2) must be contiguous fp32 tensors, got "
                             f"{tuple(cast.shape)} and {tuple(target.shape)}")
    if cmds.dtype != torch.int32 or tuple(cmds.shape) != (b,) or not cmds.is_contiguous():
        raise capi.LavbError(f"agent_view: cmds must be a contiguous ({b},) int32 tensor, got {cmds.dtype} {tuple(cmds.shape)}")
    if other_locs.dim() != 4 or not f32(other_locs, (other_locs.shape[0], other_locs.shape[1], t, 2)):
        raise capi.LavbError(f"agent_view: other_locs must be a contiguous (K, M, {t}, 2) fp32 tensor, got {other_locs.dtype} "
                             f"{tuple(other_locs.shape)}")
    k, m = other_locs.shape[:2]
    if not f32(other_cmds, (k, m)):
        raise capi.LavbError(f"agent_view: other_cmds must be a contiguous ({k}, {m}) fp32 tensor, got {other_cmds.dtype} "
                             f"{tuple(other_cmds.shape)}")
    offsets = np.ascontiguousarray(offsets.numpy() if torch.is_tensor(offsets) else offsets)
    box_offsets = np.ascontiguousarray(box_offsets.numpy() if torch.is_tensor(box_offsets) else box_offsets)
    for name, o in (("offsets", offsets), ("box_offsets", box_offsets)):
        if o.dtype != np.int32 or o.shape != (b + 1,):
            raise capi.LavbError(f"agent_view: {name} must be a host ({b + 1},) int32 array, got {o.dtype} {o.shape}")
    boxes = np.ascontiguousarray(boxes.numpy() if torch.is_tensor(boxes) else boxes)
    if boxes.dtype != np.float64 or boxes.ndim != 2 or boxes.shape[1] != 6:
        raise capi.LavbError(f"agent_view: boxes must be a host (NB, 6) fp64 array, got {boxes.dtype} {boxes.shape}")
    if not isinstance(config, capi.ViewConfig):
        raise capi.LavbError("agent_view: config must be a capi.ViewConfig")
    dev = rgbs.device
    if len({dev, tels.device, points.device, bev.device, plan.device, cast.device, cmds.device, other_locs.device,
            other_cmds.device, target.device}) != 1:
        raise capi.LavbError("agent_view: the inputs must be on one device")
    need = agent_view_scratch_bytes(b)
    if scratch is None:
        scratch = torch.empty((need,), dtype=torch.uint8, device=dev)
    elif scratch.dtype != torch.uint8 or scratch.numel() < need or not scratch.is_contiguous() or scratch.device != dev:
        raise capi.LavbError(f"agent_view: scratch must be a contiguous uint8 tensor of >= {need} bytes on {dev}")
    if out is None:
        out = torch.empty((b, 160, 1146, 3), dtype=torch.uint8, device=dev)
    elif out.dtype != torch.uint8 or tuple(out.shape) != (b, 160, 1146, 3) or not out.is_contiguous() or out.device != dev:
        raise capi.LavbError(f"agent_view: out must be a contiguous ({b}, 160, 1146, 3) uint8 tensor on {dev}")
    strides = (C.c_longlong * 4)(*bev.stride())
    ip = lambda a: a.ctypes.data_as(C.c_void_p)
    code = F32 if bev.dtype == torch.float32 else capi.h16_code()
    check(lib().lavb_agent_view(_ptr(rgbs), _ptr(tels), _ptr(points), b, points.shape[1], points.shape[2], _ptr(bev), code,
                                bev.shape[1], strides, _ptr(plan), _ptr(cast), _ptr(cmds), t, _ptr(other_locs), _ptr(other_cmds),
                                k, m, ip(offsets), ip(boxes) if boxes.size else None, boxes.shape[0], ip(box_offsets), _ptr(target),
                                C.byref(config), _ptr(scratch), scratch.numel(), _ptr(out), _stream()), "lavb_agent_view")
    if b:    # histogram, points per 256 agents, boxes per 96 (at most), compose
        _COUNT[0] += int(points.shape[1] > 0) + -(-b // 256) + -(-int(box_offsets[b] - box_offsets[0]) // 96) + 1
    return out
