"""Torch-tensor front ends of the C-ABI kernels (device pointers + current stream in, tensors out).

PyTorch is plumbing here: allocation, streams, views.  Every function launches hand-written
sm_90a kernels through lav_b200.capi; nothing falls back to torch math.

Each wrapper checks what it hands to the kernels with _tensor / _out / _host, plus one _require per rule those cannot state,
so that every pointer it passes covers what the kernel reads or writes; a bad call raises LavbError, never an assert (python -O
strips asserts).  The checks read tensor metadata only, never device data, so the wrappers can be captured into CUDA graphs.
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


def _hptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise capi.LavbError("lav_b200 kernels need CUDA tensors (there is no CPU fallback)")


def _require(ok, msg):
    if not ok:
        raise capi.LavbError(msg)


def _shape_ok(got, shape):
    return shape is None or (len(got) == len(shape) and all(s is None or s == g for s, g in zip(shape, got)))


def _want(shape, dtypes):
    """'(*, 2) torch.float32 ' for shape (None, 2) and dtypes (torch.float32,); None / () leave their part out"""
    s = "" if shape is None else "(" + ", ".join("*" if v is None else str(v) for v in shape) + ("," if len(shape) == 1 else "") + ") "
    return s + (" or ".join(str(d) for d in dtypes) + " " if dtypes else "")


def _tensor(what, name, t, dtype, shape, device=None, contiguous=True):
    """-> t's shape when t is a CUDA tensor of dtype (one or a tuple; None: any) and shape (an int entry must match, a None entry
    matches any size; None: any shape), contiguous unless told otherwise, and on ``device`` when one is given; else LavbError
    (for None too)."""
    dts = dtype if isinstance(dtype, tuple) else () if dtype is None else (dtype,)
    if not (torch.is_tensor(t) and t.is_cuda and (not dts or t.dtype in dts) and _shape_ok(t.shape, shape)
            and (not contiguous or t.is_contiguous()) and (device is None or t.device == device)):
        got = f"{t.dtype} {tuple(t.shape)} on {t.device}" if torch.is_tensor(t) else type(t).__name__
        raise capi.LavbError(f"{what}: {name} must be a {'contiguous ' if contiguous else ''}{_want(shape, dts)}tensor on "
                             f"{device or 'a CUDA device'}, got {got}")
    return tuple(t.shape)


def _out(what, name, out, dtype, shape, device):
    """a new tensor when ``out`` is None, else ``out`` once _tensor has accepted it."""
    if out is None:
        return torch.empty(shape, dtype=dtype, device=device)
    _tensor(what, name, out, dtype, shape, device)
    return out


def _apart(what, name, out, **inputs):
    """LavbError unless the bytes of ``out`` share none with those of each named input tensor (the kernels read their inputs
    while they write out)."""
    o0, o1 = out.data_ptr(), out.data_ptr() + out.numel() * out.element_size()
    for k, t in inputs.items():
        t0 = t.data_ptr()
        _require(o0 == o1 or t.numel() == 0 or not (o0 < t0 + t.numel() * t.element_size() and t0 < o1),
                 f"{what}: {name} must not overlap {k}")


def _host(what, name, a, dtype, shape, cast=False):
    """a host array a kernel reads (numpy or a CPU tensor) -> it as contiguous numpy, converted to dtype with cast=True; raises
    LavbError unless it has dtype and shape (as _tensor's)."""
    a = np.ascontiguousarray(a.numpy() if torch.is_tensor(a) else a, dtype=dtype if cast else None)
    if a.dtype != dtype or not _shape_ok(a.shape, shape):
        raise capi.LavbError(f"{what}: {name} must be a host {_want(shape, (np.dtype(dtype),))}array, got {a.dtype} {a.shape}")
    return a


def launches():
    """number of kernel launches issued through this module (bench.py reports it)."""
    return _COUNT[0]


_COUNT = [0]
PROFILE = None     # bench.py sets this to a list to collect (kind, work, start_event, end_event) per launch


def _launch(fn, *args, launches=1, prof=None):
    """lib().fn(*args, current stream), its status checked, counted as ``launches`` kernels; with prof = (kind, work) and
    PROFILE set, timed into PROFILE."""
    e0 = None
    if prof is not None and PROFILE is not None:
        e0 = torch.cuda.Event(enable_timing=True)
        e0.record()
    check(getattr(lib(), fn)(*args, _stream()), fn)
    if e0 is not None:
        e1 = torch.cuda.Event(enable_timing=True)
        e1.record()
        PROFILE.append((*prof, e0, e1))
    _COUNT[0] += launches


# ----------------------------------------------------------------------------- painting
def paint(points, sem, cams, mode, copy_cols=0, out=None, out_col0=None):
    """points (N,>=3) fp32; sem (ncam,C,H,W)-shaped tensor with ANY strides (NCHW or channels-last);
    cams (ncam,41) float32 numpy (K|lidar_to_world|world_to_cam).  See lavb_paint in include/lav_b200.h."""
    n, _ = _tensor("paint", "points", points, torch.float32, (None, None), contiguous=False)
    _require(points.stride(1) == 1, "paint: points must have unit stride along a row")
    ncam, c_in, h, w = _tensor("paint", "sem", sem, torch.float32, (None,) * 4, points.device, contiguous=False)
    c_out = c_in if mode == 0 else c_in - 1
    if out_col0 is None:
        out_col0 = copy_cols
    if out is None:
        out = torch.empty((n, out_col0 + c_out), dtype=torch.float32, device=points.device)
    _, oc = _tensor("paint", "out", out, torch.float32, (n, None), points.device, contiguous=False)
    _require(out.stride(1) == 1 and oc >= out_col0 + c_out, f"paint: out must have unit stride along a row and hold "
             f"{out_col0 + c_out} columns, got {tuple(out.shape)} with strides {out.stride()}")
    cams = _host("paint", "cams", cams, np.float32, (ncam, 41), cast=True)
    s = sem.stride()
    _launch("lavb_paint", _ptr(points), n, points.stride(0), _ptr(sem), ncam, c_in, h, w, s[0], s[1], s[2], s[3], _hptr(cams), mode,
            _ptr(out), out.stride(0), out_col0, copy_cols)
    return out


def stack_sweep(src, R, dx, dy, time_idx, n_time, dst, roof_filter=False):
    """dst (n, src_cols+n_time) <- [src[:, :3] @ R + (dx,dy,0) | src[:,3:] | one_hot(time_idx)]"""
    _tensor("stack_sweep", "src", src, torch.float32, (None, None))
    _tensor("stack_sweep", "dst", dst, torch.float32, (src.shape[0], src.shape[1] + n_time), src.device)
    R = _host("stack_sweep", "R", R, np.float32, (3, 3), cast=True)
    _launch("lavb_stack_sweep", _ptr(src), src.shape[0], src.shape[1], _hptr(R), float(dx), float(dy), time_idx, n_time,
            int(roof_filter), _ptr(dst))
    return dst


def roof_filter(sweeps, pad_nan=False, out=None):
    """LAVAgent.preprocess (lav_agent.py:448-457) on the device, order preserving.  sweeps: (n, cols) or (F, n, cols) fp32
    contiguous -> (out like sweeps with the kept rows first, counts (F,) int32).  pad_nan fills rows past the count with NaN."""
    _tensor("roof_filter", "sweeps", sweeps, torch.float32, None)
    _require(sweeps.dim() in (2, 3), f"roof_filter: sweeps must be (n, cols) or (F, n, cols), got {tuple(sweeps.shape)}")
    x = sweeps if sweeps.dim() == 3 else sweeps[None]
    f, n, cols = x.shape
    if out is None:
        out = torch.empty_like(x)
    _tensor("roof_filter", "out", out, torch.float32, x.shape, x.device)
    counts = torch.empty((f,), dtype=torch.int32, device=x.device)
    _launch("lavb_roof_filter", _ptr(x), f, n, cols, n * cols, _ptr(out), n * cols, _ptr(counts), int(pad_nan))
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


# the encoders are built for the v2 point MLP only: these fp32 parameters, and point rows of at least 11 floats
_POINT_MLP = (("w1", (64, 16)), ("s1", (64,)), ("t1", (64,)), ("w2", (64, 64)), ("s2", (64,)), ("t2", (64,)))


def pillar_forward(pts, starts, counts, grid, w1, s1, t1, w2, s2, t2):
    """pts: 2-D fp32 row buffer (rows of >= D floats); cloud b = rows [starts[b], starts[b]+counts[b]).
    Returns the NHWC canvas (B, ny, nx, H2) fp32."""
    _tensor("pillar_forward", "pts", pts, torch.float32, (None, None), contiguous=False)
    _require(pts.stride(1) == 1 and pts.shape[1] >= 11, f"pillar_forward: point rows must be unit-stride and hold at least 11 "
             f"floats, got {tuple(pts.shape)} with strides {pts.stride()}")
    for (name, shape), t in zip(_POINT_MLP, (w1, s1, t1, w2, s2, t2)):
        _tensor("pillar_forward", name, t, torch.float32, shape, pts.device)
    min_x, max_x, min_y, max_y, ppm, nx, ny = grid
    d = w1.shape[1] - 5
    b, st, ct = _clouds(starts, counts, pts, "pillar_forward")
    canvas = torch.empty((b, ny, nx, w2.shape[0]), dtype=torch.float32, device=pts.device)
    ws = _workspace(pts.device, lib().lavb_pillar_workspace_bytes(b, nx, ny))
    # algorithmic bytes (SURVEY 8d): read P x D fp32 points once + write the canvas once
    _launch("lavb_pillar_forward", _ptr(pts), pts.stride(0), d, st, ct, b, min_x, max_x, min_y, max_y, ppm, nx, ny, _ptr(w1),
            _ptr(s1), _ptr(t1), w1.shape[0], _ptr(w2), _ptr(s2), _ptr(t2), w2.shape[0], _ptr(canvas), F32, _ptr(ws), launches=4,
            prof=("pillar", float(sum(int(c) for c in counts)) * d * 4 + canvas.numel() * 4))
    return canvas


def pillar_decorate(pts, starts, counts, grid, d):
    """training stage 0: returns (feat (M,d+5) fp32, cell (M,) int32), rows in input order (clouds in batch order)."""
    _tensor("pillar_decorate", "pts", pts, torch.float32, (None, None), contiguous=False)
    _require(pts.stride(1) == 1, "pillar_decorate: pts must have unit stride along a row")
    min_x, max_x, min_y, max_y, ppm, nx, ny = grid
    b, st, ct = _clouds(starts, counts, pts, "pillar_decorate")
    ws = _workspace(pts.device, lib().lavb_pillar_workspace_bytes(b, nx, ny))
    total = int(sum(int(c) for c in counts))
    feat = torch.empty((total, d + 5), dtype=torch.float32, device=pts.device)
    cell = torch.empty((total,), dtype=torch.int32, device=pts.device)
    m = C.c_int(0)
    _launch("lavb_pillar_decorate", _ptr(pts), pts.stride(0), d, st, ct, b, min_x, max_x, min_y, max_y, ppm, nx, ny, _ptr(feat),
            _ptr(cell), C.byref(m), _ptr(ws), launches=4)
    return feat[:m.value], cell[:m.value]


def pillar_scatter_max(h, cell, n_cells, want_argmax=True):
    """training stage 1: h (M,C) fp32 >= 0, cell (M,) int32 in [0, n_cells) -> (canvas (n_cells,C) fp32, arg (n_cells,C) int32
    or None).  See lavb_pillar_scatter_max in include/lav_b200.h for the tie rule and the empty-cell values."""
    m, c = _tensor("pillar_scatter_max", "h", h, torch.float32, (None, None), contiguous=False)
    _tensor("pillar_scatter_max", "cell", cell, torch.int32, (m,), h.device)
    _require(int(n_cells) >= 0, f"pillar_scatter_max: n_cells = {n_cells} < 0")
    h = h.contiguous()
    canvas = torch.empty((n_cells, c), dtype=torch.float32, device=h.device)
    arg = torch.empty((n_cells, c), dtype=torch.int32, device=h.device) if want_argmax else None
    _launch("lavb_pillar_scatter_max", _ptr(h), _ptr(cell), m, c, n_cells, _ptr(canvas), _ptr(arg), launches=2)
    return canvas, arg


def pillar_scatter_max_bwd(gcanvas, arg, cell, m):
    """gh (m,C) fp32: gh[r, c] = gcanvas[cell[r], c] where arg[cell[r], c] == r, else 0.  gcanvas may have any strides."""
    shape = _tensor("pillar_scatter_max_bwd", "gcanvas", gcanvas, torch.float32, (None, None), contiguous=False)
    _tensor("pillar_scatter_max_bwd", "arg", arg, torch.int32, shape, gcanvas.device)
    _tensor("pillar_scatter_max_bwd", "cell", cell, torch.int32, (m,), gcanvas.device)
    gcanvas = gcanvas.contiguous()
    c = gcanvas.shape[-1]
    gh = torch.empty((m, c), dtype=torch.float32, device=gcanvas.device)
    _launch("lavb_pillar_scatter_max_bwd", _ptr(gcanvas), _ptr(arg), _ptr(cell), m, c, _ptr(gh))
    return gh


# ----------------------------------------------------------------------------- convolution
def conv_taps(x, cin, in_coff, out, cout, out_coff, hog, wog, in_s, out_s, out_o, taps, w, bias=None, scale=None, shift=None,
              res=None, res_coff=0, pre_relu=False, post_relu=False, sigmoid=False, umma=False, d2s_nout=0):
    """x, out, res: contiguous NHWC buffers (N,H,W,Ctot).  taps: list of (dy,dx).
    umma=False: CUDA-core kernel, w (ntaps,cin,cout_pad16) fp32.
    umma=True : wgmma kernel, x f16, w (ntaps,cout,cin) f16."""
    _tensor("conv_taps", "x", x, h16() if umma else None, (None,) * 4)
    _tensor("conv_taps", "out", out, torch.float32 if d2s_nout else None, (x.shape[0], None, None, d2s_nout or None))
    _tensor("conv_taps", "w", w, h16() if umma else torch.float32,
            (len(taps), (cout + 31) // 32 * 32, cin) if umma else (len(taps), cin, (cout + 15) // 16 * 16))
    _require(not d2s_nout or (umma and cout == 32 and 4 * d2s_nout <= 32),
             f"conv_taps: d2s_nout = {d2s_nout} needs the wgmma kernel, cout 32 and 4 * d2s_nout <= 32")
    d = ConvDesc()
    d.inp, d.in_dtype = x.data_ptr(), _DT[x.dtype]
    d.n, d.hin, d.win, d.in_cstride = x.shape
    d.cin, d.in_coff = cin, in_coff
    d.out, d.out_dtype = out.data_ptr(), _DT[out.dtype]
    _, d.hout, d.wout, d.out_cstride = out.shape
    d.cout, d.out_coff = cout, out_coff
    d.d2s_nout = d2s_nout
    if d2s_nout:
        d.out_cstride, d.out_coff = 32, 0        # (validated as a 32-column GEMM; addressing is done by the d2s epilogue)
    d.hog, d.wog = hog, wog
    d.in_sy, d.in_sx = in_s
    d.out_sy, d.out_sx = out_s
    d.out_oy, d.out_ox = out_o
    d.ntaps = len(taps)
    for i, (dy, dx) in enumerate(taps):
        d.dy[i], d.dx[i] = dy, dx
    d.w = w.data_ptr()
    d.bias = bias.data_ptr() if bias is not None else None
    d.scale = scale.data_ptr() if scale is not None else None
    d.shift = shift.data_ptr() if shift is not None else None
    if res is not None:
        _tensor("conv_taps", "res", res, None, (*out.shape[:3], None))
        d.res, d.res_dtype, d.res_cstride, d.res_coff = res.data_ptr(), _DT[res.dtype], res.shape[3], res_coff
    d.pre_relu, d.post_relu, d.sigmoid = int(pre_relu), int(post_relu), int(sigmoid)
    _launch("lavb_conv_umma" if umma else "lavb_conv_taps", C.byref(d),
            prof=(f"umma:{cin}->{cout}x{len(taps)}taps@{hog}x{wog}", 2.0 * x.shape[0] * hog * wog * cout * cin * len(taps))
            if umma else None)
    return out


def pool2_affine_relu(x, c, in_coff, scale, shift, out, out_coff):
    _need_cuda(x, out)
    n, h, w, cs = x.shape
    _launch("lavb_pool2_affine_relu", _ptr(x), _DT[x.dtype], n, h, w, c, cs, in_coff, _ptr(scale), _ptr(shift), _ptr(out),
            out.shape[3], out_coff)
    return out


def rgb_normalize(rgb, out_dtype=torch.float32):
    """uint8 (N,H,W,3) or float (N,3,H,W) in 0..255 -> NHWC4 normalised ((x/255-.5)*2, 4th channel 0)."""
    if torch.is_tensor(rgb) and rgb.dtype == torch.uint8:
        n, h, w, _ = _tensor("rgb_normalize", "rgb", rgb, None, (None, None, None, 3), contiguous=False)
        rgb, u8 = rgb.contiguous(), 1
    else:
        n, _, h, w = _tensor("rgb_normalize", "rgb", rgb, None, (None, 3, None, None), contiguous=False)
        rgb, u8 = rgb.float().contiguous(), 0
    out = torch.empty((n, h, w, 4), dtype=out_dtype, device=rgb.device)
    _launch("lavb_rgb_normalize", _ptr(rgb), u8, n, h, w, _ptr(out), _DT[out_dtype])
    return out


def convert(src, dtype):
    _need_cuda(src)
    src = src.contiguous()
    if src.dtype == dtype:
        return src
    dst = torch.empty(src.shape, dtype=dtype, device=src.device)
    _launch("lavb_convert", _ptr(src), _DT[src.dtype], _ptr(dst), _DT[dtype], src.numel())
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
    k, _, _ = _tensor(what, "theta", theta, None, (None, 2, 3), contiguous=False)
    _tensor(what, "frame_idx", frame_idx, None, (k,), contiguous=False)
    _require(not (frame_idx.dtype.is_floating_point or frame_idx.dtype.is_complex or frame_idx.dtype == torch.bool),
             f"{what}: frame_idx must be an integer tensor, got {frame_idx.dtype}")
    if frame_idx.dtype != torch.int32:
        frame_idx = frame_idx.clamp(0, b - 1).to(torch.int32)
    return k, frame_idx.contiguous(), theta.float().contiguous()


def crop_bilinear(feats_nhwc, frame_idx, theta, crop_size):
    """feats_nhwc (B,H,W,C) contiguous fp32 (C % 4 == 0) or h16 (C % 8 == 0); frame_idx (K,) integer; theta (K,2,3) ->
    (K,crop,crop,C) in the feature dtype.  Frame indices outside [0, B) are clamped to the nearest frame."""
    _need_cuda(feats_nhwc)
    _require(crop_supported(feats_nhwc), f"crop_bilinear: need a contiguous, 16-byte aligned (B,H,W,C) map, fp32 with C % 4 == 0 "
             f"or {h16()} with C % 8 == 0; got {feats_nhwc.dtype} {tuple(feats_nhwc.shape)}")
    b, h, w, c = feats_nhwc.shape
    k, frame_idx, theta = _crop_poses("crop_bilinear", frame_idx, theta, b)
    out = torch.empty((k, crop_size, crop_size, c), dtype=feats_nhwc.dtype, device=feats_nhwc.device)
    _launch("lavb_crop_bilinear", _ptr(feats_nhwc), _DT[feats_nhwc.dtype], b, h, w, c, _ptr(frame_idx), _ptr(theta), k, crop_size,
            _ptr(out))
    return out


def crop_bilinear_u8(bev_u8, frame_idx, theta, crop_size, out=None):
    """bev_u8 (B,C,H,W) contiguous uint8; frame_idx (K,) int32; theta (K,2,3) fp32 -> fp32 NCHW (K,C,crop,crop): the crops of
    crop_bilinear read straight from a uint8 planar map (bit-identical to crop_bilinear on its float copy).  Frame indices
    outside [0, B) are clamped to the nearest frame.  ``out`` (K,C,crop,crop) fp32 contiguous is written in full if given; it
    must not overlap the map or the poses."""
    what = "crop_bilinear_u8"
    b, c, h, w = _tensor(what, "bev_u8", bev_u8, torch.uint8, (None,) * 4)
    dev = bev_u8.device
    _tensor(what, "theta", theta, None, (None, 2, 3), dev, contiguous=False)
    _tensor(what, "frame_idx", frame_idx, None, None, dev, contiguous=False)
    _require(c >= 1 and h >= 1 and w >= 1 and b >= 1, f"{what}: bev_u8 must be a non-empty (B,C,H,W) map, got {tuple(bev_u8.shape)}")
    _require(2 <= crop_size <= 65535, f"{what}: crop_size must be in [2, 65535], got {crop_size}")
    k, frame_idx, theta = _crop_poses(what, frame_idx, theta, b)
    _require(k <= 65535, f"{what}: at most 65535 crops per call, got {k}")
    out = _out(what, "out", out, torch.float32, (k, c, crop_size, crop_size), dev)
    _apart(what, "out", out, bev_u8=bev_u8, frame_idx=frame_idx, theta=theta)
    _launch("lavb_crop_bilinear_u8", _ptr(bev_u8), b, c, h, w, _ptr(frame_idx), _ptr(theta), k, crop_size, _ptr(out))
    return out


def crop_bilinear_bwd(gout_nhwc, frame_idx, theta, feat_shape, out=None):
    """gout_nhwc (K,crop,crop,C) fp32 contiguous -> gradient of crop_bilinear w.r.t. the (B,H,W,C) fp32 feature map.
    ``out`` (B,H,W,C) fp32 contiguous is written in full if given (zeros for every frame no crop samples)."""
    _require(len(feat_shape) == 4, f"crop_bilinear_bwd: feat_shape must be (B, H, W, C), got {tuple(feat_shape)}")
    b, h, w, c = (int(v) for v in feat_shape)
    _tensor("crop_bilinear_bwd", "gout", gout_nhwc, torch.float32, (None,) * 4)
    _require(gout_nhwc.data_ptr() % 16 == 0, "crop_bilinear_bwd: gout must be 16-byte aligned")
    k, frame_idx, theta = _crop_poses("crop_bilinear_bwd", frame_idx, theta, b)
    crop = gout_nhwc.shape[1]
    _require(tuple(gout_nhwc.shape) == (k, crop, crop, c), f"crop_bilinear_bwd: gout {tuple(gout_nhwc.shape)} does not match {k} "
             f"square crops of the {c}-channel map {tuple(feat_shape)}")
    gfeat = _out("crop_bilinear_bwd", "out", out, torch.float32, (b, h, w, c), gout_nhwc.device)
    _launch("lavb_crop_bilinear_bwd", _ptr(gout_nhwc), b, h, w, c, _ptr(frame_idx), _ptr(theta), k, crop, _ptr(gfeat))
    return gfeat


class CropBilinear(torch.autograd.Function):
    """crop_bilinear with its hand-written backward (gradient to the feature map only: the crop poses are data)."""

    @staticmethod
    def forward(ctx, feats_nhwc, frame_idx, theta, crop_size):
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
    n, h, wd, cs = _tensor("deconv3x3s2_small", "x", x, None, (None,) * 4)
    _tensor("deconv3x3s2_small", "w", w, None, None)
    _tensor("deconv3x3s2_small", "bias", bias, None, None)
    outs = [torch.empty((n, 2 * h, 2 * wd, no), dtype=torch.float32, device=x.device) for no in n_outs]
    ptrs = (C.c_void_p * groups)(*[o.data_ptr() for o in outs])
    no = (C.c_int * groups)(*n_outs)
    sg = (C.c_int * groups)(*[int(s) for s in sigmoids])
    _launch("lavb_deconv3x3s2_small", _ptr(x), _DT[x.dtype], n, h, wd, cs, groups, cin_g, _ptr(w), _ptr(bias), no, sg, ptrs)
    return outs


def paint_batched(points, sem, cams, mode, copy_cols, out):
    """points (F,N,>=3) fp32 contiguous; sem logical (F,ncam,C,H,W) any strides; out (F,N,copy_cols+c_out) contiguous."""
    f, n, ps = _tensor("paint_batched", "points", points, torch.float32, (None,) * 3)
    _, ncam, c_in, h, w = _tensor("paint_batched", "sem", sem, torch.float32, (f, None, None, None, None), points.device,
                                  contiguous=False)
    _tensor("paint_batched", "out", out, torch.float32, (f, n, copy_cols + (c_in if mode == 0 else c_in - 1)), points.device)
    cams = _host("paint_batched", "cams", cams, np.float32, (ncam, 41), cast=True)
    s = sem.stride()
    _launch("lavb_paint_batched", _ptr(points), f, n, ps, n * ps, _ptr(sem), ncam, c_in, h, w, s[0], s[1], s[2], s[3], s[4],
            _hptr(cams), mode, _ptr(out), out.shape[2], n * out.shape[2], copy_cols, copy_cols)
    return out


def pack_deconv2x2(weight, bias):
    """ConvTranspose2d(16, C, 2, stride=2) parameters (weight (16,C,2,2), bias (C,)) -> the 520-float table
    lavb_paint_deconv_batched reads: w[v%2][u%2][c_in][8] | bias[8]."""
    cin, c, kh, kw = weight.shape
    _require(cin == 16 and kh == 2 and kw == 2 and c <= 8, f"pack_deconv2x2: weight must be (16, C <= 8, 2, 2), got {tuple(weight.shape)}")
    w = torch.zeros((2, 2, 16, 8), dtype=torch.float32, device=weight.device)
    w[:, :, :, :c] = weight.detach().float().permute(2, 3, 0, 1)
    b = torch.zeros((8,), dtype=torch.float32, device=weight.device)
    b[:c] = bias.detach().float()
    return torch.cat([w.reshape(-1), b]).contiguous()


def paint_deconv_batched(points, feat, n_classes, deconv, cams, copy_cols, out, image_hw):
    """points (F,N,>=3) fp32; feat NHWC (F*ncam, H/2, W/2, 16) fp32 / h16 = ERFNet decoder output before output_conv;
    deconv = pack_deconv2x2(...); out (F,N,copy_cols + n_classes-1)."""
    f, n, ps = _tensor("paint_deconv_batched", "points", points, torch.float32, (None,) * 3)
    _tensor("paint_deconv_batched", "out", out, torch.float32, (f, n, copy_cols + n_classes - 1), points.device)
    h, w = image_hw
    cams = _host("paint_deconv_batched", "cams", cams, np.float32, (None, 41), cast=True)
    ncam = cams.shape[0]
    _tensor("paint_deconv_batched", "feat", feat, (torch.float32, h16()), (f * ncam, h // 2, w // 2, 16), points.device)
    _tensor("paint_deconv_batched", "deconv", deconv, torch.float32, (520,), points.device)
    _launch("lavb_paint_deconv_batched", _ptr(points), f, n, ps, n * ps, _ptr(feat), _DT[feat.dtype], ncam, n_classes, h, w,
            _ptr(deconv), _hptr(cams), _ptr(out), out.shape[2], n * out.shape[2], copy_cols, copy_cols)
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
    n, hh, wh, _ = _tensor("seg_confusion", "feat", feat, (torch.float32, h16()), (None, None, None, 16))
    _tensor("seg_confusion", "labels", labels, torch.uint8, (n, 2 * hh, 2 * wh), feat.device)
    _tensor("seg_confusion", "table", table, torch.float32, None, feat.device)
    _require(table.numel() == 520, "seg_confusion: table must be the 520-float pack_deconv2x2 table")
    lut = _host("seg_confusion", "lut", lut, np.uint8, (256,))
    c = int(n_classes)
    out = _out("seg_confusion", "out", out, torch.int32, (n, c * c + 1), feat.device)
    _launch("lavb_seg_confusion", _ptr(feat), _DT[feat.dtype], _ptr(table), _ptr(labels), _hptr(lut), n, c, 2 * hh, 2 * wh, _ptr(out),
            launches=n > 0)
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
    c = int(n_classes)
    f, n, _ = _tensor("paint_confusion", "points", points, torch.float32, (None, None, 4))
    dev = points.device
    cams = _host("paint_confusion", "cams", cams, np.float32, (None, 41), cast=True)
    ncam = cams.shape[0]
    _require(1 <= ncam <= 4, f"paint_confusion: cams must be (ncam, 41) with 1 <= ncam <= 4, got {cams.shape}")
    _, h, w = _tensor("paint_confusion", "tags", tags, torch.uint8, (f * ncam, None, None), dev)
    _require(feat is not None or stored is not None, "paint_confusion: give feat (the online painting), stored (lidar_sem rows) or both")
    if feat is not None:
        _tensor("paint_confusion", "feat", feat, (torch.float32, h16()), (f * ncam, h // 2, w // 2, 16), dev)
        _tensor("paint_confusion", "table", table, torch.float32, None, dev)
        _require(table.numel() == 520, "paint_confusion: table must be the 520-float pack_deconv2x2 table")
    elif table is not None:      # unused without feat, but held to the inputs' device all the same
        _tensor("paint_confusion", "table", table, None, None, dev, contiguous=False)
    if stored is not None:
        _tensor("paint_confusion", "stored", stored, torch.float32, (f, n, c - 1), dev)
    if meta is not None:
        _tensor("paint_confusion", "meta", meta, torch.int32, (f, 2), dev)
    lut = _host("paint_confusion", "lut", lut, np.uint8, (256,))
    _require(int(lut.max()) < c, f"paint_confusion: lut must hold classes below {c}")
    ints = lib().lavb_paint_confusion_ints(ncam, c, feat is not None, stored is not None)
    _require(ints >= 0, f"paint_confusion: {c} classes outside 2..8")
    out = _out("paint_confusion", "out", out, torch.int32, (f, ints), dev)
    if n == 0:              # empty sweeps: every count is 0 (and an empty stored buffer has no device pointer to pass)
        return out.zero_()
    min_x, max_x, min_y, max_y = (float(v) for v in window)
    _launch("lavb_paint_confusion", _ptr(points), f, n, _ptr(meta), _ptr(feat), _DT[feat.dtype] if feat is not None else F32,
            _ptr(table), _ptr(tags), _hptr(lut), _ptr(stored), _hptr(cams), ncam, c, h, w, min_x, max_x, min_y, max_y, _ptr(out),
            launches=f > 0)
    return out


STACK_JOB_DTYPE = np.dtype([("src", np.uint64), ("dst", np.uint64), ("n", np.int32), ("time_idx", np.int32), ("R", np.float32, 9),
                            ("dx", np.float32), ("dy", np.float32), ("pad", np.int32)])


def stack_jobs(d_jobs, n_jobs, max_n, src_cols, n_time, roof_filter=False):
    """d_jobs: uint8 device tensor holding n_jobs STACK_JOB_DTYPE records."""
    _tensor("stack_jobs", "d_jobs", d_jobs, torch.uint8, (None,))
    _require(d_jobs.numel() >= n_jobs * STACK_JOB_DTYPE.itemsize,
             f"stack_jobs: d_jobs holds {d_jobs.numel()} bytes, fewer than {n_jobs} 72-byte STACK_JOB_DTYPE records")
    _launch("lavb_stack_jobs", _ptr(d_jobs), n_jobs, max_n, src_cols, n_time, int(roof_filter))


# ----------------------------------------------------------------------------- temporal BEV targets
BEV_JOB_DTYPE = np.dtype([("src", np.int64), ("dst", np.int64), ("m1", np.float64, 6), ("m2", np.float64, 6), ("dx", np.int32),
                          ("dy", np.int32), ("pad", np.int32, 2)])
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
    P, h, w = _tensor("bev_targets", "src_planes", src_planes, torch.uint8, (None,) * 3)
    jobs = np.ascontiguousarray(jobs, dtype=BEV_JOB_DTYPE)
    _require(not len(jobs) or (np.abs(jobs["dx"]).max() <= BEV_MARGIN and np.abs(jobs["dy"]).max() <= BEV_MARGIN),
             f"bev_targets: a job shifts beyond the {BEV_MARGIN}-pixel margin")
    if out is None:
        out = torch.empty((int(jobs["dst"].max()) + 1 if len(jobs) else 0, h, w), dtype=torch.uint8, device=src_planes.device)
    _tensor("bev_targets", "out", out, torch.uint8, None)
    _require(tuple(out.shape[-2:]) == (h, w), f"bev_targets: out must hold ({h}, {w}) planes, got {tuple(out.shape)}")
    n_out = out.numel() // (h * w)
    _require(not len(jobs) or (jobs["src"].max() < P and jobs["dst"].min() >= 0 and jobs["dst"].max() < n_out),
             f"bev_targets: job plane index out of range ({P} source planes, {n_out} output planes)")
    if len(jobs) == 0:
        return out
    d_jobs = _to_device(jobs.view(np.uint8), src_planes.device)
    _launch("lavb_bev_targets", _ptr(d_jobs), len(jobs), _ptr(src_planes), _ptr(out), h, w)
    return out


PNG_JOB_DTYPE = np.dtype([("off", np.int64), ("len", np.int64), ("dst", np.int32), ("h", np.int32), ("w", np.int32),
                          ("pad", np.int32)])


def png_decode_gray8(src, jobs, out, status=None):
    """8-bit grayscale PNG images -> uint8 planes in one launch (see lavb_png_decode_gray8 in include/lav_b200.h), as
    cv2.imdecode(..., IMREAD_GRAYSCALE).  src: 1-D uint8 CUDA tensor of the images' zlib streams (their IDAT payloads,
    concatenated); jobs: PNG_JOB_DTYPE records (off, len, dst, h, w); out: contiguous (P, h, w) uint8 CUDA tensor, every job's (h, w)
    equal to its planes'.  -> status (n_jobs,) int32 on the device, 0 where the image decoded; a nonzero entry marks a malformed
    stream whose plane holds garbage.  The other planes of out are not written."""
    _tensor("png_decode_gray8", "src", src, torch.uint8, (None,))
    P, h, w = _tensor("png_decode_gray8", "out", out, torch.uint8, (None,) * 3, src.device)
    jobs = np.ascontiguousarray(jobs, dtype=PNG_JOB_DTYPE)
    _require(0 < h <= 4096 and 0 < w <= 4096, f"png_decode_gray8: plane size {h}x{w} outside 1..4096")
    if len(jobs):
        _require(not ((jobs["h"] != h).any() or (jobs["w"] != w).any()), f"png_decode_gray8: a job's size differs from the {h}x{w} planes")
        _require(not ((jobs["dst"] < 0).any() or (jobs["dst"] >= P).any() or len(np.unique(jobs["dst"])) != len(jobs)),
                 f"png_decode_gray8: job planes must be distinct and in 0..{P - 1}")
        _require(not ((jobs["off"] < 0).any() or (jobs["len"] < 0).any() or (jobs["off"] + jobs["len"] > src.numel()).any()),
                 f"png_decode_gray8: a job's stream lies outside the {src.numel()}-byte source")
    if status is None:
        status = torch.empty(len(jobs), dtype=torch.int32, device=src.device)
    _tensor("png_decode_gray8", "status", status, torch.int32, None, src.device)
    _require(status.numel() == len(jobs), f"png_decode_gray8: status must hold {len(jobs)} entries, got {tuple(status.shape)}")
    if len(jobs) == 0:
        return status
    d_jobs = _to_device(jobs.view(np.uint8), src.device)
    _launch("lavb_png_decode_gray8", _ptr(src), src.numel(), _ptr(d_jobs), len(jobs), _ptr(out), P, h, w, _ptr(status))
    return status


def _to_device(a, device):
    """host array -> device tensor through pinned staging, without a host synchronisation (the pinned block is not reused
    before the copy has run: the caching host allocator records the copy's stream)."""
    return torch.from_numpy(np.ascontiguousarray(a)).pin_memory().to(device, non_blocking=True)


# ----------------------------------------------------------------------------- training batches
LIDAR_SWEEP_DTYPE = np.dtype([("R_aug", np.float32, 9), ("R_mv", np.float32, 9), ("dx", np.float32), ("dy", np.float32),
                              ("time_idx", np.int32), ("row0", np.int32)])


def lidar_batch(raw, rows, sweeps, cams, image_hw, n_time, out=None):
    """The LiDAR input of a training batch in one launch (see lavb_lidar_batch in include/lav_b200.h).  raw (N, 4+C) fp32: every
    sweep's rows [xyzr | painted]; rows (B, P) int32: the raw row of each output row, -1 for a zero row; sweeps: uint8 CUDA tensor
    of LIDAR_SWEEP_DTYPE records sorted by row0; cams (ncam, 41) float32 numpy; image_hw = the camera image size.
    -> (B, P, 4+C+n_time) fp32, bit-identical to GpuLidarStacker on each sample for the same shuffle."""
    _, cols = _tensor("lidar_batch", "raw", raw, torch.float32, (None, None))
    _require(cols >= 4, f"lidar_batch: raw must be (N, 4+C), got {tuple(raw.shape)}")
    b, p = _tensor("lidar_batch", "rows", rows, torch.int32, (None, None), raw.device)
    _tensor("lidar_batch", "sweeps", sweeps, torch.uint8, None, raw.device)
    _require(sweeps.numel() % LIDAR_SWEEP_DTYPE.itemsize == 0, "lidar_batch: sweeps must hold whole 88-byte LIDAR_SWEEP_DTYPE records")
    cams = _host("lidar_batch", "cams", cams, np.float32, (None, 41), cast=True)
    c = cols - 4
    out = _out("lidar_batch", "out", out, torch.float32, (b, p, 4 + c + n_time), raw.device)
    _launch("lavb_lidar_batch", _ptr(raw), raw.shape[0], c, _ptr(rows), b * p, _ptr(sweeps), sweeps.numel() // LIDAR_SWEEP_DTYPE.itemsize,
            _hptr(cams), cams.shape[0], image_hw[0], image_hw[1], n_time, _ptr(out))
    return out


def lidar_batch_paint(raw, rows, sweeps, slots, feat, n_classes, deconv, cams, image_hw, n_time, out=None):
    """lidar_batch with every sweep painted online (see lavb_lidar_batch_paint in include/lav_b200.h).  raw (N, 4) fp32, 16-byte
    aligned: every sweep's [xyzr] rows; rows and sweeps as lidar_batch; slots (n_sweeps,) int32 on the device: the frame slot of
    each sweep; feat NHWC (F * ncam, H/2, W/2, 16) fp32 / h16 = forward_features_nhwc of the ncam images of each of F frames;
    deconv = its pack_deconv2x2 table of ``n_classes``; cams (ncam, 41) float32 numpy, the painting cameras; image_hw = their
    image size.  -> (B, P, 3 + n_classes + n_time) fp32, bit-identical to paint_deconv_batched on each sweep followed by
    lidar_batch."""
    what = "lidar_batch_paint"
    n_raw, _ = _tensor(what, "raw", raw, torch.float32, (None, 4))
    _require(raw.data_ptr() % 16 == 0, f"{what}: raw must be 16-byte aligned")
    b, p = _tensor(what, "rows", rows, torch.int32, (None, None), raw.device)
    _tensor(what, "sweeps", sweeps, torch.uint8, None, raw.device)
    _require(sweeps.numel() % LIDAR_SWEEP_DTYPE.itemsize == 0, f"{what}: sweeps must hold whole 88-byte LIDAR_SWEEP_DTYPE records")
    n_sweeps = sweeps.numel() // LIDAR_SWEEP_DTYPE.itemsize
    _tensor(what, "slots", slots, torch.int32, (n_sweeps,), raw.device)
    cams = _host(what, "cams", cams, np.float32, (None, 41), cast=True)
    ncam, (h, w) = cams.shape[0], image_hw
    _require(1 <= ncam <= 4 and h > 0 and w > 0 and h % 2 == 0 and w % 2 == 0,
             f"{what}: 1..4 cameras and an even image size, got {ncam} cameras of {h} x {w}")
    nf, _, _, _ = _tensor(what, "feat", feat, (torch.float32, h16()), (None, h // 2, w // 2, 16), raw.device)
    _require(nf % ncam == 0, f"{what}: feat holds {nf} images, not a whole number of frames of {ncam} cameras")
    _require(feat.data_ptr() % (16 if feat.dtype == torch.float32 else 8) == 0, f"{what}: feat must be 16-byte (fp32) / 8-byte aligned")
    c = int(n_classes)
    _require(2 <= c <= 8, f"{what}: n_classes must be 2..8, got {c}")
    _tensor(what, "deconv", deconv, torch.float32, (520,), raw.device)
    out = _out(what, "out", out, torch.float32, (b, p, 3 + c + n_time), raw.device)
    _apart(what, "out", out, raw=raw, rows=rows, sweeps=sweeps, slots=slots, feat=feat, deconv=deconv)
    _launch("lavb_lidar_batch_paint", _ptr(raw), n_raw, _ptr(rows), b * p, _ptr(sweeps), _ptr(slots), n_sweeps, _ptr(feat),
            _DT[feat.dtype], nf // ncam, c, _ptr(deconv), _hptr(cams), ncam, h, w, n_time, _ptr(out))
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
    _tensor("det_heatmaps", "actors", actors, torch.float32, (None, 6))
    b1, = _tensor("det_heatmaps", "offsets", offsets, torch.int32, (None,), actors.device)
    _require(b1 >= 1, "det_heatmaps: offsets must hold B+1 >= 1 entries")
    h, w, (ppm, cx0, cy0, cy1, inv_r) = det_grid(**(grid or {}))
    b = b1 - 1
    if out is None:
        out = [torch.empty((b, 2, h, w), dtype=torch.float32, device=actors.device) for _ in range(3)]
    for o in out:
        _tensor("det_heatmaps", "out", o, torch.float32, (b, 2, h, w), actors.device)
    heat, size, orim = out
    _launch("lavb_det_heatmaps", _ptr(actors), _ptr(offsets), b, h, w, ppm, cx0, cy0, cy1, inv_r, _ptr(heat), _ptr(size), _ptr(orim))
    return heat, size, orim


def _layout(parts):
    """(name, dtype, shape, byte offset) of each of a packed result buffer's parts (name, dtype, shape), laid end to end in
    order, and the buffer's size."""
    out, pos = [], 0
    for name, dt, shape in parts:
        out.append((name, dt, shape, pos))
        pos += math.prod(shape) * dt.itemsize
    return out, pos


def _views(buf, parts):
    """the named parts of a packed result buffer (uint8, on the device or a host copy), as _layout places them."""
    return {name: buf[pos:pos + math.prod(shape) * dt.itemsize].view(dt).view(shape) for name, dt, shape, pos in _layout(parts)[0]}


def _eval_parts(b, ncols):     # 8-byte parts first
    return [("iou", torch.int64, (b, 3, 2)), ("plan_err", torch.float64, (b, 2)), ("ngt", torch.int32, (b, 2)),
            ("score", torch.float32, (b, ncols)), ("flags", torch.int32, (b, ncols))]


def eval_views(buf, b, ncols):
    """the named parts of an eval_batch result buffer (on the device or a host copy of it): iou (b,3,2) int64 = per BEV channel
    (intersection, union); plan_err (b,2) fp64 = (ADE, FDE); ngt (b,2) int32 = actors per class in the window; score / flags
    (b, ncols) = the packed scores and, per column, bit 4 for a surviving peak and bit k for a match at EVAL_THRESHOLDS_M[k]."""
    return _views(buf, _eval_parts(b, ncols))


EVAL_THRESHOLDS_M = (0.5, 1.0, 2.0, 4.0)      # centre-distance thresholds of the detection matching (evaluate.cu)


def eval_batch(seg, gt, packed, actors, offsets, plan, ego_locs, grid=None, min_score=0.2, out=None):
    """The scores of one evaluation batch in one launch (see lavb_eval_batch in include/lav_b200.h).  seg (B,H,W,3) NHWC sigmoid
    probabilities, fp32 or h16; gt (B,P>=3,H,W) uint8; packed (B,7,2*n_det) fp32 from det_peaks; actors (A,6) fp32 (the
    det_heatmaps table, on the device); offsets (B+1,) int32 on the HOST; plan (B,T,2) and ego_locs (B,T+1,2) fp32; grid: the
    keyword arguments of det_grid.  -> the uint8 result buffer (written into ``out`` when given), to be read through eval_views,
    usually after one copy to the host."""
    b, h, w, _ = _tensor("eval_batch", "seg", seg, (torch.float32, h16()), (None, None, None, 3))
    dev = seg.device
    _tensor("eval_batch", "gt", gt, torch.uint8, (b, None, h, w), dev)
    _, _, ncols = _tensor("eval_batch", "packed", packed, torch.float32, (b, 7, None), dev)
    _require(ncols % 2 == 0, f"eval_batch: packed must be (B, 7, 2*n_det), got {tuple(packed.shape)}")
    _tensor("eval_batch", "actors", actors, torch.float32, (None, 6), dev)
    offsets = _host("eval_batch", "offsets", offsets, np.int32, (b + 1,))
    _, t, _ = _tensor("eval_batch", "plan", plan, torch.float32, (b, None, 2), dev)
    _tensor("eval_batch", "ego_locs", ego_locs, torch.float32, (b, t + 1, 2), dev)
    parts = _eval_parts(b, ncols)
    out = _out("eval_batch", "out", out, torch.uint8, (_layout(parts)[1],), dev)
    v = _views(out, parts)
    _, _, (ppm, cx0, cy0, cy1, _) = det_grid(**(grid or {}))
    _launch("lavb_eval_batch", _ptr(seg), _DT[seg.dtype], _ptr(gt), gt.shape[1], b, h, w, _ptr(packed), ncols // 2, _ptr(actors),
            actors.shape[0], _hptr(offsets), ppm, cx0, cy0, cy1, float(min_score), _ptr(plan), _ptr(ego_locs), t, _ptr(v["iou"]),
            _ptr(v["ngt"]), _ptr(v["score"]), _ptr(v["flags"]), _ptr(v["plan_err"]), launches=-(-b // 256))
    return out


DET_BOX_IOU_THRESHOLDS = (0.3, 0.5, 0.7)      # rotated-box IoU thresholds of the box match (det_box_eval.cu)
DET_BOX_ERRORS = ("iou", "translation_m", "scale", "heading_rad", "range_m")


def _det_box_parts(b, ncols):  # 8-byte parts first
    return [("err", torch.float64, (b, ncols, len(DET_BOX_ERRORS))), ("score", torch.float32, (b, ncols)),
            ("flags", torch.int32, (b, ncols)), ("actor", torch.int32, (b, ncols, len(DET_BOX_IOU_THRESHOLDS) + 1)),
            ("ngt", torch.int32, (b, 2))]


def det_box_views(buf, b, ncols):
    """the named parts of a det_box_eval result buffer (on the device or a host copy of it): err (b, ncols, 5) fp64 = per column
    with a 2 m match the DET_BOX_ERRORS (the IoU with the matched actor's box, translation in metres, scale error, heading error in
    radians, the actor's distance from the ego in metres), NaN otherwise; score (b, ncols) fp32 = the packed scores; flags (b,
    ncols) int32 = bit 4 survivor, bit k an IoU match at DET_BOX_IOU_THRESHOLDS[k], bit 3 the 2 m match; actor (b, ncols, 4)
    int32 = the actor row of each of those four matches, -1 for none; ngt (b, 2) int32 = actors per class in the window."""
    return _views(buf, _det_box_parts(b, ncols))


def det_box_eval(packed, actors, offsets, grid=None, min_score=0.2, out=None):
    """The box scores of one batch's detections in one launch (see lavb_det_box_eval in include/lav_b200.h).  packed (B,7,2*n_det)
    fp32 from det_peaks, actors (A,6) fp32 on the device and offsets (B+1,) int32 on the HOST (eval_batch's actor table); grid:
    the keyword arguments of det_grid; min_score as eval_batch's.  -> the uint8 result buffer (written into ``out`` when given),
    read through det_box_views, usually after one copy to the host."""
    b, _, ncols = _tensor("det_box_eval", "packed", packed, torch.float32, (None, 7, None))
    _require(ncols % 2 == 0, f"det_box_eval: packed must be (B, 7, 2*n_det), got {tuple(packed.shape)}")
    dev = packed.device
    _tensor("det_box_eval", "actors", actors, torch.float32, (None, 6), dev)
    offsets = _host("det_box_eval", "offsets", offsets, np.int32, (b + 1,))
    parts = _det_box_parts(b, ncols)
    out = _out("det_box_eval", "out", out, torch.uint8, (_layout(parts)[1],), dev)
    v = _views(out, parts)
    h, w, (ppm, cx0, cy0, cy1, _) = det_grid(**(grid or {}))
    _launch("lavb_det_box_eval", _ptr(packed), b, w, ncols // 2, _ptr(actors), actors.shape[0], _hptr(offsets), ppm, cx0, cy0, cy1,
            float(min_score), _ptr(v["score"]), _ptr(v["flags"]), _ptr(v["actor"]), _ptr(v["err"]), _ptr(v["ngt"]),
            launches=-(-b // 256))
    return out


def _forecast_parts(k):
    return [("err", torch.float64, (k, 6)), ("branch", torch.int32, (k, 2))]


def forecast_views(buf, k):
    """the named parts of a forecast_eval result buffer (on the device or a host copy of it): err (k,6) fp64 = (min ADE, min FDE,
    top-branch ADE, top-branch FDE, ADE and FDE under the recorded command or NaN); branch (k,2) int32 = (argmin-ADE branch, top
    branch)."""
    return _views(buf, _forecast_parts(k))


def forecast_eval(cast, score, target, cmd, out=None):
    """The forecast scores of k rows in one launch (see lavb_forecast_eval in include/lav_b200.h).  cast (k,C,T,2), score (k,C)
    and target (k,T,2) fp32; cmd (k,) int32, -1 where the row has no recorded command.  -> the uint8 result buffer (written into
    ``out`` when given), to be read through forecast_views, usually after one copy to the host."""
    k, c, t, _ = _tensor("forecast_eval", "cast", cast, torch.float32, (None, None, None, 2))
    dev = cast.device
    _tensor("forecast_eval", "score", score, torch.float32, (k, c), dev)
    _tensor("forecast_eval", "target", target, torch.float32, (k, t, 2), dev)
    _tensor("forecast_eval", "cmd", cmd, torch.int32, (k,), dev)
    out = _out("forecast_eval", "out", out, torch.uint8, (_layout(_forecast_parts(k))[1],), dev)
    v = forecast_views(out, k)
    _launch("lavb_forecast_eval", _ptr(cast), _ptr(score), _ptr(target), _ptr(cmd), k, c, t, _ptr(v["err"]), _ptr(v["branch"]),
            launches=k > 0)
    return out


DET_MATCH_M = 2.0       # centre-distance radius of the detected-forecast match (det_forecast.cu)


def _det_match_parts(b, k, t):  # forecast_eval's result of the k rows first (its ``out`` is buf[:56 * k]), then the match's
    return _forecast_parts(k) + [("dist", torch.float64, (k,)), ("target", torch.float32, (k, t, 2)), ("actor", torch.int32, (k,)),
                                 ("flag", torch.int32, (k,)), ("ngt", torch.int32, (b, 2))]


def det_match_views(buf, b, k, t):
    """the named parts of a det_forecast_match result buffer of b samples, k rows and t steps (on the device or a host copy):
    err (k,6) fp64 / branch (k,2) int32 = forecast_views of the rows, once forecast_eval has written buf[:56 * k]; dist (k,) fp64 =
    match distance in metres, NaN when unmatched; target (k,t,2) fp32 = the matched track's future in the ego frame, NaN unless
    matched to a tracked actor; actor (k,) int32 = the actor row within its sample, or -1; flag (k,) int32 = bit 0 matched, bit 1
    matched to a tracked actor; ngt (b,2) int32 = vehicles in the window with and without a track."""
    return _views(buf, _det_match_parts(b, k, t))


def det_forecast_match(packed, actors, offsets, row_offsets, cols, num_objs, locs, ego_locs, grid=None, match_m=DET_MATCH_M,
                       out=None):
    """The match of one batch's forecast rows to the recorded actors in one launch (see lavb_det_forecast_match in
    include/lav_b200.h).  packed (B,7,2*n_det) fp32 from det_peaks; actors (A,6) fp32 on the device and offsets (B+1,) int32 on the
    HOST (eval_batch's actor table); row_offsets (B+1,) and cols (K,) int32 on the HOST = each sample's rows and their packed
    columns; num_objs (B,) on the HOST = the recorded tracks; locs (B,max_objs,T+1,2) and ego_locs (B,T+1,2) fp32 = the labels;
    grid: the keyword arguments of det_grid.  -> the uint8 result buffer (written into ``out`` when given), read through
    det_match_views; forecast_eval(..., out=buf[:56 * K]) puts the rows' scores in the same buffer."""
    b, _, ncols = _tensor("det_forecast_match", "packed", packed, torch.float32, (None, 7, None))
    _require(ncols % 2 == 0, f"det_forecast_match: packed must be (B, 7, 2*n_det), got {tuple(packed.shape)}")
    dev = packed.device
    _tensor("det_forecast_match", "actors", actors, torch.float32, (None, 6), dev)
    offsets = _host("det_forecast_match", "offsets", offsets, np.int32, (b + 1,))
    row_offsets = _host("det_forecast_match", "row_offsets", row_offsets, np.int32, (b + 1,))
    num_objs = _host("det_forecast_match", "num_objs", num_objs, np.int32, (b,), cast=True)
    k = int(row_offsets[-1])
    cols = _host("det_forecast_match", "cols", cols, np.int32, (k,))
    _, max_objs, t1, _ = _tensor("det_forecast_match", "locs", locs, torch.float32, (b, None, None, 2), dev)
    t = t1 - 1
    _tensor("det_forecast_match", "ego_locs", ego_locs, torch.float32, (b, t + 1, 2), dev)
    parts = _det_match_parts(b, k, t)
    out = _out("det_forecast_match", "out", out, torch.uint8, (_layout(parts)[1],), dev)
    v = _views(out, parts)
    h, w, (ppm, cx0, cy0, cy1, _) = det_grid(**(grid or {}))
    _launch("lavb_det_forecast_match", _ptr(packed), b, w, ncols // 2, _ptr(actors), actors.shape[0], _hptr(offsets), _hptr(row_offsets),
            _hptr(cols), _hptr(num_objs), _ptr(locs), _ptr(ego_locs), max_objs, t, ppm, cx0, cy0, cy1, float(match_m), _ptr(v["actor"]),
            _ptr(v["flag"]), _ptr(v["dist"]), _ptr(v["target"]), _ptr(v["ngt"]), launches=-(-b // 128))
    return out


# one (actor, step) record of plan_safety's actor table (lavb_plan_safety in include/lav_b200.h)
PLAN_SAFETY_ACTOR_DTYPE = np.dtype([("x", np.float64), ("y", np.float64), ("cos", np.float64), ("sin", np.float64),
                                    ("e1", np.float64), ("e2", np.float64), ("typ", np.int32), ("present", np.int32)])
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
    b, n, t, _ = _tensor("plan_safety", "traj", traj, torch.float32, (None, None, None, 2))
    dev = traj.device
    offsets = _host("plan_safety", "offsets", offsets, np.int32, (b + 1,))
    rec = PLAN_SAFETY_ACTOR_DTYPE.itemsize
    _tensor("plan_safety", "actors", actors, torch.uint8, (None,), dev)
    _require(actors.numel() % (rec * t) == 0, f"plan_safety: actors must hold {rec}-byte records, {t} per actor row, got {actors.numel()} bytes")
    _tensor("plan_safety", "ego_ext", ego_ext, torch.float64, (b, 2), dev)
    _, _, h, w = _tensor("plan_safety", "bev", bev, torch.uint8, (b, None, None, None), dev)
    out = _out("plan_safety", "out", out, torch.int32, (b, n, 8), dev)
    _, _, (ppm, cx0, cy0, cy1, _) = det_grid(**(grid or {}))
    _launch("lavb_plan_safety", _ptr(traj), b, n, t, _ptr(actors), actors.numel() // (rec * t), _hptr(offsets), _ptr(ego_ext), _ptr(bev),
            bev[0].numel() if b else h * w, h, w, ppm, cx0, cy0, cy1, _ptr(out), launches=-(-b // 512))
    return out


DRIVING_SCORE_STEP_S = 0.25       # default step period of the recordings (lav_b200.evaluate's driving-score protocol)
DRIVING_SCORE_COMFORT = ("lon_acceleration", "lon_jerk", "yaw_rate", "yaw_acceleration", "lat_acceleration")
DRIVING_SCORE_FIELDS = ("fault_step", "fault_row", "fault_class", "exempt_step", "exempt_row", "exempt_class", "ttc_step", "ttc_row",
                        "off_road_step", "comfort_mask") + tuple(f"{c}_step" for c in DRIVING_SCORE_COMFORT) + ("invalid_step",)


def _driving_parts(b, n):     # 8-byte part first
    return [("ep", torch.float64, (b, n, 2)), ("res", torch.int32, (b, n, len(DRIVING_SCORE_FIELDS)))]


def driving_score_views(buf, b, n):
    """the named parts of a driving_score result buffer of b samples and n trajectories (on the device or a host copy), each
    (b, n): fault_step / fault_row / fault_class = the first at-fault collision's step (1..T), actor row and class; exempt_* the
    same for the first exempt collision; ttc_step / ttc_row = the first time-to-collision violation; off_road_step; comfort_mask =
    bit q set when DRIVING_SCORE_COMFORT[q] fails, {term}_step its first failing step; invalid_step = the first invalid step;
    -1 for none.  progress / length (fp64) = the arc-length position s of the last point on the expert polyline and its length L."""
    v = _views(buf, _driving_parts(b, n))
    out = {name: v["res"][..., i] for i, name in enumerate(DRIVING_SCORE_FIELDS)}
    out["progress"], out["length"] = v["ep"][..., 0], v["ep"][..., 1]
    return out


def driving_score(traj, expert, actors, offsets, ego_ext, bev, grid=None, dt=DRIVING_SCORE_STEP_S, out=None):
    """The driving-score terms of n ego trajectories per sample in one launch (see lavb_driving_score in include/lav_b200.h).
    traj (B,n,T,2) fp32 in the label frame; expert (B,T,2) fp32 = the polyline progress is measured along; actors =
    PLAN_SAFETY_ACTOR_DTYPE records as a 1-D uint8 tensor on the device, T + 1 per actor row (steps 0..T), sample i owning rows
    [offsets[i], offsets[i+1]) (offsets (B+1,) int32 on the HOST); ego_ext (B,2) fp64; bev (B,P,H,W) uint8, plane 0 the road; grid:
    the keyword arguments of det_grid; dt the step period in seconds.  -> the uint8 result buffer (written into ``out`` when
    given), read through driving_score_views, usually after one copy to the host."""
    b, n, t, _ = _tensor("driving_score", "traj", traj, torch.float32, (None, None, None, 2))
    dev = traj.device
    _tensor("driving_score", "expert", expert, torch.float32, (b, t, 2), dev)
    offsets = _host("driving_score", "offsets", offsets, np.int32, (b + 1,))
    rec = PLAN_SAFETY_ACTOR_DTYPE.itemsize * (t + 1)
    _tensor("driving_score", "actors", actors, torch.uint8, (None,), dev)
    _require(actors.numel() % rec == 0, f"driving_score: actors must hold {t + 1} 56-byte records per actor row, got {actors.numel()} bytes")
    _tensor("driving_score", "ego_ext", ego_ext, torch.float64, (b, 2), dev)
    _, _, h, w = _tensor("driving_score", "bev", bev, torch.uint8, (b, None, None, None), dev)
    _require(isinstance(dt, (int, float)) and math.isfinite(dt) and dt > 0, f"driving_score: dt must be a finite period > 0, got {dt!r}")
    parts = _driving_parts(b, n)
    out = _out("driving_score", "out", out, torch.uint8, (_layout(parts)[1],), dev)
    _apart("driving_score", "out", out, traj=traj, expert=expert, actors=actors, ego_ext=ego_ext, bev=bev)
    v = _views(out, parts)
    _, _, (ppm, cx0, cy0, cy1, _) = det_grid(**(grid or {}))
    _launch("lavb_driving_score", _ptr(traj), _ptr(expert), b, n, t, _ptr(actors), actors.numel() // rec, _hptr(offsets), _ptr(ego_ext),
            _ptr(bev), bev[0].numel() if b else h * w, h, w, ppm, cx0, cy0, cy1, float(dt), _ptr(v["ep"]), _ptr(v["res"]),
            launches=-(-b // 512))
    return out


def agent_control_state_bytes(turn_n, speed_n):
    """bytes of one agent's controller state (lavb_agent_control_state_bytes); all-zero bytes are a new route."""
    n = int(lib().lavb_agent_control_state_bytes(int(turn_n), int(speed_n)))
    _require(n != 0, f"agent_control: PID windows {turn_n}, {speed_n} outside 1..64")
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
    b, t, _ = _tensor("agent_control", "plan", plan, torch.float32, (None, None, 2))
    dev = plan.device
    _tensor("agent_control", "cast", cast, torch.float32, (b, t, 2), dev)
    k, c, _, _ = _tensor("agent_control", "other_locs", other_locs, torch.float32, (None, None, t, 2), dev)
    _tensor("agent_control", "other_cmds", other_cmds, torch.float32, (k, c), dev)
    _tensor("agent_control", "pred_bra", pred_bra, torch.float32, (b,), dev)
    _tensor("agent_control", "speed", speed, torch.float32, (b,), dev)
    offsets = _host("agent_control", "offsets", offsets, np.int32, (b + 1,))
    dcmd = torch.is_tensor(cmds) and cmds.is_cuda
    if dcmd:
        _tensor("agent_control", "device cmds", cmds, torch.int32, (b,), dev)
    else:
        cmds = _host("agent_control", "cmds", cmds, np.int32, (b,))
    _require(isinstance(config, capi.ControlConfig), "agent_control: config must be a capi.ControlConfig")
    _tensor("agent_control", "state", state, torch.uint8, (b * agent_control_state_bytes(config.turn_n, config.speed_n),), dev)
    control = _out("agent_control", "control", control, torch.float32, (b, 3), dev)
    flags = _out("agent_control", "flags", flags, torch.int32, (b,), dev)
    _launch("lavb_agent_control_dcmd" if dcmd else "lavb_agent_control", _ptr(plan), _ptr(cast), b, t, c, _ptr(other_locs),
            _ptr(other_cmds), k, _hptr(offsets), _ptr(pred_bra), _ptr(speed), _ptr(cmds) if dcmd else _hptr(cmds), C.byref(config),
            _ptr(state), _ptr(control), _ptr(flags), launches=-(-b // 512))
    return control, flags


NAV_STATE_DTYPE = np.dtype([("ekf_x", np.float64, (3,)), ("ekf_p", np.float64, (3,)), ("wp_x", np.float64), ("wp_y", np.float64),
                            ("rp_x", np.float64), ("rp_y", np.float64), ("route_scale", np.float64), ("ekf_scale", np.float64),
                            ("frames", np.int32), ("wp_idx", np.int32), ("wp_cmd", np.int32), ("rp_idx", np.int32),
                            ("lane_counter", np.int32), ("lane_changed", np.int32), ("pad", np.int32, (2,))])   # lavb_nav_state


def agent_nav_state_bytes():
    """bytes of one agent's lavb_nav_state record (lavb_agent_nav_state_bytes)."""
    n = int(lib().lavb_agent_nav_state_bytes())
    _require(n == NAV_STATE_DTYPE.itemsize, f"agent_nav: the library's state record has {n} bytes, NAV_STATE_DTYPE {NAV_STATE_DTYPE.itemsize}")
    return n


def agent_nav_front(nodes, node_cmd, route, gnss, compass, state, cmds=None, nxps=None, poses=None, flags=None):
    """The front of B agents' tick in one launch (lavb_agent_nav_front in include/lav_b200.h): nodes (M, 2) fp64 and node_cmd (M,)
    int32 = every route's nodes; route (B, 2) int32 = (start, count) per agent; gnss (B, 2) fp64 = lat, lon; compass (B,) fp64,
    raw; state B lavb_nav_state records (uint8, updated in place).  -> (cmds (B,) int32, nxps (B, 2) fp32, poses (B, 3) fp64,
    flags (B,) int32 of LAVB_NAV_* bits), written into the given tensors when given."""
    b, _ = _tensor("agent_nav_front", "route", route, torch.int32, (None, 2))
    dev = route.device
    m, _ = _tensor("agent_nav_front", "nodes", nodes, torch.float64, (None, 2), dev)
    _tensor("agent_nav_front", "node_cmd", node_cmd, torch.int32, (m,), dev)
    _tensor("agent_nav_front", "gnss", gnss, torch.float64, (b, 2), dev)
    _tensor("agent_nav_front", "compass", compass, torch.float64, (b,), dev)
    _tensor("agent_nav_front", "state", state, torch.uint8, (b * agent_nav_state_bytes(),), dev)
    cmds = _out("agent_nav_front", "cmds", cmds, torch.int32, (b,), dev)
    nxps = _out("agent_nav_front", "nxps", nxps, torch.float32, (b, 2), dev)
    poses = _out("agent_nav_front", "poses", poses, torch.float64, (b, 3), dev)
    flags = _out("agent_nav_front", "flags", flags, torch.int32, (b,), dev)
    _launch("lavb_agent_nav_front", b, _ptr(nodes), _ptr(node_cmd), m, _ptr(route), _ptr(gnss), _ptr(compass), _ptr(state), _ptr(cmds),
            _ptr(nxps), _ptr(poses), _ptr(flags), launches=1 if b else 0)
    return cmds, nxps, poses, flags


def agent_nav_update(control, speed, gnss, compass, state):
    """EKF.step of B agents after the controls (lavb_agent_nav_update): control (B, 3) fp32 = agent_control's output (steer in
    column 0); speed (B,) fp64 m/s; gnss (B, 2) fp64; compass (B,) fp64, raw; state as in agent_nav_front, updated in place."""
    _need_cuda(state)
    b = state.numel() // agent_nav_state_bytes()
    _tensor("agent_nav_update", "control", control, torch.float32, (b, 3))
    dev = control.device
    _tensor("agent_nav_update", "speed", speed, torch.float64, (b,), dev)
    _tensor("agent_nav_update", "gnss", gnss, torch.float64, (b, 2), dev)
    _tensor("agent_nav_update", "compass", compass, torch.float64, (b,), dev)
    _tensor("agent_nav_update", "state", state, torch.uint8, None, dev)
    _require(state.numel() == b * agent_nav_state_bytes(), "agent_nav_update: state must hold whole lavb_nav_state records")
    _launch("lavb_agent_nav_update", b, _ptr(control), _ptr(speed), _ptr(gnss), _ptr(compass), _ptr(state), launches=1 if b else 0)


def stack_job_poses(d_jobs, b, t, gap, keep, tick, ring_pose, poses=None):
    """the R / dx / dy fields of stack_jobs' table from the device pose ring (lavb_stack_job_poses): d_jobs the uint8 table of
    b * t STACK_JOB_DTYPE records; ring_pose (b, keep, 3) fp64, ``poses`` (b, 3) fp64 written to slot tick % keep first."""
    _tensor("stack_job_poses", "jobs", d_jobs, torch.uint8, None)
    _require(d_jobs.numel() == b * t * STACK_JOB_DTYPE.itemsize, f"stack_job_poses: jobs must hold {b} x {t} records")
    _tensor("stack_job_poses", "ring_pose", ring_pose, torch.float64, (b, keep, 3))
    if poses is not None:
        _tensor("stack_job_poses", "poses", poses, torch.float64, (b, 3))
    _launch("lavb_stack_job_poses", _ptr(d_jobs), b, t, gap, keep, int(tick), _ptr(ring_pose), _ptr(poses), launches=1 if b else 0)


PILLAR_ENCODER ="sorted"    # name of the 16-bit pipeline's pillar encoder, reported by bench.py; it selects nothing


def pillar_forward_sorted(pts, starts, counts, grid, w1, s1, t1, w2, s2, t2, canvas16=False):
    """tensor-core pillar encoder of the 16-bit pipeline: counting sort by canvas cell + persistent mma.sync encoder
    (lavb_pillar_forward_sorted).  Returns the NHWC canvas: fp32 (B,ny,nx,H2); with canvas16, h16 (B,ny,nx,H2), saturating —
    what the 16-bit pipeline feeds the backbone."""
    _tensor("pillar_forward_sorted", "pts", pts, torch.float32, (None, None), contiguous=False)
    _require(pts.stride(1) == 1 and pts.shape[1] >= 11, f"pillar_forward_sorted: point rows must be unit-stride and hold at least "
             f"11 floats, got {tuple(pts.shape)} with strides {pts.stride()}")
    for (name, shape), t in zip(_POINT_MLP, (w1, s1, t1, w2, s2, t2)):
        _tensor("pillar_forward_sorted", name, t, torch.float32, shape, pts.device)
    min_x, max_x, min_y, max_y, ppm, nx, ny = grid
    d = w1.shape[1] - 5
    b, st, ct = _clouds(starts, counts, pts, "pillar_forward_sorted")
    total = int(sum(int(c) for c in counts))
    h2 = w2.shape[0]
    canvas = torch.empty((b, ny, nx, h2), dtype=h16() if canvas16 else torch.float32, device=pts.device)
    ws = _workspace(pts.device, lib().lavb_pillar_sorted_workspace_bytes(b, nx, ny, total))
    _launch("lavb_pillar_forward_sorted", _ptr(pts), pts.stride(0), d, st, ct, b, min_x, max_x, min_y, max_y, ppm, nx, ny, _ptr(w1),
            _ptr(s1), _ptr(t1), w1.shape[0], _ptr(w2), _ptr(s2), _ptr(t2), h2, _ptr(canvas), 2 if canvas16 else 0, _ptr(ws),
            launches=6, prof=("pillar", float(total) * d * 4 + float(b) * ny * nx * h2 * (2 if canvas16 else 4)))
    return canvas


def det_peaks(center, box, ori, min_score=0.2, max_det=15):
    """center (LOGITS) fp32 NHWC (B,H,W,ncls), box, ori: fp32 NHWC (B,H,W,2), all contiguous -> packed (B,7,ncls*max_det)
    (see lavb_det_peaks)."""
    b, h, w, ncls = _tensor("det_peaks", "center", center, torch.float32, (None,) * 4)
    _tensor("det_peaks", "box", box, torch.float32, (b, h, w, 2))
    _tensor("det_peaks", "ori", ori, torch.float32, (b, h, w, 2))
    packed = torch.empty((b, 7, ncls * max_det), dtype=torch.float32, device=center.device)
    ws = _workspace(center.device, lib().lavb_det_peaks_workspace_bytes(b, ncls))
    _launch("lavb_det_peaks", _ptr(center), _ptr(box), _ptr(ori), b, h, w, ncls, min_score, max_det, _ptr(packed), _ptr(ws), launches=2)
    return packed


def stem7x7s2_u8(img_u8, w_h16, bias, mean, std):
    """img_u8 (B, ncam, H, cam_w, 3) uint8 contiguous; w_h16 (64,160) packed by pack_stem_weights; bias (64,)
    -> f16 NHWC (B, H/2, ncam*cam_w/2, 64)."""
    b, ncam, h, cw, _ = _tensor("stem7x7s2_u8", "img_u8", img_u8, torch.uint8, (None, None, None, None, 3))
    _tensor("stem7x7s2_u8", "w_h16", w_h16, h16(), (64, 160))
    _tensor("stem7x7s2_u8", "bias", bias, torch.float32, (64,))
    _require(len(mean) == 3 and len(std) == 3, "stem7x7s2_u8: mean and std hold 3 values")
    out = torch.empty((b, (h - 1) // 2 + 1, (ncam * cw - 1) // 2 + 1, 64), dtype=h16(), device=img_u8.device)
    m = (C.c_float * 3)(*[float(v) for v in mean])
    sd = (C.c_float * 3)(*[float(v) for v in std])
    _launch("lavb_stem7x7s2_u8", _ptr(img_u8), b, ncam, h, cw, _ptr(w_h16), _ptr(bias), m, sd, _ptr(out))
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
    n, h, w, cin = _tensor("conv7x7s2_umma", "x", x, h16(), (None,) * 4)
    _require(cin % 64 == 0 and h >= 7 and w >= 7, f"conv7x7s2_umma: x must have cin % 64 == 0 and h, w >= 7, got {tuple(x.shape)}")
    _tensor("conv7x7s2_umma", "w_packed", w_packed, h16(), (49, 64, cin))
    _tensor("conv7x7s2_umma", "bias", bias, torch.float32, None)
    _require(bias.numel() == 64, f"conv7x7s2_umma: bias must hold 64 values, got {bias.numel()}")
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    out = _out("conv7x7s2_umma", "out", out, h16(), (n, ho, wo, 64), x.device)
    _launch("lavb_conv7x7s2_umma", _ptr(x), n, h, w, cin, _ptr(w_packed), _ptr(bias), _ptr(out),
            prof=(f"stem7x7s2:{cin}->64@{h}x{w}", 2.0 * n * ho * wo * 64 * cin * 49))
    return out


def conv3x3_umma(x, w, cout, stride, bias=None, scale=None, shift=None, pre_relu=False, out=None):
    """3x3 / pad 1 / stride 1 or 2 convolution with output channels in M (lavb_conv3x3_umma): x contiguous f16 NHWC (n, h, w, cin),
    cin in (64, 128, 384); w (9, cout, cin) f16, the conv_umma packing; cout in (64, 128, 256); bias / scale / shift fp32 (cout,)
    or None -> f16 NHWC (n, (h-1)//s+1, (w-1)//s+1, cout) = [relu](conv + bias) * scale + shift, written into `out` when given."""
    n, h, wd, cin = _tensor("conv3x3_umma", "x", x, h16(), (None,) * 4)
    _tensor("conv3x3_umma", "w", w, h16(), (9, cout, cin))
    for name, v in (("bias", bias), ("scale", scale), ("shift", shift)):
        if v is not None:
            _tensor("conv3x3_umma", name, v, torch.float32, None)
            _require(v.numel() == cout, f"conv3x3_umma: {name} must hold {cout} values, got {v.numel()}")
    ho, wo = (h - 1) // stride + 1, (wd - 1) // stride + 1
    out = _out("conv3x3_umma", "out", out, h16(), (n, ho, wo, cout), x.device)
    # the label format of conv_taps' wgmma launches, so that bench.py's conv roofline keeps covering the same layers
    _launch("lavb_conv3x3_umma", _ptr(x), n, h, wd, cin, stride, _ptr(w), cout, _ptr(bias), _ptr(scale), _ptr(shift), int(pre_relu),
            _ptr(out), prof=(f"umma:{cin}->{cout}x9taps@{ho}x{wo}", 2.0 * n * ho * wo * cout * cin * 9))
    return out


def pack_conv7x7s2_weights(w):
    """(64, cin, 7, 7) conv weights -> (49, 64, cin) f16 [tap = ky*7 + kx][cout][cin], the layout conv7x7s2_umma reads."""
    _require(w.dim() == 4 and tuple(w.shape[2:]) == (7, 7) and w.shape[0] == 64,
             f"pack_conv7x7s2_weights: w must be (64, cin, 7, 7), got {tuple(w.shape)}")
    return w.permute(2, 3, 0, 1).reshape(49, 64, w.shape[1]).to(h16()).contiguous()


def maxpool3x3s2_nhwc(x):
    """MaxPool2d(3, 2, 1) on a contiguous f16 NHWC tensor."""
    n, h, w, c = _tensor("maxpool3x3s2_nhwc", "x", x, h16(), (None,) * 4)
    _require(c % 8 == 0, f"maxpool3x3s2_nhwc: x must have channels a multiple of 8, got {c}")
    out = torch.empty((n, (h - 1) // 2 + 1, (w - 1) // 2 + 1, c), dtype=h16(), device=x.device)
    _launch("lavb_maxpool3x3s2_nhwc", _ptr(x), n, h, w, c, _ptr(out))
    return out


def conv_pair_umma(x, w1, bias1, w2, shift2, dil, res=None, post_relu=True, out=None):
    """fused pair: mid = relu(conv3x1_dil(x) + bias1); out = [relu](conv1x3_dil(mid) + shift2 [+ res]).  A BatchNorm affine after
    the second conv is folded by the caller: w2 <- w2 * s (per output channel), shift2 <- b2 * s + t.
    x / res: contiguous f16 NHWC (n, h, w, c), c in {64, 128}, w in {32, 64, 128}; w1 / w2: (3, c, c) f16 [tap][cout][cin];
    bias1 / shift2: fp32 (c,).  The result goes to `out` when given (contiguous, the shape of x)."""
    from .capi import ConvPairDesc
    n, h, w, c = _tensor("conv_pair_umma", "x", x, h16(), (None,) * 4)
    _tensor("conv_pair_umma", "w1", w1, h16(), (3, c, c))
    _tensor("conv_pair_umma", "w2", w2, h16(), (3, c, c))
    for name, v in (("bias1", bias1), ("shift2", shift2)):
        _tensor("conv_pair_umma", name, v, torch.float32, None)
        _require(v.numel() == c, f"conv_pair_umma: {name} must hold {c} values, got {v.numel()}")
    out = _out("conv_pair_umma", "out", out, h16(), x.shape, x.device)
    d = ConvPairDesc()
    d.inp, d.out = x.data_ptr(), out.data_ptr()
    d.n, d.h, d.w, d.c, d.dil, d.post_relu = n, h, w, c, int(dil), int(post_relu)
    d.w1, d.bias1 = w1.data_ptr(), bias1.data_ptr()
    d.w2, d.shift2 = w2.data_ptr(), shift2.data_ptr()
    if res is not None:
        _tensor("conv_pair_umma", "res", res, h16(), x.shape)
        d.res = res.data_ptr()
    _launch("lavb_conv_pair_umma", C.byref(d), prof=(f"umma_pair:{c}x{h}x{w}", 2.0 * n * h * w * c * c * 6))
    return out


def erf_stem(rgb_u8, w27, scale, shift, out_dtype):
    """fused normalize + ERFNet initial block: rgb_u8 (N,H,W,3) uint8 -> NHWC (N,H/2,W/2,16).  w27 (27,16), scale/shift (16,)
    are HOST float32 numpy arrays (kernel parameters)."""
    n, h, w, _ = _tensor("erf_stem", "rgb_u8", rgb_u8, torch.uint8, (None, None, None, 3))
    _require(out_dtype in (torch.float32, h16()), f"erf_stem: out_dtype must be float32 or {h16()}, got {out_dtype}")
    a = _host("erf_stem", "w27", w27, np.float32, (27, 16), cast=True)
    b = _host("erf_stem", "scale", scale, np.float32, (16,), cast=True)
    c = _host("erf_stem", "shift", shift, np.float32, (16,), cast=True)
    out = torch.empty((n, h // 2, w // 2, 16), dtype=out_dtype, device=rgb_u8.device)
    _launch("lavb_erf_stem", _ptr(rgb_u8), n, h, w, _hptr(a), _hptr(b), _hptr(c), _ptr(out), _DT[out_dtype])
    return out


def erf_down16(x, w9, st):
    """fused DownsamplerBlock(16, 64): x h16 NHWC (n,h,w,16) -> (n,h/2,w/2,64) (lavb_erf_down16)."""
    n, h, w, _ = _tensor("erf_down16", "x", x, h16(), (None, None, None, 16))
    _tensor("erf_down16", "w9", w9, torch.float32, (9, 16, 48))
    _tensor("erf_down16", "st", st, torch.float32, (64, 2))
    out = torch.empty((n, h // 2, w // 2, 64), dtype=x.dtype, device=x.device)
    _launch("lavb_erf_down16", _ptr(x), _ptr(out), n, h, w, _ptr(w9), _ptr(st))
    return out


def erf_nb16(x, w4, st):
    """fused non_bottleneck_1d(16, dilation 1) block: x h16 NHWC (n,h,w,16) -> same shape (lavb_erf_nb16)."""
    n, h, w, _ = _tensor("erf_nb16", "x", x, h16(), (None, None, None, 16))
    _tensor("erf_nb16", "w4", w4, torch.float32, (4, 3, 16, 16))
    _tensor("erf_nb16", "st", st, torch.float32, (4, 16, 2))
    out = torch.empty_like(x)
    _launch("lavb_erf_nb16", _ptr(x), _ptr(out), n, h, w, _ptr(w4), _ptr(st))
    return out


def cast_gru(embd, wih_t, whh_t, bih, bhh, wmlp, bmlp, steps, out=None):
    """the 6 cast branches in one launch (csrc/cast_gru.cu).  embd (N, 512) fp32; wih_t (ncmd, 512, 192), whh_t (ncmd, 64, 192) the
    TRANSPOSED GRU weights; bih / bhh (ncmd, 192); wmlp (ncmd, 2, 64); bmlp (ncmd, 2) -> (N, ncmd, steps, 2) fp32 cumulative waypoints,
    written into ``out`` (contiguous, not overlapping an input) when given."""
    n, _ = _tensor("cast_gru", "embd", embd, torch.float32, (None, 512))
    dev = embd.device
    ncmd, _, _ = _tensor("cast_gru", "wih_t", wih_t, torch.float32, (None, 512, 192), dev)
    ins = dict(embd=embd, wih_t=wih_t, whh_t=whh_t, bih=bih, bhh=bhh, wmlp=wmlp, bmlp=bmlp)
    for name, shape in (("whh_t", (ncmd, 64, 192)), ("bih", (ncmd, 192)), ("bhh", (ncmd, 192)), ("wmlp", (ncmd, 2, 64)), ("bmlp", (ncmd, 2))):
        _tensor("cast_gru", name, ins[name], torch.float32, shape, dev)
    _require(1 <= ncmd <= 65535 and steps >= 1,
             f"cast_gru: need 1 <= ncmd <= 65535 and steps >= 1, got ncmd {ncmd}, steps {steps}")
    out = _out("cast_gru", "out", out, torch.float32, (n, ncmd, steps, 2), dev)
    _apart("cast_gru", "out", out, **ins)
    _launch("lavb_cast_gru", _ptr(embd), n, _ptr(wih_t), _ptr(whh_t), _ptr(bih), _ptr(bhh), _ptr(wmlp), _ptr(bmlp), ncmd, steps, _ptr(out))
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
    b, _, _, _, _ = _tensor("agent_view", "rgbs", rgbs, torch.uint8, (None, 3, 288, 256, 3))
    dev = rgbs.device
    _tensor("agent_view", "tels", tels, torch.uint8, (b, 192, 480, 3), dev)
    _, p, s = _tensor("agent_view", "points", points, torch.float32, (b, None, None), dev)
    _require(s >= 2, f"agent_view: points rows must hold x, y, got {tuple(points.shape)}")
    _tensor("agent_view", "bev", bev, (torch.float32, h16()), (b, None, 320, 320), dev, contiguous=False)
    _, t, _ = _tensor("agent_view", "plan", plan, torch.float32, (b, None, 2), dev)
    _tensor("agent_view", "cast", cast, torch.float32, (b, t, 2), dev)
    _tensor("agent_view", "target", target, torch.float32, (b, 2), dev)
    _tensor("agent_view", "cmds", cmds, torch.int32, (b,), dev)
    k, m, _, _ = _tensor("agent_view", "other_locs", other_locs, torch.float32, (None, None, t, 2), dev)
    _tensor("agent_view", "other_cmds", other_cmds, torch.float32, (k, m), dev)
    offsets = _host("agent_view", "offsets", offsets, np.int32, (b + 1,))
    box_offsets = _host("agent_view", "box_offsets", box_offsets, np.int32, (b + 1,))
    boxes = _host("agent_view", "boxes", boxes, np.float64, (None, 6))
    _require(isinstance(config, capi.ViewConfig), "agent_view: config must be a capi.ViewConfig")
    need = agent_view_scratch_bytes(b)
    if scratch is None:
        scratch = torch.empty((need,), dtype=torch.uint8, device=dev)
    _tensor("agent_view", "scratch", scratch, torch.uint8, None, dev)
    _require(scratch.numel() >= need, f"agent_view: scratch must hold >= {need} bytes, got {scratch.numel()}")
    out = _out("agent_view", "out", out, torch.uint8, (b, 160, 1146, 3), dev)
    strides = (C.c_longlong * 4)(*bev.stride())
    code = F32 if bev.dtype == torch.float32 else capi.h16_code()
    # histogram, points per 256 agents, boxes per 96 (at most), compose
    n = int(p > 0) + -(-b // 256) + -(-int(box_offsets[b] - box_offsets[0]) // 96) + 1 if b else 0
    _launch("lavb_agent_view", _ptr(rgbs), _ptr(tels), _ptr(points), b, p, s, _ptr(bev), code, bev.shape[1], strides, _ptr(plan),
            _ptr(cast), _ptr(cmds), t, _ptr(other_locs), _ptr(other_cmds), k, m, _hptr(offsets), _hptr(boxes) if boxes.size else None,
            boxes.shape[0], _hptr(box_offsets), _ptr(target), C.byref(config), _ptr(scratch), scratch.numel(), _ptr(out), launches=n)
    return out
