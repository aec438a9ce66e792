"""The inference pillar encoders, lavb_pillar_forward ("fp32") and lavb_pillar_forward_sorted with an fp32 ("sorted") or h16
("sorted_h16") canvas, against the fp64 statement tests/util.pillar_forward_ref64 across their C-ABI contract.  Every
element of every canvas is held to the statement's per-element bound (derived in its docstring: a bound every correct
encoder meets, not a measured error); empty cells must be exactly 0.

The sorted encoder's segmented max is tested where it can go wrong: its order is cell order, so the clouds below place
pillar heads exactly on, one before and one after a 32-row quarter edge, a 128-row batch edge and a window edge, with
pillar sizes from 1 to 5000, one pillar holding a whole 40 000-point cloud, and runs of single-point pillars filling whole
quarters.  The persistent loop runs at the bench shapes (B = 32 x 40 000 and 64 x 120 000, every frame compared), at one
window per block and below one batch.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from lav_b200 import capi, ops
from lav_b200.capi import LavbError
from tests import util

pytestmark = pytest.mark.gpu

GRID4 = (-10.0, 70.0, -40.0, 40.0, 4.0, 320, 320)
SMALL = (-10.0, 70.0, -40.0, 40.0, 0.25, 20, 20)
ENCODERS = ["fp32", "sorted", "sorted_h16"]


def _weights(seed=0, device="cuda"):
    g = torch.Generator().manual_seed(seed)
    w1 = torch.randn(64, 16, generator=g) * 0.25
    w2 = torch.randn(64, 64, generator=g) * 0.125
    s1, s2 = 0.5 + torch.rand(64, generator=g), 0.5 + torch.rand(64, generator=g)
    t1, t2 = torch.randn(64, generator=g) * 0.5, torch.randn(64, generator=g) * 0.5
    return [t.to(device).contiguous() for t in (w1, s1, t1, w2, s2, t2)]


def encode(enc, pts, starts, counts, grid, ws):
    if enc == "fp32":
        return ops.pillar_forward(pts, starts, counts, grid, *ws)
    return ops.pillar_forward_sorted(pts, starts, counts, grid, *ws, canvas16=enc == "sorted_h16")


def check(enc, got, pts, starts, counts, grid, ws, frames_per_chunk=8):
    """every element of got within the statement's bound, empty cells exactly 0 -> max err / bound"""
    assert tuple(got.shape) == (len(counts), grid[6], grid[5], 64)
    assert got.dtype == (ops.h16() if enc == "sorted_h16" else torch.float32)
    worst = 0.0
    for b0 in range(0, len(counts), frames_per_chunk):
        sl = slice(b0, b0 + frames_per_chunk)
        want, bound = util.pillar_forward_ref64(pts, starts[sl], counts[sl], grid, *ws, enc)
        g = got[sl].double()
        err = (g - want).abs()
        assert bool(torch.isfinite(g).all())
        bad = err > bound
        assert not bool(bad.any()), (f"{int(bad.sum())} elements outside the bound, worst excess {float((err - bound).max()):.3e}, "
                                     f"first at {bad.nonzero()[0].tolist()} (frame offset {b0})")
        live = bound > 0
        if bool(live.any()):
            worst = max(worst, float((err[live] / bound[live]).max()))
    return worst


def run_and_check(pts, starts, counts, grid, ws, encs=ENCODERS):
    return {e: check(e, encode(e, pts, starts, counts, grid, ws), pts, starts, counts, grid, ws) for e in encs}


# ----------------------------------------------------------------------------------------------------- cloud builders
def _cell_points(cells, sizes, grid, seed, device="cuda"):
    """points of pillars of the given sizes, pillar k inside canvas cell cells[k] = row * nx + col (so sorted order is the
    order of cells), jittered inside the cell; 11 columns."""
    mn_x, _, mn_y, _, ppm, nx, ny = grid
    g = torch.Generator().manual_seed(seed)
    cells = torch.as_tensor(cells, dtype=torch.int64)
    sizes = torch.as_tensor(sizes, dtype=torch.int64)
    rc = torch.repeat_interleave(cells, sizes)
    row, col = rc // nx, rc % nx
    xi, yi = ny - 1 - row, col
    n = len(rc)
    p = torch.rand(n, 11, generator=g) * 2 - 1
    p[:, 0] = mn_x + (xi.float() + 0.05 + 0.9 * torch.rand(n, generator=g)) / ppm
    p[:, 1] = mn_y + (yi.float() + 0.05 + 0.9 * torch.rand(n, generator=g)) / ppm
    p[:, 2] = torch.randn(n, generator=g)
    perm = torch.randperm(n, generator=g)                          # the sort must undo a shuffled input order
    return p[perm].contiguous().to(device)


def _heads(targets, tail):
    """pillar sizes whose heads land exactly on the given sorted slots (first pillar at slot 0)"""
    cuts = [0] + sorted(targets)
    return [b - a for a, b in zip(cuts, cuts[1:])] + [tail]


def _segment_case(name):
    """-> list of pillar-size lists, one per frame"""
    if name == "sizes":
        return [[1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 1000, 5000, 1, 3]]
    if name == "whole_cloud":
        return [[40000]]
    if name == "heads_at_edges":    # on / one before / one after quarter (32k), batch (128k) and window edges
        t = [k * e + d for e in (32, 128) for k in range(1, 8) for d in (-1, 0, 1)]
        t += [384 * k + d for k in range(1, 5) for d in (-1, 0, 1)] + [1024, 1025, 1151, 1152, 1153, 1279]
        return [_heads(set(t), 77)]
    if name == "single_runs":       # single-point pillars filling whole quarters, between long pillars
        return [[1] * 128 + [32] + [1] * 64 + [200] + [1] * 96 + [31] + [1] * 33 + [129] + [1] * 256]
    if name == "across_frames":     # windows that begin in one frame and end in the next
        return [[1] * 50 + [100], [60, 1, 1, 300], [], [127, 1] * 5]
    raise KeyError(name)


@pytest.mark.parametrize("case", ["sizes", "whole_cloud", "heads_at_edges", "single_runs", "across_frames"])
def test_segmented_max_at_known_boundaries(cuda, case):
    grid = GRID4
    ws = _weights(1)
    frames = _segment_case(case)
    clouds = []
    for b, sizes in enumerate(frames):
        # distinct cells in increasing order, spread over the canvas so rows and columns vary
        cells = (torch.arange(len(sizes)) * 997 + 13 * b) % (320 * 320)
        cells, _ = torch.sort(cells)
        clouds.append(_cell_points(cells, sizes, grid, seed=100 + b) if sizes else torch.zeros((0, 11), device=cuda))
    counts = [len(c) for c in clouds]
    pts = torch.cat(clouds).contiguous()
    starts = list(np.cumsum([0] + counts[:-1]))
    worst = run_and_check(pts, starts, counts, grid, ws)
    print(f"\n{case}: max err / bound " + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))


def _bench_cloud(b, n, seed):
    """(b * n, 11) fp32 on the GPU: 30 % of the points in dense clusters (pillars of hundreds of points), the rest spread over
    and beyond the window."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    p = torch.rand(b * n, 11, generator=g, device="cuda")
    p[:, 0] = p[:, 0] * 84 - 12
    p[:, 1] = torch.rand(b * n, generator=g, device="cuda") * 84 - 42
    dense = torch.rand(b * n, generator=g, device="cuda") < 0.3
    p[dense, 0] = torch.randn(int(dense.sum()), generator=g, device="cuda") * 2 + 10
    p[dense, 1] = torch.randn(int(dense.sum()), generator=g, device="cuda") * 2
    p[:, 2] = torch.randn(b * n, generator=g, device="cuda")
    return p.contiguous()


@pytest.mark.parametrize("b,n", [(32, 40000), (64, 120000)])
def test_bench_shapes_every_frame(cuda, b, n):
    """more windows than blocks: the grid is min(ceil(total / 128), 3 SMs), so each block walks many windows"""
    pts = _bench_cloud(b, n, seed=b)
    starts, counts = [i * n for i in range(b)], [n] * b
    windows = math.ceil(b * n / 128)
    assert windows > 3 * torch.cuda.get_device_properties(0).multi_processor_count * 10
    worst = run_and_check(pts, starts, counts, GRID4, _weights(2))
    print(f"\nB = {b} x {n}: max err / bound " + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))


@pytest.mark.parametrize("case", ["one_window_per_block", "below_one_batch"])
def test_persistent_loop_small(cuda, case):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if case == "one_window_per_block":        # every window a whole batch of single-point pillars: one window per block
        total = 3 * sms * 128
        cells = torch.randperm(320 * 320, generator=torch.Generator().manual_seed(5))[:total].sort().values
        pts = _cell_points(cells, [1] * total, GRID4, seed=6)
    else:
        pts = _bench_cloud(1, 100, seed=7)
    run_and_check(pts, [0], [len(pts)], GRID4, _weights(3))


def test_statement_on_gpu_equals_cpu(cuda):
    pts = _bench_cloud(3, 20000, seed=8)
    ws = _weights(4)
    for mode in ENCODERS:
        a, ab = util.pillar_forward_ref64(pts, [0, 20000, 40000], [20000] * 3, GRID4, *ws, mode)
        c, cb = util.pillar_forward_ref64(pts.cpu(), [0, 20000, 40000], [20000] * 3, GRID4, *[w.cpu() for w in ws], mode)
        diff = (a.cpu() - c).abs()
        same = diff <= 1e-12 * float(c.abs().max())
        assert float(same.double().mean()) > 1 - 1e-5 and bool((diff <= cb).all()), mode   # a half rounding may flip at a tie
        assert float((ab.cpu() - cb).abs().max()) <= 1e-9 * float(cb.abs().max())


# ----------------------------------------------------------------------------------------------------- clouds and batch
def _clouds_case(name):
    """-> (pts 2-D view, starts, counts)"""
    base = _bench_cloud(1, 30000, seed=9)
    if name == "batch1":
        return base, [0], [30000]
    if name == "batch2":
        return base, [0, 17000], [17000, 13000]
    if name == "batch128":
        g = torch.Generator().manual_seed(10)
        counts = torch.randint(0, 230, (128,), generator=g).tolist()
        counts[0] = counts[64] = counts[127] = 0
        return base, [b * 230 for b in range(128)], counts
    if name == "empty_first_middle_last":
        return base, [0, 0, 5000, 9000, 30000], [0, 5000, 0, 3000, 0]
    if name == "gaps_and_shared_rows":         # gaps between clouds; clouds 1 and 2 share rows
        return base, [100, 5000, 6000, 20000], [3000, 2000, 2500, 7000]
    if name == "out_of_buffer_order":
        return base, [20000, 0, 9000], [9000, 8000, 4000]
    raise KeyError(name)


@pytest.mark.parametrize("case", ["batch1", "batch2", "batch128", "empty_first_middle_last", "gaps_and_shared_rows",
                                  "out_of_buffer_order"])
def test_clouds_and_batch(cuda, case):
    pts, starts, counts = _clouds_case(case)
    run_and_check(pts, starts, counts, GRID4, _weights(11))


@pytest.mark.parametrize("stride", [11, 12, 16, 64])
def test_point_stride(cuda, stride):
    base = _bench_cloud(1, 6000, seed=12)
    wide = torch.full((6000, stride), float("nan"), device=cuda)
    wide[:, :11] = base
    pts = wide[:, :11]
    assert pts.stride(0) == stride
    run_and_check(pts, [0, 2500], [2500, 3500], GRID4, _weights(13))


def test_frame_alone_equals_its_row_of_the_batch(cuda):
    pts, starts, counts = _clouds_case("batch128")
    ws = _weights(14)
    for enc in ENCODERS:
        batch = encode(enc, pts, starts, counts, GRID4, ws).double()
        for b in (1, 63, 126):
            alone = encode(enc, pts, [starts[b]], [counts[b]], GRID4, ws).double()
            _, cb = util.pillar_forward_ref64(pts, [starts[b]], [counts[b]], GRID4, *ws, enc, parts="centroid")
            assert bool(((alone[0] - batch[b]).abs() <= cb[0]).all()), (enc, b)


# ----------------------------------------------------------------------------------------------------- grid
def _grid_for(min_x, max_x, min_y, max_y, ppm):
    """the smallest grid the window fits, from the same fp32 rule the entry points check"""
    f32 = np.float32
    top = lambda lo, hi: int((np.nextafter(f32(hi), f32(-np.inf)) - f32(lo)) * f32(ppm))       # noqa: E731
    return (min_x, max_x, min_y, max_y, ppm, max(round((max_x - min_x) * ppm), top(min_x, max_x)),
            max(round((max_y - min_y) * ppm), top(min_y, max_y)))


@pytest.mark.parametrize("grid", [
    _grid_for(-10.0, 70.0, -40.0, 40.0, 1.0), _grid_for(-10.0, 70.0, -40.0, 40.0, 8.0), _grid_for(-10.0, 70.0, -40.0, 40.0, 3.0),
    _grid_for(-10.1, 69.9, -40.3, 39.7, 4.0),                                 # min not a multiple of 1 / ppm
    (-10.0, 70.0, -20.0, 20.0, 4.0, 320, 160),                               # nx != ny: xi >= 160 all clamp onto row 0
    (-40.0, 40.0, -40.0, 40.0, 4.0, 320, 320),                               # x and y round onto index 320 = nx = ny
], ids=["ppm1", "ppm8", "ppm3", "offset_min", "non_square", "round_onto_n"])
def test_grids(cuda, grid):
    pts = _bench_cloud(2, 15000, seed=15)
    edge = pts[:64].clone()
    edge[:, 0], edge[:, 1] = (grid[0] + grid[1]) / 2, (grid[2] + grid[3]) / 2
    hi_x = float(np.nextafter(np.float32(grid[1]), np.float32(-np.inf)))
    hi_y = float(np.nextafter(np.float32(grid[3]), np.float32(-np.inf)))
    edge[:16, 0], edge[16:32, 1] = hi_x, hi_y
    edge[32:48, 0], edge[32:48, 1] = hi_x, hi_y
    edge[48:56, 0], edge[56:, 1] = grid[0], grid[2]
    pts = torch.cat([edge, pts]).contiguous()
    keep, xi, yi = util.pillar_locate(pts[:64, 0], pts[:64, 1], grid)
    assert bool(keep.all())
    if grid[5] == 320 and grid[0] == -40.0:
        assert int(xi.max()) == 320 and int(yi.max()) == 320
    run_and_check(pts, [0, 15064], [15064, 15000], grid, _weights(16))


@pytest.mark.parametrize("case", ["all_outside", "empty_batch"])
def test_nothing_kept(cuda, case):
    pts = _bench_cloud(1, 5000, seed=17)
    if case == "all_outside":
        pts[:, 0] += 200
        counts = [2500, 2500]
    else:
        counts = [0, 0]
    for enc in ENCODERS:
        got = encode(enc, pts, [0, 2500], counts, GRID4, _weights(18))
        assert bool((got.float().view(-1) == 0).all()) and not bool(torch.signbit(got.float()).any())


# ----------------------------------------------------------------------------------------------------- values
def _value_cloud(seed=19):
    """pillars of 1..6 points; returns (pts, row index of the first point of each of 8 multi-point pillars)"""
    sizes = [1, 3, 6, 2, 5, 4, 3, 6] * 6
    cells = torch.arange(len(sizes)) * 2111 % (320 * 320)
    cells, _ = cells.sort()
    g = torch.Generator().manual_seed(seed)
    pts = _cell_points(cells, sizes, GRID4, seed).cpu()
    return pts, g


@pytest.mark.parametrize("where", ["x", "y", "z", "feature"])
@pytest.mark.parametrize("value", ["nan", "inf", "-inf"])
def test_non_finite_values(cuda, where, value):
    """NaN or +-inf in x or y drops the point.  NaN in z or a feature column: the point's hidden units are NaN and every
    ReLU makes them 0, so it contributes relu(t2); a NaN z makes its pillar's centroid, hence every point of that pillar,
    NaN.  +-inf in z or a feature: the fp32 encoder computes with the infinities (the statement in fp64 does the same) and
    may write +inf; the sorted encoder saturates the split to +-131008 and stays finite."""
    pts, g = _value_cloud()
    col = {"x": 0, "y": 1, "z": 2, "feature": 7}[where]
    hit = torch.randperm(len(pts), generator=g)[:40]
    pts[hit, col] = float(value)
    pts = pts.to(cuda)
    ws = _weights(20)
    ws[3] = ws[3].abs()                  # w2 >= 0: an infinite hidden unit reaches the fp32 canvas as +inf, not as NaN
    for enc in ENCODERS:
        got = encode(enc, pts, [0], [len(pts)], GRID4, ws).double()
        want, bound = util.pillar_forward_ref64(pts, [0], [len(pts)], GRID4, *ws, enc)
        if enc != "fp32":
            assert bool(torch.isfinite(got).all()), enc
        if value == "nan" or where in ("x", "y") or enc == "fp32":
            fin = torch.isfinite(want)
            assert torch.equal(got[~fin], want[~fin]), enc                  # the +inf the fp32 encoder writes
            ok = (got - want).abs() <= torch.nan_to_num(bound, nan=float("inf"))
            assert bool(ok[fin].all()), enc
        if value == "nan" and where in ("z", "feature"):                # a NaN point contributes exactly relu(t2)
            t2 = ws[5].double().clamp_min(0)
            keep, xi, yi = util.pillar_locate(pts[hit, 0], pts[hit, 1], GRID4)
            cells = ((319 - xi).clamp(0, 319) * 320 + yi.clamp(0, 319))
            assert bool((got.view(-1, 64)[cells] >= (util.round_h16(t2) if enc == "sorted_h16" else t2) * (1 - 2 ** -20)).all())
    if value != "nan" and where in ("z", "feature"):
        got = encode("fp32", pts, [0], [len(pts)], GRID4, ws)
        assert bool(torch.isposinf(got).any()) and not bool(torch.isnan(got).any())


@pytest.mark.parametrize("mag", [1e3, 6e4, 1e5, 1e30])
@pytest.mark.parametrize("where", ["z", "feature"])
def test_large_values(cuda, where, mag):
    """fp32 encoder: within the bound, and within 1e-5 of the canvas scale, at every magnitude.  Sorted encoder: within the
    bound while the decorated values stay inside the half range; far beyond it the hi / lo split saturates and the canvas is
    wrong without any sign (still finite).  At 1e30 the bound itself is vacuous (it scales with sum |f w|), so the sorted
    encoder's error is measured against the canvas scale there."""
    pts, g = _value_cloud(21)
    col = {"z": 2, "feature": 7}[where]
    pts[:, col] = (torch.rand(len(pts), generator=g) * 2 - 1) * mag
    pts = pts.to(cuda)
    ws = _weights(22)
    excess, rel = {}, {}
    for enc in ENCODERS:
        got = encode(enc, pts, [0], [len(pts)], GRID4, ws).double()
        want, bound = util.pillar_forward_ref64(pts, [0], [len(pts)], GRID4, *ws, enc)
        assert bool(torch.isfinite(got).all())
        excess[enc] = float(((got - want).abs() - bound).max())
        rel[enc] = float((got - want).abs().max() / want.abs().max())
    print(f"\n{where} ~ {mag:g}: max (err - bound) " + ", ".join(f"{k} {v:.3e}" for k, v in excess.items()) +
          "; max err / canvas scale " + ", ".join(f"{k} {v:.2e}" for k, v in rel.items()))
    assert excess["fp32"] <= 0 and rel["fp32"] < 1e-5
    if mag <= 1e3 or (mag <= 6e4 and where == "feature"):      # z - centroid can reach 2 mag
        assert excess["sorted"] <= 0 and excess["sorted_h16"] <= 0
    if mag >= 1e30:
        assert rel["sorted"] > 1e-2 and rel["sorted_h16"] > 1e-2


@pytest.mark.parametrize("w", [1.0, 1 / 3], ids=["w_exact_in_half", "w_third"])
def test_layer1_keeps_fp32_precision(cuda, w):
    """A hidden unit that cancels the point's coordinate (h = w x - 60 w and w y - 10 w on a strip of cells at x ~ 60): it
    needs layer 1 to carry x and w to ~fp32 accuracy, well below their half ulps (2^-6 at 60, 2^-13 at 1/3), and the
    identity layer 2 passes it through to the canvas.  w = 1 isolates the feature's lo part, w = 1/3 the weight's."""
    n = 4000
    g = torch.Generator().manual_seed(23)
    pts = torch.rand(n, 11, generator=g)
    pts[:, 0] = 60 + torch.rand(n, generator=g) * 0.2499
    pts[:, 1] = 10 + torch.rand(n, generator=g) * 20
    pts = pts.to(cuda)
    w1 = torch.zeros(64, 16)
    w1[:32, 0] = w
    w1[32:, 1] = w
    t1 = torch.cat([torch.full((32,), -60.0 * w), torch.full((32,), -10.0 * w)])
    ws = [t.to(cuda).contiguous() for t in (w1, torch.ones(64), t1, torch.eye(64), torch.ones(64), torch.zeros(64))]
    worst = run_and_check(pts, [0], [n], GRID4, ws)
    print(f"\ncancellation, w = {w:.4f}: max err / bound {worst}")


# ----------------------------------------------------------------------------------------------------- whole buffer
def _lib_call(enc, pts, starts, counts, grid, ws, canvas_addr, work_addr, stride=None, d=11, h=(64, 64), mode=None, batch=None,
              ptrs=None):
    b = len(counts)
    st, ct = (C.c_longlong * max(b, 1))(*starts), (C.c_int * max(b, 1))(*counts)
    p = {"pts": pts.data_ptr(), **{k: t.data_ptr() for k, t in zip(("w1", "s1", "t1", "w2", "s2", "t2"), ws)}}
    p.update(ptrs or {})
    v = lambda a: C.c_void_p(a)                                      # noqa: E731
    args = (v(p["pts"]), stride or pts.stride(0), d, st, ct, b if batch is None else batch, *[float(x) for x in grid[:5]],
            grid[5], grid[6], v(p["w1"]), v(p["s1"]), v(p["t1"]), h[0], v(p["w2"]), v(p["s2"]), v(p["t2"]), h[1],
            v(canvas_addr))
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    if enc == "fp32":
        rc = capi.lib().lavb_pillar_forward(*args, capi.F32 if mode is None else mode, v(work_addr), s)
    else:
        rc = capi.lib().lavb_pillar_forward_sorted(*args, (2 if enc == "sorted_h16" else 0) if mode is None else mode,
                                                   v(work_addr), s)
    torch.cuda.synchronize()
    return rc


def _ws_bytes(enc, b, grid, total):
    if enc == "fp32":
        return capi.lib().lavb_pillar_workspace_bytes(b, grid[5], grid[6])
    return capi.lib().lavb_pillar_sorted_workspace_bytes(b, grid[5], grid[6], total)


PAD = 256      # canary bytes on each side of the canvas (a multiple of 16, so the sorted encoder's canvas stays aligned)


def _canary_canvas(enc, b, grid):
    esize = 2 if enc == "sorted_h16" else 4
    nbytes = b * grid[6] * grid[5] * 64 * esize
    buf = torch.full((nbytes + 2 * PAD,), 0xFF, dtype=torch.uint8, device="cuda")      # NaN in both fp32 and half
    view = buf[PAD:PAD + nbytes].view(ops.h16() if esize == 2 else torch.float32).view(b, grid[6], grid[5], 64)
    return buf, view


@pytest.mark.parametrize("enc", ENCODERS)
def test_canvas_and_workspace_canaries(cuda, enc):
    """a NaN-filled canvas inside a canary buffer, and a 0xFF-filled workspace of exactly the reported size followed by a
    canary: every empty cell comes out exactly 0, everything within the bound, and no byte outside either buffer changes"""
    pts, starts, counts = _clouds_case("batch2")
    ws = _weights(24)
    buf, canvas = _canary_canvas(enc, 2, GRID4)
    nws = _ws_bytes(enc, 2, GRID4, sum(counts))
    work = torch.full((nws + 4096,), 0xFF, dtype=torch.uint8, device=cuda)
    work[nws:] = torch.arange(4096, device=cuda).to(torch.uint8)
    tail = work[nws:].clone()
    assert _lib_call(enc, pts, starts, counts, GRID4, ws, canvas.data_ptr(), work.data_ptr()) == 0
    assert bool((buf[:PAD] == 0xFF).all()) and bool((buf[-PAD:] == 0xFF).all())
    assert torch.equal(work[nws:], tail)
    check(enc, canvas, pts, starts, counts, GRID4, ws)
    _, bound = util.pillar_forward_ref64(pts, starts, counts, GRID4, *ws, enc)
    empty = bound.sum(-1) == 0
    assert bool(empty.any()) and bool((canvas.double()[empty] == 0).all())


@pytest.mark.parametrize("enc", ENCODERS)
def test_two_calls_differ_only_by_centroid_order(cuda, enc):
    pts = _bench_cloud(4, 40000, seed=25)
    starts, counts = [i * 40000 for i in range(4)], [40000] * 4
    ws = _weights(26)
    a = encode(enc, pts, starts, counts, GRID4, ws).double()
    b = encode(enc, pts, starts, counts, GRID4, ws).double()
    _, cb = util.pillar_forward_ref64(pts, starts, counts, GRID4, *ws, enc, parts="centroid")
    assert bool(((a - b).abs() <= cb).all())


def test_h16_canvas_is_the_fp32_canvas_rounded_once(cuda):
    pts = _bench_cloud(4, 40000, seed=27)
    starts, counts = [i * 40000 for i in range(4)], [40000] * 4
    ws = _weights(28)
    c32 = encode("sorted", pts, starts, counts, GRID4, ws)
    c16 = encode("sorted_h16", pts, starts, counts, GRID4, ws).double()
    _, cb = util.pillar_forward_ref64(pts, starts, counts, GRID4, *ws, "sorted_h16", parts="centroid")
    assert bool(((c16 - util.round_h16(c32.double())).abs() <= cb).all())
    single = cb == 0                              # cells whose pillars' centroids are order-independent: bit-equal
    assert bool(single.any()) and torch.equal(c16[single], util.round_h16(c32.double())[single])


# ----------------------------------------------------------------------------------------------------- rejections
BAD_GRIDS = {
    "ppm0": (-10.0, 70.0, -40.0, 40.0, 0.0, 320, 320), "ppm_neg": (-10.0, 70.0, -40.0, 40.0, -4.0, 320, 320),
    "ppm_nan": (-10.0, 70.0, -40.0, 40.0, float("nan"), 320, 320), "ppm_inf": (-10.0, 70.0, -40.0, 40.0, float("inf"), 320, 320),
    "min_nan": (float("nan"), 70.0, -40.0, 40.0, 4.0, 320, 320), "max_inf": (-10.0, float("inf"), -40.0, 40.0, 4.0, 320, 320),
    "min_eq_max": (-10.0, -10.0, -40.0, 40.0, 4.0, 320, 320), "min_gt_max": (-10.0, 70.0, 40.0, -40.0, 4.0, 320, 320),
    "nx0": (-10.0, 70.0, -40.0, 40.0, 4.0, 0, 320), "ny_neg": (-10.0, 70.0, -40.0, 40.0, 4.0, 320, -1),
    "grid_too_small_ppm8": (-10.0, 70.0, -40.0, 40.0, 8.0, 320, 320),
    "nx_one_short": (-10.0, 70.0, -40.0, 40.0, 4.0, 318, 320),
    "ny_one_short": (-40.0, 40.0, -40.0, 40.0, 4.0, 320, 319),        # y just below 40 reaches index 320
}
BAD_ARGS = ["batch0", "batch129", "neg_count", "neg_start", "d10", "h1_32", "stride10", "mode1", "null_pts", "null_w1",
            "null_t2", "null_canvas", "null_ws", "pts_misaligned", "w2_misaligned", "ws_misaligned", "canvas_misaligned"]


@pytest.mark.parametrize("bad", list(BAD_GRIDS) + BAD_ARGS)
@pytest.mark.parametrize("enc", ENCODERS)
def test_rejects_before_launch(cuda, enc, bad):
    pts = _bench_cloud(1, 3000, seed=29)
    ws = _weights(30)
    grid, starts, counts, kw = BAD_GRIDS.get(bad, SMALL), [0, 1000], [1000, 2000], {}
    if bad == "batch0":
        kw["batch"] = 0
    elif bad == "batch129":
        starts, counts = [0] * 129, [20] * 129
    elif bad == "neg_count":
        counts = [1000, -1]
    elif bad == "neg_start":
        starts = [-5, 1000]
    elif bad == "d10":
        kw["d"] = 10
    elif bad == "h1_32":
        kw["h"] = (32, 64)
    elif bad == "stride10":
        kw["stride"] = 10
    elif bad == "mode1":
        kw["mode"] = 1
    elif bad.startswith("null_") and bad[5:] in ("pts", "w1", "t2"):
        kw["ptrs"] = {bad[5:]: 0}
    elif bad == "pts_misaligned":
        kw["ptrs"] = {"pts": pts.data_ptr() + 2}
    elif bad == "w2_misaligned":
        kw["ptrs"] = {"w2": torch.zeros(64 * 64 + 1, device=cuda)[1:].data_ptr()}
    nb = max(len(counts), 1)
    sized = SMALL if bad in BAD_ARGS else GRID4
    buf, canvas = _canary_canvas(enc, nb, sized)
    nws = _ws_bytes(enc, nb, sized, max(sum(counts), 0)) + 64
    work = torch.full((nws,), 0x5A, dtype=torch.uint8, device=cuda)
    canvas_addr = buf.data_ptr() + PAD
    work_addr = work.data_ptr()
    if bad == "null_canvas":
        canvas_addr = 0
    elif bad == "null_ws":
        work_addr = 0
    elif bad == "ws_misaligned":
        work_addr += 8
    elif bad == "canvas_misaligned":
        canvas_addr += 2 if enc == "fp32" else 8
    if bad == "mode1" and enc == "fp32":
        kw["mode"] = capi.F16                    # the fp32 encoder's canvas_dtype must be LAVB_F32
    rc = _lib_call(enc, pts, starts, counts, grid, ws, canvas_addr, work_addr, **kw)
    assert rc != 0, bad
    assert capi.lib().lavb_last_error()
    assert bool((buf == 0xFF).all()) and bool((work == 0x5A).all())


@pytest.mark.parametrize("enc", ENCODERS)
def test_wrappers_reject(cuda, enc):
    pts = _bench_cloud(1, 3000, seed=31)
    ws = _weights(32)
    for starts, counts in (([0, 1000], [1000, 2001]), ([2990], [11]), ([0, 1], [5])):
        with pytest.raises(LavbError):
            encode(enc, pts, starts, counts, GRID4, ws)
    for k, shape in ((0, (64, 15)), (0, (32, 16)), (3, (64, 32)), (3, (32, 64)), (1, (63,)), (5, (65,))):
        bad = list(ws)
        bad[k] = torch.ones(shape, device=cuda)
        with pytest.raises(LavbError):
            encode(enc, pts, [0], [3000], GRID4, bad)
    bad = list(ws)
    bad[3] = ws[3].double()
    with pytest.raises(LavbError):
        encode(enc, pts, [0], [3000], GRID4, bad)
    with pytest.raises(LavbError):
        ops.pillar_decorate(pts, [0, 1000], [1000, 2001], GRID4, 11)
    with pytest.raises(LavbError):
        encode(enc, pts[:, :10], [0], [3000], GRID4, ws)
