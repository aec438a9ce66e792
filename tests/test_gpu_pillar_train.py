"""The training-mode pillar kernels (csrc/pillar.cu: lavb_pillar_decorate, lavb_pillar_scatter_max and its backward) against
plain references, at the shapes a LiDAR training step runs (B = 32 x 40 000 points) and at the edges where they can go wrong:
the half-open window, NaN / inf coordinates, a y that rounds onto the index nx, ragged and empty clouds, strided rows, more
than 2^20 points (the compaction scan carries across its 1024-block chunks), the tie rule of the arg-max and the layout of the
upstream gradient.  The reference helpers below are checked against oracle/lav_ref.pillar_net in test_pillar_train_ref_cpu.py.
"""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from lav_b200 import capi, ops, synth
from lav_b200.capi import LavbError
from lav_b200.point_pillar import PointPillarNet
from oracle import lav_ref as O
from tests import util

pytestmark = pytest.mark.gpu

PPM, D = 4, 11
NX = (util.GRID["max_x"] - util.GRID["min_x"]) * PPM
NY = (util.GRID["max_y"] - util.GRID["min_y"]) * PPM
GRID = (float(util.GRID["min_x"]), float(util.GRID["max_x"]), float(util.GRID["min_y"]), float(util.GRID["max_y"]), float(PPM),
        NX, NY)
EMPTY_ARG = 0x7f7f7f7f                  # arg-max of an empty cell (the kernel's byte-wise 0x7f fill)
U32 = 2.0 ** -24                        # unit roundoff of fp32
MLP_KEYS = ["0.weight", "0.bias", "1.weight", "1.bias", "3.weight", "3.bias", "4.weight", "4.bias"]
GRAD_GATES = {"0.weight": 3e-3, "0.bias": 2e-6, "1.weight": 2e-3, "1.bias": 5e-3, "3.weight": 2e-3, "3.bias": 4e-6,
              "4.weight": 3e-4, "4.bias": 3.5e-3}                # see test_train_mode_module_at_training_size
Y_HI = float(np.nextafter(np.float32(util.GRID["max_y"]), np.float32(0)))    # (y - min_y) * 4 rounds to 320 = nx in fp32


# ----------------------------------------------------------------------------------------------------- reference helpers
def canvas_cells(coords, nx=NX, ny=NY):
    """oracle coords (b, xi, yi) -> canvas cell b*ny*nx + clamp(ny-1-xi)*nx + clamp(yi) (scatter_points, point_pillar.py:87-90).
    A yi that rounded to nx clamps onto col nx-1, so two pillars can share one cell."""
    b, xi, yi = coords.long().unbind(1)
    return (b * ny + (ny - 1 - xi).clamp(0, ny - 1)) * nx + yi.clamp(0, nx - 1)


def smallest_row_argmax(h, cell):
    """Max-pool of the rows h (M, C) >= 0 into their cells, in fp64, over the occupied cells only.
    -> occ (K,) sorted occupied cell ids, canvas (K, C) fp64, arg (K, C) int64, slot (M,) index of each row's cell in occ.
    canvas[k, c] = max(0, max of h[r, c] over the rows r of cell occ[k]); arg[k, c] = the SMALLEST such row with
    h[r, c] == canvas[k, c] (channels whose rows are all 0 included).  Every row of a cell counts, so where two pillars share a
    cell (yi == nx) the cell holds the per-channel max over both: lav_b200's semantics.  The reference's index_put keeps one
    of the two pillars instead, which one being undefined (SURVEY App. C.5)."""
    h = h.detach().double().cpu()
    cell = cell.long().cpu()
    m, c = h.shape
    occ, slot = torch.unique(cell, return_inverse=True)
    idx = slot[:, None].expand(m, c)
    canvas = torch.zeros((len(occ), c), dtype=torch.float64).scatter_reduce(0, idx, h, "amax", include_self=True)
    rows = torch.arange(m)[:, None].expand(m, c)
    cand = torch.where(h == canvas[slot], rows, torch.full_like(rows, EMPTY_ARG))
    arg = torch.full((len(occ), c), EMPTY_ARG, dtype=torch.int64).scatter_reduce(0, idx, cand, "amin", include_self=True)
    return occ, canvas, arg, slot


def mlp64(feat, params):
    """Linear -> BatchNorm1d on batch statistics (biased variance, eps 1e-5) -> ReLU, twice, written out in fp64."""
    x = feat
    for w, b, g, beta in (params[:4], params[4:]):
        x = x @ w.T + b
        mu = x.mean(0)
        var = ((x - mu) ** 2).mean(0)
        x = torch.relu((x - mu) / torch.sqrt(var + 1e-5) * g + beta)
    return x


def routed_grads(feat, params, arg, g):
    """fp64 gradients of the eight point-MLP parameters for loss = sum_{k,c} g[k, c] * h[arg[k, c], c]: the canvas gradient g
    (K, C) of the occupied cells routed to the rows arg (K, C).  -> (grads, h)."""
    p64 = [p.detach().double().cpu().requires_grad_() for p in params]
    h = mlp64(feat.double().cpu(), p64)
    loss = (g.double().cpu() * h.gather(0, arg)).sum()
    return torch.autograd.grad(loss, p64), h.detach()


def centroid_tolerance(points, inv, n_pillars, got, want):
    """Bound on |got - want| of the centroid columns (x - mean of its pillar), where the two sums run in different orders.
    Per pillar of n points and axis: each fp32 sum is within (n-1) u sum|x_i| of the exact one, each division adds u |mean|,
    and each final subtraction rounds by at most half an ulp of its result."""
    xyz = points[:, :3].double()
    n = torch.bincount(inv, minlength=n_pillars).double()[:, None]
    sabs = torch.zeros((n_pillars, 3), dtype=torch.float64).index_add_(0, inv, xyz.abs())
    per_pillar = (2 * (n - 1) * U32 * sabs + 2 * U32 * sabs) / n
    top = np.maximum(np.abs(got.numpy()), np.abs(want.numpy())).astype(np.float32)
    return per_pillar[inv] + torch.from_numpy(np.spacing(top).astype(np.float64))


# ----------------------------------------------------------------------------------------------------- inputs
def _with_time(p, k):
    t = torch.zeros(len(p), 3)
    t[:, k % 3] = 1
    return torch.cat([p, t], 1)


@functools.lru_cache(maxsize=1)
def _training_batch():
    """(32, 40 000, 11): B = 32 clouds of 40 000 painted, time-stamped points, 1.28 M rows > 2^20."""
    return torch.stack([_with_time(synth.painted_sweep(40000, tag=f"ptrain{b}"), b) for b in range(32)])


def _edge_cloud():
    """A stacked cloud with edge rows at its head, in its middle and at its tail."""
    base = synth.stacked_lidar(700, tag="pedge")
    nan, inf = float("nan"), float("inf")
    xy = [(-10.0, -40.0),                                     # x = min_x, y = min_y: kept
          (70.0, 0.0), (0.0, 40.0), (70.0, 40.0),             # x = max_x or y = max_y: dropped
          (nan, 0.0), (0.0, nan), (inf, 0.0), (-inf, 0.0), (0.0, inf), (0.0, -inf),   # dropped
          (20.01, Y_HI), (20.05, Y_HI), (20.2, Y_HI),         # yi rounds to 320: its own pillar, cell clamps onto col 319
          (20.02, 39.9), (20.1, 39.8), (20.15, 39.77),        # yi = 319, same xi: the pillar that shares the cell
          (5.01, 5.01), (5.02, 5.03), (5.1, 5.1)]             # one pillar; the first row gets z = NaN below
    edge = base[:len(xy)].clone()
    edge[:, :2] = torch.tensor(xy)
    edge[len(xy) - 3, 2] = nan
    return torch.cat([edge[:7], base[:1000], edge[7:14], base[1000:], edge[14:]]).contiguous()


def _clouds(name):
    """-> list of (n, 11) clouds for the decorate cases that go through PointPillarNet._as_buffer."""
    g = synth._gen(11, name)
    if name == "one":
        return [synth.stacked_lidar(2000, tag="p1")]
    if name == "ragged3":
        return [synth.stacked_lidar(1000, tag="pr0"), synth.stacked_lidar(17, tag="pr1"), synth.stacked_lidar(600, tag="pr2")]
    if name == "empty_first_middle_last":
        e = torch.zeros((0, 11))
        return [e, synth.stacked_lidar(500, tag="pe0"), e, synth.stacked_lidar(300, tag="pe1"), e]
    if name == "all_outside_cloud":
        out = synth.stacked_lidar(400, tag="po")
        out[:, 0] += 500
        return [synth.stacked_lidar(300, tag="pi0"), out, synth.stacked_lidar(300, tag="pi1")]
    if name == "edges":
        return [_edge_cloud(), synth.stacked_lidar(200, tag="pe2")]
    if name == "batch128":
        base = synth.stacked_lidar(2000, tag="p128")
        counts = torch.randint(0, 120, (128,), generator=g)
        counts[[0, 64, 127]] = 0
        return [base[b * 40:b * 40 + int(counts[b])] for b in range(128)]
    raise KeyError(name)


def _oracle_aux(sd, clouds, counts):
    with torch.no_grad():
        _, aux = O.pillar_net(sd, clouds, counts, ppm=PPM, training=True, return_aux=True, **util.GRID)
    return aux


def _check_decorate(feat, cell, aux):
    """feat / cell of lavb_pillar_decorate against the fp32 oracle's decorated rows."""
    want, coords = aux["decorated"], aux["coords"]
    assert feat.shape == want.shape == (len(want), D + 5)
    feat, cell = feat.cpu(), cell.cpu()
    assert cell.dtype == torch.int32 and torch.equal(cell.long(), canvas_cells(coords))
    exact = list(range(D)) + [D + 3, D + 4]                         # the point, the two cell-origin columns
    assert torch.equal(feat[:, exact].view(torch.int32), want[:, exact].contiguous().view(torch.int32))
    got_c, want_c = feat[:, D:D + 3], want[:, D:D + 3]              # centroid columns: float atomics, order undefined
    nan = torch.isnan(want_c)
    assert torch.equal(torch.isnan(got_c), nan)
    tol = centroid_tolerance(aux["points"], aux["inv"], len(aux["uniq"]), got_c, want_c)
    err = (got_c.double() - want_c.double()).abs()
    assert bool((err[~nan] <= tol[~nan]).all()), float((err - tol)[~nan].max())


# ----------------------------------------------------------------------------------------------------- a. decorate
@pytest.mark.parametrize("case", ["one", "ragged3", "empty_first_middle_last", "all_outside_cloud", "edges", "batch128"])
def test_decorate_matches_fp32_oracle(cuda, case):
    _, sd = util.lidar_model()
    clouds = _clouds(case)
    counts = [len(c) for c in clouds]
    buf, starts, counts = PointPillarNet._as_buffer([c.to(cuda) for c in clouds], counts)
    feat, cell = ops.pillar_decorate(buf, starts, counts, GRID, D)
    aux = _oracle_aux(sd, clouds, counts)
    _check_decorate(feat, cell, aux)
    if case == "edges":                                              # the edge rows are really there
        b, xi, yi = aux["coords"].unbind(1)
        assert int((yi == NX).sum()) == 3 and int(((b == 0) & (xi == 0) & (yi == 0)).sum()) >= 1
        assert int(torch.isnan(feat[:, 2]).sum()) == 1 and int(torch.isnan(feat[:, D + 2]).sum()) >= 3
        assert not bool((feat[:, 0] >= 70).any() or (feat[:, 1] >= 40).any())


@pytest.mark.parametrize("case", ["empty_b1", "all_outside"])
def test_decorate_with_no_kept_point(cuda, case):
    pts = torch.zeros((0, D)) if case == "empty_b1" else synth.stacked_lidar(300, tag="pout") + torch.tensor([0, 200.0] + [0] * 9)
    feat, cell = ops.pillar_decorate(pts.to(cuda), [0], [len(pts)], GRID, D)
    assert feat.shape == (0, D + 5) and cell.shape == (0,)


def test_decorate_padded_tensor_through_module_buffer(cuda):
    """(B, P, 11) input as PointPillarNet takes it: rows past each count are padding that lies INSIDE the window."""
    _, sd = util.lidar_model()
    clouds = [synth.stacked_lidar(900, tag="pp0"), synth.stacked_lidar(500, tag="pp1"), synth.stacked_lidar(40, tag="pp2")]
    counts = [len(c) for c in clouds]
    pad = torch.full((3, max(counts) + 33, D), 3.0)
    for b, c in enumerate(clouds):
        pad[b, :len(c)] = c
    buf, starts, cnt = PointPillarNet._as_buffer(pad.to(cuda), torch.tensor(counts))
    feat, cell = ops.pillar_decorate(buf, starts, cnt, GRID, D)
    _check_decorate(feat, cell, _oracle_aux(sd, clouds, counts))


def test_decorate_strided_rows_with_gaps(cuda):
    """rows of 16 floats (a column-sliced view: pt_stride = 16 > d) and clouds that do not abut in the buffer."""
    _, sd = util.lidar_model()
    clouds = [synth.stacked_lidar(700, tag="ps0"), synth.stacked_lidar(400, tag="ps1")]
    wide = torch.full((len(clouds[0]) + 57 + len(clouds[1]), 16), 1.0)     # gap rows lie in the window
    wide[:len(clouds[0]), :D] = clouds[0]
    wide[len(clouds[0]) + 57:, :D] = clouds[1]
    pts = wide.to(cuda)[:, :D]
    assert pts.stride() == (16, 1)
    feat, cell = ops.pillar_decorate(pts, [0, len(clouds[0]) + 57], [len(c) for c in clouds], GRID, D)
    _check_decorate(feat, cell, _oracle_aux(sd, clouds, [len(c) for c in clouds]))


def test_decorate_at_training_size(cuda):
    """B = 32 x 40 000 = 1.28 M points: more than 2^20, so the compaction's block scan carries across 1024-block chunks."""
    _, sd = util.lidar_model()
    batch = _training_batch()
    counts = [batch.shape[1]] * batch.shape[0]
    buf, starts, cnt = PointPillarNet._as_buffer(batch.to(cuda), counts)
    assert buf.shape[0] > 1 << 20
    feat, cell = ops.pillar_decorate(buf, starts, cnt, GRID, D)
    _check_decorate(feat, cell, _oracle_aux(sd, list(batch), counts))


# ----------------------------------------------------------------------------------------------------- b, c. scatter-max
def _scatter_case(name):
    """-> (h (M, C) fp32 >= 0, cell (M,) int32 in [0, n_cells), n_cells)"""
    g = synth._gen(12, name)
    m, c, n_cells = 200000, 64, 9000
    if name == "dup_rows":                       # rows copied from a small pool: exact ties between whole rows
        pool = torch.relu(torch.randn(1500, c, generator=g))
        h = pool[torch.randint(0, len(pool), (m,), generator=g)]
        h[:, [3, 40]] = 0                        # channels that are 0 in every row
    elif name == "bf16":                         # bf16-rounded values, as the MLP hands them over under autocast
        h = torch.relu(torch.randn(m, c, generator=g)).bfloat16().float()
    elif name == "one_cell":                     # every row lands on one cell: all atomics hit the same 64 addresses
        h = torch.relu(torch.randn(m, c, generator=g)).floor()      # integers: several rows reach each channel's max
        return h, torch.full((m,), 4321, dtype=torch.int32), n_cells
    elif name == "c1" or name == "c3":
        c = int(name[1])
        h = torch.relu(torch.randn(m, c, generator=g)).bfloat16().float()
    elif name == "m0":
        return torch.zeros((0, c)), torch.zeros((0,), dtype=torch.int32), n_cells
    else:
        raise KeyError(name)
    cell = torch.randint(0, 6000, (m,), generator=g, dtype=torch.int32) * 3 // 2     # a third of the cells stays empty
    return h.contiguous(), cell, n_cells


def _check_scatter(h, cell, canvas, arg):
    """canvas / arg of lavb_pillar_scatter_max against the fp64 amax and the smallest-row rule, empty cells included."""
    occ, want, want_arg, _ = smallest_row_argmax(h, cell)
    assert torch.equal(canvas[occ.to(canvas.device)].cpu().view(torch.int32), want.float().view(torch.int32))
    assert torch.equal(arg[occ.to(arg.device)].cpu().long(), want_arg)
    empty = torch.ones(canvas.shape[0], dtype=torch.bool, device=canvas.device)
    empty[occ.to(canvas.device)] = False
    assert bool((canvas[empty].view(torch.int32) == 0).all()) and bool((arg[empty] == EMPTY_ARG).all())
    return occ, want_arg


def _check_routed_backward(gcanvas, arg, cell, gh):
    """gh[r, c] == gcanvas[cell[r], c] where arg[cell[r], c] == r, else 0 (bit for bit); per occupied (cell, channel) the row
    gradients sum to exactly gcanvas."""
    cl = cell.long()
    rows = torch.arange(len(cell), device=cell.device)[:, None]
    want = torch.where(arg[cl].long() == rows, gcanvas[cl], torch.zeros((), device=gh.device))
    assert torch.equal(gh.view(torch.int32), want.contiguous().view(torch.int32))
    summed = torch.zeros(gcanvas.shape, dtype=torch.float64, device=gh.device).index_add_(0, cl, gh.double())
    occ = torch.unique(cl)
    assert torch.equal(summed[occ], gcanvas[occ].double())
    hits = torch.zeros(gcanvas.shape, dtype=torch.int32, device=gh.device).index_add_(0, cl, (gh != 0).int())
    assert int(hits.max()) <= 1


@pytest.mark.parametrize("case", ["dup_rows", "bf16", "one_cell", "c1", "c3", "m0"])
def test_scatter_max_and_backward(cuda, case):
    h, cell, n_cells = _scatter_case(case)
    canvas, arg = ops.pillar_scatter_max(h.to(cuda), cell.to(cuda), n_cells)
    assert canvas.shape == arg.shape == (n_cells, h.shape[1]) and arg.dtype == torch.int32
    occ, want_arg = _check_scatter(h, cell, canvas, arg)
    if case in ("dup_rows", "bf16", "one_cell"):             # the tie rule is really exercised: several rows reach a positive max
        _, can64, _, slot = smallest_row_argmax(h, cell)
        hits = torch.zeros(can64.shape, dtype=torch.int64).index_add_(0, slot, (h.double() == can64[slot]).long())
        assert int(((hits > 1) & (can64 > 0)).sum()) > 10
    gcanvas = torch.randn((n_cells, h.shape[1]), generator=synth._gen(13, case)).to(cuda)
    gh = ops.pillar_scatter_max_bwd(gcanvas, arg, cell.to(cuda), h.shape[0])
    assert gh.shape == h.shape and gh.dtype == torch.float32
    _check_routed_backward(gcanvas, arg, cell.to(cuda), gh)


def test_scatter_max_collision_takes_max_of_both_pillars(cuda):
    """y = nextafter(40, 0) rounds to yi = 320 = nx: decorate gives that pillar the cell of its yi = 319 neighbour, and the
    cell holds, per channel, the max over the rows of both pillars."""
    _, sd = util.lidar_model()
    clouds = _clouds("edges")
    buf, starts, counts = PointPillarNet._as_buffer([c.to(cuda) for c in clouds], [len(c) for c in clouds])
    feat, cell = ops.pillar_decorate(buf, starts, counts, GRID, D)
    aux = _oracle_aux(sd, clouds, counts)
    h = torch.relu(torch.randn((len(feat), 64), generator=synth._gen(14, "coll")))
    canvas, arg = ops.pillar_scatter_max(h.to(cuda), cell, len(clouds) * NY * NX)
    _check_scatter(h, cell.cpu(), canvas, arg)
    b, xi, yi = aux["coords"].unbind(1)
    hi = (b == 0) & (xi == 120) & (yi == NX)
    lo = (b == 0) & (xi == 120) & (yi == NX - 1)
    assert int(hi.sum()) == 3 and int(lo.sum()) >= 3
    target = int(canvas_cells(aux["coords"][hi][:1]))
    assert target == (NY - 1 - 120) * NX + NX - 1 and bool((cell.cpu()[hi | lo] == target).all())
    want = torch.maximum(h[hi].max(0).values, h[lo].max(0).values)
    got = canvas[target].cpu()
    assert torch.equal(got, want)
    assert bool((got != h[hi].max(0).values).any()) and bool((got != h[lo].max(0).values).any())   # both pillars contribute


@pytest.mark.parametrize("layout", ["nchw", "channels_last", "expanded"])
def test_module_backward_for_each_gradient_layout(cuda, layout, monkeypatch):
    """PointPillarNet returns the NHWC canvas as a (B, C, ny, nx) view; whichever layout the consuming convolution hands back,
    _PillarScatterMax.backward routes it to the arg-max rows bit for bit."""
    m, _ = util.lidar_model(cuda)
    pp = m.point_pillar_net.train()
    seen = {}
    real = ops.pillar_scatter_max

    def spy(h, cell, n_cells, want_argmax=True):
        seen["cell"] = cell
        seen["canvas"], seen["arg"] = real(h, cell, n_cells, want_argmax)
        return seen["canvas"], seen["arg"]

    monkeypatch.setattr(ops, "pillar_scatter_max", spy)
    pp.point_net.net.register_forward_hook(lambda mod, inp, out: seen.setdefault("h", out))
    clouds = [c.to(cuda) for c in util.pillar_clouds()]
    out = pp(clouds, [len(c) for c in clouds])
    assert out.shape == (2, 64, NY, NX)
    g = torch.randn(out.shape, generator=synth._gen(15, "layout")).to(cuda)
    if layout == "channels_last":
        g = g.contiguous(memory_format=torch.channels_last)
    elif layout == "expanded":
        g = torch.full((1, 1, 1, 1), 0.5, device=cuda).expand(out.shape)
    (gh,) = torch.autograd.grad(out, seen["h"], g)
    g_nhwc = g.permute(0, 2, 3, 1).reshape(-1, 64)
    _check_routed_backward(g_nhwc, seen["arg"], seen["cell"], gh)
    _check_scatter(seen["h"], seen["cell"].cpu(), seen["canvas"], seen["arg"])


# ----------------------------------------------------------------------------------------------------- d. training size
def test_train_mode_module_at_training_size(cuda, monkeypatch):
    """Train-mode PointPillarNet at B = 32 x 40 000 against an fp64 restatement of its point MLP fed with the GPU's own
    decorated rows (so the rounding of the centroid sums, bounded by the decorate tests, stays out of the comparison).

    Measured on one H100 SXM 80 GB HBM3 (400 W power limit), M = 968 454 kept rows, 444 395 occupied cells: canvas within
    9.4e-7 of fp64 (max-norm relative), max |h32 - h64| 1.0e-5, the arg-max row differs from fp64 at 7-9 of 28.4 M
    (cell, channel) with candidate values at most 7.4e-7 apart.  Point-MLP gradients, 2-norm error over the 2-norm of the fp64
    gradient: 0.weight 5.8e-4, 1.weight 3.8e-4, 1.bias 9.7e-4, 3.weight 3.2e-4, 4.weight 6.1e-5, 4.bias 7.0e-4; the Linear
    biases, whose true gradient is 0, max-norm over that of the weight gradients: 0.bias 1.4-4.3e-7, 3.bias 7.4e-7.  The routing
    itself is exact (checked bit for bit below), so these errors are torch's fp32 Linear / BatchNorm1d backward: sums over ~1e6
    rows of a mixed-sign gradient.  Between runs the max-norm errors of the weights moved by up to 3.4x, so GRAD_GATES leave
    about 5x room."""
    m, _ = util.lidar_model(cuda)
    pp = m.point_pillar_net.train()
    seen = {}
    real_dec, real_sc = ops.pillar_decorate, ops.pillar_scatter_max

    def spy_dec(*a, **k):
        seen["feat"], seen["cell"] = real_dec(*a, **k)
        return seen["feat"], seen["cell"]

    def spy_sc(h, cell, n_cells, want_argmax=True):
        seen["h"] = h
        seen["canvas"], seen["arg"] = real_sc(h, cell, n_cells, want_argmax)
        return seen["canvas"], seen["arg"]

    def keep_grad(mod, inp, out):
        out.register_hook(lambda gr: seen.__setitem__("gh", gr))

    monkeypatch.setattr(ops, "pillar_decorate", spy_dec)
    monkeypatch.setattr(ops, "pillar_scatter_max", spy_sc)
    pp.point_net.net.register_forward_hook(keep_grad)
    batch = _training_batch()
    out = pp(batch.to(cuda), [batch.shape[1]] * batch.shape[0])
    gen = torch.Generator(device=cuda)
    gen.manual_seed(16)
    g = torch.randn(out.shape, generator=gen, device=cuda)
    (out * g).sum().backward()
    params = [dict(pp.point_net.net.named_parameters())[k] for k in MLP_KEYS]

    h32, cell, canvas, arg = seen["h"].detach(), seen["cell"], seen["canvas"], seen["arg"]
    # the kernel's own routing is exact on the h it was given: amax, smallest row, empty cells
    occ, _ = _check_scatter(h32, cell.cpu(), canvas, arg)
    _check_routed_backward(g.permute(0, 2, 3, 1).reshape(-1, 64), arg, cell, seen["gh"])
    occ_d = occ.to(cuda)
    arg_occ = arg[occ_d].long().cpu()
    g_occ = g.permute(0, 2, 3, 1).reshape(-1, 64)[occ_d].cpu()
    grads64, h64 = routed_grads(seen["feat"], params, arg_occ, g_occ)
    # canvas and arg-max against fp64
    occ64, can64, arg64, _ = smallest_row_argmax(h64, cell)
    assert torch.equal(occ64, occ)
    got = canvas[occ_d].cpu().double()
    canvas_err = float((got - can64).abs().max() / can64.abs().max())
    assert torch.equal((got > 0).any(1), (can64 > 0).any(1))
    h_err = float((h32.cpu().double() - h64).abs().max())
    diff = arg_occ != arg64
    gap = (h64.gather(0, arg64) - h64.gather(0, arg_occ)).abs()[diff]
    n_diff = int(diff.sum())
    # gradients of the eight point-MLP parameters
    errs, maxerr = {}, {}
    w_scale = max(float(grads64[0].abs().max()), float(grads64[4].abs().max()))
    for k, p, w in zip(MLP_KEYS, params, grads64):
        d = p.grad.detach().double().cpu() - w
        maxerr[k] = float(d.abs().max() / (w_scale if k in ("0.bias", "3.bias") else w.abs().max()))
        errs[k] = maxerr[k] if k in ("0.bias", "3.bias") else float(d.norm() / w.norm())
    print(f"\ntraining size: M = {len(h32)}, occupied cells {len(occ)}, canvas rel err {canvas_err:.2e}, max |h32 - h64| "
          f"{h_err:.2e}, arg-max differs from fp64 at {n_diff} of {diff.numel()} (cell, channel), max gap {float(gap.max()) if n_diff else 0:.2e}; "
          "grad rel err (2-norm) " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()) +
          "; (max-norm) " + ", ".join(f"{k} {v:.2e}" for k, v in maxerr.items()))
    assert len(h32) > 400000
    assert canvas_err < 1e-5
    assert n_diff <= diff.numel() * 1e-5                              # near-ties of fp32 rounding only, and rare
    if n_diff:
        assert float(gap.max()) <= 2 * h_err
    for k, v in errs.items():
        assert v < GRAD_GATES[k], (k, v)


# ----------------------------------------------------------------------------------------------------- e. autocast
def test_train_mode_module_under_bf16_autocast(cuda, monkeypatch):
    """PointPillarNet in train mode under bf16 autocast, as LAVTrainer(amp=True) runs it: the MLP hands bf16 rows to the
    scatter (cast to fp32 on the way in), ties are common, and the tie rule decides which row gets the gradient."""
    m, _ = util.lidar_model(cuda)
    pp = m.point_pillar_net.train()
    seen = {}
    real = ops.pillar_scatter_max

    def spy(h, cell, n_cells, want_argmax=True):
        seen["cell"] = cell
        seen["canvas"], seen["arg"] = real(h, cell, n_cells, want_argmax)
        return seen["canvas"], seen["arg"]

    def keep(mod, inp, out):
        out.retain_grad()
        seen["h"] = out

    monkeypatch.setattr(ops, "pillar_scatter_max", spy)
    pp.point_net.net.register_forward_hook(keep)
    batch = _training_batch()[:4]
    with torch.autocast("cuda", dtype=torch.bfloat16):
        out = pp(batch.to(cuda), [batch.shape[1]] * 4)
    h, cell, canvas, arg = seen["h"], seen["cell"], seen["canvas"], seen["arg"]
    assert h.dtype == torch.bfloat16 and canvas.dtype == torch.float32
    occ, want_arg = _check_scatter(h.detach().float(), cell.cpu(), canvas, arg)
    _, can64, _, slot = smallest_row_argmax(h.detach().float(), cell)
    ties = torch.zeros(can64.shape, dtype=torch.int64).index_add_(0, slot, (h.detach().cpu().double() == can64[slot]).long())
    assert int(((ties > 1) & (can64 > 0)).sum()) > 100               # positive ties are common under bf16
    g = torch.randn(out.shape, generator=synth._gen(17, "amp")).to(cuda)
    (out.float() * g).sum().backward()
    g_nhwc = g.permute(0, 2, 3, 1).reshape(-1, 64)
    cl = cell.long()
    rows = torch.arange(len(cl), device=cuda)[:, None]
    want = torch.where(arg[cl].long() == rows, g_nhwc[cl], torch.zeros((), device=cuda)).bfloat16()
    assert h.grad.dtype == torch.bfloat16 and torch.equal(h.grad, want)
    hits = torch.zeros((canvas.shape[0], 64), dtype=torch.int32, device=cuda).index_add_(0, cl, (h.grad != 0).int())
    assert bool((hits[occ.to(cuda)] == 1).all())                    # every (cell, channel) reaches exactly one row
    for k, p in pp.point_net.net.named_parameters():
        assert p.grad is not None and bool(torch.isfinite(p.grad).all()), k


# ----------------------------------------------------------------------------------------------------- f. rejection
def _decorate_c(pts, stride, d, starts, counts):
    """raw lavb_pillar_decorate with canary outputs -> (return code, *h_m, feat, cell)"""
    b = len(counts)
    st = (C.c_longlong * b)(*starts)
    ct = (C.c_int * b)(*counts)
    feat = torch.full((max(sum(counts), 1), d + 5), float("nan"), device=pts.device)
    cell = torch.full((max(sum(counts), 1),), -7, dtype=torch.int32, device=pts.device)
    ws = torch.empty(capi.lib().lavb_pillar_workspace_bytes(max(b, 1), NX, NY), dtype=torch.uint8, device=pts.device)
    hm = C.c_int(-5)
    rc = capi.lib().lavb_pillar_decorate(C.c_void_p(pts.data_ptr()), stride, d, st, ct, b, *GRID, C.c_void_p(feat.data_ptr()),
                                         C.c_void_p(cell.data_ptr()), C.byref(hm), C.c_void_p(ws.data_ptr()),
                                         C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return rc, hm.value, feat, cell


@pytest.mark.parametrize("bad", ["batch129", "d10", "stride8"])
def test_decorate_rejects_before_any_launch(cuda, bad):
    pts = synth.stacked_lidar(100, tag="prej").to(cuda)
    args = dict(batch129=(D, D, [0] * 129, [2] * 129), d10=(D, 10, [0], [300]), stride8=(8, D, [0], [300]))[bad]
    rc, hm, feat, cell = _decorate_c(pts, *args)
    assert rc != 0 and hm == -5 and bool(torch.isnan(feat).all()) and bool((cell == -7).all())
    with pytest.raises(LavbError):                                   # and through ops
        if bad == "stride8":
            ops.pillar_decorate(pts.flatten()[:300 * 8 + 3].as_strided((300, D), (8, 1)), [0], [300], GRID, D)
        else:
            ops.pillar_decorate(pts, args[2], args[3], GRID, args[1])


@pytest.mark.parametrize("m,c,n_cells", [(-1, 64, 100), (100, 0, 100), (100, -3, 100), (100, 64, -1)])
def test_scatter_rejects_bad_shapes_before_any_launch(cuda, m, c, n_cells):
    h = torch.ones((100, 64), device=cuda)
    cell = torch.zeros((100,), dtype=torch.int32, device=cuda)
    canvas = torch.full((100, 64), float("nan"), device=cuda)
    arg = torch.full((100, 64), -7, dtype=torch.int32, device=cuda)
    gh = torch.full((100, 64), float("nan"), device=cuda)
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: C.c_void_p(t.data_ptr())                           # noqa: E731
    with pytest.raises(LavbError):
        capi.check(capi.lib().lavb_pillar_scatter_max(p(h), p(cell), m, c, n_cells, p(canvas), p(arg), s), "scatter_max")
    if n_cells >= 0:
        with pytest.raises(LavbError):
            capi.check(capi.lib().lavb_pillar_scatter_max_bwd(p(canvas), p(arg), p(cell), m, c, p(gh), s), "scatter_max_bwd")
    torch.cuda.synchronize()
    assert bool(torch.isnan(canvas).all()) and bool((arg == -7).all()) and bool(torch.isnan(gh).all())


def test_scatter_ops_refuse_bad_dtypes_and_shapes_with_lavb_error(cuda):
    h = torch.ones((50, 64), device=cuda)
    cell = torch.zeros((50,), dtype=torch.int32, device=cuda)
    g = torch.ones((10, 64), device=cuda)
    arg = torch.zeros((10, 64), dtype=torch.int32, device=cuda)
    for hh, cc, n in [(h.bfloat16(), cell, 10), (h.double(), cell, 10), (h, cell.long(), 10), (h, cell[:49], 10),
                      (h, torch.zeros((100,), dtype=torch.int32, device=cuda)[::2], 10), (h[0], cell, 10), (h, cell, -1)]:
        with pytest.raises(LavbError):
            ops.pillar_scatter_max(hh, cc, n)
    for gg, aa, cc in [(g.bfloat16(), arg, cell), (g, arg.long(), cell), (g, arg[:9], cell), (g, arg[:, :63], cell),
                       (g, arg, cell.long()), (g, arg, cell[:49]), (g[0], arg[0], cell)]:
        with pytest.raises(LavbError):
            ops.pillar_scatter_max_bwd(gg, aa, cc, 50)
