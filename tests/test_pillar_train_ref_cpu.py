"""The reference helpers of test_gpu_pillar_train.py (cell mapping, smallest-row arg-max, fp64 point MLP, gathered gradient
routing) against oracle/lav_ref.pillar_net on small clouds, on the CPU."""
import torch

from lav_b200 import synth
from oracle import lav_ref as O
from tests import util
from tests.test_gpu_pillar_train import (MLP_KEYS, NX, NY, PPM, _edge_cloud, canvas_cells, mlp64, routed_grads,
                                         smallest_row_argmax)


def _oracle(clouds):
    _, sd = util.lidar_model()
    with torch.no_grad():
        canvas, aux = O.pillar_net(sd, clouds, [len(c) for c in clouds], ppm=PPM, training=True, return_aux=True, **util.GRID)
    return sd, canvas.permute(0, 2, 3, 1).reshape(-1, canvas.shape[1]), aux


def test_cells_and_smallest_row_argmax_rebuild_the_oracle_canvas():
    """canvas[occ] = h[arg] rebuilds the oracle's canvas, cell for cell, except where a yi == nx pillar shares the cell of its
    neighbour: there the helper takes the per-channel max over both pillars; the reference's index_put keeps, per channel,
    one of the two."""
    edge = _edge_cloud()
    edge[torch.isnan(edge[:, 2]), 2] = 0.5                  # a NaN z would make every batch statistic NaN
    clouds = [torch.cat([edge, edge[:300]]), synth.stacked_lidar(300, tag="rc1")]     # repeated rows: exact ties
    _, want, aux = _oracle(clouds)
    h = aux["point_feats"]
    cell = canvas_cells(aux["coords"])
    occ, can64, arg, slot = smallest_row_argmax(h, cell)
    rows = torch.arange(len(h))[:, None]
    hit = h.double() == can64[slot]
    assert bool((hit <= (rows >= arg[slot])).all())          # no smaller row of the cell reaches the max
    assert int(((hit.long().new_zeros(can64.shape).index_add_(0, slot, hit.long()) > 1) & (can64 > 0)).sum()) > 0
    rebuilt = torch.zeros_like(want)
    rebuilt[occ] = h.gather(0, arg)
    assert torch.equal(rebuilt[occ].double(), can64)
    pcell = canvas_cells(aux["uniq"])
    coll = (torch.bincount(pcell, minlength=len(want)) > 1).nonzero()[:, 0]
    assert coll.tolist() == [(NY - 1 - 120) * NX + NX - 1]    # the one yi == 320 pillar of the edge cloud
    rest = torch.ones(len(want), dtype=torch.bool)
    rest[coll] = False
    assert torch.equal(rebuilt[rest], want[rest])
    fmax = O.scatter_max(h, aux["inv"], len(aux["uniq"]))
    pills = (pcell == coll[0]).nonzero()[:, 0]
    assert len(pills) == 2
    assert torch.equal(rebuilt[coll[0]], fmax[pills].max(0).values)
    assert bool(((want[coll[0]] == fmax[pills[0]]) | (want[coll[0]] == fmax[pills[1]])).all())   # the reference: either, per channel


def test_routed_gradients_equal_autograd_through_amax():
    """With no ties, routing the canvas gradient through the arg-max rows (h[arg] gathered) is the gradient of the fp64
    scatter_reduce('amax'); mlp64 restates the oracle's fp32 point MLP."""
    clouds = [synth.stacked_lidar(800, tag="rg0"), synth.stacked_lidar(500, tag="rg1")]
    sd, _, aux = _oracle(clouds)
    feat = aux["decorated"].double()
    params = [sd["point_pillar_net.point_net.net." + k] for k in MLP_KEYS]
    h64 = mlp64(feat, [p.double() for p in params])
    assert float((h64 - aux["point_feats"].double()).abs().max()) < 1e-5 * float(h64.abs().max())
    cell = canvas_cells(aux["coords"])
    occ, can64, arg, slot = smallest_row_argmax(h64, cell)
    hits = torch.zeros(can64.shape, dtype=torch.int64).index_add_(0, slot, (h64 == can64[slot]).long())
    assert bool((hits[can64 > 0] == 1).all())                # no ties among the positive maxima
    g = torch.randn(can64.shape, generator=synth._gen(18, "route"), dtype=torch.float64)
    got, _ = routed_grads(feat, params, arg, g)
    p64 = [p.double().requires_grad_() for p in params]
    h = mlp64(feat, p64)
    pooled = torch.zeros(can64.shape, dtype=torch.float64).scatter_reduce(0, slot[:, None].expand_as(h), h, "amax",
                                                                          include_self=True)
    want = torch.autograd.grad((g * pooled).sum(), p64)
    scale = max(float(w.abs().max()) for w in want)
    for k, a, b in zip(MLP_KEYS, got, want):
        assert torch.allclose(a, b, rtol=1e-10, atol=1e-12 * scale), k
