"""GPU parity: painting, sweep stacking and the pillar encoder against the oracle, through the C-ABI."""
import numpy as np
import pytest
import torch

from lav_b200 import ops, synth
from oracle import lav_ref as O
from tests import util

pytestmark = pytest.mark.gpu


def _flip_ok(lidar, convs, bad_rows, tol=2e-3):
    """every mismatching point must sit within `tol` px of an integer boundary in some camera (fp32 rounding
    of the projection differs between BLAS orderings); anything else is a bug."""
    for i in bad_rows.tolist():
        near = False
        for K, l2w, w2c in convs:
            p = np.r_[lidar[i, :3].double().numpy(), 1.0]
            cam = w2c @ (l2w @ p)
            cam = np.array([cam[1], -cam[2], cam[0]])
            q = K @ cam
            for val in (q[0] / (1e-5 + q[2]), q[1] / (1e-5 + q[2]), q[2]):
                if abs(val - round(val)) < tol * max(1.0, abs(val) * 1e-3):
                    near = True
        if not near:
            return False
    return True


def test_paint_matches_oracle_and_reference(cuda, golden_dir):
    from lav_b200 import point_painting as PP
    lidar, sem5, gold = util.paint_inputs()
    convs_o = O.default_converters()
    convs = PP.make_converters()
    sem4 = O.suppress_background(sem5)
    got = PP.point_painting(lidar.to(cuda), sem4.to(cuda), convs).cpu()
    want = torch.from_numpy(gold["painted"])              # REFERENCE output (fp32 torch twin)
    bad = (got != want).any(dim=1).nonzero()[:, 0]
    assert len(bad) <= max(2, len(lidar) // 5000), f"{len(bad)} painted rows differ"
    assert _flip_ok(lidar, convs_o, bad)
    # fused background suppression (mode 1) and fused softmax (mode 2)
    fused = PP.forward_paint(lidar.to(cuda), sem5.to(cuda), convs).cpu()
    wantf = torch.from_numpy(gold["fused"])
    badf = (fused != wantf).any(dim=1).nonzero()[:, 0]
    assert set(badf.tolist()) <= set(bad.tolist())
    logits = torch.randn(3, 5, 288, 256, generator=synth._gen(5, "logits"))
    f2 = PP.forward_paint(lidar.to(cuda), logits.to(cuda), convs, logits=True).cpu()
    w2 = O.forward_paint(lidar, torch.softmax(logits, 1), convs_o)
    ok = torch.ones(len(lidar), dtype=torch.bool)
    ok[bad] = False
    assert torch.allclose(f2[ok], w2[ok], rtol=0, atol=2e-6)
    # channels-last semantic maps (what the CUDA ERFNet emits) give the same result
    sem_cl = sem4.to(cuda).permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
    got_cl = PP.point_painting(lidar.to(cuda), sem_cl, convs).cpu()
    assert torch.equal(got_cl, got)


def test_paint_edge_cases(cuda):
    from lav_b200 import point_painting as PP
    convs = PP.make_converters()
    sem = synth.sem_probs(tag="e").to(cuda)[:, 1:]
    empty = PP.point_painting(torch.zeros((0, 4), device=cuda), sem, convs)
    assert empty.shape == (0, 4)
    weird = torch.tensor([[float("nan"), 0, 0, 0], [float("inf"), 0, 0, 0], [1e30, 1e30, 1e30, 0], [-1e30, 0, 0, 0],
                          [1.5, 0, 0, 0]], device=cuda)
    out = PP.point_painting(weird, sem, convs).cpu()
    want = O.point_painting_f32(weird.cpu(), sem.cpu(), O.default_converters())
    assert torch.equal(out, want)


def test_stack_sweep_matches_oracle(cuda):
    from lav_b200 import ops
    import math
    sweeps = [synth.painted_sweep(3000, tag=f"s{i}") for i in range(3)]
    loc, ori = synth.ego_motion(3, tag="stk")
    want = O.stack_lidar(sweeps, loc, ori)
    dst = torch.empty((9000, 11), device=cuda)
    for i, s in enumerate(sweeps):
        d = ori[i] - ori[0]
        R = np.array([[math.cos(d), math.sin(d), 0], [-math.sin(d), math.cos(d), 0], [0, 0, 1]])
        c0, s0 = math.cos(ori[0]), math.sin(ori[0])
        dl = (loc[i] - loc[0]) @ np.array([[c0, -s0], [s0, c0]])
        ops.stack_sweep(s.to(cuda), R, dl[0], dl[1], i, 3, dst[i * 3000:(i + 1) * 3000])
    assert torch.allclose(dst.cpu(), want, rtol=0, atol=1e-5)


@pytest.mark.parametrize("form", ["list", "padded", "single"])
def test_pillar_canvas_matches_oracle(cuda, form):
    m, sd = util.lidar_model(cuda)
    clouds = util.pillar_clouds()
    if form == "single":
        clouds = clouds[:1]
    npts = [len(c) for c in clouds]
    with torch.no_grad():
        want = O.pillar_net(sd, clouds, npts, **util.GRID)
        if form == "padded":
            P = max(npts) + 17
            pad = torch.full((len(clouds), P, 11), 3.0)        # padding rows are in-window on purpose
            for b, c in enumerate(clouds):
                pad[b, :len(c)] = c
            got = m.point_pillar_net(pad.to(cuda), torch.tensor(npts))
        else:
            got = m.point_pillar_net([c.to(cuda) for c in clouds], npts)
    assert got.shape == want.shape
    got = got.cpu()
    assert torch.equal((got != 0).any(1), (want != 0).any(1)), "occupied cells differ"
    assert util.rel_err(got, want) < 1e-5


def test_pillar_matches_reference_golden(cuda, golden_dir):
    import os
    gold = np.load(os.path.join(golden_dir, "lidar_model.npz"))
    m, _ = util.lidar_model(cuda)
    clouds = util.pillar_clouds()
    with torch.no_grad():
        got = m.point_pillar_net([c.to(cuda) for c in clouds], [len(c) for c in clouds]).cpu()
    idx = torch.from_numpy(gold["pillar_idx"]).long()
    vals = got.permute(0, 2, 3, 1)[idx[:, 0], idx[:, 1], idx[:, 2]]
    np.testing.assert_allclose(vals.numpy(), gold["pillar_val"], rtol=1e-4, atol=1e-4)
    assert int((got != 0).any(1).sum()) == len(idx)


@pytest.mark.parametrize("mode", ["uniform", "adversarial", "empty", "all_outside"])
def test_pillar_edge_distributions(cuda, mode):
    m, sd = util.lidar_model(cuda)
    if mode == "empty":
        pts = torch.zeros((0, 11))
    elif mode == "all_outside":
        pts = synth.stacked_lidar(500, tag="o")
        pts[:, 0] += 500
    else:
        xyz = synth.lidar_sweep(6000, tag=mode, mode=mode)
        pts = torch.cat([xyz, torch.rand(6000, 7, generator=synth._gen(3, mode))], 1)
    with torch.no_grad():
        got = m.point_pillar_net([pts.to(cuda)], [len(pts)]).cpu()
        if len(pts) and mode != "all_outside":
            want = O.pillar_net(sd, [pts], [len(pts)], **util.GRID)
            assert util.rel_err(got, want) < 1e-5
        else:
            assert float(got.abs().max()) == 0.0


def test_pillar_full_size_properties(cuda):
    """BASELINE config 2 size (B=32 x 40k points): properties that need no oracle run."""
    m, _ = util.lidar_model(cuda)
    base = torch.cat([synth.painted_sweep(40000, tag="full"), torch.tensor([[1., 0, 0]]).expand(40000, 3)], 1)
    B = 32
    batch = base.to(cuda)[None].repeat(B, 1, 1)
    with torch.no_grad():
        can = m.point_pillar_net(batch, [40000] * B)
        assert can.shape == (B, 64, 320, 320)
        assert torch.equal(can[0], can[B - 1]) or util.rel_err(can[0], can[B - 1]) < 1e-6   # batch items independent
        perm = torch.randperm(40000, generator=synth._gen(1, "perm")).to(cuda)
        can_p = m.point_pillar_net(batch[:1, perm], [40000])
        assert util.rel_err(can_p[0], can[0]) < 1e-5                                        # point order irrelevant
        assert float(can.min()) >= 0.0


@pytest.mark.parametrize("out", ["fp32", "h16"])
@pytest.mark.parametrize("mode", ["carla", "uniform", "adversarial", "batch", "empty"])
def test_pillar_tensor_core_encoders_match_oracle(cuda, mode, out):
    """the tensor-core encoder of the 16-bit pipeline (cell-sorted + mma.sync) in both canvas formats (fp32, h16): same
    occupancy as the oracle, values within 1e-3 (layer 1 runs on hi/lo-split operands ~ fp32, layer 2 on h16 operands with
    fp32 accumulation; the h16 canvas adds one 2^-12 rounding)."""
    m, sd = util.lidar_model(cuda)
    m.set_precision("f16")
    if mode == "batch":
        clouds = util.pillar_clouds()
    elif mode == "empty":
        clouds = [torch.zeros((0, 11))]
    elif mode == "carla":
        clouds = [synth.stacked_lidar(20000, tag="sorted")]
    else:
        xyz = synth.lidar_sweep(9000, tag=mode, mode=mode)
        clouds = [torch.cat([xyz, torch.rand(9000, 7, generator=synth._gen(3, mode))], 1)]
    npts = [len(c) for c in clouds]
    with torch.no_grad():
        got = m.point_pillar_net.forward_nhwc([c.to(cuda) for c in clouds], npts, canvas16=(out == "h16")).float().cpu()
    if mode == "empty":
        assert float(got.abs().max()) == 0.0
        return
    with torch.no_grad():
        want = O.pillar_net(sd, clouds, npts, **util.GRID).permute(0, 2, 3, 1)
    assert got.shape == want.shape
    assert torch.equal((got != 0).any(-1), (want != 0).any(-1)), "occupied cells differ"
    assert util.rel_err(got, want) < 1e-3
    rms = float(((got - want) ** 2).mean().sqrt() / (want ** 2).mean().sqrt())
    assert rms < 3e-3, rms


def _roof_sweep(n, tag):
    """a sweep with a good share of points inside / on the faces of the ego-roof box (x in (-2.4,0), y in (-.8,.8), z in (-1.5,-1))."""
    g = synth._gen(9, tag)
    pts = synth.lidar_sweep(n, tag=tag)
    k = n // 4
    box = torch.stack([torch.rand(k, generator=g) * 3.0 - 2.7, torch.rand(k, generator=g) * 2.0 - 1.0,
                       torch.rand(k, generator=g) * 0.8 - 1.65, torch.rand(k, generator=g)], 1)
    pts[torch.randperm(n, generator=g)[:k]] = box
    edges = torch.tensor([[-2.4, 0.0, -1.2, 1.0], [0.0, 0.0, -1.2, 1.0], [-1.0, -0.8, -1.2, 1.0], [-1.0, 0.8, -1.2, 1.0],
                          [-1.0, 0.0, -1.5, 1.0], [-1.0, 0.0, -1.0, 1.0], [-1.0, 0.0, -1.25, 1.0], [float("nan"), 0.0, -1.25, 1.0]])
    pts[:len(edges)] = edges                    # faces are OUTSIDE (strict inequalities); NaN fails the test -> kept
    return pts.contiguous()


def test_roof_filter_is_an_order_preserving_drop(cuda):
    """a5: LAVAgent.preprocess (lav_agent.py:448-457) = np.delete of the rows inside the roof box.  lavb_roof_filter must give
    the oracle's rows in the oracle's order (bit-equal), for one sweep, for a batch of ragged NaN-padded sweeps, and for sweeps
    longer than one 1024-row chunk with nothing / everything dropped."""
    for n, tag in ((5000, "rf0"), (1024, "rf1"), (7, "rf2"), (40000, "rf3")):
        pts = _roof_sweep(max(n, 8), tag)[:n] if n >= 8 else _roof_sweep(8, tag)[:n]
        want = O.preprocess(pts)
        got, cnt = ops.roof_filter(pts.to(cuda))
        assert int(cnt[0]) == len(want)
        assert torch.equal(torch.nan_to_num(got[:len(want)].cpu(), nan=-7.0), torch.nan_to_num(want, nan=-7.0))
    inside = torch.tensor([[-1.0, 0.0, -1.2, 0.5]]).repeat(3000, 1)
    got, cnt = ops.roof_filter(inside.to(cuda), pad_nan=True)
    assert int(cnt[0]) == 0 and bool(torch.isnan(got).all())
    # batch of fixed-shape sweeps, padded with NaN rows (StaticFramePipeline layout): counts per frame, NaN tail
    B, N = 3, 6000
    batch = torch.full((B, N, 4), float("nan"))
    lens = [6000, 4097, 1]
    for b in range(B):
        batch[b, :lens[b]] = _roof_sweep(6000, f"rfb{b}")[:lens[b]]
    got, cnt = ops.roof_filter(batch.to(cuda), pad_nan=True)
    got = got.cpu()
    for b in range(B):
        want = O.preprocess(batch[b, :lens[b]])
        k = len(want)
        assert torch.equal(torch.nan_to_num(got[b, :k], nan=-7.0), torch.nan_to_num(want, nan=-7.0))
        assert bool(torch.isnan(got[b, k:]).all())
        assert int(cnt[b]) == k + (N - lens[b])              # NaN padding rows of the input are "kept" (they stay NaN rows)


def test_roof_filter_inside_stacking_matches_drop(cuda):
    """the fused form (roof_filter flag of lavb_stack_sweep: dropped rows are marked x = NaN in place) gives the same canvas as
    dropping first: every downstream kernel skips NaN rows."""
    m, _ = util.lidar_model(cuda)
    src = torch.cat([_roof_sweep(6000, "rfs"), torch.rand(6000, 4, generator=synth._gen(2, "rfs"))], 1).contiguous()
    R = np.eye(3, dtype=np.float32)
    marked = torch.empty((6000, 11), device=cuda)
    ops.stack_sweep(src.to(cuda), R, 0.0, 0.0, 0, 3, marked, roof_filter=True)
    keep = O.preprocess(src)
    assert int(torch.isnan(marked[:, 0]).sum()) == len(src) - len(keep) + 1          # + the NaN probe row of _roof_sweep
    dropped = torch.empty((len(keep), 11), device=cuda)
    ops.stack_sweep(keep.to(cuda).contiguous(), R, 0.0, 0.0, 0, 3, dropped)
    with torch.no_grad():
        a = m.point_pillar_net([marked], [len(marked)])
        b = m.point_pillar_net([dropped], [len(dropped)])
    assert util.rel_err(a, b) < 1e-6


@pytest.mark.parametrize("precision", ["fp32", "f16"])
def test_paint_from_decoder_features_matches_logit_path(cuda, precision):
    """lavb_paint_deconv_batched (output_conv + softmax + suppression evaluated inside the gather, erfnet.py:122-124,132 +
    model_inference.py:44-50) == materialised logits -> lavb_paint_batched mode 2, same features.  Geometry must be identical."""
    from lav_b200 import point_painting as PP
    m, _ = util.seg_model(cuda)
    m.set_precision(precision)
    F_, N = 2, 6000
    rgb = torch.cat([synth.rgb_frames(tag=f"pd{f}", smooth=True) for f in range(F_)]).to(cuda)       # (F*3,288,256,3) u8
    pts = torch.stack([synth.lidar_sweep(N, tag=f"pd{f}") for f in range(F_)]).to(cuda).contiguous()
    cams = np.stack([c.packed() for c in PP.make_converters()])
    with torch.no_grad():
        feat, table, ncls = m.forward_features_nhwc(rgb)
        assert feat.shape == (F_ * 3, 144, 128, 16) and ncls == 5
        logits = m.forward_nhwc(rgb)
    logits = logits.view(F_, 3, 288, 256, 5).permute(0, 1, 4, 2, 3)
    want = ops.paint_batched(pts, logits, cams, 2, 4, torch.empty((F_, N, 8), device=cuda))
    got = ops.paint_deconv_batched(pts, feat, ncls, table, cams, 4, torch.empty((F_, N, 8), device=cuda), (288, 256))
    assert torch.equal(got[..., :4], want[..., :4])
    assert torch.equal((got[..., 4:] != 0).any(-1), (want[..., 4:] != 0).any(-1))            # same hit / miss per point
    # fp32: accumulation order only.  f16: the materialised path multiplies h16-rounded output_conv weights (mma.sync), the fused
    # path fp32 weights — both see the same h16 features
    assert float((got[..., 4:] - want[..., 4:]).abs().max()) < (1e-5 if precision == "fp32" else 5e-3)
