"""GPU parity of the frame-level pieces: crop kernel, InferModel, FramePipeline (BASELINE config 1 analogue)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from lav_b200 import ops, synth
from oracle import lav_ref as O
from tests import util
from tests.test_heads_cpu import uniplanner

pytestmark = pytest.mark.gpu

DETS = [(150.0, 200.0, 8.0, 4.0, 0.9, 0.3), (170.0, 240.0, 8.0, 4.0, -0.2, 0.95), (161.0, 281.0, 8., 4., 1., 0.)]


@pytest.mark.parametrize("dtype", ["fp32", "h16"])
def test_crop_kernel_vs_grid_sample(cuda, dtype):
    dtype = torch.float32 if dtype == "fp32" else ops.h16()
    from lav_b200.heads import crop_theta
    g = synth._gen(4, "crop")
    feats = torch.randn(3, 64, 40, 48, generator=g)
    locs = torch.tensor([[0., 0.], [3., -5.], [-8., 2.], [30., 30.], [1., 1.]])
    oris = torch.tensor([0., 0.4, -2.0, 1.0, 3.1])
    fidx = torch.tensor([0, 1, 2, 1, 0], dtype=torch.int32)
    theta = crop_theta(locs, oris, 40, 48, 2.0, 24, torch.tensor(0.), torch.tensor(0.75))
    grids = F.affine_grid(theta, torch.Size((5, 64, 24, 24)), align_corners=True)
    want = F.grid_sample(feats[fidx.long()], grids, align_corners=True)
    x = feats.permute(0, 2, 3, 1).contiguous().to(cuda).to(dtype)
    got = ops.crop_bilinear(x, fidx.to(cuda), theta.to(cuda), 24).float().cpu().permute(0, 3, 1, 2)
    assert util.rel_err(got, want) < (1e-5 if dtype == torch.float32 else 1e-2)


@pytest.mark.parametrize("case", ["c64", "c400_many"])
def test_crop_backward_kernel_vs_grid_sample_grad(cuda, case):
    """ops.CropBilinear (gather backward, no atomics) against autograd through F.grid_sample on the CPU: windows that leave the
    map, several crops per frame, > 32 crops on one frame (second pass of the per-block crop list), channel counts below
    one warp pass (64) and above one channel pass (400)."""
    from lav_b200.heads import crop_theta
    g = synth._gen(5, "cropbwd" + case)
    C, K = (64, 7) if case == "c64" else (400, 41)
    B, H, W, S = 3, 40, 48, 24
    feats = torch.randn(B, C, H, W, generator=g)
    locs = torch.randn(K, 2, generator=g) * 8
    oris = torch.rand(K, generator=g) * 6.28 - 3.14
    fidx = torch.randint(0, B, (K,), generator=g).to(torch.int32) if case == "c64" else torch.cat([torch.zeros(36, dtype=torch.int32), torch.tensor([1, 2, 1, 2, 2], dtype=torch.int32)])
    theta = crop_theta(locs, oris, H, W, 2.0, S, torch.tensor(0.), torch.tensor(0.75))
    gout = torch.randn(K, C, S, S, generator=g)
    f_cpu = feats.clone().requires_grad_(True)
    grids = F.affine_grid(theta, torch.Size((K, C, S, S)), align_corners=True)
    want_out = F.grid_sample(f_cpu[fidx.long()], grids, align_corners=True)
    want_out.backward(gout)
    f_gpu = feats.to(cuda).requires_grad_(True)
    got_out = ops.CropBilinear.apply(f_gpu.permute(0, 2, 3, 1).contiguous(), fidx.to(cuda), theta.to(cuda), S).permute(0, 3, 1, 2)
    got_out.backward(gout.to(cuda))
    assert util.rel_err(got_out.detach().cpu(), want_out.detach()) < 1e-5
    assert util.rel_err(f_gpu.grad.cpu(), f_cpu.grad) < 1e-5
    # the training forward of UniPlanner.crop_feature takes this path and agrees with its grid_sample fallback
    import lav_b200.heads as Hd
    up, _ = uniplanner()
    up = up.to(cuda)
    f2 = feats[:, :64].to(cuda).requires_grad_(True)
    rel_locs, rel_oris = (torch.randn(5, 2, generator=g) * 3).to(cuda), (torch.rand(5, generator=g) - 0.5).to(cuda)
    fr = torch.tensor([0, 2, 1, 1, 0], device=cuda)
    outs = []
    for flag in (True, False):
        Hd.TRAIN_CROP_KERNEL = flag
        try:
            f2.grad = None
            o = up.crop_feature(f2, rel_locs, rel_oris, pixels_per_meter=2, crop_size=S, frame_idx=fr)
            o.square().sum().backward()
            outs.append((o.detach().clone(), f2.grad.clone()))
        finally:
            Hd.TRAIN_CROP_KERNEL = True
    assert util.rel_err(outs[0][0], outs[1][0]) < 1e-5 and util.rel_err(outs[0][1], outs[1][1]) < 1e-5


@pytest.mark.parametrize("n", [1, 37, 128])
def test_cast_kernel_matches_gru_modules(cuda, n):
    """lavb_cast_gru (6 branches x GRU(512,64) + Linear + cumsum in one launch) == the nn.GRU / nn.Linear module path of
    UniPlanner.cast and BEVPlanner.cast (uniplanner.py:286-301), fp32, 1e-5 of the waypoint scale; the packed weights follow
    parameter updates."""
    import lav_b200.heads as Hd
    up, _ = uniplanner()
    up = up.to(cuda).eval()
    g = synth._gen(6, f"cast{n}")
    embd = (torch.randn(n, 512, generator=g) * 0.7).to(cuda)
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            for planner in (up, up.bev_planner):
                got = planner.cast(embd)
                Hd.CAST_KERNEL = False
                try:
                    want = planner.cast(embd)
                finally:
                    Hd.CAST_KERNEL = True
                assert got.shape == want.shape == (n, planner.num_cmds, planner.num_plan, 2)
                assert util.rel_err(got, want) < 1e-5, util.rel_err(got, want)
            up.cast_mlps_ego[2].bias.add_(1.0)                        # in-place update -> the pack must be rebuilt
            got, Hd.CAST_KERNEL = up.cast(embd), False
            try:
                want = up.cast(embd)
            finally:
                Hd.CAST_KERNEL = True
            assert util.rel_err(got, want) < 1e-5
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32


def test_infer_model_matches_oracle(cuda):
    from lav_b200.model_inference import InferModel
    lm, lsd = util.lidar_model(cuda)
    up, usd = uniplanner()
    im = InferModel(lm, up, 1.5, 2.4, cuda)
    pts = synth.stacked_lidar(3000, tag="im")
    nxp = torch.tensor([0.0, -20.0])
    with torch.no_grad():
        f, center, box, ori, seg = O.lidar_model(lsd, [pts], [len(pts)], **util.GRID)
        want_det = O.det_inference(torch.sigmoid(center[0]), box[0], ori[0])
        got = im(pts.to(cuda), nxp.to(cuda), 2)
    assert [[d[:2] for d in c] for c in got[6]] == [[d[:2] for d in c] for c in want_det]
    assert util.rel_err(got[5], seg) < 1e-3
    with torch.no_grad():
        w = O.uniplanner_infer(usd, f[0], want_det[1], 2, nxp)
    sc = float(w[1].abs().max()) + 1
    assert float((got[1].cpu() - w[1]).abs().max()) < 1e-3 * sc        # ego_plan_locs
    assert float((got[2].cpu() - w[2]).abs().max()) < 1e-3 * sc        # ego_cast_locs
    # planner with a fixed detection list (vehicle branch), on CUDA features
    with torch.no_grad():
        feats = lm([pts.to(cuda)], [len(pts)])[0][0]
        ee, epl, ecl, ocl, occ = im.uniplanner_infer(feats, DETS, 2, nxp.to(cuda))
        w = O.uniplanner_infer(usd, f[0], DETS, 2, nxp)
    sc = float(w[3].abs().max()) + 1
    assert ocl.shape == w[3].shape == (2, 6, 20, 2)                     # third det is within 4 px of the ego: skipped
    assert float((epl.cpu() - w[1]).abs().max()) < 1e-3 * sc
    assert float((ocl.cpu() - w[3]).abs().max()) < 1e-3 * sc
    assert float((occ.cpu() - w[4]).abs().max()) < 1e-3


def _pipeline(cuda, precision):
    from lav_b200.agent import FramePipeline
    from lav_b200.heads import RGBBrakePredictionModel
    lm, lsd = util.lidar_model()
    sm, ssd = util.seg_model()
    up, usd = uniplanner()
    bra = RGBBrakePredictionModel([4, 6, 7, 10]).eval()
    bsd = synth.fill_state_dict_(bra.state_dict())
    bra.load_state_dict(bsd)
    return FramePipeline(sm, lm, up, bra, device=cuda, precision=precision), (ssd, lsd, usd, {k: v.clone() for k, v in bsd.items()})


def _oracle_frame(sds, rgb_u8, tel_u8, lidar, prev, loc, ori, dets):
    ssd, lsd, usd, bsd = sds
    with torch.no_grad():
        sem = torch.softmax(O.erfnet(ssd, rgb_u8.permute(0, 3, 1, 2).float()), 1)
        fused = O.forward_paint(lidar, sem, O.default_converters())
        stacked = O.stack_lidar([fused] + prev, loc, ori)
        f, center, box, orim, seg = O.lidar_model(lsd, [stacked], [len(stacked)], **util.GRID)
        det = O.det_inference(torch.sigmoid(center[0]), box[0], orim[0])
        plan = O.uniplanner_infer(usd, f[0], dets if dets is not None else det[1], 3, torch.tensor([0.0, -20.0]))
        wide = rgb_u8.permute(1, 0, 2, 3).reshape(288, 768, 3).permute(2, 0, 1)[None].float()
        bra = O.brake_model(bsd, wide, tel_u8.permute(2, 0, 1)[None].float())
    return dict(fused=fused, stacked=stacked, seg=seg, det=det, plan=plan, bra=bra, features=f)


def test_frame_pipeline_fp32_matches_oracle(cuda):
    """BASELINE config 1: one synthetic frame (3xRGB 288x256 + LiDAR sweep) -> waypoints / brake, tol 1e-3."""
    from lav_b200.agent import SweepHistory
    pipe, sds = _pipeline(cuda, "fp32")
    B = 2
    rgbs = torch.stack([synth.rgb_frames(tag=f"f{b}", smooth=True) for b in range(B)])
    tels = torch.stack([synth.rgb_frames(tag=f"t{b}", smooth=True, n_cam=1, h=192, w=480)[0] for b in range(B)])
    lidars = [synth.lidar_sweep(6000 + 500 * b, tag=f"fl{b}") for b in range(B)]
    prev = [[synth.painted_sweep(5000, tag=f"fp{b}{i}") for i in range(2)] for b in range(B)]
    poses = [synth.ego_motion(3, tag=f"fe{b}") for b in range(B)]
    hist = []
    for b in range(B):
        h = SweepHistory()
        loc, ori = poses[b]
        for t in range(10):       # slot t-5 -> prev[0], slot t-10 -> prev[1]
            k = 0 if t >= 5 else 1
            h.push(prev[b][k].to(cuda), loc[1 + k], ori[1 + k])
        hist.append(h)
    out = pipe.step(rgbs.to(cuda), tels.to(cuda), [l.to(cuda) for l in lidars], hist, torch.tensor([[0.0, -20.0]] * B).to(cuda), [3] * B,
                    poses=[(poses[b][0][0], poses[b][1][0]) for b in range(B)])
    for b in range(B):
        want = _oracle_frame(sds, rgbs[b], tels[b], lidars[b], prev[b], poses[b][0], poses[b][1], None)
        got_fused = hist[b].lidars[-1].cpu()
        bad = (got_fused != want["fused"]).any(1)
        # painting follows the CUDA ERFNet's softmax: compare painted probabilities numerically, geometry exactly
        assert torch.equal(got_fused[:, :4], want["fused"][:, :4])
        assert float((got_fused[:, 4:] - want["fused"][:, 4:]).abs().max()) < 2e-3 or int(bad.sum()) < 10
        assert util.rel_err(out["pred_bev"][b], want["seg"][0]) < 2e-3
        assert [[d[:2] for d in c] for c in out["det"][b]] == [[d[:2] for d in c] for c in want["det"]]
        sc = float(want["plan"][1].abs().max()) + 1
        assert float((out["ego_plan_locs"][b].cpu() - want["plan"][1]).abs().max()) < 1e-3 * sc
        assert abs(float(out["pred_bra"][b]) - float(want["bra"][0])) < 1e-3


def test_frame_pipeline_f16_close_to_oracle(cuda):
    from lav_b200.agent import SweepHistory
    pipe, sds = _pipeline(cuda, "f16")
    rgbs = synth.rgb_frames(tag="g0", smooth=True)[None]
    tels = synth.rgb_frames(tag="gt", smooth=True, n_cam=1, h=192, w=480)
    lidar = synth.lidar_sweep(8000, tag="gl")
    prev = [synth.painted_sweep(6000, tag=f"gp{i}") for i in range(2)]
    loc, ori = synth.ego_motion(3, tag="ge")
    h = SweepHistory()
    for t in range(10):
        k = 0 if t >= 5 else 1
        h.push(prev[k].to(cuda), loc[1 + k], ori[1 + k])
    out = pipe.step(rgbs.to(cuda), tels.to(cuda), [lidar.to(cuda)], [h], torch.tensor([[0.0, -20.0]]).to(cuda), [3], poses=[(loc[0], ori[0])])
    want = _oracle_frame(sds, rgbs[0], tels[0], lidar, prev, loc, ori, None)
    f_got, f_want = out["features"][0].float().cpu().permute(2, 0, 1), want["features"][0]
    rms = float(((f_got - f_want) ** 2).mean().sqrt() / (f_want ** 2).mean().sqrt())
    assert rms < 1e-2, rms                                   # ERFNet(f16) -> paint -> 17 f16 conv layers: north_star 1e-2
    assert util.rel_err(f_got, f_want) < 1e-2
    sc = float(want["plan"][1].abs().max()) + 1
    assert float((out["ego_plan_locs"][0].float().cpu() - want["plan"][1]).abs().max()) < 1e-2 * sc
    assert abs(float(out["pred_bra"][0]) - float(want["bra"][0])) < 1e-2


@pytest.mark.parametrize("graphs", [False, True])
def test_static_pipeline_matches_dynamic(cuda, graphs):
    """The fixed-shape / CUDA-graph pipeline (batched paint, table-driven stack, ring-buffer FIFO) must reproduce the
    dynamic FramePipeline tick by tick, including ticks where older sweeps do not exist yet."""
    from lav_b200.agent import FramePipeline, SweepHistory, StaticFramePipeline
    from lav_b200.heads import RGBBrakePredictionModel
    lm, _ = util.lidar_model()
    sm, _ = util.seg_model()
    up, _ = uniplanner()
    bra = RGBBrakePredictionModel([4, 6, 7, 10]).eval()
    bra.load_state_dict(synth.fill_state_dict_(bra.state_dict()))
    dyn = FramePipeline(sm, lm, up, bra, device=cuda, precision="fp32")
    B, N = 2, 5000
    st = StaticFramePipeline(sm, lm, up, bra, B, N, device=cuda, precision="fp32", use_graphs=graphs)
    hist = [SweepHistory() for _ in range(B)]
    nxps = torch.tensor([[0.0, -20.0], [3.0, -15.0]])
    for tick in range(12):
        rgbs = torch.stack([synth.rgb_frames(tag=f"s{tick}{b}", smooth=True) for b in range(B)])
        tels = torch.stack([synth.rgb_frames(tag=f"st{tick}{b}", smooth=True, n_cam=1, h=192, w=480)[0] for b in range(B)])
        lidars = [synth.lidar_sweep(N - 100 * b, tag=f"sl{tick}{b}") for b in range(B)]       # agent 1 has a shorter sweep
        poses = [(np.array([0.3 * tick, 0.1 * b]), 0.02 * tick) for b in range(B)]
        heavy = tick in (0, 4, 5, 10, 11)     # compare on the ticks where the set of stacked sweeps changes
        o_s = st.step(rgbs.to(cuda), tels.to(cuda), [l.to(cuda) for l in lidars], nxps, [3, 1], poses=poses, fixed_dets=DETS)
        if not heavy:
            for b in range(B):   # keep the dynamic FIFO in step without running its networks
                hist[b].push(st.cur[b, :lidars[b].shape[0]].clone(), poses[b][0], poses[b][1])
            continue
        im = dyn.infer_model
        orig = im.decode_packed
        im.decode_packed = lambda *a, **k: [[d[0], list(DETS)] for d in orig(*a, **k)]
        o_d = dyn.step(rgbs.to(cuda), tels.to(cuda), [l.to(cuda) for l in lidars], hist, nxps.to(cuda), [3, 1], poses=poses)
        im.decode_packed = orig
        for b in range(B):
            n = lidars[b].shape[0]
            assert torch.equal(st.cur[b, :n].cpu(), hist[b].lidars[-1].cpu()), tick
            assert util.rel_err(o_s["pred_bev"][b], o_d["pred_bev"][b]) < 1e-4, tick
            sc = float(o_d["ego_plan_locs"][b].abs().max()) + 1
            assert float((o_s["ego_plan_locs"][b] - o_d["ego_plan_locs"][b]).abs().max()) < 1e-3 * sc, tick
            assert float((o_s["other_cast_locs"][b] - o_d["other_cast_locs"][b]).abs().max()) < 1e-3 * sc, tick
            assert abs(float(o_s["pred_bra"][b]) - float(o_d["pred_bra"][b])) < 1e-4
            assert [d[:2] for d in o_s["det"][b][0]] == [d[:2] for d in o_d["det"][b][0]]     # class 1 was overridden with DETS


@pytest.mark.parametrize("kind", ["blobs", "noise", "flat"])
def test_det_peaks_kernel_matches_reference_decode(cuda, kind):
    """CUDA decode (sigmoid + 7x7 NMS + top-15 + map reads) vs the torch restatement of extract_peak / det_inference."""
    from lav_b200.model_inference import InferModel
    g = synth._gen(17, kind)
    B = 3
    if kind == "blobs":
        yy, xx = torch.meshgrid(torch.arange(320.), torch.arange(320.), indexing="ij")
        logit = torch.full((B, 2, 320, 320), -6.0)
        for b in range(B):
            for k in range(25):
                cx, cy = (torch.rand(2, generator=g) * 320).tolist()
                amp = 3.0 + float(torch.rand(1, generator=g)) * 8
                logit[b, k % 2] = torch.maximum(logit[b, k % 2], -6 + amp * torch.exp(-((xx - cx) ** 2 + (yy - cy) ** 2) / 8.0))
    elif kind == "noise":
        logit = torch.randn(B, 2, 320, 320, generator=g) * 1.5 - 4.0
    else:
        logit = torch.full((B, 2, 320, 320), -9.0)          # nothing above the threshold
    size = torch.rand(B, 2, 320, 320, generator=g) * 3
    ori = torch.randn(B, 2, 320, 320, generator=g)
    stub = type("S", (), {"pixels_per_meter": 4})()
    want = InferModel.decode_packed(stub, InferModel.pack_peaks(torch.sigmoid(logit), size, ori))
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous().to(cuda)
    got = InferModel.decode_packed(stub, ops.det_peaks(nhwc(logit), nhwc(size), nhwc(ori)))
    for b in range(B):
        for c in range(2):
            assert sorted(got[b][c]) == sorted(want[b][c]), (kind, b, c)
            if kind == "blobs":
                assert got[b][c] == want[b][c]            # distinct scores: same (descending) order as torch.topk


def test_brake_real_weights_match_reference_golden(cuda, golden_dir):
    """a19 with the RELEASED weights (weights/bra_v2_9.pt, staged by oracle/pin_against_reference.py): the CUDA paths — fp32
    forward, and the 16-bit forward_u8 path with the lav_b200 stem / pool kernels — against the reference module's own output
    (tests/golden/brake.npz["real"]) on the same frames."""
    import os
    from lav_b200.heads import RGBBrakePredictionModel
    path = os.path.join(util.ROOT, "oracle", "_ref", "bra_v2_9.state_dict.pt")
    gold = np.load(os.path.join(golden_dir, "brake.npz"))
    if not os.path.exists(path) or "real" not in gold:
        pytest.skip("oracle/_ref/bra_v2_9.state_dict.pt not staged")
    sd = torch.load(path, map_location="cpu")
    n_lab = sd["seg_head.upconv.9.weight"].shape[0]
    m = RGBBrakePredictionModel(list(range(n_lab - 1))).eval()
    m.load_state_dict(sd, strict=True)
    wide_u8 = synth.rgb_frames(smooth=True, tag="wide", n_cam=1, h=288, w=768)         # (1,288,768,3) — the pin script's frames
    tel_u8 = synth.rgb_frames(smooth=True, tag="tele", n_cam=1, h=192, w=480)
    m = m.to(cuda)
    with torch.no_grad():
        got32 = m(wide_u8.permute(0, 3, 1, 2).float().to(cuda), tel_u8.permute(0, 3, 1, 2).float().to(cuda)).float().cpu()
    np.testing.assert_allclose(got32.numpy(), gold["real"], atol=1e-4)
    # 16-bit product path: the three 256-wide cameras side by side ARE the 768-wide image
    rgbs = wide_u8.view(1, 288, 3, 256, 3).permute(0, 2, 1, 3, 4).contiguous()
    m.conv_backbone.to(ops.h16()).to(memory_format=torch.channels_last)
    m.attn1.to(ops.h16()); m.attn2.to(ops.h16())
    with torch.no_grad():
        got16 = m.forward_u8(rgbs.to(cuda), tel_u8.to(cuda)).float().cpu()
    assert abs(float(got16[0]) - float(gold["real"][0])) < 1e-2, (got16, gold["real"])


def test_resnet18_folded_weights_follow_the_parameters(cuda):
    """The BN-folded eval weights are a cache: an optimizer step, a parent's load_state_dict or train()/eval() must never leave
    a stale fold behind (the reference's per-step pattern: eval() -> infer under no_grad -> train(), lav_final_v2.py:228-236)."""
    up, usd = uniplanner()
    up = up.to(cuda)
    emb = up.lidar_conv_emb
    x = torch.randn(2, 384, 96, 96, generator=torch.Generator().manual_seed(3)).to(cuda)
    with torch.no_grad():
        a = emb(x).clone()
    opt = torch.optim.SGD(emb.parameters(), lr=0.5)
    emb.train()
    emb(x).sum().backward()
    opt.step()
    emb.eval()
    with torch.no_grad():
        b = emb(x).clone()
        want = emb[0].maxpool(emb[0].relu(emb[0].bn1(emb[0].conv1(x))))
        want = emb[1:](emb[0].layer4(emb[0].layer3(emb[0].layer2(emb[0].layer1(want)))))
    assert not torch.allclose(a, b), "fold cache survived an optimizer step"
    assert util.rel_err(b, want) < 1e-3
    up.load_state_dict({k: v.to(cuda) for k, v in usd.items()})              # PARENT load: nn.Module recursion never calls the child's
    with torch.no_grad():
        c = emb(x)
    assert util.rel_err(c, a) < 1e-5, "fold cache survived a parent load_state_dict"
