"""GPU parity at the BASELINE.json configuration SIZES (SURVEY.md §8d "Config 1/2/3").

The small-cloud tests elsewhere pin the arithmetic; these pin the multi-tile / persistent / binary-search paths at the sizes
bench.py runs: 40 k-point sweeps, 120 k stacked points, B = 32 (fp32) and B = 64 (16-bit tensor-core path).  The oracle
(oracle/lav_ref.py, CPU fp32) checks EVERY frame where it is cheap (painting) and sampled frames of the batch where it is not.
"""
import numpy as np
import pytest
import torch

from lav_b200 import ops, synth
from oracle import lav_ref as O
from tests import util
from tests.test_heads_cpu import uniplanner

pytestmark = pytest.mark.gpu

N_SWEEP = 40000        # BASELINE.json: "40k LiDAR pts"


def _rms(a, b):
    return float(((a - b) ** 2).mean().sqrt() / (b ** 2).mean().sqrt())


def test_config1_full_size_frame_fp32(cuda):
    """Config 1: one frame — 3 x RGB 288x256 + a 40 000-point sweep, stacked with two 40 000-point history sweeps (120 000 x 11)
    — through the fp32 frame pipeline vs the oracle of the reference modules: waypoints (20,2) and brake, tol 1e-3."""
    from lav_b200.agent import SweepHistory
    from tests.test_gpu_frame import _oracle_frame, _pipeline
    pipe, sds = _pipeline(cuda, "fp32")
    rgbs = synth.rgb_frames(tag="c1", smooth=True)[None]
    tels = synth.rgb_frames(tag="c1t", smooth=True, n_cam=1, h=192, w=480)
    lidar = synth.lidar_sweep(N_SWEEP, tag="c1l")
    prev = [synth.painted_sweep(N_SWEEP, tag=f"c1p{i}") for i in range(2)]
    loc, ori = synth.ego_motion(3, tag="c1e")
    h = SweepHistory()
    for t in range(10):
        k = 0 if t >= 5 else 1
        h.push(prev[k].to(cuda), loc[1 + k], ori[1 + k])
    out = pipe.step(rgbs.to(cuda), tels.to(cuda), [lidar.to(cuda)], [h], torch.tensor([[0.0, -20.0]]).to(cuda), [3], poses=[(loc[0], ori[0])])
    want = _oracle_frame(sds, rgbs[0], tels[0], lidar, prev, loc, ori, None)
    assert want["stacked"].shape == (3 * N_SWEEP, 11)
    got_fused = h.lidars[-1].cpu()
    assert torch.equal(got_fused[:, :4], want["fused"][:, :4])
    bad = (got_fused != want["fused"]).any(1)
    assert float((got_fused[:, 4:] - want["fused"][:, 4:]).abs().max()) < 2e-3 or int(bad.sum()) < 40
    f_got = out["features"][0].float().cpu().permute(2, 0, 1)
    assert util.rel_err(f_got, want["features"][0]) < 1e-3
    assert util.rel_err(out["pred_bev"][0], want["seg"][0]) < 1e-3
    assert [[d[:2] for d in c] for c in out["det"][0]] == [[d[:2] for d in c] for c in want["det"]]
    sc = float(want["plan"][1].abs().max()) + 1
    assert float((out["ego_plan_locs"][0].cpu() - want["plan"][1]).abs().max()) < 1e-3 * sc
    assert float((out["ego_cast_locs"][0].cpu() - want["plan"][2]).abs().max()) < 1e-3 * sc
    assert abs(float(out["pred_bra"][0]) - float(want["bra"][0])) < 1e-3


def _config2_inputs(B):
    lidars = torch.stack([synth.lidar_sweep(N_SWEEP, tag=f"c2l{b}") for b in range(B)])            # (B,40000,4)
    sems = torch.stack([synth.sem_probs(tag=f"c2s{b % 4}") for b in range(B)])                    # (B,3,5,288,256) softmaxed
    return lidars, sems


@pytest.mark.parametrize("precision", ["fp32", "f16"])
def test_config2_paint_and_voxelise_b32(cuda, precision):
    """Config 2: point painting + PointPillars voxeliser forward, B = 32 x 40 000 points (time one-hot [1,0,0], D = 11).
    Painted features must be index-equal to the oracle on every frame; the canvas within 1e-3 on sampled frames, with
    identical occupancy.  fp32 = the exact kernel; f16 = the tensor-core encoder the benchmark runs, with its h16 canvas
    (same 1e-3 gate for both)."""
    from lav_b200 import point_painting as PP
    B = 32
    lidars, sems = _config2_inputs(B)
    convs, convs_o = PP.make_converters(), O.default_converters()
    cams = np.stack([c.packed() for c in convs])
    fused = torch.empty((B, N_SWEEP, 8), device=cuda)
    ops.paint_batched(lidars.to(cuda).contiguous(), sems.to(cuda), cams, 1, 4, fused)
    got_fused = fused.cpu()
    n_bad = 0
    for b in range(B):
        want = O.forward_paint(lidars[b], sems[b], convs_o)
        assert torch.equal(got_fused[b, :, :4], want[:, :4])
        n_bad += int((got_fused[b] != want).any(1).sum())
    assert n_bad <= B * N_SWEEP // 5000, f"{n_bad} painted rows differ over the batch"           # pixel-boundary flips only
    pts = torch.cat([fused, torch.tensor([1.0, 0.0, 0.0], device=cuda).expand(B, N_SWEEP, 3)], 2).contiguous()
    m, sd = util.lidar_model(cuda)
    m.set_precision(precision)
    with torch.no_grad():
        canvas = m.point_pillar_net.forward_nhwc(pts, [N_SWEEP] * B, canvas16=(precision != "fp32")).float()
    assert canvas.shape == (B, 320, 320, 64)
    for b in (0, 13, 31):
        with torch.no_grad():
            want = O.pillar_net(sd, [pts[b].cpu()], [N_SWEEP], **util.GRID)[0].permute(1, 2, 0)
        got = canvas[b].cpu()
        assert torch.equal((got != 0).any(-1), (want != 0).any(-1)), f"frame {b}: occupied cells differ"
        assert util.rel_err(got, want) < 1e-3, (b, util.rel_err(got, want))


def test_config3_backbone_heads_planner_b64_f16(cuda):
    """Config 3: B = 64 frames of 120 000 stacked points through the 16-bit tensor-core path — pillar encoder (h16 canvas),
    BEV backbone, the four heads and UniPlanner (cuDNN's plan GRU) with K = 3 fixed vehicles per frame — vs the fp32 oracle on
    sampled frames of the batch: north_star tolerance 1e-2 (max-norm and rms of every output)."""
    B, K = 64, 3
    dets = [(150.0, 200.0, 8.0, 4.0, 0.9, 0.3), (170.0, 240.0, 8.0, 4.0, -0.2, 0.95), (120.0, 150.0, 8., 4., 1., 0.)]
    clouds = [synth.stacked_lidar(N_SWEEP, tag=f"c3{b % 8}") for b in range(8)]
    batch = torch.stack([clouds[b % 8] for b in range(B)]).to(cuda)                                  # (64,120000,11)
    # make the frames of a group differ (not only 8 distinct inputs): a per-frame shift of the intensity column
    batch[:, :, 3] += torch.arange(B, device=cuda).view(B, 1) * 1e-3
    m, lsd = util.lidar_model(cuda)
    m.set_precision("f16")
    up, usd = uniplanner()
    up = up.to(cuda)
    up.lidar_conv_emb.to(ops.h16()).to(memory_format=torch.channels_last)
    H = W = 320
    locs, oris, fidx = [], [], []
    for b in range(B):
        l, o = up.det_to_locs(dets, H, W)
        locs += l; oris += o; fidx += [b] * len(l)
    assert len(locs) == B * K
    all_locs = torch.cat([torch.tensor(locs), torch.zeros(B, 2)]).to(cuda)
    all_oris = torch.cat([torch.tensor(oris), torch.zeros(B)]).to(cuda)
    all_fidx = torch.cat([torch.tensor(fidx), torch.arange(B)]).to(torch.int32).to(cuda)
    nxps = torch.tensor([[0.0, -20.0]] * B, device=cuda)
    cmds = torch.full((B,), 3, dtype=torch.long, device=cuda)
    with torch.no_grad():
        feats, center, box, ori, seg = m.forward_nhwc(batch, [3 * N_SWEEP] * B)
        ee, epl, ecl, ocl, occ = up.infer_device(feats.permute(0, 3, 1, 2), all_locs, all_oris, all_fidx, B * K, nxps, cmds)
    worst = {}
    for b in (0, 37, 63):
        pts = batch[b].cpu()
        with torch.no_grad():
            wf, wc, wb, wo, ws = O.lidar_model(lsd, [pts], [len(pts)], **util.GRID)
            wplan = O.uniplanner_infer(usd, wf[0], dets, 3, torch.tensor([0.0, -20.0]))
        for name, got, want in (("features", feats[b], wf[0]), ("center", center[b], wc[0]), ("box", box[b], wb[0]),
                                ("ori", ori[b], wo[0]), ("seg", seg[b], ws[0])):
            g = got.float().cpu().permute(2, 0, 1)
            e, r = util.rel_err(g, want), _rms(g, want)
            if name == "seg":          # sigmoid output: max-norm on the logits over the logit scale (util.seg_logit_err)
                e = util.seg_logit_err(g[None], wf, lsd)
            worst[name] = max(worst.get(name, 0.0), e, r)
            assert e < 1e-2 and r < 1e-2, (b, name, e, r)
        # planner: embedding, cast and the other vehicles' forecasts against the oracle directly; the 5 x 20-step plan roll-out is a
        # NON-contractive recurrent map on seeded weights (a 1e-3 embedding difference grows to 1e-1 of the waypoint scale over
        # 100 GRU steps), so the roll-out is checked as an operator: our plan vs the oracle's roll-out fed OUR embedding and cast
        rel = lambda a, w: float((a.float().cpu() - w).abs().max()) / (float(w.abs().max()) + 1)
        e_embd, e_cast = rel(ee[b], wplan[0][0]), rel(ecl[b], wplan[2])
        e_other = rel(ocl[b * K:(b + 1) * K], wplan[3])
        with torch.no_grad():
            own_cast = O.up_cast(usd, ee[b:b + 1].float().cpu())
            own_plan = O.up_plan(usd, ee[b:b + 1].float().cpu(), torch.tensor([[0.0, -20.0]]), own_cast, 4, 192)[0, -1, 3]
        e_plan = rel(epl[b], own_plan)
        worst["plan"] = max(worst.get("plan", 0.0), e_embd, e_cast, e_other, e_plan)
        assert max(e_embd, e_cast, e_other, e_plan) < 1e-2, (b, e_embd, e_cast, e_other, e_plan)
    print("config 3 worst errors:", {k: f"{v:.2e}" for k, v in worst.items()})
