"""GPU: lavb_agent_view (lav_b200.view.AgentView) against the numpy statement oracle/view_ref.py bit for bit, on seeded inputs and on
ticks of StaticFramePipeline + AgentController; AgentRecorder against render + annotate; the C ABI's refusals."""
import ctypes as C
import json
import os
import types

import numpy as np
import pytest
import torch

from lav_b200 import capi, ops, synth
from lav_b200.capi import LavbError, lib
from lav_b200.control import AgentController
from lav_b200.view import AgentRecorder, AgentView, annotate, box_table, view_config
from oracle import view_ref as V
from tests import util
from tests.test_gpu_frame import DETS
from tests.test_heads_cpu import uniplanner

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "agent_control.npz")
CFG = json.loads(str(np.load(GOLD)["config"]))          # the reference's config.yaml values (pixels_per_meter, cmd_thresh)
C_BEV, T, M = 4, 20, 6


def inputs(B, P, rows, bev_dtype, seed, cuda):
    """seeded view inputs of B agents: sweeps of up to P rows with NaN padding (bin edges for some agents), NaN plan / cast /
    forecast points, scores at fp32 0.2 and one ulp either side, NaN and > 1, boxes partly off the image, targets past pixel
    255 and NaN, all six commands; rows[i] forecast vehicles for agent i"""
    rng = np.random.default_rng(seed)
    x = dict(rgbs=rng.integers(0, 256, (B, 3, 288, 256, 3), dtype=np.uint8), tels=rng.integers(0, 256, (B, 192, 480, 3), dtype=np.uint8))
    pts = np.full((B, P, 11), np.nan, np.float32)
    edges = np.stack([V.XBINS.astype(np.float32), V.YBINS.astype(np.float32)], 1)
    for b in range(B):
        n = int(rng.integers(P // 3, P + 1))
        pts[b, :n, :4] = rng.uniform([-12, -42, -3, 0], [73, 43, 2, 1], (n, 4))
        pts[b, :n // 4, :2] = rng.normal([15, 0], [1.5, 1.5], (n // 4, 2))
        if b % 3 == 0:
            e = np.concatenate([edges, np.nextafter(edges, np.float32(np.inf)), np.nextafter(edges, -np.float32(np.inf)),
                                np.float32([[71, 41], [np.inf, 0], [0, -np.inf], [np.nan, 3]])])
            pts[b, n - len(e):n, :2] = e
    x["points"] = pts
    logits = rng.normal(0, 3, (B, 320, 320, C_BEV)).astype(np.float32)            # channels-last, as the pipeline holds it
    x["bev"] = torch.from_numpy(logits).to(cuda).to(torch.float32 if bev_dtype == "fp32" else ops.h16()).permute(0, 3, 1, 2)
    x["plan"] = np.cumsum(rng.normal([0, -1.5], [0.4, 0.5], (B, T, 2)), 1).astype(np.float32)
    x["cast"] = np.cumsum(rng.normal([0.3, -1.5], [0.4, 0.5], (B, T, 2)), 1).astype(np.float32)
    x["plan"][1 % B, 3] = np.nan
    x["cast"][B - 1, 5, 1] = np.nan
    x["cmds"] = (np.arange(B) % 6).astype(np.int32)
    locs, scores, boxes = [], [], []
    for b in range(B):
        k = rows[b]
        start = rng.uniform([-30, -60], [30, 10], (k, 1, 1, 2))
        l = (start + np.cumsum(rng.normal(0, 0.8, (k, M, T, 2)), 2)).astype(np.float32)
        s = rng.uniform(0, 1, (k, M)).astype(np.float32)
        if k:
            t = np.float32(0.2)
            s[0, :5] = [np.nextafter(t, np.float32(0)), t, np.nextafter(t, np.float32(1)), np.nan, 1.5]
            l[0, 2, 4] = np.nan
        locs.append(l)
        scores.append(s)
        bx = []
        for _ in range(k):
            a = rng.uniform(0, 2 * np.pi)
            bx.append((float(rng.integers(-20, 340)), float(rng.integers(-20, 340)), float(np.float32(rng.uniform(0.5, 14))),
                       float(np.float32(rng.uniform(0.5, 14))), float(np.float32(np.cos(a))), float(np.float32(np.sin(a)))))
        boxes.append(bx)
    x["locs"], x["scores"], x["boxes"] = locs, scores, boxes
    x["target"] = rng.normal(0, 20, (B, 2)).astype(np.float32)
    x["target"][0] = [45.0, -90.0]
    if B > 2:
        x["target"][2, 1] = np.nan
    return x


def statement(x, b, sig):
    rgb = x["rgbs"][b].transpose(1, 0, 2, 3).reshape(288, 768, 3)
    plan = x["cast"][b] if x["cmds"][b] in (4, 5) else x["plan"][b]
    return V.frame(rgb, x["tels"][b], x["points"][b], sig[b], plan, x["locs"][b], x["scores"][b], x["boxes"][b], x["target"][b],
                   CFG["pixels_per_meter"], CFG["cmd_thresh"])


def device_args(x, cuda):
    B = len(x["locs"])
    offsets = np.zeros(B + 1, np.int32)
    np.cumsum([len(l) for l in x["locs"]], out=offsets[1:])
    table, box_offsets = box_table([[[], bx] for bx in x["boxes"]])
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    locs = np.concatenate(x["locs"]) if offsets[-1] else np.zeros((0, M, T, 2), np.float32)
    scores = np.concatenate(x["scores"]) if offsets[-1] else np.zeros((0, M), np.float32)
    return [d(x["rgbs"]), d(x["tels"]), d(x["points"]), x["bev"], d(x["plan"]), d(x["cast"]), d(x["cmds"]), d(locs), d(scores),
            offsets, table, box_offsets, d(x["target"])]


def compare(got, want, where):
    bad = np.argwhere((got != want).any(-1))
    assert len(bad) == 0, f"{where}: {len(bad)} pixels differ, first {bad[:5].tolist()}"


@pytest.mark.parametrize("B, P, bev_dtype", [(1, 4000, "fp32"), (7, 40000, "h16"), (7, 40000, "fp32"), (64, 120000, "h16")])
def test_kernel_equals_statement(cuda, B, P, bev_dtype):
    rows = [(0, 1, 15)[b % 3] for b in range(B)]
    x = inputs(B, P, rows, bev_dtype, seed=B * 7 + P, cuda=cuda)
    args = device_args(x, cuda)
    cfg = view_config(CFG)
    out = ops.agent_view(*args, cfg)
    sig = torch.sigmoid(x["bev"].float()).cpu().numpy()
    got = out.cpu().numpy()
    for b in range(B):
        compare(got[b], statement(x, b, sig), f"B={B} agent {b} ({rows[b]} vehicles, cmd {x['cmds'][b]})")
    # the same frames from a captured graph, and again after the scratch held another tick
    g = torch.cuda.CUDAGraph()
    scratch = torch.empty((ops.agent_view_scratch_bytes(B),), dtype=torch.uint8, device=cuda)
    again = torch.zeros_like(out)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.agent_view(*args, cfg, scratch=scratch, out=again)
    torch.cuda.current_stream().wait_stream(s)
    with torch.cuda.graph(g):
        ops.agent_view(*args, cfg, scratch=scratch, out=again)
    again.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(again, out)


def _models():
    from lav_b200.heads import RGBBrakePredictionModel
    lm, _ = util.lidar_model()
    sm, _ = util.seg_model()
    up, _ = uniplanner()
    bra = RGBBrakePredictionModel([4, 6, 7, 10]).eval()
    bra.load_state_dict(synth.fill_state_dict_(bra.state_dict()))
    return sm, lm, up, bra


@pytest.mark.parametrize("precision", ["fp32", "f16"])
def test_pipeline_ticks_render_the_statement_and_record(cuda, precision):
    from lav_b200.agent import StaticFramePipeline
    sm, lm, up, bra = _models()
    B, N = 4, 4000
    pipe = StaticFramePipeline(sm, lm, up, bra, B, N, device=cuda, precision=precision)
    ctl, view = AgentController(B, CFG, cuda), AgentView(B, CFG, cuda)
    rec = AgentRecorder(view)
    nxps = torch.tensor([[0.0, -20.0], [3.0, -15.0], [-4.0, -10.0], [50.0, -90.0]])
    rs = np.random.RandomState(5)
    want_rec = []
    for tick in range(3):
        rgbs = torch.stack([synth.rgb_frames(tag=f"av{tick}{b}", smooth=True) for b in range(B)]).to(cuda)
        tels = torch.stack([synth.rgb_frames(tag=f"avt{tick}{b}", smooth=True, n_cam=1, h=192, w=480)[0] for b in range(B)]).to(cuda)
        lidars = [synth.lidar_sweep(N - 100 * b, tag=f"avl{tick}{b}").to(cuda) for b in range(B)]
        cmds = [3, 4, 1, 5] if tick % 2 == 0 else [0, 2, 5, 3]
        out = pipe.step(rgbs, tels, lidars, nxps, cmds, fixed_dets=DETS)
        speeds = rs.uniform(0.0, 11.0, B).astype(np.float32)
        res = ctl.step(out, speeds, cmds)
        frames = view.render(pipe, out).clone()
        recorded = rec.record(pipe, out, res, speeds)
        torch.cuda.synchronize()
        assert torch.equal(recorded, frames)
        # the statement on this tick's copied tensors
        x = dict(rgbs=pipe.rgbs.cpu().numpy(), tels=pipe.tels.cpu().numpy(), points=pipe.stacked.cpu().numpy(),
                 plan=out["ego_plan_locs"].float().cpu().numpy(), cast=out["ego_cast_locs"].float().cpu().numpy(),
                 cmds=pipe.cmds.cpu().numpy(), locs=[o.float().cpu().numpy() for o in out["other_cast_locs"]],
                 scores=[o.float().cpu().numpy() for o in out["other_cast_cmds"]], boxes=[d[1] for d in out["det"]],
                 target=pipe.nxps.cpu().numpy())
        sig = torch.sigmoid(out["pred_bev"].float()).cpu().numpy()
        got = frames.cpu().numpy()
        for b in range(B):
            compare(got[b], statement(x, b, sig), f"{precision} tick {tick} agent {b}")
        want_rec.append(annotate(got.copy(), speeds, cmds, res["control"].cpu().numpy(), out["pred_bra"].float().cpu().numpy()))
    flushed = rec.flush([0, 3])
    assert sorted(flushed) == [0, 3] and rec.pending(0) == 0 and rec.pending(1) == 3
    for b in (0, 3):
        np.testing.assert_array_equal(flushed[b], np.stack([w[b] for w in want_rec]))
    rest = rec.flush()
    np.testing.assert_array_equal(rest[1], np.stack([w[1] for w in want_rec]))
    assert rest[0].shape == (0, 160, 1146, 3)
    rec.close()


def test_malformed_calls_are_refused_with_output_untouched(cuda):
    B = 3
    x = inputs(B, 4000, [1, 0, 2], "fp32", seed=1, cuda=cuda)
    rgbs, tels, pts, bev, plan, cast, cmds, locs, scores, offsets, table, box_offsets, target = device_args(x, cuda)
    cfg = view_config(CFG)
    out = torch.full((B, 160, 1146, 3), 7, dtype=torch.uint8, device=cuda)
    scratch = torch.empty((ops.agent_view_scratch_bytes(B),), dtype=torch.uint8, device=cuda)
    strides = (C.c_longlong * 4)(*bev.stride())
    ip = lambda a: a.ctypes.data_as(C.c_void_p)
    p = lambda t: C.c_void_p(t.data_ptr())
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call(**o):
        a = dict(rgbs=p(rgbs), tels=p(tels), points=p(pts), b=B, p=pts.shape[1], stride=11, bev=p(bev), dtype=capi.F32, c=C_BEV,
                 strides=strides, plan=p(plan), cast=p(cast), cmds=p(cmds), t=T, locs=p(locs), scores=p(scores), k=locs.shape[0],
                 m=M, offsets=ip(offsets), boxes=ip(table), nbox=table.shape[0], box_offsets=ip(box_offsets), target=p(target),
                 cfg=C.byref(cfg), scratch=p(scratch), scratch_bytes=scratch.numel(), out=p(out))
        a.update(o)
        return lib().lavb_agent_view(*a.values(), stream)

    bad_off = offsets.copy(); bad_off[1], bad_off[2] = 2, 1
    far_off = offsets.copy(); far_off[-1] = locs.shape[0] + 1
    far_box = box_offsets.copy(); far_box[-1] = table.shape[0] + 1
    cfg_zero, cfg_nan, cfg_inexact, cfg_thresh = (view_config(dict(CFG, pixels_per_meter=v)) for v in (0.0, float("nan"), 0.1, 4))
    cfg_thresh.cmd_thresh = float("nan")
    refused = dict(neg_b=dict(b=-1), many_b=dict(b=70000), neg_p=dict(p=-1), stride=dict(stride=1), t0=dict(t=0), t_big=dict(t=65),
                   m0=dict(m=0), m9=dict(m=9), neg_k=dict(k=-1), dtype=dict(dtype=7), c0=dict(c=0), c_big=dict(c=65),
                   no_cfg=dict(cfg=None), no_strides=dict(strides=None), no_offsets=dict(offsets=None),
                   no_box_offsets=dict(box_offsets=None), no_boxes=dict(boxes=None),
                   ppm0=dict(cfg=C.byref(cfg_zero)), ppm_nan=dict(cfg=C.byref(cfg_nan)), ppm_inexact=dict(cfg=C.byref(cfg_inexact)),
                   thresh_nan=dict(cfg=C.byref(cfg_thresh)), offsets_order=dict(offsets=ip(bad_off)),
                   offsets_past_k=dict(offsets=ip(far_off)), boxes_past_n=dict(box_offsets=ip(far_box)),
                   neg_stride=dict(strides=(C.c_longlong * 4)(-1, 0, 0, 0)), small_scratch=dict(scratch_bytes=scratch.numel() - 1),
                   null_rgbs=dict(rgbs=None), null_tels=dict(tels=None), null_points=dict(points=None), null_bev=dict(bev=None),
                   null_plan=dict(plan=None), null_cast=dict(cast=None), null_cmds=dict(cmds=None), null_locs=dict(locs=None),
                   null_target=dict(target=None), null_scratch=dict(scratch=None), null_out=dict(out=None),
                   odd_plan=dict(plan=C.c_void_p(plan.data_ptr() + 4)), odd_scratch=dict(scratch=C.c_void_p(scratch.data_ptr() + 4)),
                   odd_points=dict(points=C.c_void_p(pts.data_ptr() + 2)))
    for name, o in refused.items():
        assert call(**o) != 0, name
        assert lib().lavb_last_error(), name
    torch.cuda.synchronize()
    assert bool((out == 7).all()), "a refused call wrote the output"
    assert call() == 0
    torch.cuda.synchronize()
    assert not bool((out == 7).all())
    with pytest.raises(LavbError):
        ops.agent_view(rgbs[:, :2].contiguous(), tels, pts, bev, plan, cast, cmds, locs, scores, offsets, table, box_offsets, target, cfg)
    with pytest.raises(LavbError):
        ops.agent_view(rgbs, tels, pts, bev, plan, cast, cmds.long(), locs, scores, offsets, table, box_offsets, target, cfg)
    with pytest.raises(LavbError):
        ops.agent_view(rgbs, tels, pts, bev, plan, cast, cmds, locs, scores, offsets, table.astype(np.float32), box_offsets, target, cfg)
    with pytest.raises(LavbError):
        AgentView(B + 1, CFG, cuda).render(types.SimpleNamespace(B=B), {})
