"""GPU: lavb_agent_control (lav_b200.control.AgentController) against the numpy statement oracle/control_ref.ControlTail over long
seeded sequences, its argument checks, reset, and AgentController.step on the outputs of both frame pipelines."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from lav_b200 import ops, synth
from lav_b200.capi import LavbError, lib
from lav_b200.control import AgentController, control_config
from oracle.control_ref import ControlTail, control_sequence
from tests import util
from tests.test_gpu_frame import DETS
from tests.test_heads_cpu import uniplanner

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "agent_control.npz")
CFG = json.loads(str(np.load(GOLD)["config"]))          # the reference's config.yaml values


def device_out(x, cuda):
    """a pipeline-shaped output dict of one tick of control_sequence, on the device: each agent's forecast rows are views of one
    (K, C, T, 2) tensor, as the pipelines return them"""
    counts = [len(o) for o in x["other_locs"]]
    locs = torch.from_numpy(np.concatenate(x["other_locs"])).to(cuda)
    cmds = torch.from_numpy(np.concatenate(x["other_cmds"])).to(cuda)
    return dict(ego_plan_locs=torch.from_numpy(x["plan"]).to(cuda), ego_cast_locs=torch.from_numpy(x["cast"]).to(cuda),
                other_cast_locs=torch.split(locs, counts), other_cast_cmds=torch.split(cmds, counts),
                pred_bra=torch.from_numpy(x["pred_bra"]).to(cuda))


def check_tick(tail, want, ctl, got, where):
    flags, control = got["flags"].cpu().numpy(), got["control"].cpu().numpy()
    np.testing.assert_array_equal(flags, want["flags"], err_msg=where)
    np.testing.assert_array_equal(control[:, 1:], want["control"][:, 1:].astype(np.float32), err_msg=where)
    assert np.abs(control[:, 0].astype(np.float64) - want["control"][:, 0].astype(np.float32)).max() <= 1e-12, where
    s = ctl.state_views()
    np.testing.assert_array_equal(s["stop"], tail.stop, err_msg=where)
    np.testing.assert_array_equal(s["creep"], tail.force, err_msg=where)
    np.testing.assert_array_equal(s["speed"], tail.speed, err_msg=where)
    assert np.abs(s["turn"] - tail.turn).max() <= 1e-12, where


@pytest.mark.parametrize("B, T, n", [(1, 20, 40), (7, 10, 7), (64, 20, 40), (64, 10, 7), (300, 10, 7), (300, 20, 40)])
def test_kernel_equals_statement(cuda, B, T, n):
    cfg = dict(CFG, turn_n=n, speed_n=n, aim_point=[min(a, T - 1) for a in CFG["aim_point"]])
    tail, ctl = ControlTail(B, cfg), AgentController(B, cfg, cuda)
    stopped, halts = ((2,), (3,)) if B > 3 else ((B - 1,), ())
    for tick, x in enumerate(control_sequence(100 + B + T + n, B, 700, T=T, stopped=stopped, halts=halts)):
        want = tail.step(**x)
        got = ctl.step(device_out(x, cuda), x["speed"], x["cmd"])
        check_tick(tail, want, ctl, got, f"B {B} T {T} n {n} tick {tick}")


def test_reset_touches_only_the_named_agents(cuda):
    B = 6
    tail, ctl = ControlTail(B, CFG), AgentController(B, CFG, cuda)
    for x in control_sequence(5, B, 30, stopped=(1, 4)):
        tail.step(**x)
        ctl.step(device_out(x, cuda), x["speed"], x["cmd"])
    before = ctl.state.view(B, -1).cpu().clone()
    assert before.any(dim=1).all()
    ctl.reset([1, 4])
    tail.reset([1, 4])
    after = ctl.state.view(B, -1).cpu()
    assert not after[[1, 4]].any()
    keep = [0, 2, 3, 5]
    assert torch.equal(after[keep], before[keep])
    for tick, x in enumerate(control_sequence(6, B, 20, stopped=(1,))):     # and the reset agents start a new route
        want = tail.step(**x)
        check_tick(tail, want, ctl, ctl.step(device_out(x, cuda), x["speed"], x["cmd"]), f"after reset, tick {tick}")
    ctl.reset()
    assert not ctl.state.any()


def _call(args, **over):
    a = dict(args, **over)
    return lib().lavb_agent_control(*[a[k] for k in ("plan", "cast", "b", "t", "c", "locs", "cmds", "k", "offsets", "bra", "speed",
                                                      "cmd", "cfg", "state", "control", "flags")], None)


def test_rejects_malformed_arguments(cuda):
    B, T, Cn, K = 3, 20, 6, 5
    cfg = control_config(CFG)
    x = next(control_sequence(9, B, 1, T=T))
    plan = torch.from_numpy(x["plan"]).to(cuda)
    locs = torch.randn(K, Cn, T, 2, device=cuda)
    scores = torch.rand(K, Cn, device=cuda)
    bra, speed = torch.zeros(B, device=cuda), torch.ones(B, device=cuda)
    state = torch.full((B * ops.agent_control_state_bytes(cfg.turn_n, cfg.speed_n),), 7, dtype=torch.uint8, device=cuda)
    control = torch.full((B, 3), -5.0, device=cuda)
    flags = torch.full((B,), -5, dtype=torch.int32, device=cuda)
    offsets = np.array([0, 2, 2, 5], np.int32)
    cmd = np.array([0, 4, 5], np.int32)
    p = lambda t: C.c_void_p(t.data_ptr())
    keep = []                                     # the host arrays behind the pointers stay alive for the calls
    ip = lambda a: (keep.append(a), a.ctypes.data_as(C.c_void_p))[1]
    args = dict(plan=p(plan), cast=p(plan), b=B, t=T, c=Cn, locs=p(locs), cmds=p(scores), k=K, offsets=ip(offsets), bra=p(bra),
                speed=p(speed), cmd=ip(cmd), cfg=C.byref(cfg), state=p(state), control=p(control), flags=p(flags))

    def cfg_with(**kw):
        c = control_config(CFG)
        for k, v in kw.items():
            if k == "aim0":
                c.aim_point[0] = v
            else:
                setattr(c, k, v)
        return C.byref(c)

    bad = [dict(t=33), dict(t=1), dict(c=9), dict(c=0), dict(b=-1), dict(k=-1),
           dict(offsets=ip(np.array([0, 3, 2, 5], np.int32))), dict(offsets=ip(np.array([0, 2, 2, 6], np.int32))),
           dict(offsets=ip(np.array([-1, 2, 2, 5], np.int32))), dict(offsets=None),
           dict(cmd=ip(np.array([0, 6, 1], np.int32))), dict(cmd=ip(np.array([0, -1, 1], np.int32))), dict(cmd=None),
           dict(cfg=None), dict(cfg=cfg_with(turn_n=65)), dict(cfg=cfg_with(speed_n=0)), dict(cfg=cfg_with(aim0=T)),
           dict(cfg=cfg_with(aim0=-1)), dict(cfg=cfg_with(pixels_per_meter=0.0)),
           dict(plan=None), dict(cast=None), dict(locs=None), dict(cmds=None), dict(bra=None), dict(speed=None), dict(state=None),
           dict(control=None), dict(flags=None), dict(plan=C.c_void_p(plan.data_ptr() + 4))]
    for over in bad:
        assert _call(args, **over) != 0, over
    torch.cuda.synchronize()
    assert (control == -5.0).all() and (flags == -5).all() and (state == 7).all()
    assert _call(args, b=0, offsets=ip(np.zeros(1, np.int32))) == 0                 # no agent: nothing to do
    assert _call(args, locs=None, cmds=None, k=0, offsets=ip(np.zeros(B + 1, np.int32))) == 0   # no forecast rows at all
    torch.cuda.synchronize()
    assert (flags != -5).all()
    with pytest.raises(LavbError):
        ops.agent_control(plan, plan, locs, scores, offsets, bra, speed, cmd.astype(np.int64), cfg, state)
    with pytest.raises(LavbError):
        ops.agent_control(plan, plan, locs, scores, offsets, bra, speed, cmd, cfg, state[1:])
    with pytest.raises(LavbError):
        ops.agent_control(plan, plan[:, :10].contiguous(), locs, scores, offsets, bra, speed, cmd, cfg, state)
    with pytest.raises(KeyError):
        AgentController(B, {k: v for k, v in CFG.items() if k != "clip_delta"}, cuda)


def _models():
    from lav_b200.heads import RGBBrakePredictionModel
    lm, _ = util.lidar_model()
    sm, _ = util.seg_model()
    up, _ = uniplanner()
    bra = RGBBrakePredictionModel([4, 6, 7, 10]).eval()
    bra.load_state_dict(synth.fill_state_dict_(bra.state_dict()))
    return sm, lm, up, bra


def _host_copy(out, B):
    return dict(plan=out["ego_plan_locs"].cpu().numpy(), cast=out["ego_cast_locs"].cpu().numpy(),
                other_locs=[o.cpu().numpy() for o in out["other_cast_locs"]], other_cmds=[o.cpu().numpy() for o in out["other_cast_cmds"]],
                pred_bra=out["pred_bra"].float().cpu().numpy().reshape(B))


def _snapshot(out):
    keys = ("ego_plan_locs", "ego_cast_locs", "pred_bra")
    return {k: out[k].clone() for k in keys}, [o.clone() for o in out["other_cast_locs"]], [o.clone() for o in out["other_cast_cmds"]]


@pytest.mark.parametrize("kind", ["static", "dynamic"])
def test_controller_on_pipeline_outputs(cuda, kind):
    from lav_b200.agent import FramePipeline, StaticFramePipeline, SweepHistory
    sm, lm, up, bra = _models()
    B, N = 4, 4000
    if kind == "static":
        pipe = StaticFramePipeline(sm, lm, up, bra, B, N, device=cuda, precision="fp32")
    else:
        pipe = FramePipeline(sm, lm, up, bra, device=cuda, precision="fp32")
        hist = [SweepHistory() for _ in range(B)]
        orig = pipe.infer_model.decode_packed
        pipe.infer_model.decode_packed = lambda *a, **k: [[d[0], list(DETS)] for d in orig(*a, **k)]
    tail, ctl = ControlTail(B, CFG), AgentController(B, CFG, cuda)
    nxps = torch.tensor([[0.0, -20.0], [3.0, -15.0], [-4.0, -10.0], [1.0, -30.0]])
    rs = np.random.RandomState(11)
    for tick in range(3):
        rgbs = torch.stack([synth.rgb_frames(tag=f"ac{tick}{b}", smooth=True) for b in range(B)]).to(cuda)
        tels = torch.stack([synth.rgb_frames(tag=f"act{tick}{b}", smooth=True, n_cam=1, h=192, w=480)[0] for b in range(B)]).to(cuda)
        lidars = [synth.lidar_sweep(N - 100 * b, tag=f"acl{tick}{b}").to(cuda) for b in range(B)]
        cmds = [3, 4, 1, 5] if tick % 2 == 0 else [0, 2, 5, 3]
        if kind == "static":
            out = pipe.step(rgbs, tels, lidars, nxps, cmds, fixed_dets=DETS)
        else:
            out = pipe.step(rgbs, tels, lidars, hist, nxps.to(cuda), cmds)
        assert sum(len(o) for o in out["other_cast_locs"]) > 0
        speeds = rs.uniform(0.0, 11.0, B).astype(np.float32)
        before = _snapshot(out)
        got = ctl.step(out, speeds, cmds)
        torch.cuda.synchronize()
        after = _snapshot(out)
        assert all(torch.equal(before[0][k], after[0][k]) for k in before[0])
        assert all(torch.equal(a, b) for a, b in zip(before[1] + before[2], after[1] + after[2]))
        want = tail.step(**_host_copy(out, B), speed=speeds, cmd=cmds)
        check_tick(tail, want, ctl, got, f"{kind} tick {tick}")
