"""GPU: lavb_agent_nav_front / lavb_agent_nav_update (lav_b200.navigation.AgentNavigator) against the numpy statement
oracle/nav_ref.AgentNavRef over 1000-tick sequences, set_routes' isolation, lavb_stack_job_poses against
StaticFramePipeline._fill_jobs and the stacked sweeps of both pose paths, AgentController.step with device commands, and the
argument checks."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from lav_b200 import ops, synth
from lav_b200.agent import GAP, StaticFramePipeline
from lav_b200.capi import LavbError, lib
from lav_b200.control import FLAG_BAD_CMD, AgentController
from lav_b200.navigation import FLAG_NO_ROUTE, AgentNavigator
from oracle import nav_ref as N
from oracle.nav_ref import nav_drive
from oracle.control_ref import control_sequence
from tests import util
from tests.test_gpu_agent_control import device_out
from tests.test_gpu_frame import DETS
from tests.test_heads_cpu import uniplanner

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CFG = json.loads(str(np.load(os.path.join(GOLD, "agent_control.npz"))["config"]))
# fp64 state against the statement.  Only CUDA's cos / sin / tan / atan differ from the host's, by an ulp or two, but kbm_step's
# tan(theta) has its pole at a compass of pi: there the predicted heading theta_p grows large, and the update theta_p + K (z -
# theta_p) with K = 1 - 3e-11 cancels it back to the compass, so theta keeps an error of a few ulp of theta_p (1e-5 rad and more
# when the compass lies within 1e-9 of pi), and the next cos(theta + beta) carries speed * dt times that into x and y, where the
# EKF's small position gain keeps it.  Heading: |d theta| <= TOL_THETA * max(1, |theta_p|).  x, y (and the poses, which are the
# previous state): |d| <= TOL_XY * max(|value|, 1 m) + the sum over the route's ticks of speed * dt * the heading bound of the
# state the tick started from.  P: no transcendental function, bit-equal.
TOL_THETA, TOL_XY = 1e-12, 1e-12


def ulp_close(a, b):
    """fp32 arrays equal, or 1 ulp apart; NaN where the other is NaN"""
    nan = np.isnan(b)
    assert np.array_equal(np.isnan(a), nan)
    ia, ib = a[~nan].view(np.int32).astype(np.int64), b[~nan].view(np.int32).astype(np.int64)
    return int(np.abs(ia - ib).max()) if ia.size else 0


@pytest.mark.parametrize("B", [1, 7, 64, 300, 600])
def test_kernels_equal_statement(cuda, B):
    ticks = 1000
    routes, x = nav_drive(B, (2, 500, 5000), ticks, seed=40 + B)
    ref, nav = N.AgentNavRef(B), AgentNavigator(B, cuda)
    control = torch.zeros((B, 3), dtype=torch.float32, device=cuda)
    worst, ulps = dict(xy=0.0, theta=0.0), 0
    theta_scale = np.ones(B)                                     # max(1, |theta_p|) of the state the poses hold
    carried = np.zeros(B)                                        # the position error the heading bounds carry, per route

    def check_state(x_got, x_want, scale, carry, where):
        fin = np.isfinite(x_want)
        assert np.array_equal(fin, np.isfinite(x_got)), where
        d = np.where(fin, np.abs(np.nan_to_num(x_got - x_want)), 0.0)
        bound = TOL_XY * np.maximum(np.abs(np.nan_to_num(x_want[:, :2])), 1.0) + carry[:, None]
        worst["xy"] = max(worst["xy"], float((d[:, :2] / bound).max()))
        worst["theta"] = max(worst["theta"], float((d[:, 2] / scale).max()))
        assert worst["xy"] <= 1 and worst["theta"] <= TOL_THETA, (where, worst)

    for t in range(ticks):
        if t in routes:
            agents, plans = [a for a, _ in routes[t]], [r for _, r in routes[t]]
            ref.set_routes(agents, plans)
            nav.set_routes(agents, plans)
            carried[agents] = 0.0
        want = ref.front(x["gnss"][t], x["compass"][t])
        got = {k: v.cpu().numpy() for k, v in nav.front(x["gnss"][t], x["compass"][t]).items()}
        where = f"B {B} tick {t}"
        np.testing.assert_array_equal(got["cmds"], want["cmds"], err_msg=where)
        np.testing.assert_array_equal(got["flags"], want["flags"], err_msg=where)
        ulps = max(ulps, ulp_close(got["nxps"], want["nxps"]))
        theta_scale = np.where(ref.frames == 1, 1.0, theta_scale)
        check_state(got["poses"], want["poses"], theta_scale, carried, where + " poses")
        carried += np.where(ref.frames >= 2, x["speed"][t] * N.DT * TOL_THETA * theta_scale, 0.0)
        control[:, 0] = torch.from_numpy(x["steer"][t].astype(np.float32))
        ref.update(x["steer"][t], x["speed"][t], x["gnss"][t], x["compass"][t])
        nav.update(control, x["speed"][t])
        s = nav.state_views()
        live = s["frames"] >= 2
        for f, r in (("frames", ref.frames), ("lane_counter", ref.lane_counter), ("lane_changed", ref.lane_changed)):
            np.testing.assert_array_equal(s[f], r, err_msg=f"{where} {f}")
        for f, r in (("wp_idx", ref.wp_idx), ("wp_cmd", ref.wp_cmd), ("rp_idx", ref.rp_idx)):
            np.testing.assert_array_equal(s[f][live], r[live], err_msg=f"{where} {f}")
        assert np.array_equal(s["wp_x"][live], ref.wp[live, 0]) and np.array_equal(s["rp_y"][live], ref.rp[live, 1]), where
        theta_scale = np.where(live, np.maximum(1.0, np.abs(ref.theta_pred)), 1.0)
        check_state(s["ekf_x"], ref.x, theta_scale, carried, where + " ekf_x")
        np.testing.assert_array_equal(s["ekf_p"], ref.p, err_msg=where)
        assert ulps <= 1, (where, ulps)
    print(f"B {B}: max fp64 difference x, y {worst['xy']:.2e} of their bound, theta {worst['theta']:.2e} of max(1, |theta_p|); "
          f"nxps within {ulps} ulp")


def test_set_routes_leaves_other_agents_alone(cuda):
    B = 9
    routes, x = nav_drive(B, (2, 500), 120, seed=3, reset_at=10 ** 9)
    nav = AgentNavigator(B, cuda)
    nav.set_routes([a for a, _ in routes[0]], [r for _, r in routes[0]])
    control = torch.zeros((B, 3), dtype=torch.float32, device=cuda)
    for t in range(100):
        nav.front(x["gnss"][t], x["compass"][t])
        nav.update(control, x["speed"][t])
    before = nav.state.view(B, -1).clone()
    nav.set_routes([2, 5], [routes[0][7][1], routes[0][0][1]])
    after = nav.state.view(B, -1)
    for b in range(B):
        assert torch.equal(after[b], before[b]) == (b not in (2, 5)), b
    res = nav.front(x["gnss"][100], x["compass"][100])
    assert (res["flags"][[2, 5]].cpu() == 1).all()


def _job_stub(B, N, cuda):
    T, KEEP = 3, StaticFramePipeline.KEEP
    import types
    return types.SimpleNamespace(
        B=B, T=T, N=N, KEEP=KEEP, tick=0, ring=torch.randn((B, KEEP, N, 8), device=cuda), cur=torch.randn((B, N, 8), device=cuda),
        stacked=torch.full((B, T * N, 8 + T), float("nan"), device=cuda), ring_pose=np.zeros((B, KEEP, 3)),
        ring_valid=np.zeros((B, KEEP), dtype=bool), jobs_host=torch.zeros(B * T * ops.STACK_JOB_DTYPE.itemsize, dtype=torch.uint8),
        jobs_dev=torch.zeros(B * T * ops.STACK_JOB_DTYPE.itemsize, dtype=torch.uint8, device=cuda))


def test_job_poses_equal_fill_jobs(cuda):
    B, N = 37, 64
    host, dev = _job_stub(B, N, cuda), _job_stub(B, N, cuda)
    dev.ring, dev.cur = host.ring, host.cur
    ring_pose = torch.zeros((B, host.KEEP, 3), dtype=torch.float64, device=cuda)
    rs = np.random.RandomState(5)
    equal_ticks = 0
    for tick in range(3 * GAP + 4):
        poses = np.stack([rs.uniform(-3e6, 3e6, B), rs.uniform(-3e6, 3e6, B), rs.uniform(-7, 7, B)], -1)
        StaticFramePipeline._fill_jobs(host, [(p[:2], p[2]) for p in poses])
        StaticFramePipeline._fill_jobs(dev, None, device_poses=True)
        ops.stack_job_poses(dev.jobs_dev, B, dev.T, GAP, dev.KEEP, dev.tick, ring_pose, torch.from_numpy(poses).to(cuda))
        torch.cuda.synchronize()
        a = host.jobs_dev.cpu().numpy().view(ops.STACK_JOB_DTYPE)
        b = dev.jobs_dev.cpu().numpy().view(ops.STACK_JOB_DTYPE)
        for f in ("src", "n", "time_idx"):
            np.testing.assert_array_equal(a[f], b[f], err_msg=f"tick {tick} {f}")
        np.testing.assert_array_equal(a["dst"] - np.uint64(host.stacked.data_ptr()), b["dst"] - np.uint64(dev.stacked.data_ptr()))
        for f in ("R", "dx", "dy"):
            assert ulp_close(np.ascontiguousarray(b[f]), np.ascontiguousarray(a[f])) <= 1, (tick, f)
        np.testing.assert_array_equal(ring_pose[:, tick % host.KEEP].cpu().numpy(), poses)
        # the stacked sweeps of the two tables: bit-equal wherever the tables are
        host.stacked.fill_(float("nan")); dev.stacked.fill_(float("nan"))
        ops.stack_jobs(host.jobs_dev.to(cuda), B * host.T, N, 8, host.T)
        ops.stack_jobs(dev.jobs_dev, B * dev.T, N, 8, dev.T)
        same = np.array([all(np.array_equal(a.reshape(B, -1)[i][f], b.reshape(B, -1)[i][f]) for f in ("R", "dx", "dy"))
                         for i in range(B)])
        sh, sd = host.stacked.cpu().numpy()[same], dev.stacked.cpu().numpy()[same]
        assert np.array_equal(sh.view(np.uint32), sd.view(np.uint32)), tick
        equal_ticks += int(same.sum())
        for s in (host, dev):
            s.ring[:, s.tick % s.KEEP] = s.cur
            s.tick += 1
    assert equal_ticks > 0


def _models():
    from lav_b200.heads import RGBBrakePredictionModel
    lm, _ = util.lidar_model()
    sm, _ = util.seg_model()
    up, _ = uniplanner()
    bra = RGBBrakePredictionModel([4, 6, 7, 10]).eval()
    bra.load_state_dict(synth.fill_state_dict_(bra.state_dict()))
    return sm, lm, up, bra


def test_pipeline_with_navigator_stacks_as_the_host_poses(cuda):
    """StaticFramePipeline(navigator=nav).begin(gnss=, compass=) against the host-pose path fed nav.front's outputs: the planner
    inputs equal, and the stacked sweeps bit-equal on every agent whose job table equals _fill_jobs'.  Two agents get new routes
    mid-run from the default stream right before a begin() that runs the front on the pipeline's stream, and the navigator
    pipeline takes host poses for two ticks in between (its host ring must catch up with the device ring, and back)."""
    sm, lm, up, bra = _models()
    B, N, ticks, reset_at, host_ticks = 3, 3000, 16, 8, (11, 12)
    routes, x = nav_drive(B, (2, 500), ticks, seed=11)
    new_routes, _ = nav_drive(B, (500, 2), ticks, seed=12)
    nav, shadow = AgentNavigator(B, cuda), AgentNavigator(B, cuda)
    for n in (nav, shadow):
        n.set_routes([a for a, _ in routes[0]], [r for _, r in routes[0]])
    p_dev = StaticFramePipeline(sm, lm, up, bra, B, N, device=cuda, precision="f16", navigator=nav)
    p_host = StaticFramePipeline(sm, lm, up, bra, B, N, device=cuda, precision="f16")
    control = torch.zeros((B, 3), dtype=torch.float32, device=cuda)
    compared = 0
    for t in range(ticks):
        if t == reset_at:
            for n_ in (nav, shadow):
                n_.set_routes([0, 2], [new_routes[0][0][1], new_routes[0][2][1]])
        rgbs = torch.stack([synth.rgb_frames(tag=f"n{t}{b}", smooth=True) for b in range(B)]).to(cuda)
        tels = torch.stack([synth.rgb_frames(tag=f"nt{t}{b}", smooth=True, n_cam=1, h=192, w=480)[0] for b in range(B)]).to(cuda)
        lidars = [synth.lidar_sweep(N - 50 * b, tag=f"nl{t}{b}").to(cuda) for b in range(B)]
        want = {k: v.clone() for k, v in shadow.front(x["gnss"][t], x["compass"][t]).items()}
        poses = [(p[:2], p[2]) for p in want["poses"].cpu().numpy()]
        if t in host_ticks:
            got = nav.front(x["gnss"][t], x["compass"][t])
            p_dev.begin(rgbs, tels, lidars, got["nxps"].cpu(), got["cmds"].cpu().tolist(), poses=poses)
        else:
            got = p_dev.begin(rgbs, tels, lidars, gnss=x["gnss"][t], compass=x["compass"][t])
        p_host.begin(rgbs, tels, lidars, want["nxps"].cpu(), want["cmds"].cpu().tolist(), poses=poses)
        torch.cuda.synchronize()
        # bit for bit: a NaN compass gives NaN targets (x carries one at tick 13)
        assert torch.equal(p_dev.nxps.view(torch.int32), p_host.nxps.view(torch.int32)) and torch.equal(p_dev.cmds, p_host.cmds), t
        assert torch.equal(got["flags"], want["flags"]) and torch.equal(got["poses"].view(torch.int64), want["poses"].view(torch.int64)), t
        if t == reset_at:
            assert (got["flags"][[0, 2]] == 1).all() and got["flags"][1] != 1, got["flags"]
        a = p_host.jobs_dev.cpu().numpy().view(ops.STACK_JOB_DTYPE).reshape(B, -1)
        b = p_dev.jobs_dev.cpu().numpy().view(ops.STACK_JOB_DTYPE).reshape(B, -1)
        for f in ("n", "time_idx"):
            np.testing.assert_array_equal(a[f], b[f], err_msg=f"tick {t} {f}")
        base = lambda p: np.where(np.arange(p.T)[None] == 0, np.uint64(p.cur.data_ptr()), np.uint64(p.ring.data_ptr()))
        np.testing.assert_array_equal(a["src"] - base(p_host), b["src"] - base(p_dev), err_msg=f"tick {t} src")
        rows = [i for i in range(B) if all(np.array_equal(a[i][f], b[i][f]) for f in ("R", "dx", "dy"))]
        for i in rows:
            assert np.array_equal(p_host.stacked[i].cpu().numpy().view(np.uint32), p_dev.stacked[i].cpu().numpy().view(np.uint32)), t
        compared += len(rows)
        p_dev.finish(fixed_dets=DETS); p_host.finish(fixed_dets=DETS)
        for n_ in (nav, shadow):
            n_.update(control, x["speed"][t])
    assert compared >= B * 8


def test_controller_device_cmds_equal_host_cmds(cuda):
    B = 70
    ctl_h, ctl_d = AgentController(B, CFG, cuda), AgentController(B, CFG, cuda)
    for tick, x in enumerate(control_sequence(77, B, 60)):
        out = device_out(x, cuda)
        h = ctl_h.step(out, x["speed"], x["cmd"])
        d = ctl_d.step(out, x["speed"], torch.from_numpy(x["cmd"].astype(np.int32)).to(cuda))
        assert torch.equal(h["control"], d["control"]) and torch.equal(h["flags"], d["flags"]), tick
        assert torch.equal(ctl_h.state, ctl_d.state), tick
    # an out-of-range device command: NaN controls, FLAG_BAD_CMD, the agent's state untouched, the others as the host path
    x = next(control_sequence(78, B, 1))
    out = device_out(x, cuda)
    cmds = torch.from_numpy(x["cmd"].astype(np.int32)).to(cuda)
    cmds[4], cmds[9] = 6, -1
    before = ctl_d.state.view(B, -1).clone()
    d = ctl_d.step(out, x["speed"], cmds)
    h = ctl_h.step(out, x["speed"], np.where((np.arange(B) == 4) | (np.arange(B) == 9), 0, x["cmd"]).astype(np.int32))
    bad = torch.zeros(B, dtype=torch.bool, device=cuda)
    bad[[4, 9]] = True
    assert torch.isnan(d["control"][bad]).all() and (d["flags"][bad] == FLAG_BAD_CMD).all()
    assert torch.equal(d["control"][~bad], h["control"][~bad]) and torch.equal(d["flags"][~bad], h["flags"][~bad])
    assert torch.equal(ctl_d.state.view(B, -1)[bad], before[bad])


def test_malformed_calls_are_rejected_untouched(cuda):
    B = 4
    routes, x = nav_drive(B, (3,), 4, seed=1)
    nav = AgentNavigator(B, cuda)
    nav.set_routes([a for a, _ in routes[0]], [r for _, r in routes[0]])
    g = torch.from_numpy(x["gnss"][0][:, :2].copy()).to(cuda)
    c = torch.from_numpy(x["compass"][0].copy()).to(cuda)
    outs = [torch.full((B,), 77, dtype=torch.int32, device=cuda), torch.full((B, 2), 7.0, device=cuda),
            torch.full((B, 3), 7.0, dtype=torch.float64, device=cuda), torch.full((B,), 77, dtype=torch.int32, device=cuda)]
    state0 = nav.state.clone()
    args = [nav.nodes, nav.node_cmd, nav.route, g, c, nav.state]
    bad = [(1, nav.node_cmd.to(torch.int64)), (2, nav.route[:, :1].contiguous()), (3, g.float()), (3, g[:3]), (4, c[:2]),
           (5, nav.state[:-1]), (0, nav.nodes.float())]
    for k, v in bad:
        a = list(args)
        a[k] = v
        with pytest.raises(LavbError):
            ops.agent_nav_front(*a, *outs)
    with pytest.raises(LavbError):
        ops.agent_nav_front(*args, outs[0], outs[1].double(), outs[2], outs[3])
    with pytest.raises(LavbError):
        ops.agent_nav_update(torch.zeros((B, 2), device=cuda), torch.zeros(B, dtype=torch.float64, device=cuda), g, c, nav.state)
    # the C entry points themselves: unaligned pointers and bad sizes
    p = lambda t, off=0: C.c_void_p(t.data_ptr() + off)
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert lib().lavb_agent_nav_front(B, p(nav.nodes, 8), p(nav.node_cmd), nav.nodes.shape[0], p(nav.route), p(g), p(c),
                                      p(nav.state), p(outs[0]), p(outs[1]), p(outs[2]), p(outs[3]), s) != 0
    assert lib().lavb_agent_nav_front(B, p(nav.nodes), p(nav.node_cmd), -2, p(nav.route), p(g), p(c), p(nav.state), p(outs[0]),
                                      p(outs[1]), p(outs[2]), p(outs[3]), s) != 0
    assert lib().lavb_agent_nav_update(B, p(outs[1]), p(outs[2]), p(g, 8), p(c), p(nav.state), s) != 0
    torch.cuda.synchronize()
    assert torch.equal(nav.state, state0)
    assert (outs[0] == 77).all() and (outs[1] == 7).all() and (outs[2] == 7).all() and (outs[3] == 77).all()
    # a device route entry that is no route: NO_ROUTE, NaN target and pose, the agent's state untouched; the others run
    nav.route[1] = torch.tensor([0, 10 ** 6], dtype=torch.int32)
    nav.route[2] = torch.tensor([-1, 2], dtype=torch.int32)
    res = nav.front(x["gnss"][0], x["compass"][0])
    torch.cuda.synchronize()
    f = res["flags"].cpu().numpy()
    assert f[1] == f[2] == FLAG_NO_ROUTE and f[0] == f[3] == 1
    assert torch.isnan(res["nxps"][1:3]).all() and torch.isnan(res["poses"][1:3]).all()
    assert torch.equal(nav.state.view(B, -1)[1:3], state0.view(B, -1)[1:3])
