"""Measurements of the agent's localisation and route following on the GPU (DESIGN §4): the two navigation launches per tick
(lavb_agent_nav_front + lavb_agent_nav_update) at B agents with CUDA events, the host work they replace on this machine's CPU,
and a two-group StaticFramePipeline + AgentController loop like scripts/control_measure.py's that alternates host navigation
(poses, commands and targets computed on the host and uploaded) with the navigator.

    python scripts/nav_measure.py --out-dir OUT [--batch 64] [--reference DIR]

Host work: the reference's Waypointer.tick + RoutePlanner.run_step + EKF.step per agent when ``--reference`` (team_code_v2 of the
reference) is readable, and always the O(1) numpy statement (oracle/nav_ref) and StaticFramePipeline._fill_jobs, at 100- and
500-node routes.  Results go to OUT/nav_measure.json with the GPU's name, power limit and clocks read in the same run.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from control_measure import config  # noqa: E402
from eval_measure import gpu_info  # noqa: E402


def inputs(B, nodes, ticks, seed):
    from oracle.nav_ref import nav_drive
    return nav_drive(B, (nodes,), ticks, seed, reset_at=10 ** 9)


def launches(B, rounds, reps, dev):
    """the two launches per tick on prepared device inputs, and AgentNavigator.front + update with the host-to-device staging"""
    from lav_b200 import ops
    from lav_b200.navigation import AgentNavigator
    routes, x = inputs(B, 500, 40, 1)
    nav = AgentNavigator(B, dev)
    nav.set_routes([a for a, _ in routes[0]], [r for _, r in routes[0]])
    control = torch.zeros((B, 3), dtype=torch.float32, device=dev)
    for t in range(20):
        nav.front(x["gnss"][t], x["compass"][t])
        nav.update(control, x["speed"][t])
    g, c = torch.from_numpy(x["gnss"][20][:, :2].copy()).to(dev), torch.from_numpy(x["compass"][20].copy()).to(dev)
    sp = torch.from_numpy(x["speed"][20].copy()).to(dev)
    out = [nav.out[k] for k in ("cmds", "nxps", "poses", "flags")]
    raw, full = [], []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            ops.agent_nav_front(nav.nodes, nav.node_cmd, nav.route, g, c, nav.state, *out)
            ops.agent_nav_update(control, sp, g, c, nav.state)
        e1.record()
        torch.cuda.synchronize()
        raw.append(e0.elapsed_time(e1) / reps)
        t0 = time.perf_counter()
        for k in range(reps):
            nav.front(x["gnss"][21 + k % 19], x["compass"][21 + k % 19])
            nav.update(control, x["speed"][21 + k % 19])
        torch.cuda.synchronize()
        full.append((time.perf_counter() - t0) * 1e3 / reps)
    return dict(agents=B, route_nodes=500, two_launches_ms_median=float(np.median(raw)),
                navigator_front_update_wall_ms_median=float(np.median(full)), rounds_ms=raw)


def host_costs(B, reference, rounds, dev):
    """per tick, B agents: the reference objects (when readable), the O(1) statement, and _fill_jobs' pose work"""
    import types
    from lav_b200 import ops
    from lav_b200.agent import StaticFramePipeline
    from oracle.nav_ref import AgentNavRef
    res = {}
    for nodes in (100, 500):
        routes, x = inputs(B, nodes, 60, 2)
        r = {}
        if reference:
            sys.path.insert(0, os.path.join(ROOT, "oracle", "refshim"))
            sys.path.insert(0, reference)
            from agents.navigation.local_planner import RoadOption
            from ekf import EKF
            from planner import RoutePlanner
            from waypointer import Waypointer
            plans = [[(g, RoadOption(c)) for g, c in rt] for _, rt in routes[0]]
            objs = []
            for b in range(B):
                gps = x["gnss"][0, b]
                e = EKF(1, 1.477531, 1.393600)
                e.init(gps[0], gps[1], 0.0)
                objs.append((Waypointer(plans[b], gps, pop_lane_change=True), RoutePlanner(plans[b]), e))
            ms = []
            for _ in range(rounds):
                t0 = time.perf_counter()
                for t in range(1, 21):
                    for b, (wp, rp, e) in enumerate(objs):
                        gps = x["gnss"][t, b]
                        wp.tick(gps)
                        rp.run_step(gps)
                        e.step(x["speed"][t, b], 0.1, gps[0], gps[1], 0.0)
                ms.append((time.perf_counter() - t0) * 1e3 / 20)
            r["reference_objects_ms_per_tick_median"] = float(np.median(ms))
        ref = AgentNavRef(B)
        ref.set_routes([a for a, _ in routes[0]], [rt for _, rt in routes[0]])
        ms = []
        for _ in range(rounds):
            t0 = time.perf_counter()
            for t in range(1, 21):
                ref.front(x["gnss"][t], x["compass"][t])
                ref.update(x["steer"][t], x["speed"][t], x["gnss"][t], x["compass"][t])
            ms.append((time.perf_counter() - t0) * 1e3 / 20)
        r["numpy_statement_ms_per_tick_median"] = float(np.median(ms))
        res[str(nodes)] = r
    T, KEEP, N = 3, StaticFramePipeline.KEEP, 16
    stub = types.SimpleNamespace(B=B, T=T, N=N, KEEP=KEEP, tick=0, ring=torch.zeros((B, KEEP, N, 8), device=dev),
                                 cur=torch.zeros((B, N, 8), device=dev), stacked=torch.zeros((B, T * N, 8 + T), device=dev),
                                 ring_pose=np.zeros((B, KEEP, 3)), ring_valid=np.zeros((B, KEEP), dtype=bool),
                                 jobs_host=torch.zeros(B * T * ops.STACK_JOB_DTYPE.itemsize, dtype=torch.uint8).pin_memory(),
                                 jobs_dev=torch.zeros(B * T * ops.STACK_JOB_DTYPE.itemsize, dtype=torch.uint8, device=dev))
    poses = [(np.array([1.0 * b, 2.0]), 0.1 * b) for b in range(B)]
    ms = {"host_poses": [], "device_poses": []}
    for _ in range(rounds):
        for name, dp in (("host_poses", False), ("device_poses", True)):
            t0 = time.perf_counter()
            for _ in range(50):
                StaticFramePipeline._fill_jobs(stub, None if dp else poses, device_poses=dp)
                stub.tick += 1
            torch.cuda.synchronize()
            ms[name].append((time.perf_counter() - t0) * 1e3 / 50)
    res["fill_jobs_ms_median"] = {k: float(np.median(v)) for k, v in ms.items()}
    return res


def pipeline_loop(B, groups, steps, rounds, dev):
    import bench
    from lav_b200 import synth
    from lav_b200.agent import StaticFramePipeline
    from lav_b200.control import AgentController
    from lav_b200.navigation import AgentNavigator
    from oracle.nav_ref import AgentNavRef
    cfg = config()
    Bp = B // groups
    N = synth.SWEEP_POINTS
    routes, x = inputs(B, 100, steps * (rounds + 3) * 2 + 4, 3)
    plans = [rt for _, rt in routes[0]]
    (seg, lid, uni, bra), _ = bench.build_models()
    navs = [AgentNavigator(Bp, dev) for _ in range(groups)]
    refs = [AgentNavRef(Bp) for _ in range(groups)]
    sl = [slice(pi * Bp, (pi + 1) * Bp) for pi in range(groups)]
    for pi in range(groups):
        navs[pi].set_routes(range(Bp), plans[sl[pi]])
        refs[pi].set_routes(range(Bp), plans[sl[pi]])
    p_nav = [StaticFramePipeline(seg, lid, uni, bra, Bp, N, device=dev, precision="f16", navigator=navs[pi]) for pi in range(groups)]
    p_host = [StaticFramePipeline(seg, lid, uni, bra, Bp, N, device=dev, precision="f16") for _ in range(groups)]
    rgbs, tels, lidars, _, _ = bench.synth_frames(B)
    h_rgbs, h_tels, h_lidar = rgbs.pin_memory(), tels.pin_memory(), torch.stack(lidars).pin_memory()
    ctls = [AgentController(Bp, cfg, dev) for _ in range(groups)]
    h_ctl = [torch.empty((Bp, 3), dtype=torch.float32).pin_memory() for _ in range(groups)]
    tick = [0]

    def step_device():
        t = tick[0]; tick[0] += 1
        for pi, pp in enumerate(p_nav):
            pp.begin(h_rgbs[sl[pi]], h_tels[sl[pi]], h_lidar[sl[pi]], gnss=x["gnss"][t, sl[pi]], compass=x["compass"][t, sl[pi]])
        outs = [pp.finish(fixed_dets=bench.FIXED_DETS) for pp in p_nav]
        for pi, o in enumerate(outs):
            res = ctls[pi].step(o, x["speed"][t, sl[pi]].astype(np.float32), navs[pi].out["cmds"])
            navs[pi].update(res["control"], x["speed"][t, sl[pi]])
            h_ctl[pi].copy_(res["control"], non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return [c.numpy() for c in h_ctl]

    def step_host():
        t = tick[0]; tick[0] += 1
        fr = [refs[pi].front(x["gnss"][t, sl[pi]], x["compass"][t, sl[pi]]) for pi in range(groups)]
        for pi, pp in enumerate(p_host):
            pp.begin(h_rgbs[sl[pi]], h_tels[sl[pi]], h_lidar[sl[pi]], torch.from_numpy(fr[pi]["nxps"]), fr[pi]["cmds"].tolist(),
                     poses=[(p[:2], p[2]) for p in fr[pi]["poses"]])
        outs = [pp.finish(fixed_dets=bench.FIXED_DETS) for pp in p_host]
        for pi, o in enumerate(outs):
            h_ctl[pi].copy_(ctls[pi].step(o, x["speed"][t, sl[pi]].astype(np.float32), fr[pi]["cmds"])["control"],
                            non_blocking=True)
        torch.cuda.current_stream().synchronize()
        for pi in range(groups):
            refs[pi].update(h_ctl[pi].numpy()[:, 0], x["speed"][t, sl[pi]], x["gnss"][t, sl[pi]], x["compass"][t, sl[pi]])
        return [c.numpy() for c in h_ctl]

    for _ in range(3):
        step_device(); step_host()
    ms = {"device": [], "host": []}
    for _ in range(rounds):
        for name, fn in (("device", step_device), ("host", step_host)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                fn()
            ms[name].append((time.perf_counter() - t0) * 1e3 / steps)
    return dict(agents=B, groups=groups, steps_per_round=steps, rounds=rounds, route_nodes=100,
                navigator_ms_per_tick_median=float(np.median(ms["device"])),
                host_navigation_ms_per_tick_median=float(np.median(ms["host"])),
                device_rounds_ms=ms["device"], host_rounds_ms=ms["host"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", required=True)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reference", default=None, help="team_code_v2 of the reference, to time its own classes")
    args = ap.parse_args()
    dev = torch.device("cuda")
    from lav_b200 import capi
    capi.lib()
    ref = args.reference if args.reference and os.path.isdir(args.reference) else None
    res = dict(gpu=gpu_info(), torch=torch.__version__, numpy=np.__version__, host_cpus=os.cpu_count())
    res["launches"] = launches(args.batch, args.rounds, 200, dev)
    res["host"] = host_costs(args.batch, ref, args.rounds, dev)
    res["pipeline"] = pipeline_loop(args.batch, 2, 20, args.rounds, dev)
    res["gpu_after"] = gpu_info()
    os.makedirs(args.out_dir, exist_ok=True)
    path = os.path.join(args.out_dir, "nav_measure.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
