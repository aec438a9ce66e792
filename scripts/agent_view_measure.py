"""Measurements of the agent's debug view on the GPU (DESIGN §4): the lavb_agent_view launches per tick at B agents with 40 k and
120 k points per sweep, three sweeps stacked (CUDA events, medians over alternating rounds, with the bytes the launches must
move computed from the shapes), the device-to-host copy of the frames into pinned memory, the host statement (oracle/view_ref.frame) per agent on this
machine's CPU, and a two-group StaticFramePipeline + AgentController loop like control_measure.py's, without a view and with
AgentRecorder recording every tick.

    python scripts/agent_view_measure.py --out-dir OUT [--batch 64]

The GPU's name, power limit and clocks are read in the same run.  Results go to OUT/agent_view_measure.json.
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

from eval_measure import gpu_info  # noqa: E402

FRAME_BYTES = 160 * 1146 * 3


def view_bytes(B, P, c_bev, bev_elem):
    """bytes the launches must move: the cameras and tele view read once, x / y of every stacked row (its 44-byte row), the BEV
    logits, the scratch planes zeroed, written and read, the frames written"""
    sensors = 3 * 288 * 256 * 3 + 192 * 480 * 3
    scratch = 320 * 320 * 12
    return B * (sensors + P * 44 + c_bev * 320 * 320 * bev_elem + 3 * scratch + FRAME_BYTES)


def render_times(B, sizes, rounds, reps, dev):
    from lav_b200 import ops
    from lav_b200.view import view_config
    from tests.test_gpu_agent_view import CFG, inputs, device_args
    cases = {}
    for P in sizes:
        x = inputs(B, 3 * P, [3] * B, "h16", seed=P, cuda=dev)             # t, t-5 and t-10 stacked
        args = device_args(x, dev)
        scratch = torch.empty((ops.agent_view_scratch_bytes(B),), dtype=torch.uint8, device=dev)
        out = torch.empty((B, 160, 1146, 3), dtype=torch.uint8, device=dev)
        cases[P] = (args, scratch, out, x["bev"].shape[1], x["bev"].element_size(), x)
    cfg = view_config(CFG)
    for P, (args, scratch, out, *_rest) in cases.items():
        for _ in range(3):
            ops.agent_view(*args, cfg, scratch=scratch, out=out)
    ms = {P: [] for P in sizes}
    for _ in range(rounds):
        for P in sizes:
            args, scratch, out = cases[P][:3]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                ops.agent_view(*args, cfg, scratch=scratch, out=out)
            e1.record()
            e1.synchronize()
            ms[P].append(e0.elapsed_time(e1) / reps)
    res = {}
    host = torch.empty((B, 160, 1146, 3), dtype=torch.uint8).pin_memory()
    for P in sizes:
        args, scratch, out, c, elem, x = cases[P]
        med = float(np.median(ms[P]))
        nbytes = view_bytes(B, 3 * P, c, elem)
        res[f"points_{P}"] = dict(render_ms_median=med, render_rounds_ms=ms[P], bytes_moved=nbytes,
                                  achieved_GBps=nbytes / med / 1e6, points_per_sweep=P, stacked_rows=3 * P, vehicles_per_agent=3)
    copies = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        host.copy_(cases[sizes[0]][2], non_blocking=True)
        e1.record()
        e1.synchronize()
        copies.append(e0.elapsed_time(e1))
    res["d2h_frames"] = dict(bytes=B * FRAME_BYTES, ms_median=float(np.median(copies)), rounds_ms=copies,
                             GBps=B * FRAME_BYTES / float(np.median(copies)) / 1e6)
    return res, cases


def host_statement(cases, sizes):
    """oracle/view_ref.frame of agent 0 on the host CPU, from host copies of its inputs (the copies are not timed)"""
    from oracle import view_ref as V
    from tests.test_gpu_agent_view import statement
    res = {}
    for P in sizes:
        x = cases[P][5]
        sig = torch.sigmoid(x["bev"][:1].float()).cpu().numpy()
        t = []
        for _ in range(3):
            t0 = time.perf_counter()
            statement(x, 0, sig)
            t.append((time.perf_counter() - t0) * 1e3)
        res[f"points_{P}_ms_per_agent_median"] = float(np.median(t))
    res["statement"] = V.__name__
    return res


def pipeline_loop(B, groups, steps, rounds, dev):
    import bench
    from lav_b200 import synth
    from lav_b200.agent import StaticFramePipeline
    from lav_b200.control import AgentController
    from lav_b200.view import AgentRecorder, AgentView
    from tests.test_gpu_agent_view import CFG
    Bp = B // groups
    N = synth.SWEEP_POINTS
    (seg, lid, uni, bra), _ = bench.build_models()
    pipes = [StaticFramePipeline(seg, lid, uni, bra, Bp, N, device=dev, precision="f16") for _ in range(groups)]
    rgbs, tels, lidars, prev, poses = bench.synth_frames(B)
    h_rgbs, h_tels, h_lidar = rgbs.pin_memory(), tels.pin_memory(), torch.stack(lidars).pin_memory()
    nxps = torch.tensor([[0.0, -20.0]] * B).pin_memory()
    cmds = np.array([3] * B, dtype=np.int32)
    for pi, pp in enumerate(pipes):
        pp.tick = 10
        for b in range(Bp):
            loc, ori = poses[pi * Bp + b]
            pp.preload_history(b, [(prev[pi * Bp + b][k % 2].to(dev), loc[1 + (k % 2)], ori[1 + (k % 2)]) for k in range(10)])
    step_poses = [(poses[b][0][0], poses[b][1][0]) for b in range(B)]
    sl = [slice(pi * Bp, (pi + 1) * Bp) for pi in range(groups)]
    ctls = [AgentController(Bp, CFG, dev) for _ in range(groups)]
    recs = [AgentRecorder(AgentView(Bp, CFG, dev)) for _ in range(groups)]
    speeds = np.random.RandomState(0).uniform(0.0, 10.0, B).astype(np.float32)
    h_ctl = [torch.empty((Bp, 3), dtype=torch.float32).pin_memory() for _ in range(groups)]

    def step(record):
        for pi, pp in enumerate(pipes):
            pp.begin(h_rgbs[sl[pi]], h_tels[sl[pi]], h_lidar[sl[pi]], nxps[sl[pi]], cmds[sl[pi]].tolist(), poses=step_poses[sl[pi]])
        for pi, pp in enumerate(pipes):
            o = pp.finish(fixed_dets=bench.FIXED_DETS)
            res = ctls[pi].step(o, speeds[sl[pi]], cmds[sl[pi]])
            if record:
                recs[pi].record(pp, o, res, speeds[sl[pi]])
            h_ctl[pi].copy_(res["control"], non_blocking=True)
        torch.cuda.current_stream().synchronize()

    for _ in range(3):
        step(False); step(True)
    for r in recs:
        r.flush()
    ms = {"controls": [], "controls_and_recorder": []}
    for _ in range(rounds):
        for name, rec in (("controls", False), ("controls_and_recorder", True)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                step(rec)
            if rec:           # the writer thread's queued ticks are part of the cost
                for r in recs:
                    r.pending(0)
            ms[name].append((time.perf_counter() - t0) * 1e3 / steps)
            if rec:           # the frames are handed out outside the timed window
                frames = [r.flush() for r in recs]
                assert all(len(f[0]) == steps for f in frames)
    for r in recs:
        r.close()
    return dict(agents=B, groups=groups, steps_per_round=steps, rounds=rounds,
                **{f"{k}_ms_per_tick_median": float(np.median(v)) for k, v in ms.items()},
                **{f"{k}_rounds_ms": v for k, v in ms.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", required=True)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=7)
    args = ap.parse_args()
    dev = torch.device("cuda")
    from lav_b200 import capi
    capi.lib()
    res = dict(gpu=gpu_info(), torch=torch.__version__, numpy=np.__version__, host_cpus=os.cpu_count())
    sizes = (40000, 120000)
    res["render"], cases = render_times(args.batch, sizes, args.rounds, 20, dev)
    res["host_statement"] = host_statement(cases, sizes)
    del cases
    res["pipeline"] = pipeline_loop(args.batch, 2, 10, args.rounds, dev)
    res["gpu_after"] = gpu_info()
    os.makedirs(args.out_dir, exist_ok=True)
    path = os.path.join(args.out_dir, "agent_view_measure.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
