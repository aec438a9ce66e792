"""Measurements of the agent's controls on the GPU (DESIGN §4): the lavb_agent_control time per tick, the host statement of the same
tail (oracle/control_ref.ControlTail, vectorised numpy) with the device-to-host copies it needs, and a two-group
StaticFramePipeline loop like bench.py's end-to-end leg that alternates "controls on the device + one copy" with "copy plans,
casts and forecasts + host tail".

    python scripts/control_measure.py --out-dir OUT [--batch 64]

Kernel and host times are medians over alternating rounds on seeded ticks of control_sequence with 3 and 15 forecast rows per
agent (T = 20, 6 branches, the reference config's controller); the loop uses bench.build_models and bench.FIXED_DETS (3 vehicles
per agent).  The GPU's name, power limit and clocks are read in the same run.  Results go to OUT/control_measure.json.
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

CFG_PATH = os.path.join(ROOT, "tests", "golden", "agent_control.npz")


def config():
    return json.loads(str(np.load(CFG_PATH)["config"]))


def tick_inputs(B, rows, seed, dev):
    """one seeded tick with exactly ``rows`` forecast rows per agent: the host dict and its pipeline-shaped device copy"""
    from oracle.control_ref import control_sequence
    x = next(control_sequence(seed, B, 1, max_rows=rows))
    rs = np.random.RandomState(seed)
    for b in range(B):                                      # control_sequence draws 0..max_rows: pad / cut to ``rows``
        o, c = x["other_locs"][b], x["other_cmds"][b]
        idx = rs.randint(0, max(len(o), 1), rows) if len(o) else None
        x["other_locs"][b] = o[idx] if idx is not None else np.zeros((rows,) + x["other_locs"][1].shape[1:], np.float32)
        x["other_cmds"][b] = c[idx] if idx is not None else np.zeros((rows, c.shape[1]), np.float32)
    counts = [rows] * B
    locs = torch.from_numpy(np.concatenate(x["other_locs"])).to(dev)
    cmds = torch.from_numpy(np.concatenate(x["other_cmds"])).to(dev)
    out = dict(ego_plan_locs=torch.from_numpy(x["plan"]).to(dev), ego_cast_locs=torch.from_numpy(x["cast"]).to(dev),
               other_cast_locs=torch.split(locs, counts), other_cast_cmds=torch.split(cmds, counts),
               pred_bra=torch.from_numpy(x["pred_bra"]).to(dev))
    return x, out


def host_tail(tail, out, speeds, cmds, per_agent):
    """the host baseline: copy what the tail reads to the host (per agent like run_step's to_numpy calls, or one copy per
    tensor) and run the statement"""
    B = tail.B
    if per_agent:
        locs = [o.cpu().numpy() for o in out["other_cast_locs"]]
        scores = [o.cpu().numpy() for o in out["other_cast_cmds"]]
    else:
        counts = [len(o) for o in out["other_cast_locs"]]
        locs = np.split(torch.cat(list(out["other_cast_locs"])).cpu().numpy(), np.cumsum(counts)[:-1])
        scores = np.split(torch.cat(list(out["other_cast_cmds"])).cpu().numpy(), np.cumsum(counts)[:-1])
    return tail.step(out["ego_plan_locs"].cpu().numpy(), out["ego_cast_locs"].cpu().numpy(), locs, scores,
                     out["pred_bra"].float().cpu().numpy().reshape(B), speeds, cmds)


def kernel_and_host(B, rows_list, rounds, reps, dev):
    from lav_b200.control import AgentController
    from oracle.control_ref import ControlTail
    cfg = config()
    res = {}
    inputs = {r: tick_inputs(B, r, 10 + r, dev) for r in rows_list}
    ctls = {r: AgentController(B, cfg, dev) for r in rows_list}
    tails = {r: ControlTail(B, cfg) for r in rows_list}
    d_speed = {r: torch.from_numpy(inputs[r][0]["speed"]).to(dev) for r in rows_list}
    k_ms = {r: [] for r in rows_list}
    h_ms = {(r, p): [] for r in rows_list for p in (False, True)}
    for _ in range(rounds):
        for r in rows_list:
            x, out = inputs[r]
            ctls[r].step(out, d_speed[r], x["cmd"])
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                ctls[r].step(out, d_speed[r], x["cmd"])
            e1.record()
            torch.cuda.synchronize()
            k_ms[r].append(e0.elapsed_time(e1) / reps)
            for per_agent in (False, True):
                t0 = time.perf_counter()
                n = max(1, reps // 10)
                for _ in range(n):
                    host_tail(tails[r], out, x["speed"], x["cmd"], per_agent)
                h_ms[(r, per_agent)].append((time.perf_counter() - t0) * 1e3 / n)
    # the launch alone: ops.agent_control on prepared arguments, without AgentController.step's host-side preparation
    from lav_b200 import ops
    for r in rows_list:
        x, out = inputs[r]
        offsets = np.arange(0, B * r + 1, r, dtype=np.int32)
        args = (out["ego_plan_locs"], out["ego_cast_locs"], torch.cat(list(out["other_cast_locs"])),
                torch.cat(list(out["other_cast_cmds"])), offsets, out["pred_bra"], d_speed[r], x["cmd"].astype(np.int32),
                ctls[r].config, ctls[r].state)
        ops.agent_control(*args)
        times = []
        for _ in range(rounds):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                ops.agent_control(*args)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1) / reps)
        res[str(r)] = dict(agents=B, rows_per_agent=r, steps=20, branches=6,
                           controller_step_ms_median=float(np.median(k_ms[r])), launch_ms_median=float(np.median(times)),
                           host_statement_one_copy_per_tensor_ms_median=float(np.median(h_ms[(r, False)])),
                           host_statement_per_agent_copies_ms_median=float(np.median(h_ms[(r, True)])))
    return res


def pipeline_loop(B, groups, steps, rounds, dev):
    import bench
    from lav_b200 import synth
    from lav_b200.agent import StaticFramePipeline
    from lav_b200.control import AgentController
    from oracle.control_ref import ControlTail
    cfg = config()
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
    ctls = [AgentController(Bp, cfg, dev) for _ in range(groups)]
    tails = [ControlTail(Bp, cfg) for _ in range(groups)]
    speeds = np.random.RandomState(0).uniform(0.0, 10.0, B).astype(np.float32)
    h_ctl = [torch.empty((Bp, 3), dtype=torch.float32).pin_memory() for _ in range(groups)]

    def run():
        for pi, pp in enumerate(pipes):
            pp.begin(h_rgbs[sl[pi]], h_tels[sl[pi]], h_lidar[sl[pi]], nxps[sl[pi]], cmds[sl[pi]].tolist(), poses=step_poses[sl[pi]])
        return [pp.finish(fixed_dets=bench.FIXED_DETS) for pp in pipes]

    def step_device():
        outs = run()
        for pi, o in enumerate(outs):
            h_ctl[pi].copy_(ctls[pi].step(o, speeds[sl[pi]], cmds[sl[pi]])["control"], non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return [c.numpy() for c in h_ctl]

    def step_host():
        outs = run()
        return [host_tail(tails[pi], o, speeds[sl[pi]], cmds[sl[pi]], per_agent=True)["control"] for pi, o in enumerate(outs)]

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
    return dict(agents=B, groups=groups, steps_per_round=steps, rounds=rounds,
                device_controls_ms_per_tick_median=float(np.median(ms["device"])),
                host_tail_ms_per_tick_median=float(np.median(ms["host"])),
                device_rounds_ms=ms["device"], host_rounds_ms=ms["host"])


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
    res["kernel"] = kernel_and_host(args.batch, (3, 15), args.rounds, 200, dev)
    res["pipeline"] = pipeline_loop(args.batch, 2, 20, args.rounds, dev)
    res["gpu_after"] = gpu_info()
    os.makedirs(args.out_dir, exist_ok=True)
    path = os.path.join(args.out_dir, "control_measure.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
