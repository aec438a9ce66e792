"""Pillar encoder A/B: sorted vs tile-binned kernels (mma.sync / wgmma MLP) on B frames of 120k stacked points (and B x 40k,
config 2).  python scripts/pillar_ab.py [B]"""
import os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from lav_b200 import ops, synth
from tests import util

B = int(sys.argv[1]) if len(sys.argv) > 1 else 32
dev = torch.device("cuda:0")
m, _ = util.lidar_model(dev)


def graph_time(fn, iters=20):
    for _ in range(2):
        out = fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        g.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters, out


with torch.no_grad():
    for n_sweep, label in ((40000, "120k stacked"), (13334, "40k stacked")):
        clouds = [synth.stacked_lidar(n_sweep, tag=f"ab{i}") for i in range(4)]
        pts = torch.stack([clouds[b % 4] for b in range(B)]).to(dev).contiguous()
        P = pts.shape[1]
        m.set_precision("fp32")
        ms, ref = graph_time(lambda: m.point_pillar_net.forward_nhwc(pts, [P] * B))
        alg32 = (P * 11 * 4 + 320 * 320 * 64 * 4) * B
        print(f"{label} B={B}: exact fp32 kernel {ms * 1e3 / B:.2f} us/frame ({alg32 / ms / 1e6:.0f} GB/s algorithmic)", flush=True)
        ref = ref.clone()
        m.set_precision("f16")
        for enc, kw, nm in (("sorted", dict(split_out=True), "split"), ("sorted", dict(), "fp32"), ("sorted", dict(canvas16=True), "h16"), ("tiled", dict(split_out=True), "split"),
                            ("tiled", dict(), "fp32"), ("tiled", dict(canvas16=True), "h16")):
            ops.PILLAR_ENCODER = enc
            ms, out = graph_time(lambda: m.point_pillar_net.forward_nhwc(pts, [P] * B, **kw))
            o = out.float()
            if nm == "split":
                o = o[..., :64] + o[..., 64:]
            alg = (P * 11 * 4 + 320 * 320 * 64 * (2 if nm == "h16" else 4)) * B
            err = float((o - ref).abs().max() / ref.abs().max())
            occ = bool(torch.equal((o != 0).any(-1), (ref != 0).any(-1)))
            print(f"{label} B={B}: {enc:6s} out={nm:5s}: {ms * 1e3 / B:.2f} us/frame ({alg / ms / 1e6:.0f} GB/s algorithmic), "
                  f"max-norm err vs exact {err:.2e}, occupancy equal {occ}", flush=True)
        ops.PILLAR_ENCODER = "sorted"
