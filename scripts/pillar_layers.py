"""one sorted pillar-encoder forward (B x 120k points) inside a cudaProfiler range"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from lav_b200 import synth
from tests import util
B = int(sys.argv[1]) if len(sys.argv) > 1 else 16
KW = dict(canvas16=True)
dev = torch.device("cuda:0")
m, _ = util.lidar_model(dev)
m.set_precision("f16")
pts = torch.stack([synth.stacked_lidar(tag=f"pl{b % 4}") for b in range(B)]).to(dev).contiguous()
with torch.no_grad():
    for _ in range(2):
        m.point_pillar_net.forward_nhwc(pts, [pts.shape[1]] * B, **KW)
    torch.cuda.synchronize()
    torch.cuda.profiler.start()
    m.point_pillar_net.forward_nhwc(pts, [pts.shape[1]] * B, **KW)
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()
