"""End-to-end A/B of two builds of liblavb200.so on the 16-bit LiDAR + planner path, separating the kernels under comparison from
the pillar canvas, which is not reproducible from run to run (its centroid sums are float atomic adds).

    python scripts/lidar_planner_ab.py OTHER/liblavb200.so

On the inputs of tests/test_gpu_config_sizes.py config 3 (B = 64 frames of 120 000 stacked points) it prints
  - how many canvas elements differ between three runs of the pillar encoder, for each build;
  - for ONE canvas fed to both builds: whether features, the four heads and every planner output are bit-identical;
  - whether the 16-bit ERFNet logits of four 3-camera frames are bit-identical.
The base build runs every layer on the kernels it has (layers.cmajor_wins off), whatever this tree routes elsewhere.
"""
import ctypes
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from lav_b200 import capi, layers as L, ops, synth
from tests import util
from tests.test_heads_cpu import uniplanner


def load(path):
    """capi.lib() of the library at `path`, binding only the entry points it exports (an older build lacks the newer ones)"""
    saved = dict(capi._SIGS)
    handle = ctypes.CDLL(path)
    for name in [k for k in capi._SIGS if not hasattr(handle, k)]:
        del capi._SIGS[name]
    capi._lib, capi.LIB_PATH = None, path
    try:
        return capi.lib()
    finally:
        capi._SIGS.clear()
        capi._SIGS.update(saved)


if not torch.cuda.is_available():
    sys.exit("lidar_planner_ab.py needs a CUDA device")
here = capi.LIB_PATH
libs = {"base": load(os.path.abspath(sys.argv[1])), "this": load(here)}
cuda = torch.device("cuda:0")
B, K, N = 64, 3, 40000
dets = [(150.0, 200.0, 8.0, 4.0, 0.9, 0.3), (170.0, 240.0, 8.0, 4.0, -0.2, 0.95), (120.0, 150.0, 8., 4., 1., 0.)]
clouds = [synth.stacked_lidar(N, tag=f"c3{b % 8}") for b in range(8)]
batch = torch.stack([clouds[b % 8] for b in range(B)]).to(cuda)
batch[:, :, 3] += torch.arange(B, device=cuda).view(B, 1) * 1e-3
m, lsd = util.lidar_model(cuda)
m.set_precision("f16")
up, usd = uniplanner()
up = up.to(cuda)
up.lidar_conv_emb.to(ops.h16()).to(memory_format=torch.channels_last)
locs, oris, fidx = [], [], []
for b in range(B):
    l, o = up.det_to_locs(dets, 320, 320)
    locs += l; oris += o; fidx += [b] * len(l)
all_locs = torch.cat([torch.tensor(locs), torch.zeros(B, 2)]).to(cuda)
all_oris = torch.cat([torch.tensor(oris), torch.zeros(B)]).to(cuda)
all_fidx = torch.cat([torch.tensor(fidx), torch.arange(B)]).to(torch.int32).to(cuda)
nxps = torch.tensor([[0.0, -20.0]] * B, device=cuda)
cmds = torch.full((B,), 3, dtype=torch.long, device=cuda)
wins = L.cmajor_wins


def use(k):              # the base build has no lavb_conv3x3_umma: keep its layers on conv_umma
    capi._lib = libs[k]
    L.cmajor_wins = wins if k == "this" else (lambda *a: False)


def canvas():
    return m.point_pillar_net.forward_nhwc(batch, [3 * N] * B, canvas16=True).clone()

with torch.no_grad():
    for k in libs:
        use(k)
        cs = [canvas() for _ in range(3)]
        for i in (1, 2):
            d = (cs[0].float() - cs[i].float()).abs()
            print(f"[{k}] canvas run 0 vs {i}: {int((d > 0).sum())} of {d.numel()} elements differ, max {float(d.max()):.3e}")
    use("base")
    cv = canvas()
    outs = {}
    for k in libs:
        use(k)
        feats = m.backbone.forward_nhwc(cv)
        heads = m.heads_nhwc(feats)
        plan = up.infer_device(feats.permute(0, 3, 1, 2), all_locs, all_oris, all_fidx, B * K, nxps, cmds)
        torch.cuda.synchronize()
        outs[k] = [feats.clone(), *[t.clone() for t in heads], *[t.clone() for t in plan]]
    names = ["features", "center", "box", "ori", "seg", "ego_embd", "ego_plan", "ego_cast", "other_cast", "other_cmd"]
    for n, a, b in zip(names, outs["base"], outs["this"]):
        d = (a.float() - b.float()).abs()
        print(f"same canvas, base vs this: {n:10s} {'bit-identical' if torch.equal(a, b) else f'{int((d > 0).sum())} differ, max {float(d.max()):.3e} = {float(d.max() / a.float().abs().max()):.2e} of scale'}")
    # ERFNet f16 on three camera frames
    sm, _ = util.seg_model(cuda)
    sm.set_precision("f16")
    rgb = torch.stack([synth.rgb_frames(tag=f"e2e{i}", smooth=True) for i in range(4)]).view(-1, 288, 256, 3).to(cuda)
    seg = {}
    for k in libs:
        use(k)
        seg[k] = sm.forward_u8(rgb).clone()
    print("erfnet f16 logits base vs this:", "bit-identical" if torch.equal(seg["base"], seg["this"]) else
          f"max diff {float((seg['base'].float() - seg['this'].float()).abs().max()):.3e}")
