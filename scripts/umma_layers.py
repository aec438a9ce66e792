"""Run a few representative wgmma conv layers once and time them with events."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from lav_b200 import ops
from lav_b200.layers import TapConv

dev = torch.device("cuda:0")
B = int(sys.argv[1]) if len(sys.argv) > 1 else 8
cfgs = [("erf64_3x1", 3 * B, 72, 64, 64, 64, (3, 1), (1, 0)), ("erf128_3x1", 3 * B, 36, 32, 128, 128, (3, 1), (1, 0)),
        ("bb64_3x3", B, 160, 160, 64, 64, (3, 3), (1, 1)), ("bb128_3x3", B, 80, 80, 128, 128, (3, 3), (1, 1)),
        ("heads_384_256", B, 160, 160, 384, 256, (3, 3), (1, 1))]
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
for name, n, h, w, cin, cout, k, p in cfgs:
    wgt = torch.randn(cout, cin, *k, device=dev) * 0.05
    layer = TapConv(wgt, False, 1, p, 1, 0, None, pre_relu=True, scale=torch.ones(cout, device=dev), shift=torch.zeros(cout, device=dev))
    x = torch.randn(n, h, w, cin, device=dev).to(ops.h16())
    out = torch.empty(n, h, w, cout, device=dev, dtype=ops.h16())
    for _ in range(3):
        layer(x, out=out)
    ts = []
    for _ in range(5):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); layer(x, out=out); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    t = sorted(ts)[2]
    fl = 2.0 * n * h * w * cout * cin * k[0] * k[1]
    by = n * h * w * (cin + cout) * 2
    tiles = n * ((h + 7) // 8) * ((w + 15) // 16)
    print(f"{name:14s} {t*1e3:8.1f} us  {fl/t/1e9:7.1f} TFLOP/s  {by/t/1e6:7.1f} GB/s(alg)  tiles={tiles} ({tiles/132:.1f}/SM on 132 SMs)")
