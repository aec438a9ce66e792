"""Planner embedder stem (conv 7x7 / s2 / p3, 384 -> 64, folded BN + ReLU) at the bench shape (128 crops of 96 x 96 x 384, one
agent group of 32 frames x (3 vehicles + ego)) and the batch-1 latency leg's 9 crops: the lav_b200 wgmma kernel
(ops.conv7x7s2_umma) against the cuDNN call it replaces, with cuDNN autotune off (the bench setting) and on.  CUDA events
over >= 20 launches after warm-up; FLOPs from the shapes.

    python scripts/planner_stem_layer.py [--out results.json]
"""
import argparse, json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from lav_b200 import ops

PEAK = 989.0      # H100 SXM dense f16 TFLOP/s (data sheet, 700 W)
ITERS = 20


def timed(fn):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(ITERS):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / ITERS


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", help="also write the results as JSON to this path")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("gpu:", gpu)
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(0)
    res = {"gpu": gpu, "iters": ITERS, "rows": []}
    for n in (128, 9):
        x = torch.randn(n, 96, 96, 384, generator=g).to(dev, ops.h16())
        w = (torch.randn(64, 384, 7, 7, generator=g) / (49 * 384) ** 0.5).to(dev)
        b = torch.randn(64, generator=g).to(dev)
        wk = ops.pack_conv7x7s2_weights(w)
        x_cl = x.permute(0, 3, 1, 2)                                  # NCHW view of the channels-last memory
        w_cl = w.to(ops.h16()).contiguous(memory_format=torch.channels_last)
        b16 = b.to(ops.h16())
        flop = 2.0 * n * 48 * 48 * 64 * 384 * 49
        arms = {"conv7x7s2_umma": lambda: ops.conv7x7s2_umma(x, wk, b)}
        for bm in (False, True):
            def cudnn(bm=bm):
                torch.backends.cudnn.benchmark = bm
                return torch.cudnn_convolution_relu(x_cl, w_cl, b16, (2, 2), (3, 3), (1, 1), 1)
            arms[f"cudnn (benchmark={bm})"] = cudnn
        for name, fn in arms.items():
            ms = timed(fn)
            tf = flop / ms / 1e9
            row = {"crops": n, "arm": name, "ms": ms, "tflops": tf, "frac_of_989": tf / PEAK}
            res["rows"].append(row)
            print(f"n={n:4d} {name:26s} {ms:9.3f} ms  {tf:7.1f} TFLOP/s  {tf / PEAK:6.3f} of {PEAK:.0f}")
        torch.backends.cudnn.benchmark = False
        got = ops.conv7x7s2_umma(x, wk, b).float().permute(0, 3, 1, 2)
        want = torch.cudnn_convolution_relu(x_cl, w_cl, b16, (2, 2), (3, 3), (1, 1), 1).float()
        print(f"n={n:4d} max |kernel - cudnn| / max |cudnn| = {float((got - want).abs().max() / want.abs().max()):.2e}")
    if args.out:
        json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
