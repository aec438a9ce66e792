"""A/B timing of the product's conv_umma layers (and the fused ERFNet pairs of conv_pair_umma) at bench shapes (B = 32 frames
per agent group) for two builds of liblavb200.so, and of the two wgmma kernels of the 3x3 BEV convolutions in one build.

    python scripts/conv_umma_ab.py [--base-lib OTHER/liblavb200.so] [--rounds 5] [--reps 10]

Both libraries are loaded into one process; the rounds alternate base / this tree's build on the same inputs and weights.
For every layer it prints the median kernel time (CUDA events over `reps` back-to-back launches), the GEMM rate and its
fraction of the 989 TFLOP/s dense fp16 peak, whether the two builds' outputs are bit-identical (else the largest difference
relative to the output's scale), and byte counts derived from the shapes:
  smem KB  : shared-memory operand bytes the MMAs read per 64-deep K-block of one CTA (conv_umma: 128 pixels x cout_mma)
  fill KB  : bytes the TMA moves from L2 into shared memory per tile (conv_umma: one A and one B box per tap and chunk;
             stem: one pixel box per tap (base) -> one per kernel row and kx parity (this tree))
  fill TB/s: all tiles' fill bytes of this tree over its median time
The planner stem (conv7x7s2_umma, 128 and 9 crops of 96 x 96 x 384) is timed the same way, and so is every shape of the fused
ERFNet pair a tick runs; the last line sums the pair times at their launch counts per tick.
The base build runs every layer on the kernels it has (layers.cmajor_wins off), whatever this tree routes elsewhere.

Kernel arm (this build only, always run): every 3x3 / pad-1 BEV layer on conv_umma_kernel (pixels in M, 8 x 16 tiles) and on
lavb_conv3x3_umma (output channels in M, 16 x 16 tiles), alternating, with the same columns; fill KB/tile is per 256 output
pixels for both (two conv_umma tiles, one conv3x3 tile per 128-channel CTA column).
The card name, power limit and SM clocks are read in the same run.
"""
import argparse
import ctypes
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from lav_b200 import capi, layers as L, ops
from lav_b200.layers import TapConv

PEAK = 989e12


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


KERNEL_ARM = []   # (name, TapConv, input, GEMM flop) of the layers lavb_conv3x3_umma can run


def layers(dev, B):
    """(name, run() -> output, GEMM flop, cout_mma, [(cin, ntaps, tiles) per launch] or None for the pair kernel,
    or ("stem", crops, cin, tiles))"""
    g = torch.Generator(device=dev).manual_seed(0)
    rn = lambda *s: torch.randn(*s, device=dev, generator=g)
    h16 = ops.h16()
    out = []

    def tap(name, n, hin, win, cin, cout, k, stride=1, pad=1, transposed=False, opad=0, **kw):
        wshape = (cin, cout, k, k) if transposed else (cout, cin, k, k)
        layer = TapConv(rn(*wshape) * (2.0 / (cin * k * k)) ** 0.5, transposed, stride, pad, 1, opad, **kw)
        x = rn(n, hin, win, cin).to(h16)
        ho, wo = layer.out_size(hin, win)
        y = torch.empty(n, ho, wo, cout, device=dev, dtype=h16)
        fl = 0
        for ph in layer.phases:
            (osy, osx), (ooy, oox) = ph["out_s"], ph["out_o"]
            fl += 2 * n * ((ho - ooy + osy - 1) // osy) * ((wo - oox + osx - 1) // osx) * cin * len(ph["taps"]) * layer.cout
        tiles = lambda ph: n * -(-((ho - ph["out_o"][0] + ph["out_s"][0] - 1) // ph["out_s"][0]) // 8) * \
            -(-((wo - ph["out_o"][1] + ph["out_s"][1] - 1) // ph["out_s"][1]) // 16)
        out.append((name, lambda: layer(x, out=y), fl, (cout + 31) // 32 * 32,
                    [(cin, len(ph["taps"]), tiles(ph)) for ph in layer.phases]))
        if layer.cmajor_ok:
            KERNEL_ARM.append((name, layer, x, fl))

    bn = lambda c: dict(pre_relu=True, scale=rn(c).abs() + 0.5, shift=rn(c) * 0.1)
    tap("heads 384->256 160x160", B, 160, 160, 384, 256, 3, **bn(256))
    tap("bb 64->64 s1 160x160", B, 160, 160, 64, 64, 3, **bn(64))
    tap("bb 64->64 s2 320->160", B, 320, 320, 64, 64, 3, stride=2, **bn(64))
    tap("bb 128->128 s1 80x80", B, 80, 80, 128, 128, 3, **bn(128))
    tap("bb 64->128 s2 160->80", B, 160, 160, 64, 128, 3, stride=2, **bn(128))
    tap("bb 128->128 s2 80->40", B, 80, 80, 128, 128, 3, stride=2, **bn(128))
    tap("bb 128->128 s1 40x40", B, 40, 40, 128, 128, 3, **bn(128))
    tap("erf down 64->64 s2 72x64", 3 * B, 72, 64, 64, 64, 3, stride=2, bias=rn(64) * 0.1, scale=rn(64).abs() + 0.5,
        shift=rn(64) * 0.1, post_relu=True)
    tap("erf up 128->64 36x32", 3 * B, 36, 32, 128, 64, 3, stride=2, transposed=True, opad=1, bias=rn(64) * 0.1,
        scale=rn(64).abs() + 0.5, shift=rn(64) * 0.1, post_relu=True)
    tap("erf up 64->16 72x64", 3 * B, 72, 64, 64, 16, 3, stride=2, transposed=True, opad=1, bias=rn(16) * 0.1,
        scale=rn(16).abs() + 0.5, shift=rn(16) * 0.1, post_relu=True)

    # the four head output layers: 2x2-tap GEMMs over the 64-channel slices of the heads conv output, depth-to-space epilogue
    hid = rn(B, 160, 160, 256).to(h16)
    heads = []
    for gi, no in enumerate((2, 2, 2, 3)):
        wu = (rn(4, 32, 64) * 0.1).to(h16).contiguous()
        b32 = torch.zeros(32, device=dev)
        b32[:4 * no] = rn(no).repeat(4) * 0.1
        heads.append((gi, no, wu, b32, torch.empty(B, 320, 320, no, device=dev)))

    def d2s():
        for gi, no, wu, b32, o in heads:
            ops.conv_taps(hid, 64, 64 * gi, o, 32, 0, 160, 160, (1, 1), (2, 2), (0, 0), [(0, 0), (0, 1), (1, 0), (1, 1)], wu,
                          bias=b32, sigmoid=gi == 3, umma=True, d2s_nout=no)
        return torch.cat([h[4].flatten() for h in heads])

    out.append(("head outputs 4x(64->32 2x2 d2s)", d2s, 4 * 2 * B * 160 * 160 * 64 * 4 * 32, 32,
                [(64, 4, B * 20 * 10)] * 4))

    # the planner embedder's 7x7 / s2 stem: 4 crops per agent (ego + K = 3 vehicles) -> 128 crops, and the batch-1 leg's 9
    def stem(name, crops):
        x = rn(crops, 96, 96, 384).to(h16)
        wp = ops.pack_conv7x7s2_weights(rn(64, 384, 7, 7) / (49 * 384) ** 0.5)
        b = rn(64) * 0.1
        y = torch.empty(crops, 48, 48, 64, device=dev, dtype=h16)
        out.append((name, lambda: ops.conv7x7s2_umma(x, wp, b, out=y), 2 * crops * 48 * 48 * 64 * 384 * 49, 64,
                    ("stem", crops, 384, crops * 9)))

    stem(f"planner stem {4 * B} crops 96x96x384", 4 * B)
    stem("planner stem 9 crops 96x96x384", 9)

    # the fused ERFNet (3x1 -> 1x3) pairs (conv_pair_umma_kernel), every shape a tick runs, with its launch count per tick:
    # each non_bottleneck_1d block is a dilation-1 pair without the residual, then a dilation-d pair with it
    for c, h, w, dil, res, count in PAIR_SHAPES:
        x = rn(3 * B, h, w, c).to(h16)
        r = rn(3 * B, h, w, c).to(h16) if res else None
        w1, w2 = ((rn(3, c, c) / (3 * c) ** 0.5).to(h16).contiguous() for _ in range(2))
        b1, t2 = rn(c) * 0.1, rn(c) * 0.1
        y = torch.empty(3 * B, h, w, c, device=dev, dtype=h16)
        out.append((pair_name(c, h, w, dil, res, count),
                    lambda x=x, r=r, w1=w1, w2=w2, b1=b1, t2=t2, y=y, dil=dil: ops.conv_pair_umma(x, w1, b1, w2, t2, dil, res=r, out=y),
                    2 * 2 * 3 * B * h * w * c * c * 3, c, None))
    return out


# (c, h, w, dilation, residual, launches per tick): 7 blocks of 64 channels at 72 x 64, 8 of 128 channels at 36 x 32
PAIR_SHAPES = [(64, 72, 64, 1, False, 7), (64, 72, 64, 1, True, 7), (128, 36, 32, 1, False, 8),
               (128, 36, 32, 2, True, 2), (128, 36, 32, 4, True, 2), (128, 36, 32, 8, True, 2), (128, 36, 32, 16, True, 2)]


def pair_name(c, h, w, dil, res, count):
    return f"erf pair {c} {h}x{w} d{dil}{' +res' if res else ''} x{count}"


def fill_bytes_per_tile(cin, ntaps, cout_mma):
    """TMA bytes from L2 into shared memory for one 8 x 16 tile of conv_umma: per 64-channel chunk and tap one A box of
    8 x 16 pixels x 128 B and one B box of cout_mma x 128 B"""
    return cin // 64 * ntaps * (8 * 16 * 128 + cout_mma * 128)


def stem_fill_bytes_per_tile(cin, grouped):
    """the same for one 16 x 16 tile of conv7x7s2_umma: 49 weight boxes of 8 KB plus 49 pixel boxes of 16 x 16 x 128 B
    (one per tap) or 14 of 19 x 16 x 128 B (one per kernel row and kx parity)"""
    return cin // 64 * (49 * 8192 + (14 * 19 if grouped else 49 * 16) * 16 * 128)


def kblock_bytes(cout_mma, old_width=32):
    """(smem operand bytes per K-block with one wgmma per `old_width` columns, with one full-width wgmma, L2 -> SM bytes)"""
    a_per_wgmma = 64 * 16 * 2                      # one warpgroup's 64 x 16 A fragment
    b = 2 * 4 * cout_mma * 16 * 2                  # 2 warpgroups x 4 K16 steps x the whole B slice
    old = 2 * 4 * max(1, cout_mma // old_width) * a_per_wgmma + b
    return old, 2 * 4 * a_per_wgmma + b, 128 * 128 + cout_mma * 128


def cmajor_fill_bytes_per_tile(cin, cout, stride):
    """TMA bytes from L2 into shared memory for one 16 x 16 tile of lavb_conv3x3_umma and one CTA column of min(cout, 128)
    channels: per chunk and kernel row `stride` pixel boxes of 16 rows x (18 or 17) columns x 128 B, per tap and chunk one
    weight box of that column's channels x 128 B"""
    cols = 18 if stride == 1 else 17
    return cin // 64 * (3 * stride * cols * 16 * 128 + 9 * min(cout, 128) * 128)


def kernel_arm(rounds, reps):
    """conv_umma_kernel against lavb_conv3x3_umma on every 3x3 BEV layer, in this build"""
    med = lambda v: sorted(v)[len(v) // 2]
    span = lambda v: f"{med(v):.3f} [{min(v):.3f}-{max(v):.3f}]"
    print(f"\n{'layer (conv_umma vs conv3x3_umma)':34s} {'conv_umma ms':>24s} {'conv3x3 ms':>24s} {'TF/s':>7s} {'TF/s':>7s} "
          f"{'/989':>5s} {'speedup':>7s} {'bitwise':>8s} {'fill KB/256px':>14s} {'fill TB/s':>10s}")
    for name, layer, x, fl in KERNEL_ARM:
        n, h, w, cin = x.shape
        ho, wo = layer.out_size(h, w)
        s = layer.stride[0]
        ph = layer.phases[0]
        ya = torch.empty(n, ho, wo, layer.cout, device=x.device, dtype=x.dtype)
        yb = torch.empty_like(ya)
        arms = {
            "umma": lambda: ops.conv_taps(x, cin, 0, ya, layer.cout, 0, ho, wo, (s, s), (1, 1), (0, 0), ph["taps"], ph["w_umma"],
                                          layer.bias, layer.scale, layer.shift, pre_relu=layer.pre_relu, umma=True),
            "cmajor": lambda: ops.conv3x3_umma(x, ph["w_umma"], layer.cout, s, layer.bias, layer.scale, layer.shift, layer.pre_relu,
                                               out=yb),
        }
        for f in arms.values():
            f(); f()
        torch.cuda.synchronize()
        same = bool(torch.equal(ya, yb))
        diff = "same" if same else f"{float((ya.float() - yb.float()).abs().max() / ya.float().abs().max()):.1e}"
        t = {k: [] for k in arms}
        for _ in range(rounds):
            for k, f in arms.items():
                t[k].append(time_ms(f, reps))
        ncol = max(1, layer.cout // 128)
        f_umma = 2 * fill_bytes_per_tile(cin, 9, layer.cout)
        f_cm = ncol * cmajor_fill_bytes_per_tile(cin, layer.cout, s)
        tiles_cm = n * -(-ho // 16) * -(-wo // 16)
        rate = tiles_cm * f_cm / (med(t["cmajor"]) * 1e-3) / 1e12
        print(f"{name:34s} {span(t['umma']):>24s} {span(t['cmajor']):>24s} {fl / med(t['umma']) / 1e9:7.1f} "
              f"{fl / med(t['cmajor']) / 1e9:7.1f} {fl / (med(t['cmajor']) * 1e-3) / PEAK:5.2f} "
              f"{med(t['umma']) / med(t['cmajor']):7.3f} {diff:>8s} {f'{f_umma // 1024}->{f_cm // 1024}':>14s} {rate:10.2f}")


def time_ms(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base-lib", help="liblavb200.so of the tree to compare against (without it: the kernel arm only)")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("conv_umma_ab.py needs a CUDA device")
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(f"device: {torch.cuda.get_device_name(dev)} | nvidia-smi name, power limit, SM clock, max SM clock: {q}")
    ls = layers(dev, args.batch)
    kernel_arm(args.rounds, args.reps)
    if not args.base_lib:
        return
    new_path = capi.LIB_PATH
    libs = {"base": load(os.path.abspath(args.base_lib)), "this": load(new_path)}
    wins = L.cmajor_wins

    def use(k):                                   # the base build has no lavb_conv3x3_umma: keep its layers on conv_umma
        capi._lib = libs[k]
        L.cmajor_wins = wins if k == "this" else (lambda *a: False)
    times = {(n, k): [] for n, *_ in ls for k in libs}
    same = {}
    for name, run, *_ in ls:                      # warm up both builds on every shape; compare their outputs
        res = {}
        for k in libs:
            use(k)
            for _ in range(2):
                y = run()
            torch.cuda.synchronize()
            res[k] = y.clone()
        same[name] = (bool(torch.equal(res["base"], res["this"])),
                      float((res["base"].float() - res["this"].float()).abs().max() / res["base"].float().abs().max()))
    for _ in range(args.rounds):
        for name, run, *_ in ls:
            for k in libs:
                use(k)
                times[(name, k)].append(time_ms(run, args.reps))
    use("this")
    med = lambda v: sorted(v)[len(v) // 2]
    span = lambda v: f"{med(v):.3f} [{min(v):.3f}-{max(v):.3f}]"
    print(f"{'layer':34s} {'base ms [min-max]':>24s} {'this ms [min-max]':>24s} {'base TF/s':>9s} {'this TF/s':>9s} {'/989':>5s} "
          f"{'speedup':>7s} {'bitwise':>8s} {'smem KB':>7s} {'fill KB/tile':>13s} {'fill TB/s':>9s}")
    for name, run, fl, cm, launches in ls:
        tb, tt = times[(name, "base")], times[(name, "this")]
        diff = "same" if same[name][0] else f"{same[name][1]:.1e}"
        if launches is None:                       # fused pair kernel: no tap boxes
            s_new, fill, rate = kblock_bytes(cm, 64)[1] // 1024, "-", "-"
        elif launches[0] == "stem":
            _, crops, cin, tiles = launches
            f0, f1 = stem_fill_bytes_per_tile(cin, False), stem_fill_bytes_per_tile(cin, True)
            s_new, fill, rate = (8192 + 16384) * 2 // 1024, f"{f0 // 1024}->{f1 // 1024}", f"{tiles * f1 / (med(tt) * 1e-3) / 1e12:.2f}"
        else:
            s_new = kblock_bytes(cm)[1] // 1024
            f1 = [fill_bytes_per_tile(ci, nt, cm) for ci, nt, _ in launches]
            total = sum(f * t for f, (*_, t) in zip(f1, launches))
            fill = f"{f1[0] // 1024}" + ("" if len(set(f1)) == 1 else f" ({len(f1)} launches)")
            rate = f"{total / (med(tt) * 1e-3) / 1e12:.2f}"
        print(f"{name:34s} {span(tb):>24s} {span(tt):>24s} {fl / med(tb) / 1e9:9.1f} {fl / med(tt) / 1e9:9.1f} "
              f"{fl / (med(tt) * 1e-3) / PEAK:5.2f} {med(tb) / med(tt):7.3f} {diff:>8s} {s_new:7d} {fill:>13s} {rate:>9s}")
    # all pair launches of one tick: each round's per-shape times weighted by the launch counts, median over rounds
    tick = {k: [sum(s[5] * times[(pair_name(*s), k)][r] for s in PAIR_SHAPES) for r in range(args.rounds)] for k in libs}
    print(f"{'erf pairs, one tick (' + str(sum(s[5] for s in PAIR_SHAPES)) + ' launches)':34s} {span(tick['base']):>24s} "
          f"{span(tick['this']):>24s} {'':9s} {'':9s} {'':5s} {med(tick['base']) / med(tick['this']):7.3f}")


if __name__ == "__main__":
    main()
