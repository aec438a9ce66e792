"""Per-tile pipeline timing of lavb_conv_pair_umma from its clock64 trace (lavb_conv_pair_set_trace): where a CTA's tile period goes."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from lav_b200 import ops, capi

def run(n, h, w, c, dil, use_res, tiles=16):
    g = torch.Generator().manual_seed(1)
    x = torch.randn(n, h, w, c, generator=g).to(ops.h16()).cuda()
    w1 = (torch.randn(3, c, c, generator=g) / (3 * c) ** 0.5).to(ops.h16()).cuda()
    w2 = (torch.randn(3, c, c, generator=g) / (3 * c) ** 0.5).to(ops.h16()).cuda()
    b1, t2 = torch.randn(c, generator=g).cuda() * 0.1, torch.randn(c, generator=g).cuda() * 0.1
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctas = 2 * sms if c == 64 else sms
    buf = torch.zeros(ctas * tiles * 8, dtype=torch.int64, device="cuda")
    for _ in range(3):
        ops.conv_pair_umma(x, w1, b1, w2, t2, dil, res=x if use_res else None)
    capi.lib().lavb_conv_pair_set_trace(buf.data_ptr(), tiles)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    ops.conv_pair_umma(x, w1, b1, w2, t2, dil, res=x if use_res else None)
    e1.record()
    torch.cuda.synchronize()
    capi.lib().lavb_conv_pair_set_trace(None, 0)
    t = buf.cpu().numpy().reshape(ctas, tiles, 8).astype(np.float64)
    ntile = n * ((h + 128 // w - 1) // (128 // w))
    per_cta = ntile / ctas
    ok = (t[:, :, 3] > 0) & (t[:, :, 0] > 0)
    it = min(int(per_cta) - 1, tiles - 1)
    sel = slice(1, max(2, it))                      # steady-state iterations
    d = lambda a, b: np.nanmean(np.where(ok[:, sel], t[:, sel, a] - t[:, sel, b], np.nan))
    period = np.nanmean(np.where(ok[:, sel][:, 1:], t[:, sel, 0][:, 1:] - t[:, sel, 0][:, :-1], np.nan))
    print(f"c={c} {n}x{h}x{w} dil={dil} res={use_res}: launch {e0.elapsed_time(e1) * 1e3:.1f} us, {per_cta:.1f} tiles/CTA, tile period {period:.0f} cyc")
    print(f"   epilogue warp: E1 (acc1 ready -> mid written) {d(1, 0):.0f} | wait stage 2 (mid written -> acc2 ready) {d(2, 1):.0f} | "
          f"E2 (acc2 ready -> stored) {d(3, 2):.0f} | next acc1 wait {period - d(3, 0):.0f}")
    print(f"   MMA thread: stage-1(next) issued -> mid_full seen {d(5, 4):.0f} | mid_full -> stage-2 issued+committed {d(6, 5):.0f} | "
          f"epilogue's mid_full arrive -> MMA sees it {d(5, 1):.0f} | stage-2 commit -> epilogue sees acc2 {d(2, 6):.0f}")

B = int(sys.argv[1]) if len(sys.argv) > 1 else 32
run(3 * B, 72, 64, 64, 1, False)
run(3 * B, 72, 64, 64, 1, True)
run(3 * B, 36, 32, 128, 2, True)
