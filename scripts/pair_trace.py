"""Per-tile pipeline timing of lavb_conv_pair_umma from its clock64 trace (lavb_conv_pair_set_trace): where a CTA's tile period goes.

    python scripts/pair_trace.py [B]

Thread 0 of each CTA stamps, per tile iteration: [0] stage-1 accumulators ready, [1] `mid` written (end of epilogue 1),
[2] stage-2 accumulators ready, [3] tile stored (end of epilogue 2).  Printed per shape, in SM clocks, averaged over the
steady-state iterations of all CTAs:
  S1 wait : end of the previous tile's epilogue 2 -> this tile's stage-1 accumulators ready
  E1      : epilogue 1 (bias, ReLU, three shifted copies of `mid`, two barriers)
  S2      : stage-2 MMAs (from `mid` written to accumulators ready)
  E2      : epilogue 2 (shift, residual, ReLU, store)
  period  : stamp [0] of one tile to stamp [0] of the next
"""
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
    r = x.clone() if use_res else None
    y = torch.empty_like(x)
    for _ in range(3):
        ops.conv_pair_umma(x, w1, b1, w2, t2, dil, res=r, out=y)
    buf = torch.zeros(2 * torch.cuda.get_device_properties(0).multi_processor_count * tiles * 8, dtype=torch.int64, device="cuda")
    capi.lib().lavb_conv_pair_set_trace(buf.data_ptr(), tiles)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    ops.conv_pair_umma(x, w1, b1, w2, t2, dil, res=r, out=y)
    e1.record()
    torch.cuda.synchronize()
    capi.lib().lavb_conv_pair_set_trace(None, 0)
    t = buf.cpu().numpy().reshape(-1, tiles, 8).astype(np.float64)
    t = t[t[:, 0, 0] > 0]                            # the CTAs the launch had
    ctas = t.shape[0]
    ntile = n * -(-h // (128 // w))
    per_cta = ntile / ctas
    it = min(int(per_cta), tiles)
    ok = (t[:, :it, 3] > 0) & (t[:, :it, 0] > 0)
    t = np.where(ok[:, :, None], t[:, :it], np.nan)
    mean = lambda v: float(np.nanmean(v[:, 1:]))      # iteration 0 carries the prologue
    s1 = mean(np.concatenate([np.full((ctas, 1), np.nan), t[:, 1:, 0] - t[:, :-1, 3]], 1))
    period = mean(np.concatenate([np.full((ctas, 1), np.nan), t[:, 1:, 0] - t[:, :-1, 0]], 1))
    print(f"c={c} {n}x{h}x{w} dil={dil} res={use_res}: launch {e0.elapsed_time(e1) * 1e3:.1f} us, {ctas} CTAs, "
          f"{per_cta:.2f} tiles/CTA | S1 wait {s1:.0f} | E1 {mean(t[:, :, 1] - t[:, :, 0]):.0f} | "
          f"S2 {mean(t[:, :, 2] - t[:, :, 1]):.0f} | E2 {mean(t[:, :, 3] - t[:, :, 2]):.0f} | period {period:.0f} cyc")


B = int(sys.argv[1]) if len(sys.argv) > 1 else 32
print(f"device: {torch.cuda.get_device_name(0)}")
run(3 * B, 72, 64, 64, 1, False)
run(3 * B, 72, 64, 64, 1, True)
run(3 * B, 36, 32, 128, 1, False)
for d in (2, 4, 8, 16):
    run(3 * B, 36, 32, 128, d, True)
