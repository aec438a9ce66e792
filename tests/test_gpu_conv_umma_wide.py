"""GPU: conv_umma at the MMA widths that run one CTA per SM (cout > 128; in the product the fused 384 -> 256 heads conv), at the
tile counts a persistent grid of 132 CTAs meets at its edges: a single tile, fewer tiles than CTAs, an odd count above the grid,
and a count that is not a multiple of twice the grid; plus stride 2 and an output channel slice with a residual slice.

Each case compares with fp64 F.conv2d on h16-rounded operands (2e-5 of the output scale with fp32 output, 1e-3 with h16 output).
The output buffer is filled with a NaN bit pattern first; every element inside the written slice must be replaced and every
element outside it (other channels, a spare image past the end) must keep it.
"""
import pytest
import torch
import torch.nn.functional as F

from lav_b200 import ops, synth

pytestmark = pytest.mark.gpu

CANARY = {torch.float32: (torch.int32, 0x7FC0DEAD), torch.float16: (torch.int16, 0x7E5A), torch.bfloat16: (torch.int16, 0x7FDA)}

# (n, h, w) -> tiles of 8 x 16 output pixels: n * ceil(h / 8) * ceil(w / 16)
CASES = {
    "tiles1": dict(shape=(1, 8, 16)),                              # 1 tile
    "tiles3": dict(shape=(3, 5, 13)),                              # 3 ragged tiles
    "tiles135": dict(shape=(5, 24, 140)),                          # 5 x 3 x 9: odd, above the grid
    "tiles300": dict(shape=(4, 40, 240)),                          # 4 x 5 x 15: 300 = 2 x 132 + 36
    "stride2": dict(shape=(3, 37, 67), stride=2),                  # 3 x 3 x 3 tiles of a stride-2 conv, ragged
    "slices_res": dict(shape=(2, 21, 50), out_cs=384, out_off=64, res_cs=320, res_off=32),
}


def q(x):
    return x.to(ops.h16()).double()


@pytest.mark.parametrize("cout", [160, 256])
@pytest.mark.parametrize("name", list(CASES))
def test_conv_umma_wide(cuda, name, cout):
    cfg = CASES[name]
    (n, h, w), s, cin = cfg["shape"], cfg.get("stride", 1), 64
    out_cs, out_off = cfg.get("out_cs", cout), cfg.get("out_off", 0)
    res_cs, res_off = cfg.get("res_cs", cout), cfg.get("res_off", 0)
    g = synth._gen(37, f"wide{name}{cout}")
    x = q(torch.randn(n, h, w, cin, generator=g)).to(cuda)
    wt = q(torch.randn(cout, cin, 3, 3, generator=g) / (9 * cin) ** 0.5).to(cuda)
    b = torch.randn(cout, generator=g).to(cuda)
    sc = (torch.rand(cout, generator=g) + 0.5).to(cuda)
    sh = torch.randn(cout, generator=g).to(cuda)
    a = F.conv2d(x.permute(0, 3, 1, 2), wt, None, s, 1).permute(0, 2, 3, 1)
    ho, wo = a.shape[1:3]
    rbuf = q(torch.randn(n, ho, wo, res_cs, generator=g)).to(cuda)
    want = F.relu(F.relu(a + b.double()) * sc.double() + sh.double() + rbuf[..., res_off:res_off + cout])
    wu = wt.permute(2, 3, 0, 1).reshape(9, cout, cin).to(ops.h16()).contiguous()      # cout % 32 == 0: no padding rows
    taps = [(ky - 1, kx - 1) for ky in range(3) for kx in range(3)]
    for odt, tol in ((torch.float32, 2e-5), (ops.h16(), 1e-3)):
        it, bits = CANARY[odt]
        full = torch.empty((n + 1, ho, wo, out_cs), dtype=odt, device=cuda)
        full.view(it).fill_(bits)
        ops.conv_taps(x.to(ops.h16()).contiguous(), cin, 0, full[:n], cout, out_off, ho, wo, (s, s), (1, 1), (0, 0), taps, wu,
                      bias=b, scale=sc, shift=sh, res=rbuf.to(ops.h16()).contiguous(), res_coff=res_off, pre_relu=True,
                      post_relu=True, umma=True)
        torch.cuda.synchronize()
        canary = full.view(it) == bits
        inside = torch.zeros(full.shape, dtype=torch.bool, device=cuda)
        inside[:n, ..., out_off:out_off + cout] = True
        assert not bool(canary[inside].any()), f"{int(canary[inside].sum())} outputs never written ({odt})"
        assert bool(canary[~inside].all()), f"{int((~canary)[~inside].sum())} elements written outside the slice ({odt})"
        got = full[:n, ..., out_off:out_off + cout].double()
        err = float((got - want).abs().max() / want.abs().max())
        assert err < tol, (odt, err)
