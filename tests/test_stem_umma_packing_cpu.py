"""Host-side logic of the planner embedder's stem kernel (no GPU): the [tap][cout][cin] layout of ops.pack_conv7x7s2_weights and
the kernel's tile addressing (csrc/stem_umma.cu), restated in numpy, reproduce conv 7x7 / stride 2 / pad 3."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from lav_b200 import ops

TILE = 16     # kTile of csrc/stem_umma.cu


def emulate(x, wk):
    """numpy restatement of conv7x7s2_umma_kernel's K loop without bias / ReLU: per 16 x 16 output tile and K-block (tap t,
    chunk kc), B[pixel (py, px)][k] = x[2 (oy0 + py) - 3 + t // 7, 2 (ox0 + px) - 3 + t % 7, 64 kc + k] (zero outside the image,
    as TMA fills), A[cout][k] = wk[t, cout, 64 kc + k], D[cout][pixel] += A @ B.T."""
    n, h, w, cin = x.shape
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    out = np.zeros((n, ho, wo, 64), np.float64)
    for img in range(n):
        for oy0 in range(0, ho, TILE):
            for ox0 in range(0, wo, TILE):
                d = np.zeros((64, TILE * TILE))
                for t in range(49):
                    ky, kx = t // 7, t % 7
                    iy = 2 * (oy0 + np.arange(TILE)) - 3 + ky
                    ix = 2 * (ox0 + np.arange(TILE)) - 3 + kx
                    ok = (iy[:, None] >= 0) & (iy[:, None] < h) & (ix[None, :] >= 0) & (ix[None, :] < w)
                    for kc in range(cin // 64):
                        px = x[img, np.clip(iy, 0, h - 1)][:, np.clip(ix, 0, w - 1), 64 * kc:64 * kc + 64]   # (16, 16, 64)
                        b = np.where(ok[..., None], px, 0).reshape(TILE * TILE, 64)
                        d += wk[t, :, 64 * kc:64 * kc + 64] @ b.T
                for n_ in range(TILE * TILE):
                    oy, ox = oy0 + n_ // TILE, ox0 + n_ % TILE
                    if oy < ho and ox < wo:
                        out[img, oy, ox] = d[:, n_]
    return out


@pytest.mark.parametrize("shape", [(1, 9, 13, 64), (2, 37, 20, 128)])
def test_stem_umma_packing_and_tiling(shape):
    n, h, w, cin = shape
    rng = np.random.default_rng(1)
    x = rng.standard_normal(shape).astype(np.float32)
    wt = torch.from_numpy(rng.standard_normal((64, cin, 7, 7)).astype(np.float32) * 0.05)
    wk = ops.pack_conv7x7s2_weights(wt)
    assert tuple(wk.shape) == (49, 64, cin) and wk.dtype == ops.h16() and wk.is_contiguous()
    wq = wk.float().numpy()
    wr = wt.to(ops.h16()).float().numpy()
    for t in (0, 6, 7, 24, 48):
        assert np.array_equal(wq[t], wr[:, :, t // 7, t % 7])     # tap t = ky * 7 + kx, rows = cout, K = cin contiguous
    got = emulate(x.astype(np.float64), wq.astype(np.float64))
    ref = F.conv2d(torch.from_numpy(x).permute(0, 3, 1, 2).double(), torch.from_numpy(wr).double(), None, 2, 3)
    ref = ref.permute(0, 2, 3, 1).numpy()
    assert got.shape == ref.shape
    assert np.abs(got - ref).max() < 1e-9 * max(1.0, np.abs(ref).max())
