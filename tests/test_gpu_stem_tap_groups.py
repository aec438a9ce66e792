"""GPU: the planner stem (ops.conv7x7s2_umma) with shared pixel boxes.  The tile is column-major in shared memory, and the
taps of one kernel row with the same kx parity read one 19-column box, each from strided column kx // 2 on.

Compared with fp64 F.conv2d on h16-rounded operands (1e-3 of the output scale; the output is h16) at the bench crop with
1 and 9 crops, at the smallest legal image (the 19-column box covers it several times over), at odd and non-square sizes
with edge tiles on both axes, and at cin = 64 (one chunk) and 128.  Larger batches are covered by test_gpu_stem_umma.py.
"""
import pytest
import torch
import torch.nn.functional as F

from lav_b200 import ops, synth

pytestmark = pytest.mark.gpu


def q(x):
    return x.to(ops.h16()).double()


@pytest.mark.parametrize("shape", [(1, 96, 96, 384), (9, 96, 96, 384), (3, 7, 7, 64), (2, 49, 51, 64), (2, 33, 70, 128),
                                   (1, 70, 21, 64)])
def test_conv7x7s2_umma_tap_groups_fp64(cuda, shape):
    n, h, w, cin = shape
    g = synth._gen(46, f"stem_groups{shape}")
    x = q(torch.randn(n, h, w, cin, generator=g)).to(cuda)
    wt = q(torch.randn(64, cin, 7, 7, generator=g) / (49 * cin) ** 0.5).to(cuda)
    b = (torch.randn(64, generator=g) * 0.5).to(cuda)
    got = ops.conv7x7s2_umma(x.to(ops.h16()).contiguous(), ops.pack_conv7x7s2_weights(wt.float()), b).double()
    want = F.relu(F.conv2d(x.permute(0, 3, 1, 2), wt, b.double(), 2, 3)).permute(0, 2, 3, 1)
    assert got.shape == want.shape
    err = float((got - want).abs().max() / want.abs().max())
    del x, wt, got, want
    torch.cuda.empty_cache()
    assert err < 1e-3, err
