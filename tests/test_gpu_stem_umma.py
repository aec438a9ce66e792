"""GPU parity of the planner embedder's stem kernel (ops.conv7x7s2_umma, csrc/stem_umma.cu): the kernel against fp32
F.conv2d, and resnet18(num_channels=384) with the kernel against the same module on its cuDNN stem."""
import pytest
import torch
import torch.nn.functional as F

from lav_b200 import heads, ops, synth

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("shape", [(1, 96, 96, 384), (9, 96, 96, 384), (130, 96, 96, 384), (3, 50, 38, 64)])
def test_conv7x7s2_umma_vs_fp32_conv(cuda, shape):
    """bench crop shape at batch 1, 9 (batch-1 latency leg) and 130 (past one wave of tiles); (3, 50, 38, 64) has edge tiles
    on both axes, a non-square map and a single 64-channel K chunk."""
    n, h, w, cin = shape
    g = synth._gen(5, str(shape))
    x = torch.randn(n, h, w, cin, generator=g).to(cuda, ops.h16())
    wt = (torch.randn(64, cin, 7, 7, generator=g) / (49 * cin) ** 0.5).to(cuda)
    b = (torch.randn(64, generator=g) * 0.5).to(cuda)
    got = ops.conv7x7s2_umma(x, ops.pack_conv7x7s2_weights(wt), b).float()
    want = F.relu(F.conv2d(x.permute(0, 3, 1, 2).float(), wt.to(ops.h16()).float(), b, 2, 3)).permute(0, 2, 3, 1)
    assert got.shape == want.shape == (n, (h - 1) // 2 + 1, (w - 1) // 2 + 1, 64)
    err = float((got - want).abs().max() / want.abs().max())
    assert err < 2e-3, err


def _embedder(cuda):
    m = heads.resnet18(num_channels=384).eval()
    m.load_state_dict(synth.fill_state_dict_(m.state_dict()))
    return m.to(cuda).to(ops.h16()).to(memory_format=torch.channels_last)


def _both_stems(m, x):
    with torch.no_grad():
        try:
            heads.STEM_KERNEL = False
            want = m(x).float()
        finally:
            heads.STEM_KERNEL = True
        got = m(x).float()
    return got, want


def _rms(got, want):
    return float(((got - want) ** 2).mean().sqrt() / (want ** 2).mean().sqrt())


def test_resnet18_384_stem_kernel_matches_cudnn(cuda):
    m = _embedder(cuda)
    x = torch.randn(4, 384, 96, 96, generator=synth._gen(6, "emb")).to(cuda, ops.h16()).contiguous(memory_format=torch.channels_last)
    got, want = _both_stems(m, x)
    assert got.shape == want.shape == (4, 512, 3, 3)
    assert _rms(got, want) < 5e-3, _rms(got, want)    # both f16, different rounding points (cuDNN keeps BN folded in h16 weights)


def test_resnet18_384_stem_kernel_not_stale_after_step(cuda):
    """the packed stem lives in the fold cache: an optimizer step on the stem followed by eval() must be seen by the kernel."""
    m = _embedder(cuda)
    x = torch.randn(2, 384, 96, 96, generator=synth._gen(7, "emb")).to(cuda, ops.h16()).contiguous(memory_format=torch.channels_last)
    with torch.no_grad():
        before = m(x).float()
    m.train()
    opt = torch.optim.SGD(m.parameters(), lr=0.5)
    m(x).float().square().mean().backward()
    opt.step()
    m.eval()
    got, want = _both_stems(m, x)
    assert _rms(want, before) > 1e-2                   # the step moved the output
    assert _rms(got, want) < 5e-3, _rms(got, want)
