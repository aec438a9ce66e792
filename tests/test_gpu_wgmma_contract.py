"""GPU: the wgmma convolutions lavb_conv_umma, lavb_conv3x3_umma, lavb_conv7x7s2_umma and lavb_conv_pair_umma against their
whole C-ABI contract (include/lav_b200.h): the fp64 statements of tests/util.py on the operands as the kernels read them
(h16 values; tests/test_wgmma_ref_cpu.py ties them to F.conv2d / F.conv_transpose2d and shows that each plausible wrong
kernel lands at least 100 x these tolerances away at these inputs), within util.WGMMA_TOL of the output scale after the NaN
pattern and every infinity have matched exactly.  The tolerances are bounds the kernels must meet, not measured errors.

Outputs are filled beforehand with a NaN canary bit pattern and carry a spare image past the end; every element of the
documented slice and pixel lattice must be written and every other element must keep the canary bit for bit.  Every case
names the instantiation it reaches: conv_umma_kernel<cout_mma / 32>, the
conv_cmajor_kernel<KS, S, CO, SC> variants and conv_pair_umma_kernel<c>.

The instantiation is asserted in a fresh interpreter (test_instantiations_in_a_fresh_process reruns the value cases there with
tracing on): torch.profiler sessions in a process that has already run many of them can come back without kernel records, so
the in-process cases only compute and compare.

Refused calls change one field of a valid call each.  Out-of-range fields are built so that, were their check missing, the
call would still only touch the test's own canary arena (operands are views into the middle of it); misaligned pointers are
refused by checks that exist, so they reach no kernel either.
"""
import ctypes as C
import math
import os
import subprocess
import sys

import pytest
import torch

from lav_b200 import capi, ops, synth
from tests import util
from tests.util import INT, canary, is_canary, kernels

pytestmark = pytest.mark.gpu
TRACE = os.environ.get("LAVB_WGMMA_TRACE") == "1"
TOL = dict(util.WGMMA_TOL, stem=2e-3)


def odt(out):
    return torch.float32 if out == "f32" else ops.h16()


def bits(t):
    return t.contiguous().view(INT[t.dtype])


def assert_kernel(launched, name, count=1):
    names = [k[0].replace("(int)", "") for k in launched]
    assert len(names) == count and all(name in k for k in names), f"expected {count} x {name}, launched {names}"


def run_traced(fn, name, tmp_path):
    """fn(), one call of a wgmma entry on device operands.  Under LAVB_WGMMA_TRACE=1 (test_instantiations_in_a_fresh_process)
    also asserts, from the kernel records torch.profiler takes, that fn launched exactly one kernel, the instantiation `name`"""
    if TRACE:
        assert_kernel(kernels(fn, tmp_path), name)
    else:
        fn()
        torch.cuda.synchronize()


def assert_err(got, want, tol, what):
    err = util.wgmma_err(got, want)
    print(f"{what}: {err / tol:.3g} of the tolerance")
    assert err < tol, (what, err)


# ------------------------------------------------------------------------------------------------------------------ conv_umma
def umma_operands(c, cuda):
    """c's weights, bias, scale and shift on the device (None where the case has none)"""
    dev = lambda t: None if t is None else t.to(cuda)                      # noqa: E731
    return c.w.to(ops.h16()).to(cuda), dev(c.bias), dev(c.scale), dev(c.shift)


def umma_call(c, dev_ops, x, out, res):
    """one lavb_conv_umma call of case c on device operands only, so that a traced call launches nothing else"""
    w, b, sc, sh = dev_ops
    ops.conv_taps(x, c.cin, c.in_off, out, c.cout, c.out_off, c.hog, c.wog, c.in_s, (1, 1), (0, 0), c.taps, w, bias=b, scale=sc,
                  shift=sh, res=res, res_coff=c.res_off, pre_relu=c.pre, post_relu=c.post, sigmoid=c.sig, umma=True)


@pytest.mark.parametrize("name", list(util.UMMA_CASES))
def test_conv_umma_contract(cuda, tmp_path, name):
    c = util.UmmaCase(name, h16=ops.h16(), **util.UMMA_CASES[name])
    dt = odt(c.out)
    x = c.x.to(ops.h16()).to(cuda)
    res = None if c.res is None else c.res.to(ops.h16()).to(cuda)
    dev_ops = umma_operands(c, cuda)
    full = canary((c.n + 1, c.hog, c.wog, c.out_cs), dt, cuda)
    run_traced(lambda: umma_call(c, dev_ops, x, full[:c.n], res), f"conv_umma_kernel<{(c.cout + 31) // 32}>", tmp_path)
    sl = slice(c.out_off, c.out_off + c.cout)
    inside = torch.zeros(full.shape, dtype=torch.bool, device=cuda)
    inside[:c.n, ..., sl] = True
    assert torch.equal(~is_canary(full), inside), "written elements differ from the documented slice"
    assert_err(full[:c.n, ..., sl].cpu(), c.want(), TOL[c.out], name)


@pytest.mark.parametrize("name", list(util.UMMA_CONVT))
def test_conv_umma_transposed_phases(cuda, tmp_path, name):
    """ConvTranspose2d(k3, s2, p1) as four phase calls (out_s 2, out_o in {0, 1}^2, 1 / 2 / 2 / 4 taps) on the input's h x w
    grid into a channel slice of a wider map: after each call only that phase's lattice of the slice has changed (the odd
    phases' last row / column lies outside an odd hout / wout and is skipped); weight rows past cout hold NaN"""
    c = util.ConvTCase(name, h16=ops.h16(), **util.UMMA_CONVT[name])
    cs, off = c.cout + 16, 8
    x = c.x.to(ops.h16()).to(cuda)
    b, sc, sh = c.bias.to(cuda), c.scale.to(cuda), c.shift.to(cuda)
    full = canary((c.n + 1, c.hout, c.wout, cs), torch.float32, cuda)
    cm = (c.cout + 31) // 32 * 32
    for (py, px), taps, wp in c.phases:
        w = torch.full((len(taps), cm, c.cin), math.nan)
        w[:, :c.cout] = wp
        w = w.to(ops.h16()).to(cuda)
        before = bits(full).clone()
        run_traced(lambda: ops.conv_taps(x, c.cin, 0, full[:c.n], c.cout, off, c.h, c.w, (1, 1), (2, 2), (py, px), taps, w,
                                                 bias=b, scale=sc, shift=sh, post_relu=True, umma=True),
                   f"conv_umma_kernel<{cm // 32}>", tmp_path)
        lattice = torch.zeros(full.shape, dtype=torch.bool, device=cuda)
        lattice[:c.n, py::2, px::2, off:off + c.cout] = True
        changed = bits(full) != before
        assert torch.equal(changed, lattice), (py, px, int((changed & ~lattice).sum()), int((lattice & ~changed).sum()))
    assert_err(full[:c.n, ..., off:off + c.cout].cpu(), c.want(), TOL["f32"], name)


@pytest.mark.parametrize("no,hw,out_o", [(3, (25, 35), (0, 0)), (2, (25, 36), (0, 0)), (8, (26, 35), (0, 0)), (3, (26, 36), (1, 1))])
def test_conv_umma_depth_to_space_clipped(cuda, tmp_path, no, hw, out_o):
    """the d2s epilogue on 13 x 18 grids into maps that end inside a 2 x 2 block (odd hout and / or wout) or whose lattice is
    shifted by out_o = (1, 1): each of the four positions is clipped to hout x wout on its own, the rest written exactly once"""
    g = synth._gen(59, f"d2s{no}{hw}{out_o}")
    n, h, w, cin = 2, 13, 18, 64
    x = torch.randn(n, h, w, 2 * cin, generator=g).to(ops.h16())
    wt = (torch.randn(cin, no, 3, 3, generator=g) / (9 * cin) ** 0.5).to(ops.h16()).float()
    b = torch.randn(no, generator=g)
    b32 = torch.zeros(32)
    b32[:4 * no] = b.repeat(4)
    wu = util.pack_d2s(wt, no)
    v = util.tap_conv64(x[..., cin:].double(), [(0, 0), (0, 1), (1, 0), (1, 1)], wu, (1, 1), h, w) + b32.double()
    want, written = util.d2s_scatter64(v, no, *hw, out_o)
    xd, wd, bd = x.to(cuda), wu.to(ops.h16()).to(cuda), b32.to(cuda)
    full = canary((n + 1, *hw, no), torch.float32, cuda)
    run_traced(lambda: ops.conv_taps(xd, cin, cin, full[:n], 32, 0, h, w, (1, 1), (2, 2), out_o, [(0, 0), (0, 1), (1, 0), (1, 1)],
                                     wd, bias=bd, umma=True, d2s_nout=no), "conv_umma_kernel<1>", tmp_path)
    got_w = ~is_canary(full).cpu()
    assert not bool(got_w[n:].any()), "written past the end"
    assert torch.equal(got_w[:n], written), (int((got_w[:n] & ~written).sum()), int((written & ~got_w[:n]).sum()))
    assert_err(full[:n].cpu()[written], want[written], TOL["f32"], f"d2s {no} {hw}")


def test_conv_umma_inplace_residual(cuda):
    """out may be res element for element (h16, same stride and offset): the result is the out-of-place one, bit for bit"""
    c = util.UmmaCase("inplace", h16=ops.h16(), cout=64, res=True, res_cs=96, res_off=16, out="h16", post=True)
    c.out_cs, c.out_off = 96, 16
    x = c.x.to(ops.h16()).to(cuda)
    res = c.res.to(ops.h16()).to(cuda)
    dev_ops = umma_operands(c, cuda)
    sep = canary((c.n, c.hog, c.wog, 96), ops.h16(), cuda)
    umma_call(c, dev_ops, x, sep, res)
    inplace = res.clone()
    umma_call(c, dev_ops, x, inplace, inplace)
    torch.cuda.synchronize()
    assert torch.equal(bits(inplace[..., 16:80]), bits(sep[..., 16:80]))
    assert torch.equal(bits(inplace[..., :16]), bits(res[..., :16])) and torch.equal(bits(inplace[..., 80:]), bits(res[..., 80:]))
    assert_err(sep[..., 16:80].cpu(), c.want(), TOL["h16"], "in place")


# ------------------------------------------------------------------------------------------------------------- conv3x3_umma
# (cin, cout, stride) -> the conv_cmajor_kernel<KS, S, CO, SC> instantiation lavb_conv3x3_umma launches for it
CMAJOR = {(64, 64, 1): "3, 1, 64, 1", (128, 64, 1): "3, 1, 64, 2", (64, 128, 1): "3, 1, 128, 1", (128, 128, 1): "3, 1, 128, 2",
          (64, 64, 2): "3, 2, 64, 1", (64, 128, 2): "3, 2, 128, 1", (384, 256, 1): "3, 1, 128, 1", (128, 256, 2): "3, 2, 128, 1"}


def _nan_inf_image(g, n, h, w, cin, nan, inf):
    x = torch.randn(n, h, w, cin, generator=g)
    if nan:
        x[n - 1, h // 2, w // 3, 5] = math.nan
    if inf:
        x[0, 1, w - 2, 7] = math.inf
        x[n - 1, h - 1, 2, cin - 4] = -math.inf
    return x.to(ops.h16())


@pytest.mark.parametrize("pre", [False, True])
@pytest.mark.parametrize("special", ["nan", "inf", "none"])
@pytest.mark.parametrize("cin,cout,stride", list(CMAJOR))
def test_conv3x3_umma_contract(cuda, tmp_path, cin, cout, stride, special, pre):
    """every instantiation on a 2-image 19 x 37 map (ragged tiles) with bias and an affine of mixed sign, with and without the
    pre-ReLU, clean and with one NaN pixel or two infinite pixels: the NaN pattern is the receptive field without the ReLU
    (none with it), infinities are stored as +-65504"""
    g = synth._gen(60, f"c3{cin}{cout}{stride}{special}{pre}")
    n, h, w = 2, 19, 37
    x = _nan_inf_image(g, n, h, w, cin, special == "nan", special == "inf")
    wt = (torch.randn(9, cout, cin, generator=g) / (9 * cin) ** 0.5).to(ops.h16())
    b, sc, sh = torch.randn(cout, generator=g), torch.rand(cout, generator=g) + 0.5, torch.randn(cout, generator=g)
    sc[::3] *= -1
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    a = util.tap_conv64(x.double(), util._taps(3, 1), wt.double(), (stride, stride), ho, wo)
    want = util.store64(util.wgmma_epilogue64(a, b, sc, sh, None, pre), "h16")
    full = canary((n + 1, ho, wo, cout), ops.h16(), cuda)
    dev = [t.to(cuda) for t in (x, wt, b, sc, sh)]
    run_traced(lambda: ops.conv3x3_umma(dev[0], dev[1], cout, stride, *dev[2:], pre, out=full[:n]),
               f"conv_cmajor_kernel<{CMAJOR[(cin, cout, stride)]}>", tmp_path)
    assert not bool(is_canary(full[:n]).any()) and bool(is_canary(full[n:]).all())
    assert bool(torch.isnan(want).any()) == (special == "nan" and not pre)
    assert_err(full[:n].cpu(), want, TOL["h16"], f"conv3x3 {cin}->{cout} s{stride} {special} pre={pre}")


@pytest.mark.parametrize("special", ["nan", "inf"])
@pytest.mark.parametrize("cin", [64, 128])
def test_conv7x7s2_umma_nan_inf(cuda, tmp_path, cin, special):
    """the stem's ReLU turns a NaN into 0 (no output is NaN); an infinite pixel gives +inf or 0, stored as 65504 or 0"""
    g = synth._gen(61, f"stem{cin}{special}")
    n, h, w = 2, 23, 30
    x = _nan_inf_image(g, n, h, w, cin, special == "nan", special == "inf")
    wt = (torch.randn(64, cin, 7, 7, generator=g) / (49 * cin) ** 0.5).to(ops.h16())
    b = torch.randn(64, generator=g) * 0.5
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    a = util.tap_conv64(x.double(), util._taps(7, 3), wt.double().permute(2, 3, 0, 1).reshape(49, 64, cin), (2, 2), ho, wo)
    want = util.store64(util.wgmma_epilogue64(a, b, pre=True), "h16")
    full = canary((n + 1, ho, wo, 64), ops.h16(), cuda)
    xd, wp, bd = x.to(cuda), ops.pack_conv7x7s2_weights(wt.to(cuda)), b.to(cuda)
    run_traced(lambda: ops.conv7x7s2_umma(xd, wp, bd, out=full[:n]), "conv_cmajor_kernel<7, 2, 64, 1>", tmp_path)
    assert not bool(is_canary(full[:n]).any()) and bool(is_canary(full[n:]).all())
    assert not bool(torch.isnan(full[:n].float()).any())
    assert_err(full[:n].cpu(), want, TOL["stem"], f"stem {cin} {special}")


# ------------------------------------------------------------------------------------------------------------- conv_pair_umma
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("special", ["res_nan", "x_nan", "x_inf"])
@pytest.mark.parametrize("c", [64, 128])
def test_conv_pair_umma_nan_inf(cuda, tmp_path, c, special, relu):
    """one NaN pixel in the residual stays NaN without the ReLU and is 0 with it, on both residual paths; a NaN input pixel
    is stopped by the inner ReLU (0); an infinite one saturates the inner h16 store at 65504"""
    g = synth._gen(62, f"pair{c}{special}{relu}")
    n, h, w, dil = 2, 6, 32, 2
    q = lambda t: t.to(ops.h16())                                           # noqa: E731
    x = _nan_inf_image(g, n, h, w, c, special == "x_nan", special == "x_inf")
    w1, w2 = (q(torch.randn(3, c, c, generator=g) / (3 * c) ** 0.5) for _ in range(2))
    b1, t2 = torch.randn(c, generator=g) * 0.1, torch.randn(c, generator=g) * 0.1
    r = torch.randn(n, h, w, c, generator=g)
    if special == "res_nan":
        r[1, 3, 5, 9] = math.nan
    r = q(r)
    want = util.pair_ref64(x.double(), w1.double(), b1, w2.double(), t2, dil, r.double(), relu, h16=ops.h16())
    full = canary((n + 1, h, w, c), ops.h16(), cuda)
    dev = [t.to(cuda) for t in (x, w1, b1, w2, t2, r)]
    run_traced(lambda: ops.conv_pair_umma(*dev[:5], dil, res=dev[5], post_relu=relu, out=full[:n]), f"conv_pair_umma_kernel<{c}>",
               tmp_path)
    assert not bool(is_canary(full[:n]).any()) and bool(is_canary(full[n:]).all())
    assert bool(torch.isnan(want).any()) == (special == "res_nan" and not relu)
    assert_err(full[:n].cpu(), want, TOL["pair"], f"pair {c} {special} relu={relu}")


def test_conv_pair_umma_needs_dense_bias(cuda):
    """bias1 / shift2 are read as c dense floats: a strided view is refused rather than read wrong"""
    c = 64
    x = torch.zeros(1, 2, 32, c, device=cuda).to(ops.h16())
    wz = torch.zeros(3, c, c, device=cuda).to(ops.h16())
    strided = torch.zeros(2 * c, device=cuda)[::2]
    dense = torch.zeros(c, device=cuda)
    for b1, t2 in ((strided, dense), (dense, strided)):
        with pytest.raises(capi.LavbError):
            ops.conv_pair_umma(x, wz, b1, wz, t2, 1)


# ------------------------------------------------------------------------------------------------------ batch independence
def test_batch_independence(cuda):
    """image k alone equals image k of a batch of 3, bit for bit, on conv_umma, conv3x3_umma, conv7x7s2_umma and the pair"""
    g = synth._gen(63, "batch")
    q = lambda t: t.to(ops.h16()).to(cuda)                                  # noqa: E731
    x = q(torch.randn(3, 21, 37, 128, generator=g))
    b, sc, sh = (torch.randn(128, generator=g).to(cuda) for _ in range(3))
    w9 = q(torch.randn(9, 128, 128, generator=g) / 34)
    w49 = q(torch.randn(49, 64, 128, generator=g) / 80)
    wp = q(torch.randn(3, 128, 128, generator=g) / 20)
    r = q(torch.randn(3, 21, 37, 128, generator=g))
    xp, rp = q(torch.randn(3, 5, 64, 128, generator=g)), q(torch.randn(3, 5, 64, 128, generator=g))
    taps = util._taps(3, 1)
    calls = {
        "conv_umma": lambda xi, ri: ops.conv_taps(xi, 128, 0, torch.empty(xi.shape[0], 21, 37, 128, device=cuda), 128, 0, 21, 37, (1, 1),
                                                  (1, 1), (0, 0), taps, w9, b, sc, sh, ri, 0, True, True, umma=True),
        "conv3x3_umma": lambda xi, ri: ops.conv3x3_umma(xi, w9, 128, 2, b, sc, sh, True),
        "conv7x7s2_umma": lambda xi, ri: ops.conv7x7s2_umma(xi, w49, b[:64].contiguous()),
        "conv_pair_umma": lambda xi, ri: ops.conv_pair_umma(xi, wp, b, wp, sh, 3, res=ri),
    }
    for name, f in calls.items():
        xs, rs = (xp, rp) if name == "conv_pair_umma" else (x, r)
        whole = f(xs, rs)
        for k in range(3):
            one = f(xs[k:k + 1].contiguous(), rs[k:k + 1].contiguous())
            torch.cuda.synchronize()
            assert torch.equal(bits(one[0]), bits(whole[k])), (name, k)


# -------------------------------------------------------------------------------------------------------------- rejections
class Arena:
    """one canary buffer per dtype; every operand of a rejection case is a view into its middle, so that a call whose check
    were missing would still only touch the arena"""

    def __init__(self, cuda, elems=1 << 20):
        self.f = canary((elems,), torch.float32, cuda)
        self.h = canary((elems,), ops.h16(), cuda)
        self.mid = elems // 2

    def at(self, dtype, shape, off=0):
        buf = self.f if dtype == torch.float32 else self.h
        n = math.prod(shape)
        return buf[self.mid + off:self.mid + off + n].view(shape)

    def snapshot(self):
        torch.cuda.synchronize()
        self.before = (bits(self.f).clone(), bits(self.h).clone())

    def intact(self):
        """nothing in the arena changed since snapshot()"""
        return torch.equal(bits(self.f), self.before[0]) and torch.equal(bits(self.h), self.before[1])


def _umma_desc(ar, cuda):
    """a valid lavb_conv_umma call: 1 x 8 x 8 x 64 h16 input, one tap, cout 32 fp32 output with an h16 residual and a bias"""
    x, r = ar.at(ops.h16(), (1, 8, 8, 64), -1 << 17), ar.at(ops.h16(), (1, 8, 8, 32), 1 << 17)
    w = ar.at(ops.h16(), (1, 32, 64), 1 << 18)
    w.zero_()
    b = torch.zeros(32, device=cuda)
    out = ar.at(torch.float32, (1, 8, 8, 32))
    d = capi.ConvDesc()
    d.inp, d.in_dtype, d.n, d.hin, d.win, d.cin, d.in_cstride, d.in_coff = x.data_ptr(), capi.lib().lavb_h16_dtype(), 1, 8, 8, 64, 64, 0
    d.out, d.out_dtype, d.hout, d.wout, d.cout, d.out_cstride, d.out_coff = out.data_ptr(), capi.F32, 8, 8, 32, 32, 0
    d.hog, d.wog, d.in_sy, d.in_sx, d.out_sy, d.out_sx, d.out_oy, d.out_ox = 8, 8, 1, 1, 1, 1, 0, 0
    d.ntaps = 1
    d.w, d.bias = w.data_ptr(), b.data_ptr()
    d.res, d.res_dtype, d.res_cstride, d.res_coff = r.data_ptr(), capi.lib().lavb_h16_dtype(), 32, 0
    return d, (x, r, w, b, out)


UMMA_REJECT = {
    "ntaps0": dict(ntaps=0), "ntaps17": dict(ntaps=17), "cin0": dict(cin=0), "cin32": dict(cin=32), "cout0": dict(cout=0),
    "cout12": dict(cout=12), "cout264": dict(cout=264), "in_f32": dict(in_dtype=0), "out_dtype_bad": dict(out_dtype=99),
    "in_coff_neg": dict(in_coff=-8), "in_coff4": dict(in_coff=4), "in_slice_past": dict(in_coff=8),
    "out_coff_neg": dict(out_coff=-8), "out_cstride36": dict(out_cstride=36), "out_slice_past": dict(out_coff=8),
    "res_coff_neg": dict(res_coff=-8), "res_slice_past": dict(res_coff=8), "res_cstride24": dict(res_cstride=24),
    "res_f32": dict(res_dtype=0), "res_cout40": dict(cout=40, out_cstride=40),
    "n0": dict(n=0), "hog0": dict(hog=0), "wog_neg": dict(wog=-1), "hin0": dict(hin=0), "win_neg": dict(win=-8),
    "hout0": dict(hout=0), "wout_neg": dict(wout=-1),
    "in_sy0": dict(in_sy=0), "in_sx9": dict(in_sx=9), "out_sy0": dict(out_sy=0), "out_sx_neg": dict(out_sx=-1),
    "out_oy_neg": dict(out_oy=-1), "out_ox_neg": dict(out_ox=-2), "scale_without_shift": dict(scale="bias"),
    "null_in": dict(inp=None), "null_out": dict(out=None), "null_w": dict(w=None),
    "out_8B_offset": dict(out=8), "res_8B_offset": dict(res=8), "bias_misaligned": dict(bias=2),
    "out_overlaps_in": dict(out="x"), "out_overlaps_w": dict(out="w"), "out_f32_is_res": dict(res="out"),
    "d2s_cout64": dict(d2s_nout=2, cout=64, out_cstride=64, res=None), "d2s_nout9": dict(d2s_nout=9, res=None),
    "d2s_out_s1": dict(d2s_nout=2, res=None), "d2s_with_res": dict(d2s_nout=2, out_sy=2, out_sx=2),
}


@pytest.mark.parametrize("name", list(UMMA_REJECT))
def test_conv_umma_rejects(cuda, name):
    """each check refuses before launch (LavbError) and nothing in the arena changes; the unchanged call is accepted"""
    ar = Arena(cuda)
    d, keep = _umma_desc(ar, cuda)
    ar.snapshot()
    named = dict(x=keep[0], w=keep[2], bias=keep[3])
    for k, v in UMMA_REJECT[name].items():
        if isinstance(v, str):
            setattr(d, k, getattr(d, "out") if v == "out" else named[v].data_ptr())
        elif k in ("inp", "out", "res", "w", "bias") and v is not None:
            setattr(d, k, getattr(d, k) + v)                  # a byte offset from the aligned base
        else:
            setattr(d, k, v)
    with pytest.raises(capi.LavbError):
        capi.check(capi.lib().lavb_conv_umma(C.byref(d), ops._stream()), "lavb_conv_umma")
    torch.cuda.synchronize()
    assert ar.intact()
    d, keep = _umma_desc(ar, cuda)
    capi.check(capi.lib().lavb_conv_umma(C.byref(d), ops._stream()), "lavb_conv_umma")
    torch.cuda.synchronize()
    assert not bool(is_canary(keep[4]).any())


def _cmajor_call(ar, cuda, which, ch):
    """a valid lavb_conv3x3_umma (1 x 16 x 16 x 64 -> 64, stride 1) or lavb_conv7x7s2_umma (1 x 16 x 16 x 64 -> 8 x 8 x 64) call
    with one field changed: -> (return code, output view)"""
    lib = capi.lib()
    x = ar.at(ops.h16(), (1, 16, 16, 64), -1 << 17)
    w = ar.at(ops.h16(), (49 if which == "7x7" else 9, 64, 64), 1 << 17)
    w.zero_()
    b = torch.zeros(64 + 4, device=cuda)
    ho = 8 if which == "7x7" else 16
    out = ar.at(ops.h16(), (1, ho, ho, 64))
    ptr = dict(x=x.data_ptr(), w=w.data_ptr(), b=b.data_ptr(), out=out.data_ptr())
    for k in ("x", "w", "b", "out"):
        v = ch.get(k)
        if isinstance(v, str):
            ptr[k] = ptr[v]
        elif isinstance(v, int):
            ptr[k] += v
        elif k in ch:
            ptr[k] = None
    n, h, wd, cin = ch.get("n", 1), ch.get("h", 16), ch.get("wd", 16), ch.get("cin", 64)
    vp = lambda k: C.c_void_p(ptr[k])                                      # noqa: E731
    torch.cuda.synchronize()
    if which == "7x7":
        code = lib.lavb_conv7x7s2_umma(vp("x"), n, h, wd, cin, vp("w"), vp("b"), vp("out"), ops._stream())
    else:
        sc = vp("b") if ch.get("scale_only") else C.c_void_p(0)
        code = lib.lavb_conv3x3_umma(vp("x"), n, h, wd, cin, ch.get("stride", 1), vp("w"), ch.get("cout", 64), vp("b"), sc, C.c_void_p(0),
                                     1, vp("out"), ops._stream())
    torch.cuda.synchronize()
    return code, out


CMAJOR_REJECT = {
    "3x3": {"null_in": dict(x=None), "null_out": dict(out=None), "n_neg": dict(n=-1), "h0": dict(h=0), "stride3": dict(stride=3),
            "cin96": dict(cin=96), "cout96": dict(cout=96), "scale_without_shift": dict(scale_only=True),
            "out_8B_offset": dict(out=8), "bias_misaligned": dict(b=2), "out_overlaps_in": dict(out="x"),
            "out_overlaps_w": dict(out="w"), "out_overlaps_bias": dict(b="out"), "tiles_2_31": dict(n=1 << 30, cout=256)},
    "7x7": {"null_bias": dict(b=None), "n_neg": dict(n=-1), "h6": dict(h=6), "cin32": dict(cin=32), "out_8B_offset": dict(out=8),
            "bias_misaligned": dict(b=2), "out_overlaps_in": dict(out="x"), "out_overlaps_w": dict(out="w"),
            "tiles_2_31": dict(n=(1 << 31) - 1, h=48, wd=16)},
}


@pytest.mark.parametrize("which,name", [(k, n) for k, v in CMAJOR_REJECT.items() for n in v])
def test_conv3x3_conv7x7s2_umma_rejects(cuda, which, name):
    ar = Arena(cuda)
    _cmajor_call(ar, cuda, which, dict(n=0))                 # the operands in place (n = 0 writes nothing)
    ar.snapshot()
    code, _ = _cmajor_call(ar, cuda, which, CMAJOR_REJECT[which][name])
    assert code != 0
    if name.startswith("tiles"):
        assert "2^31 tiles" in capi.lib().lavb_last_error().decode()
    assert ar.intact()
    code, out = _cmajor_call(ar, cuda, which, {})
    assert code == 0 and not bool(is_canary(out).any())


def _pair_call(ar, cuda, ch):
    """a valid lavb_conv_pair_umma call (2 x 4 x 32 x 64, dilation 1, residual) with one field changed"""
    x, r = ar.at(ops.h16(), (2, 4, 32, 64), -1 << 17), ar.at(ops.h16(), (2, 4, 32, 64), 1 << 17)
    w = ar.at(ops.h16(), (3, 64, 64), 1 << 18)
    w.zero_()
    b = torch.zeros(64 + 4, device=cuda)
    out = ar.at(ops.h16(), (2, 4, 32, 64))
    d = capi.ConvPairDesc()
    d.inp, d.out, d.res = x.data_ptr(), out.data_ptr(), r.data_ptr()
    d.n, d.h, d.w, d.c, d.dil, d.post_relu = 2, 4, 32, 64, 1, 1
    d.w1, d.bias1, d.w2, d.shift2 = w.data_ptr(), b.data_ptr(), w.data_ptr(), b.data_ptr()
    for k, v in ch.items():
        if isinstance(v, str):
            setattr(d, k, dict(x=x, r=r)[v].data_ptr())
        elif k in ("bias1", "shift2") and v is not None:
            setattr(d, k, getattr(d, k) + v)
        else:
            setattr(d, k, v)
    code = capi.lib().lavb_conv_pair_umma(C.byref(d), ops._stream())
    torch.cuda.synchronize()
    return code, out


PAIR_REJECT = {"c96": dict(c=96), "w48": dict(w=48), "dil0": dict(dil=0), "dil_w": dict(dil=32), "n_neg": dict(n=-1), "h0": dict(h=0),
               "null_bias1": dict(bias1=None), "null_w2": dict(w2=None), "bias1_misaligned": dict(bias1=2),
               "shift2_misaligned": dict(shift2=2), "out_overlaps_in": dict(out="x"), "out_overlaps_res": dict(out="r"),
               "tiles_2_31": dict(n=1 << 30, h=8)}


@pytest.mark.parametrize("name", list(PAIR_REJECT))
def test_conv_pair_umma_rejects(cuda, name):
    ar = Arena(cuda)
    _pair_call(ar, cuda, dict(n=0))                          # the operands in place (n = 0 writes nothing)
    ar.snapshot()
    code, _ = _pair_call(ar, cuda, PAIR_REJECT[name])
    assert code != 0
    if name.startswith("tiles"):
        assert "2^31 tiles" in capi.lib().lavb_last_error().decode()
    assert ar.intact()
    code, out = _pair_call(ar, cuda, {})
    assert code == 0 and not bool(is_canary(out).any())


# ------------------------------------------------------------------------------------------------------------ instantiations
def test_instantiations_in_a_fresh_process(cuda):
    """every value case above again, in a new interpreter with LAVB_WGMMA_TRACE=1: each call launches exactly the kernel
    instantiation its case names (conv_umma_kernel<cout_mma / 32>, conv_cmajor_kernel<KS, S, CO, SC>, conv_pair_umma_kernel<c>)"""
    cases = "not rejects and not fresh_process and not inplace and not dense_bias and not batch_independence"
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", os.path.abspath(__file__), "-k", cases],
                       cwd=util.ROOT, env={**os.environ, "LAVB_WGMMA_TRACE": "1", "PYTHONDONTWRITEBYTECODE": "1"},
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert " passed" in r.stdout and " failed" not in r.stdout, r.stdout[-2000:]
