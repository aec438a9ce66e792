"""GPU: the CUDA-core tap convolution lavb_conv_taps and its helper kernels (lavb_deconv3x3s2_small, lavb_pool2_affine_relu,
lavb_rgb_normalize, lavb_convert) against their whole C-ABI contract (include/lav_b200.h), called through ops / capi directly
so that every descriptor field is set here rather than by TapConv.

lavb_conv_taps picks one of four bodies from the descriptor: conv_c16_mma_kernel (16-bit input, cin 16, <= 9 taps),
conv_small_kernel (cin <= 16), and conv_taps_kernel with 128 x 64 tiles (cout_pad % 64 == 0) or 256 x 16 tiles.  Every case
names the body it is meant to reach and asserts, from the kernel names torch.profiler records, that it did.  The reference is
fp64 F.conv2d / F.conv_transpose2d on the operands as the kernel reads them (16-bit inputs and residuals rounded, and the c16
body's weights rounded to the 16-bit type, as the header states), within 2e-5 of the output scale for fp32 output and 1e-3 for
16-bit output.  These tolerances are bounds the kernels must meet, not measured errors.  Outputs are filled beforehand with a
NaN canary bit pattern and carry a spare image past the end; every element of the documented slice and pixel lattice must be
written and every other element must keep the canary bit for bit.

Misaligned or out-of-range arguments appear only in cases the entry points refuse before launching anything, or (pool2,
convert) route to their element-wise bodies.
"""
import ctypes as C
import math
import os

import pytest
import torch
import torch.nn.functional as F

from lav_b200 import capi, ops, synth
from tests.util import INT, canary, is_canary, kernels

pytestmark = pytest.mark.gpu

CNAME = {torch.float32: "float", torch.float16: "__half", torch.bfloat16: "__nv_bfloat16"}
TOL = {torch.float32: 2e-5, torch.float16: 1e-3, torch.bfloat16: 1e-2}


def dt(code):
    return torch.float32 if code == "f" else ops.h16()


def bits(t):
    return t.contiguous().view(INT[t.dtype])


def q(x):
    return x.to(ops.h16()).double()


def nhwc(t):
    return t.permute(0, 2, 3, 1)


def nchw(t):
    return t.permute(0, 3, 1, 2)


def fmax0(a):
    """fmaxf(a, 0.f): a NaN comes out as 0 (torch.relu would keep it)"""
    return torch.where(torch.isnan(a), torch.zeros_like(a), a.clamp_min(0))


def num_sms():
    """the SM count lavb sizes its grids with: the device's, capped by LAVB_NUM_SMS when that is set"""
    n = torch.cuda.get_device_properties(0).multi_processor_count
    cap = int(os.environ.get("LAVB_NUM_SMS", "0") or 0)
    return cap if 0 < cap < n else n


def body_name(body, in_dt, out_dt, ntaps, cin):
    if body == "c16":
        return f"conv_c16_mma_kernel<{CNAME[out_dt]}, {3 if ntaps <= 3 else 4 if ntaps <= 4 else 9}>"
    if body == "small":
        return f"conv_small_kernel<{CNAME[in_dt]}, {CNAME[out_dt]}, {4 if cin <= 4 else 16}>"
    tile = "128, 64, 8, 2" if body == "gemm64" else "256, 16, 8, 1"
    return f"conv_taps_kernel<{CNAME[in_dt]}, {CNAME[out_dt]}, {tile}>"


def assert_body(launched, name, count=1):
    hits = [k for k in launched if name in k[0]]
    assert len(hits) == count and len(launched) == count, f"expected {count} x {name}, launched {launched}"
    return hits


def pack(wt, taps_of):
    """(cout, cin, kh, kw) weight -> (ntaps, cin, cout_pad16) fp32, tap t = ky * kw + kx; the padding columns hold NaN, which
    must never reach a stored channel"""
    cout, cin, kh, kw = wt.shape
    cp = (cout + 15) // 16 * 16
    w = torch.full((kh * kw, cin, cp), float("nan"), dtype=torch.float32, device=wt.device)
    w[:, :, :cout] = wt.permute(2, 3, 1, 0).reshape(kh * kw, cin, cout).float()
    return taps_of(kh, kw), w.contiguous()


def epilogue(a, b, sc, sh, r, pre, post, sig):
    if b is not None:
        a = a + b.double()
    if pre:
        a = fmax0(a)
    if sc is not None:
        a = a * sc.double() + sh.double()
    if r is not None:
        a = a + r
    if post:
        a = fmax0(a)
    if sig:
        a = torch.sigmoid(a)
    return a


def assert_close(got, want, tol, what=""):
    g, w = got.double(), want.double()
    nan_w = torch.isnan(w)
    assert torch.equal(torch.isnan(g), nan_w), f"{what}: NaN where the reference has {int(nan_w.sum())} NaN, got {int(torch.isnan(g).sum())}"
    if bool((~nan_w).any()):
        scale = float(w[~nan_w].abs().max()) or 1.0
        err = float((g - w)[~nan_w].abs().max()) / scale
        assert err < tol, f"{what}: error {err:.3e} of the output scale > {tol}"


class Conv:
    """one Conv2d (kh x kw, stride, padding, dilation) as a tap list: seeded operands, the fp64 reference and the call"""

    def __init__(self, cuda, body, in_dt="h", out_dt="h", n=2, hw=(11, 13), cin=16, cout=32, k=(3, 3), pad=(1, 1), dil=1,
                 stride=1, in_cs=None, in_off=0, out_cs=None, out_off=0, res=True, res_cs=None, res_off=0, bias=True, affine=True,
                 pre=True, post=True, sig=False, nan_at=None, seed=""):
        self.cuda, self.body = cuda, body
        self.in_dt, self.out_dt = dt(in_dt), dt(out_dt)
        self.n, (h, w), self.cin, self.cout = n, hw, cin, cout
        self.in_off, self.out_off, self.res_off = in_off, out_off, res_off
        self.in_cs, self.out_cs = in_cs or cin, out_cs or cout
        self.pre, self.post, self.sig, self.stride = pre, post, sig, stride
        g = synth._gen(51, f"taps:{body}:{seed}")
        kh, kw = k
        x = torch.randn(n, h, w, self.in_cs, generator=g)
        if nan_at is not None:
            x[nan_at[0], nan_at[1], nan_at[2], in_off + 1] = float("nan")
        self.x = x.to(self.in_dt).to(cuda)
        wt = (torch.randn(cout, cin, kh, kw, generator=g) / (cin * kh * kw) ** 0.5).to(cuda)
        self.taps, self.w = pack(wt, lambda kh_, kw_: [(ky * dil - pad[0], kx * dil - pad[1]) for ky in range(kh_) for kx in range(kw_)])
        self.b = torch.randn(cout, generator=g).to(cuda) if bias else None
        self.sc = (torch.rand(cout, generator=g) + 0.5).to(cuda) if affine else None
        self.sh = torch.randn(cout, generator=g).to(cuda) if affine else None
        self.ho = (h + 2 * pad[0] - dil * (kh - 1) - 1) // stride + 1
        self.wo = (w + 2 * pad[1] - dil * (kw - 1) - 1) // stride + 1
        self.r = (torch.randn(n, self.ho, self.wo, res_cs or cout, generator=g).to(self.out_dt).to(cuda) if res else None)
        self.wt64 = q(wt) if body == "c16" else wt.double()      # the c16 body multiplies by 16-bit weights
        self.conv_args = dict(stride=stride, padding=pad, dilation=dil)
        self.nan_at = nan_at

    def conv64(self, wt64):
        x = self.x[..., self.in_off:self.in_off + self.cin].double()
        if self.nan_at is None:
            return nhwc(F.conv2d(nchw(x), wt64, None, **self.conv_args))
        # NaN outputs are exactly those whose receptive field holds the NaN pixel (computed apart, so that the fp64
        # convolution's algorithm cannot spread the NaN)
        nan = torch.isnan(x)
        a = nhwc(F.conv2d(nchw(torch.where(nan, torch.zeros_like(x), x)), wt64, None, **self.conv_args))
        hit = nhwc(F.conv2d(nchw(nan.any(-1, keepdim=True).double()), torch.ones_like(wt64[:1, :1]), None, **self.conv_args)) > 0.5
        return torch.where(hit, torch.full_like(a, float("nan")), a)

    def want(self, wt64=None):
        r = None if self.r is None else self.r[..., self.res_off:self.res_off + self.cout].double()
        return epilogue(self.conv64(self.wt64 if wt64 is None else wt64), self.b, self.sc, self.sh, r, self.pre, self.post, self.sig)

    def call(self, x, out, r):
        ops.conv_taps(x, self.cin, self.in_off, out, self.cout, self.out_off, self.ho, self.wo, (self.stride, self.stride), (1, 1),
                      (0, 0), self.taps, self.w, self.b, self.sc, self.sh, r, self.res_off, self.pre, self.post, self.sig)

    def run(self, tmp_path, n_kernels=1):
        """one call into a canary buffer with a spare image: the launched kernels, and the written slice"""
        self.full = canary((self.n + 1, self.ho, self.wo, self.out_cs), self.out_dt, self.cuda)
        launched = kernels(lambda: self.call(self.x, self.full[:self.n], self.r), tmp_path)
        hits = assert_body(launched, body_name(self.body, self.in_dt, self.out_dt, len(self.taps), self.cin), n_kernels)
        sl = slice(self.out_off, self.out_off + self.cout)
        got = self.full[:self.n, ..., sl]
        written = ~is_canary(self.full)
        inside = torch.zeros_like(written)
        inside[:self.n, ..., sl] = True
        assert bool(written[inside].all()), f"{int((~written[inside]).sum())} outputs of the slice never written"
        assert not bool(written[~inside].any()), f"{int(written[~inside].sum())} elements written outside the slice"
        return got, hits

    def check(self, tmp_path):
        got, hits = self.run(tmp_path)
        assert_close(got, self.want(), TOL[self.out_dt], f"{self.body} {self.in_dt}->{self.out_dt}")
        return got, hits


# ---------------------------------------------------------------------------------------------------------- conv_taps cases
H, FL = "h", "f"
CASES = {
    # every body x every dtype pair, full epilogue with a residual, 11 x 13 maps (no tile multiple), n = 2
    **{f"c16_{i}{o}": dict(body="c16", in_dt=i, out_dt=o, cin=16, cout=32) for i, o in ((H, H), (H, FL))},
    **{f"small_{i}{o}": dict(body="small", in_dt=i, out_dt=o, cin=12, cout=24) for i, o in ((H, H), (H, FL), (FL, H), (FL, FL))},
    **{f"gemm64_{i}{o}": dict(body="gemm64", in_dt=i, out_dt=o, cin=32, cout=64) for i, o in ((H, H), (H, FL), (FL, H), (FL, FL))},
    **{f"gemm16_{i}{o}": dict(body="gemm16", in_dt=i, out_dt=o, cin=32, cout=40) for i, o in ((H, H), (H, FL), (FL, H), (FL, FL))},
    # c16 tap counts: 3 (1 x 3), 4 (2 x 2), 5 (1 x 5, the 9-slot body part full), 9 with stride 2; odd cout
    "c16_taps3": dict(body="c16", out_dt=FL, k=(1, 3), pad=(0, 1)),
    "c16_taps4": dict(body="c16", k=(2, 2), pad=(0, 0)),
    "c16_taps5": dict(body="c16", out_dt=FL, k=(1, 5), pad=(0, 2), cout=13),
    "c16_taps9_s2": dict(body="c16", stride=2, hw=(17, 23), cout=40),
    "c16_cout13": dict(body="c16", cout=13, res=False),
    # small: cin 4, 8, 12 and three 16-column chunks
    **{f"small_cin{c}": dict(body="small", in_dt=FL, out_dt=FL, cin=c, cout=40) for c in (4, 8, 12)},
    # the 256 x 16 GEMM: three column blocks (cout 40, above), the scalar epilogue (cout 13); the 128 x 64 GEMM at 128, 192
    "gemm16_cout13": dict(body="gemm16", in_dt=FL, out_dt=FL, cin=32, cout=13),
    "gemm16_cout13_h": dict(body="gemm16", cin=32, cout=13),
    "gemm64_cout128": dict(body="gemm64", in_dt=FL, out_dt=FL, cin=48, cout=128),
    "gemm64_cout192": dict(body="gemm64", cin=32, cout=192, hw=(9, 15)),
    # the tap table's maximum, a 4 x 4 kernel: GEMM, small on fp32 and on the 16-bit cin-16 input the c16 body declines
    "taps16_gemm64": dict(body="gemm64", in_dt=FL, out_dt=FL, cin=32, cout=64, k=(4, 4), pad=(1, 2)),
    "taps16_gemm16": dict(body="gemm16", cin=20, cout=24, k=(4, 4), pad=(2, 1)),
    "taps16_small": dict(body="small", in_dt=FL, out_dt=FL, cin=8, cout=24, k=(4, 4), pad=(1, 1)),
    "taps16_small_h16": dict(body="small", out_dt=FL, cin=16, cout=24, k=(4, 4), pad=(1, 1)),
    "taps10_small_h16": dict(body="small", cin=16, cout=16, k=(2, 5), pad=(1, 2)),
    "taps12_gemm16": dict(body="gemm16", in_dt=FL, out_dt=H, cin=24, cout=16, k=(3, 4), pad=(1, 1)),
}
# descriptor fields on every body: channel slices of wider buffers (an unaligned output slice as well), dilated taps, stride 2
for _b, _base in (("c16", dict(cin=16, cout=24)), ("small", dict(cin=8, cout=24, in_dt=FL)), ("gemm64", dict(cin=32, cout=64)),
                  ("gemm16", dict(cin=32, cout=24, in_dt=FL))):
    CASES[f"{_b}_slices"] = dict(body=_b, **_base, in_cs=_base["cin"] + 24, in_off=12, out_cs=_base["cout"] + 40, out_off=20,
                                 res_cs=_base["cout"] + 16, res_off=8)
    CASES[f"{_b}_out_off3"] = dict(body=_b, **_base, out_dt=FL, out_cs=_base["cout"] + 7, out_off=3, res_cs=_base["cout"] + 6, res_off=5)
    CASES[f"{_b}_concat"] = dict(body=_b, **_base, out_cs=_base["cout"] + 16, out_off=0, res=False)      # DownsamplerBlock's concat
    CASES[f"{_b}_dil2"] = dict(body=_b, **_base, dil=2, pad=(2, 2), hw=(13, 17))
    CASES[f"{_b}_s2"] = dict(body=_b, **_base, stride=2, hw=(15, 21), out_dt=FL)
    # the epilogue: each step alone and in combinations (null bias, null scale/shift, no residual)
    for _name, _epi in (("plain", dict(bias=False, affine=False, res=False, pre=False, post=False)),
                        ("bias", dict(affine=False, res=False, pre=False, post=False)),
                        ("affine", dict(bias=False, res=False, pre=False, post=False)),
                        ("pre", dict(bias=False, affine=False, res=False, post=False)),
                        ("res_post", dict(bias=False, affine=False, pre=False)),
                        ("sigmoid", dict(post=False, sig=True)),
                        ("pre_post_no_bias", dict(bias=False, affine=False))):
        CASES[f"{_b}_epi_{_name}"] = dict(body=_b, **_base, **_epi)


@pytest.mark.parametrize("name", list(CASES))
def test_conv_taps_descriptor(cuda, tmp_path, name):
    Conv(cuda, seed=name, **CASES[name]).check(tmp_path)


def test_c16_rounds_its_weights(cuda, tmp_path):
    """the c16 body multiplies by the weights rounded to the 16-bit type (header): with weights that are not representable
    it matches the rounded-weight reference and misses the fp32-weight one; the same layer with 10 taps (small body) uses
    the fp32 weights"""
    c = Conv(cuda, "c16", out_dt=FL, cin=16, cout=32, res=False, affine=False, pre=False, post=False, seed="round")
    got, _ = c.run(tmp_path)
    fp32_w = c.w[:, :, :32].reshape(3, 3, 16, 32).permute(3, 2, 0, 1).double()
    assert bool((q(fp32_w) != fp32_w).any())
    assert_close(got, c.want(), 2e-5, "rounded weights")
    miss = float((got.double() - c.want(fp32_w)).abs().max() / c.want(fp32_w).abs().max())
    assert miss > 2e-5, miss
    s = Conv(cuda, "small", out_dt=FL, cin=16, cout=32, k=(2, 5), pad=(1, 2), res=False, seed="round10")
    got, _ = s.run(tmp_path)
    assert_close(got, s.want(), 2e-5, "fp32 weights")


# ----------------------------------------------------------------------------------------------------------- c16 schedule
@pytest.mark.parametrize("rows_pb", [8, 3])
def test_c16_rows_per_block(cuda, tmp_path, rows_pb):
    """rows_pb = clamp(row_blocks / (SMs * 16), 1, 8): a map tall enough for 8 rows per block with hog % 8 != 0, and one for
    an intermediate 3 with a short last group; wog = 200 (> 128, not a multiple of 32: the last segment's fourth warp returns
    at once) and four 16-column chunks.  The grid the profiler records confirms rows_pb."""
    sms = num_sms()
    hog = 8 * sms + 5 if rows_pb == 8 else 3 * sms + 1
    assert hog % rows_pb != 0
    c = Conv(cuda, "c16", cin=16, cout=64, hw=(hog, 200), seed=f"rows{rows_pb}")
    row_blocks = c.n * hog * 2 * 4
    assert max(1, min(8, row_blocks // (sms * 16))) == rows_pb
    got, hits = c.check(tmp_path)
    grid = hits[0][1]
    assert grid is not None and list(grid) == [c.n * -(-hog // rows_pb), 2, 4], grid


# ------------------------------------------------------------------------------------------------------ transposed convolution
@pytest.mark.parametrize("body,in_dt,cin,cout", [("c16", H, 16, 24), ("small", FL, 8, 13), ("gemm64", H, 32, 64), ("gemm16", FL, 32, 24)])
def test_conv_transpose_phases(cuda, tmp_path, body, in_dt, cin, cout):
    """ConvTranspose2d(k3, s2, p1) as four output phases (1, 2, 2 and 4 taps), each called on the full h x w grid, so the
    odd phases' last row / column falls past hout = 2h - 1, wout = 2w - 1 and must be skipped.  After each call only that
    phase's (2 oy + py, 2 ox + px) lattice of the channel slice has changed; the result is fp64 F.conv_transpose2d."""
    n, h, w = 2, 7, 9
    ho, wo = 2 * h - 1, 2 * w - 1
    g = synth._gen(52, f"convT{body}")
    idt, odt = dt(in_dt), ops.h16()
    x = torch.randn(n, h, w, cin, generator=g).to(idt).to(cuda)
    wt = (torch.randn(cin, cout, 3, 3, generator=g) / (cin * 2.25) ** 0.5).to(cuda)
    b = torch.randn(cout, generator=g).to(cuda)
    sc, sh = (torch.rand(cout, generator=g) + 0.5).to(cuda), torch.randn(cout, generator=g).to(cuda)
    r = torch.randn(n, ho, wo, cout + 8, generator=g).to(odt).to(cuda)
    wt64 = q(wt) if body == "c16" else wt.double()
    want = epilogue(nhwc(F.conv_transpose2d(nchw(x.double()), wt64, None, 2, 1)), b, sc, sh, r[..., 4:4 + cout].double(), True, True, False)
    out_cs, out_off = cout + 12, 6
    full = canary((n + 1, ho, wo, out_cs), odt, cuda)
    for py in range(2):
        for px in range(2):
            taps, blocks = [], []
            for ky in range(3):
                if (py + 1 - ky) % 2:
                    continue
                for kx in range(3):
                    if (px + 1 - kx) % 2:
                        continue
                    taps.append(((py + 1 - ky) // 2, (px + 1 - kx) // 2))
                    blocks.append(wt[:, :, ky, kx])
            wp = torch.full((len(taps), cin, (cout + 15) // 16 * 16), float("nan"), device=cuda)
            wp[:, :, :cout] = torch.stack(blocks)
            before = bits(full).clone()
            launched = kernels(lambda: ops.conv_taps(x, cin, 0, full[:n], cout, out_off, h, w, (1, 1), (2, 2), (py, px), taps,
                                                     wp.contiguous(), b, sc, sh, r, 4, True, True), tmp_path)
            assert_body(launched, body_name(body, idt, odt, len(taps), cin))
            lattice = torch.zeros(full.shape, dtype=torch.bool, device=cuda)
            lattice[:n, py::2, px::2, out_off:out_off + cout] = True
            changed = bits(full) != before
            assert torch.equal(changed, lattice), (py, px, int((changed & ~lattice).sum()), int((lattice & ~changed).sum()))
    assert_close(full[:n, ..., out_off:out_off + cout], want, TOL[odt], f"convT {body}")


# ------------------------------------------------------------------------------------------------------ batch independence
@pytest.mark.parametrize("body,in_dt,cin,cout", [("c16", H, 16, 40), ("small", H, 12, 24), ("gemm64", FL, 32, 64), ("gemm16", H, 32, 40)])
def test_conv_taps_batch_independence(cuda, tmp_path, body, in_dt, cin, cout):
    """image k alone equals image k of a batch of 3, bit for bit (the c16 body's rows_pb and the GEMM tiles differ)"""
    c = Conv(cuda, body, in_dt=in_dt, n=3, cin=cin, cout=cout, hw=(21, 37), seed="batch")
    got, _ = c.run(tmp_path)
    for k in range(3):
        one = canary((1, c.ho, c.wo, c.out_cs), c.out_dt, cuda)
        c.call(c.x[k:k + 1].contiguous(), one, c.r[k:k + 1].contiguous())
        torch.cuda.synchronize()
        assert torch.equal(bits(one[0]), bits(got[k])), k


# ---------------------------------------------------------------------------------------------------------------------- NaN
@pytest.mark.parametrize("relu", ["none", "pre", "post"])
@pytest.mark.parametrize("body,in_dt,cin,cout", [("c16", H, 16, 24), ("small", FL, 8, 24), ("gemm64", H, 32, 64), ("gemm16", FL, 32, 24)])
def test_conv_taps_nan(cuda, tmp_path, body, in_dt, cin, cout, relu):
    """one NaN input pixel: without a ReLU the outputs whose receptive field holds it are NaN on every body; a ReLU is
    fmaxf(a, 0), which turns the NaN into 0 (header), so with one every output is finite and follows that rule"""
    c = Conv(cuda, body, in_dt=in_dt, cin=cin, cout=cout, pre=relu == "pre", post=relu == "post", nan_at=(1, 5, 6), seed="nan")
    got, _ = c.check(tmp_path)
    if relu == "none":
        assert int(torch.isnan(got.float()).sum()) == 9 * cout
    else:
        assert bool(torch.isfinite(got.float()).all())


# -------------------------------------------------------------------------------------------------------------- rejections
def _desc(cuda, in_dt=torch.float32, cin=16, cout=16):
    """a valid descriptor (1 x 8 x 8 map, 1 tap) and the tensors behind it; the output is canary-filled"""
    x = torch.zeros(1, 8, 8, cin, dtype=in_dt, device=cuda)
    out = canary((1, 8, 8, cout), torch.float32, cuda)
    r = torch.zeros(1, 8, 8, cout, device=cuda)
    w = torch.zeros(1, cin, 16, device=cuda)
    b = torch.zeros(32, device=cuda)
    d = capi.ConvDesc()
    d.inp, d.in_dtype, d.n, d.hin, d.win, d.cin, d.in_cstride, d.in_coff = x.data_ptr(), ops._DT[in_dt], 1, 8, 8, cin, cin, 0
    d.out, d.out_dtype, d.hout, d.wout, d.cout, d.out_cstride, d.out_coff = out.data_ptr(), capi.F32, 8, 8, cout, cout, 0
    d.hog, d.wog, d.in_sy, d.in_sx, d.out_sy, d.out_sx, d.out_oy, d.out_ox = 8, 8, 1, 1, 1, 1, 0, 0
    d.ntaps = 1
    d.w, d.bias = w.data_ptr(), b.data_ptr()
    d.res, d.res_dtype, d.res_cstride, d.res_coff = r.data_ptr(), capi.F32, cout, 0
    return d, (x, out, r, w, b)


REJECT = {
    "cin0": dict(cin=0), "cin_neg": dict(cin=-4), "in_coff_neg": dict(in_coff=-4), "out_coff_neg": dict(out_coff=-1),
    "res_coff_neg": dict(res_coff=-4), "res_slice_past_end": dict(res_coff=4), "res_cstride_small": dict(res_cstride=8),
    "in_sy0": dict(in_sy=0), "in_sx_neg": dict(in_sx=-1), "out_sy0": dict(out_sy=0), "out_sx_neg": dict(out_sx=-2),
    "out_oy_neg": dict(out_oy=-1), "out_ox_neg": dict(out_ox=-1), "hin0": dict(hin=0), "win0": dict(win=0), "hout0": dict(hout=0),
    "wout_neg": dict(wout=-3), "null_in": dict(inp=None), "null_out": dict(out=None), "null_w": dict(w=None),
    "in_misaligned": dict(inp=4), "out_misaligned": dict(out=4), "res_misaligned": dict(res=8), "w_misaligned": dict(w=4),
    "bias_misaligned": dict(bias=2), "in_h16_misaligned": dict(inp=4, in_dt=True),
}


@pytest.mark.parametrize("name", list(REJECT))
def test_conv_taps_rejects(cuda, name):
    """each argument check refuses before launch (LavbError) and writes nothing"""
    change = dict(REJECT[name])
    d, keep = _desc(cuda, in_dt=ops.h16() if change.pop("in_dt", False) else torch.float32)
    for k, v in change.items():
        if k in ("inp", "out", "res", "w", "bias") and v is not None:
            setattr(d, k, getattr(d, k) + v)                  # a byte offset from the aligned base
        else:
            setattr(d, k, v)
    with pytest.raises(capi.LavbError):
        capi.check(capi.lib().lavb_conv_taps(C.byref(d), ops._stream()), "lavb_conv_taps")
    torch.cuda.synchronize()
    assert bool(is_canary(keep[1]).all())
    # the unchanged descriptor is accepted (so each case above is refused for its own field)
    d, keep = _desc(cuda)
    capi.check(capi.lib().lavb_conv_taps(C.byref(d), ops._stream()), "lavb_conv_taps")
    torch.cuda.synchronize()
    assert not bool(is_canary(keep[1]).any())


# --------------------------------------------------------------------------------------------------------- deconv3x3s2_small
def _deconv(x, groups, cin_g, w, bias, n_outs, sigmoids, outs):
    return capi.lib().lavb_deconv3x3s2_small(
        ops._ptr(x), ops._DT[x.dtype], x.shape[0], x.shape[1], x.shape[2], x.shape[3], groups, cin_g, ops._ptr(w), ops._ptr(bias),
        (C.c_int * groups)(*n_outs), (C.c_int * groups)(*[int(s) for s in sigmoids]),
        (C.c_void_p * groups)(*[o.data_ptr() for o in outs]), ops._stream())


@pytest.mark.parametrize("dtype", [FL, H])
@pytest.mark.parametrize("groups,cin_g", [(g, c) for g in (1, 3, 8) for c in (8, 24, 64)])
def test_deconv3x3s2_small_contract(cuda, tmp_path, groups, cin_g, dtype):
    """groups x cin_g over the header's range, input channel stride past groups * cin_g, 1..4 outputs and the sigmoid mixed
    across groups, maps (1, 1), (8, 16), (9, 17), (13, 40): against fp64 conv_transpose2d(k3, s2, p1, op1) of each group's
    channels within 2e-5, every output element written and nothing past the end"""
    g = synth._gen(53, f"deconv{groups}{cin_g}{dtype}")
    idt = dt(dtype)
    n_outs = [1 + (i + cin_g // 8) % 4 for i in range(groups)]
    sigmoids = [(i + groups) % 2 == 1 for i in range(groups)]
    wt = [torch.randn(cin_g, no, 3, 3, generator=g) / (cin_g * 2.25) ** 0.5 for no in n_outs]
    wp = torch.randn(groups, cin_g, 9, 4, generator=g)              # the unused padding columns hold noise
    for k, (t, no) in enumerate(zip(wt, n_outs)):
        wp[k, :, :, :no] = t.permute(0, 2, 3, 1).reshape(cin_g, 9, no)
    wp, wt = wp.to(cuda).contiguous(), [t.to(cuda) for t in wt]
    bias = torch.randn(groups, 4, generator=g).to(cuda)
    for n, h, w in ((2, 1, 1), (2, 8, 16), (1, 9, 17), (2, 13, 40)):
        cs = groups * cin_g + 8
        x = torch.randn(n, h, w, cs, generator=g).to(idt).to(cuda)
        fulls = [canary((n + 1, 2 * h, 2 * w, no), torch.float32, cuda) for no in n_outs]
        launched = kernels(lambda: capi.check(_deconv(x, groups, cin_g, wp, bias, n_outs, sigmoids, [f[:n] for f in fulls]),
                                              "lavb_deconv3x3s2_small"), tmp_path)
        assert_body(launched, f"deconv3x3s2_small_kernel<{CNAME[idt]}>")
        for k in range(groups):
            want = nhwc(F.conv_transpose2d(nchw(x[..., k * cin_g:(k + 1) * cin_g].double()), wt[k].double(), bias[k, :n_outs[k]].double(),
                                           2, 1, 1))
            if sigmoids[k]:
                want = torch.sigmoid(want)
            got = fulls[k][:n]
            assert not bool(is_canary(got).any()), (k, h, w)
            assert bool(is_canary(fulls[k][n:]).all()), (k, h, w)
            assert_close(got, want, 2e-5, f"group {k} map {h}x{w}")


DECONV_REJECT = {"cin_g_neg": dict(cin_g=-8), "cin_g0": dict(cin_g=0), "n_neg": dict(n=-1), "h_neg": dict(h=-2),
                 "w_neg": dict(w=-16), "null_bias": dict(bias=None), "in_misaligned": dict(x_off=1)}


@pytest.mark.parametrize("name", list(DECONV_REJECT))
def test_deconv3x3s2_small_rejects(cuda, name):
    ch = DECONV_REJECT[name]
    buf = torch.zeros(2 * 4 * 4 * 16 + 4, device=cuda)
    off = ch.get("x_off", 0)
    x = buf[off:off + 2 * 4 * 4 * 16].view(2, 4, 4, 16)
    out = canary((2, 8, 8, 2), torch.float32, cuda)
    wp, bias = torch.zeros(1, 16, 9, 4, device=cuda), torch.zeros(1, 4, device=cuda)
    n, h, w = ch.get("n", 2), ch.get("h", 4), ch.get("w", 4)
    code = capi.lib().lavb_deconv3x3s2_small(ops._ptr(x), capi.F32, n, h, w, 16, 1, ch.get("cin_g", 16), ops._ptr(wp),
                                             ops._ptr(ch.get("bias", bias)), (C.c_int * 1)(2), (C.c_int * 1)(0),
                                             (C.c_void_p * 1)(out.data_ptr()), ops._stream())
    torch.cuda.synchronize()
    assert code != 0
    assert bool(is_canary(out).all())


# ----------------------------------------------------------------------------------------------------------- pool2_affine_relu
POOL = {
    # vector body: c, offsets and strides multiples of 4, aligned pointers
    "vec": dict(c=8, in_cs=16, in_off=4, out_cs=24, out_off=12, body="pool2_vec4_kernel"),
    # scalar body: c = 6; an input offset of 2; an input pointer one element past an aligned one
    "c6": dict(c=6, in_cs=8, in_off=0, out_cs=10, out_off=3, body="pool2_kernel"),
    "in_off2": dict(c=8, in_cs=12, in_off=2, out_cs=8, out_off=0, body="pool2_kernel"),
    "in_ptr_unaligned": dict(c=8, in_cs=8, in_off=0, out_cs=8, out_off=0, ptr_off=1, body="pool2_kernel"),
}


@pytest.mark.parametrize("dtype", [FL, H])
@pytest.mark.parametrize("name", list(POOL))
@pytest.mark.parametrize("affine", ["identity", "random"])
def test_pool2_affine_relu_contract(cuda, tmp_path, name, dtype, affine):
    """both bodies x both dtypes with channel slices: the 2 x 2 max exact; after y * scale + shift and the ReLU within one
    output ulp of fp64 (bit for bit with the identity affine); only the output slice written"""
    cfg = POOL[name]
    tdt = dt(dtype)
    n, h, w, c = 2, 10, 14, cfg["c"]
    g = synth._gen(54, f"pool{name}{dtype}{affine}")
    off = cfg.get("ptr_off", 0)
    buf = torch.randn(n * h * w * cfg["in_cs"] + off, generator=g).to(tdt).to(cuda)
    x = buf[off:].view(n, h, w, cfg["in_cs"])
    assert (x.data_ptr() % (4 * x.element_size()) == 0) == (off == 0)
    if affine == "identity":
        sc, sh = torch.ones(c, device=cuda), torch.zeros(c, device=cuda)
    else:
        sc, sh = (torch.randn(c, generator=g) * 2).to(cuda), torch.randn(c, generator=g).to(cuda)
    full = canary((n + 1, h // 2, w // 2, cfg["out_cs"]), tdt, cuda)
    launched = kernels(lambda: ops.pool2_affine_relu(x, c, cfg["in_off"], sc, sh, full[:n], cfg["out_off"]), tmp_path)
    assert_body(launched, f"{cfg['body']}<{CNAME[tdt]}>")
    xs = x[..., cfg["in_off"]:cfg["in_off"] + c]
    mx = torch.maximum(torch.maximum(xs[:, 0::2, 0::2], xs[:, 0::2, 1::2]), torch.maximum(xs[:, 1::2, 0::2], xs[:, 1::2, 1::2]))
    sl = slice(cfg["out_off"], cfg["out_off"] + c)
    got = full[:n, ..., sl]
    written = ~is_canary(full)
    inside = torch.zeros_like(written)
    inside[:n, ..., sl] = True
    assert torch.equal(written, inside)
    if affine == "identity":
        assert torch.equal(got.float(), fmax0(mx.double()).float())
    else:
        want = fmax0(mx.double() * sc.double() + sh.double())
        mant = {torch.float32: 23, torch.float16: 10, torch.bfloat16: 7}[tdt]
        tiny = {torch.float32: -126, torch.float16: -14, torch.bfloat16: -126}[tdt]
        ulp = torch.exp2(torch.floor(torch.log2(want.abs().clamp_min(2.0 ** tiny))) - mant)
        err = (got.double() - want).abs()
        assert bool((err <= ulp).all()), float((err / ulp).max())


POOL_REJECT = {"in_slice": dict(in_off=12), "out_slice": dict(out_off=9), "in_off_neg": dict(in_off=-4), "c0": dict(c=0),
               "n_neg": dict(n=-1), "hin_odd": dict(hin=5), "null_scale": dict(scale=None), "in_misaligned_byte": dict(in_byte=2)}


@pytest.mark.parametrize("name", list(POOL_REJECT))
def test_pool2_affine_relu_rejects(cuda, name):
    ch = POOL_REJECT[name]
    buf = torch.zeros(2 * 4 * 4 * 16 * 4 + 16, dtype=torch.uint8, device=cuda)
    ptr = buf.data_ptr() + ch.get("in_byte", 0)
    out = canary((2, 2, 2, 16), torch.float32, cuda)
    sc, sh = torch.ones(16, device=cuda), torch.zeros(16, device=cuda)
    code = capi.lib().lavb_pool2_affine_relu(C.c_void_p(ptr), capi.F32, ch.get("n", 2), ch.get("hin", 4), 4, ch.get("c", 8), 16,
                                             ch.get("in_off", 0), ops._ptr(ch.get("scale", sc)), ops._ptr(sh), ops._ptr(out), 16,
                                             ch.get("out_off", 8), ops._stream())
    torch.cuda.synchronize()
    assert code != 0
    assert bool(is_canary(out).all())


# ------------------------------------------------------------------------------------------------------------- rgb_normalize
@pytest.mark.parametrize("out_dtype", [FL, H])
@pytest.mark.parametrize("src", ["u8_nhwc", "float_nchw"])
def test_rgb_normalize_contract(cuda, tmp_path, src, out_dtype):
    """both sources x both output dtypes on n * h * w = 266 (not a multiple of 256): bit for bit fp32 (x / 255 - 0.5) * 2 (the
    kernel's three roundings) stored in the output dtype, the 4th channel exactly 0, nothing written past the end"""
    n, h, w = 2, 7, 19
    g = synth._gen(55, f"rgb{src}{out_dtype}")
    odt = dt(out_dtype)
    if src == "u8_nhwc":
        rgb = torch.randint(0, 256, (n, h, w, 3), generator=g, dtype=torch.uint8)
        x32 = rgb.float()
    else:
        rgb = torch.rand(n, 3, h, w, generator=g) * 255
        rgb[0, :, 0, :3] = torch.tensor([0.0, 255.0, 127.5])
        x32 = rgb.permute(0, 2, 3, 1)
    want = ((x32 / 255.0) - 0.5) * 2.0                 # fp32 on the host: IEEE division, subtraction and product
    full = canary((n + 1, h, w, 4), odt, cuda)
    rgb = rgb.to(cuda).contiguous()
    launched = kernels(lambda: capi.check(capi.lib().lavb_rgb_normalize(ops._ptr(rgb), int(src == "u8_nhwc"), n, h, w, ops._ptr(full),
                                                                         ops._DT[odt], ops._stream()), "lavb_rgb_normalize"), tmp_path)
    assert_body(launched, f"rgb_norm_kernel<{CNAME[odt]}>")
    got = full[:n].cpu()
    assert torch.equal(bits(got[..., :3]), bits(want.to(odt)))
    assert torch.equal(bits(got[..., 3]), bits(torch.zeros(n, h, w, dtype=odt)))
    assert bool(is_canary(full[n:]).all())
    # ops.rgb_normalize returns the same bits
    assert torch.equal(bits(ops.rgb_normalize(rgb, odt).cpu()), bits(got))


@pytest.mark.parametrize("args", [(-1, 4, 4), (2, -4, 4), (2, 4, -1)])
def test_rgb_normalize_rejects(cuda, args):
    out = canary((2, 4, 4, 4), torch.float32, cuda)
    rgb = torch.zeros(2, 4, 4, 3, dtype=torch.uint8, device=cuda)
    assert capi.lib().lavb_rgb_normalize(ops._ptr(rgb), 1, *args, ops._ptr(out), capi.F32, ops._stream()) != 0
    torch.cuda.synchronize()
    assert bool(is_canary(out).all())


# ------------------------------------------------------------------------------------------------------------------- convert
def _convert_src(count, src_dt, g):
    if src_dt == torch.float32:
        mag = torch.exp(torch.empty(count).uniform_(math.log(1e-8), math.log(3e4), generator=g))
        x = torch.randn(count, generator=g).sign() * mag
        special = torch.tensor([0.0, -0.0, float("nan"), 6e-8, -3e-8, 5.96e-8, 6.1e-5, -6.09e-5, 1.0 + 2.0 ** -11, 65504.0, -1e-30])
        x[:min(count, special.numel())] = special[:count]
        return x
    u = torch.randint(-32768, 32768, (count,), generator=g, dtype=torch.int32).to(torch.int16)
    special = torch.tensor([0x0000, -0x8000, 0x0001, -0x7FFF, 0x03FF, 0x7E00, 0x3C00], dtype=torch.int32).to(torch.int16)
    u[:min(count, special.numel())] = special[:count]
    return u.view(ops.h16())


@pytest.mark.parametrize("unaligned", [False, True])
@pytest.mark.parametrize("direction", ["f32_to_h16", "h16_to_f32"])
@pytest.mark.parametrize("count", [1, 3, 4, 5, 1027])
def test_convert_contract(cuda, count, direction, unaligned):
    """counts 1, 3, 4, 5, 1027 (vector body plus tail) both ways, from 4-element aligned buffers and from buffers one
    element past that (element-wise body): bit for bit Tensor.to on the host, +-0 and 16-bit subnormals included, NaN stays
    NaN; nothing written outside the count"""
    src_dt, dst_dt = (torch.float32, ops.h16()) if direction == "f32_to_h16" else (ops.h16(), torch.float32)
    g = synth._gen(56, f"convert{count}{direction}")
    x = _convert_src(count, src_dt, g)
    off = int(unaligned)
    sbuf = canary((count + 8,), src_dt, cuda)
    sbuf[off:off + count] = x.to(cuda)
    dbuf = canary((count + 8,), dst_dt, cuda)
    src, dst = sbuf[off:off + count], dbuf[off:off + count]
    capi.check(capi.lib().lavb_convert(ops._ptr(src), ops._DT[src_dt], ops._ptr(dst), ops._DT[dst_dt], count, ops._stream()),
               "lavb_convert")
    torch.cuda.synchronize()
    want = x.to(dst_dt)
    got = dst.cpu()
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan)
    assert torch.equal(bits(got)[~nan], bits(want)[~nan])
    outside = torch.ones(count + 8, dtype=torch.bool)
    outside[off:off + count] = False
    assert bool(is_canary(dbuf).cpu()[outside].all())


def test_convert_rejects(cuda):
    src = torch.zeros(16, device=cuda)
    dst = canary((16,), ops.h16(), cuda)
    lib = capi.lib()
    assert lib.lavb_convert(ops._ptr(src), capi.F32, ops._ptr(dst), ops._DT[ops.h16()], -4, ops._stream()) != 0
    assert lib.lavb_convert(C.c_void_p(src.data_ptr() + 2), capi.F32, ops._ptr(dst), ops._DT[ops.h16()], 4, ops._stream()) != 0
    assert lib.lavb_convert(ops._ptr(src), capi.F32, ops._ptr(dst), capi.F32, 4, ops._stream()) != 0
    torch.cuda.synchronize()
    assert bool(is_canary(dst).all())
