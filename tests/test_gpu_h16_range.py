"""GPU: the saturation contract of the 16-bit path (include/lav_b200.h: every fp32 -> h16 conversion saturates at +-65504).

Each test scales weights or inputs (inside the h16 range) so that a good share of the outputs falls past +-65504 while a
comparable share stays inside, and compares with the same operation in fp64 on the h16-rounded operands.  The reference
applies `store` (clamp to +-65504, then round to h16) at every point where the kernel stores h16, intermediates in shared
memory included.  Asserted: no inf / NaN anywhere; every element whose reference lies past the range is exactly +-65504;
the others meet the tolerance of the kernel's existing parity test.
"""
import pytest
import torch
import torch.nn.functional as F

from lav_b200 import ops, synth
from oracle import lav_ref as O
from tests import util

pytestmark = pytest.mark.gpu

H = 65504.0                      # largest finite IEEE half


@pytest.fixture(autouse=True)
def _ieee_half(cuda):
    if ops.h16() != torch.float16:
        pytest.skip("the +-65504 saturation contract is the IEEE-half build's")


def q(x):
    """operand rounded to h16 (the kernel reads h16), kept in fp64"""
    return x.to(torch.float16).double()


def store(x):
    """the kernel's h16 store: saturate to the finite range, then round to nearest"""
    return x.clamp(-H, H).to(torch.float16).double()


def gain(raw, frac=0.15):
    """factor that puts the largest `frac` of |raw| past the h16 range"""
    a = raw.detach().double().abs().flatten().cpu()
    k = max(1, int(a.numel() * (1 - frac)))
    return H / float(a.kthvalue(k).values)


def check(got, raw, want, tol, both_signs, live=None, scale=None):
    """got: kernel output; raw: reference value before the final h16 store; want: store(raw) (or the equivalent).
    The in-range error is measured as a fraction of `scale` (default: max |want|); live: the elements that count for coverage."""
    got, raw, want = got.double().cpu(), raw.double().cpu(), want.double().cpu()
    assert got.shape == want.shape == raw.shape
    assert bool(torch.isfinite(got).all()), f"{int((~torch.isfinite(got)).sum())} inf/NaN elements in an h16 output"
    over = raw.abs() > H * (1 + 1e-3)         # clear of the boundary, where accumulation order could decide
    inside = raw.abs() < H
    n = raw.numel() if live is None else int(live.sum())
    assert int(over.sum()) >= 0.05 * n, f"only {int(over.sum())} of {n} outputs past the range: the case does not test saturation"
    assert int((inside if live is None else inside & live).sum()) >= 0.05 * n, "too few outputs inside the range"
    if both_signs:
        assert bool((raw[over] > 0).any()) and bool((raw[over] < 0).any()), "overflow of one sign only"
    sat = got[over]
    assert torch.equal(sat, torch.sign(raw[over]) * H), \
        f"{int((sat != torch.sign(raw[over]) * H).sum())} out-of-range outputs are not +-65504, e.g. {sat[sat != torch.sign(raw[over]) * H][:4].tolist()}"
    rest = ~over
    err = float((got[rest] - want[rest]).abs().max() / (want.abs().max() if scale is None else scale))
    assert err < tol, err


def conv(x, w, b=None, stride=1, pad=0, dil=1):
    """fp64 conv of an NHWC tensor with an OIHW weight -> NHWC"""
    y = F.conv2d(x.double().permute(0, 3, 1, 2), w.double(), None if b is None else b.double(), stride, pad, dil)
    return y.permute(0, 2, 3, 1)


def taps3x3():
    return [(ky - 1, kx - 1) for ky in range(3) for kx in range(3)]


def gen(*tag):
    return synth._gen(71, "h16range" + str(tag))


# ----------------------------------------------------------------------------------------------------------- tap convolutions
@pytest.mark.parametrize("path", ["cuda_core", "c16"])
def test_conv_taps_h16_output_saturates(cuda, path):
    """lavb_conv_taps with h16 in and out: the CUDA-core tile kernel (cin = 64) and the 16-channel mma.sync kernel (cin = 16);
    no ReLU, so both signs overflow."""
    g = gen(path)
    cin, cout, n, h, w = (64 if path == "cuda_core" else 16), 32, 2, 20, 24
    x = q(torch.randn(n, h, w, cin, generator=g)).to(cuda)
    wt = (torch.randn(cout, cin, 3, 3, generator=g) / (9 * cin) ** 0.5).to(cuda)
    b = torch.randn(cout, generator=g).to(cuda)
    k = gain(conv(x, q(wt), b, pad=1))
    wt, b = q(wt * k), (b * k).float()
    raw = conv(x, wt, b, pad=1)
    out = torch.empty((n, h, w, cout), dtype=torch.float16, device=cuda)
    wp = wt.permute(2, 3, 1, 0).reshape(9, cin, cout).float().contiguous()          # [tap][cin][cout], cout already % 16
    ops.conv_taps(x.half(), cin, 0, out, cout, 0, h, w, (1, 1), (1, 1), (0, 0), taps3x3(), wp, bias=b)
    check(out, raw, store(raw), 5e-3, both_signs=True)


@pytest.mark.parametrize("res", [False, True])
def test_conv_umma_h16_output_saturates(cuda, res):
    """lavb_conv_umma with h16 output, bias folded into the shift (no pre-ReLU), no post-ReLU; with a residual of up to
    +-40000 the sum overflows as well."""
    g = gen("umma", res)
    cin, cout, n, h, w = 64, 64, 2, 16, 32
    x = q(torch.randn(n, h, w, cin, generator=g)).to(cuda)
    wt = (torch.randn(cout, cin, 3, 3, generator=g) / (9 * cin) ** 0.5).to(cuda)
    b = torch.randn(cout, generator=g).to(cuda)
    k = gain(conv(x, q(wt), b, pad=1), 0.08 if res else 0.15)
    wt, b = q(wt * k), (b * k).float()
    raw = conv(x, wt, b, pad=1)
    r = None
    if res:
        r = q((torch.rand(n, h, w, cout, generator=g) * 2 - 1) * 40000).to(cuda)
        raw = raw + r
    out = torch.empty((n, h, w, cout), dtype=torch.float16, device=cuda)
    wu = wt.permute(2, 3, 0, 1).reshape(9, cout, cin).half().contiguous()            # [tap][cout][cin]
    ops.conv_taps(x.half(), cin, 0, out, cout, 0, h, w, (1, 1), (1, 1), (0, 0), taps3x3(), wu, bias=b,
                  res=None if r is None else r.half(), umma=True)
    check(out, raw, store(raw), 1e-3, both_signs=True)


def pair_ref(x, w1, b1, w2, t2, dil, res, relu):
    """fp64 restatement of lavb_conv_pair_umma with its three h16 stores: mid, conv + shift, and the residual sum.
    x / res NHWC, w1 / w2 [cout][cin][tap] (h16 values).  -> (want, raw before the last store, conv + shift before its store)"""
    xc = x.double().permute(0, 3, 1, 2)
    mid = store(F.relu(F.conv2d(xc, w1[:, :, :, None].double(), b1.double(), padding=(dil, 0), dilation=(dil, 1))))
    a = F.conv2d(mid, w2[:, :, None, :].double(), t2.double(), padding=(0, dil), dilation=(1, dil))
    raw = a if res is None else store(a) + res.double().permute(0, 3, 1, 2)
    if relu:
        raw = F.relu(raw)
    nhwc = lambda t: t.permute(0, 2, 3, 1)
    return nhwc(store(raw)), nhwc(raw), nhwc(a)


@pytest.mark.parametrize("case", [(64, False, 0), (64, False, 1), (64, True, 0), (64, True, 1),
                                  (128, False, 0), (128, False, 1), (128, True, 0), (128, True, 1),
                                  (64, "overflow", 0), (64, "overflow", 1), (128, "overflow", 0)])
def test_conv_pair_umma_saturates(cuda, case):
    """lavb_conv_pair_umma: c in {64, 128}, with / without the residual, post_relu 0 / 1.  The first conv is scaled so that ~3 %
    of `mid` saturates.  "overflow": conv + shift stays inside the range and only the residual add goes past it — the packed
    h16 add of epilogue 2 must saturate like every other h16 store."""
    c, res, relu = case
    g = gen("pair", case)
    n, h, w, dil = 2, 6, 64, 2
    x = q(torch.randn(n, h, w, c, generator=g)).to(cuda)
    w1 = (torch.randn(c, c, 3, generator=g) / (3 * c) ** 0.5).to(cuda)
    w2 = (torch.randn(c, c, 3, generator=g) / (3 * c) ** 0.5).to(cuda)
    b1, t2 = (torch.randn(c, generator=g) * 0.1).to(cuda), (torch.randn(c, generator=g) * 0.1).to(cuda)
    overflow = res == "overflow"
    if not overflow:                            # ~3 % of mid past the range
        k1 = gain(F.conv2d(x.permute(0, 3, 1, 2), q(w1)[:, :, :, None], b1.double(), padding=(dil, 0), dilation=(dil, 1)), 0.03)
        w1, b1 = w1 * k1, b1 * k1
    w1 = q(w1)
    _, _, a = pair_ref(x, w1, b1, q(w2), t2, dil, None, False)
    if overflow:                                # conv + shift within +-0.7 * 65504, residual of 40000..65504 of either sign
        k2 = 0.7 * H / float(a.abs().max())
        r = torch.rand(n, h, w, c, generator=g) * (H - 40000) + 40000
        r = q(torch.where(torch.rand(n, h, w, c, generator=g) < 0.5, -r, r)).to(cuda)
    else:
        k2 = gain(a, 0.08 if res else 0.15)
        r = q((torch.rand(n, h, w, c, generator=g) * 2 - 1) * 40000).to(cuda) if res else None
    w2, t2 = q(w2 * k2), (t2 * k2).float()
    want, raw, a = pair_ref(x, w1, b1, w2, t2, dil, r, relu)
    if overflow:
        assert float(a.abs().max()) < H
    out = ops.conv_pair_umma(x.half(), w1.permute(2, 0, 1).half().contiguous(), b1.float(), w2.permute(2, 0, 1).half().contiguous(),
                             t2, dil, res=None if r is None else r.half(), post_relu=bool(relu))
    check(out, raw, want, 1e-2, both_signs=not relu)


# ------------------------------------------------------------------------------------------------------------------ stems
def test_conv7x7s2_umma_saturates(cuda):
    g = gen("stem7")
    n, h, w, cin = 2, 23, 30, 64
    x = q(torch.randn(n, h, w, cin, generator=g)).to(cuda)
    wt = (torch.randn(64, cin, 7, 7, generator=g) / (49 * cin) ** 0.5).to(cuda)
    b = (torch.randn(64, generator=g) * 0.5).to(cuda)
    k = gain(F.relu(conv(x, q(wt), b, 2, 3)))
    wt, b = q(wt * k), (b * k).float()
    raw = F.relu(conv(x, wt, b, 2, 3))
    out = ops.conv7x7s2_umma(x.half(), ops.pack_conv7x7s2_weights(wt), b)
    check(out, raw, store(raw), 2e-3, both_signs=False)


def test_stem7x7s2_u8_saturates(cuda):
    """the brake model's stem on raw camera bytes, weights scaled"""
    g = gen("stem_u8")
    b_, ncam, h, cw = 2, 2, 32, 24
    img = torch.randint(0, 256, (b_, ncam, h, cw, 3), generator=g, dtype=torch.uint8)
    wt = torch.randn(64, 3, 7, 7, generator=g) * 0.1
    bias = torch.randn(64, generator=g) * 0.1
    mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
    wide = img.permute(0, 2, 1, 3, 4).reshape(b_, h, ncam * cw, 3).double()
    xn = q((wide / 255. - torch.tensor(mean, dtype=torch.float64)) / torch.tensor(std, dtype=torch.float64))
    k = gain(F.relu(conv(xn, q(wt), bias, 2, 3)))
    wt, bias = q(wt * k), (bias * k).float()
    raw = F.relu(conv(xn, wt, bias, 2, 3))
    out = ops.stem7x7s2_u8(img.to(cuda), ops.pack_stem_weights(wt.float().to(cuda)), bias.to(cuda), mean, std)
    check(out, raw, store(raw), 1e-2, both_signs=False)


def test_erf_stem_h16_saturates(cuda):
    """fused normalize + DownsamplerBlock(3, 16) with h16 output: the 13 conv and the 3 pooled channels, scale enlarged"""
    g = gen("erf_stem")
    n, h, w = 2, 18, 70
    rgb = torch.randint(0, 256, (n, h, w, 3), generator=g, dtype=torch.uint8)
    w27 = torch.randn(27, 16, generator=g) / 27 ** 0.5
    w27[:, 13:] = 0
    s, t = torch.rand(16, generator=g) + 0.5, torch.randn(16, generator=g) * 0.1
    xn = ((rgb.double() / 255. - .5) * 2).permute(0, 3, 1, 2)
    wc = w27.double().reshape(3, 3, 3, 16).permute(3, 2, 0, 1)[:13]                  # [(ky*3+kx)*3+c][co] -> [co][c][ky][kx]
    pre = torch.cat([F.conv2d(xn, wc, stride=2, padding=1), F.max_pool2d(xn, 2)], 1).permute(0, 2, 3, 1)
    k = gain(F.relu(pre * s.double() + t.double()))
    s, t = s * k, t * k
    raw = F.relu(pre * s.double() + t.double())
    out = ops.erf_stem(rgb.to(cuda), w27.numpy(), s.numpy(), t.numpy(), torch.float16)
    check(out, raw, store(raw), 1e-3, both_signs=False)


# --------------------------------------------------------------------------------------------------- 16-channel ERFNet blocks
def test_erf_down16_saturates(cuda):
    """DownsamplerBlock(16, 64): conv channels 0-47 and pooled channels 48-63, BatchNorm scale enlarged"""
    g = gen("down16")
    n, h, w = 2, 12, 40
    x = q(torch.randn(n, h, w, 16, generator=g))
    w9 = torch.randn(9, 16, 48, generator=g) / 144 ** 0.5
    st = torch.stack([torch.rand(64, generator=g) + 0.5, torch.randn(64, generator=g) * 0.1], 1)
    wc = q(w9).reshape(3, 3, 16, 48).permute(3, 2, 0, 1)                              # [tap][cin][cout] -> [cout][cin][ky][kx]
    pre = torch.cat([conv(x, wc, stride=2, pad=1), F.max_pool2d(x.permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1)], 3)
    k = gain(F.relu(pre * st[:, 0].double() + st[:, 1].double()))
    st = (st * k).contiguous()
    raw = F.relu(pre * st[:, 0].double() + st[:, 1].double())
    out = ops.erf_down16(x.half().to(cuda), w9.to(cuda), st.to(cuda))
    check(out, raw, store(raw), 3e-3, both_signs=False)


def nb16_ref(x, w4, st):
    """fp64 non_bottleneck_1d(16) as lavb_erf_nb16 computes it: four convs, each result stored as h16 (three intermediates in
    shared memory), the residual added before the last store.  -> (want, raw before the last store, last conv's affine output)"""
    xc = x.double().permute(0, 3, 1, 2)
    t = xc
    for cv in range(4):
        wk = q(w4[cv]).permute(2, 1, 0)                                               # [tap][cin][cout] -> [cout][cin][tap]
        vert = cv % 2 == 0
        a = F.conv2d(t, wk[:, :, :, None] if vert else wk[:, :, None, :], padding=(1, 0) if vert else (0, 1))
        a = a * st[cv, :, 0].double()[None, :, None, None] + st[cv, :, 1].double()[None, :, None, None]
        raw = F.relu(a + xc if cv == 3 else a)
        t = store(raw)
    return t.permute(0, 2, 3, 1), raw.permute(0, 2, 3, 1), a


def test_erf_nb16_saturates(cuda):
    """non_bottleneck_1d(16): the last conv's affine enlarged, so the block output overflows after the residual add; the
    reference stores every intermediate as h16 too"""
    g = gen("nb16")
    n, h, w = 2, 13, 32
    x = q(torch.randn(n, h, w, 16, generator=g))
    w4 = torch.randn(4, 3, 16, 16, generator=g) / 48 ** 0.5
    st = torch.stack([torch.rand(4, 16, generator=g) + 0.5, torch.randn(4, 16, generator=g) * 0.1], 2)
    _, _, a = nb16_ref(x, w4, st)
    st[3] *= gain(a, 0.25)                       # a's sign is symmetric: ~12 % of the outputs past +65504
    want, raw, _ = nb16_ref(x, w4, st)
    out = ops.erf_nb16(x.half().to(cuda), w4.to(cuda), st.contiguous().to(cuda))
    check(out, raw, want, 5e-3, both_signs=False)


def test_pool2_affine_relu_h16_saturates(cuda):
    g = gen("pool2")
    n, h, w, c = 2, 8, 12, 32
    x = q(torch.randn(n, h, w, c, generator=g))
    s, t = torch.rand(c, generator=g) + 0.5, torch.randn(c, generator=g) * 0.1
    pooled = F.max_pool2d(x.permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1)
    k = gain(F.relu(pooled * s.double() + t.double()))
    s, t = (s * k).contiguous(), (t * k).contiguous()
    raw = F.relu(pooled * s.double() + t.double())
    out = torch.empty((n, h // 2, w // 2, c), dtype=torch.float16, device=cuda)
    ops.pool2_affine_relu(x.half().to(cuda), c, 0, s.to(cuda), t.to(cuda), out, 0)
    check(out, raw, store(raw), 1e-3, both_signs=False)


# ------------------------------------------------------------------------------------------------------------ pillar encoders
def test_pillar_encoders_h16_canvas_saturates(cuda):
    """the tensor-core pillar encoder with the second layer's BatchNorm affine enlarged: the h16 canvas (out_mode 2) saturates."""
    m, sd = util.lidar_model(cuda)
    m.set_precision("f16")
    pp = m.point_pillar_net
    clouds = util.pillar_clouds()
    npts = [len(c) for c in clouds]
    with torch.no_grad():
        unit = O.pillar_net(sd, clouds, npts, **util.GRID).permute(0, 2, 3, 1).double()
    live = (unit != 0).any(-1, keepdim=True).expand_as(unit)
    k = gain(unit[live])
    raw = unit * k
    w1, s1, t1, w2, s2, t2 = pp._build(cuda)
    buf, starts, counts = pp._as_buffer([c.to(cuda) for c in clouds], npts)
    with torch.no_grad():
        got = ops.pillar_forward_sorted(buf, starts, counts, pp._grid(), w1, s1, t1, w2, (s2 * k).contiguous(), (t2 * k).contiguous(),
                                        canvas16=True).double().cpu()
    # layer 2 on h16 operands: the existing parity test allows 1e-3 of the canvas scale, here that of the unsaturated canvas
    check(got, raw, store(raw), 1e-3, both_signs=False, live=live, scale=float(raw.abs().max()))


# ------------------------------------------------------------------------------------------------------------- dtype helpers
def test_convert_f32_to_h16_saturates_at_the_boundaries(cuda):
    """65504 is the largest half; 65519.99 rounds to it; from 65520 on, round-to-nearest gives inf and the contract 65504.
    This is the conversion ConvBackbone applies to an fp32 canvas on the 16-bit path."""
    edge = [65504.0, 65505.0, 65519.0, 65519.99, 65520.0, 65536.0, 1e5, 3.0e38, 65503.0, 65488.0, 1.0, 0.0]
    x = torch.tensor(edge + [-v for v in edge], dtype=torch.float32)
    got = ops.convert(x.to(cuda), torch.float16).cpu()
    want = x.double().clamp(-H, H).to(torch.float16)
    assert torch.equal(got, want), (x[got != want].tolist(), got[got != want].tolist())


def test_crop_bilinear_h16_full_range_stays_finite(cuda):
    """the planner's rotated crop on an h16 feature map of +-65504 blocks: bilinear weights summing to 1 in fp32 must not
    round a full-scale sample to inf"""
    from lav_b200.heads import crop_theta
    g = gen("crop")
    sign = torch.where(torch.rand(3, 16, 10, 12, generator=g) < 0.5, -1.0, 1.0)
    feats = (sign.repeat_interleave(4, 2).repeat_interleave(4, 3) * H)                 # (3, 16, 40, 48) in 4x4 blocks
    locs = torch.tensor([[0., 0.], [3., -5.], [-8., 2.], [30., 30.], [1., 1.]])
    oris = torch.tensor([0., 0.4, -2.0, 1.0, 3.1])
    fidx = torch.tensor([0, 1, 2, 1, 0], dtype=torch.int32)
    theta = crop_theta(locs, oris, 40, 48, 2.0, 24, torch.tensor(0.), torch.tensor(0.75))
    grids = F.affine_grid(theta.double(), torch.Size((5, 16, 24, 24)), align_corners=True)
    want = store(F.grid_sample(feats.double()[fidx.long()], grids, align_corners=True)).permute(0, 2, 3, 1)
    x = feats.permute(0, 2, 3, 1).contiguous().to(cuda).half()
    got = ops.crop_bilinear(x, fidx.to(cuda), theta.to(cuda), 24).double().cpu()
    assert bool(torch.isfinite(got).all())
    assert float(got.abs().max()) == H
    assert util.rel_err(got, want) < 1e-2
