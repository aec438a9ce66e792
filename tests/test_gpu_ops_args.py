"""The kernel wrappers' argument checks: for each wrapper one valid call, then each of its checked conditions broken once (wrong
dtype, wrong shape, non-contiguous where the kernel needs dense memory, a host tensor).  A broken call raises LavbError naming the
wrapper before anything is launched, and leaves a given output untouched."""
import numpy as np
import pytest
import torch

from lav_b200 import ops, synth
from lav_b200 import point_painting as PP
from lav_b200.capi import LavbError

pytestmark = pytest.mark.gpu

GRID = (-10.0, 70.0, -40.0, 40.0, 0.25, 20, 20)


def nc(t):
    """a non-contiguous tensor of t's shape, dtype and values"""
    return torch.stack([t, t], -1)[..., 0]


def _cases(dev):
    """(wrapper, valid keyword arguments, output, bad overrides of those arguments).  The output is the name of the argument the
    wrapper writes, None, or the tensor itself when the call reaches it only through a device table (stack_jobs): the case then
    holds the tensor, so it outlives every call that writes through the table."""
    g = torch.Generator().manual_seed(7)
    r = lambda *s, dt=torch.float32: torch.rand(s, generator=g).to(dt).to(dev)             # noqa: E731
    z = lambda *s, dt=torch.float32: torch.zeros(s, dtype=dt, device=dev)                 # noqa: E731
    h, u8, i32 = ops.h16(), torch.uint8, torch.int32
    pts = synth.lidar_sweep(64, tag="args").to(dev).contiguous()
    cams = np.stack([c.packed() for c in PP.make_converters(rgb_h=32, rgb_w=32)])
    sem = r(3, 5, 32, 32)
    sw = pts.clone()
    p11 = torch.cat([pts, r(64, 7)], 1)
    mlp = [(t * 0.1).contiguous() for t in (r(64, 16), r(64), r(64), r(64, 64), r(64), r(64))]
    pill = dict(pts=p11, starts=[0, 30], counts=[30, 34], grid=GRID, w1=mlp[0], s1=mlp[1], t1=mlp[2], w2=mlp[3], s2=mlp[4], t2=mlp[5])
    pill_bad = [dict(pts=p11.double()), dict(pts=p11[:, :10]), dict(pts=nc(p11)), dict(pts=p11.cpu()), dict(w1=mlp[0].double()),
                dict(w2=mlp[3][:32]), dict(s1=nc(mlp[1])), dict(t2=mlp[5].cpu())]
    h64, cell = r(50, 64), torch.randint(0, 10, (50,), generator=g).to(i32).to(dev)
    g10, arg = r(10, 64), z(10, 64, dt=i32)
    tx, tw = r(1, 8, 8, 16), r(1, 16, 16)
    deconv = ops.pack_deconv2x2(r(16, 5, 2, 2), r(5))
    x64 = r(1, 16, 16, 64, dt=h)
    c33 = r(1, 8, 8, 64, dt=h)
    xp = r(1, 8, 32, 64, dt=h)
    gru = [r(2, 512), r(6, 512, 192), r(6, 64, 192), r(6, 192), r(6, 192), r(6, 2, 64), r(6, 2)]
    dst7 = z(64, 7)
    job = np.zeros(1, ops.STACK_JOB_DTYPE)
    job[0] = (pts.data_ptr(), dst7.data_ptr(), 64, 0, np.eye(3, dtype=np.float32).ravel(), 0.0, 0.0, 0)   # pts: held by the cases
    jobs = torch.from_numpy(job.view(np.uint8)).to(dev)
    return [
        (ops.paint, dict(points=pts, sem=sem, cams=cams, mode=0, out=z(64, 5)), "out",
         [dict(points=pts.double()), dict(points=pts[None]), dict(points=pts.t()), dict(points=pts.cpu()), dict(sem=sem.half()),
          dict(sem=sem[0]), dict(sem=sem.cpu()), dict(cams=cams[:2]), dict(out=z(64, 5).t()), dict(out=z(64, 5).double()),
          dict(out=z(63, 5)), dict(out=z(64, 4)), dict(cams=cams[:, :40])]),
        (ops.stack_sweep, dict(src=pts, R=np.eye(3), dx=1.0, dy=2.0, time_idx=1, n_time=3, dst=z(64, 7)), "dst",
         [dict(src=nc(pts)), dict(src=pts.cpu()), dict(dst=nc(z(64, 7))), dict(dst=z(64, 6)), dict(dst=z(63, 7)),
          dict(src=pts.half()), dict(dst=z(64, 7).double()), dict(R=np.eye(2)), dict(R=np.ones(8))]),
        (ops.roof_filter, dict(sweeps=sw, out=z(1, 64, 4)), "out",
         [dict(sweeps=pts.double()), dict(sweeps=nc(pts)), dict(sweeps=pts.flatten()), dict(sweeps=pts.cpu()), dict(out=z(1, 64, 5)),
          dict(out=nc(z(1, 64, 4))), dict(out=sw[None]), dict(out=z(1, 64, 4).double())]),
        (ops.pillar_forward, pill, None, pill_bad),
        (ops.pillar_forward_sorted, pill, None, pill_bad),
        (ops.pillar_decorate, dict(pts=p11, starts=[0], counts=[64], grid=GRID, d=11), None,
         [dict(pts=p11.double()), dict(pts=p11.flatten()), dict(pts=nc(p11)), dict(pts=p11.cpu())]),
        (ops.pillar_scatter_max, dict(h=h64, cell=cell, n_cells=10), None,
         [dict(h=h64.double()), dict(h=h64[0]), dict(h=h64.cpu()), dict(cell=cell.long()), dict(cell=cell[:49]), dict(cell=nc(cell)),
          dict(cell=cell.cpu()), dict(n_cells=-1)]),
        (ops.pillar_scatter_max_bwd, dict(gcanvas=g10, arg=arg, cell=cell, m=50), None,
         [dict(gcanvas=g10.bfloat16()), dict(gcanvas=g10[0]), dict(gcanvas=g10.cpu()), dict(arg=arg.long()), dict(arg=arg[:9]),
          dict(arg=nc(arg)), dict(cell=cell.long()), dict(cell=cell[:49]), dict(cell=nc(cell)), dict(cell=cell.cpu())]),
        (ops.conv_taps, dict(x=tx, cin=16, in_coff=0, out=z(1, 8, 8, 16), cout=16, out_coff=0, hog=8, wog=8, in_s=(1, 1), out_s=(1, 1),
                             out_o=(0, 0), taps=[(0, 0)], w=tw, res=r(1, 8, 8, 16)), "out",
         [dict(x=nc(tx)), dict(x=tx[0]), dict(x=tx.cpu()), dict(w=tw.double()), dict(w=tw[:, :8]), dict(w=nc(tw)), dict(umma=True),
          dict(out=z(2, 8, 8, 16)), dict(out=nc(z(1, 8, 8, 16))), dict(res=r(1, 8, 7, 16)), dict(res=nc(r(1, 8, 8, 16))),
          dict(d2s_nout=4)]),
        (ops.rgb_normalize, dict(rgb=r(1, 8, 8, 3, dt=u8)), None,
         [dict(rgb=r(1, 8, 8, 4, dt=u8)), dict(rgb=r(1, 8, 3, dt=u8)), dict(rgb=r(1, 4, 8, 8)), dict(rgb=r(1, 8, 8, 3, dt=u8).cpu())]),
        (ops.deconv3x3s2_small, dict(x=tx, groups=1, cin_g=16, w=r(1, 16, 9, 4), bias=r(1, 4), n_outs=[2], sigmoids=[0]), None,
         [dict(x=nc(tx)), dict(x=tx[0]), dict(x=tx.cpu()), dict(w=nc(r(1, 16, 9, 4))), dict(bias=nc(r(1, 4)))]),
        (ops.paint_batched, dict(points=pts[None], sem=sem[None], cams=cams, mode=1, copy_cols=4, out=z(1, 64, 8)), "out",
         [dict(points=pts[None].double()), dict(points=nc(pts[None])), dict(points=pts), dict(points=pts[None].cpu()),
          dict(sem=sem[None].half()), dict(sem=sem), dict(out=nc(z(1, 64, 8))), dict(out=z(1, 64, 7)), dict(out=z(1, 64, 8).double()),
          dict(out=z(1, 63, 8)), dict(sem=sem[None].expand(2, -1, -1, -1, -1)), dict(cams=cams[:2]), dict(cams=cams[:, :40])]),
        (ops.pack_deconv2x2, dict(weight=r(16, 5, 2, 2), bias=r(5)), None,
         [dict(weight=r(16, 9, 2, 2), bias=r(9)), dict(weight=r(8, 5, 2, 2)), dict(weight=r(16, 5, 3, 3))]),
        (ops.paint_deconv_batched, dict(points=pts[None], feat=r(3, 16, 16, 16), n_classes=5, deconv=deconv, cams=cams, copy_cols=4,
                                        out=z(1, 64, 8), image_hw=(32, 32)), "out",
         [dict(points=pts[None].double()), dict(points=nc(pts[None])), dict(points=pts[None].cpu()), dict(feat=r(3, 16, 16, 8)),
          dict(feat=nc(r(3, 16, 16, 16))), dict(deconv=deconv[:519]), dict(out=nc(z(1, 64, 8))), dict(deconv=deconv.half()),
          dict(feat=r(3, 16, 16, 16).double()), dict(out=z(1, 64, 7)), dict(out=z(1, 64, 8).double()), dict(cams=cams[:, :40]),
          dict(n_classes=9)]),
        (ops.stack_jobs, dict(d_jobs=jobs, n_jobs=1, max_n=64, src_cols=4, n_time=3), dst7,
         [dict(d_jobs=jobs[:71]), dict(n_jobs=2), dict(d_jobs=jobs.cpu()), dict(d_jobs=jobs.view(torch.int32)), dict(max_n=-1)]),
        (ops.bev_targets, dict(src_planes=r(2, 320, 320, dt=u8), jobs=ops.bev_jobs([(0, 0, 10.0, -5.0, 3, 2), (1, 1, 0.0, 0.0, 0, 0)]),
                               out=z(2, 320, 320, dt=u8)), "out",
         [dict(src_planes=r(2, 320, 320, dt=i32)), dict(src_planes=r(320, 320, dt=u8)), dict(src_planes=nc(r(2, 320, 320, dt=u8))),
          dict(src_planes=r(2, 320, 320, dt=u8).cpu()), dict(out=z(2, 320, 320)), dict(out=z(2, 320, 321, dt=u8)),
          dict(out=nc(z(2, 320, 320, dt=u8)))]),
        (ops.det_peaks, dict(center=r(1, 16, 16, 1), box=r(1, 16, 16, 2), ori=r(1, 16, 16, 2)), None,
         [dict(center=r(1, 16, 16, 1).double()), dict(center=r(16, 16, 1)), dict(center=nc(r(1, 16, 16, 2))),
          dict(center=r(1, 16, 16, 1).cpu()), dict(box=r(1, 16, 15, 2)), dict(ori=r(1, 16, 16, 3)), dict(box=nc(r(1, 16, 16, 2))),
          dict(ori=r(1, 16, 16, 2).half())]),
        (ops.conv7x7s2_umma, dict(x=x64, w_packed=ops.pack_conv7x7s2_weights(r(64, 64, 7, 7)), bias=r(64), out=z(1, 8, 8, 64, dt=h)), "out",
         [dict(x=x64.float()), dict(x=r(1, 16, 16, 32, dt=h)), dict(x=nc(x64)), dict(x=x64.cpu()), dict(w_packed=r(49, 64, 128, dt=h)),
          dict(bias=r(64).double()), dict(bias=r(32)), dict(out=z(1, 8, 9, 64, dt=h)), dict(out=nc(z(1, 8, 8, 64, dt=h))),
          dict(out=z(1, 8, 8, 64))]),
        (ops.conv3x3_umma, dict(x=c33, w=r(9, 64, 64, dt=h), cout=64, stride=1, bias=r(64), out=z(1, 8, 8, 64, dt=h)), "out",
         [dict(x=c33.float()), dict(x=c33[0]), dict(x=nc(c33)), dict(x=c33.cpu()), dict(w=r(9, 64, 128, dt=h)), dict(w=r(9, 64, 64)),
          dict(bias=r(32)), dict(bias=r(64).double()), dict(out=z(1, 8, 8, 128, dt=h)), dict(out=nc(z(1, 8, 8, 64, dt=h)))]),
        (ops.pack_conv7x7s2_weights, dict(w=r(64, 3, 7, 7)), None, [dict(w=r(64, 3, 5, 5)), dict(w=r(32, 3, 7, 7))]),
        (ops.conv_pair_umma, dict(x=xp, w1=r(3, 64, 64, dt=h), bias1=r(64), w2=r(3, 64, 64, dt=h), shift2=r(64), dil=1,
                                  res=r(1, 8, 32, 64, dt=h), out=z(1, 8, 32, 64, dt=h)), "out",
         [dict(x=xp.float()), dict(x=nc(xp)), dict(x=xp.cpu()), dict(w1=r(3, 64, 32, dt=h)), dict(w2=r(3, 64, 64)),
          dict(w1=nc(r(3, 64, 64, dt=h))), dict(bias1=r(32)), dict(shift2=r(64).double()), dict(res=r(1, 8, 16, 64, dt=h)),
          dict(res=nc(r(1, 8, 32, 64, dt=h))), dict(out=nc(z(1, 8, 32, 64, dt=h))), dict(out=z(1, 8, 32, 64))]),
        (ops.cast_gru, dict(embd=gru[0], wih_t=gru[1], whh_t=gru[2], bih=gru[3], bhh=gru[4], wmlp=gru[5], bmlp=gru[6], steps=4), None,
         [dict(embd=gru[0].double()), dict(embd=r(2, 256)), dict(embd=nc(gru[0])), dict(embd=gru[0].cpu()), dict(whh_t=r(6, 64, 96)),
          dict(bih=r(5, 192)), dict(wmlp=nc(gru[5])), dict(bmlp=gru[6].double())]),
    ]


def test_wrappers_refuse_bad_arguments_with_lavb_error(cuda):
    for fn, kw, out_key, bad in _cases(cuda):
        name = fn.__name__
        fn(**kw)
        for over in bad:
            call = {**kw, **over}
            out = out_key if torch.is_tensor(out_key) else call.get(out_key)
            if out is not None:
                out.fill_(7)
            before = ops.launches()
            with pytest.raises(LavbError, match=name):
                fn(**call)
            assert ops.launches() == before, (name, over.keys())
            if out is not None:
                assert bool((out == 7).all()), (name, over.keys())
    torch.cuda.synchronize()
