"""Pin the oracle against the REAL reference and (re)generate tests/golden/.

Runs only in the authoring container (needs /root/reference).  It
  1. imports the reference modules unmodified from /root/reference (with the
     torch_scatter / carla stand-ins of oracle/refshim on sys.path),
  2. fills their state_dicts with lav_b200.synth.fill_state_dict_ (seeded),
  3. runs reference and oracle/lav_ref.py on the same seeded synthetic inputs,
     asserting agreement,
  4. stores (sub-sampled) REFERENCE outputs + state_dict key/shape manifests in
     tests/golden/, and real-weight state_dicts (ERFNet, brake) in the
     git-ignored oracle/_ref/ so they travel to the GPU box.

    python oracle/pin_against_reference.py
"""
import json
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("LAV_REFERENCE", "/root/reference")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "refshim"))
sys.path.insert(0, os.path.join(REF, "team_code_v2"))
sys.path.insert(0, REF)

from lav_b200 import synth  # noqa: E402
from oracle import lav_ref as O  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
if "--weights-only" in sys.argv:    # only the real-weight state_dicts of oracle/_ref/; the fixtures go to a scratch directory
    import atexit
    import shutil
    import tempfile
    GOLD = tempfile.mkdtemp(prefix="lavb_pin_")
    atexit.register(shutil.rmtree, GOLD, True)
REFOUT = os.path.join(ROOT, "oracle", "_ref")
os.makedirs(GOLD, exist_ok=True)
os.makedirs(REFOUT, exist_ok=True)
torch.set_grad_enabled(False)


def maxdiff(a, b):
    return float((torch.as_tensor(a).double() - torch.as_tensor(b).double()).abs().max())


def check(name, a, b, tol):
    d = maxdiff(a, b)
    print(f"  {name:38s} max|ref-oracle| = {d:.3e} (tol {tol:g})")
    assert d <= tol, name
    return d


def manifest(sd):
    return {k: list(v.shape) for k, v in sd.items()}


def main():
    # ---- reference imports (unmodified files) -------------------------------------------
    from models.lidar import LiDARModel
    from models.uniplanner import UniPlanner
    from models.bev_planner import BEVPlanner
    from models.rgb import RGBSegmentationModel, RGBBrakePredictionModel
    import model_inference as MI
    import point_painting as PP

    report = {}

    # ---- painting (a2-a4) -----------------------------------------------------------------
    print("[paint]")
    convs_ref_t = [MI.CoordConverter(yaw, lidar_xyz=[0, 0, 2.4], cam_xyz=[1.5, 0, 2.4], rgb_h=288, rgb_w=256, fov=64)
                   for yaw in MI.CAMERA_YAWS]
    convs_ref_n = [PP.CoordConverter(yaw, lidar_xyz=[0, 0, 2.4], cam_xyz=[1.5, 0, 2.4], rgb_h=288, rgb_w=256, fov=64)
                   for yaw in MI.CAMERA_YAWS]
    convs = O.default_converters()
    lidar = synth.lidar_sweep(8192, tag="paint")
    # add edge cases: points near the camera plane / image border / behind
    edge = torch.tensor([[1.5001, 0, 0, .5], [1.49, 0.3, 0.1, .5], [2.0, 0.6247, 0.0, .5], [2.3, -0.2, 0.7, .5],
                         [-5, 0, 0, .5], [1.6, 5, -2, .5], [0, 0, 0, .5], [1.5, 0, 0, .5]])
    lidar = torch.cat([lidar, edge]).contiguous()
    sem5 = synth.sem_probs(tag="paint")
    sem4 = O.suppress_background(sem5)
    self_stub = types.SimpleNamespace(coord_converters=convs_ref_t)
    ref_painted = MI.InferModel.point_painting(self_stub, lidar, sem4)
    ref_uvz = torch.stack([c(lidar) for c in convs_ref_t])
    ref_painted64 = PP.point_painting(lidar.numpy(), sem4.numpy(), convs_ref_n)
    ora_uvz = torch.stack([O.lidar_to_cam_f32(lidar, c) for c in convs])
    check("uvz fp32 twin", ref_uvz, ora_uvz, 0)
    check("painted fp32 twin", ref_painted, O.point_painting_f32(lidar, sem4, convs), 0)
    check("painted fp64 numpy", ref_painted64, O.point_painting_f64(lidar.numpy(), sem4.numpy(), convs), 0)
    self_stub2 = types.SimpleNamespace(coord_converters=convs_ref_t, point_painting=lambda l, s: MI.InferModel.point_painting(self_stub, l, s))
    ref_fused = MI.InferModel.forward_paint(self_stub2, lidar, sem5)
    check("forward_paint", ref_fused, O.forward_paint(lidar, sem5, convs), 0)
    flips = int((torch.from_numpy(ref_painted64).float() != ref_painted).any(dim=1).sum())
    print(f"  fp32-vs-fp64 painter boundary flips: {flips} / {len(lidar)} points")
    report["paint_flips_fp32_vs_fp64"] = flips
    np.savez_compressed(os.path.join(GOLD, "paint.npz"), edge=edge.numpy(), painted=ref_painted.numpy(),
                        uvz=ref_uvz.numpy().astype(np.int32), painted64=ref_painted64, fused=ref_fused.numpy())

    # ---- LiDARModel (a6-a12) -----------------------------------------------------------------
    print("[lidar model]")
    grid = dict(min_x=-10, max_x=70, min_y=-40, max_y=40)
    lm = LiDARModel(num_input=4 + 10 + 2, num_features=[64, 64], backbone="cnn", pixels_per_meter=4, **grid).eval()
    sd = synth.fill_state_dict_(lm.state_dict())
    lm.load_state_dict(sd)
    json.dump(manifest(sd), open(os.path.join(GOLD, "keys_lidar_model.json"), "w"), indent=0)
    clouds = [synth.stacked_lidar(2000, tag="pp0"), synth.stacked_lidar(1500, tag="pp1")]
    # padded batch tensor form (B,P,D) + num_points, as train_lidar feeds it (lav_final_v2.py:147-169)
    npts = [len(c) for c in clouds]
    ref_canvas = lm.point_pillar_net(clouds, npts)
    ora_canvas = O.pillar_net(sd, clouds, npts, **grid)
    check("canvas", ref_canvas, ora_canvas, 1e-5)
    ref_out = lm(clouds, npts)
    ora_out = O.lidar_model(sd, clouds, npts, **grid)
    names = ["features", "center", "box", "ori", "seg"]
    for n, a, b in zip(names, ref_out, ora_out):
        check(n, a, b, 2e-4)
    nz = ref_canvas.permute(0, 2, 3, 1).abs().sum(-1).nonzero()
    vals = ref_canvas.permute(0, 2, 3, 1)[nz[:, 0], nz[:, 1], nz[:, 2]]
    print(f"  occupied pillars: {len(nz)}")
    np.savez_compressed(os.path.join(GOLD, "lidar_model.npz"), pillar_idx=nz.numpy().astype(np.int32),
                        pillar_val=vals.numpy(), features_s8=ref_out[0][:, :, ::8, ::8].numpy(),
                        **{n + "_s4": t[:, :, ::4, ::4].numpy() for n, t in zip(names[1:], ref_out[1:])})

    # training-mode forward/backward of the pillar encoder + backbone (batch-stat BN), loss = weighted sums
    torch.set_grad_enabled(True)
    lm.train()
    outs = lm(clouds, npts)
    gw = [torch.randn(o.shape, generator=synth._gen(7, f"gw{i}")) for i, o in enumerate(outs)]
    loss = sum((o * g).sum() for o, g in zip(outs, gw)) / 1e3
    loss.backward()
    ref_grads = {k: p.grad.clone() for k, p in lm.named_parameters()}
    sd_t = {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in sd.items()}
    o_outs = O.lidar_model(sd_t, clouds, npts, training=True, **grid)
    o_loss = sum((o * g).sum() for o, g in zip(o_outs, gw)) / 1e3
    o_loss.backward()
    check("train loss", loss.detach(), o_loss.detach(), 1e-3 * abs(float(loss)) + 1e-4)
    worst = 0.0
    for k, g in ref_grads.items():
        rel = maxdiff(g, sd_t[k].grad) / (float(g.abs().max()) + 1e-6)
        worst = max(worst, rel)
    print(f"  train grads worst rel diff = {worst:.3e}")
    assert worst < 5e-3
    sel = ["point_pillar_net.point_net.net.0.weight", "point_pillar_net.point_net.net.3.weight",
           "backbone.conv1.0.weight", "backbone.upconv3.0.weight", "center_head.net.3.bias", "backbone.conv2.2.weight"]
    digest = {}
    for k, g_ in ref_grads.items():      # compact fingerprint of EVERY parameter gradient: l2 norm, sum, projection on a seeded vector
        r = torch.randn(g_.shape, generator=synth._gen(13, "dg:" + k))
        digest[k] = [float(g_.norm()), float(g_.sum()), float((g_ * r).sum()), float(g_.abs().max())]
    json.dump(digest, open(os.path.join(GOLD, "lidar_model_train_grad_digest.json"), "w"), indent=0)
    np.savez_compressed(os.path.join(GOLD, "lidar_model_train.npz"), loss=float(loss),
                        **{"grad:" + k: ref_grads[k].numpy() for k in sel},
                        **{"out_" + n: o.detach()[:, :, ::8, ::8].numpy() for n, o in zip(names, outs)})
    torch.set_grad_enabled(False)
    lm.eval()
    lm.load_state_dict(sd)   # running stats were updated by the train forward

    # ---- ERFNet (a1) ------------------------------------------------------------------------------
    print("[erfnet]")
    seg = RGBSegmentationModel([4, 6, 7, 10]).eval()
    sd_seg = synth.fill_state_dict_(seg.state_dict())
    seg.load_state_dict(sd_seg)
    json.dump(manifest(sd_seg), open(os.path.join(GOLD, "keys_seg_model.json"), "w"), indent=0)
    rgb = synth.rgb_frames(smooth=True).permute(0, 3, 1, 2).float()
    ref_logits = seg(rgb)
    check("erfnet seeded", ref_logits, O.erfnet(sd_seg, rgb), 2e-4 * float(ref_logits.abs().max()))
    gold = dict(seeded_s4=ref_logits[:, :, ::4, ::4].numpy(), seeded_absmax=float(ref_logits.abs().max()))
    real = os.path.join(REF, "weights", "seg_1.pt")
    if os.path.getsize(real) > 10000:
        ts = torch.jit.load(real, map_location="cpu").eval()
        sd_real = {k: v.clone() for k, v in ts.state_dict().items()}
        seg.load_state_dict(sd_real, strict=True)
        r = seg(rgb)
        check("erfnet real eager-vs-trace", r, ts(rgb), 1e-4)
        check("erfnet real oracle", r, O.erfnet(sd_real, rgb), 1e-3)
        torch.save(sd_real, os.path.join(REFOUT, "seg_1.state_dict.pt"))
        gold.update(real_s4=r[:, :, ::4, ::4].numpy(), real_argmax=r.argmax(1).to(torch.uint8).numpy())
    np.savez_compressed(os.path.join(GOLD, "erfnet.npz"), **gold)

    # ---- UniPlanner.infer + whole frame (a13-a16) ------------------------------------------------
    print("[uniplanner]")
    kw = dict(pixels_per_meter=4, crop_size=96, feature_x_jitter=1.5, feature_angle_jitter=20, x_offset=0,
              y_offset=1 + (-10) / ((70 + 10) / 2), num_cmds=6, num_plan=20, num_plan_iter=5)
    bevp = BEVPlanner(num_frame_stack=2, **kw)
    up = UniPlanner(bevp, num_input_feature=384, **kw).eval()
    sd_up = synth.fill_state_dict_(up.state_dict())
    up.load_state_dict(sd_up)
    json.dump(manifest(sd_up), open(os.path.join(GOLD, "keys_uniplanner.json"), "w"), indent=0)
    feats = ref_out[0][0]
    det = [(150.0, 200.0, 8.0, 4.0, 0.9, 0.3), (170.0, 240.0, 8.0, 4.0, -0.2, 0.95), (161.0, 281.0, 8., 4., 1., 0.)]
    nxp = torch.tensor([0.0, -20.0])
    r_epl, r_ecl, r_ocl, r_occ = up.infer(feats, det, 2, nxp)
    o_ee, o_epl, o_ecl, o_ocl, o_occ = O.uniplanner_infer(sd_up, feats, det, 2, nxp)
    sc = float(r_ocl.abs().max()) + 1
    check("ego_plan_locs", r_epl, o_epl, 1e-4 * sc)
    check("ego_cast_locs", r_ecl, o_ecl, 1e-4 * sc)
    check("other_cast_locs", r_ocl, o_ocl, 1e-4 * sc)
    check("other_cast_cmds", r_occ, o_occ, 1e-5)
    # fast-agent functional twin (model_inference.py:123-187) must agree with the module path
    stub = types.SimpleNamespace(offset_x=up.offset_x, offset_y=up.offset_y, pixels_per_meter=4, crop_size=96, num_cmds=6,
                                 num_plan=20, lidar_conv_emb=up.lidar_conv_emb, cast=up.cast, plan=up.plan,
                                 cast_cmd_pred=up.cast_cmd_pred)
    f_ee, f_epl, f_ecl, f_ocl, f_occ = MI.InferModel.uniplanner_infer(stub, feats, det, 2, nxp)
    check("fast twin ego_plan", f_epl, r_epl, 1e-4 * sc)
    check("ego_embd", f_ee, o_ee, 1e-4 * float(f_ee.abs().max()))
    ref_dets = MI.InferModel.det_inference(types.SimpleNamespace(pixels_per_meter=4), torch.sigmoid(ref_out[1][0]),
                                           ref_out[2][0], ref_out[3][0])
    ora_dets = O.det_inference(torch.sigmoid(ora_out[1][0]), ora_out[2][0], ora_out[3][0])
    assert [[d[:2] for d in c] for c in ref_dets] == [[d[:2] for d in c] for c in ora_dets], "det peaks differ"
    print(f"  det_inference peaks (random heads): {[len(c) for c in ref_dets]}")
    # blob heat-maps so the decode has something to find (incl. filtered cases: near ego, far, tiny)
    gb = synth._gen(11, "blobs")
    yy, xx = torch.meshgrid(torch.arange(320.), torch.arange(320.), indexing="ij")
    heat = torch.full((2, 320, 320), -6.0)
    centres = [(100, 200), (161, 281), (250, 150), (30, 30), (160, 100), (200, 260), (120, 250)]
    for ci, (cx_, cy_) in enumerate(centres):
        amp = 4.0 + float(torch.rand(1, generator=gb)) * 6
        heat[ci % 2] = torch.maximum(heat[ci % 2], -6 + amp * torch.exp(-((xx - cx_) ** 2 + (yy - cy_) ** 2) / 8.0))
    sizem = torch.rand(2, 320, 320, generator=gb) * 3
    orim = torch.randn(2, 320, 320, generator=gb)
    ref_dets2 = MI.InferModel.det_inference(types.SimpleNamespace(pixels_per_meter=4), torch.sigmoid(heat), sizem, orim)
    ora_dets2 = O.det_inference(torch.sigmoid(heat), sizem, orim)
    assert ref_dets2 == ora_dets2 and sum(len(c) for c in ref_dets2) > 0, "blob det differ"
    print(f"  det_inference peaks (blobs): {[len(c) for c in ref_dets2]}")
    ref_dets = ref_dets2
    np.savez_compressed(os.path.join(GOLD, "uniplanner.npz"), det=np.array(det), ego_embd=f_ee.numpy(), ego_plan=r_epl.numpy(),
                        ego_cast=r_ecl.numpy(), other_cast=r_ocl.numpy(), other_cmds=r_occ.numpy(),
                        det0=np.array(ref_dets[0]).reshape(-1, 6), det1=np.array(ref_dets[1]).reshape(-1, 6))

    # ---- UniPlanner training forward with its frozen teacher (a17) -----------------------------------------------
    print("[uniplanner train]")
    import importlib
    pkg = types.ModuleType("lavm")                      # lav/models as a package WITHOUT running its __init__ (it imports an absent unet)
    pkg.__path__ = [os.path.join(REF, "lav", "models")]
    sys.modules["lavm"] = pkg
    UP2 = importlib.import_module("lavm.uniplanner").UniPlanner
    BP2 = importlib.import_module("lavm.bev_planner_v2").BEVPlanner
    from lav_b200.heads import UniPlanner as MyUP, BEVPlanner as MyBP
    ref_up = UP2(BP2(num_frame_stack=2, **kw), num_input_feature=384, **kw).train()
    assert list(ref_up.state_dict().keys()) == list(sd_up.keys())
    ref_up.load_state_dict(sd_up)
    my_up = MyUP(MyBP(num_frame_stack=2, **kw), num_input_feature=384, **kw).train()
    my_up.load_state_dict(sd_up)
    gt = synth._gen(23, "uptrain")
    Bt, No = 2, 5
    feats_t = (ref_out[0][:Bt] * 0.5).clone()                                  # (2,384,160,160)
    bev_t = (torch.rand(Bt, 9, 320, 320, generator=gt) > 0.7).float()
    ego_locs_t = torch.cumsum(torch.rand(Bt, 21, 2, generator=gt) * torch.tensor([0.2, -1.0]), dim=1)
    locs_t = torch.randn(Bt, No + 1, 21, 2, generator=gt) * 6 + torch.tensor([0.0, -8.0])
    locs_t[:, 0] = ego_locs_t
    oris_t = torch.rand(Bt, No + 1, generator=gt) * 0.6 - 0.3
    typs_t = torch.tensor([[1, 1, 1, 0, 1, 1], [1, 1, 0, 1, 1, 0]])
    nxps_t = torch.tensor([[0.0, -20.0], [3.0, -15.0]])
    torch.set_grad_enabled(True)
    torch.manual_seed(1234)
    r_out = ref_up(feats_t, bev_t, ego_locs_t, locs_t, oris_t, nxps_t, typs_t)
    torch.manual_seed(1234)
    m_out = my_up(feats_t, bev_t, ego_locs_t, locs_t, oris_t, nxps_t, typs_t)
    names_t = ["other_locs", "other_cast_locs", "other_cast_cmds", "other_cast_locs_expert", "other_cast_cmds_expert", "ego_locs",
               "ego_plan_locs", "ego_cast_locs", "ego_cast_cmds", "ego_cast_locs_expert", "ego_plan_locs_expert"]
    assert len(r_out) == len(m_out) == 11
    for n, a_, b_ in zip(names_t, r_out, m_out):
        check("train " + n, a_.detach(), b_.detach(), 2e-4 * (float(a_.abs().max()) + 1))
    torch.set_grad_enabled(False)
    np.savez_compressed(os.path.join(GOLD, "uniplanner_train.npz"), **{n: a_.detach().numpy() for n, a_ in zip(names_t, r_out)})

    # ---- train_lidar loss block (a18): the REFERENCE's own LAV.train_lidar, sub-models stubbed ------------------------------
    print("[train_lidar losses]")
    import yaml
    from lav.lav_final_v2 import LAV
    from lav.models.loss import DetLoss as RefDetLoss
    from lav_b200 import train as T
    cfg = yaml.safe_load(open(os.path.join(REF, "config_v2.yaml")))
    outs_l, planner_l, tg = synth.loss_block_inputs()
    gold_l = {}
    for distill in (True, False):
        for mode in ("full", "perceive_only", "motion_only"):
            torch.set_grad_enabled(True)
            leaf = torch.zeros((), requires_grad=True)                      # so that the reference's backward()/step() have a graph
            obj = object.__new__(LAV)                                       # LAV.__init__ loads checkpoints: set what train_lidar reads
            for k in ("box_weight", "ori_weight", "seg_weight", "other_weight", "cmd_weight", "perception_weight", "cmd_smooth",
                      "num_plan", "num_plan_iter", "num_cmds", "pixels_per_meter"):
                setattr(obj, k, cfg[k])
            obj.device, obj.distill = torch.device("cpu"), distill
            obj.perceive_only, obj.motion_only = mode == "perceive_only", mode == "motion_only"
            obj.branch_weights = torch.tensor(cfg["branch_weights"]).float()
            obj.det_criterion = RefDetLoss()
            obj.bev_center = [160.0, 280.0]
            obj.seg_mask = LAV.build_seg_mask(obj, h=320, w=320, cx=160, cy=280)
            obj.lidar_model = lambda lidars, num_points: tuple(t + leaf for t in outs_l[:4]) + (outs_l[4],)
            obj.uniplanner = lambda *a: tuple(t + leaf for t in planner_l)
            obj.lidar_optim = torch.optim.SGD([leaf], lr=0.0)
            obj.det_inference = lambda *a, **k: [[], []]
            obj.mot_inference = lambda *a, **k: (torch.zeros(20, 2), torch.zeros(0, 6, 20, 2), torch.zeros(0, 6))
            B_ = tg["cmds"].shape[0]
            res = LAV.train_lidar(obj, torch.zeros(B_, 4, 11), torch.tensor([4] * B_), tg["heatmaps"], tg["sizemaps"], tg["orimaps"], tg["bev"],
                                  tg["ego_locs"], tg["cmds"], torch.zeros(B_, 2), tg["bras"], torch.zeros(B_, 6, 21, 2), torch.zeros(B_, 6),
                                  torch.zeros(B_, 6).long(), torch.tensor([6] * B_))
            torch.set_grad_enabled(False)
            names_l = ["hm_loss", "box_loss", "ori_loss", "seg_loss", "plan_loss", "ego_cast_loss", "other_cast_loss", "cmd_loss"]
            ref_l = np.array([res[k] for k in names_l], dtype=np.float64)
            mine, parts = T.train_losses(outs_l, planner_l, tg["heatmaps"], tg["sizemaps"], tg["orimaps"], tg["bev"], tg["ego_locs"],
                                         tg["cmds"], tg["bras"], T.build_seg_mask(), T.LossConfig(distill=distill, perceive_only=obj.perceive_only,
                                                                                             motion_only=obj.motion_only))
            my_l = np.array([float(parts[k]) for k in names_l])
            d = float(np.abs(ref_l - my_l).max() / (np.abs(ref_l).max()))
            print(f"  distill={distill} {mode:14s} max rel |ref-mine| over the 8 losses = {d:.2e}")
            assert d < 1e-5
            gold_l[f"{'distill' if distill else 'nodistill'}_{mode}"] = ref_l
    np.savez_compressed(os.path.join(GOLD, "train_losses.npz"), names=np.array(names_l), **gold_l)

    # ---- brake model (a19) -------------------------------------------------------------------------
    print("[brake]")
    bra = RGBBrakePredictionModel([4, 6, 7, 10], pretrained=False).eval()
    sd_bra = synth.fill_state_dict_(bra.state_dict())
    bra.load_state_dict(sd_bra)
    json.dump(manifest(sd_bra), open(os.path.join(GOLD, "keys_brake.json"), "w"), indent=0)
    rgb1 = synth.rgb_frames(smooth=True, tag="wide", n_cam=1, h=288, w=768).permute(0, 3, 1, 2).float()
    rgb2 = synth.rgb_frames(smooth=True, tag="tele", n_cam=1, h=192, w=480).permute(0, 3, 1, 2).float()
    r = bra(rgb1, rgb2)
    check("brake seeded", r, O.brake_model(sd_bra, rgb1, rgb2), 1e-5)
    gold = dict(seeded=r.numpy())
    real = os.path.join(REF, "weights", "bra_v2_9.pt")
    if os.path.getsize(real) > 10000:
        ts = torch.jit.load(real, map_location="cpu").eval()
        sd_real = {k: v.clone() for k, v in ts.state_dict().items()}
        n_lab = sd_real["seg_head.upconv.9.weight"].shape[0]      # released brake net has 4 seg labels
        bra = RGBBrakePredictionModel(list(range(n_lab - 1)), pretrained=False).eval()
        bra.load_state_dict(sd_real, strict=True)
        r = bra(rgb1, rgb2)
        try:   # the released trace hard-codes a cuda device for the positional encoding
            check("brake real eager-vs-trace", r, ts(rgb1, rgb2), 1e-5)
        except RuntimeError as e:
            print("  brake trace not runnable on CPU (device baked into the trace):", str(e).splitlines()[-1][:60])
        check("brake real oracle", r, O.brake_model(sd_real, rgb1, rgb2), 1e-5)
        torch.save(sd_real, os.path.join(REFOUT, "bra_v2_9.state_dict.pt"))
        gold.update(real=r.numpy())
    np.savez_compressed(os.path.join(GOLD, "brake.npz"), **gold)

    json.dump(report, open(os.path.join(GOLD, "pin_report.json"), "w"), indent=1)
    print("golden fixtures written to", GOLD)


if __name__ == "__main__":
    main()
