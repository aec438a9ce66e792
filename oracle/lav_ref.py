"""ORACLE — test infrastructure, never the product path.

A CPU (PyTorch fp32 / numpy fp64) functional restatement of the LAV per-frame
forward path (SURVEY.md §8a).  Every function takes plain tensors plus a
``state_dict`` (the reference's serialized key layout) and cites the reference
file:line it follows.  Only ``tests/``, ``__graft_entry__.smoke()`` and
``bench.py``'s cpu_baseline / ``--impl reference`` legs may import this module.

Pinning: ``oracle/pin_against_reference.py`` imports the real reference modules
from /root/reference (authoring container only), checks this restatement
against them on seeded inputs and writes ``tests/golden/*.npz``.  The reference
has no tests or golden vectors of its own (SURVEY.md §4), so the pin is "outputs
of the reference itself run here".  Two third-party pieces are NOT in
/root/reference and are restated from their published behaviour (unpinned):
``torch-scatter==2.0.7`` scatter_max/scatter_mean (Dockerfile:74) and
``carla.Transform.get_matrix`` (CARLA 0.9.10.1).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

CAMERA_YAWS = (-60, 0, 60)  # team_code_v2/model_inference.py:12


# ----------------------------------------------------------------------------
# a3: camera geometry — lav/utils/point_painting.py:5-43, model_inference.py:255-297
# ----------------------------------------------------------------------------

def carla_matrix(x=0.0, y=0.0, z=0.0, yaw=0.0, pitch=0.0, roll=0.0):
    """carla.Transform(...).get_matrix() restated (UE4 convention, degrees).
    CARLA 0.9.10 LibCarla/source/carla/geom/Transform.h GetMatrix — third party."""
    cy, sy = math.cos(math.radians(yaw)), math.sin(math.radians(yaw))
    cr, sr = math.cos(math.radians(roll)), math.sin(math.radians(roll))
    cp, sp = math.cos(math.radians(pitch)), math.sin(math.radians(pitch))
    return np.array([
        [cp * cy, cy * sp * sr - sy * cr, -cy * sp * cr - sy * sr, x],
        [cp * sy, sy * sp * sr + cy * cr, -sy * sp * cr + cy * sr, y],
        [sp, -cp * sr, cp * cr, z],
        [0.0, 0.0, 0.0, 1.0]], dtype=np.float64)


def converter_matrices(cam_yaw, lidar_xyz, cam_xyz, rgb_h, rgb_w, fov):
    """K (3,3), lidar_to_world (4,4), world_to_cam (4,4) in fp64.
    point_painting.py:6-25 / model_inference.py:259-274."""
    focal = rgb_w / (2.0 * np.tan(fov * np.pi / 360.0))
    K = np.identity(3)
    K[0, 0] = K[1, 1] = focal
    K[0, 2] = rgb_w / 2.0
    K[1, 2] = rgb_h / 2.0
    l2w = carla_matrix(*lidar_xyz)
    w2c = np.linalg.inv(carla_matrix(*cam_xyz, yaw=cam_yaw))
    return K, l2w, w2c


def default_converters(camera_x=1.5, camera_z=2.4, rgb_h=288, rgb_w=256, fov=64):
    """The three converters the agent builds (lav_agent_fast.py:131-134, model_inference.py:20-23)."""
    return [converter_matrices(yaw, [0, 0, camera_z], [camera_x, 0, camera_z], rgb_h, rgb_w, fov)
            for yaw in CAMERA_YAWS]


def lidar_to_cam_f32(lidar, conv):
    """fp32 torch twin: CoordConverter.forward, model_inference.py:280-297.  Returns (N,3) int64."""
    K, l2w, w2c = (torch.from_numpy(np.asarray(m)).float() for m in conv)
    xyz1 = torch.cat([lidar[:, :3], torch.ones_like(lidar[:, 0:1])], dim=-1).T
    world = l2w @ xyz1
    cam = w2c @ world
    cam = torch.stack([cam[1], -cam[2], cam[0]], dim=0)
    c2 = K @ cam
    c2 = torch.stack([c2[0] / (1e-5 + c2[2]), c2[1] / (1e-5 + c2[2]), c2[2]], dim=0).T
    return c2.long()


def lidar_to_cam_f64(lidar, conv):
    """numpy fp64 painter: CoordConverter.lidar_to_cam, point_painting.py:27-43."""
    K, l2w, w2c = conv
    lidar = np.asarray(lidar)
    xyz = lidar[:, :3].T
    xyz1 = np.r_[xyz, [np.ones(xyz.shape[1])]]
    world = l2w @ xyz1
    cam = w2c @ world
    cam = np.array([cam[1], -cam[2], cam[0]])
    c2 = K @ cam
    c2 = np.array([c2[0] / (1e-5 + c2[2]), c2[1] / (1e-5 + c2[2]), c2[2]]).T
    return c2.astype(int)


# ----------------------------------------------------------------------------
# a2/a4: painting — model_inference.py:44-50,75-93 ; point_painting.py:46-66
# ----------------------------------------------------------------------------

def suppress_background(pred_sem):
    """model_inference.py:45: p[:,1:] * (1 - p[:,:1])."""
    return pred_sem[:, 1:] * (1 - pred_sem[:, :1])


def point_painting_f32(lidar, sems, convs):
    """InferModel.point_painting, model_inference.py:75-93.  sems (ncam,C,H,W)."""
    sem_c, sem_h, sem_w = sems[0].shape
    painted = torch.zeros((len(lidar), sem_c), dtype=torch.float32)
    for sem, conv in zip(sems, convs):
        uvz = lidar_to_cam_f32(lidar, conv)
        u, v, z = uvz[:, 0], uvz[:, 1], uvz[:, 2]
        valid = (z >= 0) & (u >= 0) & (u < sem_w) & (v >= 0) & (v < sem_h)
        sel = uvz[valid]
        painted[valid] = sem[:, sel[:, 1], sel[:, 0]].T
    return painted


def point_painting_f64(lidar, sems, convs):
    """numpy painter, point_painting.py:46-66 (fp64 buffer and projection)."""
    lidar = np.asarray(lidar)
    sems = np.asarray(sems)
    sem_c, sem_h, sem_w = sems[0].shape
    painted = np.zeros((len(lidar), sem_c))
    for sem, conv in zip(sems, convs):
        uvz = lidar_to_cam_f64(lidar, conv)
        u, v, z = uvz[:, 0], uvz[:, 1], uvz[:, 2]
        valid = (z >= 0) & (u >= 0) & (u < sem_w) & (v >= 0) & (v < sem_h)
        sel = uvz[valid]
        painted[valid] = sem[:, sel[:, 1], sel[:, 0]].T
    return painted


def forward_paint(cur_lidar, pred_sem, convs):
    """InferModel.forward_paint, model_inference.py:44-50: (N,4)+(3,5,H,W softmaxed) -> (N,8)."""
    sem = suppress_background(pred_sem)
    painted = point_painting_f32(cur_lidar, sem, convs)
    return torch.cat([cur_lidar, painted], dim=-1)


# ----------------------------------------------------------------------------
# a5: ego-roof filter + sweep stacking — lav_agent.py:448-457, lav_agent_fast.py:363-383,547-565
# ----------------------------------------------------------------------------

def preprocess(lidar):
    """Drop the ego-roof box, lav_agent.py:448-457 (order preserving)."""
    x, y, z = lidar[:, 0], lidar[:, 1], lidar[:, 2]
    idx = (x > -2.4) & (x < 0) & (y > -0.8) & (y < 0.8) & (z > -1.5) & (z < -1)
    return lidar[~idx]


def move_lidar_points(xyz, dloc, ori0, ori1):
    """lav_agent_fast.py:547-565 (fp32 matmul of points, fp64 host trig)."""
    dloc = np.asarray(dloc, dtype=np.float64) @ np.array(
        [[np.cos(ori0), -np.sin(ori0)], [np.sin(ori0), np.cos(ori0)]])
    ori = ori1 - ori0
    R = torch.tensor([[np.cos(ori), np.sin(ori), 0], [-np.sin(ori), np.cos(ori), 0], [0, 0, 1]], dtype=torch.float)
    out = xyz @ R
    out[:, 0] += dloc[0]
    out[:, 1] += dloc[1]
    return out


def stack_lidar(sweeps, locs, oris, num_frame_stack=2):
    """get_stacked_lidar, lav_agent_fast.py:363-383.  ``sweeps`` newest first:
    sweeps[i] is the fused (n_i,8) sweep GAP*i ticks ago, locs/oris its ego pose."""
    loc0, ori0 = np.asarray(locs[0]), oris[0]
    rel = []
    for i, (s, loc, ori) in enumerate(zip(sweeps, locs, oris)):
        xyz = move_lidar_points(s[:, :3], np.asarray(loc) - loc0, ori0, ori)
        t = torch.zeros((len(xyz), num_frame_stack + 1), dtype=xyz.dtype)
        t[:, i] = 1
        rel.append(torch.cat([xyz, s[:, 3:], t], dim=-1))
    return torch.cat(rel)


# ----------------------------------------------------------------------------
# torch-scatter 2.0.7 restatement (third party, absent): segment max / mean
# ----------------------------------------------------------------------------

def scatter_max(src, index, num_segments):
    out = torch.full((num_segments, src.shape[1]), -float("inf"), dtype=src.dtype)
    out = out.scatter_reduce(0, index[:, None].expand_as(src), src, reduce="amax", include_self=True)
    return out


def scatter_mean(src, index, num_segments):
    s = torch.zeros((num_segments, src.shape[1]), dtype=src.dtype).index_add_(0, index, src)
    c = torch.zeros((num_segments,), dtype=src.dtype).index_add_(0, index, torch.ones_like(src[:, 0]))
    return s / c.clamp_min(1)[:, None]


# ----------------------------------------------------------------------------
# a6-a9: PointPillarNet — lav/models/point_pillar.py:55-116
# ----------------------------------------------------------------------------

def _bn(x, sd, p, eps, training=False, momentum=0.1):
    return F.batch_norm(x, None if training else sd[p + "running_mean"], None if training else sd[p + "running_var"],
                        sd[p + "weight"], sd[p + "bias"], training, momentum, eps)


def pillar_net(sd, lidar_list, num_points, prefix="point_pillar_net.", min_x=-10, max_x=70, min_y=-40, max_y=40,
               ppm=4, training=False, return_aux=False):
    """PointPillarNet.forward, point_pillar.py:92-116 -> canvas (B,C,ny,nx) NCHW fp32."""
    nx = (max_x - min_x) * ppm
    ny = (max_y - min_y) * ppm
    B = len(lidar_list)
    coords, pts = [], []
    for b, p in enumerate(lidar_list):
        p = p[:int(num_points[b])]
        keep = (p[:, 0] >= min_x) & (p[:, 0] < max_x) & (p[:, 1] >= min_y) & (p[:, 1] < max_y)   # :71-73
        p = p[keep]
        c = ((p[:, [0, 1]] - torch.tensor([min_x, min_y], dtype=p.dtype)) * ppm).long()            # :75-77
        coords.append(F.pad(c, (1, 0), value=b))
        pts.append(p)
    coords = torch.cat(coords)
    pts = torch.cat(pts)
    uniq, inv = coords.unique(return_inverse=True, dim=0)                                         # :82
    M = len(uniq)
    # decorate :55-68 (note the axis-swapped, un-centred cell origins)
    x_c = uniq[inv][:, 2:3].to(pts.dtype) / ppm + min_x
    y_c = uniq[inv][:, 1:2].to(pts.dtype) / ppm + min_y
    xyz = pts[:, :3]
    cluster = xyz - scatter_mean(xyz, inv, M)[inv]
    feat = torch.cat([pts, cluster, xyz[:, :1] - x_c, xyz[:, 1:2] - y_c], dim=-1)
    # DynamicPointNet :28-35 : Linear-BN1d-ReLU x2 then scatter_max
    q = prefix + "point_net.net."
    h = F.linear(feat, sd[q + "0.weight"], sd[q + "0.bias"])
    h = F.relu(_bn(h, sd, q + "1.", 1e-5, training))
    h = F.linear(h, sd[q + "3.weight"], sd[q + "3.bias"])
    h = F.relu(_bn(h, sd, q + "4.", 1e-5, training))
    fmax = scatter_max(h, inv, M)
    # scatter_points :87-90
    canvas = torch.zeros(B, fmax.shape[1], ny, nx, dtype=fmax.dtype)
    canvas[uniq[:, 0], :, torch.clamp(ny - 1 - uniq[:, 1], 0, ny - 1), torch.clamp(uniq[:, 2], 0, nx - 1)] = fmax
    if return_aux:
        return canvas, dict(decorated=feat, coords=coords, uniq=uniq, inv=inv, points=pts, point_feats=h)
    return canvas


# ----------------------------------------------------------------------------
# a10-a12: ConvBackbone / Head / LiDARModel — lav/models/lidar.py
# ----------------------------------------------------------------------------

def _crb(x, sd, p_conv, p_bn, stride, training=False):
    """Conv3x3(no bias) -> ReLU -> BN(eps 1e-3, momentum 0.01): lidar.py:57-60."""
    x = F.conv2d(x, sd[p_conv + "weight"], None, stride, 1)
    return _bn(F.relu(x), sd, p_bn, 1e-3, training, 0.01)


def conv_backbone(sd, x, prefix="backbone.", training=False):
    """ConvBackbone.forward, lidar.py:133-143."""
    def stage(x, name, n):
        for i in range(n):
            x = _crb(x, sd, f"{prefix}{name}.{3 * i}.", f"{prefix}{name}.{3 * i + 2}.", 2 if i == 0 else 1, training)
        return x
    x1 = stage(x, "conv1", 4)      # :56-70
    x2 = stage(x1, "conv2", 6)     # :72-91
    x3 = stage(x2, "conv3", 6)     # :93-112

    def up(x, name, stride, pad, opad):
        y = F.conv_transpose2d(x, sd[f"{prefix}{name}.0.weight"], None, stride, pad, opad)
        return _bn(F.relu(y), sd, f"{prefix}{name}.2.", 1e-3, training, 0.01)
    u1 = up(x1, "upconv1", 1, 0, 0)    # :114-118
    u2 = up(x2, "upconv2", 2, 1, 0)    # :120-125
    u3 = up(x3, "upconv3", 4, 1, 2)    # :127-131
    return torch.cat([u1, u2, u3], dim=1)


def head(sd, x, prefix, sigmoid=False, training=False):
    """Head.forward, lidar.py:147-164."""
    y = _crb(x, sd, prefix + "net.0.", prefix + "net.2.", 1, training)
    y = F.conv_transpose2d(y, sd[prefix + "net.3.weight"], sd[prefix + "net.3.bias"], 2, 1, 1)
    return torch.sigmoid(y) if sigmoid else y


def lidar_model(sd, lidars, num_points, training=False, **grid):
    """LiDARModel.forward, lidar.py:34-45 -> (features, center, box, ori, seg)."""
    canvas = pillar_net(sd, lidars, num_points, training=training, **grid)
    f = conv_backbone(sd, canvas, training=training)
    return (f, head(sd, f, "center_head.", training=training), head(sd, f, "box_head.", training=training),
            head(sd, f, "ori_head.", training=training), head(sd, f, "seg_head.", True, training=training))


# ----------------------------------------------------------------------------
# a1: ERFNet — lav/models/erfnet.py, rgb.py:41-45
# ----------------------------------------------------------------------------

def _erf_down(x, sd, p):
    """DownsamplerBlock, erfnet.py:12-23."""
    y = torch.cat([F.conv2d(x, sd[p + "conv.weight"], sd[p + "conv.bias"], 2, 1), F.max_pool2d(x, 2, 2)], 1)
    return F.relu(_bn(y, sd, p + "bn.", 1e-3))


def _erf_nb1d(x, sd, p, d):
    """non_bottleneck_1d, erfnet.py:26-61 (dropout inactive in eval)."""
    y = F.relu(F.conv2d(x, sd[p + "conv3x1_1.weight"], sd[p + "conv3x1_1.bias"], 1, (1, 0)))
    y = F.conv2d(y, sd[p + "conv1x3_1.weight"], sd[p + "conv1x3_1.bias"], 1, (0, 1))
    y = F.relu(_bn(y, sd, p + "bn1.", 1e-3))
    y = F.relu(F.conv2d(y, sd[p + "conv3x1_2.weight"], sd[p + "conv3x1_2.bias"], 1, (d, 0), (d, 1)))
    y = F.conv2d(y, sd[p + "conv1x3_2.weight"], sd[p + "conv1x3_2.bias"], 1, (0, d), (1, d))
    y = _bn(y, sd, p + "bn2.", 1e-3)
    return F.relu(y + x)


def _erf_up(x, sd, p):
    """UpsamplerBlock, erfnet.py:99-108."""
    y = F.conv_transpose2d(x, sd[p + "conv.weight"], sd[p + "conv.bias"], 2, 1, 1)
    return F.relu(_bn(y, sd, p + "bn.", 1e-3))


ERF_ENC_DILATIONS = [1] * 5 + [None] + [2, 4, 8, 16, 2, 4, 8, 16]   # erfnet.py:73-82


def erfnet(sd, rgb, prefix="erfnet."):
    """RGBSegmentationModel.forward, rgb.py:43-45: rgb (B,3,H,W) float 0..255 -> logits (B,5,H,W)."""
    x = (rgb / 255. - .5) * 2
    e = prefix + "encoder."
    x = _erf_down(x, sd, e + "initial_block.")
    x = _erf_down(x, sd, e + "layers.0.")
    for i in range(1, 6):
        x = _erf_nb1d(x, sd, f"{e}layers.{i}.", 1)
    x = _erf_down(x, sd, e + "layers.6.")
    for i, d in enumerate([2, 4, 8, 16, 2, 4, 8, 16]):
        x = _erf_nb1d(x, sd, f"{e}layers.{7 + i}.", d)
    d_ = prefix + "decoder."
    x = _erf_up(x, sd, d_ + "layers.0.")
    x = _erf_nb1d(x, sd, d_ + "layers.1.", 1)
    x = _erf_nb1d(x, sd, d_ + "layers.2.", 1)
    x = _erf_up(x, sd, d_ + "layers.3.")
    x = _erf_nb1d(x, sd, d_ + "layers.4.", 1)
    x = _erf_nb1d(x, sd, d_ + "layers.5.", 1)
    return F.conv_transpose2d(x, sd[d_ + "output_conv.weight"], sd[d_ + "output_conv.bias"], 2)


# ----------------------------------------------------------------------------
# a13: detection decode — model_inference.py:95-121,189-202 (fast agent thresholds)
# ----------------------------------------------------------------------------

def extract_peak(heatmap, max_pool_ks=7, max_det=15):
    """model_inference.py:189-202."""
    max_cls = F.max_pool2d(heatmap[None, None], max_pool_ks, 1, max_pool_ks // 2)[0, 0]
    possible = heatmap - (max_cls > heatmap).float() * 1e5
    max_det = min(max_det, possible.numel())
    return torch.topk(possible.view(-1), max_det)


def det_inference(heatmaps, sizemaps, orimaps, ppm=4, min_score=0.2):
    """InferModel.det_inference, model_inference.py:95-121 (heatmaps already sigmoided)."""
    dets = []
    for i, c in enumerate(heatmaps):
        det = []
        score, loc = extract_peak(c)
        peaks = [(float(s), int(l) % c.size(1), int(l) // c.size(1)) for s, l in zip(score, loc) if s > min_score]
        for s, x, y in peaks:
            w, h = float(sizemaps[0, y, x]), float(sizemaps[1, y, x])
            cos, sin = float(orimaps[0, y, x]), float(orimaps[1, y, x])
            if i == 1 and max(w, h) < 0.1 * ppm:
                continue
            dist = np.linalg.norm([x - 160, y - 280])
            if dist <= 2 or dist >= 30 * ppm:
                continue
            det.append((x, y, w, h, cos, sin))
        dets.append(det)
    return dets


# ----------------------------------------------------------------------------
# a14-a16: UniPlanner.infer — team_code_v2/models/uniplanner.py:186-352, resnet.py
# ----------------------------------------------------------------------------

def _cbr(x, sd, pc, pb, stride, pad, relu=True):
    y = F.conv2d(x, sd[pc + "weight"], sd.get(pc + "bias"), stride, pad)
    y = _bn(y, sd, pb, 1e-5)
    return F.relu(y) if relu else y


def resnet18_features(sd, x, p):
    """ResNet._forward_impl with BasicBlock [2,2,2,2], resnet.py:235-247,37-84 (no avgpool/fc)."""
    x = _cbr(x, sd, p + "conv1.", p + "bn1.", 2, 3)
    x = F.max_pool2d(x, 3, 2, 1)
    for li, stride in zip(range(1, 5), (1, 2, 2, 2)):
        for bi in range(2):
            q = f"{p}layer{li}.{bi}."
            s = stride if bi == 0 else 1
            idt = x
            y = _cbr(x, sd, q + "conv1.", q + "bn1.", s, 1)
            y = _cbr(y, sd, q + "conv2.", q + "bn2.", 1, 1, relu=False)
            if (q + "downsample.0.weight") in sd:
                idt = _cbr(x, sd, q + "downsample.0.", q + "downsample.1.", s, 0, relu=False)
            x = F.relu(y + idt)
    return x


def conv_emb(sd, x, p):
    """nn.Sequential(resnet18, AdaptiveAvgPool2d(1), Flatten): uniplanner.py:36-40."""
    return resnet18_features(sd, x, p + "0.").mean(dim=(2, 3))


def crop_feature(features, rel_locs, rel_oris, ppm, crop_size, offset_x, offset_y):
    """UniPlanner.crop_feature, team_code_v2/models/uniplanner.py:303-340 (= model_inference.py:204-238)."""
    B, C, H, W = features.shape
    rel_locs = rel_locs.view(-1, 2) * ppm / torch.tensor([H / 2, W / 2], dtype=rel_locs.dtype)
    cos, sin = torch.cos(rel_oris), torch.sin(rel_oris)
    rx, ry = rel_locs[..., 0], rel_locs[..., 1]
    k = crop_size / H
    rxo = -k * offset_x * cos + k * offset_y * sin + offset_x
    ryo = -k * offset_x * sin - k * offset_y * cos + offset_y
    theta = torch.stack([torch.stack([k * cos, k * -sin, rxo + rx], dim=-1),
                         torch.stack([k * sin, k * cos, ryo + ry], dim=-1)], dim=-2)
    grids = F.affine_grid(theta, torch.Size((B, C, crop_size, crop_size)), align_corners=True)
    return F.grid_sample(features, grids, align_corners=True)


def transform_points(locs, oris):
    """uniplanner.py:349-356."""
    cos, sin = torch.cos(oris), torch.sin(oris)
    R = torch.stack([torch.stack([cos, sin], dim=-1), torch.stack([-sin, cos], dim=-1)], dim=-2)
    return locs @ R


def gru_forward(sd, p, x, h0=None):
    """nn.GRU(batch_first=True, 1 layer) restated: gates r,z,n in PyTorch order."""
    w_ih, w_hh, b_ih, b_hh = (sd[p + n] for n in ("weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0"))
    B, T, _ = x.shape
    Hd = w_hh.shape[1]
    h = torch.zeros(B, Hd, dtype=x.dtype) if h0 is None else h0
    outs = []
    for t in range(T):
        gi = F.linear(x[:, t], w_ih, b_ih)
        gh = F.linear(h, w_hh, b_hh)
        i_r, i_z, i_n = gi.chunk(3, 1)
        h_r, h_z, h_n = gh.chunk(3, 1)
        r = torch.sigmoid(i_r + h_r)
        z = torch.sigmoid(i_z + h_z)
        n = torch.tanh(i_n + r * h_n)
        h = (1 - z) * n + z * h
        outs.append(h)
    return torch.stack(outs, dim=1)


def up_cast(sd, embd, num_cmds=6, num_plan=20, p=""):
    """UniPlanner.cast, team_code_v2/models/uniplanner.py:282-301 — 'other' mode re-uses the ego GRUs."""
    B = embd.size(0)
    u = embd.expand(num_plan, B, -1).permute(1, 0, 2)
    locs = []
    for i in range(num_cmds):
        out = gru_forward(sd, f"{p}cast_grus_ego.{i}.", u)
        locs.append(torch.cumsum(F.linear(out, sd[f"{p}cast_mlps_ego.{i}.weight"], sd[f"{p}cast_mlps_ego.{i}.bias"]), dim=1))
    return torch.stack(locs, dim=1)


def up_plan(sd, embd, nxp, cast_locs, ppm=4, crop_size=192, num_cmds=6, num_plan=20, num_plan_iter=5, p=""):
    """UniPlanner.plan/_plan, team_code_v2/models/uniplanner.py:249-280."""
    B = embd.size(0)
    plan_loc = cast_locs
    plans = []
    u0 = nxp * ppm / crop_size * 2 - 1
    for _ in range(num_plan_iter):
        locs = []
        for i in range(num_cmds):
            u = torch.cat([u0.expand(num_plan, B, -1).permute(1, 0, 2), plan_loc[:, i]], dim=2)
            out = gru_forward(sd, p + "plan_gru.", u, embd)
            locs.append(torch.cumsum(F.linear(out, sd[p + "plan_mlp.weight"], sd[p + "plan_mlp.bias"]), dim=1))
        plan_loc = torch.stack(locs, dim=1) + plan_loc
        plans.append(plan_loc)
    return torch.stack(plans, dim=1)


def uniplanner_infer(sd, features, det, cmd, nxp, ppm=4, crop_size=96, num_cmds=6, num_plan=20, num_plan_iter=5, p=""):
    """UniPlanner.infer, team_code_v2/models/uniplanner.py:186-247.
    features (384,160,160); det = list of (X,Y,w,h,cos,sin); returns
    (ego_embd, ego_plan_locs (20,2), ego_cast_locs (20,2), other_cast_locs (K,6,20,2), other_cast_cmds (K,6))."""
    offset_x, offset_y = sd[p + "offset_x"], sd[p + "offset_y"]   # 0-dim fp32 tensors, as in the module
    H, W = features.size(1) * 2, features.size(2) * 2
    cx = float(W / 2 + offset_x * W / 2)
    cy = float(H / 2 + offset_y * H / 2)
    locs, oris = [], []
    for X, Y, h, w, cos, sin in det:
        if np.linalg.norm([X - cx, Y - cy]) <= 4:
            continue
        locs.append([(X - cx) / ppm, (Y - cy) / ppm])
        oris.append(float(np.arctan2(sin, cos)))
    locs = torch.tensor(locs, dtype=torch.float32).view(-1, 2)
    oris = torch.tensor(oris, dtype=torch.float32)
    N = len(locs)
    if N > 0:
        crops = crop_feature(features.expand(N, *features.size()), locs, oris, ppm / 2, crop_size, offset_x, offset_y)
        oe = conv_emb(sd, crops, p + "lidar_conv_emb.")
        ocl = up_cast(sd, oe, num_cmds, num_plan, p)
        occ = torch.sigmoid(F.linear(oe, sd[p + "cast_cmd_pred.0.weight"], sd[p + "cast_cmd_pred.0.bias"]))
        ocl = transform_points(ocl, oris[:, None].repeat(1, num_cmds))
        ocl = ocl + locs.view(N, 1, 1, 2)
    else:
        ocl = torch.zeros((N, num_cmds, num_plan, 2))
        occ = torch.zeros((N, num_cmds))
    ego_crop = crop_feature(features[None], torch.zeros((1, 2)), torch.zeros((1,)), ppm / 2, crop_size, offset_x, offset_y)
    ee = conv_emb(sd, ego_crop, p + "lidar_conv_emb.")
    ecl = up_cast(sd, ee, num_cmds, num_plan, p)
    epl = up_plan(sd, ee, nxp[None], ecl, ppm, crop_size * 2, num_cmds, num_plan, num_plan_iter, p)[0, -1, cmd]
    return ee, epl, ecl[0, cmd], ocl, occ


# ----------------------------------------------------------------------------
# a19: brake model — team_code_v2/models/rgb.py:48-83, attention.py:6-56
# ----------------------------------------------------------------------------

def positional_encoding_1d(d_model, length):
    """attention.py:40-56."""
    pe = torch.zeros(length, d_model)
    position = torch.arange(0, length).unsqueeze(1)
    div = torch.exp(torch.arange(0, d_model, 2, dtype=torch.float) * -(math.log(10000.0) / d_model))
    pe[:, 0::2] = torch.sin(position.float() * div)
    pe[:, 1::2] = torch.cos(position.float() * div)
    return pe


def attention_pool(sd, p, x, num_heads=8):
    """Attention.forward, attention.py:20-38."""
    b, d, h, w = x.shape
    x = x.flatten(2).transpose(1, 2)
    kv = F.linear(x, sd[p + "linear_kv.weight"], sd[p + "linear_kv.bias"])
    k, v = kv.chunk(2, dim=-1)
    dh = d // num_heads
    k = k.view(b, h * w, num_heads, dh).transpose(1, 2) + positional_encoding_1d(dh, h * w)
    v = v.view(b, h * w, num_heads, dh).transpose(1, 2)
    q = sd[p + "q"].expand(b, -1, -1, -1)
    dots = torch.matmul(q, k.transpose(-1, -2)) * dh ** -0.5
    out = torch.matmul(torch.softmax(dots, dim=-1), v)
    return out.transpose(1, 2).reshape(b, d)


def brake_model(sd, rgb1, rgb2):
    """RGBBrakePredictionModel.forward(mask=False), team_code_v2/models/rgb.py:66-83."""
    mean = sd["normalize.mean"][None, :, None, None]
    std = sd["normalize.std"][None, :, None, None]
    x1 = resnet18_features(sd, (rgb1 / 255. - mean) / std, "conv_backbone.")
    x2 = resnet18_features(sd, (rgb2 / 255. - mean) / std, "conv_backbone.")
    h = torch.cat([attention_pool(sd, "attn1.", x1), attention_pool(sd, "attn2.", x2)], dim=1)
    return torch.sigmoid(F.linear(h, sd["classifier.0.weight"], sd["classifier.0.bias"]))[:, 0]


# ----------------------------------------------------------------------------
# whole frame (InferModel.forward, model_inference.py:53-73)
# ----------------------------------------------------------------------------

def infer_frame(lidar_sd, uni_sd, lidar_points, nxp, cmd, **grid):
    f, center, box, ori, seg = lidar_model(lidar_sd, [lidar_points], [len(lidar_points)], **grid)
    det = det_inference(torch.sigmoid(center[0]), box[0], ori[0])
    ee, epl, ecl, ocl, occ = uniplanner_infer(uni_sd, f[0], det[1], cmd, nxp)
    return ee, epl, ecl, ocl, occ, seg, det
