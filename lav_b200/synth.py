"""Seeded synthetic frames and weights (SURVEY.md §8d).

Nothing here touches the reference or the oracle: it only manufactures inputs
of the shapes the LAV frame path consumes (3 RGB cameras 288x256, a 40k-point
LiDAR sweep, ego poses for sweep stacking) and deterministic state_dict
contents for models whose released ``.th`` weights are git-LFS pointers.

All generators are CPU, seeded, and independent of module construction order,
so the authoring container, the GPU box and the golden fixtures agree.
"""
import hashlib
import math

import numpy as np
import torch

SEED = 2021  # reference default seed: lav/train_full_v2.py:68

RGB_H, RGB_W = 288, 256          # team_code_v2/lav_agent.py:53-55
SWEEP_POINTS = 40_000            # CARLA 600k pts/s, 2 ticks @20 Hz
CAMERA_YAWS = (-60, 0, 60)       # team_code_v2/lav_agent.py:35
CAMERA_X, CAMERA_Z = 1.5, 2.4    # team_code_v2/config.yaml:4-5


def _gen(seed, tag=""):
    h = hashlib.sha256(f"{seed}:{tag}".encode()).digest()
    g = torch.Generator(device="cpu")
    g.manual_seed(int.from_bytes(h[:7], "little"))
    return g


def lidar_sweep(n=SWEEP_POINTS, seed=SEED, tag="sweep", mode="carla"):
    """(n,4) fp32 x,y,z,intensity in the LiDAR frame (sensor at z=0).

    mode 'carla'   : r~U(2,85), az~U(-pi,pi), el~U(-30deg,+10deg), ground clip at z=-2.4
    mode 'uniform' : uniform in the BEV window (worst-case pillar count)
    mode 'adversarial': all points in 16 cells (atomic contention)
    """
    g = _gen(seed, tag + mode)
    if mode == "carla":
        r = torch.rand(n, generator=g) * 83.0 + 2.0
        az = (torch.rand(n, generator=g) * 2 - 1) * math.pi
        el = torch.rand(n, generator=g) * math.radians(40.0) - math.radians(30.0)
        down = el < 0
        rmax = torch.where(down, CAMERA_Z / torch.sin(-el).clamp_min(1e-3), torch.full_like(r, 1e9))
        r = torch.minimum(r, rmax)
        x = r * torch.cos(el) * torch.cos(az)
        y = r * torch.cos(el) * torch.sin(az)
        z = r * torch.sin(el)
    elif mode == "uniform":
        x = torch.rand(n, generator=g) * 79.9 - 9.95
        y = torch.rand(n, generator=g) * 79.9 - 39.95
        z = torch.rand(n, generator=g) * 3.0 - 2.4
    elif mode == "adversarial":
        cell = torch.randint(0, 16, (n,), generator=g)
        x = 10.0 + (cell % 4).float() * 0.25 + torch.rand(n, generator=g) * 0.24
        y = -2.0 + (cell // 4).float() * 0.25 + torch.rand(n, generator=g) * 0.24
        z = torch.rand(n, generator=g) * 2.0 - 2.0
    else:
        raise ValueError(mode)
    inten = torch.rand(n, generator=g)
    return torch.stack([x, y, z, inten], dim=1).float().contiguous()


def rgb_frames(seed=SEED, tag="rgb", smooth=False, n_cam=3, h=RGB_H, w=RGB_W):
    """(n_cam,h,w,3) uint8 RGB.  smooth=True gives low-pass noise so a trained
    segmenter's softmax is not degenerate."""
    g = _gen(seed, tag + str(smooth))
    if not smooth:
        return torch.randint(0, 256, (n_cam, h, w, 3), generator=g, dtype=torch.int64).to(torch.uint8)
    low = torch.rand(n_cam, 3, h // 16 + 1, w // 16 + 1, generator=g)
    img = torch.nn.functional.interpolate(low, size=(h, w), mode="bilinear", align_corners=True)
    img = img + 0.05 * torch.randn(n_cam, 3, h, w, generator=g)
    return (img.clamp(0, 1) * 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()


def sem_probs(seed=SEED, tag="sem", n_cam=3, c=5, h=RGB_H, w=RGB_W):
    """softmax of N(0,1) logits, (n_cam,c,h,w) fp32 (paint-only tests)."""
    g = _gen(seed, tag)
    return torch.softmax(torch.randn(n_cam, c, h, w, generator=g), dim=1).contiguous()


def ego_motion(n_sweeps=3, seed=SEED, tag="ego"):
    """poses (loc (n,2) fp64, ori (n,) fp64) for the stacked sweeps; index 0 = current."""
    g = _gen(seed, tag)
    loc = (torch.rand(n_sweeps, 2, generator=g, dtype=torch.float64) * 4 - 2)
    ori = (torch.rand(n_sweeps, generator=g, dtype=torch.float64) * 0.4 - 0.2)
    loc[0] = 0
    return loc.numpy(), ori.numpy()


def painted_sweep(n=SWEEP_POINTS, seed=SEED, tag="painted"):
    """(n,8) fp32: xyzI + 4 painted class probabilities (zeros for ~40% of points)."""
    g = _gen(seed, tag + "p")
    pts = lidar_sweep(n, seed, tag)
    sem = torch.rand(n, 4, generator=g) * (torch.rand(n, 1, generator=g) > 0.4)
    return torch.cat([pts, sem], dim=1).contiguous()


def stacked_lidar(n_per_sweep=SWEEP_POINTS, n_sweeps=3, seed=SEED, tag="stack"):
    """(P,11) fp32 stacked, ego-motion compensated sweeps with a one-hot time channel
    (same layout as lav_agent_fast.get_stacked_lidar, lav_agent_fast.py:363-383)."""
    loc, ori = ego_motion(n_sweeps, seed, tag)
    out = []
    for i in range(n_sweeps):
        s = painted_sweep(n_per_sweep, seed, f"{tag}{i}")
        d = ori[i] - ori[0]
        R = torch.tensor([[math.cos(d), math.sin(d), 0], [-math.sin(d), math.cos(d), 0], [0, 0, 1]], dtype=torch.float32)
        xyz = s[:, :3] @ R
        c0, s0 = math.cos(ori[0]), math.sin(ori[0])
        dl = (loc[i] - loc[0]) @ np.array([[c0, -s0], [s0, c0]])
        xyz[:, 0] += float(dl[0])
        xyz[:, 1] += float(dl[1])
        t = torch.zeros(n_per_sweep, n_sweeps)
        t[:, i] = 1
        out.append(torch.cat([xyz, s[:, 3:], t], dim=1))
    return torch.cat(out).contiguous()


# --------------------------------------------------------------------------- weights

def fill_state_dict_(sd, seed=SEED):
    """Deterministically overwrite every tensor of a state_dict in place.

    Values depend only on (seed, key, shape) so any process that builds a module
    with the same keys gets bit-identical weights.  BatchNorm statistics are
    non-trivial on purpose (identity BN hides folding bugs, SURVEY.md §7).
    """
    for k, v in sd.items():
        g = _gen(seed, "w:" + k)
        leaf = k.rsplit(".", 1)[-1]
        if leaf == "num_batches_tracked":
            v.fill_(100)
        elif leaf == "running_mean":
            v.copy_(torch.randn(v.shape, generator=g) * 0.1)
        elif leaf == "running_var":
            v.copy_(torch.rand(v.shape, generator=g) * 1.0 + 0.5)
        elif v.dim() == 0:
            pass  # scalar buffers/params (offset_x/offset_y) keep constructor values
        elif v.dim() == 1 and leaf == "weight" and ".bn2." in k:
            # last norm of a residual branch (ResNet BasicBlock / ERFNet nb1d): keep the branch
            # small so stacked residual adds stay O(1) with un-trained weights
            v.copy_(torch.rand(v.shape, generator=g) * 0.2 + 0.2)
        elif v.dim() == 1 and leaf == "weight":      # norm scale
            v.copy_(torch.rand(v.shape, generator=g) * 1.0 + 0.5)
        elif v.dim() == 1:                            # any bias
            v.copy_(torch.randn(v.shape, generator=g) * 0.1)
        elif k.endswith(".q") or leaf == "q":
            v.copy_(torch.randn(v.shape, generator=g))
        else:
            # conv / linear / gru weights.  ConvTranspose weights are (Cin,Cout,kh,kw);
            # Kaiming-ish scale on the contracted fan so deep ReLU stacks stay O(1).
            if v.dim() >= 3:
                rf = int(np.prod(v.shape[2:]))
                fan = v.shape[1] * rf
                if ".upconv" in k or ".output_conv" in k or _is_transposed_key(k):
                    fan = v.shape[0] * max(1, rf // 4)
            else:
                fan = v.shape[-1]
            std = math.sqrt(2.0 / max(fan, 1))
            if "gru" in k:
                std = 1.0 / math.sqrt(v.shape[-1])
            v.copy_(torch.randn(v.shape, generator=g) * std)
    return sd


def _is_transposed_key(k):
    # Head.net.3 (lidar.py:155), ERFNet UpsamplerBlock.conv / decoder.output_conv (erfnet.py:102,122)
    return k.endswith("_head.net.3.weight") or ("decoder.layers.0.conv" in k) or ("decoder.layers.3.conv" in k)


def bev_planner_batch(seed=SEED, B=3, n_actors=8, T=21, no_vehicles=False):
    """Seeded train_bev batch for the privileged planner: bev (B,9,320,320) uint8 0/1, ego_locs (B,T,2), cmds (B,), nxps (B,2),
    bras (B,), locs (B,n_actors,T,2) with slot 0 = the ego, oris (B,n_actors), typs (B,n_actors) int64.  Sample 0 has every actor
    a vehicle ahead (more than max_num_cars = 5: the multinomial path), sample 1 a mix, the last none.  ``no_vehicles``: no
    actor is a vehicle (the zero-placeholder path).  Used by oracle/pin_bev.py and the tests."""
    g = _gen(seed, f"bevbatch{B}{n_actors}{int(no_vehicles)}")
    bev = (torch.rand(B, 9, 320, 320, generator=g) > 0.7).to(torch.uint8)
    ego_locs = torch.cumsum(torch.rand(B, T, 2, generator=g) * torch.tensor([0.2, -1.0]), dim=1)
    locs = torch.randn(B, n_actors, T, 2, generator=g) * torch.tensor([5.0, 4.0]) + torch.tensor([0.0, -12.0])
    locs[:, 0] = ego_locs
    locs[-1, 1:, :, 1] = locs[-1, 1:, :, 1].abs() + 2.0                      # last sample: every actor behind the ego
    oris = torch.rand(B, n_actors, generator=g) * 0.6 - 0.3
    typs = torch.ones(B, n_actors, dtype=torch.int64)
    typs[1, 1::2] = 0
    if no_vehicles:
        typs[:] = 0
    cmds = torch.randint(0, 6, (B,), generator=g)
    nxps = torch.tensor([[0.0, -20.0]]).repeat(B, 1) + torch.randn(B, 2, generator=g)
    bras = torch.zeros(B, dtype=torch.int64)
    bras[1] = 1
    return bev, ego_locs, cmds, nxps, bras, locs, oris, typs


def loss_block_inputs(B=4, K=5, seed=SEED, num_cmds=6, num_plan=20, num_plan_iter=5):
    """Seeded stand-ins for everything the loss block of LAV.train_lidar consumes (lav/lav_final_v2.py:177-225): the five
    LiDARModel outputs, the eleven UniPlanner outputs and the targets.  Used by oracle/pin_against_reference.py (which feeds
    them to the REFERENCE's own train_lidar through stub sub-models) and by the tests (which feed lav_b200.train)."""
    g = _gen(seed, f"lossblock{B}")
    r = lambda *s: torch.randn(*s, generator=g)
    u = lambda *s: torch.rand(*s, generator=g)
    outs = (r(B, 384, 8, 8), r(B, 2, 320, 320) * 2, u(B, 2, 320, 320) * 3, r(B, 2, 320, 320), torch.sigmoid(r(B, 3, 320, 320)))
    planner = (r(K, num_plan, 2), r(K, num_cmds, num_plan, 2), torch.sigmoid(r(K, num_cmds)), r(K, num_cmds, num_plan, 2),
               torch.sigmoid(r(K, num_cmds)), r(B, num_plan, 2), r(B, num_plan_iter, num_cmds, num_plan, 2),
               r(B, num_cmds, num_plan, 2), torch.sigmoid(r(B, num_cmds)), r(B, num_cmds, num_plan, 2),
               r(B, num_plan_iter, num_cmds, num_plan, 2))
    yy, xx = torch.meshgrid(torch.arange(320.), torch.arange(320.), indexing="ij")
    heat = torch.zeros(B, 2, 320, 320)
    for b in range(B):
        for k in range(5):
            cx, cy = (u(2) * 320).tolist()
            heat[b, k % 2] = torch.maximum(heat[b, k % 2], torch.exp(-((xx - cx) ** 2 + (yy - cy) ** 2) / 18.0))
    targets = dict(heatmaps=heat, sizemaps=u(B, 2, 320, 320) * 3, orimaps=r(B, 2, 320, 320),
                   bev=(u(B, 9, 320, 320) > 0.7).to(torch.uint8), ego_locs=r(B, num_plan + 1, 2),
                   cmds=torch.randint(0, num_cmds, (B,), generator=g), bras=torch.tensor([0, 1, 0, 0][:B] + [0] * max(0, B - 4)))
    return outs, planner, targets


# --------------------------------------------------------------------------- recorded trajectories
def encode_png(gray):
    """(h, w) uint8 -> grayscale PNG bytes (cv2 when it imports, else a stored-filter zlib writer; both lossless)."""
    gray = np.ascontiguousarray(gray, dtype=np.uint8)
    try:
        import cv2
    except ImportError:
        cv2 = None
    if cv2 is not None:
        return cv2.imencode(".png", gray)[1].tobytes()
    import struct
    import zlib
    h, w = gray.shape

    def chunk(tag, data):
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)
    raw = b"".join(b"\x00" + gray[r].tobytes() for r in range(h))
    return (b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 0, 0, 0, 0)) +
            chunk(b"IDAT", zlib.compress(raw, 6)) + chunk(b"IEND", b""))


def decode_png(data):
    """grayscale PNG bytes -> (h, w) uint8, as cv2.imdecode(..., IMREAD_GRAYSCALE) (torchvision when cv2 is missing)."""
    try:
        import cv2
    except ImportError:
        cv2 = None
    buf = np.frombuffer(data, np.uint8)
    if cv2 is not None:
        return cv2.imdecode(buf, cv2.IMREAD_GRAYSCALE)
    from torchvision.io import ImageReadMode, decode_png as tv_decode
    return tv_decode(torch.from_numpy(buf.copy()), ImageReadMode.GRAY)[0].numpy()


def _road_planes(rs, h=320, w=320):
    """12 binary (0/255) map planes of one frame: a road band, lane lines, a crossing and a few boxes."""
    yy, xx = np.mgrid[:h, :w].astype(np.float64)
    planes = np.zeros((12, h, w), np.uint8)
    th = rs.uniform(-0.4, 0.4)
    off = rs.uniform(-30, 30)
    u = (xx - 160 - off) * np.cos(th) - (yy - 280) * np.sin(th)              # distance across the road
    v = (xx - 160 - off) * np.sin(th) + (yy - 280) * np.cos(th)              # along it
    cross = np.abs(v + rs.uniform(80, 200)) < rs.uniform(18, 30)
    road = (np.abs(u) < rs.uniform(25, 40)) | cross
    planes[0] = road * 255
    planes[1] = (road & (np.abs(np.abs(u) - 12) < 1.5)) * 255                # lane lines
    planes[2] = (road & (np.abs(u) < 1.2) & (np.mod(v, 24) < 12)) * 255       # dashed centre line
    for c in range(3, 12):
        for _ in range(rs.randint(0, 4)):
            cx, cy, a, b = rs.uniform(40, 280), rs.uniform(40, 300), rs.uniform(3, 9), rs.uniform(2, 5)
            planes[c] |= ((np.abs(xx - cx) < a) & (np.abs(yy - cy) < b)).astype(np.uint8) * 255
    return planes


TEL_H, TEL_W = 288, 480          # the telephoto camera before crop_tel_bottom (team_code_v2/lav_agent.py:53-55)


def _blobs(rs, h, w, n, values, base):
    """(h, w) uint8: ``base`` with ``n`` axis-aligned rectangles, each filled with one draw from ``values``."""
    img = np.full((h, w), base, np.uint8)
    for _ in range(n):
        y0, x0 = rs.randint(0, h), rs.randint(0, w)
        img[y0:y0 + rs.randint(4, h // 3), x0:x0 + rs.randint(4, w // 3)] = rs.choice(values)
    return img


def _camera_images(rs, n_cameras, jpeg):
    """the camera keys of one frame: rgb_{c} (288 x 256 colour, PNG or ``jpeg``), sem_{c} (grayscale PNG of tags 0..22 on a
    background of 0, so listed tags, unlisted tags and background all occur) for each of ``n_cameras``, and tel_rgb (288 x 480)."""
    import cv2
    enc = (lambda im: cv2.imencode(".jpg", im, [cv2.IMWRITE_JPEG_QUALITY, 90])[1].tobytes()) if jpeg else \
        (lambda im: cv2.imencode(".png", im)[1].tobytes())

    def colour(h, w):
        low = rs.randint(0, 256, (h // 16 + 1, w // 16 + 1, 3)).astype(np.uint8)
        return cv2.resize(low, (w, h), interpolation=cv2.INTER_LINEAR)
    keys = {}
    for c in range(n_cameras):
        keys[f"rgb_{c}"] = enc(colour(RGB_H, RGB_W))
        keys[f"sem_{c}"] = encode_png(_blobs(rs, RGB_H, RGB_W, 12, np.arange(23), 0))
    keys["tel_rgb"] = enc(colour(TEL_H, TEL_W))
    return keys


def record_trajectories(root, n_traj=2, n_frames=30, seed=SEED, n_points=600, n_actors=12, seg_channels=4,
                        towns=("Town01", "Town03", "Town02", "Town04", "Town05", "Town06"), images=False, n_cameras=3):
    """Write ``n_traj`` seeded synthetic trajectories of ``n_frames`` frames under ``root`` in the reference's record layout
    (basic_dataset.py:52-53,82-157, temporal_lidar_painted_dataset.py:29-30), through data_paint.DirEnv (one file per key):
      len, town; lidar_%05d (n,4) f32; lidar_sem_%05d (n,C) f32; map_{0..11}_%05d grayscale PNG (0/255);
      id (int32, ego first), loc (f32 (n,2) metres), ori (f32 degrees), bbox (f32 (n,2)), type (uint8), cmd / bra (uint8),
      nxp (f32 (2,)) per frame.
    With ``images`` every frame also holds the camera keys of the image datasets (seg_dataset.py, bra_dataset.py):
      rgb_{c}_%05d for c < n_cameras (PNG; JPEG in trajectory 1), sem_{c}_%05d (grayscale PNG of CARLA tags), tel_rgb_%05d
      (288 x 480, encoded as the rgb keys).  They come from a RandomState of their own, so every other key keeps its bytes.
    The ego drives a smooth arc; the other actors move smoothly, some leave before the last frame, some are out of range.
    Returns the trajectory directories."""
    import os
    from .data_paint import DirEnv
    paths = []
    for k in range(n_traj):
        rs = np.random.RandomState(int.from_bytes(hashlib.sha256(f"{seed}:traj{k}".encode()).digest()[:4], "little"))
        path = os.path.join(root, f"traj_{k:03d}")
        env = DirEnv(path)
        env.put("len", str(n_frames).encode())
        env.put("town", towns[k % len(towns)].encode())
        speed, yaw0, yaw_rate = rs.uniform(6, 12) / 20, rs.uniform(-180, 180), rs.uniform(-3, 3)
        start = rs.uniform(-100, 100, 2)
        ego_id = int(rs.randint(1, 100))
        ids = ego_id + 1 + rs.choice(5000, n_actors, replace=False)
        a_typ = (rs.rand(n_actors) > 0.35).astype(np.uint8)                  # 1 vehicle, 0 pedestrian
        a_off = rs.uniform(-25, 25, (n_actors, 2))
        a_off[-2:] *= 3                                                       # two actors beyond the radius cuts
        a_vel = rs.uniform(-0.4, 0.4, (n_actors, 2))
        a_ori = rs.uniform(-180, 180, n_actors)
        a_box = np.where(a_typ[:, None] == 1, rs.uniform(1.8, 2.6, (n_actors, 2)), rs.uniform(0.3, 0.5, (n_actors, 2)))
        a_last = np.where(rs.rand(n_actors) < 0.3, rs.randint(n_frames // 3, n_frames, n_actors), n_frames)   # leaves after a_last
        rs_img = np.random.RandomState(int.from_bytes(hashlib.sha256(f"{seed}:img{k}".encode()).digest()[:4], "little"))
        for f in range(n_frames):
            if images:
                for key, data in _camera_images(rs_img, n_cameras, jpeg=k == 1).items():
                    env.put(f"{key}_{f:05d}", data)
            yaw = yaw0 + yaw_rate * f
            heading = np.deg2rad(yaw0 + yaw_rate * f / 2)
            ego_loc = start + speed * f * np.array([np.cos(heading), np.sin(heading)])
            here = np.nonzero(f < a_last)[0]
            locs = np.concatenate([ego_loc[None], ego_loc + a_off[here] + a_vel[here] * f])
            env.put(f"id_{f:05d}", np.concatenate([[ego_id], ids[here]]).astype(np.int32).tobytes())
            env.put(f"loc_{f:05d}", locs.astype(np.float32).tobytes())
            env.put(f"ori_{f:05d}", np.concatenate([[yaw], a_ori[here] + 2 * f]).astype(np.float32).tobytes())
            env.put(f"bbox_{f:05d}", np.concatenate([[[2.4, 1.1]], a_box[here]]).astype(np.float32).tobytes())
            env.put(f"type_{f:05d}", np.concatenate([[1], a_typ[here]]).astype(np.uint8).tobytes())
            env.put(f"cmd_{f:05d}", np.array([rs.randint(0, 6)], np.uint8).tobytes())
            env.put(f"bra_{f:05d}", np.array([rs.rand() < 0.2], np.uint8).tobytes())
            env.put(f"nxp_{f:05d}", (ego_loc + rs.uniform(-20, 20, 2)).astype(np.float32).tobytes())
            pts = lidar_sweep(n_points, seed, f"rec{k}_{f}").numpy()
            pts[:25, :3] = np.array([-1.2, 0.0, -1.25]) + rs.uniform(-0.3, 0.3, (25, 3)) * [1, 1, 0.5]   # ego-roof returns
            sem = rs.rand(n_points, seg_channels) * (rs.rand(n_points, 1) > 0.4)
            env.put(f"lidar_{f:05d}", pts.astype(np.float32).tobytes())
            env.put(f"lidar_sem_{f:05d}", sem.astype(np.float32).tobytes())
            for c, plane in enumerate(_road_planes(rs)):
                env.put(f"map_{c}_{f:05d}", encode_png(plane))
        paths.append(path)
    return paths
