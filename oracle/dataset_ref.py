"""numpy restatement of TemporalLiDARPaintedDataset.__getitem__ (lav/utils/datasets/temporal_lidar_painted_dataset.py:15-179) and
the helpers it calls (basic_dataset.py:81-157, lidar_dataset.py:14-23,92-182), for the tests and for oracle/pin_dataset.py.

No cv2: ``warp_affine_u8`` restates cv2.warpAffine for uint8 images with INTER_LINEAR and a constant-zero border in OpenCV's own
fixed-point arithmetic (imgwarp.cpp: AB_BITS = 10, INTER_BITS = 5, INTER_REMAP_COEF_BITS = 15), so it is bit-identical to it.
The random draws of the sample (rotation jitter, stack jitters, shuffle permutation) are arguments, so a run of the reference
with seeded generators can be replayed exactly.
"""
import math

import numpy as np
import torch

BEV_CENTER = (160, 280)          # rotate_image's default image_center (lidar_dataset.py:159)


# --------------------------------------------------------------------------- OpenCV's fixed-point warp
def rotation_matrix_2d(center, angle_deg):
    """cv2.getRotationMatrix2D(center, angle, 1.0): the angle is scaled by the constant pi/180 (not multiplied by pi, then divided)."""
    a = angle_deg * (math.pi / 180)
    c, s = math.cos(a), math.sin(a)
    cx, cy = center
    return np.array([[c, s, (1 - c) * cx - s * cy], [-s, c, s * cx + (1 - c) * cy]], dtype=np.float64)


def invert_affine(M):
    """the inverse cv::warpAffine computes from the forward matrix (same operation order, so the same roundings)."""
    det = M[0, 0] * M[1, 1] - M[0, 1] * M[1, 0]
    d = 1.0 / det if det != 0 else 0.0
    a11, a22, a12, a21 = M[1, 1] * d, M[0, 0] * d, -M[0, 1] * d, -M[1, 0] * d
    b1 = -a11 * M[0, 2] - a12 * M[1, 2]
    b2 = -a21 * M[0, 2] - a22 * M[1, 2]
    return np.array([[a11, a12, b1], [a21, a22, b2]], dtype=np.float64)


def fixed_coords(Minv, h, w):
    """source coordinates of every output pixel in 1/32 pixel: (X, Y) int64 (h, w).  np.rint is round-half-to-even like cvRound."""
    xs, ys = np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64)
    rint = lambda v: np.rint(v).astype(np.int64)
    X = (rint((Minv[0, 1] * ys + Minv[0, 2]) * 1024)[:, None] + 16 + rint(Minv[0, 0] * xs * 1024)[None, :]) >> 5
    Y = (rint((Minv[1, 1] * ys + Minv[1, 2]) * 1024)[:, None] + 16 + rint(Minv[1, 0] * xs * 1024)[None, :]) >> 5
    return X, Y


def warp_affine_u8(img, M, dsize=None):
    """cv2.warpAffine(img, M, dsize, flags=INTER_LINEAR) for uint8 (h, w) or (h, w, c) with the default zero border."""
    h, w = img.shape[:2]
    ow, oh = dsize if dsize is not None else (w, h)
    X, Y = fixed_coords(invert_affine(np.asarray(M, dtype=np.float64)), oh, ow)
    sx, fx, sy, fy = X >> 5, X & 31, Y >> 5, Y & 31
    src = img.reshape(h, w, -1).astype(np.int64)
    acc = np.zeros((oh, ow, src.shape[2]), np.int64)
    for ox, oy, wt in ((0, 0, (32 - fx) * (32 - fy)), (1, 0, fx * (32 - fy)), (0, 1, (32 - fx) * fy), (1, 1, fx * fy)):
        tx, ty = sx + ox, sy + oy
        inside = (tx >= 0) & (tx < w) & (ty >= 0) & (ty < h)
        v = src[np.clip(ty, 0, h - 1), np.clip(tx, 0, w - 1)] * inside[..., None]
        acc += v * (wt * 32)[..., None]
    out = np.minimum((acc + 16384) >> 15, 255).astype(np.uint8)
    return out.reshape((oh, ow) + img.shape[2:])


def rotate_image(img, angle_deg, center=BEV_CENTER):
    """lidar_dataset.rotate_image (:159-163)."""
    return warp_affine_u8(img, rotation_matrix_2d(center, angle_deg))


def load_bev_channels(planes, angle=0.0, angle_offset=0.0, loc=(0, 0), margin=32):
    """load_bev_channels (temporal_lidar_painted_dataset.py:182-198) after load_bev: planes (h, w, c) uint8 -> (c, h, w) 0/1.
    Raises ValueError when the shift leaves the margin (the reference's slice assignment fails there)."""
    dx, dy = (int(v) for v in loc)
    if abs(dx) > margin or abs(dy) > margin:
        raise ValueError(f"BEV shift ({dx}, {dy}) exceeds the {margin}-pixel margin")
    h, w = planes.shape[:2]
    a = rotate_image(planes, -angle * 180 / math.pi)
    padded = np.zeros((h + 2 * margin, w + 2 * margin) + planes.shape[2:], np.uint8)
    padded[margin:margin + h, margin:margin + w] = a
    crop = np.ascontiguousarray(padded[dx + margin:dx + margin + h, dy + margin:dy + margin + w])
    b = rotate_image(crop, angle_offset)
    return (b > 0).astype(np.uint8).reshape(h, w, -1).transpose(2, 0, 1)


# --------------------------------------------------------------------------- record access and the actor filter
def access(get, tag, index, dtype=np.float32):
    """BasicDataset.access(tag, txn, index, 1, dtype) for one frame; ``get(key: str) -> bytes``."""
    return np.frombuffer(get(f"{tag}_{index:05d}"), dtype)[None]


def filter_actors(get, index, max_pedestrian_radius=10, max_vehicle_radius=20, T=10):
    """BasicDataset.filter (basic_dataset.py:103-157): the actors of frame ``index`` seen in every frame index..index+T and inside
    their type's radius.  -> ego_id, ego_locs (T+1,2), ego_oris (T+1,), {id: locs}, {id: oris}, {id: bbox}, {id: typs}."""
    ids0 = access(get, "id", index, np.int32).ravel()
    ego = ids0[0]
    seen = {a: np.zeros(T + 1) for a in ids0}
    locs = {a: np.zeros((T + 1, 2)) for a in ids0}
    oris = {a: np.zeros(T + 1) for a in ids0}
    bbox = {a: np.zeros((T + 1, 2)) for a in ids0}
    typs = {a: np.zeros(T + 1) for a in ids0}
    for k in range(T + 1):
        f = index + k
        rows = zip(access(get, "id", f, np.int32).ravel(), access(get, "loc", f).reshape(-1, 2), access(get, "ori", f).ravel(),
                   access(get, "bbox", f).reshape(-1, 2), access(get, "type", f, np.uint8).ravel())
        for a, l, o, b, ty in rows:
            if a in seen:
                seen[a][k], locs[a][k], oris[a][k], bbox[a][k], typs[a][k] = 1, l, np.deg2rad(o), b, ty
    ego_locs, ego_oris = locs[ego], oris[ego]
    drop = {a for a in seen if not seen[a].all()}
    for a in seen:
        r = np.linalg.norm(locs[a][0] - ego_locs[0])
        if (typs[a][0] == 0 and r > max_pedestrian_radius) or (typs[a][0] == 1 and r > max_vehicle_radius):
            drop.add(a)
    keep = [a for a in seen if a not in drop]
    pick = lambda d: {a: d[a] for a in keep}
    return ego, ego_locs, ego_oris, pick(locs), pick(oris), pick(bbox), pick(typs)


def transform_ego(ego_locs, locs, oris, bbox, typs, ego_ori, T=11):
    """lidar_dataset.transform_ego: actors sorted by id, positions rotated into the ego frame."""
    keys = sorted(locs)
    stack = lambda d, shape: np.array([d[k] for k in keys]).reshape(shape)
    L, O, B, Y = stack(locs, (-1, T, 2)), stack(oris, (-1, T)), stack(bbox, (-1, T, 2)), stack(typs, (-1, T))
    R = [[np.sin(ego_ori), np.cos(ego_ori)], [-np.cos(ego_ori), np.sin(ego_ori)]]
    origin = ego_locs[0]
    return (ego_locs - origin) @ R, (L - origin) @ R, O - ego_ori, B, Y


def rotate_points(points, angle_deg, center):
    r = np.deg2rad(angle_deg)
    return (points - center) @ [[np.cos(r), np.sin(r)], [-np.sin(r), np.cos(r)]] + center


def detections_to_heatmap(locs, oris, bbox, typs, min_x=-10, max_x=70, min_y=-40, max_y=40, pixels_per_meter=4, radius=1):
    """LiDARDataset.detections_to_heatmap (lidar_dataset.py:92-127) in fp32 torch on the CPU."""
    h, w = (max_y - min_y) * pixels_per_meter, (max_x - min_x) * pixels_per_meter
    heat, size, orim = torch.zeros((2, h, w)), torch.zeros((2, h, w)), torch.zeros((2, h, w))
    for c in (0, 1):
        sel = typs == c
        if sel.sum() == 0:
            continue
        loc, ori, box = (torch.tensor(a[sel], dtype=torch.float32) for a in (locs, oris, bbox))
        cx = -loc[:, 0] * pixels_per_meter + (max_y - min_y) * pixels_per_meter / 2
        cy = -loc[:, 1] * pixels_per_meter + h + min_x * pixels_per_meter
        gx = (-((torch.arange(w)[:, None] - cx[None]) / radius) ** 2).exp()
        gy = (-((torch.arange(h)[:, None] - cy[None]) / radius) ** 2).exp()
        g, who = (gx[None] * gy[:, None]).max(dim=-1)
        m = g > heat.max(dim=0)[0]
        size[:, m] = box.T[:, who[m]] * pixels_per_meter
        orim[0, m] = torch.cos(ori[who[m]])
        orim[1, m] = torch.sin(ori[who[m]])
        heat[c] = g
    return heat, size, orim


# --------------------------------------------------------------------------- the whole sample
def decode_png_gray(data):
    from lav_b200.synth import decode_png
    return decode_png(data)


def get_item(get, index, cfg, angle, jitters, perm, convs):
    """TemporalLiDARPaintedDataset.__getitem__ for frame ``index`` of one recording (``get(key) -> bytes``), with the draws given:
    angle (degrees), jitters[i] = (loc_jitter (2,), ori_jitter) of the i-th stacked frame (ignored for i = 0), perm = the
    shuffle permutation of the stacked rows (None: unshuffled).  ``convs``: oracle.lav_ref converters of cameras camera_yaws[1:-1].
    Returns the reference's 14-tuple (numpy / torch as the reference returns them)."""
    from oracle import lav_ref as O
    T, ppm = cfg["num_plan"], cfg["pixels_per_meter"]
    radii = dict(max_pedestrian_radius=cfg["max_pedestrian_radius"], max_vehicle_radius=cfg["max_vehicle_radius"], T=T)
    nseg = len(cfg["seg_channels"])
    frames = [i for i in range(index, index - cfg["num_frame_stack"] - 1, -1) if i >= 0]
    rows = []
    poses = {i: filter_actors(get, i, **radii)[1:3] for i in frames}
    loc0, ori0 = poses[index][0][0], poses[index][1][0]
    for t, i in enumerate(frames):
        xyzr = access(get, "lidar", i).reshape(-1, 4)
        painted = access(get, "lidar_sem", i).reshape(-1, nseg)
        roof = (xyzr[:, 0] > -2.4) & (xyzr[:, 0] < 0) & (xyzr[:, 1] > -0.8) & (xyzr[:, 1] < 0.8) & (xyzr[:, 2] > -1.5) & (xyzr[:, 2] < -1)
        xyzr, painted = xyzr[~roof], painted[~roof]
        r = np.deg2rad(-angle)
        xyzr = xyzr @ [[np.cos(r), np.sin(r), 0, 0], [-np.sin(r), np.cos(r), 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]]
        painted = painted * O.point_painting_f64(xyzr, np.ones((len(convs), 1, 288, 256)), convs)
        lj, oj = (0, 0) if t == 0 else jitters[t]
        loc, ori = poses[i][0][0], poses[i][1][0]
        dloc = (loc - loc0 + lj) @ [[np.cos(ori0), -np.sin(ori0)], [np.sin(ori0), np.cos(ori0)]]
        d = ori + oj - ori0
        xyzr = xyzr @ [[np.cos(d), np.sin(d), 0, 0], [-np.sin(d), np.cos(d), 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]]
        xyzr[:, :2] += dloc
        one_hot = np.zeros((len(xyzr), cfg["num_frame_stack"] + 1), np.float32)
        one_hot[:, t] = 1
        rows.append(np.concatenate([xyzr.astype(np.float32), painted.astype(np.float32), one_hot], 1))
    lidar = np.concatenate(rows)
    lidar = lidar[(np.arange(len(lidar)) if perm is None else np.asarray(perm))[:cfg["max_lidar_points"]]]
    num_points = min(cfg["max_lidar_points"], sum(len(r) for r in rows))
    padded_lidar = np.zeros((cfg["max_lidar_points"], lidar.shape[1]), np.float32)
    padded_lidar[:num_points] = lidar[:num_points]

    cmd = int(access(get, "cmd", index, np.uint8)[0, 0])
    bra = int(access(get, "bra", index, np.uint8)[0, 0])
    nxp = access(get, "nxp", index).reshape(2)
    _, e_locs, e_oris, locs, oris, bbox, typs = filter_actors(get, index, **radii)
    ego_locs, locs, oris, bbox, typs = transform_ego(e_locs, locs, oris, bbox, typs, e_oris[0], T + 1)

    bev = np.zeros((3 + 2 * (cfg["num_frame_stack"] + 1), 320, 320), np.uint8)
    bev[:3] = load_bev_channels(load_planes(get, index, (0, 9, 10)), angle_offset=angle)
    for t, i in enumerate(frames):
        loc, ori = poses[i][0][0], poses[i][1][0]
        dl = (loc - loc0) @ [[np.cos(ori0), -np.sin(ori0)], [np.sin(ori0), np.cos(ori0)]] * ppm
        bev[3 + 2 * t:5 + 2 * t] = load_bev_channels(load_planes(get, i, (1, 2)), angle=ori - ori0, angle_offset=angle, loc=dl)

    locs = rotate_points(locs, -angle, ego_locs[0])
    oris[1:] = oris[1:] - np.deg2rad(angle)
    grid = {k: cfg[k] for k in ("min_x", "max_x", "min_y", "max_y", "pixels_per_meter")}
    heat, size, orim = detections_to_heatmap(locs[:, 0], oris[:, 0], bbox[:, 0], typs[:, 0], **grid)
    n_obj = min(len(locs), cfg["max_objs"])
    p_locs = np.zeros((cfg["max_objs"], T + 1, 2), np.float32)
    p_oris = np.zeros((cfg["max_objs"],), np.float32)
    p_typs = np.zeros((cfg["max_objs"],), np.int32)
    p_locs[:n_obj], p_oris[:n_obj], p_typs[:n_obj] = locs[:n_obj], oris[:n_obj, 0], typs[:n_obj, 0]
    # the reference's second filter (max_mot_vehicle_radius) only re-derives ego_locs, which no radius changes
    ego_locs = rotate_points(ego_locs, -angle, ego_locs[0])
    nxp = rotate_points(nxp, -angle, ego_locs[0])
    return (padded_lidar, num_points, heat, size, orim, bev, -ego_locs, cmd, -nxp, bra, -p_locs, p_oris, p_typs, n_obj)


def load_planes(get, index, channels):
    """BasicDataset.load_bev: grayscale PNG planes map_{c}_%05d stacked (h, w, c)."""
    return np.stack([decode_png_gray(get(f"map_{c}_{index:05d}")) for c in channels], axis=-1)
