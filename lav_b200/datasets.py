"""Training data from recorded trajectories: TemporalLiDARPaintedDataset (lav/utils/datasets/temporal_lidar_painted_dataset.py)
with its per-sample work on the GPU and a batch loader for LAVTrainer.train_lidar; TemporalBEVDataset
(lav/utils/datasets/temporal_bev_dataset.py) and its loader for BEVTrainer.train_bev.

Recording layout: the reference's keys (basic_dataset.py:52-53,82-101; data_paint.py writes lidar_sem_%05d), one key-value
environment per trajectory directory (LMDB when the `lmdb` package imports and data.mdb exists, else data_paint.DirEnv).

What runs where:
    record reads, PNG chunk walk (png.parse)                      host, a background thread of the loader
    PNG inflate and unfilter of the map planes                     device, one ops.png_decode_gray8 launch per batch on a side
                                                                   stream (PNGs other than 8-bit grayscale: synth.decode_png)
    actor filter, ego transform, label padding (a few hundred floats)   host, vectorised numpy
    LiDAR: roof filter, rotation, FOV re-mask, stacking, shuffle   device, data_pipeline.GpuLidarStacker (per sample), or for a
                                                                   batch its index tables on the host and one ops.lidar_batch
    heat / size / orientation maps                                 device, data_pipeline.detections_to_heatmap (per sample), or
                                                                   one ops.det_heatmaps launch per batch
    the 9-plane temporal BEV target (2 warpAffine per plane)       device, ops.bev_targets: one launch per batch, bit-identical
                                                                   to the reference's OpenCV chain
"""
import glob
import math
import os
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch
import yaml

from . import data_paint, ops, png
from .capi import LavbError
from .data_pipeline import GpuLidarStacker, detections_to_heatmap

TRAIN_TOWNS = ("Town01", "Town03", "Town04", "Town06")          # basic_dataset.py:9
BEV_SIZE = 320


def index_trajectories(data_dir, percentage_data, all_towns, num_plan, seed):
    """BasicDataset.__init__'s sample list (basic_dataset.py:29-72): one coin toss per entry of ``data_dir`` (seeded like
    np.random.seed(seed)), entries without a data.mdb (or a directory store) skipped, the TRAIN_TOWNS filter unless all_towns;
    frame indices 0 .. len - num_plan - 1 of each kept trajectory.  Entries are visited in sorted order (the reference takes
    the file system's order).  -> (list of trajectory paths, list of (trajectory number, frame index))."""
    rs = np.random.RandomState(seed)
    paths, index = [], []
    for path in sorted(glob.glob(os.path.join(data_dir, "*"))):
        if rs.random_sample() > percentage_data:
            continue
        if not (os.path.exists(os.path.join(path, "data.mdb")) or os.path.isdir(os.path.join(path, "kv"))):
            continue
        env = data_paint.open_env(path)
        n, town = int(env.get("len")), env.get("town").decode()
        env.close()
        if not all_towns and town not in TRAIN_TOWNS:
            continue
        paths.append(path)
        index += [(len(paths) - 1, i) for i in range(n - num_plan)]
    return paths, index


def _frame(env, tag, i, dtype=np.float32):
    return np.frombuffer(env.get(f"{tag}_{i:05d}"), dtype)


def ego_pose(env, i):
    """world pose of the ego (the first id of frame i) as BasicDataset.filter reads it: loc (2,) f64, yaw in radians."""
    ids = _frame(env, "id", i, np.int32)
    r = np.nonzero(ids == ids[0])[0][-1]
    return _frame(env, "loc", i).reshape(-1, 2)[r].astype(np.float64), float(np.deg2rad(_frame(env, "ori", i)[r:r + 1])[0])


def _read_tracks(env, index, T):
    """the records of frames index .. index + T for the actors of frame ``index``, sorted by id: seen (N,T+1), world locs
    (N,T+1,2), oris (N,T+1) in radians, bbox (N,T+1,2), typs (N,T+1), zero where unseen; and the ego's row."""
    ids0 = _frame(env, "id", index, np.int32)
    ego = ids0[0]
    uid = np.unique(ids0)
    n = len(uid)
    seen = np.zeros((n, T + 1), bool)
    locs, oris = np.zeros((n, T + 1, 2)), np.zeros((n, T + 1))
    bbox, typs = np.zeros((n, T + 1, 2)), np.zeros((n, T + 1))
    for k in range(T + 1):
        ids = _frame(env, "id", index + k, np.int32)
        pos = np.clip(np.searchsorted(uid, ids), 0, n - 1)
        hit = uid[pos] == ids
        p = pos[hit]
        seen[p, k] = True
        locs[p, k] = _frame(env, "loc", index + k).reshape(-1, 2)[hit]
        oris[p, k] = np.deg2rad(_frame(env, "ori", index + k)[hit])
        bbox[p, k] = _frame(env, "bbox", index + k).reshape(-1, 2)[hit]
        typs[p, k] = _frame(env, "type", index + k, np.uint8)[hit]
    return seen, locs, oris, bbox, typs, int(np.searchsorted(uid, ego))


def _ego_transform(locs, oris, e):
    """(origin, R, ego yaw) of transform_ego: ego-frame points are (p - origin) @ R."""
    ego_ori = oris[e, 0]
    return locs[e, 0].copy(), [[np.sin(ego_ori), np.cos(ego_ori)], [-np.cos(ego_ori), np.sin(ego_ori)]], ego_ori


def _label_tracks(tracks, max_pedestrian_radius, max_vehicle_radius):
    seen, locs, oris, bbox, typs, e = tracks
    ego_locs = locs[e].copy()
    r = np.linalg.norm(locs[:, 0] - ego_locs[0], axis=1)
    keep = seen.all(1) & ~((typs[:, 0] == 0) & (r > max_pedestrian_radius)) & ~((typs[:, 0] == 1) & (r > max_vehicle_radius))
    origin, R, ego_ori = _ego_transform(locs, oris, e)
    return (ego_locs - origin) @ R, (locs[keep] - origin) @ R, oris[keep] - ego_ori, bbox[keep], typs[keep]


def actor_tracks(env, index, T, max_pedestrian_radius, max_vehicle_radius):
    """BasicDataset.filter + transform_ego (basic_dataset.py:103-157, lidar_dataset.py:132-148), vectorised.
    -> ego_locs (T+1,2), locs (N,T+1,2), oris (N,T+1), bbox (N,T+1,2), typs (N,T+1) in the ego frame of ``index``, actors sorted
    by id (the ego is one of them)."""
    return _label_tracks(_read_tracks(env, index, T), max_pedestrian_radius, max_vehicle_radius)


def _safety_table(tracks, first=1):
    """the actor table of steps first .. T of ``tracks`` (plan_safety_table: first = 1, driving_score_table: first = 0)."""
    seen, locs, oris, bbox, typs, e = tracks
    origin, R, ego_ori = _ego_transform(locs, oris, e)
    others = np.arange(len(seen)) != e
    present = seen[others, first:]
    yaw = oris[others, first:] - ego_ori
    only = lambda a: np.where(present.reshape(present.shape + (1,) * (a.ndim - 2)), a, 0)
    return dict(locs=only(-((locs[others, first:] - origin) @ R)), cos=only(np.cos(yaw)), sin=only(np.sin(yaw)),
                bbox=only(bbox[others, first:]), typ=only(typs[others, first:]).astype(np.int32), present=present,
                ego_bbox=bbox[e, 0].copy())


def plan_safety_table(env, index, T):
    """The actors an ego plan of sample ``index`` is checked against (lav_b200.evaluate, --plan-safety): every actor of frame
    ``index`` but the ego, with no radius filter, at steps 1..T (frames index + 1 .. index + T), in actor_tracks' id order.
    -> dict: locs (N,T,2) fp64 in the label frame (actor_tracks' ego frame, negated as the labels are), cos / sin (N,T) fp64 of
    the yaw relative to the ego (the actor heads along (sin, -cos) there), bbox (N,T,2) = the recorded half extents, typ (N,T)
    int32, present (N,T) bool (the id appears in that frame; the other entries are zero); ego_bbox (2,) = the ego's bbox at
    frame ``index``."""
    return _safety_table(_read_tracks(env, index, T))


def _plan_safety_of(tracks, wanted, augmented):
    """the plan_safety_table of a prepared sample when ``wanted``; its label frame is the unaugmented one."""
    if not wanted:
        return None
    if augmented:
        raise LavbError("plan_safety_table: the table is in the unaugmented label frame; the sample is rotated or shifted")
    return _safety_table(tracks)


def driving_score_table(env, index, T):
    """The actors an ego plan of sample ``index`` is scored against by the driving score (lav_b200.evaluate, --driving-score):
    plan_safety_table's actors, records and layout, at steps 0..T (frames index .. index + T), so that step 0 gives each actor's
    pose before the plan's first step.  -> the dict of plan_safety_table with T + 1 steps per actor."""
    return _safety_table(_read_tracks(env, index, T), first=0)


def _driving_score_of(tracks, wanted, augmented):
    """the driving_score_table of a prepared sample when ``wanted``; its label frame is the unaugmented one."""
    if not wanted:
        return None
    if augmented:
        raise LavbError("driving_score_table: the table is in the unaugmented label frame; the sample is rotated or shifted")
    return _safety_table(tracks, first=0)


def stage_plan_safety(tables, pin):
    """the plan_safety_table (or driving_score_table) of each sample of a batch packed for ops.plan_safety (ops.driving_score):
    actors = PLAN_SAFETY_ACTOR_DTYPE records as a 1-D uint8 tensor (sample i's rows, then within a row its steps), offsets (B+1,)
    int32 = the actor rows of each sample, ego_ext (B,2) fp64; pinned on ``pin``."""
    T = tables[0]["locs"].shape[1] if tables else 0
    rec = np.zeros((sum(len(s["locs"]) for s in tables), T), ops.PLAN_SAFETY_ACTOR_DTYPE)
    offsets = np.concatenate([[0], np.cumsum([len(s["locs"]) for s in tables])]).astype(np.int32)
    for s, a0, a1 in zip(tables, offsets[:-1], offsets[1:]):
        r = rec[a0:a1]
        r["x"], r["y"], r["cos"], r["sin"] = s["locs"][..., 0], s["locs"][..., 1], s["cos"], s["sin"]
        r["e1"], r["e2"], r["typ"], r["present"] = s["bbox"][..., 0], s["bbox"][..., 1], s["typ"], s["present"]
    ego = np.array([s["ego_bbox"] for s in tables], np.float64).reshape(-1, 2)
    tensor = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    out = dict(actors=tensor(rec.reshape(-1).view(np.uint8)), offsets=tensor(offsets), ego_ext=tensor(ego))
    return {k: v.pin_memory() for k, v in out.items()} if pin else out


def rotate_points(points, angle_deg, center):
    r = np.deg2rad(angle_deg)
    return (points - center) @ [[np.cos(r), np.sin(r)], [-np.sin(r), np.cos(r)]] + center


class TemporalLiDARPaintedDataset:
    """TemporalLiDARPaintedDataset (temporal_lidar_painted_dataset.py) over a recording, built on ``device``.

    Same constructor, YAML keys, ``len`` and index mapping as the reference (BasicDataset, with the trajectories in sorted order);
    ``ds[i]`` returns its 14-tuple as device tensors: lidar (max_lidar_points, 4+C+T) f32, num_points, heatmaps / sizemaps /
    orimaps (2,320,320) f32, bev (9,320,320) uint8, -ego_locs (T+1,2) f64, cmd, -nxp (2,) f64, bra, -locs (max_objs,T+1,2) f32,
    oris (max_objs,) f32, typs (max_objs,) int32, num_objs.  ``sample(idx, angle, jitters, generator)`` takes the random draws
    explicitly; ``ds[i]`` draws them from generators seeded with ``seed``.  The draws have the reference's distributions but not
    its random streams: the same seed gives other (equally distributed) augmentations than the reference.  ``overrides``
    replaces keys of the YAML (the evaluator's --data-dir)."""

    def __init__(self, config_path, seed=2021, device=torch.device("cuda"), overrides=None):
        with open(config_path) as f:
            cfg = yaml.safe_load(f)
        cfg.update(overrides or {})
        self.cfg = cfg
        for k, v in cfg.items():
            setattr(self, k, v)
        self.device = torch.device(device)
        self.margin = ops.BEV_MARGIN
        self.paths, self.index = index_trajectories(self.data_dir, self.percentage_data, self.all_towns, self.num_plan, seed)
        self._envs, self._env_lock = {}, threading.Lock()
        self._decode_stream = None
        self.stacker = GpuLidarStacker(self.num_frame_stack, len(self.seg_channels), self.max_lidar_points, self.camera_x,
                                       self.camera_z, device=self.device)
        self.rng = np.random.RandomState(seed)
        self.gen = torch.Generator(device="cpu").manual_seed(seed)

    def __len__(self):
        return len(self.index)

    def env(self, traj):
        with self._env_lock:                        # the loaders' threads share it: open each environment once per process
            if traj not in self._envs:
                self._envs[traj] = data_paint.open_env(self.paths[traj])
            return self._envs[traj]

    def draw(self, rng):
        """(angle in degrees, stack jitters) with the reference's distributions (temporal_lidar_painted_dataset.py:21,50-51)."""
        angle = float(rng.uniform(-1, 1)) * self.angle_jitter
        jit = [(np.zeros(2), 0.0)] + [(rng.uniform(-self.stack_loc_jitter, self.stack_loc_jitter, 2),
                                       float(rng.uniform(-self.stack_ori_jitter, self.stack_ori_jitter)))
                                      for _ in range(self.num_frame_stack)]
        return angle, jit

    def no_draw(self):
        """the draws of an unaugmented sample: angle 0 and zero stack jitters."""
        return 0.0, [(np.zeros(2), 0.0)] * (self.num_frame_stack + 1)

    # ---- host part: record reads, PNG chunk walks, labels, BEV job rows
    def prepare(self, idx, angle, jitters, plan_safety=False, cameras=False, paint=False, driving_score=False):
        """the host record of sample ``idx``; with ``plan_safety`` (unaugmented samples only) it also holds the sample's
        plan_safety_table, from the same record reads, and with ``driving_score`` its driving_score_table; with ``cameras``, under "cameras", what CameraDataset reads for the brake
        model (read_cameras: the three middle cameras of camera_yaws and tel_rgb[:-crop_tel_bottom]).  With ``paint`` (online
        painting) no lidar_sem key is read: each sweep carries its frame index where the painted rows would be, and "traj" the
        trajectory, for stage_batch's frame table."""
        traj, index = self.index[idx]
        env = self.env(traj)
        cams = read_cameras(env, index, brake_cameras(len(self.camera_yaws), "TemporalLiDARPaintedDataset"),
                            self.crop_tel_bottom) if cameras else None
        T, nseg = self.num_plan, len(self.seg_channels)
        radii = (self.max_pedestrian_radius, self.max_vehicle_radius)
        frames = [i for i in range(index, index - self.num_frame_stack - 1, -1) if i >= 0]
        tracks = _read_tracks(env, index, T)
        table = _plan_safety_of(tracks, plan_safety, angle != 0)
        driving = _driving_score_of(tracks, driving_score, angle != 0)
        ego_locs, locs, oris, bbox, typs = _label_tracks(tracks, *radii)
        poses = {i: ego_pose(env, i) for i in frames}
        loc0, ori0 = poses[index]
        sweeps = [(_frame(env, "lidar", i).reshape(-1, 4), i if paint else _frame(env, "lidar_sem", i).reshape(-1, nseg), poses[i][0],
                   poses[i][1]) for i in frames]
        pngs = [self.map_png(traj, env, c, index) for c in (0, 9, 10)]
        rows = [(c, c, 0.0, angle, 0, 0) for c in range(3)]                                   # load_bev_channels(angle=0, loc=0)
        ppm = self.pixels_per_meter
        for t, i in enumerate(frames):
            loc, ori = poses[i]
            dl = (loc - loc0) @ [[np.cos(ori0), -np.sin(ori0)], [np.sin(ori0), np.cos(ori0)]] * ppm
            dx, dy = map(int, dl)
            if abs(dx) > self.margin or abs(dy) > self.margin:
                raise LavbError(f"frame {i} of {self.paths[traj]}: BEV shift ({dx}, {dy}) px exceeds the {self.margin}-pixel margin")
            for c in (1, 2):
                rows.append((len(pngs), 3 + 2 * t + c - 1, -(ori - ori0) * 180 / math.pi, angle, dx, dy))
                pngs.append(self.map_png(traj, env, c, i))
        rows += [(-1, 3 + 2 * t + c, 0.0, 0.0, 0, 0) for t in range(len(frames), self.num_frame_stack + 1) for c in (0, 1)]

        locs = rotate_points(locs, -angle, ego_locs[0])
        oris[1:] = oris[1:] - np.deg2rad(angle)
        n_obj = min(len(locs), self.max_objs)
        p_locs = np.zeros((self.max_objs, T + 1, 2), np.float32)
        p_oris = np.zeros((self.max_objs,), np.float32)
        p_typs = np.zeros((self.max_objs,), np.int32)
        p_locs[:n_obj], p_oris[:n_obj], p_typs[:n_obj] = locs[:n_obj], oris[:n_obj, 0], typs[:n_obj, 0]
        ego_rot = rotate_points(ego_locs, -angle, ego_locs[0])
        nxp = rotate_points(_frame(env, "nxp", index).reshape(2), -angle, ego_rot[0])
        h = dict(sweeps=sweeps, angle=angle, jitters=jitters, pngs=pngs, rows=rows,
                 det=(locs[:, 0], oris[:, 0], bbox[:, 0], typs[:, 0]), ego_locs=-ego_rot, nxp=-nxp,
                 cmd=int(_frame(env, "cmd", index, np.uint8)[0]), bra=int(_frame(env, "bra", index, np.uint8)[0]),
                 locs=-p_locs, oris=p_oris, typs=p_typs, num_objs=n_obj)
        if table is not None:
            h["plan_safety"] = table
        if driving is not None:
            h["driving_score"] = driving
        if cams is not None:
            h["cameras"] = cams
        if paint:
            h["traj"] = traj
        return h

    def paint_images(self, traj, i):
        """the painting cameras' images of frame ``i`` of trajectory ``traj``: rgb_0 .. rgb_2 (point_painting.CAMERA_YAWS, the
        cameras data_paint reads) decoded by load_img -> (3, 288, 256, 3) uint8 RGB.  A missing key or an image of another size is
        a LavbError naming the trajectory and the key."""
        env, what = self.env(traj), self.paths[traj]
        h, w = self.stacker.rgb_hw
        imgs = []
        for c in range(len(self.stacker.cams)):
            key = f"rgb_{c}_{i:05d}"
            try:
                img = load_img(env, f"rgb_{c}", i)
            except LavbError as e:
                raise LavbError(f"{what}: {e}") from None
            if img.shape != (h, w, 3):
                raise LavbError(f"{what}: record key {key} is {img.shape[1]} x {img.shape[0]}, the painting cameras' images are "
                                f"{w} x {h}")
            imgs.append(img)
        return np.stack(imgs)

    def stage_paint(self, hs, pin, pool=None):
        """the frame table of a batch prepared with ``paint``: its distinct (trajectory, frame) pairs in first-use order (sample
        order, each sample's sweeps newest first), each pair's images decoded once by paint_images (on ``pool`` when given) into
        one (F, 3, 288, 256, 3) uint8 buffer (pinned on ``pin``), and the samples' sweeps with each frame index replaced by its
        slot.  -> (dict(images, pairs), [sweeps of each sample])."""
        slot, pairs, sweeps = {}, [], []
        for h in hs:
            mine = []
            for xyzr, i, loc, ori in h["sweeps"]:
                key = (h["traj"], int(i))
                if key not in slot:
                    slot[key] = len(pairs)
                    pairs.append(key)
                mine.append((xyzr, slot[key], loc, ori))
            sweeps.append(mine)
        imgs = list((pool.map if pool is not None else map)(lambda k: self.paint_images(*k), pairs))
        h, w = self.stacker.rgb_hw
        buf = torch.empty((len(pairs), len(self.stacker.cams), h, w, 3), dtype=torch.uint8, pin_memory=pin)
        dst = buf.numpy()
        for f, img in enumerate(imgs):
            dst[f] = img
        return dict(images=buf, pairs=pairs), sweeps

    # ---- device part
    def lidar_and_maps(self, h, generator=None):
        lidar, num = self.stacker(h["sweeps"], h["angle"], h["jitters"], generator=generator)
        grid = dict(min_x=self.min_x, max_x=self.max_x, min_y=self.min_y, max_y=self.max_y, pixels_per_meter=self.pixels_per_meter)
        heat, size, orim = detections_to_heatmap(*h["det"], device=self.device, **grid)
        return lidar, num, heat, size, orim

    def map_png(self, traj, env, c, i):
        """("trajectory path: key", png.parse of map plane c of frame i): the zlib stream for the device decoder, or a
        host-decoded plane."""
        key = f"map_{c}_{i:05d}"
        what = f"{self.paths[traj]}: {key}"
        return what, png.parse(env.get(key), what, BEV_SIZE)

    def decode_maps(self, maps):
        """the map planes staged by stage_maps -> (planes (P, 320, 320) uint8 on the device, the event after which they are ready).
        Decodes on a side stream and waits for that stream's event, not the device; raises LavbError naming the key of a
        malformed plane, so no batch is built from it.  The caller's stream does not wait: see planes_on_stream."""
        dev = self.device
        with torch.cuda.device(dev):
            if self._decode_stream is None:
                self._decode_stream = torch.cuda.Stream(dev)
            with torch.cuda.stream(self._decode_stream):
                planes = torch.empty((maps["n_planes"], BEV_SIZE, BEV_SIZE), dtype=torch.uint8, device=dev)
                status = ops.png_decode_gray8(maps["src"].to(dev, non_blocking=True), maps["jobs"], planes)
                for p, plane in maps["host"]:
                    planes[p].copy_(plane, non_blocking=True)
                status_h = torch.empty(status.shape, dtype=torch.int32, pin_memory=True)
                status_h.copy_(status, non_blocking=True)
                ready = torch.cuda.Event()
                ready.record()
        ready.synchronize()
        bad = np.nonzero(status_h.numpy())[0]
        if len(bad):
            raise LavbError("malformed PNG map plane(s): " + ", ".join(f"{maps['keys'][maps['jobs']['dst'][j]]} (status "
                                                                        f"{int(status_h[j])})" for j in bad))
        return planes, ready

    def planes_on_stream(self, decoded):
        """the planes of decode_maps, ordered after the decode on the current stream."""
        planes, ready = decoded
        torch.cuda.current_stream(self.device).wait_event(ready)
        planes.record_stream(torch.cuda.current_stream(self.device))
        return planes

    def bev_batch(self, hs, decoded=None):
        """one map decode and one bev_targets launch for the samples ``hs`` -> (len(hs), 9, 320, 320) uint8 on the device;
        ``decoded`` = decode_maps of their stage_maps when done ahead."""
        n_bev = 3 + 2 * (self.num_frame_stack + 1)
        planes = self.planes_on_stream(decoded or self.decode_maps(stage_maps(hs, self.device.type == "cuda")))
        out = torch.empty((len(hs), n_bev, BEV_SIZE, BEV_SIZE), dtype=torch.uint8, device=self.device)
        return ops.bev_targets(planes, bev_job_table(hs, n_bev), out)

    def sample(self, idx, angle, jitters, generator=None):
        """the 14-tuple of sample ``idx`` for the given draws: angle (degrees), jitters[i] = (loc (2,), ori) of stacked frame i
        (index - i; entry 0 is unused), generator = torch generator of the LiDAR row shuffle."""
        h = self.prepare(idx, angle, jitters)
        lidar, num, heat, size, orim = self.lidar_and_maps(h, generator)
        bev = self.bev_batch([h])[0]
        dev = self.device
        return (lidar, num, heat, size, orim, bev, torch.as_tensor(h["ego_locs"], device=dev), h["cmd"],
                torch.as_tensor(h["nxp"], device=dev), h["bra"], torch.as_tensor(h["locs"], device=dev),
                torch.as_tensor(h["oris"], device=dev), torch.as_tensor(h["typs"], device=dev), h["num_objs"])

    def __getitem__(self, idx):
        angle, jit = self.draw(self.rng)
        return self.sample(idx, angle, jit, self.gen)

    # ---- a whole batch: host tables (any thread), then a fixed number of launches and H2D copies (the caller's thread)
    def stage_batch(self, hs, generator=None, pool=None):
        """the host tables of a batch of prepared samples ``hs``, in pinned memory on a CUDA dataset.  Draws the LiDAR
        shuffles from ``generator`` (CPU) in sample order, as one sample() per entry of ``hs`` would.  Samples prepared with
        ``paint`` also stage their frame table and images under "paint" (stage_paint, the decodes on ``pool``), and the LiDAR
        tables carry raw (N, 4) rows and a frame slot per sweep."""
        pin = self.device.type == "cuda"
        pinned = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory() if pin else torch.from_numpy(np.ascontiguousarray(a))
        paint = bool(hs) and "traj" in hs[0]
        painting, sweeps = self.stage_paint(hs, pin, pool) if paint else (None, [h["sweeps"] for h in hs])
        lidar = self.stacker.batch_tables([(sw, h["angle"], h["jitters"]) for sw, h in zip(sweeps, hs)], generator, paint=paint)
        dets = [np.column_stack([np.reshape(locs, (-1, 2)), oris, np.reshape(bbox, (-1, 2)), typs]) for locs, oris, bbox, typs in
                (h["det"] for h in hs)]
        offsets = np.concatenate([[0], np.cumsum([len(d) for d in dets])]).astype(np.int32)
        f32 = lambda key: np.stack([h[key] for h in hs]).astype(np.float32)
        labels = dict(ego_locs=f32("ego_locs"), nxp=f32("nxp"), locs=f32("locs"), oris=f32("oris"),
                      typs=np.stack([h["typs"] for h in hs]).astype(np.int32),
                      cmd=np.array([h["cmd"] for h in hs], np.int64), bra=np.array([h["bra"] for h in hs], np.int64))
        st = dict(lidar=lidar, actors=pinned(np.concatenate(dets + [np.zeros((0, 6))]).astype(np.float32)),
                  offsets=pinned(offsets), maps=stage_maps(hs, pin),
                  bev_jobs=bev_job_table(hs, 3 + 2 * (self.num_frame_stack + 1)),
                  labels={k: pinned(v) for k, v in labels.items()}, num_objs=[h["num_objs"] for h in hs])
        if hs and "plan_safety" in hs[0]:                                       # prepared with plan_safety (the evaluator)
            st["plan_safety"] = stage_plan_safety([h["plan_safety"] for h in hs], pin)
        if hs and "driving_score" in hs[0]:                                     # prepared with driving_score (the evaluator)
            st["driving_score"] = stage_plan_safety([h["driving_score"] for h in hs], pin)
        if hs and "cameras" in hs[0]:                                           # prepared with cameras (the brake evaluation)
            st["cameras"] = stage_images([h["cameras"] for h in hs], ("rgbs", "tel"), pin, "TemporalLiDARPaintedDataset")
        if painting is not None:
            st["paint"] = painting
        return st

    def paint_features(self, st, seg_model):
        """forward_features_nhwc of ``seg_model`` over the F x 3 staged images of a batch staged with "paint", in one call ->
        (features, deconv table, n_classes)."""
        if seg_model is None:
            raise LavbError("the batch was prepared for online painting: launch_batch needs the segmentation model")
        imgs = st["paint"]["images"]
        F_, ncam, h, w, _ = imgs.shape
        return seg_model.forward_features_nhwc(imgs.to(self.device, non_blocking=True).view(F_ * ncam, h, w, 3))

    @torch.no_grad()
    def launch_batch(self, st, seg_model=None):
        """the device half of a batch staged by stage_batch: the map decode (unless decode_maps ran ahead), lidar_batch,
        det_heatmaps and bev_targets, and the H2D copies; the only device-to-host read is the decode's status, on its own stream
        -> the loader's 14-tuple.  A batch staged with "paint" runs ``seg_model`` once over its frame table's images
        (paint_features) and takes lidar_batch_paint's one launch instead of lidar_batch."""
        dev = self.device
        to = lambda t: t.to(dev, non_blocking=True)
        painting = self.paint_features(st, seg_model) if "paint" in st else None
        lidar = self.stacker.batch_launch(st["lidar"], painting)
        grid = dict(min_x=self.min_x, max_x=self.max_x, min_y=self.min_y, max_y=self.max_y, pixels_per_meter=self.pixels_per_meter)
        heat, size, orim = ops.det_heatmaps(to(st["actors"]), to(st["offsets"]), grid)
        planes = self.planes_on_stream(st.get("decoded") or self.decode_maps(st["maps"]))
        bev = torch.empty((len(st["num_objs"]), 3 + 2 * (self.num_frame_stack + 1), BEV_SIZE, BEV_SIZE), dtype=torch.uint8, device=dev)
        ops.bev_targets(planes, st["bev_jobs"], bev)
        lab = {k: to(v) for k, v in st["labels"].items()}
        return (lidar, torch.tensor(st["lidar"]["nums"], dtype=torch.int64), heat, size, orim, bev, lab["ego_locs"], lab["cmd"],
                lab["nxp"], lab["bra"], lab["locs"], lab["oris"], lab["typs"], torch.tensor(st["num_objs"], dtype=torch.int64))

    def sample_batch(self, idxs, draws, generator=None):
        """the loader's 14-tuple for the samples ``idxs`` with the draws ``draws[i] = (angle, jitters)``; the LiDAR shuffles come
        from ``generator`` (CPU) in sample order.  Equal, tensor for tensor, to stacking sample(idxs[i], *draws[i], generator) in
        order, with the device work in a fixed number of launches."""
        hs = [self.prepare(int(i), *d) for i, d in zip(idxs, draws)]
        return self.launch_batch(self.stage_batch(hs, generator))


def stage_maps(hs, pin):
    """the map planes of the prepared samples ``hs``, concatenated in order: their zlib streams packed into one (pinned on
    ``pin``) buffer with the PNG_JOB_DTYPE job table, the host-decoded planes, and each plane's key."""
    parsed = [p for h in hs for _, p in h["pngs"]]
    src, jobs, host = png.pack(parsed, BEV_SIZE)
    src = torch.from_numpy(src.copy())
    host = [(p, torch.from_numpy(plane.copy())) for p, plane in host]
    if pin:
        src, host = src.pin_memory(), [(p, t.pin_memory()) for p, t in host]
    return dict(src=src, jobs=jobs, host=host, keys=[k for h in hs for k, _ in h["pngs"]], n_planes=len(parsed))


def bev_job_table(hs, n_bev):
    """BEV_JOB_DTYPE records of the prepared samples ``hs``, their planes concatenated in order, sample b's output planes at
    b * n_bev + d."""
    rows, base = [], 0
    for b, h in enumerate(hs):
        rows += [(s + base if s >= 0 else -1, b * n_bev + d, a1, a2, dx, dy) for s, d, a1, a2, dx, dy in h["rows"]]
        base += len(h["pngs"])
    return ops.bev_jobs(rows)


class TemporalBatchLoader:
    """Batches of ``dataset`` for LAVTrainer.train_lidar, one rank of ``world``.

    Each epoch shuffles the sample list with a permutation seeded by (seed, epoch) — the same on every rank — and rank r takes
    every world-th entry; every rank yields the same number of batches (len // world // batch_size with drop_last).  The draws
    of an epoch come from a RandomState (angle and jitters, on the caller's thread) and a torch CPU generator (the LiDAR
    shuffles), both seeded by (seed, epoch, rank) and taken in sample order.  While batch k is on the GPU, a background thread
    builds batch k+1: record reads, PNG chunk walks and labels on ``num_workers`` threads, then the tables of
    TemporalLiDARPaintedDataset.stage_batch and the map decode on a side stream (decode_maps, which raises before a batch with
    a malformed map is yielded); the rest of the device part is launch_batch.  A batch is the 14-tuple
    lidars (B,P,4+C+T) f32, num_points (B,) int64 (host), heatmaps / sizemaps / orimaps (B,2,320,320) f32, bev (B,9,320,320)
    uint8, ego_locs (B,T+1,2) f32, cmds (B,) int64, nxps (B,2) f32, bras (B,) int64, locs (B,max_objs,T+1,2) f32, oris
    (B,max_objs) f32, typs (B,max_objs) int32, num_objs (B,) int64; train_lidar takes the first 13.

    With ``ordered`` (evaluation) the samples come in index order with no augmentation, rank r taking the contiguous range
    [r * n // world, (r + 1) * n // world): every draw is dataset.no_draw(), and the LiDAR shuffles still come from the
    generator of (seed, epoch, rank).  With ``plan_safety`` (ordered only) every sample is
    prepared with its plan_safety_table, and the staged tables carry them packed under "plan_safety" (stage_plan_safety); with
    ``driving_score`` (ordered only) the same with its driving_score_table, under "driving_score".  With
    ``cameras`` every sample is prepared with the brake model's camera images, and the staged tables carry them under "cameras"
    as one pinned uint8 buffer per key: rgbs (B, 3, h, w, 3), tel (B, h_tel, w_tel, 3).

    With ``seg_model`` (an RGBSegmentationModel, set to the caller's precision) the sweeps are painted online instead of read
    from lidar_sem: every sample is prepared with ``paint``, the batch's distinct (trajectory, frame) pairs are decoded once each
    on the ``num_workers`` threads (stage_paint; in ordered mode a batch of 32 consecutive samples has about 34 of them), and
    launch_batch runs the model once over their images and lidar_batch_paint once; the staged tables carry them under "paint"."""

    def __init__(self, dataset, batch_size, seed=2021, rank=0, world=1, drop_last=True, num_workers=8, ordered=False,
                 plan_safety=False, cameras=False, seg_model=None, driving_score=False):
        self.ds, self.B, self.seed, self.rank, self.world, self.drop_last = dataset, batch_size, seed, rank, world, drop_last
        self.num_workers = max(1, int(num_workers))
        self.ordered = ordered
        self.plan_safety = plan_safety
        self.driving_score = driving_score
        self.cameras = cameras
        self.seg_model = seg_model
        if plan_safety and not ordered:
            raise LavbError("plan_safety tables need the ordered, unaugmented loader")
        if driving_score and not ordered:
            raise LavbError("driving_score tables need the ordered, unaugmented loader")
        self.epoch = 0

    def _prepare(self, pool, idxs, draws):
        kw = dict(plan_safety=True) if self.plan_safety else {}
        if self.driving_score:
            kw["driving_score"] = True
        if self.cameras:
            kw["cameras"] = True
        if self.seg_model is not None:
            kw["paint"] = True
        return list(pool.map(lambda a: self.ds.prepare(int(a[0]), *a[1], **kw), zip(idxs, draws)))

    def shard(self, epoch):
        """this rank's sample indices of ``epoch``: training takes every world-th entry of the epoch's shuffle (the remainder
        dropped, so every rank runs as many steps); ordered mode takes the contiguous range [rank * n // world,
        (rank + 1) * n // world), so the ranks together score every sample once, in index order."""
        n = len(self.ds)
        if self.ordered:
            return np.arange(self.rank * n // self.world, (self.rank + 1) * n // self.world)
        return np.random.RandomState([self.seed, epoch]).permutation(n)[self.rank::self.world][:n // self.world]

    def __len__(self):
        n = len(self.shard(0)) if self.ordered else len(self.ds) // self.world
        return n // self.B if self.drop_last else -(-n // self.B)

    def generators(self, epoch):
        """(RandomState of the angle and jitter draws, torch CPU generator of the LiDAR shuffles) of ``epoch`` on this rank."""
        return (np.random.RandomState([self.seed, epoch, self.rank]),
                torch.Generator(device="cpu").manual_seed(self.seed * 1000003 + epoch * 1009 + self.rank))

    def _host(self, idxs, draws, gen, pool):
        hs = self._prepare(pool, idxs, draws)
        st = self.ds.stage_batch(hs, gen, **(dict(pool=pool) if self.seg_model is not None else {}))
        st["decoded"] = self.ds.decode_maps(st["maps"])
        return st

    def __iter__(self):
        for batch, _ in self.staged_batches():
            yield batch

    def staged_batches(self):
        """the batches of the next epoch as (14-tuple, the host tables stage_batch made for it): the evaluator reads the actor
        table ("actors", "offsets") that the tuple does not carry."""
        epoch, self.epoch = self.epoch, self.epoch + 1
        order = self.shard(epoch)
        batches = [order[k * self.B:(k + 1) * self.B] for k in range(len(self))]
        rng, gen = self.generators(epoch)
        if not batches:
            return
        draw = self.ds.no_draw if self.ordered else lambda: self.ds.draw(rng)
        draws = lambda idxs: [draw() for _ in idxs]                             # on this thread, in sample order
        launch = self.ds.launch_batch if self.seg_model is None else lambda st: self.ds.launch_batch(st, self.seg_model)
        with ThreadPoolExecutor(1) as ahead, ThreadPoolExecutor(self.num_workers) as pool:
            nxt = ahead.submit(self._host, batches[0], draws(batches[0]), gen, pool)
            for k in range(len(batches)):
                staged = nxt.result()
                if k + 1 < len(batches):
                    nxt = ahead.submit(self._host, batches[k + 1], draws(batches[k + 1]), gen, pool)
                yield launch(staged), staged


class TemporalBEVDataset:
    """TemporalBEVDataset (lav/utils/datasets/temporal_bev_dataset.py), the data of the privileged planner, over a recording.

    Same constructor, YAML keys, ``len`` and index mapping as the reference (BasicDataset, trajectories in sorted order).
    ``ds[i]`` returns its 9-tuple: bev (3+2*(num_frame_stack+1), 320, 320) uint8 on ``device`` (one bev_targets launch),
    -ego_locs (T+1,2) f64, cmd, -nxp (2,) f64, bra, -locs (max_objs,T+1,2) f32, oris (max_objs,) f32, typs (max_objs,) int32,
    num_objs.  ``sample(idx, offset, angle)`` takes the draws explicitly: the column shift ``offset`` in pixels and the rotation
    ``angle`` in degrees.  ``ds[i]`` draws them from ``self.gen``, a torch CPU generator seeded with ``seed``, exactly as the
    reference draws them from torch's global generator (temporal_bev_dataset.py:28-30), so a seeded stream replays.  ``overrides``
    replaces keys of the YAML (the evaluator's --data-dir)."""

    def __init__(self, config_path, seed=2021, device=torch.device("cuda"), overrides=None):
        with open(config_path) as f:
            cfg = yaml.safe_load(f)
        cfg.update(overrides or {})
        self.cfg = cfg
        for k, v in cfg.items():
            setattr(self, k, v)
        self.device = torch.device(device)
        self.margin = ops.BEV_MARGIN
        self.paths, self.index = index_trajectories(self.data_dir, self.percentage_data, self.all_towns, self.num_plan, seed)
        self._envs, self._env_lock = {}, threading.Lock()
        self._decode_stream = None
        self.gen = torch.Generator(device="cpu").manual_seed(seed)

    __len__ = TemporalLiDARPaintedDataset.__len__
    bev_batch = TemporalLiDARPaintedDataset.bev_batch
    map_png = TemporalLiDARPaintedDataset.map_png
    decode_maps = TemporalLiDARPaintedDataset.decode_maps
    planes_on_stream = TemporalLiDARPaintedDataset.planes_on_stream
    env = TemporalLiDARPaintedDataset.env

    def draw(self, gen):
        """(offset in pixels, angle in degrees): int of the fp32 draw clipped to the margin, then the angle — the reference's
        expressions and order (temporal_bev_dataset.py:28-30)."""
        offset = int((torch.rand(1, generator=gen) * 2 - 1) * self.x_jitter)
        offset = int(np.clip(offset, -self.margin, self.margin))
        angle = float(torch.rand(1, generator=gen) * 2 - 1) * self.angle_jitter
        return offset, angle

    def no_draw(self):
        """the draws of an unaugmented sample: no shift, no rotation."""
        return 0, 0.0

    # ---- host part: record reads, PNG chunk walks, labels, BEV job rows
    def prepare(self, idx, offset, angle, plan_safety=False, driving_score=False):
        """the host record of sample ``idx``; with ``plan_safety`` (unaugmented samples only) it also holds the sample's
        plan_safety_table, from the same record reads, and with ``driving_score`` its driving_score_table."""
        traj, index = self.index[idx]
        env = self.env(traj)
        T = self.num_plan
        tracks = _read_tracks(env, index, T)
        table = _plan_safety_of(tracks, plan_safety, offset != 0 or angle != 0)
        driving = _driving_score_of(tracks, driving_score, offset != 0 or angle != 0)
        ego_locs, locs, oris, _, typs = _label_tracks(tracks, self.max_pedestrian_radius, self.max_vehicle_radius)
        frames = [i for i in range(index, index - self.num_frame_stack - 1, -1) if i >= 0]
        poses = {i: ego_pose(env, i) for i in frames}
        loc0, ori0 = poses[index]
        pngs = [self.map_png(traj, env, c, index) for c in (0, 9, 10)]
        rows = [(c, c, 0.0, angle, 0, offset) for c in range(3)]                          # load_bev_channels(y_offset=offset)
        ppm = self.pixels_per_meter
        for t, i in enumerate(frames):
            loc, ori = poses[i]
            dl = (loc - loc0) @ [[np.cos(ori0), -np.sin(ori0)], [np.sin(ori0), np.cos(ori0)]] * ppm
            dx, dy = map(int, dl)
            if abs(dx) > self.margin or abs(dy + offset) > self.margin:
                raise LavbError(f"frame {i} of {self.paths[traj]}: BEV shift ({dx}, {dy + offset}) px exceeds the "
                                f"{self.margin}-pixel margin")
            for c in (1, 2):
                rows.append((len(pngs), 3 + 2 * t + c - 1, -(ori - ori0) * 180 / math.pi, angle, dx, dy + offset))
                pngs.append(self.map_png(traj, env, c, i))
        rows += [(-1, 3 + 2 * t + c, 0.0, 0.0, 0, 0) for t in range(len(frames), self.num_frame_stack + 1) for c in (0, 1)]

        shift = [offset / ppm, 0]
        locs = rotate_points(locs, -angle, ego_locs[0]) + shift                           # about the unshifted ego origin
        oris[1:] = oris[1:] - np.deg2rad(angle)
        ego = rotate_points(ego_locs, -angle, ego_locs[0]) + shift
        nxp = rotate_points(_frame(env, "nxp", index).reshape(2), -angle, ego[0]) + shift  # about the SHIFTED ego origin
        n_obj = min(len(locs), self.max_objs)
        p_locs = np.zeros((self.max_objs, T + 1, 2), np.float32)
        p_oris = np.zeros((self.max_objs,), np.float32)
        p_typs = np.zeros((self.max_objs,), np.int32)
        p_locs[:n_obj], p_oris[:n_obj], p_typs[:n_obj] = locs[:n_obj], oris[:n_obj, 0], typs[:n_obj, 0]
        h = dict(pngs=pngs, rows=rows, ego_locs=-ego, nxp=-nxp, cmd=int(_frame(env, "cmd", index, np.uint8)[0]),
                 bra=int(_frame(env, "bra", index, np.uint8)[0]), locs=-p_locs, oris=p_oris, typs=p_typs, num_objs=n_obj)
        if table is not None:
            h["plan_safety"] = table
        if driving is not None:
            h["driving_score"] = driving
        return h

    def sample(self, idx, offset, angle):
        """the 9-tuple of sample ``idx`` for the given draws (offset in pixels, angle in degrees)."""
        h = self.prepare(idx, offset, angle)
        dev = self.device
        return (self.bev_batch([h])[0], torch.as_tensor(h["ego_locs"], device=dev), h["cmd"], torch.as_tensor(h["nxp"], device=dev),
                h["bra"], torch.as_tensor(h["locs"], device=dev), torch.as_tensor(h["oris"], device=dev),
                torch.as_tensor(h["typs"], device=dev), h["num_objs"])

    def __getitem__(self, idx):
        return self.sample(idx, *self.draw(self.gen))


class TemporalBEVBatchLoader(TemporalBatchLoader):
    """Batches of a TemporalBEVDataset for BEVTrainer.train_bev, one rank of ``world``: the shuffle and sharding of
    TemporalBatchLoader.  The draws of a batch come from one torch CPU generator seeded by (seed, epoch, rank), in sample
    order; record reads and PNG chunk walks run on ``num_workers`` threads and the batch's maps (about 2,300 planes at 256) are
    decoded in one launch on a side stream, one batch ahead of the GPU.  A batch is the 9-tuple bev (B,9,320,320) uint8, ego_locs (B,T+1,2) f32, cmds (B,) int64, nxps (B,2) f32,
    bras (B,) int64, locs (B,max_objs,T+1,2) f32, oris (B,max_objs) f32, typs (B,max_objs) int32, num_objs (B,) int64 (host),
    with one bev_targets launch per batch.  With ``ordered`` (evaluation) the samples come in index order and every draw is
    dataset.no_draw(); with ``plan_safety`` as well, every host record holds its plan_safety_table under "plan_safety", and with
    ``driving_score`` its driving_score_table under "driving_score"."""

    def _host_bev(self, idxs, draws, pool):
        hs = self._prepare(pool, idxs, draws)
        return hs, self.ds.decode_maps(stage_maps(hs, self.ds.device.type == "cuda"))

    def staged_batches(self):
        """the batches of the next epoch as (9-tuple, the host records dataset.prepare made for it): the evaluator reads the
        recorded commands there without a copy back from the device."""
        epoch, self.epoch = self.epoch, self.epoch + 1
        order = self.shard(epoch)
        batches = [order[k * self.B:(k + 1) * self.B] for k in range(len(self))]
        gen = torch.Generator(device="cpu").manual_seed(self.seed * 1000003 + epoch * 1009 + self.rank)
        if not batches:
            return
        draw = self.ds.no_draw if self.ordered else lambda: self.ds.draw(gen)
        draws = lambda idxs: [draw() for _ in idxs]                             # on this thread, in sample order
        with ThreadPoolExecutor(1) as ahead, ThreadPoolExecutor(self.num_workers) as pool:
            nxt = ahead.submit(self._host_bev, batches[0], draws(batches[0]), pool)
            for k in range(len(batches)):
                hs, decoded = nxt.result()
                if k + 1 < len(batches):
                    nxt = ahead.submit(self._host_bev, batches[k + 1], draws(batches[k + 1]), pool)
                yield self._device_bev(hs, decoded), hs

    def _device_bev(self, hs, decoded):
        ds, dev = self.ds, self.ds.device
        bev = ds.bev_batch(hs, decoded)
        f32 = lambda key: torch.as_tensor(np.stack([h[key] for h in hs]), dtype=torch.float32).to(dev)
        ints = lambda key: torch.tensor([h[key] for h in hs], dtype=torch.int64)
        return (bev, f32("ego_locs"), ints("cmd").to(dev), f32("nxp"), ints("bra").to(dev), f32("locs"), f32("oris"),
                torch.as_tensor(np.stack([h["typs"] for h in hs])).to(dev), ints("num_objs"))


def load_img(env, tag, i):
    """BasicDataset.load_img (basic_dataset.py:86-94) with the BGR -> RGB flip of the image datasets: key ``tag_%05d`` decoded by
    cv2.imdecode, IMREAD_COLOR for an rgb tag (-> (h, w, 3) RGB), IMREAD_GRAYSCALE for a sem tag (-> (h, w))."""
    import cv2
    key = f"{tag}_{i:05d}"
    data = env.get(key)
    if data is None:
        raise LavbError(f"record key {key} is missing")
    img = cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR if "rgb" in tag else cv2.IMREAD_GRAYSCALE)
    if img is None:
        raise LavbError(f"record key {key} is not a decodable image")
    return img[..., ::-1] if img.ndim == 3 else img


def brake_cameras(ncam, what):
    """the three middle cameras ncam//2 - 1 .. ncam//2 + 1 of ``ncam`` (BrakePredictionDataset's, bra_dataset.py:17-31), the
    ones the brake model sees side by side; fewer than three cameras is a LavbError of ``what``."""
    mid = [ncam // 2 - 1, ncam // 2, ncam // 2 + 1]
    if mid[0] < 0 or mid[2] >= ncam:
        raise LavbError(f"{what}: the brake model needs three middle cameras, the config has {ncam}")
    return mid


def read_cameras(env, i, cams, crop_tel_bottom=None):
    """the colour images of frame ``i``, decoded by load_img: rgbs (len(cams), h, w, 3) of the cameras ``cams``, and with
    ``crop_tel_bottom`` tel = tel_rgb[:-crop_tel_bottom] (h_tel - crop_tel_bottom, w_tel, 3); uint8 numpy."""
    h = dict(rgbs=np.stack([load_img(env, f"rgb_{c}", i) for c in cams]))
    if crop_tel_bottom is not None:
        h["tel"] = load_img(env, "tel_rgb", i)[:-crop_tel_bottom]
    return h


def stage_images(hs, keys, pin, what):
    """the images under ``keys`` of the prepared records ``hs`` stacked into one uint8 host buffer per key (pinned on ``pin``),
    record b at index b; a key missing from the first record is skipped, images of different sizes are a LavbError of ``what``."""
    st = {}
    for key in keys:
        if key in hs[0]:
            shapes = {h[key].shape for h in hs}
            if len(shapes) != 1:
                raise LavbError(f"{what}: the {key} images of a batch differ in size: {sorted(shapes)}")
            buf = torch.empty((len(hs),) + hs[0][key].shape, dtype=torch.uint8, pin_memory=pin)
            dst = buf.numpy()
            for b, h in enumerate(hs):
                dst[b] = h[key]
            st[key] = buf
    return st


class CameraDataset:
    """The camera samples of a recording, for scoring the segmentation and brake models (lav_b200.evaluate_rgb): the frames of
    BasicDataset (index_trajectories, the same YAML keys and ``overrides``), unaugmented.

    Frame k holds, with ``seg``, every camera 0 .. len(camera_yaws) - 1 and its labels, SegmentationDataset's samples k * ncam + c
    (seg_dataset.py:16-25); with ``brake``, the three middle cameras ncam//2 - 1 .. ncam//2 + 1, the telephoto view cut by
    [:-crop_tel_bottom] and the brake label, BrakePredictionDataset's sample k (bra_dataset.py:17-31).  ``cams`` are the cameras
    read (all with ``seg``, else the middle three) and ``brake_cams`` the positions of the middle three among them.  Images are
    decoded on the host as BasicDataset.load_img decodes them, colour images flipped BGR -> RGB; no key a run does not need is
    read.  The reference's augment(0.5) is training-only and not applied."""

    def __init__(self, config_path, seg=True, brake=True, seed=2021, device=torch.device("cuda"), overrides=None):
        if not (seg or brake):
            raise LavbError("CameraDataset: nothing to load (neither seg nor brake)")
        with open(config_path) as f:
            cfg = yaml.safe_load(f)
        cfg.update(overrides or {})
        self.cfg = cfg
        for k, v in cfg.items():
            setattr(self, k, v)
        self.device = torch.device(device)
        self.seg, self.brake = seg, brake
        ncam = len(self.camera_yaws)
        mid = brake_cameras(ncam, "CameraDataset") if brake else [ncam // 2 - 1, ncam // 2, ncam // 2 + 1]
        self.cams = list(range(ncam)) if seg else mid
        self.brake_cams = [self.cams.index(c) for c in mid] if brake else []
        self.paths, self.index = index_trajectories(self.data_dir, self.percentage_data, self.all_towns, self.num_plan, seed)
        self._envs, self._env_lock = {}, threading.Lock()

    __len__ = TemporalLiDARPaintedDataset.__len__
    env = TemporalLiDARPaintedDataset.env

    def no_draw(self):
        """no augmentation: nothing to draw."""
        return ()

    def prepare(self, idx):
        """the decoded host images of frame ``idx``: rgbs (len(cams), h, w, 3), with seg labels (len(cams), h, w), with brake tel
        (h_tel - crop_tel_bottom, w_tel, 3) and bra; uint8 numpy."""
        traj, i = self.index[idx]
        env = self.env(traj)
        h = read_cameras(env, i, self.cams, self.crop_tel_bottom if self.brake else None)
        if self.seg:
            h["labels"] = np.stack([load_img(env, f"sem_{c}", i) for c in self.cams])
        if self.brake:
            h["bra"] = int(_frame(env, "bra", i, np.uint8)[0])
        return h

    def stage_batch(self, hs):
        """the prepared frames ``hs`` stacked into one host buffer per key (pinned on a CUDA dataset): rgbs (B, ncam, h, w, 3),
        labels (B, ncam, h, w), tel (B, h_tel, w_tel, 3) uint8, bra (B,) int64."""
        pin = self.device.type == "cuda"
        st = stage_images(hs, ("rgbs", "labels", "tel"), pin, "CameraDataset")
        if self.brake:
            bra = torch.tensor([h["bra"] for h in hs], dtype=torch.int64)
            st["bra"] = bra.pin_memory() if pin else bra
        return st

    def launch_batch(self, st):
        """the staged host buffers copied to the device, one copy each."""
        return {k: v.to(self.device, non_blocking=True) for k, v in st.items()}


class PaintDataset:
    """The painted LiDAR samples of a recording, for scoring the point painting (lav_b200.evaluate_paint): the frames of
    BasicDataset (index_trajectories, the same YAML keys and ``overrides``), unaugmented.

    Frame k holds the recorded sweep lidar_%05d and the recorded tags sem_{c} of the painting cameras c = 0 .. 2
    (point_painting.CAMERA_YAWS, the three cameras data_paint reads; not the config's camera_yaws, which lists five); with
    ``online`` their colour images rgb_{c}, with ``stored`` the painted rows lidar_sem_%05d.  Images are decoded on the host as
    BasicDataset.load_img decodes them; an image of another size than the painting geometry (288 x 256) is a LavbError.  A
    lidar_sem key that is missing or whose size is not the sweep's rows x (len(seg_channels)) floats marks the frame
    mismatched: its stored rows are not scored, and nothing is raised."""

    def __init__(self, config_path, online=True, stored=False, seed=2021, device=torch.device("cuda"), overrides=None):
        from . import point_painting
        if not (online or stored):
            raise LavbError("PaintDataset: nothing to score (neither online nor stored)")
        with open(config_path) as f:
            cfg = yaml.safe_load(f)
        cfg.update(overrides or {})
        self.cfg = cfg
        for k, v in cfg.items():
            setattr(self, k, v)
        self.device = torch.device(device)
        self.online, self.stored = online, stored
        self.converters = point_painting.make_converters(self.camera_x, self.camera_z)
        self.cams = list(range(len(self.converters)))
        self.image_hw = (self.converters[0].rgb_h, self.converters[0].rgb_w)
        self.window = (self.min_x, self.max_x, self.min_y, self.max_y)
        self.n_classes = len(self.seg_channels) + 1
        self.paths, self.index = index_trajectories(self.data_dir, self.percentage_data, self.all_towns, self.num_plan, seed)
        self._envs, self._env_lock = {}, threading.Lock()

    __len__ = TemporalLiDARPaintedDataset.__len__
    env = TemporalLiDARPaintedDataset.env

    def no_draw(self):
        """no augmentation: nothing to draw."""
        return ()

    def _image(self, env, tag, i):
        img = load_img(env, tag, i)
        if img.shape[:2] != self.image_hw:
            raise LavbError(f"record key {tag}_{i:05d} is {img.shape[1]} x {img.shape[0]}, the painting cameras' images are "
                            f"{self.image_hw[1]} x {self.image_hw[0]}")
        return img

    def prepare(self, idx):
        """the host record of frame ``idx``: lidar (n, 4) f32, labels (ncam, h, w) uint8, with online rgbs (ncam, h, w, 3) uint8,
        with stored the lidar_sem rows (n, C - 1) f32 or None when the frame is mismatched."""
        traj, i = self.index[idx]
        env = self.env(traj)
        key = f"lidar_{i:05d}"
        raw = env.get(key)
        if raw is None:
            raise LavbError(f"record key {key} is missing")
        h = dict(lidar=np.frombuffer(raw, np.float32).reshape(-1, 4))
        h["labels"] = np.stack([self._image(env, f"sem_{c}", i) for c in self.cams])
        if self.online:
            h["rgbs"] = np.stack([self._image(env, f"rgb_{c}", i) for c in self.cams])
        if self.stored:
            sem = env.get(f"lidar_sem_{i:05d}")
            w = self.n_classes - 1
            ok = sem is not None and len(sem) == len(h["lidar"]) * w * 4
            h["stored"] = np.frombuffer(sem, np.float32).reshape(-1, w) if ok else None
        return h

    def stage_batch(self, hs):
        """the prepared frames ``hs`` in host buffers (pinned on a CUDA dataset): points (B, Nmax, 4) f32 NaN-padded (Nmax >= 1),
        meta (B, 2) int32 = (rows, stored scored), labels (B, ncam, h, w) and rgbs (B, ncam, h, w, 3) uint8, stored (B, Nmax,
        C - 1) f32 (zero where not scored)."""
        pin = self.device.type == "cuda"
        B, n_max = len(hs), max(1, max(len(h["lidar"]) for h in hs))
        empty = lambda shape, dtype: torch.empty(shape, dtype=dtype, pin_memory=pin)
        st = dict(points=empty((B, n_max, 4), torch.float32), meta=empty((B, 2), torch.int32))
        pts, meta = st["points"].numpy(), st["meta"].numpy()
        pts[:] = np.nan
        for b, h in enumerate(hs):
            pts[b, :len(h["lidar"])] = h["lidar"]
            meta[b] = (len(h["lidar"]), int(h.get("stored") is not None))
        for key in ("labels", "rgbs"):
            if key in hs[0]:
                st[key] = empty((B,) + hs[0][key].shape, torch.uint8)
                dst = st[key].numpy()
                for b, h in enumerate(hs):
                    dst[b] = h[key]
        if self.stored:
            st["stored"] = empty((B, n_max, self.n_classes - 1), torch.float32)
            dst = st["stored"].numpy()
            dst[:] = 0
            for b, h in enumerate(hs):
                if h["stored"] is not None:
                    dst[b, :len(h["stored"])] = h["stored"]
        return st

    def launch_batch(self, st):
        """the staged host buffers copied to the device, one copy each."""
        return {k: v.to(self.device, non_blocking=True) for k, v in st.items()}


class CameraBatchLoader(TemporalBatchLoader):
    """Batches of a CameraDataset in frame order, unaugmented, the last batch possibly short: TemporalBatchLoader's ordered mode,
    with the record reads and image decodes of a batch on ``num_workers`` threads one batch ahead of the GPU.  A batch is the
    dict of CameraDataset.launch_batch; staged_batches also yields the host buffers."""

    def __init__(self, dataset, batch_size, num_workers=8):
        super().__init__(dataset, batch_size, drop_last=False, num_workers=num_workers, ordered=True)

    def _host(self, idxs, draws, gen, pool):
        return self.ds.stage_batch(self._prepare(pool, idxs, draws))


def get_data_loader(data_type, args):
    """lav.utils.datasets.get_data_loader for 'temporal_lidar_painted' and 'temporal_bev' (args: config_path, seed, batch_size;
    optional rank, world_size, device, num_workers).  The other dataset types are not provided."""
    if data_type not in ("temporal_lidar_painted", "temporal_bev"):
        raise NotImplementedError(f"data type {data_type!r}: only 'temporal_lidar_painted' and 'temporal_bev' are provided")
    dev = getattr(args, "device", None) or torch.device("cuda", torch.cuda.current_device())
    rank, world = getattr(args, "rank", 0), getattr(args, "world_size", 1)
    if data_type == "temporal_bev":
        ds = TemporalBEVDataset(args.config_path, seed=args.seed, device=dev)
        return TemporalBEVBatchLoader(ds, args.batch_size, args.seed, rank, world, num_workers=getattr(args, "num_workers", 8))
    ds = TemporalLiDARPaintedDataset(args.config_path, seed=args.seed, device=dev)
    return TemporalBatchLoader(ds, args.batch_size, args.seed, rank, world, num_workers=getattr(args, "num_workers", 8))
