"""numpy restatement (no cv2) of the reference's TemporalBEVDataset.__getitem__ (lav/utils/datasets/temporal_bev_dataset.py:12-97),
built on the pieces of oracle/dataset_ref.py.  Pinned against the reference by oracle/pin_bev.py."""
import numpy as np

from oracle.dataset_ref import access, filter_actors, load_bev_channels, load_planes, rotate_points, transform_ego


def get_bev_item(get, index, cfg, offset, angle):
    """TemporalBEVDataset.__getitem__ for frame ``index`` of one recording (``get(key) -> bytes``) with the draws given: the column
    shift ``offset`` (pixels, already clipped to the margin) and the rotation ``angle`` (degrees).  Returns the reference's 9-tuple
    (bev, -ego_locs, cmd, -nxp, bra, -locs, oris, typs, num_objs)."""
    T, ppm = cfg["num_plan"], cfg["pixels_per_meter"]
    radii = dict(max_pedestrian_radius=cfg["max_pedestrian_radius"], max_vehicle_radius=cfg["max_vehicle_radius"], T=T)
    _, e_locs, e_oris, locs, oris, bbox, typs = filter_actors(get, index, **radii)
    ego_locs, locs, oris, bbox, typs = transform_ego(e_locs, locs, oris, bbox, typs, e_oris[0], T + 1)

    bev = np.zeros((3 + 2 * (cfg["num_frame_stack"] + 1), 320, 320), np.uint8)
    bev[:3] = load_bev_channels(load_planes(get, index, (0, 9, 10)), angle_offset=angle, loc=(0, offset))
    frames = [i for i in range(index, index - cfg["num_frame_stack"] - 1, -1) if i >= 0]
    poses = {i: filter_actors(get, i, **radii)[1:3] for i in frames}
    loc0, ori0 = poses[index][0][0], poses[index][1][0]
    for t, i in enumerate(frames):
        loc, ori = poses[i][0][0], poses[i][1][0]
        dl = (loc - loc0) @ [[np.cos(ori0), -np.sin(ori0)], [np.sin(ori0), np.cos(ori0)]] * ppm
        dx, dy = (int(v) for v in dl)
        bev[3 + 2 * t:5 + 2 * t] = load_bev_channels(load_planes(get, i, (1, 2)), angle=ori - ori0, angle_offset=angle,
                                                     loc=(dx, dy + offset))

    shift = [offset / ppm, 0]
    locs = rotate_points(locs, -angle, ego_locs[0]) + shift
    oris[1:] = oris[1:] - np.deg2rad(angle)
    nxp = access(get, "nxp", index).reshape(2)
    ego_locs = rotate_points(ego_locs, -angle, ego_locs[0]) + shift
    nxp = rotate_points(nxp, -angle, ego_locs[0]) + shift
    cmd = int(access(get, "cmd", index, np.uint8)[0, 0])
    bra = int(access(get, "bra", index, np.uint8)[0, 0])
    n_obj = min(len(locs), cfg["max_objs"])
    p_locs = np.zeros((cfg["max_objs"], T + 1, 2), np.float32)
    p_oris = np.zeros((cfg["max_objs"],), np.float32)
    p_typs = np.zeros((cfg["max_objs"],), np.int32)
    p_locs[:n_obj], p_oris[:n_obj], p_typs[:n_obj] = locs[:n_obj], oris[:n_obj, 0], typs[:n_obj, 0]
    return bev, -ego_locs, cmd, -nxp, bra, -p_locs, p_oris, p_typs, n_obj
