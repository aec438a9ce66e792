"""CPU: the host half of the batched LiDAR path (GpuLidarStacker.batch_tables) against a numpy restatement of the stacker's row
order — roof filter, then the permutation, then truncation and zero padding — and the loader's new argument."""
import math

import numpy as np
import torch

from lav_b200 import ops
from lav_b200.data_pipeline import GpuLidarStacker


def make_sweep(rs, n, c=4, roof_frac=0.1):
    xyz = rs.uniform(-40, 40, (n, 3)).astype(np.float32)
    xyz[:, 2] = rs.uniform(-3, 2, n)
    roof = rs.rand(n) < roof_frac                                     # inside the ego-roof box: dropped
    xyz[roof] = np.stack([rs.uniform(-2.3, -0.1, roof.sum()), rs.uniform(-0.7, 0.7, roof.sum()), rs.uniform(-1.4, -1.1, roof.sum())], 1)
    xyzr = np.concatenate([xyz, rs.rand(n, 1).astype(np.float32)], 1)
    return xyzr, rs.rand(n, c).astype(np.float32)


def make_sample(rs, sizes, angle=None):
    sweeps = []
    for i, n in enumerate(sizes):
        xyzr, painted = make_sweep(rs, n)
        sweeps.append((xyzr, painted, rs.uniform(-5, 5, 2), float(rs.uniform(-math.pi, math.pi))))
    jit = [(np.zeros(2), 0.0)] + [(rs.uniform(-0.4, 0.4, 2), float(rs.uniform(-0.1, 0.1))) for _ in range(2)]
    return sweeps, float(rs.uniform(-20, 20)) if angle is None else angle, jit


def restated_rows(samples, P, seed):
    """output row -> raw row, as GpuLidarStacker orders them: each sweep's kept rows (np.delete of the roof box) newest first,
    shuffled by randperm(total) drawn per sample in order, truncated to P, padded with -1."""
    g = torch.Generator().manual_seed(seed)
    out, base, nums = np.full((len(samples), P), -1, np.int64), 0, []
    for b, (sweeps, _, _) in enumerate(samples):
        kept = []
        for xyzr, _, _, _ in sweeps:
            x, y, z = (xyzr[:, k].astype(np.float64) for k in range(3))
            on_roof = (x > np.float32(-2.4)) & (x < 0) & (y > np.float32(-0.8)) & (y < np.float32(0.8)) & (z > -1.5) & (z < -1)
            kept.append(base + np.delete(np.arange(len(xyzr)), np.nonzero(on_roof)[0]))
            base += len(xyzr)
        kept = np.concatenate(kept)
        perm = torch.randperm(len(kept), generator=g).numpy()
        num = min(P, len(kept))
        out[b, :num] = kept[perm][:num]
        nums.append(num)
    return out, nums


def test_batch_tables_follow_the_stacker_row_order():
    rs = np.random.RandomState(0)
    P = 5000
    samples = [make_sample(rs, s) for s in ([3000], [2000, 2500], [2500, 2500, 2500], [0, 100, 0], [1000, 0, 4000])]
    samples.append(make_sample(rs, [400]))
    samples[-1][0][0][0][:, :3] = [-1.0, 0.0, -1.2]                    # every point on the roof: nothing kept
    st = GpuLidarStacker(2, 4, P, device=torch.device("cpu"))
    t = st.batch_tables(samples, torch.Generator().manual_seed(7))
    want, nums = restated_rows(samples, P, 7)
    assert t["nums"] == nums and nums[2] == P and nums[0] < P and nums[-1] == 0
    assert t["rows"].dtype == torch.int32 and np.array_equal(t["rows"].numpy(), want)
    raw = np.concatenate([np.concatenate([x, p], 1) for sweeps, _, _ in samples for x, p, _, _ in sweeps])
    assert np.array_equal(t["raw"].numpy(), raw)
    sw = t["sweeps"]
    assert sw.dtype == ops.LIDAR_SWEEP_DTYPE and len(sw) == sum(len(s[0]) for s in samples)
    assert np.array_equal(sw["row0"], np.cumsum([0] + [len(x) for s in samples for x, _, _, _ in s[0]])[:-1])
    assert sw["time_idx"].tolist() == [i for s in samples for i in range(len(s[0]))]
    # the transforms are the stacker's: R_aug of the sample's angle, dloc rounded to fp32 as lavb_stack_sweep's float arguments
    sweeps, angle, jit = samples[2]
    rad = math.radians(-angle)
    k = 3                                                              # first sweep of sample 2
    assert np.array_equal(sw["R_aug"][k].reshape(3, 3), np.array([[math.cos(rad), math.sin(rad), 0], [-math.sin(rad), math.cos(rad), 0],
                                                                  [0, 0, 1]], np.float32))
    loc0, ori0 = sweeps[0][2], sweeps[0][3]
    dloc = (sweeps[1][2] - loc0 + jit[1][0]) @ np.array([[math.cos(ori0), -math.sin(ori0)], [math.sin(ori0), math.cos(ori0)]])
    assert (sw["dx"][k + 1], sw["dy"][k + 1]) == (np.float32(dloc[0]), np.float32(dloc[1]))
    assert sw["dx"][k] == 0 and sw["dy"][k] == 0


def test_det_grid_is_the_torch_scalars():
    h, w, (ppm, cx0, cy0, cy1, inv_r) = ops.det_grid()
    assert (h, w, ppm, cx0, cy0, cy1, inv_r) == (320, 320, 4, 160.0, 320, -40, 1.0)
    assert ops.det_grid(radius=3)[2][4] == float(np.float32(1) / np.float32(3))


def test_train_full_num_workers_argument():
    from lav_b200 import train_full
    assert train_full.parse_args([]).num_workers == 16
    assert train_full.parse_args(["--num-workers", "4"]).num_workers == 4
