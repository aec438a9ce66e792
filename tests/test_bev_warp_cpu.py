"""CPU: the fixed-point restatement of cv2.warpAffine (oracle/dataset_ref.py), the rotation matrix and its inverse (also the
host-side copy in lav_b200.ops that fills the bev_targets job table), and load_bev_channels, against OpenCV itself.
Skipped where cv2 does not import."""
import math

import numpy as np
import pytest

from lav_b200 import ops
from oracle import dataset_ref as D

cv2 = pytest.importorskip("cv2")


def _cv_rotate(img, angle):
    return cv2.warpAffine(img, cv2.getRotationMatrix2D((160, 280), angle, 1.0), img.shape[1::-1], flags=cv2.INTER_LINEAR)


def test_rotation_matrix_and_inverse_equal_opencv():
    rs = np.random.RandomState(0)
    for angle in np.concatenate([rs.uniform(-30, 30, 200), [0.0, -0.0, 20.0, -20.0, 90.0]]):
        angle = float(angle)
        M = cv2.getRotationMatrix2D((160, 280), angle, 1.0)
        assert np.array_equal(D.rotation_matrix_2d((160, 280), angle), M), angle
        inv = cv2.invertAffineTransform(M)
        assert np.array_equal(D.invert_affine(M), inv), angle
        assert np.array_equal(np.array(ops._inverse_rotation(angle, (160, 280))).reshape(2, 3), inv), angle


@pytest.mark.parametrize("channels", [1, 2, 3])
@pytest.mark.parametrize("kind", ["random", "binary"])
def test_fixed_point_warp_equals_opencv(channels, kind):
    rs = np.random.RandomState(channels * 7 + (kind == "binary"))
    for angle in rs.uniform(-30, 30, 200 // 4):
        shape = (320, 320) if channels == 1 else (320, 320, channels)
        img = rs.randint(0, 256, shape).astype(np.uint8) if kind == "random" else ((rs.rand(*shape) > 0.8) * 255).astype(np.uint8)
        M = cv2.getRotationMatrix2D((160, 280), float(angle), 1.0)
        want = cv2.warpAffine(img, M, (320, 320), flags=cv2.INTER_LINEAR)
        assert np.array_equal(D.warp_affine_u8(img, M), want), angle


def test_fixed_point_warp_other_sizes_equal_opencv():
    rs = np.random.RandomState(5)
    for h, w in ((40, 56), (97, 33)):
        img = rs.randint(0, 256, (h, w)).astype(np.uint8)
        for angle in rs.uniform(-30, 30, 10):
            M = cv2.getRotationMatrix2D((w / 2, h * 0.8), float(angle), 1.0)
            assert np.array_equal(D.warp_affine_u8(img, M), cv2.warpAffine(img, M, (w, h), flags=cv2.INTER_LINEAR))


def test_load_bev_channels_equals_cv2_chain():
    """load_bev_channels (temporal_lidar_painted_dataset.py:182-198) with cv2 vs the restatement, shifts across [-32, 32]."""
    rs = np.random.RandomState(11)
    shifts = [(-32, 32), (32, -32), (0, 0), (-32, -32), (32, 32)] + [tuple(rs.uniform(-32.99, 32.99, 2)) for _ in range(20)]
    for loc in shifts:
        planes = ((rs.rand(320, 320, 2) > 0.85) * 255).astype(np.uint8)
        yaw, jitter = float(rs.uniform(-0.3, 0.3)), float(rs.uniform(-20, 20))
        dx, dy = map(int, loc)
        a = _cv_rotate(planes, -yaw * 180 / math.pi)
        a = np.pad(a, [[32, 32], [32, 32], [0, 0]])[dx + 32:dx + 352, dy + 32:dy + 352, :]
        want = (_cv_rotate(a, jitter) > 0).astype(np.uint8).transpose(2, 0, 1)
        assert np.array_equal(D.load_bev_channels(planes, yaw, jitter, loc), want), loc
    with pytest.raises(ValueError):
        D.load_bev_channels(planes, 0.0, 0.0, (33, 0))
