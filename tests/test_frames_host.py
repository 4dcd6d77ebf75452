"""CPU checks of the add_frame restatement (frames_oracle.py): the odometry rotation, the point depths, the keyframe
selection and the 8-bit decode, against independent float64 computations, known answers and OpenCV when it imports."""
import numpy as np
import pytest

import frames_oracle as fo


def _independent_R(q):
    """R = I + 2 w [v]x + 2 [v]x^2 with v = (x, y, z): the same map as Eigen's toRotationMatrix, without normalisation."""
    x, y, z, w = q
    K = np.array([[0.0, -z, y], [z, 0.0, -x], [-y, x, 0.0]])
    return np.eye(3) + 2.0 * w * K + 2.0 * K @ K


def _quats(n, seed):
    rng = np.random.default_rng(seed)
    q = rng.normal(size=(n, 4))
    return q / np.linalg.norm(q, axis=1, keepdims=True)


def test_rotation_matches_independent_float64():
    for q in _quats(200, 1):
        R = fo.quat_rotation(q)
        assert np.abs(R - _independent_R(q)).max() <= 1e-12
        assert np.abs(R.T @ R - np.eye(3)).max() <= 1e-12 and abs(np.linalg.det(R) - 1.0) <= 1e-12
    scipy_rot = pytest.importorskip("scipy.spatial.transform").Rotation
    for q in _quats(50, 2):                                             # scipy takes (x, y, z, w) too
        assert np.abs(fo.quat_rotation(q) - scipy_rot.from_quat(q).as_matrix()).max() <= 1e-12


def test_rotation_known_answers():
    assert np.array_equal(fo.quat_rotation([0.0, 0.0, 0.0, 1.0]), np.eye(3))
    s = np.sqrt(0.5)
    want = {0: [[1, 0, 0], [0, 0, -1], [0, 1, 0]],                      # 90 degrees about x, y, z
            1: [[0, 0, 1], [0, 1, 0], [-1, 0, 0]],
            2: [[0, -1, 0], [1, 0, 0], [0, 0, 1]]}
    for axis, R in want.items():
        q = [0.0, 0.0, 0.0, s]
        q[axis] = s
        assert np.abs(fo.quat_rotation(q) - np.array(R, np.float64)).max() <= 1e-15, axis
    # Eigen does not normalise: q = 2 * (90 degrees about x) gives the unit formula's answer for the longer quaternion
    r2 = np.sqrt(2.0)
    R = fo.quat_rotation([r2, 0.0, 0.0, r2])
    assert np.abs(R - np.array([[1, 0, 0], [0, -3, -4], [0, 4, -3]], np.float64)).max() <= 1e-14
    assert np.abs(R - _independent_R([r2, 0.0, 0.0, r2])).max() <= 1e-14


def test_depth_matches_independent_float64():
    rng = np.random.default_rng(3)
    for q in _quats(20, 4):
        t = rng.uniform(-50, 50, 3)
        xyz = (rng.uniform(-100, 100, (1000, 3))).astype(np.float32)
        R = _independent_R(q)
        want = (xyz.astype(np.float64) - t) @ R[:, 2]                    # z of R_cw (p - t_wc)
        got = fo.depth_rsp64(q, t, xyz)
        assert np.abs(got - want).max() <= 1e-12 * max(1.0, np.abs(want).max())
        assert np.array_equal(fo.depth_rsp(q, t, xyz), got.astype(np.float32))
    # identity pose: the depth is the point's z
    xyz = rng.uniform(-5, 5, (100, 3)).astype(np.float32)
    assert np.array_equal(fo.depth_rsp([0, 0, 0, 1], [0, 0, 0], xyz), xyz[:, 2])


@pytest.mark.parametrize("k,train", [(1, list(range(12))), (2, [1, 3, 5, 7, 9, 11]), (5, [4, 9])])
def test_keyframe_selection(k, train):
    """(all_frame_num_ + 1) % select_every_k_frame == 0 over the first 12 frames"""
    assert [i for i in range(12) if fo.is_train(i, k)] == train


def test_decode_table():
    x = np.arange(256)
    tab = np.float32(x) * np.float32(1 / 255)
    assert np.array_equal(fo.DECODE.view(np.uint32), tab.astype(np.float32).view(np.uint32))
    naive = (x / 255.0).astype(np.float32)
    assert int(np.sum(fo.DECODE != naive)) == 126                      # the "obvious" formula differs in 126 byte values
    assert fo.DECODE[0] == 0.0 and fo.DECODE[255] == 1.0
    rng = np.random.default_rng(5)
    bgr = rng.integers(0, 256, (7, 9, 3), dtype=np.uint8)
    img = fo.decode(bgr)
    assert img.shape == (3, 7, 9) and img.dtype == np.float32
    for c in range(3):
        assert np.array_equal(img[c], tab[bgr[..., 2 - c]])


def test_decode_matches_opencv():
    """cvtColor(BGR2RGB) gives the channel order; cv::normalize(NORM_MINMAX, CV_32F) of an image spanning 0..255 calls
    Mat::convertTo(CV_32F, 1/255, 0), the 8U -> 32F conversion Dataset::addFrame uses, so it pins the scale's rounding."""
    cv2 = pytest.importorskip("cv2")
    x = np.arange(256, dtype=np.uint8)
    bgr = np.stack([x, x[::-1], np.roll(x, 77)], 1).reshape(16, 16, 3).copy()
    rgb = cv2.cvtColor(bgr, cv2.COLOR_BGR2RGB)
    assert np.array_equal(rgb, bgr[..., ::-1])
    conv = cv2.normalize(rgb, None, 0.0, 1.0, cv2.NORM_MINMAX, cv2.CV_32F)
    assert np.array_equal(conv.transpose(2, 0, 1).view(np.uint32), fo.decode(bgr).view(np.uint32))


def test_colours():
    c = np.arange(256, dtype=np.uint8).reshape(-1, 1).repeat(3, 1)
    assert np.array_equal(fo.colours_init(c), np.arange(256)[:, None].repeat(3, 1) / 255.0)
    assert fo.colours_extend(c).dtype == np.float32
