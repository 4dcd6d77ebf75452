"""The vectorised restatement of extend()'s selection (tests/extend_oracle.py) checked on the host against the CPU oracle's
O(n^2) restatement (glic_oracle_extend_select, float32), on random scenes and on hand-made pixel borders, depth ties, negative
depths and filter thresholds -- before any GPU test relies on it."""
import numpy as np
import pytest

import extend_oracle as eo

F32 = np.float32


def _rot(rng):
    q = rng.normal(size=4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]], F32)


def _both(oracle32, pts, rsp, R, t, fx, fy, cx, cy, W, H, T):
    got = eo.select(pts, rsp, R, t, fx, fy, cx, cy, W, H, T)["keep"]
    want = oracle32.extend_select(pts, rsp, R, t, fx, fy, cx, cy, W, H, T)
    assert np.array_equal(got, want), (got[:20], want[:20])
    return got


@pytest.mark.parametrize("seed", range(4))
def test_random_scenes_match_the_c_oracle(oracle32, seed):
    rng = np.random.default_rng(seed)
    W, H = [(40, 30), (1, 17), (23, 1), (64, 48)][seed]
    n = 1500
    fx, fy = F32(0.6 * max(W, H)), F32(0.55 * max(W, H))
    cx, cy = F32(W * 0.43), F32(H * 0.57)
    pts = np.c_[rng.uniform(-6, 6, n), rng.uniform(-4, 4, n), rng.uniform(-3, 12, n)].astype(F32)
    pts[: n // 3] = np.round(pts[: n // 3] * 4) / 4                       # coarse grid: many shared pixels and equal depths
    rsp = rng.uniform(-0.5, 12, n).astype(F32)
    rsp[rng.uniform(size=n) < 0.05] = 0.0
    T = rng.uniform(0, 0.02, (H, W)).astype(F32)
    T[rng.uniform(size=(H, W)) < 0.6] = 1.0
    keep = _both(oracle32, pts, rsp, _rot(rng), rng.uniform(-1, 1, 3).astype(F32), fx, fy, cx, cy, W, H, T)
    assert keep.size > 0


def alpha_thresholds():
    """final_T values whose 1 - T is exactly one ulp below 0.99f, 0.99f, and one ulp above (all three exact)"""
    a = np.array([np.nextafter(F32(0.99), F32(0)), F32(0.99), np.nextafter(F32(0.99), F32(1))], F32)
    T = F32(1) - a
    assert np.array_equal(F32(1) - T, a)
    return T


def test_constructed_edges_match_the_c_oracle(oracle32):
    W, H, fx, fy, cx, cy = 8, 6, F32(4.0), F32(4.0), F32(0.0), F32(0.0)
    R, t = np.eye(3, dtype=F32), np.zeros(3, F32)
    tiny = np.nextafter(F32(0), F32(1))
    below_W = np.nextafter(F32(W), F32(0))
    pts = np.array([[1.0, 1.0, 2.0],                     # 0: pixel (2,2)
                    [1.0, 1.0, 2.0],                     # 1: same pixel, same depth, later index: loses to 0
                    [0.0, 1.0, 2.0],                     # 2: x exactly 0 -> column 0 (in)
                    [-tiny, 1.0, 4.0],                   # 3: x one ulp below 0 -> column -1 (out)
                    [below_W, 1.0, 4.0],                 # 4: x one ulp below W -> column 7 (in)
                    [W, 1.0, 4.0],                       # 5: x exactly W -> out
                    [-1.5, -1.0, -2.0],                  # 6: behind the camera, projects to (3,2): takes part
                    [1.5, 1.0, 2.0],                     # 7: pixel (3,2) at depth 2: loses to 6 (depth -2)
                    [2.0, 2.0, 2.0],                     # 8: pixel (4,4), depth_rsp 0 -> not inserted
                    [1.0, H, 4.0],                       # 9: y exactly H -> out
                    [-0.0, 3.0, 4.0]], F32)              # 10: x = -0.0 -> column 0 (in)
    rsp = np.ones(len(pts), F32)
    rsp[8] = 0.0
    T = np.ones((H, W), F32)
    sel = eo.select(pts, rsp, R, t, fx, fy, cx, cy, W, H, T)
    assert sel["xf"][2] == 0 and sel["xf"][3] == -tiny and sel["xf"][4] == below_W and sel["xf"][5] == W
    assert sel["yf"][9] == H and sel["xf"][10] == 0
    assert sel["in_image"].tolist() == [True, True, True, False, True, False, True, True, True, False, True]
    assert _both(oracle32, pts, rsp, R, t, fx, fy, cx, cy, W, H, T).tolist() == [0, 2, 4, 6, 10]
    # the 0.99 threshold: alpha one ulp below 0.99f is in, exactly 0.99f and one ulp above are out; T = 0 is out
    T_below, T_at, T_above = alpha_thresholds()
    T2 = T.copy()
    T2[2, 2], T2[2, 0], T2[1, 7], T2[2, 3] = T_at, T_below, T_above, 0.0
    assert _both(oracle32, pts, rsp, R, t, fx, fy, cx, cy, W, H, T2).tolist() == [2, 10]
    # a dropped winner does not hand its pixel to the runner-up
    assert 1 not in _both(oracle32, pts, rsp, R, t, fx, fy, cx, cy, W, H, T2).tolist()
    # depth_rsp at 0.0, -0.0 and the smallest subnormal
    rsp2 = rsp.copy()
    rsp2[[0, 2, 4]] = [0.0, -0.0, tiny]
    assert _both(oracle32, pts, rsp2, R, t, fx, fy, cx, cy, W, H, T).tolist() == [4, 6, 10]


def test_ties_and_signed_zero_depths():
    """Equal depths go to the smaller index whatever the input order; -0.0 and +0.0 are one depth.  A zero camera depth
    projects to +-inf or NaN and never takes part, so the fold only matters to the restatement's own sort."""
    W, H = 4, 4
    R, t = np.eye(3, dtype=F32), np.zeros(3, F32)
    T = np.ones((H, W), F32)
    pts = np.array([[0.1, 0.1, 1.0]] * 3 + [[0.12, 0.13, 1.0]], F32)
    for perm in ([0, 1, 2, 3], [3, 2, 1, 0]):
        sel = eo.select(pts[perm], np.ones(4, F32), R, t, 1.0, 1.0, 2.0, 2.0, W, H, T)
        assert sel["keep"].tolist() == [0]
    cam = np.array([[0.0, 0.0, -0.0], [0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, np.inf], [1.0, 1.0, -np.inf],
                    [np.nan, 0.0, 1.0], [0.0, np.nan, 1.0], [0.0, 0.0, np.nan]], F32)
    sel = eo.select(None, np.ones(len(cam), F32), None, None, 1.0, 1.0, 2.0, 2.0, W, H, T, cam=cam)
    assert sel["in_image"].tolist() == [False, False, False, True, True, False, False, False]
    # z = +inf and z = -inf both land on the principal point (x / +-inf = +-0): the -inf depth wins the pixel
    assert sel["keep"].tolist() == [4]
