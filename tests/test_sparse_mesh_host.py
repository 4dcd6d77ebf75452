"""The sparse grid's allocation rule on the CPU (tests/sparse_mesh_oracle.py): a hand-worked pixel, and its sufficiency against
the dense restatement of mesh_oracle.py on random views, a plane at 85 degrees, lattice points on pixel borders, depths at
max_depth, a box near the +2^19 lattice edge and a clipped view: every point some view gives t < 0, with its +-1
neighbourhood, lies in an allocated block, and the dense mesh restricted to the allocated blocks is the dense mesh."""
import numpy as np

import mesh_oracle as mo
import sparse_mesh_oracle as so
from test_mesh_oracle_host import CENTRE, R_S, _sphere_views


def test_one_pixel_by_hand():
    """identity camera, f = 10, c = 0: pixel (0, 0) at depth 1, trunc 1 covers x, y in [0, 0.2], z in [1, 2]"""
    view = mo.view_of(np.eye(3), np.zeros(3))
    depth = np.zeros((4, 4), np.float32)
    depth[0, 0] = 1.0
    L, H, clipped = so.pixel_ranges(view, 4, 4, 10.0, 10.0, 0.0, 0.0, depth, None, 1.0, 0.0, (0, 0, 0), 0.25)
    assert L.tolist() == [[-2, -2, 2]] and H.tolist() == [[3, 3, 10]] and not clipped.any()
    keys, n = so.block_set(view, 4, 4, 10.0, 10.0, 0.0, 0.0, depth, None, 1.0, 0.0, (0, 0, 0), 0.25)
    bi, bj, bk = so.key_blocks(keys)
    assert n == 0 and sorted(set(bi.tolist())) == [-1, 0] and sorted(set(bk.tolist())) == [0, 1] and keys.size == 8
    assert (np.diff(keys) > 0).all()


def _plane_depth(R, t, W, H, f, n, c):
    """z-depth [H,W] of the plane n . X = c along the rays through pixel centres"""
    R = np.asarray(R, np.float64)
    C = -R.T @ np.asarray(t, np.float64)
    u = (np.arange(W) + 0.5 - W / 2.0) / f
    v = (np.arange(H) + 0.5 - H / 2.0) / f
    dx, dy = np.meshgrid(u, v)
    dirs = np.stack([dx, dy, np.ones_like(dx)], -1) @ R             # world direction per unit z
    z = (c - np.dot(n, C)) / (dirs @ np.asarray(n, np.float64))
    return np.where(z > 0, z, 0).astype(np.float32)


def check_sufficient(views, W, H, f, trunc, max_depth, origin, s, dims, shift=(0, 0, 0)):
    """views: (view, depth, rgb, mask); the sparse lattice has origin `origin`, the dense box starts at lattice point `shift`"""
    keys, clipped = [], 0
    for view, depth, rgb, mask in views:
        k, c = so.block_set(view, W, H, f, f, W / 2.0, H / 2.0, depth, mask, trunc, max_depth, origin, s)
        keys.append(k)
        clipped += c
    keys = np.unique(np.concatenate(keys))
    dense_origin = np.asarray(origin, np.float32) + np.float32(s) * np.asarray(shift, np.float32)
    g = mo.new_grid(dense_origin, s, dims)
    neg = np.zeros(int(np.prod(dims)), bool)
    for view, depth, rgb, mask in views:
        neg |= so.negative_points(g, view, W, H, f, f, W / 2.0, H / 2.0, depth, mask, trunc, max_depth)
        mo.integrate(g, view, W, H, f, f, W / 2.0, H / 2.0, depth, rgb, mask, trunc, max_depth)
    keep = so.allocated(g, keys, shift)
    assert neg.any()
    assert keep[so.dilate(neg, dims)].all(), "a point with t < 0 or a neighbour of one is in no allocated block"
    want = mo.extract(g)
    got = mo.extract(so.restrict(g, keep))
    assert want[2].shape[0] > 50
    for a, b in zip(got, want):
        assert a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))
    assert (g["weight"][keep] > 0).sum() <= (g["weight"] > 0).sum()
    return keys, clipped


def _sphere_scene(rng, W=64, H=48, f=50.0):
    views = []
    for R, t in _sphere_views()[:5]:
        depth = mo.sphere_depth(R, t, W, H, f, f, W / 2.0, H / 2.0, CENTRE, R_S)
        depth += (rng.standard_normal(depth.shape) * 0.01).astype(np.float32) * (depth > 0)
        mask = rng.random((H, W)) > 0.1
        views.append((mo.view_of(R, t), depth, rng.random((3, H, W)).astype(np.float32), mask))
    return views


def test_random_views():
    rng = np.random.default_rng(7)
    s = 0.08
    keys, clipped = check_sufficient(_sphere_scene(rng), 64, 48, 50.0, 0.2, 0.0, (-2.0, -2.1, -2.05), s, (52, 52, 52))
    assert clipped == 0 and keys.size > 20


def test_grazing_plane():
    """the plane y = 0.3 seen at 85 degrees from its normal"""
    W, H, f = 64, 48, 40.0
    a = np.radians(85.0)
    R, t = mo.look_at((0.0, 0.3 - 2.0 * np.cos(a), -2.0 * np.sin(a)), (0.0, 0.3, 0.0))
    depth = _plane_depth(R, t, W, H, f, np.array([0.0, 1.0, 0.0]), 0.3)
    depth[depth > 12] = 0
    views = [(mo.view_of(R, t), depth, np.full((3, H, W), 0.5, np.float32), None)]
    check_sufficient(views, W, H, f, 0.15, 0.0, (-3.0, -0.5, -3.0), 0.05, (120, 30, 200))


def test_points_on_pixel_borders():
    """identity camera, f = 16, c integral, s = 1/16: lattice points at z = 1 project onto pixel borders exactly"""
    W, H, f = 32, 32, 16.0
    view = mo.view_of(np.eye(3), np.zeros(3))
    depth = np.full((H, W), 1.0, np.float32)
    depth[8:12, 8:12] = 1.25
    views = [(view, depth, np.full((3, H, W), 0.25, np.float32), None)]
    check_sufficient(views, W, H, f, 0.125, 0.0, (-1.0, -1.0, 0.5), 0.0625, (34, 34, 20))


def test_far_depths_at_max_depth():
    W, H, f = 48, 40, 30.0
    R, t = mo.look_at((0.0, 0.0, 0.0), (0.1, 0.05, 1.0))
    depth = _plane_depth(R, t, W, H, f, np.array([0.05, 0.02, 1.0]), 3.0)
    max_depth = float(np.median(depth))
    depth[depth > max_depth] = np.float32(max_depth)                  # exactly at max_depth: used
    depth[:, :6] = np.float32(max_depth) * np.float32(1.001)          # beyond it: not used
    views = [(mo.view_of(R, t), depth, np.full((3, H, W), 0.5, np.float32), None)]
    check_sufficient(views, W, H, f, 0.2, max_depth, (-1.5, -1.5, 1.5), 0.05, (60, 50, 40))


def test_box_near_the_lattice_edge():
    """s = 2^-4 and integral origins: the dense box from lattice point 2^19 - 64 rounds as the sparse lattice does"""
    W, H, f = 48, 40, 40.0
    s, i0 = 0.0625, (1 << 19) - 64
    o = (-32760.0, -32760.0, -32760.0)
    base = np.asarray(o) + s * i0                                     # world position of the box's first point
    R, t = mo.look_at(base + (1.5, 1.5, -0.5), base + (1.6, 1.4, 2.0))
    depth = _plane_depth(R, t, W, H, f, np.array([0.0, 0.0, 1.0]), base[2] + 1.5)
    views = [(mo.view_of(R, t), depth, np.full((3, H, W), 0.5, np.float32), None)]
    keys, clipped = check_sufficient(views, W, H, f, 0.25, 0.0, o, s, (60, 60, 40), shift=(i0, i0, i0))
    assert clipped == 0 and (np.stack(so.key_blocks(keys)) >= (1 << 16) - 8).all()


def test_clipped_view_is_reported():
    """the same camera pushed past the lattice edge: its far pixels are clipped and counted"""
    W, H, f = 48, 40, 40.0
    s, i0 = 0.0625, (1 << 19) - 64
    o = np.array([-32760.0, -32760.0, -32760.0])
    base = o + s * i0
    R, t = mo.look_at(base + (1.5, 1.5, 1.0), base + (1.5, 1.5, 9.0))
    depth = np.full((H, W), 2.8, np.float32)                          # the truncation band crosses the last lattice point
    L, Hh, clipped = so.pixel_ranges(mo.view_of(R, t), W, H, f, f, W / 2.0, H / 2.0, depth, None, 0.25, 0.0, o, s)
    assert clipped.all() and (Hh[:, 2] == (1 << 19) - 1).all()
    keys, n = so.block_set(mo.view_of(R, t), W, H, f, f, W / 2.0, H / 2.0, depth, None, 0.25, 0.0, o, s)
    assert n == W * H and keys.size > 0
