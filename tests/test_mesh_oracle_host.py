"""The meshing restatement on the CPU (tests/mesh_oracle.py): the exact fma it uses, a fronto-parallel plane with known fused values
and a known mesh, a sphere fused from analytic depth maps around it (closed, consistently oriented, Euler characteristic 2, its
volume, every vertex near the surface), and glic_mesh_ply_write byte for byte against a writer of its own."""
import ctypes as C
import fractions
import math

import numpy as np
import pytest

import mesh_oracle as mo

f32 = np.float32


def test_fma32_is_the_exact_fma():
    rng = np.random.default_rng(3)
    a = rng.standard_normal(2000).astype(np.float32)
    b = rng.standard_normal(2000).astype(np.float32)
    c = (rng.standard_normal(2000) * 1e-3).astype(np.float32)
    # products whose exact sum with c sits on a float32 rounding midpoint, where rounding twice goes wrong
    a[:4] = [f32(1.0) + f32(2.0 ** -12)] * 4
    b[:4] = [f32(1.0) + f32(2.0 ** -12)] * 4
    c[:4] = [f32(-2.0 ** -30), f32(2.0 ** -30), f32(0.0), f32(-1.0)]
    got = mo.fma32(a, b, c)
    for x, y, z, g in zip(a, b, c, got):
        exact = fractions.Fraction(float(x)) * fractions.Fraction(float(y)) + fractions.Fraction(float(z))
        lo = f32(float(exact))                                  # float(Fraction) rounds once to float64; adjust to the float32 RN
        cand = [np.nextafter(lo, f32(-np.inf)), lo, np.nextafter(lo, f32(np.inf))]
        err = [abs(fractions.Fraction(float(v)) - exact) for v in cand]
        best = min(err)
        ties = [v for v, e in zip(cand, err) if e == best]
        want = ties[0] if len(ties) == 1 else [v for v in ties if (np.array(v).view(np.uint32) & 1) == 0][0]
        assert np.array(g).view(np.uint32) == np.array(want).view(np.uint32), (x, y, z)


def _plane_setup(d=f32(2.03), trunc=0.08):
    W, H, fx = 64, 48, 40.0
    g = mo.new_grid((-1.0, -0.75, 1.6), 0.05, (41, 31, 19))
    depth = np.full((H, W), d, np.float32)
    rgb = np.stack([np.full((H, W), v, np.float32) for v in (0.2, 0.5, 0.8)])
    view = mo.view_of(np.eye(3), np.zeros(3))
    upd = mo.integrate(g, view, W, H, fx, fx, W / 2.0, H / 2.0, depth, rgb, trunc=trunc)
    return g, upd, d, trunc


def test_plane_fused_values():
    g, upd, d, trunc = _plane_setup()
    _, (X, Y, Z) = mo.lattice(g)
    assert upd.any()
    # the identity view: z = Z exactly, so every fused point holds t = min(1, (d - z) / trunc) with weight 1
    want = np.fmin(f32(1), (d - Z[upd]) / f32(trunc))
    assert np.array_equal(g["tsdf"][upd].view(np.uint32), want.view(np.uint32))
    assert (g["weight"][upd] == 1).all() and not g["weight"][~upd].any() and not g["tsdf"][~upd].any()
    assert (Z[upd] <= d + f32(trunc)).all() and not (Z[~upd] <= d).any()
    assert np.array_equal(g["col"][:, upd], np.array([[0.2], [0.5], [0.8]], np.float32) * np.ones(upd.sum(), np.float32))


def test_plane_mesh_is_a_flat_sheet():
    g, _, d, _ = _plane_setup()
    nx, ny, nz = g["dims"]
    xyz, rgb, faces = mo.extract(g)
    assert xyz.shape == ((nx - 1) * (ny - 1), 3)                       # one layer of active cells
    assert faces.shape == (2 * (nx - 2) * (ny - 2), 3)                 # one quad per interior z-edge
    assert np.abs(xyz[:, 2] - d).max() <= 4 * np.spacing(d)
    assert (rgb == np.array([51, 128, 204], np.uint8)).all()
    # normals point out of the surface, into the free space in front of the camera (-z)
    p = xyz.astype(np.float64)[faces]
    n = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    assert (n[:, 2] < 0).all()
    und, dirc = mo.edge_counts(faces)
    assert (dirc == 1).all()                                           # consistently oriented


R_S, CENTRE = 1.0, np.array([0.1, -0.05, 0.02])


def _sphere_views():
    dirs = [(1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1)]
    dirs += [(s1, s2, s3) for s1 in (1, -1) for s2 in (1, -1) for s3 in (1, -1)]
    out = []
    for dv in dirs:
        dv = np.asarray(dv, np.float64) / np.linalg.norm(dv)
        out.append(mo.look_at(CENTRE + 3.0 * R_S * dv, CENTRE, up=(0.3, -1.0, 0.1)))
    return out


def sphere_grid(s=0.05, W=160, H=160, f=150.0, trunc=None):
    """the restatement grid of the sphere fused from 14 views at 3 r"""
    trunc = 3 * s if trunc is None else trunc
    m = int(math.ceil((R_S + 4 * s) / s))
    g = mo.new_grid(CENTRE - m * s, s, (2 * m + 1,) * 3)
    rgb = np.stack([np.full((H, W), v, np.float32) for v in (0.9, 0.4, 0.1)])
    for R, t in _sphere_views():
        depth = mo.sphere_depth(R, t, W, H, f, f, W / 2.0, H / 2.0, CENTRE, R_S)
        mo.integrate(g, mo.view_of(R, t), W, H, f, f, W / 2.0, H / 2.0, depth, rgb, trunc=trunc)
    return g


def check_sphere_mesh(xyz, faces, s, f=150.0, dist=3.0):
    """the sphere properties of a mesh fused by sphere_grid; returns the largest vertex distance from the sphere"""
    assert faces.shape[0] > 1000
    und, dirc = mo.edge_counts(faces)
    assert (und == 2).all(), "not closed: %d edges not in exactly two faces" % (und != 2).sum()
    assert (dirc == 1).all(), "not consistently oriented"
    assert mo.euler_characteristic(xyz, faces) == 2
    vol = mo.signed_volume(xyz, faces)
    assert vol > 0 and abs(vol / (4.0 / 3.0 * math.pi * R_S ** 3) - 1.0) < 0.03, vol
    # Bound: a vertex is a mean of crossing points on the edges of its cell, so it lies in the cell, and the cell has corners of
    # both signs.  A lattice point's fused sign is right wherever every view that fuses it has the surface within the sampling
    # error e of the true depth along its ray: the depth of the pixel centre instead of the point's own ray, at most half a pixel
    # diagonal (sqrt(2)/2 px) from it, i.e. e <= (sqrt(2)/2) (z / f) on a surface seen head-on.  So a vertex is within one voxel
    # of the sphere (a cell with corners of both signs), plus e at the largest depth the views see, plus the sag of the sphere
    # over a cell diagonal (3 s^2 / (8 r)).
    e = math.sqrt(2) / 2 * dist * R_S / f
    bound = s + e + 3 * s * s / (8 * R_S)
    err = np.abs(np.linalg.norm(xyz.astype(np.float64) - CENTRE, axis=1) - R_S)
    assert err.max() <= bound, (err.max(), bound)
    return err.max(), bound


def test_sphere_mesh_is_closed_and_on_the_sphere():
    s = 0.05
    g = sphere_grid(s)
    xyz, rgb, faces = mo.extract(g)
    err, bound = check_sphere_mesh(xyz, faces, s)
    print("sphere: %d vertices, %d faces, max distance %.4f (bound %.4f)" % (xyz.shape[0], faces.shape[0], err, bound))
    assert (np.abs(rgb.astype(np.int32) - [230, 102, 26]) <= 1).all()      # means of one colour: 0.9 * 255 = 229.5 rounds either way


# ---- the PLY writer ---------------------------------------------------------------------------------------------------------
def _numpy_mesh_ply(xyz, rgb, faces):
    V, F = xyz.shape[0], faces.shape[0]
    head = ("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n"
            "property uchar red\nproperty uchar green\nproperty uchar blue\nelement face %d\nproperty list uchar int vertex_indices\n"
            "end_header\n" % (V, F)).encode()
    vt = np.dtype([("p", "<f4", 3), ("c", "u1", 3)])
    ft = np.dtype([("n", "u1"), ("i", "<i4", 3)])
    v = np.empty(V, vt)
    v["p"], v["c"] = xyz, rgb
    fa = np.empty(F, ft)
    fa["n"], fa["i"] = 3, faces
    return head + v.tobytes() + fa.tobytes()


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a.size else None


@pytest.mark.parametrize("V,F", [(0, 0), (5, 3), (5000, 9001)])
def test_mesh_ply_writer_bytes(tmp_path, V, F):
    from gaussian_lic_b200 import capi
    rng = np.random.default_rng(V + F)
    xyz = rng.standard_normal((V, 3)).astype(np.float32)
    rgb = rng.integers(0, 256, (V, 3)).astype(np.uint8)
    faces = rng.integers(0, max(V, 1), (F, 3)).astype(np.int32)
    path = tmp_path / "m.ply"
    capi.check(capi.lib.glic_mesh_ply_write(str(path).encode(), V, _ptr(xyz), _ptr(rgb), F, _ptr(faces)), "mesh_ply_write")
    data = path.read_bytes()
    assert data == _numpy_mesh_ply(xyz, rgb, faces)
    # read back through the header
    end = data.index(b"end_header\n") + len(b"end_header\n")
    body = data[end:]
    v = np.frombuffer(body[:15 * V], np.dtype([("p", "<f4", 3), ("c", "u1", 3)]))
    fa = np.frombuffer(body[15 * V:], np.dtype([("n", "u1"), ("i", "<i4", 3)]))
    assert np.array_equal(v["p"], xyz) and np.array_equal(v["c"], rgb) and (fa["n"] == 3).all() and np.array_equal(fa["i"], faces)


def test_mesh_ply_writer_fails_loudly(tmp_path):
    from gaussian_lic_b200 import capi
    xyz = np.zeros((1, 3), np.float32)
    rgb = np.zeros((1, 3), np.uint8)
    assert capi.lib.glic_mesh_ply_write(str(tmp_path / "no" / "such" / "dir.ply").encode(), 1, _ptr(xyz), _ptr(rgb), 0, None) == -1
    assert b"cannot open" in capi.lib.glic_last_error()
    assert capi.lib.glic_mesh_ply_write(str(tmp_path / "a.ply").encode(), 1, None, _ptr(rgb), 0, None) == -1
    assert capi.lib.glic_mesh_ply_write(None, 0, None, None, 0, None) == -1
    if __import__("os").path.exists("/dev/full"):
        assert capi.lib.glic_mesh_ply_write(b"/dev/full", 1, _ptr(xyz), _ptr(rgb), 0, None) == -1


def test_grid_sizes():
    from gaussian_lic_b200 import capi
    d = (C.c_int * 3)(512, 512, 512)
    assert capi.lib.glic_tsdf_bytes(d) == 20 * 512 ** 3
    assert capi.lib.glic_mesh_scratch_bytes(d) < 512 ** 3 // 3
    for bad in ((1, 4, 4), (4, 4, 2049), (2048, 2048, 512), (-3, 4, 4)):
        d = (C.c_int * 3)(*bad)
        assert capi.lib.glic_tsdf_bytes(d) == 0 and capi.lib.glic_mesh_scratch_bytes(d) == 0
