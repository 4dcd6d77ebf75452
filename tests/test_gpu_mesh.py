"""Meshing on the GPU (mesh.cu, glic_mapper_extract_mesh): integration and extraction against the NumPy restatement bit for bit
(including a grid of more than 2^24 cells), the sphere properties of the GPU's own mesh, repeatability, argument checks with
nothing enqueued, and the mapper call: equal to render_camera(sky=False) -> glic_tsdf_integrate -> glic_mesh_extract bit for bit
(pose refinement, exposure, a masked keyframe), the frozen map, the binning overflow, allocation failures and the geometry of a
map of opaque Gaussians on a known plane."""
import ctypes as C
import math

import numpy as np
import pytest

import mesh_oracle as mo
from test_mesh_oracle_host import CENTRE, R_S, _sphere_views, check_sphere_mesh

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

DEV = "cuda:0"


def _bits(x):
    return np.ascontiguousarray(x).view(np.uint32 if np.asarray(x).dtype == np.float32 else np.asarray(x).dtype)


def _planes(data, N):
    d = data.cpu().numpy()
    return dict(tsdf=d[:N], weight=d[N:2 * N], col=d[2 * N:].reshape(3, N))


def _same_grid(got, want, what=""):
    for k in ("tsdf", "weight", "col"):
        assert np.array_equal(_bits(got[k]), _bits(want[k])), (what, k)


def _upload_grid(g):
    """a device grid holding the restatement grid g's values"""
    from gaussian_lic_b200 import ops
    grid, data = ops.tsdf_grid(g["origin"], g["s"], g["dims"], DEV)
    data.copy_(torch.from_numpy(np.concatenate([g["tsdf"], g["weight"], g["col"].reshape(-1)])))
    return grid, data


def _gpu_extract(grid):
    from gaussian_lic_b200 import ops
    xyz, rgb, faces = ops.mesh_extract(grid, DEV)
    torch.cuda.synchronize()
    return xyz.cpu().numpy(), rgb.cpu().numpy(), faces.cpu().numpy()


def _same_mesh(got, want, what=""):
    assert got[0].shape == want[0].shape and got[2].shape == want[2].shape, (what, got[0].shape, want[0].shape, got[2].shape, want[2].shape)
    assert np.array_equal(_bits(got[0]), _bits(want[0])), what
    assert np.array_equal(got[1], want[1]), what
    assert np.array_equal(got[2], want[2]), what


def _pack(mask):
    """a [H,W] bool mask -> (device words, words per row) in glic_pack_mask's layout"""
    from gaussian_lic_b200 import capi
    H, W = mask.shape
    wpr = capi.lib.glic_mask_words_per_row(W)
    valid = torch.from_numpy(np.ascontiguousarray(mask, np.uint8)).to(DEV)
    words = torch.empty(H * wpr, dtype=torch.int32, device=DEV)
    count = torch.empty(1, dtype=torch.int32, device=DEV)
    capi.check(capi.lib.glic_pack_mask(H, W, capi.ptr(valid), capi.ptr(words), capi.ptr(count), None), "pack_mask")
    torch.cuda.synchronize()
    return words, wpr


# ---- integration -----------------------------------------------------------------------------------------------------------------
W0, H0, F0 = 96, 72, 70.0


def _views(rng):
    """three views with perturbed analytic depth maps: zeros, NaNs, depths beyond max_depth, masked pixels; the grid reaches
    behind the first camera (z <= 0) and past every frame border"""
    out = []
    for v, pos in enumerate(((0.0, 0.0, -0.5), (0.8, -0.3, -0.2), (-0.6, 0.4, 0.1))):
        R, t = mo.look_at(pos, (0.05, -0.02, 1.6), up=(0.1 * v, -1.0, 0.0))
        depth = mo.sphere_depth(R, t, W0, H0, F0, F0, W0 / 2.0, H0 / 2.0, (0.0, 0.0, 1.6), 0.7)
        depth += (rng.standard_normal(depth.shape) * 0.01).astype(np.float32) * (depth > 0)
        depth[rng.random(depth.shape) < 0.05] = 0.0
        depth[rng.random(depth.shape) < 0.03] = np.nan
        depth[rng.random(depth.shape) < 0.03] = 9.0                      # beyond max_depth
        depth[:, 0] = depth[:, -1] = depth[0, :] = depth[-1, :] = 1.2     # the frame border
        rgb = rng.random((3, H0, W0)).astype(np.float32)
        mask = rng.random((H0, W0)) > 0.1
        mask[10:20, 30:50] = False
        out.append((mo.view_of(R, t), depth.astype(np.float32), rgb, mask if v != 1 else None))
    return out


def _integrate_both(views, dims=(41, 37, 45), origin=(-1.1, -0.9, -0.7), s=0.06, trunc=0.15, max_depth=5.0):
    from gaussian_lic_b200 import ops
    g = mo.new_grid(origin, s, dims)
    grid, data = ops.tsdf_grid(origin, s, dims, DEV)
    N = int(np.prod(dims))
    for q, (view, depth, rgb, mask) in enumerate(views):
        mo.integrate(g, view, W0, H0, F0, F0, W0 / 2.0, H0 / 2.0, depth, rgb, mask, trunc, max_depth)
        words, wpr = _pack(mask) if mask is not None else (None, 0)
        ops.tsdf_integrate(grid, torch.from_numpy(view).to(DEV), W0, H0, F0, F0, W0 / 2.0, H0 / 2.0, torch.from_numpy(depth).to(DEV),
                           torch.from_numpy(rgb).to(DEV), words, wpr, trunc, max_depth)
        torch.cuda.synchronize()
        _same_grid(_planes(data, N), g, "after view %d" % q)
    return g, grid, data


def test_integration_matches_restatement():
    g, grid, data = _integrate_both(_views(np.random.default_rng(1)))
    w = g["weight"]
    _, (X, Y, Z) = mo.lattice(g)
    assert (w == 3).any() and (w == 1).any() and (w == 0).mean() > 0.2 and (Z <= 0.0).any()
    # rgb = None leaves the colour alone
    from gaussian_lic_b200 import ops
    view, depth, _, _ = _views(np.random.default_rng(1))[0]
    before = data.clone()
    ops.tsdf_integrate(grid, torch.from_numpy(view).to(DEV), W0, H0, F0, F0, W0 / 2.0, H0 / 2.0, torch.from_numpy(depth).to(DEV),
                       trunc=0.15, max_depth=5.0)
    mo.integrate(g, view, W0, H0, F0, F0, W0 / 2.0, H0 / 2.0, depth, None, None, 0.15, 5.0)
    N = g["tsdf"].size
    _same_grid(_planes(data, N), g, "without rgb")
    assert torch.equal(data[2 * N:], before[2 * N:])


# ---- extraction --------------------------------------------------------------------------------------------------------------
def test_extraction_matches_restatement():
    g, grid, data = _integrate_both(_views(np.random.default_rng(2)))
    want = mo.extract(g)
    assert want[0].shape[0] > 200 and want[2].shape[0] > 200
    _same_mesh(_gpu_extract(grid), want, "fused grid")


def _analytic_grid(dims, s, seed, holes=True):
    """a grid holding the signed distance (clipped to [-1, 1] in units of 3 s) of two spheres, random colours and unobserved
    patches"""
    rng = np.random.default_rng(seed)
    nx, ny, nz = dims
    g = mo.new_grid((0.0, 0.0, 0.0), s, dims)
    _, (X, Y, Z) = mo.lattice(g)
    ext = np.array([nx, ny, nz], np.float64) * s
    d1 = np.sqrt((X - 0.45 * ext[0]) ** 2 + (Y - 0.5 * ext[1]) ** 2 + (Z - 0.5 * ext[2]) ** 2) - 0.3 * ext.min()
    d2 = np.sqrt((X - 0.7 * ext[0]) ** 2 + (Y - 0.4 * ext[1]) ** 2 + (Z - 0.6 * ext[2]) ** 2) - 0.2 * ext.min()
    g["tsdf"][:] = np.clip(np.minimum(d1, d2) / (3 * s), -1, 1).astype(np.float32)
    g["weight"][:] = rng.integers(1, 4, g["tsdf"].size).astype(np.float32)
    if holes:
        g["weight"][rng.random(g["tsdf"].size) < 0.001] = 0.0
    g["col"][:] = rng.random(g["col"].shape).astype(np.float32) * 1.2 - 0.1
    return g


@pytest.mark.parametrize("dims", [(2, 2, 2), (3, 5, 2), (33, 17, 9), (260, 258, 256)])
def test_extraction_of_analytic_grids(dims):
    g = _analytic_grid(dims, 0.01, sum(dims))
    if dims == (2, 2, 2):
        g["tsdf"][:] = [-0.5, 0.25, 0.5, 0.5, 0.5, 0.5, 0.5, 0.5]
    cells = (dims[0] - 1) * (dims[1] - 1) * (dims[2] - 1)
    want = mo.extract(g)
    grid, data = _upload_grid(g)
    got = _gpu_extract(grid)
    _same_mesh(got, want, str(dims))
    if cells > 2 ** 24:
        print("%s: %d cells, %d vertices, %d faces" % (dims, cells, want[0].shape[0], want[2].shape[0]))
        assert want[2].shape[0] > 2 ** 16


# ---- the sphere on the GPU, repeatability ------------------------------------------------------------------------------------
def _gpu_sphere(s=0.05, W=160, H=160, f=150.0):
    from gaussian_lic_b200 import ops
    trunc = 3 * s
    m = int(math.ceil((R_S + 4 * s) / s))
    dims = (2 * m + 1,) * 3
    grid, data = ops.tsdf_grid(CENTRE - m * s, s, dims, DEV)
    rgb = torch.from_numpy(np.stack([np.full((H, W), v, np.float32) for v in (0.9, 0.4, 0.1)])).to(DEV)
    for R, t in _sphere_views():
        depth = mo.sphere_depth(R, t, W, H, f, f, W / 2.0, H / 2.0, CENTRE, R_S)
        ops.tsdf_integrate(grid, torch.from_numpy(mo.view_of(R, t)).to(DEV), W, H, f, f, W / 2.0, H / 2.0, torch.from_numpy(depth).to(DEV),
                           rgb, trunc=trunc)
    return grid, data


def test_sphere_on_the_gpu():
    grid, data = _gpu_sphere()
    xyz, rgb, faces = _gpu_extract(grid)
    err, bound = check_sphere_mesh(xyz, faces, 0.05)
    print("GPU sphere: %d vertices, %d faces, max distance %.4f (bound %.4f)" % (xyz.shape[0], faces.shape[0], err, bound))


def test_repeatable():
    a_grid, a_data = _gpu_sphere()
    b_grid, b_data = _gpu_sphere()
    torch.cuda.synchronize()
    assert torch.equal(a_data.view(torch.int32), b_data.view(torch.int32))
    _same_mesh(_gpu_extract(a_grid), _gpu_extract(b_grid), "repeat")


# ---- argument checks ------------------------------------------------------------------------------------------------------------
def test_rejected_arguments_enqueue_nothing():
    from gaussian_lic_b200 import capi, ops
    lib = capi.lib
    grid, data = ops.tsdf_grid((0, 0, 0), 0.1, (8, 8, 8), DEV)
    view = torch.eye(4, dtype=torch.float32, device=DEV).reshape(16)
    depth = torch.ones(16, 16, device=DEV)
    need = lib.glic_mesh_scratch_bytes(grid.dims)
    scratch = torch.empty(need, dtype=torch.uint8, device=DEV)
    cnt = (C.c_uint64 * 2)()
    out = torch.empty(64, dtype=torch.int32, device=DEV)
    torch.cuda.synchronize()

    def bad(**kw):
        g = capi.TsdfGrid()
        g.origin[:], g.voxel_size, g.dims[:], g.data = list(grid.origin), grid.voxel_size, list(grid.dims), grid.data
        for k, v in kw.items():
            if k in ("origin", "dims"):
                getattr(g, k)[:] = v
            elif k in ("voxel_size", "data"):
                setattr(g, k, v)
        return g

    def integ(g, **kw):
        a = dict(view=capi.ptr(view), W=16, H=16, fx=10.0, fy=10.0, cx=8.0, cy=8.0, depth=capi.ptr(depth), rgb=None, mask=None, wpr=0,
                 trunc=0.1, max_depth=0.0)
        a.update(kw)
        return lib.glic_tsdf_integrate(C.byref(g), a["view"], a["W"], a["H"], a["fx"], a["fy"], a["cx"], a["cy"], a["depth"], a["rgb"],
                                       a["mask"], a["wpr"], a["trunc"], a["max_depth"], None)

    launches = capi.launch_count()
    ok = bad()
    cases = [integ(bad(data=None)), integ(bad(dims=(1, 8, 8))), integ(bad(dims=(8, 2049, 8))), integ(bad(dims=(2048, 2048, 512))),
             integ(bad(voxel_size=0.0)), integ(bad(voxel_size=float("inf"))), integ(bad(origin=(float("nan"), 0, 0))),
             integ(ok, view=None), integ(ok, depth=None), integ(ok, W=0), integ(ok, H=-1), integ(ok, W=4096, H=4097),
             integ(ok, fx=0.0), integ(ok, fy=float("nan")), integ(ok, cx=float("inf")), integ(ok, trunc=0.0), integ(ok, trunc=-1.0),
             integ(ok, trunc=float("inf")), integ(ok, max_depth=-1.0), integ(ok, max_depth=float("nan")),
             integ(ok, mask=capi.ptr(out), wpr=0),
             lib.glic_tsdf_clear(C.byref(bad(dims=(8, 8, 1))), None), lib.glic_tsdf_clear(None, None),
             lib.glic_mesh_count(C.byref(bad(dims=(0, 8, 8))), capi.ptr(scratch), need, cnt, None),
             lib.glic_mesh_count(C.byref(ok), None, need, cnt, None), lib.glic_mesh_count(C.byref(ok), capi.ptr(scratch), need, None, None),
             lib.glic_mesh_extract(C.byref(ok), capi.ptr(scratch), need, None, capi.ptr(out), capi.ptr(out), None),
             lib.glic_mesh_extract(C.byref(bad(voxel_size=-1.0)), capi.ptr(scratch), need, capi.ptr(out), capi.ptr(out), capi.ptr(out), None)]
    assert cases == [-1] * len(cases), cases
    assert lib.glic_mesh_count(C.byref(ok), capi.ptr(scratch), need - 1, cnt, None) == -2
    assert lib.glic_mesh_extract(C.byref(ok), capi.ptr(scratch), need - 1, capi.ptr(out), capi.ptr(out), capi.ptr(out), None) == -2
    assert capi.launch_count() == launches
    torch.cuda.synchronize()


# ---- the mapper ----------------------------------------------------------------------------------------------------------------
MESH = dict(origin=(-3.0, -2.5, 3.0), voxel_size=0.08, dims=(76, 64, 120), trunc=0.3)


def _masked_trained():
    from test_gpu_align import _trained
    from test_gpu_mapper_grads import H, W, _keyframes, _scene
    raw = _scene(3)
    poses, cams, gts = _keyframes(seed=61)
    m = _trained(raw, poses, gts)
    mask = np.ones((H, W), bool)
    mask[40:120, 100:220] = False
    m.set_mask(True, 1, mask)
    return m, poses


def _composition(m, views, p):
    """extract_mesh restated through the public calls: render_camera(sky=False) -> glic_tsdf_integrate -> glic_mesh_extract"""
    from gaussian_lic_b200 import ops
    c = m.cfg
    grid, data = ops.tsdf_grid(p["origin"], p["voxel_size"], p["dims"], DEV)
    for k in views:
        R, t, cam = m.pose(k, camera=True)
        out = m.render_camera(R, t, sky=False, outputs=("rgb", "median_depth"))
        mask, n = m.mask(True, k)
        words, wpr = _pack(mask.astype(bool)) if n else (None, 0)
        ops.tsdf_integrate(grid, torch.from_numpy(cam["view"]).to(DEV), m.W, m.H, c.fx, c.fy, c.cx, c.cy,
                           torch.from_numpy(out["median_depth"]).to(DEV), torch.from_numpy(out["rgb"]).to(DEV), words, wpr, p["trunc"],
                           p.get("max_depth", 0.0))
    return _gpu_extract(grid), data


def _mesh_tuple(d):
    return d["vertices"], d["colors"], d["faces"]


def test_mapper_mesh_is_the_composition():
    m, poses = _masked_trained()
    for views, extra in ((None, {}), ([2, 0], dict(max_depth=9.0)), ([1, 1], {})):
        p = dict(MESH, **extra)
        got = m.extract_mesh(views=views, **p)
        want, data = _composition(m, range(3) if views is None else views, p)
        assert got["n_vertices"] > 100 and got["n_faces"] > 100, got["n_vertices"]
        _same_mesh(_mesh_tuple(got), want, str(views))
        N = int(np.prod(p["dims"]))
        assert got["observed_voxels"] == int((data[N:2 * N] > 0).sum())
    m.close()


def test_masked_pixels_are_not_fused():
    m, poses = _masked_trained()
    a = m.extract_mesh(views=[1], **MESH)
    m.set_mask(True, 1, None)
    b = m.extract_mesh(views=[1], **MESH)
    assert a["observed_voxels"] < b["observed_voxels"]
    m.close()


def test_mapper_mesh_leaves_the_map_frozen(tmp_path):
    from test_gpu_align import _same, _snapshot
    m, poses = _masked_trained()
    twin, _ = _masked_trained()
    before = _snapshot(m, 3)
    got = m.extract_mesh(**MESH)
    _same(before, _snapshot(m, 3))
    assert m.sample_views() == twin.sample_views()                    # the sampler's state is the twin's
    twin.close()
    path = tmp_path / "mesh.ply"
    m.save_mesh(path)
    data = path.read_bytes()
    assert data.startswith(b"ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % got["n_vertices"])
    assert len(data) == data.index(b"end_header\n") + 11 + 15 * got["n_vertices"] + 13 * got["n_faces"]
    m.close()


def test_binning_overflow_is_redrawn():
    m, poses = _masked_trained()
    want = m.extract_mesh(**MESH)
    m.set_binning_pairs(1000)
    regrows = m.stats().overflow_regrows
    got = m.extract_mesh(**MESH)
    assert m.stats().overflow_regrows > regrows
    _same_mesh(_mesh_tuple(got), _mesh_tuple(want), "overflow")
    m.close()


def test_allocation_failures_change_nothing():
    from gaussian_lic_b200 import capi
    from test_gpu_align import _same, _snapshot
    m, poses = _masked_trained()
    first = m.extract_mesh(views=[0], **MESH)
    p = dict(MESH, dims=(80, 60, 100))
    failures = 0
    for k in range(1, 20):
        m.set_binning_pairs(5000)
        before = _snapshot(m, 3)
        assert capi.lib.glic_debug_fail_allocation(k) == 0
        try:
            got = m.extract_mesh(**p)
            ok = True
        except capi.GlicError as e:
            assert "(-3)" in str(e), (k, str(e))
            ok = False
        finally:
            capi.lib.glic_debug_fail_allocation(0)
        if ok:
            break
        failures += 1
        _same(before, _snapshot(m, 3))
        _same_mesh(_mesh_tuple(m.mesh()), _mesh_tuple(first), "allocation %d" % k)
    else:
        raise AssertionError("extract_mesh never succeeded")
    print("extract_mesh: %d allocations failed in turn" % failures)
    assert failures >= 5 and got["n_vertices"] > 0
    m.close()


def test_mapper_rejected_arguments_change_nothing():
    from gaussian_lic_b200 import capi, mapper
    from test_gpu_mapper_grads import F, H, W
    m, poses = _masked_trained()
    first = m.extract_mesh(views=[0], **MESH)
    launches = capi.launch_count()
    for kw in (dict(dims=(1, 64, 64)), dict(dims=(2049, 8, 8)), dict(voxel_size=0.0), dict(voxel_size=float("nan")), dict(trunc=0.0),
               dict(trunc=float("inf")), dict(max_depth=-1.0), dict(max_depth=float("nan")), dict(views=[3]), dict(views=[-1]),
               dict(origin=(float("inf"), 0, 0))):
        with pytest.raises(capi.GlicError, match=r"\(-1\)"):
            m.extract_mesh(**dict(MESH, **kw))
    p = capi.MeshParams()
    p.n_views, p.voxel_size, p.dims[:], p.trunc = -1, 0.1, [8, 8, 8], 0.1
    keep = (C.c_int * 1)(0)
    p.views = C.cast(keep, C.c_void_p)
    assert capi.lib.glic_mapper_extract_mesh(m._h, C.byref(p), None) == -1
    assert capi.launch_count() == launches
    _same_mesh(_mesh_tuple(m.mesh()), _mesh_tuple(first), "rejected")
    m.close()
    empty = mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=0)
    with pytest.raises(capi.GlicError, match="no non-sky rows"):
        empty.extract_mesh(**MESH)
    with pytest.raises(capi.GlicError, match="no mesh"):
        empty.save_mesh("/tmp/never-written.ply")
    empty.close()


def test_plane_of_opaque_gaussians():
    """opaque flat Gaussians tiling the plane z = Z_P in front of the orbit cameras: every vertex near the plane"""
    from gaussian_lic_b200 import mapper, synthetic as syn
    from test_gpu_mapper_grads import F, H, W
    Z_P, step, sigma = 12.0, 0.05, 0.04
    xs = np.arange(-4.0, 4.0 + 1e-9, step)
    X, Y = np.meshgrid(xs, xs * 0.75)
    P = X.size
    raw = dict(means=np.stack([X.ravel(), Y.ravel(), np.full(P, Z_P)], 1).astype(np.float32),
               log_scales=np.log(np.tile([sigma, sigma, 0.002], (P, 1))).astype(np.float32),
               rots=np.tile([1.0, 0.0, 0.0, 0.0], (P, 1)).astype(np.float32), opacity_logits=np.full(P, 6.0, np.float32),
               dc=np.full((P, 3), 0.3, np.float32), sh=np.zeros((P, 0, 3), np.float32), degree=0)
    m = mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=0)
    m.initialize(raw)
    for v in (0, 1, 7):
        m.add_keyframe(*syn.orbit_pose(v, radius=2.0), np.zeros((3, H, W), np.float32))
    s = 0.05
    got = m.extract_mesh(origin=(-3.0, -2.0, 11.0), voxel_size=s, dims=(121, 81, 41), trunc=4 * s)
    xyz = got["vertices"]
    assert got["n_vertices"] > 1000 and got["n_faces"] > 1000
    # Bound: the median depth of a pixel is the view-space depth of a splat centre whose 3-sigma footprint covers the pixel, so it
    # differs from the plane's depth along that ray by at most 3 sigma tan(theta), theta the largest angle between a ray and the
    # plane's normal (a camera's axis tilt plus the half diagonal of its field of view); a vertex then lies in a cell whose corners
    # straddle that depth: one voxel more.
    tilt = max(math.acos(float(np.asarray(syn.orbit_pose(v, radius=2.0)[0])[2, 2])) for v in (0, 1, 7))
    theta = tilt + math.atan(math.hypot(W, H) / (2 * F))
    bound = s + 3 * sigma * math.tan(theta)
    err = np.abs(xyz[:, 2].astype(np.float64) - Z_P)
    print("plane: %d vertices, max |z - Z_P| %.4f (bound %.4f)" % (xyz.shape[0], err.max(), bound))
    assert err.max() <= bound
    m.close()
