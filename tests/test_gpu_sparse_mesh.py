"""The sparse block TSDF on the GPU (sparse_mesh.cu, glic_mapper_extract_mesh_sparse): the block set equals the float64
restatement of the allocation rule in any insertion order and after an overflow, grow and repeat; every voxel of every block and
the whole mesh equal the dense kernels' bit for bit (random views with masks, the analytic sphere, negative lattice indices);
repeatability; argument checks with nothing enqueued; and the mapper call equal to glic_mapper_extract_mesh on a trained map."""
import ctypes as C

import numpy as np
import pytest

import mesh_oracle as mo
import sparse_mesh_oracle as so
from test_gpu_mesh import DEV, F0, H0, MESH, W0, _bits, _gpu_extract, _masked_trained, _pack, _planes, _same_mesh, _sphere_views, _views
from test_mesh_oracle_host import CENTRE, R_S, check_sphere_mesh

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


def _dev(views):
    """views as device tensors: (view, depth, rgb, (words, wpr)), and the host mask"""
    out = []
    for view, depth, rgb, mask in views:
        out.append((torch.from_numpy(view).to(DEV), torch.from_numpy(depth).to(DEV), torch.from_numpy(rgb).to(DEV),
                    _pack(mask) if mask is not None else (None, 0), mask, view, depth))
    return out


def _insert_all(dv, origin, s, trunc, max_depth, W=W0, H=H0, f=F0, capacity=1 << 14, order=None):
    from gaussian_lic_b200 import ops
    st, data = ops.block_set(capacity, DEV)
    keep = [data]
    n = clipped = 0
    for q in (order if order is not None else range(len(dv))):
        view, depth, rgb, (words, wpr) = dv[q][:4]
        while True:
            n, c, over = ops.block_set_insert(st, origin, s, view, W, H, f, f, W / 2.0, H / 2.0, depth, words, wpr, trunc, max_depth)
            if not over:
                clipped += c
                break
            bigger, bdata = ops.block_set(2 * st.capacity, DEV)
            ops.block_set_copy(st, bigger)
            st, keep = bigger, keep + [bdata]
    return st, keep, n, clipped


def _restated_keys(dv, origin, s, trunc, max_depth, W=W0, H=H0, f=F0):
    keys = [so.block_set(v[5], W, H, f, f, W / 2.0, H / 2.0, v[6], v[4], trunc, max_depth, origin, s)[0] for v in dv]
    return np.unique(np.concatenate(keys))


def _sparse(dv, origin, s, trunc, max_depth, W=W0, H=H0, f=F0, **kw):
    """insert every view, build the grid, integrate every view: (grid, data, n, clipped, set memory kept alive)"""
    from gaussian_lic_b200 import ops
    st, keep, n, clipped = _insert_all(dv, origin, s, trunc, max_depth, W, H, f, **kw)
    grid, data = ops.sparse_tsdf(origin, s, st, n, DEV)
    for view, depth, rgb, (words, wpr) in (v[:4] for v in dv):
        ops.sparse_tsdf_integrate(grid, view, W, H, f, f, W / 2.0, H / 2.0, depth, rgb, words, wpr, trunc, max_depth)
    torch.cuda.synchronize()
    return grid, data, n, clipped, keep


def _dense(dv, origin, s, dims, trunc, max_depth, W=W0, H=H0, f=F0):
    from gaussian_lic_b200 import ops
    grid, data = ops.tsdf_grid(origin, s, dims, DEV)
    for view, depth, rgb, (words, wpr) in (v[:4] for v in dv):
        ops.tsdf_integrate(grid, view, W, H, f, f, W / 2.0, H / 2.0, depth, rgb, words, wpr, trunc, max_depth)
    torch.cuda.synchronize()
    return grid, data


def _check_equivalent(sgrid, dgrid, ddata, dims, shift=(0, 0, 0)):
    """(a) every voxel of every block equals the dense grid's, (b) the meshes are equal, (c) observed counts.  With a shifted
    dense box, a vertex o + s ((float)i + offset) rounds (float)i + offset at a different i, so vertex positions are compared
    within that rounding there and everything else bit for bit."""
    from gaussian_lic_b200 import ops
    keys, pool = ops.sparse_tsdf_planes(sgrid, DEV)
    keys, pool = keys.cpu().numpy(), pool.cpu().numpy()
    assert (np.diff(keys) > 0).all()
    bi, bj, bk = so.key_blocks(keys)
    v = np.arange(512)
    i = (bi[:, None] * 8 + (v & 7)) - shift[0]
    j = (bj[:, None] * 8 + ((v >> 3) & 7)) - shift[1]
    k = (bk[:, None] * 8 + (v >> 6)) - shift[2]
    nx, ny, nz = dims
    assert i.min() >= 0 and j.min() >= 0 and k.min() >= 0 and i.max() < nx and j.max() < ny and k.max() < nz, "the dense box is too small"
    N = nx * ny * nz
    d = _planes(ddata, N)
    L = (i + nx * (j + ny * k)).ravel()
    assert np.array_equal(_bits(pool[:, 0].ravel()), _bits(d["tsdf"][L]))
    assert np.array_equal(_bits(pool[:, 1].ravel()), _bits(d["weight"][L]))
    for c in range(3):
        assert np.array_equal(_bits(pool[:, 2 + c].ravel()), _bits(d["col"][c][L]))
    xyz, rgb, faces, counts = ops.sparse_mesh_extract(sgrid, DEV)
    torch.cuda.synchronize()
    got = (xyz.cpu().numpy(), rgb.cpu().numpy(), faces.cpu().numpy())
    want = _gpu_extract(dgrid)
    if shift == (0, 0, 0):
        _same_mesh(got, want, "sparse vs dense")
    else:
        assert got[0].shape == want[0].shape and np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2])
        assert np.abs(got[0] - want[0]).max() <= sgrid.voxel_size * 2.0 ** -8
    obs = int((pool[:, 1] > 0).sum())
    assert counts.observed_voxels == obs <= int((d["weight"] > 0).sum())
    assert counts.blocks == keys.size
    assert tuple(counts.lattice_lo) == (8 * bi.min(), 8 * bj.min(), 8 * bk.min())
    assert tuple(counts.lattice_hi) == (8 * bi.max() + 7, 8 * bj.max() + 7, 8 * bk.max() + 7)
    return got, counts


ORIGIN, S, TRUNC, MAXD = (-3.0, -3.0, -2.0), 0.06, 0.15, 5.0
DIMS = (110, 110, 130)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_block_set_is_the_restatement_in_any_order(seed):
    from gaussian_lic_b200 import ops
    dv = _dev(_views(np.random.default_rng(seed)))
    want = _restated_keys(dv, ORIGIN, S, TRUNC, MAXD)
    for order in ((0, 1, 2), (2, 0, 1), (1, 2, 0)):
        grid, data, n, clipped, keep = _sparse(dv, ORIGIN, S, TRUNC, MAXD, order=order)
        keys, _ = ops.sparse_tsdf_planes(grid, DEV)
        assert clipped == 0 and n == want.size
        assert np.array_equal(keys.cpu().numpy(), want), order


def test_overflow_grow_and_repeat_gives_the_same_set():
    from gaussian_lic_b200 import ops
    dv = _dev(_views(np.random.default_rng(4)))
    want = _restated_keys(dv, ORIGIN, S, TRUNC, MAXD)
    assert want.size > 64
    grid, data, n, clipped, keep = _sparse(dv, ORIGIN, S, TRUNC, MAXD, capacity=16)
    assert len(keep) > 2                                              # it grew more than once
    keys, _ = ops.sparse_tsdf_planes(grid, DEV)
    assert np.array_equal(keys.cpu().numpy(), want)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_scenes_equal_the_dense_grid(seed):
    dv = _dev(_views(np.random.default_rng(seed)))
    sgrid, sdata, n, clipped, keep = _sparse(dv, ORIGIN, S, TRUNC, MAXD)
    dgrid, ddata = _dense(dv, ORIGIN, S, DIMS, TRUNC, MAXD)
    got, counts = _check_equivalent(sgrid, dgrid, ddata, DIMS)
    assert got[2].shape[0] > 200 and clipped == 0


def test_sphere_equals_the_dense_grid_and_is_closed():
    s, W, H, f = 0.05, 160, 160, 150.0
    rgb = np.stack([np.full((H, W), v, np.float32) for v in (0.9, 0.4, 0.1)])
    views = [(mo.view_of(R, t), mo.sphere_depth(R, t, W, H, f, f, W / 2.0, H / 2.0, CENTRE, R_S), rgb, None) for R, t in _sphere_views()]
    dv = _dev(views)
    m = 40
    origin = tuple(np.asarray(CENTRE - m * s, np.float32))
    sgrid, sdata, n, clipped, keep = _sparse(dv, origin, s, 3 * s, 0.0, W, H, f)
    dgrid, ddata = _dense(dv, origin, s, (2 * m + 1,) * 3, 3 * s, 0.0, W, H, f)
    (xyz, rgb8, faces), counts = _check_equivalent(sgrid, dgrid, ddata, (2 * m + 1,) * 3)
    check_sphere_mesh(xyz, faces, s)
    assert mo.euler_characteristic(xyz, faces) == 2


def test_negative_lattice_indices():
    """s = 2^-4 and an integral origin inside the scene: a dense grid from lattice point -64 computes every lattice position,
    hence every voxel, identically"""
    s, shift = 0.0625, (-64, -64, -40)
    views = _views(np.random.default_rng(5))
    dv = _dev(views)
    origin = (1.0, 1.0, 1.0)
    sgrid, sdata, n, clipped, keep = _sparse(dv, origin, s, TRUNC, MAXD)
    dense_origin = tuple(np.float32(o) + np.float32(s) * np.float32(d) for o, d in zip(origin, shift))
    dims = (104, 100, 120)
    dgrid, ddata = _dense(dv, dense_origin, s, dims, TRUNC, MAXD)
    got, counts = _check_equivalent(sgrid, dgrid, ddata, dims, shift)
    assert min(counts.lattice_lo) < 0 and got[2].shape[0] > 200


def test_large_extent_is_the_union_of_dense_clusters():
    """two copies of a scene 8000 lattice points apart (s = 2^-4, integral origins, so every lattice position is exact): each
    cluster's voxels equal a dense grid's at its own origin bit for bit, and the sparse mesh is the union of the two dense meshes.
    A vertex is o + s ((float)i + offset), and (float)i + offset keeps fewer bits of the offset at i near 8000 than near 0, so
    vertices far from the dense grid's origin are compared within that rounding; the face lists must match exactly."""
    from scipy.spatial import cKDTree
    from gaussian_lic_b200 import ops
    s, gap = 0.0625, 8000
    base = _views(np.random.default_rng(6))
    far = []
    for view, depth, rgb, mask in base:                               # the same cameras moved by gap voxels along x
        m = view.reshape(4, 4).T.copy()
        m[:3, 3] -= m[:3, :3] @ np.array([gap * s, 0.0, 0.0], np.float32)
        far.append((np.ascontiguousarray(m.T).reshape(16).astype(np.float32), depth, rgb, mask))
    origin = (-3.0, -3.0, -1.0)
    sgrid, sdata, n, clipped, keep = _sparse(_dev(base + far), origin, s, TRUNC, MAXD)
    xyz, rgb8, faces, counts = ops.sparse_mesh_extract(sgrid, DEV)
    assert counts.lattice_hi[0] - counts.lattice_lo[0] > 8000
    keys, pool = ops.sparse_tsdf_planes(sgrid, DEV)
    keys, pool = keys.cpu().numpy(), pool.cpu().numpy()
    bi = so.key_blocks(keys)[0]
    parts = []
    for group, shift in ((base, 0), (far, gap)):
        o = (origin[0] + shift * s, origin[1], origin[2])
        sub = _dev(group)
        dgrid, ddata = _dense(sub, o, s, (112, 112, 128), TRUNC, MAXD)
        # the blocks of this cluster against the dense grid at its own origin
        sel = (bi >= shift // 8 - 16) & (bi < shift // 8 + 16)
        d = _planes(ddata, 112 * 112 * 128)
        v = np.arange(512)
        b = so.key_blocks(keys[sel])
        i = b[0][:, None] * 8 + (v & 7) - shift
        j = b[1][:, None] * 8 + ((v >> 3) & 7)
        k = b[2][:, None] * 8 + (v >> 6)
        assert i.min() >= 0 and i.max() < 112 and j.min() >= 0 and j.max() < 112 and k.min() >= 0 and k.max() < 128
        L = (i + 112 * (j + 112 * k)).ravel()
        for c in range(5):
            plane = (d["tsdf"], d["weight"], d["col"][0], d["col"][1], d["col"][2])[c]
            assert np.array_equal(_bits(pool[sel][:, c].ravel()), _bits(plane[L]))
        parts.append(_gpu_extract(dgrid))
    xyz, faces = xyz.cpu().numpy(), faces.cpu().numpy()
    V0, V1 = parts[0][0].shape[0], parts[1][0].shape[0]
    assert xyz.shape[0] == V0 + V1 and faces.shape[0] == parts[0][2].shape[0] + parts[1][2].shape[0]
    union = np.concatenate([parts[0][0], parts[1][0]]).astype(np.float64)
    dist, idx = cKDTree(union).query(xyz.astype(np.float64))
    assert dist.max() <= s * 2.0 ** -8, dist.max()
    assert np.array_equal(np.sort(idx), np.arange(V0 + V1))           # a one-to-one match
    dense_faces = np.concatenate([parts[0][2], parts[1][2] + V0])
    mapped = idx[faces]
    as_sets = lambda f: sorted(map(tuple, f.tolist()))
    assert as_sets(mapped) == as_sets(dense_faces)


def test_repeatable():
    from gaussian_lic_b200 import ops
    dv = _dev(_views(np.random.default_rng(7)))
    a = _sparse(dv, ORIGIN, S, TRUNC, MAXD)
    b = _sparse(dv, ORIGIN, S, TRUNC, MAXD)
    for x, y in zip(ops.sparse_tsdf_planes(a[0], DEV), ops.sparse_tsdf_planes(b[0], DEV)):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))
    ma, mb = ops.sparse_mesh_extract(a[0], DEV), ops.sparse_mesh_extract(b[0], DEV)
    for x, y in zip(ma[:3], mb[:3]):
        assert torch.equal(x, y)


def test_rejected_arguments_enqueue_nothing():
    from gaussian_lic_b200 import capi, ops
    lib = capi.lib
    dv = _dev(_views(np.random.default_rng(1)))
    grid, data, n, clipped, keep = _sparse(dv, ORIGIN, S, TRUNC, MAXD)
    st, sdata = ops.block_set(64, DEV)
    view, depth = dv[0][0], dv[0][1]
    o = (C.c_float * 3)(*ORIGIN)
    cnt = (C.c_int64 * 3)()
    need = lib.glic_sparse_mesh_scratch_bytes(grid.n_blocks)
    scratch = torch.empty(need, dtype=torch.uint8, device=DEV)
    mc = capi.SparseMeshCounts()
    out = torch.empty(64, dtype=torch.int32, device=DEV)
    torch.cuda.synchronize()

    def ins(set_=st, **kw):
        a = dict(o=o, s=S, view=capi.ptr(view), W=W0, H=H0, fx=F0, depth=capi.ptr(depth), trunc=TRUNC, max_depth=0.0, cnt=cnt)
        a.update(kw)
        return lib.glic_block_set_insert(C.byref(set_) if set_ is not None else None, a["o"], a["s"], a["view"], a["W"], a["H"], a["fx"],
                                         a["fx"], 48.0, 36.0, a["depth"], None, 0, a["trunc"], a["max_depth"], a["cnt"], None)
    bad_set = capi.BlockSet(0, sdata.data_ptr())
    big_set = capi.BlockSet(1 << 25, sdata.data_ptr())
    bad_grid = capi.SparseTsdf()
    bad_grid.origin[:], bad_grid.voxel_size, bad_grid.n_blocks, bad_grid.data = list(grid.origin), 0.0, grid.n_blocks, grid.data
    launches = capi.launch_count()
    cases = [ins(None), ins(bad_set), ins(big_set), ins(o=None), ins(cnt=None), ins(s=0.0), ins(s=float("nan")), ins(view=None),
             ins(depth=None), ins(W=0), ins(fx=0.0), ins(trunc=0.0), ins(max_depth=-1.0),
             lib.glic_block_set_clear(C.byref(bad_set), None), lib.glic_block_set_copy(C.byref(st), C.byref(st), None),
             lib.glic_block_set_copy(C.byref(st), C.byref(capi.BlockSet(100, sdata.data_ptr())), None),
             lib.glic_sparse_tsdf_init(C.byref(bad_grid), C.byref(st), None), lib.glic_sparse_tsdf_init(C.byref(grid), C.byref(bad_set), None),
             lib.glic_sparse_tsdf_integrate(C.byref(bad_grid), capi.ptr(view), W0, H0, F0, F0, 48.0, 36.0, capi.ptr(depth), None, None, 0, TRUNC, 0.0, None),
             lib.glic_sparse_tsdf_integrate(C.byref(grid), capi.ptr(view), W0, H0, F0, F0, 48.0, 36.0, capi.ptr(depth), None, None, 0, -1.0, 0.0, None),
             lib.glic_sparse_mesh_count(C.byref(grid), None, need, C.byref(mc), None),
             lib.glic_sparse_mesh_count(C.byref(grid), capi.ptr(scratch), need, None, None),
             lib.glic_sparse_mesh_extract(C.byref(grid), capi.ptr(scratch), need, None, capi.ptr(out), 1 << 20, capi.ptr(out), capi.ptr(out),
                                          capi.ptr(out), None)]
    assert cases == [-1] * len(cases), cases
    assert lib.glic_sparse_mesh_count(C.byref(grid), capi.ptr(scratch), need - 1, C.byref(mc), None) == -2
    assert capi.launch_count() == launches
    torch.cuda.synchronize()


# ---- the mapper ----------------------------------------------------------------------------------------------------------------
def test_mapper_sparse_mesh_equals_extract_mesh(tmp_path):
    from test_gpu_align import _same, _snapshot
    m, poses = _masked_trained()
    before = _snapshot(m, 3)
    s = MESH["voxel_size"]
    lo = m.extract_mesh_sparse(origin=MESH["origin"], voxel_size=s, trunc=MESH["trunc"])["lattice_lo"]
    # an origin 8 voxels before the lowest block, so that a dense grid from it holds every block
    origin = tuple(float(np.float32(o) + np.float32(s) * np.float32(l - 8)) for o, l in zip(MESH["origin"], lo))
    p = dict(origin=origin, voxel_size=s, trunc=MESH["trunc"])
    for views, extra in ((None, {}), ([2, 0], dict(max_depth=9.0))):
        c = m.extract_mesh_sparse(views=views, **p, **extra)
        sparse = m.mesh()
        assert c["clipped_pixels"] == 0 and c["vertices"] > 100 and min(c["lattice_lo"]) >= 0, c
        dims = tuple(h + 1 for h in c["lattice_hi"])
        dense = m.extract_mesh(views=views, dims=dims, **p, **extra)
        for k in ("vertices", "colors", "faces"):
            assert np.array_equal(sparse[k].view(np.uint8), dense[k].view(np.uint8)), (views, k)
        assert c["observed_voxels"] <= dense["observed_voxels"]
    _same(before, _snapshot(m, 3))
    m.extract_mesh_sparse(**p)
    path = tmp_path / "sparse.ply"
    m.save_mesh(path)
    got = m.mesh()
    assert path.read_bytes().startswith(b"ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % got["n_vertices"])
    m.close()


def test_mapper_sparse_binning_overflow_and_max_blocks():
    from gaussian_lic_b200 import capi
    m, poses = _masked_trained()
    p = dict(origin=MESH["origin"], voxel_size=MESH["voxel_size"], trunc=MESH["trunc"])
    c = m.extract_mesh_sparse(**p)
    want = m.mesh()
    m.set_binning_pairs(1000)
    regrows = m.stats().overflow_regrows
    m.extract_mesh_sparse(**p)
    assert m.stats().overflow_regrows > regrows
    got = m.mesh()
    for k in ("vertices", "colors", "faces"):
        assert np.array_equal(got[k], want[k])
    assert m.extract_mesh_sparse(max_blocks=c["blocks"], **p)["blocks"] == c["blocks"]
    with pytest.raises(capi.GlicError, match=r"\(-2\)"):
        m.extract_mesh_sparse(max_blocks=c["blocks"] - 1, **p)
    got = m.mesh()
    for k in ("vertices", "colors", "faces"):
        assert np.array_equal(got[k], want[k])
    m.close()


def test_mapper_sparse_allocation_failures_change_nothing():
    from gaussian_lic_b200 import capi
    from test_gpu_align import _same, _snapshot
    m, poses = _masked_trained()
    first = m.extract_mesh(views=[0], **MESH)
    p = dict(origin=MESH["origin"], voxel_size=0.07, trunc=MESH["trunc"])
    failures = 0
    for k in range(1, 20):
        m.set_binning_pairs(5000)
        before = _snapshot(m, 3)
        assert capi.lib.glic_debug_fail_allocation(k) == 0
        try:
            m.extract_mesh_sparse(**p)
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
        cur = m.mesh()
        for key in ("vertices", "colors", "faces"):
            assert np.array_equal(cur[key], first[key]), k
    else:
        raise AssertionError("extract_mesh_sparse never succeeded")
    assert failures >= 5
    m.close()


def test_mapper_sparse_rejected_arguments():
    from gaussian_lic_b200 import capi
    m, poses = _masked_trained()
    p = dict(origin=MESH["origin"], voxel_size=MESH["voxel_size"], trunc=MESH["trunc"])
    launches = capi.launch_count()
    for kw in (dict(voxel_size=0.0), dict(trunc=float("inf")), dict(max_depth=-1.0), dict(views=[3]), dict(origin=(float("nan"), 0, 0))):
        with pytest.raises(capi.GlicError, match=r"\(-1\)"):
            m.extract_mesh_sparse(**dict(p, **kw))
    assert capi.launch_count() == launches
    m.close()
