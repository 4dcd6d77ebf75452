"""initialize() on the GPU (csrc/initialize.cu, glic_mapper_initialize_lidar; gaussian.cpp:212-304) and the sky-less map
export (saveMap, gaussian.cpp:305-397).

Checkers: the CPU restatement of initialize() (initialize_oracle.py: LiDAR rows bit for bit, the sky generator's uniforms
bit for bit), the reference's own torch expression for the sky positions evaluated on the GPU from the same uniforms,
torch + distCUDA2 for the sky scales (and the reference's distCUDA2 when the reference build exists),
glic_mapper_initialize fed the restatement's rows, and the reference's own PLY writer for the saved map (oracle/_ref/ply_ref
on the sliced rows, oracle/_ref/ply_ref_sky with saveMap's own row counts on all of them).
"""
import ctypes as C
import importlib.util
import os
import subprocess

import numpy as np
import pytest

import initialize_oracle as io

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, H, F = 320, 208, 250.0
FX, FY = 431.795259219, 431.550090267                     # config/fastlivo.yaml:3-4
FOCAL = (FX + FY) / 2
RADIUS = 1000                                             # config/fastlivo.yaml:28
KEYS = ("means", "dc", "sh", "opacity_logits", "log_scales", "rots")


def _scan(n, seed, R_wc=None, t_wc=None):
    """n LiDAR points in front of a camera (world frame), 8-bit colours as the Dataset's doubles, depths 0.1 .. 200 m."""
    rng = np.random.default_rng(seed)
    z = rng.uniform(0.5, 15.0, n)
    pts = np.stack([z * rng.uniform(-0.6, 0.6, n), z * rng.uniform(-0.4, 0.4, n), z], 1)
    if R_wc is not None:
        pts = pts @ np.asarray(R_wc, np.float64).T + np.asarray(t_wc, np.float64)
    cols = rng.integers(0, 256, (n, 3)) / 255.0
    dep = np.exp(rng.uniform(np.log(0.1), np.log(200.0), n)).astype(np.float32)
    return pts.astype(np.float32), cols, dep


def _mapper(capacity=0, seed=0, **kw):
    from gaussian_lic_b200 import mapper
    return mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=3, capacity=capacity, seed=seed, **kw)


def _bits(a):
    a = a.detach().cpu().numpy() if hasattr(a, "detach") else np.asarray(a)
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same(a, b, what):
    assert np.array_equal(_bits(a), _bits(b)), what


@pytest.mark.parametrize("n,scaling_scale", [(1, 1.0), (1000, 2.0), (200_000, 1.0)])
def test_lidar_kernel_matches_oracle(n, scaling_scale):
    from gaussian_lic_b200 import ops
    pts, cols, dep = _scan(n, 100 + n)
    if n >= 256:
        cols[:256] = np.arange(256)[:, None] / 255.0                  # every 8-bit value in every channel
    dev = "cuda:0"
    d = ops.lidar_init(torch.as_tensor(pts, device=dev), torch.as_tensor(cols, device=dev), torch.as_tensor(dep, device=dev),
                       scaling_scale, FOCAL)
    torch.cuda.synchronize()
    o = io.lidar_init(pts, cols, dep, scaling_scale, FOCAL)
    for k in ("xyz", "f_dc", "log_scale", "rot", "opacity_logit"):
        _same(d[k], o[k], k)


def _torch_sky_xyz(uv, radius):
    """gaussian.cpp:247-253, op for op, on the GPU from the given uniforms (torch.rand's draws replaced by uv)."""
    u = torch.as_tensor(uv, device="cuda:0")
    r1, r2 = u[:, 0].contiguous(), u[:, 1].contiguous()
    pi = torch.acos(torch.tensor(-1.0, dtype=torch.float32, device="cuda:0"))
    theta = 2.0 * pi * r1
    phi = torch.acos(1.0 - 1.4 * r2)
    xyz = torch.zeros(u.shape[0], 3, dtype=torch.float32, device="cuda:0")
    radius = float(radius)                                            # double radius = skybox_radius_
    xyz[:, 0] = radius * 10 * torch.cos(theta) * torch.sin(phi)
    xyz[:, 1] = radius * 10 * torch.sin(theta) * torch.sin(phi)
    xyz[:, 2] = radius * 10 * torch.cos(phi)
    return xyz


def _reference_ext():
    so = os.path.join(ROOT, "oracle", "_ref", "glic_ref_ext.so")
    if not os.path.isfile(so):
        return None
    spec = importlib.util.spec_from_file_location("glic_ref_ext", so)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


@pytest.mark.parametrize("S", [1, 3, 4, 100_000])
def test_sky_kernel(S):
    from gaussian_lic_b200 import ops
    d = ops.skybox_init(S, RADIUS, 42, uniforms=True)
    torch.cuda.synchronize()
    uv = io.sky_uniforms(S, 42)
    _same(d["uv"], uv, "uniforms")
    _same(d["xyz"], _torch_sky_xyz(uv, RADIUS), "positions")
    want = torch.log(torch.sqrt(torch.clamp_min(ops.distCUDA2(d["xyz"]), 1e-7)))
    _same(d["log_scale"], want[:, None].repeat(1, 3), "log-scales")
    _same(d["f_dc"], np.tile(np.array([0.7, 0.8, 0.95], np.float32), (S, 1)), "f_dc")
    _same(d["rot"], np.tile(np.array([1, 0, 0, 0], np.float32), (S, 1)), "rot")
    _same(d["opacity_logit"], np.full(S, io.logit32(0.7), np.float32), "opacity logit")
    r = torch.linalg.norm(d["xyz"].double(), dim=1)
    assert float((r / (10.0 * RADIUS) - 1).abs().max()) < 1e-6
    ref = _reference_ext()
    if ref is not None and S >= 4:                                    # every point has three neighbours: finite distances
        ref_ls = torch.log(torch.sqrt(torch.clamp_min(ref.distCUDA2(d["xyz"].clone()), 1e-7)))
        assert float((ref_ls - d["log_scale"][:, 0]).abs().max()) <= 2e-6


def _oracle_rows(pts, cols, dep, S, seed, scaling_scale=1.0):
    """(sky rows from the GPU sky kernel, LiDAR rows from the oracle) as download() dicts"""
    from gaussian_lic_b200 import ops
    lid = io.lidar_init(pts, cols, dep, scaling_scale, FOCAL)
    rows = dict(means=lid["xyz"], dc=lid["f_dc"], opacity_logits=lid["opacity_logit"], log_scales=lid["log_scale"], rots=lid["rot"])
    if S:
        sky = {k: v.cpu().numpy() for k, v in ops.skybox_init(S, RADIUS, seed).items()}
        rows = dict(means=np.concatenate([sky["xyz"], rows["means"]]), dc=np.concatenate([sky["f_dc"], rows["dc"]]),
                    opacity_logits=np.concatenate([sky["opacity_logit"], rows["opacity_logits"]]),
                    log_scales=np.concatenate([sky["log_scale"], rows["log_scales"]]), rots=np.concatenate([sky["rot"], rows["rots"]]))
    return rows


def test_mapper_layout_and_growth():
    """sky rows [0, S), then the LiDAR rows in input order; zero SH rest and moments; the arena grows past cfg.capacity"""
    n, S = 5000, 3000
    pts, cols, dep = _scan(n, 1)
    m = _mapper(capacity=4096, seed=11)
    m.initialize_lidar(pts, cols, dep, FOCAL, S, RADIUS)
    st = m.stats()
    assert st.num_gaussians == S + n and st.capacity >= S + n and st.capacity > 4096
    assert m.sky_rows() == S
    dl = m.download(moments=True)
    want = _oracle_rows(pts, cols, dep, S, 11)
    for k in want:
        _same(dl[k], want[k], k)
    assert np.all(dl["sh"] == 0) and np.all(dl["exp_avg"] == 0) and np.all(dl["exp_avg_sq"] == 0)
    m.close()


def test_mapper_without_sky_equals_initialize():
    """sky_points = 0: the arena is glic_mapper_initialize's on the oracle's rows, and the view sampler is untouched"""
    n = 4000
    pts, cols, dep = _scan(n, 2)
    a, b, c = _mapper(seed=5), _mapper(seed=5), _mapper(seed=5)
    a.initialize_lidar(pts, cols, dep, FOCAL, 0, 0)
    o = _oracle_rows(pts, cols, dep, 0, 5)
    b.initialize(dict(o, sh=np.zeros((n, 15, 3), np.float32)))
    c.initialize_lidar(pts, cols, dep, FOCAL, 2000, RADIUS)               # a sky does not advance the sampler either
    assert a.sky_rows() == 0 and b.sky_rows() == 0 and c.sky_rows() == 2000
    da, db = a.download(moments=True), b.download(moments=True)
    for k in da:
        _same(da[k], db[k], k)
    img = np.full((3, H, W), 0.5, np.float32)
    from gaussian_lic_b200 import synthetic as syn
    R, t = syn.orbit_pose(0, radius=2.0)
    for m in (a, b, c):
        for _ in range(150):
            m.add_keyframe(R, t, img)
    for _ in range(3):
        va, vb, vc = a.sample_views(), b.sample_views(), c.sample_views()
        assert va == vb == vc and len(va) == 100
    for m in (a, b, c):
        m.close()


def test_determinism_and_seeds():
    n, S = 2000, 5000
    pts, cols, dep = _scan(n, 3)
    out = []
    for seed in (7, 7, 8):
        m = _mapper(seed=seed)
        m.initialize_lidar(pts, cols, dep, FOCAL, S, RADIUS)
        out.append(m.download())
        m.close()
    for k in KEYS:
        _same(out[0][k], out[1][k], k)
        _same(out[0][k][S:], out[2][k][S:], k)                          # the LiDAR rows do not depend on the seed
    assert np.mean(np.any(out[0]["means"][:S] != out[2]["means"][:S], axis=1)) > 0.99


def test_two_ranks_draw_the_same_sky():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    n, S = 2000, 5000
    pts, cols, dep = _scan(n, 4)
    dl = []
    for rank in range(2):
        with torch.cuda.device(rank):
            m = _mapper(seed=21, rank=rank, world=2)
            m.initialize_lidar(pts, cols, dep, FOCAL, S, RADIUS)
            dl.append(m.download(moments=True))
            m.close()
    for k in dl[0]:
        _same(dl[0][k], dl[1][k], k)


def _blob(path, d, rows):
    P, M = len(rows), d["sh"].shape[1]
    parts = [np.array([P, M], np.uint32).tobytes()] + [np.ascontiguousarray(d[k][rows], np.float32).tobytes()
                                                       for k in ("means", "dc", "sh", "opacity_logits", "log_scales", "rots")]
    with open(path, "wb") as f:
        f.write(b"".join(parts))


def _ply_write(path, d, rows):
    from gaussian_lic_b200 import capi
    a = {k: np.ascontiguousarray(d[k][rows], np.float32) for k in KEYS}
    p = lambda x: x.ctypes.data_as(C.c_void_p) if x.size else None
    capi.check(capi.lib.glic_ply_write(str(path).encode(), len(rows), a["sh"].shape[1], p(a["means"]), p(a["dc"]), p(a["sh"]),
                                       p(a["opacity_logits"]), p(a["log_scales"]), p(a["rots"])), "ply_write")


def test_end_to_end_with_sky(tmp_path):
    """initialize_lidar (sky + first scan) -> add_keyframe -> extend -> optimize -> save_map without the sky rows"""
    from gaussian_lic_b200 import synthetic as syn
    n, S = 6000, 4000
    poses = [syn.orbit_pose(v, radius=2.0) for v in (0, 1)]
    gts = [syn.make_gt_image(W, H, seed=3 + i) for i in range(2)]
    pts, cols, dep = _scan(n, 5, *poses[0])
    m = _mapper(seed=3, max_iters=8)
    m.initialize_lidar(pts, cols, dep, FOCAL, S, RADIUS)
    m.add_keyframe(*poses[0], gts[0])
    st = m.optimize([0, 0])
    assert np.isfinite(st.last_loss)
    m.add_keyframe(*poses[1], gts[1])
    p2, c2, d2 = _scan(8000, 6, *poses[1])
    inserted = m.extend(p2, c2.astype(np.float32), d2)
    for _ in range(2):
        st = m.optimize()
    assert np.isfinite(st.last_loss) and st.num_gaussians == S + n + inserted and inserted > 0
    assert m.sky_rows() == S
    dl = m.download()
    r = np.linalg.norm(dl["means"].astype(np.float64), axis=1)
    assert np.all(np.abs(r[:S] / (10.0 * RADIUS) - 1) < 1e-3) and np.all(r[S:] < 100.0)   # the sky kept its rows
    P = st.num_gaussians
    m.save_map(tmp_path / "mine.ply")
    mine = (tmp_path / "mine.ply").read_bytes()
    _ply_write(tmp_path / "fg.ply", dl, np.arange(S, P))
    assert mine == (tmp_path / "fg.ply").read_bytes()
    ply_ref = os.path.join(ROOT, "oracle", "_ref", "ply_ref")
    if os.path.isfile(ply_ref):                                       # the reference's own tinyply on rows [S, P)
        _blob(tmp_path / "fg.blob", dl, np.arange(S, P))
        subprocess.check_call([ply_ref, str(tmp_path / "fg.blob"), str(tmp_path / "ref_fg.ply")])
        assert mine == (tmp_path / "ref_fg.ply").read_bytes()
    ply_ref_sky = os.path.join(ROOT, "oracle", "_ref", "ply_ref_sky")
    if os.path.isfile(ply_ref_sky):                                   # ... driven like saveMap, with its unsliced f_dc / f_rest counts
        _blob(tmp_path / "all.blob", dl, np.arange(P))
        subprocess.check_call([ply_ref_sky, str(tmp_path / "all.blob"), str(tmp_path / "ref_sky.ply"), str(S)])
        assert mine == (tmp_path / "ref_sky.ply").read_bytes()
    m.close()
    # a map without a sky still saves every row
    m = _mapper(seed=3)
    m.initialize_lidar(pts, cols, dep, FOCAL, 0, 0)
    m.save_map(tmp_path / "nosky.ply")
    dl = m.download()
    _ply_write(tmp_path / "all.ply", dl, np.arange(n))
    assert (tmp_path / "nosky.ply").read_bytes() == (tmp_path / "all.ply").read_bytes()
    m.close()


def test_rejected_arguments_leave_the_model_untouched():
    from gaussian_lic_b200 import capi
    n, S = 1000, 500
    pts, cols, dep = _scan(n, 7)
    m = _mapper(seed=9)
    m.initialize_lidar(pts, cols, dep, FOCAL, S, RADIUS)
    before, st0 = m.download(moments=True), m.stats()
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    col = np.ascontiguousarray(cols, np.float64)
    lib = capi.lib
    calls = [(0, vp(pts), vp(col), vp(dep), 100, RADIUS),                 # n < 1
             (-3, vp(pts), vp(col), vp(dep), 100, RADIUS),
             (n, vp(pts), vp(col), vp(dep), -1, RADIUS),                  # sky_points < 0
             (n, vp(pts), vp(col), vp(dep), 100, 0),                      # sky_radius <= 0 with a sky
             (n, vp(pts), vp(col), vp(dep), 100, -5),
             (n, None, vp(col), vp(dep), 100, RADIUS),                    # null pointers
             (n, vp(pts), None, vp(dep), 100, RADIUS),
             (n, vp(pts), vp(col), None, 100, RADIUS)]
    for args in calls:
        nn, p, c, d, sp, sr = args
        assert lib.glic_mapper_initialize_lidar(m._h, nn, p, c, d, FOCAL, sp, sr) == -1, args
        after = m.download(moments=True)
        for k in before:
            _same(after[k], before[k], k)
        assert m.sky_rows() == S and m.stats().num_gaussians == st0.num_gaussians and m.stats().capacity == st0.capacity
    assert lib.glic_mapper_initialize_lidar(None, n, vp(pts), vp(col), vp(dep), FOCAL, 0, 0) == -1
    m.close()
