"""Rendering from any camera on the GPU: glic_render (the inference form of the forward) against glic_forward bit for bit, its
expected and median depth against a float64 restatement on the GPU's own sorted lists, known answers, and
glic_mapper_render_camera: the glic_mapper_render equalities, the sky, other frame sizes, the frozen map (one mapper, its twin,
two ranks), the binning overflow and allocation failures."""
import os
import socket

import numpy as np
import pytest

from helpers import small_scene
from render_camera_oracle import depth_planes
from test_gpu_align import _same, _snapshot, _trained
from test_gpu_mapper_grads import F, GROUPS, H, W, _keyframes, _mapper, _scene, _state

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GOLDEN = ["scene_deg0", "scene_deg1", "scene_deg3", "scene_rot_deg2", "scene_rot_deg3"]


def _bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def _golden_scene(name):
    z = np.load(os.path.join(GOLD, name + ".npz"))
    P, W_, H_, seed, deg = (int(z[k]) for k in ("P", "W", "H", "seed", "degree"))
    view = int(z["view"]) if "view" in z.files else 0
    pp = tuple(float(x) for x in z["pp"]) if "pp" in z.files else (0.0, 0.0)
    return small_scene(P, W_, H_, seed, deg, view=view, pp=pp)


SCENES = GOLDEN + ["small_scene_pp"]


def _scene_of(name):
    if name == "small_scene_pp":
        return small_scene(3000, 320, 208, 11, 3, view=3, pp=(17.5, -9.25))
    return _golden_scene(name)


def _forward_and_render(g, cam):
    from gaussian_lic_b200 import ops
    dev = torch.device("cuda:0")
    r = ops.CRasterizer(cam["W"], cam["H"], dev)
    gd = ops.scene_to_device(g, dev)
    view = r.make_view(cam)
    color, T, radii = r.forward(gd, view)
    fwd = dict(color=color.cpu().numpy(), final_T=T.cpu().numpy(), radii=radii.cpu().numpy(), R=r.R, state=r.debug_state())
    ren = r.render(gd, view)
    ren = {k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in ren.items()}
    return fwd, ren


# ---- 2. glic_render against glic_forward ------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SCENES)
def test_render_equals_forward(name):
    g, cam = _scene_of(name)
    fwd, ren = _forward_and_render(g, cam)
    assert ren["counters"] == (fwd["R"], 0, 0)
    assert np.array_equal(ren["radii"], fwd["radii"])
    assert np.array_equal(_bits(ren["color"]), _bits(fwd["color"]))
    assert np.array_equal(_bits(ren["final_T"]), _bits(fwd["final_T"]))
    assert (fwd["final_T"] < 1.0).mean() > 0.3                        # the scene covers the frame


# ---- 3. depth against the float64 restatement -------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SCENES)
def test_depth_matches_restatement(name):
    g, cam = _scene_of(name)
    fwd, ren = _forward_and_render(g, cam)
    st = fwd["state"]
    R = st["R"]
    T64, D64, med64, flag = depth_planes(cam["W"], cam["H"], st["xy"].cpu().numpy(), st["conic_opacity"].cpu().numpy(),
                                         st["depth"].cpu().numpy(), st["point_list"].cpu().numpy()[:R].view(np.uint32),
                                         st["ranges"].cpu().numpy().view(np.uint32))
    ok = ~flag
    print("%s: %d of %d pixels excluded (a decision within rounding of a threshold)" % (name, flag.sum(), flag.size))
    assert flag.mean() < 0.01
    assert np.abs(ren["final_T"][ok] - T64[ok]).max() <= 1e-4
    # expected depth: float32 FMAs against float64, relative to the depth a pixel has gathered (z up to ~25)
    D = ren["depth"].astype(np.float64)
    err = np.abs(D - D64)[ok]
    print("%s: expected depth max abs err %.3g (max depth %.3g)" % (name, err.max(), D64.max()))
    assert (err <= 1e-4 * D64[ok] + 1e-6).all()
    # median depth: the chosen splat's float32 depth exactly
    assert np.array_equal(_bits(ren["median_depth"][ok]), _bits(med64[ok].astype(np.float32)))
    assert (med64[ok] > 0).mean() > 0.1


# ---- 4. known answers ---------------------------------------------------------------------------------------------------------
def test_single_opaque_gaussian():
    from gaussian_lic_b200 import ops, synthetic as syn
    W_, H_, f, z = 64, 64, 64.0, 5.0
    cam = syn.make_camera(W_, H_, f, f, 32.0, 32.0)
    g = dict(means=np.array([[0.0, 0.0, z]], np.float32), scales=np.full((1, 3), 0.5, np.float32),
             rots=np.array([[1.0, 0.0, 0.0, 0.0]], np.float32), opacity=np.array([[0.9999]], np.float32),
             dc=np.full((1, 3), 0.5, np.float32), sh=np.zeros((1, 0, 3), np.float32), degree=0)
    dev = torch.device("cuda:0")
    r = ops.CRasterizer(W_, H_, dev)
    out = r.render(ops.scene_to_device(g, dev), r.make_view(cam))
    T, D, med = (out[k].cpu().numpy() for k in ("final_T", "depth", "median_depth"))
    assert out["counters"][0] > 0 and np.float32(T[32, 32]) == np.float32(1.0) - np.float32(0.99)
    seen = (1.0 - T.astype(np.float64)) >= 0.05                       # 1 - T rounds to 3e-8 absolute: 1e-6 relative needs alpha >= 0.03
    ratio = D[seen] / (1.0 - T[seen].astype(np.float64))
    assert seen.sum() > 100 and np.abs(ratio / z - 1.0).max() <= 1e-6
    assert np.array_equal(med[T < 0.5], np.full((T < 0.5).sum(), z, np.float32)) and (T < 0.5).sum() > 20
    assert not med[T >= 0.5].any()
    # pixels no splat reaches: colour 0, depth 0, T 1, median 0
    far = np.zeros((H_, W_), bool)
    far[:4, :4] = far[-4:, -4:] = True
    assert (T[far] == 1.0).all() and not D[far].any() and not med[far].any() and not out["color"].cpu().numpy()[:, far].any()


# ---- 5. the mapper's equalities ---------------------------------------------------------------------------------------------
def _device_rows(m, first=0):
    """the mapper's rows [first, P), downloaded and activated by the library's activation kernel"""
    from gaussian_lic_b200 import model
    d = m.download()
    d = {k: v[first:] for k, v in d.items()}
    d["degree"] = int(m.cfg.sh_degree)
    mdl = model.PackedModel(d, torch.device("cuda:0"))
    mdl.activate()
    torch.cuda.synchronize()
    return mdl


def _glic_render(mdl, W_, H_, fx, fy, cx, cy, R, t):
    from gaussian_lic_b200 import mapper, ops
    r = ops.CRasterizer(W_, H_, torch.device("cuda:0"))
    out = r.render(mdl.inputs, r.make_view(mapper.camera_block(W_, H_, fx, fy, cx, cy, R, t)))
    return {k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in out.items()}


def _same_as_glic_render(got, want, what):
    assert np.array_equal(_bits(got["final_T"]), _bits(want["final_T"])), what
    assert np.array_equal(_bits(got["depth"]), _bits(want["depth"])), what
    assert np.array_equal(_bits(got["median_depth"]), _bits(want["median_depth"])), what
    assert np.array_equal(_bits(got["rgb"]), _bits(np.clip(want["color"], 0.0, 1.0))), what


def test_render_camera_equals_render_at_keyframes():
    raw = _scene(3)
    poses, cams, gts = _keyframes(seed=45)
    m = _trained(raw, poses, gts)
    for k in range(3):
        R, t = m.pose(k)
        assert not np.array_equal(R, np.asarray(poses[k][0], np.float32))          # refined
        out = m.render_camera(R, t, exposure=k)
        assert np.array_equal(_bits(out["rgb"]), _bits(m.render(k, True))), k
        # the identity exposure is the raw colour, clamped; the other planes do not depend on it
        plain = m.render_camera(R, t)
        assert not np.array_equal(plain["rgb"], out["rgb"])
        for key in ("final_T", "depth", "median_depth"):
            assert np.array_equal(_bits(plain[key]), _bits(out[key])), (k, key)
    out = m.render_camera(*poses[1])
    assert np.array_equal(_bits(out["rgb"]), _bits(m.render(0, False)))
    # final_T and the depth planes are glic_render's on the activated rows
    mdl = _device_rows(m)
    R, t = m.pose(2)
    _same_as_glic_render(m.render_camera(R, t), _glic_render(mdl, W, H, F, F, W / 2.0, H / 2.0, R, t), "keyframe 2")
    m.close()


def _sky_mapper():
    from test_gpu_densify import _lidar_scan
    from gaussian_lic_b200 import mapper, synthetic as syn
    pts, cols, dep = _lidar_scan(3000, 5, *syn.orbit_pose(0, radius=2.0))
    m = mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=3)
    m.initialize_lidar(pts, cols, dep, F, 500, 1000)
    poses, cams, gts = _keyframes(seed=47)
    for (R, t), img in zip(poses, gts):
        m.add_keyframe(R, t, img)
    m.optimize([0, 1, 2])
    return m, poses


def test_sky_rows_in_and_out():
    m, poses = _sky_mapper()
    S = m.sky_rows()
    assert S == 500
    R, t = poses[1]
    with_sky, without = m.render_camera(R, t, sky=True), m.render_camera(R, t, sky=False)
    _same_as_glic_render(with_sky, _glic_render(_device_rows(m), W, H, F, F, W / 2.0, H / 2.0, R, t), "all rows")
    _same_as_glic_render(without, _glic_render(_device_rows(m, S), W, H, F, F, W / 2.0, H / 2.0, R, t), "rows [S, P)")
    assert (without["final_T"] >= with_sky["final_T"]).all() and (without["final_T"] > with_sky["final_T"]).any()
    m.close()


# ---- 6. other frames ----------------------------------------------------------------------------------------------------------
def test_other_frames():
    from gaussian_lic_b200 import capi
    raw = _scene(1)
    poses, cams, gts = _keyframes(seed=49)
    m = _mapper(raw, poses, gts)
    m.optimize([0, 1])
    mdl = _device_rows(m)
    R, t = poses[2]
    frames = [dict(width=1, height=1, cx=0.5, cy=0.5), dict(width=17, height=9, cx=8.0, cy=4.0),
              dict(width=2 * W, height=2 * H, fx=2 * F, fy=2 * F, cx=float(W), cy=float(H)),
              dict(cx=W / 2.0 + 23.5, cy=H / 2.0 - 11.25), dict(width=1000, height=600, fx=600.0, fy=650.0, cx=480.0, cy=310.0)]
    for fr in frames:
        Wf, Hf = fr.get("width", W), fr.get("height", H)
        k = dict(fx=fr.get("fx", F), fy=fr.get("fy", F), cx=fr["cx"], cy=fr["cy"])
        out = m.render_camera(R, t, width=Wf, height=Hf, **k)
        assert out["rgb"].shape == (3, Hf, Wf)
        _same_as_glic_render(out, _glic_render(mdl, Wf, Hf, k["fx"], k["fy"], k["cx"], k["cy"], R, t), str(fr))
    # a frame of exactly GLIC_MAX_TILES tiles renders; one tile more is refused before any launch
    big = m.render_camera(R, t, width=4096, height=4096, fx=3200.0, fy=3200.0, cx=2048.0, cy=2048.0, outputs=("final_T", "depth"))
    T = big["final_T"]
    assert T.shape == (4096, 4096) and (T >= 0).all() and (T <= 1).all() and (T < 1).mean() > 0.3 and np.isfinite(big["depth"]).all()
    launches = capi.launch_count()
    with pytest.raises(capi.GlicError, match="GLIC_MAX_TILES"):
        m.render_camera(R, t, width=4096, height=4097)
    assert capi.launch_count() == launches
    m.close()


# ---- 7. the frozen map ----------------------------------------------------------------------------------------------------------
def _render_some(m, poses):
    R, t = m.pose(1)
    m.render_camera(R, t, exposure=1)
    m.render_camera(*poses[1], width=2 * W, height=2 * H, fx=2 * F, fy=2 * F, cx=float(W), cy=float(H), sky=False)
    m.render_camera(*poses[0], width=33, height=17, cx=16.0, cy=8.0, outputs=("depth",))


def test_render_camera_leaves_the_mapper_unchanged():
    raw = _scene(3)
    poses, cams, gts = _keyframes(seed=51)
    m, twin = _trained(raw, poses, gts), _trained(raw, poses, gts)
    before = _snapshot(m, 3)
    _render_some(m, poses)
    _same(before, _snapshot(m, 3))
    assert m.sample_views() == twin.sample_views()
    m.optimize()                                                       # the sampler draws the same views for both
    twin.optimize()
    assert m.stats().iterations == twin.stats().iterations
    assert m.sample_views() == twin.sample_views()
    m.close()
    twin.close()


BATCHES_2R = [1, 2, 0, 1, 2, 2]


def _render_rank_worker(rank, world, port, q):
    try:
        import torch.distributed as dist
        from test_gpu_mapper_grads import P
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
        torch.cuda.set_device(rank % torch.cuda.device_count())
        raw = _scene(3)
        poses, cams, gts = _keyframes(seed=33)
        m = _mapper(raw, poses, gts, capacity=P, rank=rank, world=world, views_per_rank=1)
        got = [None] * world
        dist.all_gather_object(got, m.export_handle())
        m.connect(got)
        m.enable_pose_refinement(1e-3, 1e-3)
        m.enable_exposure(1e-3)
        shapes = []
        for i in range(3):
            m.optimize(BATCHES_2R[2 * i:2 * i + 2])
            if rank == 0:
                R, t = m.pose(i)
                shapes.append(m.render_camera(R, t, exposure=i, width=W + 7 * i, height=H - 5 * i)["rgb"].shape)
        out = dict(state=_state(m), pose=[m.pose(i) for i in range(3)], expo=[m.exposure(i) for i in range(3)], shapes=shapes)
        dist.barrier()
        m.close()
        dist.destroy_process_group()
        q.put((rank, "ok", out))
    except Exception as e:          # noqa: BLE001 - reported to the parent
        import traceback
        q.put((rank, "%r\n%s" % (e, traceback.format_exc()), None))


@pytest.mark.timeout(300)
def test_two_ranks_stay_identical_when_one_renders():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    q = ctx.Queue()
    procs = [ctx.Process(target=_render_rank_worker, args=(r, 2, port, q)) for r in range(2)]
    for p_ in procs:
        p_.start()
    res = sorted([q.get(timeout=240) for _ in procs], key=lambda r: r[0])
    for p_ in procs:
        p_.join(timeout=30)
    assert all(r[1] == "ok" for r in res), [r[1] for r in res]
    a, b = res[0][2], res[1][2]
    assert a["shapes"] == [(3, H - 5 * i, W + 7 * i) for i in range(3)] and b["shapes"] == []
    for key in ("p", "m", "v"):
        for grp in GROUPS:
            assert np.array_equal(_bits(a["state"][key][grp]), _bits(b["state"][key][grp])), "replicas diverged in %s / %s" % (key, grp)
    for k in range(3):
        for x, y in zip(a["pose"][k] + (a["expo"][k],), b["pose"][k] + (b["expo"][k],)):
            assert np.array_equal(_bits(x), _bits(y)), "replicas diverged in keyframe %d" % k


# ---- 8. overflow ----------------------------------------------------------------------------------------------------------------
def test_overflow_regrows_and_redraws():
    raw = _scene(0)
    poses, cams, gts = _keyframes()
    m = _mapper(raw, poses, gts)
    m.set_binning_pairs(1000)
    regrows = m.stats().overflow_regrows
    R, t = poses[1]
    first = m.render_camera(R, t)
    assert m.stats().overflow_regrows == regrows + 1
    again = m.render_camera(R, t)                                      # now with room to spare
    assert m.stats().overflow_regrows == regrows + 1
    for k in first:
        assert np.array_equal(_bits(first[k]), _bits(again[k])), k
    assert (first["final_T"] < 1).mean() > 0.3
    m.close()


def test_training_after_a_render_grows_the_binning():
    """a render that overflows grows the binning workspace alone; training afterwards, whose capacity is then bounded by the
    unchanged sample workspace, must still carve the binning workspace in the backward as its forward did: it trains like a twin
    that never rendered (up to the float atomics of the render backward)"""
    raw = _scene(3)
    poses, cams, gts = _keyframes(seed=61)
    m, twin = _mapper(raw, poses, gts), _mapper(raw, poses, gts)
    mdl = _device_rows(m)
    train_pairs = max(_glic_render(mdl, W, H, F, F, W / 2.0, H / 2.0, R, t)["counters"][0] for R, t in poses)
    big = dict(width=8 * W, height=8 * H, fx=8 * F, fy=8 * F, cx=4.0 * W, cy=4.0 * H)
    big_pairs = _glic_render(mdl, 8 * W, 8 * H, 8 * F, 8 * F, 4.0 * W, 4.0 * H, *poses[1])["counters"][0]
    pairs = 2 * train_pairs                                            # room for every training view, not for the large frame
    print("pairs: training view %d, large frame %d, capacity %d" % (train_pairs, big_pairs, pairs))
    assert big_pairs > 1.5 * pairs
    for x in (m, twin):
        x.set_binning_pairs(pairs)
    regrows = m.stats().overflow_regrows
    m.render_camera(*poses[1], **big)
    assert m.stats().overflow_regrows == regrows + 1
    views = [0, 1, 2, 2, 1, 0]
    m.optimize(views)
    twin.optimize(views)
    assert m.stats().overflow_regrows == regrows + 1 and twin.stats().overflow_regrows == regrows      # training never overflowed
    a, b = _state(m), _state(twin)
    for grp in GROUPS:
        close = np.isclose(a["p"][grp], b["p"][grp], rtol=1e-4, atol=1e-6)
        assert close.mean() > 0.99, (grp, close.mean())
    la, lb = m.stats().last_loss, twin.stats().last_loss
    assert abs(la - lb) <= 1e-4 * abs(lb), (la, lb)
    m.close()
    twin.close()


def test_empty_scene_draws_nothing():
    """glic_render with no Gaussians: T = 1 everywhere (nothing covers a pixel), colour and both depths 0, counters zero"""
    from gaussian_lic_b200 import ops, synthetic as syn
    dev = torch.device("cuda:0")
    z = lambda *shape: np.zeros(shape, np.float32)                     # noqa: E731
    g = dict(means=z(0, 3), scales=z(0, 3), rots=z(0, 4), opacity=z(0, 1), dc=z(0, 3), sh=z(0, 0, 3), degree=0)
    r = ops.CRasterizer(40, 24, dev)
    out = r.render(ops.scene_to_device(g, dev), r.make_view(syn.make_camera(40, 24, 30.0, 30.0, 20.0, 12.0)))
    assert out["counters"] == (0, 0, 0)
    assert (out["final_T"].cpu().numpy() == 1.0).all()
    for k in ("color", "depth", "median_depth"):
        assert not out[k].cpu().numpy().any(), k


# ---- 9. allocation failures -----------------------------------------------------------------------------------------------------
def test_allocation_failures_change_nothing():
    """a first large-frame call on a fresh mapper allocates its render workspace, then regrows the binning workspace (alone:
    the render has no use for the training's sample workspace) for the frame's pairs; failing each allocation in turn leaves the
    snapshot as it was, and the next call succeeds"""
    from gaussian_lic_b200 import capi
    raw = _scene(3)
    poses, cams, gts = _keyframes(seed=53)
    big = dict(width=3 * W, height=3 * H, fx=3 * F, fy=3 * F, cx=1.5 * W, cy=1.5 * H)
    failures = 0
    for k in range(1, 10):
        m = _trained(raw, poses, gts)
        m.set_binning_pairs(5000)
        before = _snapshot(m, 3)
        R, t = m.pose(0)
        want = _glic_render(_device_rows(m), big["width"], big["height"], big["fx"], big["fy"], big["cx"], big["cy"], R, t)
        assert capi.lib.glic_debug_fail_allocation(k) == 0
        try:
            out = m.render_camera(R, t, **big)
            ok = True
        except capi.GlicError as e:
            assert "(-3)" in str(e), (k, str(e))
            ok = False
        finally:
            capi.lib.glic_debug_fail_allocation(0)
        _same(before, _snapshot(m, 3))
        if not ok:
            failures += 1
            out = m.render_camera(R, t, **big)                         # the next call succeeds
        _same_as_glic_render(out, want, "allocation %d" % k)           # float atomics make every trained map its own
        m.close()
        if ok:
            break
    else:
        raise AssertionError("render_camera never succeeded")
    print("render_camera: %d allocations failed in turn" % failures)
    assert failures == 2                                               # the render workspace, then the binning workspace


def test_rejected_arguments_change_nothing():
    import ctypes as C
    from gaussian_lic_b200 import capi, mapper
    raw = _scene(0)
    poses, cams, gts = _keyframes()
    m = _trained(raw, poses, gts)
    before = _snapshot(m, 3)
    R, t = poses[0]
    bad_R = np.asarray(R, np.float32) * 1.01
    refl = np.asarray(R, np.float32) @ np.diag([1.0, 1.0, -1.0]).astype(np.float32)
    nan_t = np.array([0.0, float("nan"), 0.0])
    cases = [dict(width=0), dict(height=0), dict(width=4096, height=4097), dict(fx=0.0), dict(fy=-1.0), dict(fx=float("inf")),
             dict(cx=float("nan")), dict(cy=float("inf")), dict(R_wc=bad_R), dict(R_wc=refl), dict(t_wc=nan_t),
             dict(exposure=3), dict(exposure=-2), dict(outputs=())]
    for kw in cases:
        args = dict(R_wc=R, t_wc=t)
        args.update(kw)
        with pytest.raises(capi.GlicError):
            m.render_camera(**args)
    cam = capi.RenderCamera()
    cam.R_wc[:] = [float(x) for x in np.asarray(R, np.float32).reshape(9)]
    cam.fx, cam.fy, cam.cx, cam.cy, cam.width, cam.height = F, F, W / 2.0, H / 2.0, W, H
    buf = np.zeros((H, W), np.float32)
    for sky in (2, -1):
        assert capi.lib.glic_mapper_render_camera(m._h, C.byref(cam), -1, sky, None, buf.ctypes.data_as(C.c_void_p), None, None) == -1
    assert capi.lib.glic_mapper_render_camera(m._h, None, -1, 1, None, buf.ctypes.data_as(C.c_void_p), None, None) == -1
    assert not buf.any()
    _same(before, _snapshot(m, 3))
    m.close()
    # exposure on a mapper without it; a mapper with no rows
    plain = _mapper(raw, poses, gts)
    with pytest.raises(capi.GlicError, match="exposure"):
        plain.render_camera(R, t, exposure=0)
    plain.close()
    empty = mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=0)
    with pytest.raises(capi.GlicError, match="no rows"):
        empty.render_camera(R, t)
    empty.close()


def test_device_outputs_equal_host_outputs():
    raw = _scene(1)
    poses, cams, gts = _keyframes(seed=55)
    m = _trained(raw, poses, gts)
    import ctypes as C
    from gaussian_lic_b200 import capi
    R, t = m.pose(1)
    host = m.render_camera(R, t, exposure=1)
    cam = capi.RenderCamera()
    cam.R_wc[:] = [float(x) for x in np.asarray(R, np.float32).reshape(9)]
    cam.t_wc[:] = [float(x) for x in np.asarray(t, np.float32).reshape(3)]
    cam.fx, cam.fy, cam.cx, cam.cy, cam.width, cam.height = F, F, W / 2.0, H / 2.0, W, H
    dev = {k: torch.full(v.shape, float("nan"), dtype=torch.float32, device="cuda:0") for k, v in host.items()}
    capi.check(capi.lib.glic_mapper_render_camera(m._h, C.byref(cam), 1, 1, *[capi.ptr(dev[k]) for k in
                                                                               ("rgb", "final_T", "depth", "median_depth")]),
               "mapper_render_camera")
    for k in host:
        assert np.array_equal(_bits(dev[k].cpu().numpy()), _bits(host[k])), k
    m.close()


def test_exposures_of_other_keyframes():
    """exposure_index picks any training keyframe's E: the image of keyframe 0's pose coloured by keyframe 2's E"""
    raw = _scene(0)
    poses, cams, gts = _keyframes(seed=57)
    m = _trained(raw, poses, gts)
    R, t = m.pose(0)
    a, b = m.render_camera(R, t, exposure=2), m.render_camera(R, t, exposure=0)
    assert not np.array_equal(a["rgb"], b["rgb"]) and np.array_equal(_bits(a["final_T"]), _bits(b["final_T"]))
    m.close()
