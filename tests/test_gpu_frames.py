"""Raw frames into the native mapper (glic_mapper_enable_frames / add_frame / keyframe_image / frames_get, csrc/frames.cu's
8-bit decode; Dataset::addFrame, gaussian.cpp:41-111, and mapping.cpp:158-174).

Checkers: the CPU restatement frames_oracle.py (decode, rotation, depths, colours, keyframe selection) and the existing
float-image API fed the restated inputs (initialize_lidar, add_keyframe, extend), which must give the same map, images,
scores, exposure and pose state bit for bit, and after training the same parameters up to the render backward's
atomic-order noise.
"""
import ctypes as C

import numpy as np
import pytest

import frames_oracle as fo

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

W, H = 320, 208
FX, FY = 250.3, 249.7
SKY, RADIUS = 1000, 1000
LR = dict(rots=0.001, means=1.6e-4, log_scales=0.005, opacity_logits=0.05, dc=2.5e-3, sh=2.5e-3 / 20)   # config/fastlivo.yaml:18-22
STAT_FIELDS = ("num_gaussians", "capacity", "iterations", "last_inserted", "last_loss", "mean_visible", "overflow_regrows")


def _mapper(w=W, h=H, **kw):
    from gaussian_lic_b200 import mapper
    return mapper.Mapper(w, h, FX, FY, w / 2.0, h / 2.0, sh_degree=3, seed=17, **kw)


def _focal():
    return (float(np.float32(FX)) + float(np.float32(FY))) / 2


def _padded(bgr, pad=64):
    """the image as rows of 3 W + pad bytes (a row-padded sensor buffer)"""
    h, w, _ = bgr.shape
    buf = np.zeros((h, 3 * w + pad), np.uint8)
    buf[:, :3 * w] = bgr.reshape(h, 3 * w)
    return np.lib.stride_tricks.as_strided(buf, shape=(h, w, 3), strides=(3 * w + pad, 3, 1))


def _frames(n_frames, n_points, seed, w=W, h=H):
    """frames in random orientations (odometry quaternions 1e-7 off unit length: Eigen does not normalise them), a BGR8
    image each, and a scan in front of its own camera (the reference asserts a positive depth, gaussian.cpp:69) that reaches
    well outside the image; with the orientations apart, much of each scan lies behind the other frames' cameras"""
    from gaussian_lic_b200 import synthetic as syn
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n_frames):
        q = rng.normal(size=4)
        q *= (1.0 + 1e-7) / np.linalg.norm(q)
        t = rng.normal(0, 1.0, 3)
        img = syn.make_gt_image(w, h, seed=seed + i)
        bgr = np.ascontiguousarray(np.round(img * 255).astype(np.uint8).transpose(1, 2, 0)[..., ::-1])
        z = rng.uniform(0.3, 15.0, n_points)
        pc = np.stack([z * rng.uniform(-1.2, 1.2, n_points), z * rng.uniform(-0.9, 0.9, n_points), z], 1)
        xyz = (pc @ fo.quat_rotation(q).T + t).astype(np.float32)
        rgb = rng.integers(0, 256, (n_points, 3), dtype=np.uint8)
        out.append(dict(q=q, t=t, bgr=bgr, xyz=xyz, rgb=rgb))
    return out


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same_map(a, b, what):
    da, db = a.download(moments=True), b.download(moments=True)
    for k in da:
        assert np.array_equal(_bits(da[k]), _bits(db[k])), "%s: %s" % (what, k)
    assert a.sky_rows() == b.sky_rows(), what
    sa, sb = a.stats(), b.stats()
    for f in STAT_FIELDS:
        assert np.array_equal(np.float64(getattr(sa, f)), np.float64(getattr(sb, f))), "%s: stats.%s" % (what, f)


def _feed_b(b, frames, lo, hi, k):
    """the existing API on the restated inputs for frames [lo, hi); the scan goes to initialize_lidar (the first scan) or
    extend at the training keyframe, as add_frame hands it off"""
    pts, col, dep = [], [], []
    for i in range(lo, hi):
        f = frames[i]
        R, t = fo.float_pose(f["q"], f["t"])
        b.add_keyframe(R, t, fo.decode(f["bgr"]), train=fo.is_train(i, k))
        pts.append(f["xyz"]); col.append(f["rgb"]); dep.append(fo.depth_rsp(f["q"], f["t"], f["xyz"]))
    pts, rgb, dep = np.concatenate(pts), np.concatenate(col), np.concatenate(dep)
    return pts, rgb, dep


def _compare(da, db, steps, what):
    """test_gpu_mapper._compare's criterion: per group, 99.9 % of the entries within 2 % of one learning rate and none beyond
    the sign-flip bound (the render backward sums with float atomics, so two runs differ in the last bits)"""
    for k, lr in LR.items():
        a, b = np.asarray(da[k], np.float64).reshape(-1), np.asarray(db[k], np.float64).reshape(-1)
        if a.size == 0:
            continue
        d = np.abs(a - b)
        q, mx = np.quantile(d, 0.999) / lr, d.max() / lr
        assert q <= 0.02 + 1e-7 / lr, "%s: %s q99.9 %.3g" % (what, k, q)
        assert mx <= 6.4 * steps + 1e-7 / lr, "%s: %s max %.3g" % (what, k, mx)


def _same_loss(la, lb):
    """The first iteration's loss of two mappers with bit-identical maps and images.  The loss kernel adds its per-CTA
    partial sums with float atomics, so the scalar is order-dependent in its last bits (the per-pixel gradient is not)."""
    assert np.isfinite(la) and abs(la - lb) <= 1e-5 * abs(lb), (la, lb)


def test_decode_bit_exact_at_1080p():
    """keyframe_image of 8-bit frames (row padding 64 bytes) equals the restated decode: a random 1920x1080 frame and a frame
    with every byte value in every channel"""
    w, h = 1920, 1080
    rng = np.random.default_rng(1)
    rand = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    every = np.stack([np.arange(w * h) % 256, (np.arange(w * h) * 7 + 3) % 256, 255 - np.arange(w * h) % 256], 1)
    every = every.astype(np.uint8).reshape(h, w, 3)
    m = _mapper(w, h)
    m.enable_frames(1, 0, 0)
    xyz = np.array([[0.0, 0.0, 5.0]], np.float32)
    rgb = np.array([[10, 20, 30]], np.uint8)
    for img in (rand, every):
        assert m.add_frame([0, 0, 0, 1], [0, 0, 0], _padded(img), xyz, rgb)
    for i, img in enumerate((rand, every)):
        assert np.array_equal(_bits(m.keyframe_image(i)), _bits(fo.decode(img))), i
    st = m.frames_get()
    assert (st.frames, st.train, st.test, st.pending_points) == (2, 2, 0, 0)
    assert st.image_bytes >= 2 * 3 * w * h
    m.close()


@pytest.mark.parametrize("h,w,offset", [(5, 37, 0), (64, 64, 0), (33, 100, 1), (1080, 1920, 0)])
def test_decode_kernel(h, w, offset):
    """glic_decode_bgr8 on device buffers: full tiles, a partial last tile, H*W not a multiple of 4, an unaligned input"""
    from gaussian_lic_b200 import capi
    rng = np.random.default_rng(h * w)
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    buf = torch.zeros(3 * h * w + 16, dtype=torch.uint8, device="cuda:0")
    buf[offset:offset + 3 * h * w] = torch.as_tensor(img.reshape(-1), device="cuda:0")
    out = torch.full((3, h, w), -1.0, dtype=torch.float32, device="cuda:0")
    capi.check(capi.lib.glic_decode_bgr8(h, w, C.c_void_p(buf.data_ptr() + offset), C.c_void_p(out.data_ptr()), None), "decode_bgr8")
    torch.cuda.synchronize()
    assert np.array_equal(_bits(out.cpu().numpy()), _bits(fo.decode(img)))
    assert capi.lib.glic_decode_bgr8(0, w, C.c_void_p(buf.data_ptr()), C.c_void_p(out.data_ptr()), None) == -1
    assert capi.lib.glic_decode_bgr8(h, w, None, C.c_void_p(out.data_ptr()), None) == -1


def test_same_map_as_float_api_and_training():
    """12 frames, k = 5: keyframes at frames 4 and 9, 10 held out; 20 000-point scans (outside the image and behind the
    extending keyframe's camera too), 1000 sky points.  Mapper A takes raw frames, mapper B the existing API on the
    restated inputs.  Identical map, sky, stats, images and scores before any training; the same first loss and
    (atomic-order noise aside) the same parameters after five iterations."""
    k, n = 5, 20_000
    frames = _frames(12, n, 2)
    a, b = _mapper(), _mapper()
    a.enable_frames(k, SKY, RADIUS)
    flags = [a.add_frame(f["q"], f["t"], _padded(f["bgr"]), f["xyz"], f["rgb"]) for f in frames[:5]]
    assert flags == [False] * 4 + [True]
    pts, rgb, dep = _feed_b(b, frames, 0, 5, k)
    b.initialize_lidar(pts, fo.colours_init(rgb), dep, _focal(), SKY, RADIUS)
    _same_map(a, b, "after keyframe 4 (initialize)")
    assert a.sky_rows() == SKY and a.stats().num_gaussians == SKY + 5 * n
    flags = [a.add_frame(f["q"], f["t"], _padded(f["bgr"]), f["xyz"], f["rgb"]) for f in frames[5:10]]
    assert flags == [False] * 4 + [True]
    pts, rgb, dep = _feed_b(b, frames, 5, 10, k)
    inserted = b.extend(pts, fo.colours_extend(rgb), dep)
    assert inserted > 0 and a.stats().last_inserted == inserted
    _same_map(a, b, "after keyframe 9 (extend)")
    for f in frames[10:]:
        assert not a.add_frame(f["q"], f["t"], f["bgr"], f["xyz"], f["rgb"])
    for i in (10, 11):
        R, t = fo.float_pose(frames[i]["q"], frames[i]["t"])
        b.add_keyframe(R, t, fo.decode(frames[i]["bgr"]), train=False)
    st = a.frames_get()
    assert (st.frames, st.train, st.test, st.pending_points) == (12, 2, 10, 2 * n)
    assert st.image_bytes >= 12 * 3 * W * H
    train = [i for i in range(12) if fo.is_train(i, k)]
    test = [i for i in range(12) if not fo.is_train(i, k)]
    for is_train, order in ((True, train), (False, test)):
        for j, i in enumerate(order):
            want = fo.decode(frames[i]["bgr"])
            assert np.array_equal(_bits(a.keyframe_image(j, is_train)), _bits(want)), (is_train, j)
            assert np.array_equal(_bits(b.keyframe_image(j, is_train)), _bits(want)), (is_train, j)
            sa, sb = a.evaluate(j, is_train), b.evaluate(j, is_train)
            assert _bits(np.array(sa)).tolist() == _bits(np.array(sb)).tolist(), (is_train, j, sa, sb)
    # training on the same explicit view lists, both mappers restarted from one anisotropic copy of the map: the initial
    # LiDAR Gaussians are spheres, so their rotation gradients are rounding noise whose sign Adam's first step would take
    g = a.download()
    rng = np.random.default_rng(9)
    P = g["means"].shape[0]
    g["log_scales"] = (g["log_scales"] + rng.normal(0, 0.3, (P, 3))).astype(np.float32)
    g["rots"] = rng.normal(size=(P, 4)).astype(np.float32)
    a.initialize(g); b.initialize(g)
    sa, sb = a.optimize([1]), b.optimize([1])
    _same_loss(sa.last_loss, sb.last_loss)
    a.optimize([0, 1, 1, 0]); b.optimize([0, 1, 1, 0])
    assert a.stats().iterations == b.stats().iterations == 5
    _compare(a.download(), b.download(), 5, "after five iterations")
    a.close(); b.close()


def test_exposure_and_pose_start_state():
    """with exposure and pose refinement on, a frame keyframe starts at E = [I | 0] and at its restated float pose, with the
    camera block glic_camera_block gives for it: exposure_get and pose_get equal the float-image mapper's"""
    from gaussian_lic_b200 import mapper
    k = 3
    frames = _frames(6, 2000, 3)
    a, b = _mapper(), _mapper()
    for m in (a, b):
        m.enable_exposure(0.001)
        m.enable_pose_refinement(1e-4, 1e-4)
    a.enable_frames(k, 0, 0)
    for f in frames:
        a.add_frame(f["q"], f["t"], f["bgr"], f["xyz"], f["rgb"])
    pts, rgb, dep = _feed_b(b, frames, 0, 3, k)
    b.initialize_lidar(pts, fo.colours_init(rgb), dep, _focal(), 0, 0)
    pts, rgb, dep = _feed_b(b, frames, 3, 6, k)
    b.extend(pts, fo.colours_extend(rgb), dep)
    _same_map(a, b, "exposure + pose")
    eye = np.concatenate([np.eye(3), np.zeros((3, 1))], 1).astype(np.float32)
    for j, i in enumerate((2, 5)):
        assert np.array_equal(a.exposure(j), eye) and np.array_equal(b.exposure(j), eye)
        (Ra, ta, ca), (Rb, tb, cb) = a.pose(j, camera=True), b.pose(j, camera=True)
        R, t = fo.float_pose(frames[i]["q"], frames[i]["t"])
        assert np.array_equal(_bits(Ra), _bits(R)) and np.array_equal(_bits(ta), _bits(t))
        assert np.array_equal(_bits(Ra), _bits(Rb)) and np.array_equal(_bits(ta), _bits(tb))
        want = mapper.camera_block(W, H, FX, FY, W / 2.0, H / 2.0, R, t)
        for key in ("view", "proj", "campos", "lims"):
            assert np.array_equal(_bits(ca[key]), _bits(want[key])) and np.array_equal(_bits(ca[key]), _bits(cb[key])), key
    sa, sb = a.optimize([0]), b.optimize([0])
    _same_loss(sa.last_loss, sb.last_loss)
    a.close(); b.close()


def _state(m):
    st, fs = m.stats(), m.frames_get()
    dl = m.download(moments=True)
    return ([getattr(st, f) for f in STAT_FIELDS], (fs.frames, fs.train, fs.test, fs.pending_points, fs.image_bytes),
            {k: _bits(v).copy() for k, v in dl.items()}, m.sky_rows())


def _same_state(s0, s1, what):
    assert s0[0] == s1[0] and s0[1] == s1[1] and s0[3] == s1[3], what
    for k in s0[2]:
        assert np.array_equal(s0[2][k], s1[2][k]), (what, k)


def test_rejected_frames_change_nothing():
    from gaussian_lic_b200 import capi
    lib = capi.lib
    frames = _frames(3, 500, 4)
    f0 = frames[0]
    img, xyz, rgb = np.ascontiguousarray(f0["bgr"]), f0["xyz"], f0["rgb"]

    def frame(**kw):
        f = capi.Frame()
        f.q_wc[:] = list(f0["q"]); f.t_wc[:] = list(f0["t"])
        f.bgr, f.row_bytes, f.n_points = img.ctypes.data, 3 * W, len(xyz)
        f.xyz, f.rgb = xyz.ctypes.data, rgb.ctypes.data
        for key, v in kw.items():
            setattr(f, key, v)
        return f

    flag = C.c_int(-7)
    # frames not enabled
    m = _mapper()
    assert lib.glic_mapper_add_frame(m._h, C.byref(frame()), C.byref(flag)) == -1 and flag.value == -7
    assert lib.glic_mapper_enable_frames(m._h, 0, 0, 0) == -1                       # k < 1
    assert lib.glic_mapper_enable_frames(m._h, 2, -1, 0) == -1                      # sky_points < 0
    assert lib.glic_mapper_enable_frames(m._h, 2, 10, 0) == -1                      # a sky without a radius
    assert lib.glic_mapper_enable_frames(None, 2, 0, 0) == -1
    assert m.frames_get().frames == 0
    m.enable_frames(2, 100, RADIUS)
    assert lib.glic_mapper_enable_frames(m._h, 2, 100, RADIUS) == -1               # once per mapper
    # a first keyframe with an empty accumulated scan (frame 1 of k = 2 after a frame without points)
    assert m.add_frame(f0["q"], f0["t"], img, xyz[:0], rgb[:0]) is False
    s0 = _state(m)
    rejected = [frame(n_points=0),                                                  # empty scan at the first keyframe
                frame(bgr=None), frame(xyz=None), frame(rgb=None),                  # null pointers
                frame(row_bytes=3 * W - 1),                                          # row_bytes < 3 W
                frame(n_points=-1)]
    for f in rejected:
        assert lib.glic_mapper_add_frame(m._h, C.byref(f), C.byref(flag)) == -1 and flag.value == -7
        _same_state(s0, _state(m), "rejected frame")
    assert lib.glic_mapper_add_frame(m._h, None, None) == -1 and lib.glic_mapper_add_frame(None, C.byref(frame()), None) == -1
    _same_state(s0, _state(m), "null frame")
    out = np.empty((3, H, W), np.float32)
    assert lib.glic_mapper_keyframe_image(m._h, 0, 1, out.ctypes.data) == -1          # only held-out keyframe 0 exists
    assert lib.glic_mapper_keyframe_image(m._h, 1, 0, out.ctypes.data) == -1
    assert lib.glic_mapper_keyframe_image(m._h, 0, 0, None) == -1
    assert lib.glic_mapper_frames_get(m._h, None) == -1
    assert lib.glic_mapper_add_frame(m._h, C.byref(frame()), C.byref(flag)) == 0 and flag.value == 1   # now a valid frame
    st = m.frames_get()
    assert (st.frames, st.train, st.test, st.pending_points) == (2, 1, 1, 0) and m.sky_rows() == 100
    m.close()


def test_mixing_float_and_frame_keyframes_trains():
    """initialize_lidar + a float keyframe, then raw frames: the first frame hand-off extends the map (the mapper is already
    initialized) and optimize trains over both kinds of keyframe"""
    from gaussian_lic_b200 import synthetic as syn
    frames = _frames(4, 3000, 5)
    m = _mapper(max_iters=8)
    f0 = frames[0]
    m.initialize_lidar(f0["xyz"], fo.colours_init(f0["rgb"]), fo.depth_rsp(f0["q"], f0["t"], f0["xyz"]), _focal(), 0, 0)
    R, t = fo.float_pose(f0["q"], f0["t"])
    m.add_keyframe(R, t, syn.make_gt_image(W, H, seed=40))
    P0 = m.stats().num_gaussians
    m.enable_frames(2, 0, 0)
    for f in frames[1:]:
        m.add_frame(f["q"], f["t"], f["bgr"], f["xyz"], f["rgb"])
    st = m.stats()
    assert st.num_gaussians > P0 and m.sky_rows() == 0
    assert (m.frames_get().train, m.frames_get().test) == (1, 2)
    st = m.optimize([0, 1, 0, 1, 1])
    assert np.isfinite(st.last_loss) and st.iterations == 5
    for j in (0, 1):
        psnr, ssim = m.evaluate(j)
        assert np.isfinite(psnr) and np.isfinite(ssim)
    m.close()
