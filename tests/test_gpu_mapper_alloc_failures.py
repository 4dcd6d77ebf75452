"""The native mapper's failure contract (include/glic_b200.h, "Native mapping host"): a call that cannot allocate returns
GLIC_ERR_CUDA and leaves everything the getters return unchanged, except capacities.

glic_debug_fail_allocation(k) makes the k-th allocation from now fail on the host, without a CUDA call.  Every call that can
grow a buffer is run with k = 1, 2, ... until it succeeds; after each failed attempt the mapper's state must be bit-identical to
the state before the call.  A twin mapper makes the same calls without injection: after every successful call the two are
bit-identical, and after all of them they train alike.  (Training itself is compared with test_gpu_mapper's atomic-order
criterion: the render backward adds with float atomics, so two runs of one step differ in the last bits.)  No allocation
outlives the mappers (glic_debug_mapper_allocations).
"""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

W, H, F = 320, 208, 250.0
SKY, RADIUS = 40, 1000
GLIC_ERR_CUDA = -3
LR = dict(rots=0.001, means=1.6e-4, log_scales=0.005, opacity_logits=0.05, dc=2.5e-3, sh=2.5e-3 / 20)   # config/fastlivo.yaml:18-22
STATS = ("num_gaussians", "iterations", "last_inserted", "last_loss", "mean_visible", "overflow_regrows")


def _lib():
    from gaussian_lic_b200 import capi
    return capi.lib


def _mapper():
    from gaussian_lic_b200 import mapper
    return mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=3, capacity=256, seed=5)


def _points(n, seed):
    """n points in front of a camera at the origin looking down +z, most of them inside the image; depth = z"""
    rng = np.random.default_rng(seed)
    z = rng.uniform(2.0, 10.0, n)
    xyz = np.stack([z * rng.uniform(-0.6, 0.6, n) * W / (2 * F), z * rng.uniform(-0.6, 0.6, n) * H / (2 * F), z], 1).astype(np.float32)
    return xyz, rng.integers(0, 256, (n, 3), dtype=np.uint8), z.astype(np.float32)


def _frame(i, n):
    rng = np.random.default_rng(1000 + i)
    xyz, rgb, _ = _points(n, 2000 + i)
    bgr = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    return (0.0, 0.0, 0.0, 1.0), (0.0, 0.0, 0.0), bgr, xyz, rgb


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32).copy()


def _state(m, timings=True):
    """everything the getters return, capacities excepted (timings: the device times of the last extend / optimize)"""
    st, fs = m.stats(), m.frames_get()
    names = STATS + (("ms_extend", "ms_optimize") if timings else ())
    out = {"stats": [np.float64(getattr(st, f)).tobytes() for f in names], "sky": m.sky_rows(),
           "frames": (fs.frames, fs.train, fs.test, fs.pending_points, fs.image_bytes)}
    out.update({k: _bits(v) for k, v in m.download(moments=True).items()})
    for i in range(fs.train + m._extra_train):
        if m._expo:
            E, m1, m2, t = m.exposure_state(i)
            out["expo%d" % i] = [_bits(x) for x in (E, m1, m2)] + [t]
        if m._pose:
            R, tr, cam = m.pose(i, camera=True)
            p1, p2, pt = m.pose_state(i)
            out["pose%d" % i] = [_bits(x) for x in (R, tr, p1, p2)] + [pt] + [_bits(cam[k]) for k in ("view", "proj", "campos", "lims")]
    return out


def _same(a, b, what):
    assert a.keys() == b.keys(), what
    for k in a:
        va, vb = a[k], b[k]
        if isinstance(va, np.ndarray):
            assert va.shape == vb.shape and np.array_equal(va, vb), "%s: %s" % (what, k)
        elif isinstance(va, list):
            assert len(va) == len(vb) and all(np.array_equal(x, y) for x, y in zip(va, vb)), "%s: %s" % (what, k)
        else:
            assert va == vb, "%s: %s" % (what, k)


def _until_success(m, twin, call, what):
    """call(m) with the k-th allocation failing, k = 1, 2, ... until it succeeds; then call(twin) once without injection"""
    from gaussian_lic_b200 import capi
    lib = _lib()
    before = _state(m)
    failures = 0
    for k in range(1, 200):
        assert lib.glic_debug_fail_allocation(k) == 0
        try:
            call(m)
            ok = True
        except capi.GlicError as e:
            assert "(%d)" % GLIC_ERR_CUDA in str(e), (what, k, str(e))
            ok = False
        finally:
            lib.glic_debug_fail_allocation(0)
        if ok:
            break
        failures += 1
        _same(before, _state(m), "%s: failed attempt %d" % (what, k))
    else:
        raise AssertionError("%s never succeeded" % what)
    call(twin)
    _same(_state(m, timings=False), _state(twin, timings=False), "%s: against the twin" % what)
    return failures


def _lpips_weights(tmp_path):
    root = os.path.dirname(os.path.abspath(__file__))
    spec = importlib.util.spec_from_file_location("make_lpips_golden", os.path.join(root, "golden", "make_lpips_golden.py"))
    G = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(G)
    from gaussian_lic_b200 import lpips_weights
    path = tmp_path / "synthetic.bin"
    lpips_weights.write(path, G.synthetic_payload(1))
    return str(path)


def test_create_fails_cleanly_at_every_allocation():
    lib = _lib()
    base = lib.glic_debug_mapper_allocations()
    m = _mapper()
    cfg = m.cfg
    held = lib.glic_debug_mapper_allocations() - base
    m.close()
    assert held > 0 and lib.glic_debug_mapper_allocations() == base
    for k in range(1, held + 1):
        h = C.c_void_p()
        assert lib.glic_debug_fail_allocation(k) == 0
        rc = lib.glic_mapper_create(C.byref(cfg), C.byref(h))
        lib.glic_debug_fail_allocation(0)
        assert rc == GLIC_ERR_CUDA and not h.value, (k, rc)
        assert lib.glic_debug_mapper_allocations() == base, k
    assert lib.glic_debug_fail_allocation(-1) != 0


def test_every_growth_path_fails_without_a_trace(tmp_path):
    lib = _lib()
    base = lib.glic_debug_mapper_allocations()
    a, b = _mapper(), _mapper()
    pair = (a, b)
    for m in pair:
        m._extra_train = 0                      # training keyframes that did not come from add_frame
        m._expo = m._pose = False               # which per-keyframe state _state reads
        m.enable_frames(3, SKY, RADIUS)
        # frames 1-3 initialize the map at the first training keyframe (frame 3), 4-6 extend it, 7-8 leave 4000 points pending
        for i, n in enumerate((60, 60, 60, 10, 10, 10, 2000, 2000)):
            m.add_frame(*_frame(i, n))
    _same(_state(a, False), _state(b, False), "the twins' start")
    img = np.random.default_rng(7).uniform(0, 1, (3, H, W)).astype(np.float32)
    failures = {}

    def enable_exposure(m):
        m.enable_exposure(0.001)
        m._expo = True

    def enable_pose(m):
        m.enable_pose_refinement(1e-4, 1e-4)
        m._pose = True
    failures["enable_exposure"] = _until_success(a, b, enable_exposure, "enable_exposure")
    failures["enable_pose_refinement"] = _until_success(a, b, enable_pose, "enable_pose_refinement")
    for m in pair:                              # exposures that are not the starting one
        for i in range(m.frames_get().train):
            m.set_exposure(i, np.float32(1.0 + 0.01 * i) * np.eye(3, 4, dtype=np.float32))
    # the 9th frame: a new frame-store chunk, the scan past 4096 points, the hand-off's extend past the capacity
    cap = a.stats().capacity
    failures["add_frame"] = _until_success(a, b, lambda m: m.add_frame(*_frame(8, 2000)), "add_frame")
    assert a.frames_get().train == 3 and a.frames_get().pending_points == 0 and a.stats().capacity > cap
    # extend past the capacity
    st = a.stats()
    n = st.capacity - st.num_gaussians + 100
    xyz, rgb, dep = _points(n, 31)
    failures["extend"] = _until_success(a, b, lambda m: m.extend(xyz, rgb.astype(np.float32) / 255.0, dep), "extend")
    assert a.stats().capacity > st.capacity
    # add_keyframe crossing 64 rows of per-keyframe state
    for m in pair:
        while m.frames_get().train + m._extra_train < 64:
            m.add_keyframe(np.eye(3), np.zeros(3), img, train=True)
            m._extra_train += 1

    def add65(m):
        m.add_keyframe(np.eye(3), np.zeros(3), img, train=True)
        m._extra_train += 1
    failures["add_keyframe"] = _until_success(a, b, add65, "add_keyframe")
    failures["set_binning_pairs"] = _until_success(a, b, lambda m: m.set_binning_pairs(1 << 23), "set_binning_pairs")
    # prune the LiDAR and extend() rows (opacity 0.1), keep the sky (0.7)
    failures["prune"] = _until_success(a, b, lambda m: m.prune(0.5), "prune")
    assert a.stats().num_gaussians == SKY
    # initialize_lidar past the capacity
    st = a.stats()
    xyz, rgb, dep = _points(st.capacity + 100, 41)
    col = rgb.astype(np.float64) / 255.0
    failures["initialize_lidar"] = _until_success(a, b, lambda m: m.initialize_lidar(xyz, col, dep, F, SKY, RADIUS), "initialize_lidar")
    assert a.stats().capacity > st.capacity
    path = _lpips_weights(tmp_path)
    failures["load_lpips"] = _until_success(a, b, lambda m: m.load_lpips(path), "load_lpips")
    scores = {}
    failures["evaluate_lpips"] = _until_success(a, b, lambda m: scores.__setitem__(id(m), m.evaluate_lpips(0)), "evaluate_lpips")
    assert np.allclose(scores[id(a)], scores[id(b)], rtol=1e-6, atol=0), scores
    print("failed attempts per path:", failures)
    for what in ("add_frame", "extend", "add_keyframe", "set_binning_pairs", "prune", "initialize_lidar", "load_lpips", "evaluate_lpips"):
        assert failures[what] >= 1, what        # each of these allocates at least once

    # the grown mappers train alike
    steps = 8
    views = list(range(steps))
    sa, sb = a.optimize(views), b.optimize(views)
    assert np.isfinite(sa.last_loss) and abs(sa.last_loss - sb.last_loss) <= 1e-4 * abs(sb.last_loss), (sa.last_loss, sb.last_loss)
    # Every row of the map initialize_lidar built is isotropic with the identity rotation, so the first step's rotation gradient
    # is rounding noise (see test_gpu_mapper_built_maps), which Adam turns into a step of either sign, and the rows it turns
    # move apart in the other groups too: the parameters are held to the sign-flip bound only.
    da, db = a.download(), b.download()
    for k, lr in LR.items():
        d = np.abs(np.asarray(da[k], np.float64) - np.asarray(db[k], np.float64))
        assert d.max() / lr <= 6.4 * steps + 1e-7 / lr, k
    a.close(); b.close()
    assert lib.glic_debug_mapper_allocations() == base
