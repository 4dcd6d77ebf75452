"""Per-keyframe valid-pixel masks in the native mapper (glic_mapper_set_keyframe_mask, glic_mapper_keyframe_mask,
glic_mapper_add_frame_masked), with the deterministic option on wherever bits are compared.

* All-ones masks on every keyframe train, evaluate and align bit for bit like no masks, with the same launches per iteration.
* A painted "moving object" in the ground truth under the mask changes no bit of training, evaluation or alignment.
* Masks cost no launch per iteration.
* A map trained on keyframes with a transient object scores a higher held-out PSNR when the object is masked.
* extend() on a masked newest keyframe inserts exactly the unmasked selection's points whose pixel is used (the selection of
  glic_extend with final_T = 0 at masked pixels); add_frame_masked does the same at its hand-off.
* The setter's validation, clearing and the getter round trip; every allocation of the new paths failed in turn."""
import numpy as np
import pytest

import extend_oracle
import loss_mask_reference as mr
from test_gpu_densify import F, SEED, VIEWS, _lidar_scan, _poses

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

W, H = 320, 208
N_KF = len(VIEWS)


def _gts(seed=40):
    from gaussian_lic_b200 import synthetic as syn
    return [syn.make_gt_image(W, H, seed=seed + i).astype(np.float32) for i in range(N_KF)]


def _paint(img, k):
    """a bright 'moving object' at a keyframe-dependent place, and the mask that leaves it out"""
    out = img.copy()
    y0, x0 = 30 + 11 * k, 40 + 23 * k
    out[:, y0:y0 + 70, x0:x0 + 90] = np.array([1.0, 0.1, 0.9], np.float32)[:, None, None]
    w = np.ones((H, W), bool)
    w[y0:y0 + 70, x0:x0 + 90] = False
    return out, w


def _mapper(gts, masks=None, test_gts=None, test_masks=None, expo=True, pose=True):
    from gaussian_lic_b200 import mapper
    pts, cols, dep = _lidar_scan(3000, 5, *_poses([0])[0])
    m = mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=3, capacity=4000, seed=SEED, views_per_rank=2)
    m.initialize_lidar(pts, cols, dep, F, 500, 1000)
    for i, (R, t) in enumerate(_poses()):
        m.add_keyframe(R, t, gts[i])
        if masks is not None:
            m.set_mask(True, i, masks[i])
    for i, (R, t) in enumerate(_poses()[:2] if test_gts is not None else []):
        m.add_keyframe(R, t, test_gts[i], train=False)
        if test_masks is not None:
            m.set_mask(False, i, test_masks[i])
    if expo:
        m.enable_exposure(0.001)
    if pose:
        m.enable_pose_refinement(1e-3, 1e-3)
    m.set_deterministic(True)
    return m


def _train(m, steps=12):
    from gaussian_lic_b200 import capi
    launches = []
    for i in range(steps):
        before = capi.launch_count()
        m.optimize([VIEWS[(2 * i) % 8], VIEWS[(2 * i + 1) % 8]])
        launches.append(capi.launch_count() - before)
    return launches


def _bits(x):
    return np.ascontiguousarray(np.asarray(x, np.float32)).view(np.uint32)


def _state(m):
    out = {"map." + k: np.asarray(v) for k, v in m.download(moments=True).items()}
    for i in range(N_KF):
        R, t = m.pose(i)
        out["pose%d" % i] = np.concatenate([np.ravel(R), np.ravel(t)])
        out["E%d" % i] = np.ravel(m.exposure(i))
    for i in (0, 3):
        out["evaluate%d" % i] = np.asarray(m.evaluate(i), np.float32)
    for i in (0, 1):
        out["evaluate_test%d" % i] = np.asarray(m.evaluate(i, train=False), np.float32)
        a = m.align(i, train=False, iterations=5, exposure_lr=1e-3, split=True)
        out["align%d" % i] = np.concatenate([np.ravel(a["R_wc"]), np.ravel(a["t_wc"]), np.ravel(a["E"]),
                                             np.asarray([a["psnr"], a["ssim"], a["first_loss"], a["last_loss"]], np.float32)])
    return out


def _same(a, b):
    assert set(a) == set(b)
    for k in a:
        assert np.array_equal(_bits(a[k]), _bits(b[k])), k


def test_all_ones_masks_change_no_bit_and_no_launch():
    gts = _gts()
    ones = [np.ones((H, W), bool)] * N_KF
    a = _mapper(gts, test_gts=gts[:2])
    b = _mapper(gts, masks=ones, test_gts=gts[:2], test_masks=ones[:2])
    try:
        la, lb = _train(a), _train(b)
        assert la == lb
        _same(_state(a), _state(b))
    finally:
        a.close(); b.close()


def test_ground_truth_under_the_mask_changes_no_bit():
    gts = _gts()
    painted = [_paint(g, k) for k, g in enumerate(gts)]
    masks = [w for _, w in painted]
    a = _mapper(gts, masks=masks, test_gts=gts[:2], test_masks=masks[:2])
    b = _mapper([p for p, _ in painted], masks=masks, test_gts=[p for p, _ in painted[:2]], test_masks=masks[:2])
    c = _mapper(gts, test_gts=gts[:2])
    try:
        la, lb, lc = _train(a), _train(b), _train(c)
        assert la == lb and max(la) <= min(lc)                  # a mask adds no launch to an iteration
        _same(_state(a), _state(b))
    finally:
        a.close(); b.close(); c.close()


def test_masked_training_scores_higher_on_clean_held_out_views():
    """keyframes carry a transient object; the held-out views at the first two poses are clean"""
    gts = _gts()
    painted = [_paint(g, 0) for g in gts]                     # the object at one screen place in every keyframe
    imgs, masks = [p for p, _ in painted], [w for _, w in painted]
    a = _mapper(imgs, test_gts=gts[:2], expo=False, pose=False)
    b = _mapper(imgs, masks=masks, test_gts=gts[:2], expo=False, pose=False)
    try:
        _train(a, 150); _train(b, 150)
        pa = [a.evaluate(i, train=False)[0] for i in range(2)]
        pb = [b.evaluate(i, train=False)[0] for i in range(2)]
        print("\nheld-out PSNR unmasked %s masked %s margin %.3f dB" % (pa, pb, np.mean(pb) - np.mean(pa)))
        assert np.mean(pb) > np.mean(pa) + 0.5
    finally:
        a.close(); b.close()


def _inserted(m, P0):
    return m.download()["means"][P0:]


def test_extend_leaves_masked_pixels_out():
    from gaussian_lic_b200 import mapper
    gts = _gts()
    R, t = _poses()[N_KF - 1]
    pts, cols, dep = _lidar_scan(20000, 9, R, t)
    w = mr.mask_family("straddle", H, W, seed=3) & mr.mask_family("random", H, W, seed=4)
    got = {}
    for name, mk in (("none", None), ("mask", w), ("ones", np.ones((H, W), bool))):
        m = _mapper(gts, expo=False, pose=False)
        try:
            _train(m, 4)
            if mk is not None:
                m.set_mask(True, N_KF - 1, mk)
            P0 = m.stats().num_gaussians
            m.extend(pts, cols.astype(np.float32), dep)
            got[name] = _inserted(m, P0)
        finally:
            m.close()
    assert np.array_equal(got["none"], got["ones"])
    # the unmasked selection's points whose pixel is used, in order: extend()'s camera from the keyframe's camera block
    cb = mapper.camera_block(W, H, F, F, W / 2.0, H / 2.0, R, t)
    view = cb["view"].reshape(4, 4).T                       # row-major Rt
    Rcw, tcw = view[:3, :3].astype(np.float32), view[:3, 3].astype(np.float32)
    cam = extend_oracle.camera_coords(pts, Rcw, tcw)
    xf, yf = extend_oracle.pixel_coords(cam, F, F, W / 2.0, H / 2.0)
    px, py = np.floor(xf).astype(np.int64), np.floor(yf).astype(np.int64)
    row = {tuple(p): i for i, p in enumerate(pts)}
    keep = [row[tuple(p)] for p in got["none"]]
    want = np.array([i for i in keep if w[py[i], px[i]]], np.int64)
    assert 0 < len(want) < len(keep)
    assert np.array_equal(got["mask"], pts[want])


def test_add_frame_masked_hand_off():
    """frames through add_frame_masked (every second one a training keyframe): an all-ones mask builds the add_frame map bit
    for bit; a real mask inserts fewer points at the extend() hand-off, and every keyframe keeps its mask"""
    from test_gpu_frames import FX, FY, _frames
    from gaussian_lic_b200 import mapper
    frames = _frames(6, 3000, 31)
    w = mr.mask_family("straddle", H, W, seed=8) & mr.mask_family("random", H, W, seed=9)
    runs = {}
    for name in ("none", "ones", "mask"):
        m = mapper.Mapper(W, H, FX, FY, W / 2.0, H / 2.0, sh_degree=1, capacity=40000, seed=SEED)
        m.enable_frames(2)
        try:
            for f in frames:
                mk = None if name == "none" else (np.ones((H, W), bool) if name == "ones" else w)
                m.add_frame(f["q"], f["t"], f["bgr"], f["xyz"], f["rgb"], mask=mk)
            runs[name] = (m.download()["means"], [m.mask(True, i) for i in range(3)], [m.mask(False, i) for i in range(3)])
        finally:
            m.close()
    assert np.array_equal(_bits(runs["none"][0]), _bits(runs["ones"][0]))
    assert len(runs["mask"][0]) < len(runs["none"][0])
    assert runs["none"][1][0] == (None, 0)
    for kind in (1, 2):
        for got, n in runs["mask"][kind]:
            assert n == int(w.sum()) and np.array_equal(got.astype(bool), w)


def test_setter_validation_clearing_and_round_trip():
    from gaussian_lic_b200 import capi
    gts = _gts()
    m = _mapper(gts, test_gts=gts[:2], expo=False, pose=False)
    try:
        assert m.mask(True, 0) == (None, 0)
        w = mr.mask_family("random", H, W, seed=1)
        m.set_mask(True, 0, w)
        got, n = m.mask(True, 0)
        assert n == int(w.sum()) and np.array_equal(got, w.astype(np.uint8))
        with pytest.raises(capi.GlicError):
            m.set_mask(True, 0, np.zeros((H, W), bool))          # no used pixel: refused, the old mask stays
        with pytest.raises(capi.GlicError):
            m.set_mask(True, N_KF, w)
        with pytest.raises(capi.GlicError):
            m.set_mask(False, 2, w)
        got2, n2 = m.mask(True, 0)
        assert n2 == n and np.array_equal(got2, got)
        m.set_mask(False, 1, ~w)
        assert m.mask(False, 1)[1] == int((~w).sum())
        m.set_mask(True, 0, None)
        assert m.mask(True, 0) == (None, 0)
        # a mask that leaves the split fit columns empty is refused by align
        left_empty = np.zeros((H, W), bool)
        left_empty[:, W // 2:] = True
        m.set_mask(False, 0, left_empty)
        with pytest.raises(capi.GlicError):
            m.align(0, train=False, iterations=2, split=True)
        m.align(0, train=False, iterations=2, split=False)
    finally:
        m.close()


def test_failed_allocations_change_nothing():
    from gaussian_lic_b200 import capi
    gts = _gts()
    m = _mapper(gts, expo=False, pose=False)
    try:
        w = mr.mask_family("random", H, W, seed=2)
        m.set_mask(True, 1, w)
        before = m.mask(True, 1)
        for k in (1, 2):                                           # the bit buffer, then the staging
            assert capi.lib.glic_debug_fail_allocation(k) == 0
            with pytest.raises(capi.GlicError):
                m.set_mask(True, 1, ~w)
            capi.lib.glic_debug_fail_allocation(0)
            after = m.mask(True, 1)
            assert after[1] == before[1] and np.array_equal(after[0], before[0])
        m.set_mask(True, 1, ~w)
        assert m.mask(True, 1)[1] == int((~w).sum())
    finally:
        capi.lib.glic_debug_fail_allocation(0)
        m.close()
