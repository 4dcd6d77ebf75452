"""The native mapper's optimisation step (csrc/mapper.cu) against the float64 CPU oracle on maps the mapper builds itself:
the first LiDAR scan and the skybox (glic_mapper_initialize_lidar), and raw BGR8 frames with their scans
(glic_mapper_add_frame), which initialize the map and then extend it.

The other gradient tests train on small_scene's random anisotropic splats at depths of about 8-10.  A built map puts the step
somewhere else:
  - sky rows at |p| = 10 * skybox_radius = 10 000, far beyond zfar and behind every other splat, with knn scales of 10-200,
    so that most pixels' lists end in them.  Their pose-gradient lever arm p_view x g is formed per Gaussian in float32, and
    their SH direction adjoint divides by |o|^3 ~ 1e12;
  - LiDAR rows whose scales are scaling_scale * depth / focal for depths of 0.1-200 m: sub-pixel splats whose 2-D covariance
    is mostly the 0.3 low-pass term next to splats wider than the image, all at opacity 0.1;
  - every row isotropic with the identity rotation: the first step's rotation gradient is zero in exact arithmetic.  It is
    held to a noise bound whose scale is the rotation gradient the same rows get on the second step, once Adam has made
    their scales anisotropic;
  - 8-bit ground truth, and a keyframe with a black band where nothing is drawn: residuals of exactly zero (the sign(0)
    branch of the L1 term's gradient, which reaches the exposure's offsets through dL/dE).

The pose gradient is held to test_gpu_pose's 2e-3 of the f64 restatement.  Its sky and LiDAR parts and sum_i |term_i| are
printed so that the conditioning of the float32 per-Gaussian terms is on record.  On the raw frames' map the f32 oracle
itself lands up to ~4e-3 from the f64 one (alpha and transmittance threshold flips), so there each group is held to
max(2e-3, twice that measured distance).

The frame is 320 x 208 at the fastlivo field of view (its 640 x 512 focal lengths halved), and the sky has the config's
100 000 points at radius 1000.
"""
import numpy as np
import pytest

from helpers import GRAD_RTOL
from test_gpu_exposure import EXPO_LR, _reference_expo
from test_gpu_initialize import _scan
from test_gpu_mapper_grads import (B1, C1, GROUPS, H, W, _check_step, _check_untouched, _compare, _lr6, _raw, _recovered,
                                   _reference, _state)
from test_gpu_mapper_wide import _step_against_oracle
from test_gpu_pose import LR_R, LR_T, _pose_reference

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

FX, FY = 431.795259219 / 2, 431.550090267 / 2          # config/fastlivo.yaml:3-4 (640 x 512), halved for 320 x 208
FOCAL = (float(np.float32(FX)) + float(np.float32(FY))) / 2   # the focal add_frame derives from the float config
SKY, RADIUS = 100_000, 1000                            # config/fastlivo.yaml: skybox_points_num, skybox_radius
VIEWS = (0, 2, 5)                                      # rig views (synthetic.orbit_pose) of the three training keyframes
N_SCAN = 3000                                          # LiDAR points in front of each keyframe's camera
# Step 1 rotation gradient of an isotropic map over its step 2 scale.  The noise is a few float32 ulp of the covariance
# gradient; the step 2 gradient is that gradient times the anisotropy of one Adam step (+-3.2 scaling_lr per log-scale,
# ~0.03), so the ratio is ~1e-7 / 0.03.  An H100 run measured at most 2.2e-6 (sky and LiDAR rows, SH degree 1 and 3).
ROT_NOISE = 2e-5
IDENT = np.float32([1, 0, 0, 0])


def _new_mapper(deg, S):
    from gaussian_lic_b200 import mapper
    return mapper.Mapper(W, H, FX, FY, W / 2.0, H / 2.0, sh_degree=deg, seed=5 + deg, views_per_rank=S)


def _lidar_map(deg, S):
    """initialize_lidar with the config's sky and one scan made of N_SCAN points in front of each of three rig cameras, then
    the three training keyframes; returns the mapper, their camera blocks and ground truths"""
    from gaussian_lic_b200 import mapper, synthetic as syn
    poses = [syn.orbit_pose(v, radius=2.0) for v in VIEWS]
    pts, cols, dep = (np.concatenate(x) for x in zip(*[_scan(N_SCAN, 40 + i, R, t) for i, (R, t) in enumerate(poses)]))
    m = _new_mapper(deg, S)
    m.initialize_lidar(pts, cols, dep, FOCAL, SKY, RADIUS)
    assert m.sky_rows() == SKY and m.stats().num_gaussians == SKY + 3 * N_SCAN
    gts = [syn.make_gt_image(W, H, seed=60 + i) for i in range(len(VIEWS))]
    for (R, t), img in zip(poses, gts):
        m.add_keyframe(R, t, img)
    cams = [mapper.camera_block(W, H, FX, FY, W / 2.0, H / 2.0, R, t) for R, t in poses]
    return m, cams, gts


def _row_sets(vis, sky):
    rows = np.flatnonzero(vis)
    return dict(sky=rows[rows < sky], LiDAR=rows[rows >= sky])


def _check_fresh_rots(before, got, ref1, ref2, sets, what):
    """Step 1 of a map whose rows are all isotropic with the identity rotation: the covariance does not depend on the
    rotation, so its gradient is zero in exact arithmetic.  The recovered gradient must stay below ROT_NOISE times, and the
    f64 oracle's below 1e-12 times, the largest f64 rotation gradient the same rows get on step 2 (ref2)."""
    p = before["p"]
    vis2 = np.flatnonzero(ref2["vis"])
    for name, rows in sets.items():
        assert np.all(p["log_scales"][rows] == p["log_scales"][rows][:, :1]) and np.all(p["rots"][rows] == IDENT), (what, name)
        both = np.intersect1d(rows, vis2)
        scale = np.abs(ref2["grads"]["float64"]["rots"][both]).max()
        noise = np.abs(got["rots"][rows]).max()
        want = np.abs(ref1["grads"]["float64"]["rots"][rows]).max()
        print("%s, %s rows: step 1 max |d rots| recovered %.3e, f64 oracle %.3e; step 2 f64 scale %.3e over %d rows "
              "(ratios %.2e, %.2e)" % (what, name, noise, want, scale, both.size, noise / scale, want / scale))
        assert scale > 0 and noise <= ROT_NOISE * scale and want <= 1e-12 * scale, (what, name, noise, want, scale)


# ---- 1. LiDAR + sky map, plain steps -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("deg", [3, 1])
def test_lidar_sky_map_steps_match_oracle(oracle32, oracle64, deg):
    m, cams, gts = _lidar_map(deg, 3)
    batch = [0, 1, 2]
    sky = m.sky_rows()
    hist = []
    for step in (1, 2):
        what = "LiDAR + sky, degree %d, step %d" % (deg, step)
        before = _state(m)
        st = m.optimize(batch)
        after = _state(m)
        ref = _reference(_raw(before), cams, gts, batch, (oracle64, oracle32))
        assert abs(st.last_loss - ref["loss"]) <= 1e-5 * ref["loss"], (what, st.last_loss, ref["loss"])
        got = _recovered(before, after)
        sets = _row_sets(ref["vis"], sky)
        print("%s: %d sky rows and %d LiDAR rows visible in the batch" % (what, sets["sky"].size, sets["LiDAR"].size))
        assert sets["sky"].size >= 300 and sets["LiDAR"].size >= 300, what
        for name, rows in sets.items():
            _compare(got, ref, rows, "%s, %s rows" % (what, name), GROUPS if step == 2 else GROUPS[1:])
        rows = np.flatnonzero(ref["vis"])
        _check_step(before, after, got, rows, _lr6(), what)
        _check_untouched(before, after, ~ref["vis"], what)
        hist.append((before, got, ref, sets))
    (before, got, ref1, sets), (_, _, ref2, _) = hist
    _check_fresh_rots(before, got, ref1, ref2, sets, "LiDAR + sky, degree %d" % deg)
    m.close()


# ---- 2. the same map with exposure and pose refinement -------------------------------------------------------------------
def _pose_parts(m, batch, gts, oracle64, what):
    """Per keyframe of the batch, the f64 pose restatement summed over the sky rows and over the LiDAR rows alone, each
    with sum_i |term_i| of its per-Gaussian terms, weighted like the mapper's gradient (slots holding it / S)"""
    raw = _raw(_state(m))
    sky, n = m.sky_rows(), raw["means"].shape[0]
    out = {}
    for k in dict.fromkeys(batch):
        cam, Es = {k: m.pose(k, camera=True)[2]}, {k: m.exposure(k)}
        w = batch.count(k) / len(batch)
        out[k] = {name: w * _pose_reference(raw, cam, gts, [k], [oracle64], Es=Es, rows=rows, magnitude=True)[0]["float64"][k]
                  for name, rows in (("sky", np.arange(sky)), ("LiDAR", np.arange(sky, n)))}
        for name, (g, mag) in out[k].items():
            print("%s: keyframe %d, %s rows: dL/d(rho, omega) part %s, sum |term| %s" % (what, k, name, g, mag))
    return out


def test_lidar_sky_map_with_exposure_and_pose(oracle32, oracle64):
    """S = 4, exposure and pose refinement on: two steps through _step_against_oracle.  Before each, the f64 pose
    restatement is split into its sky and LiDAR parts; after it, the recovered pose gradient's error is printed against
    2^-24 * sum_i |term_i|, the size of the rounding of the float32 per-Gaussian terms."""
    m, _, gts = _lidar_map(3, 4)
    m.enable_exposure(EXPO_LR)
    m.enable_pose_refinement(LR_T, LR_R)
    batch = [0, 1, 2, 1]
    hist = []
    for step in (1, 2):
        what = "LiDAR + sky with exposure and pose, step %d" % step
        parts = _pose_parts(m, batch, gts, oracle64, what)
        before, pm0 = _state(m), {k: m.pose_state(k)[0] for k in parts}
        ref = _step_against_oracle(m, batch, 3, gts, (oracle32, oracle64), what, GROUPS if step == 2 else GROUPS[1:])
        after = _state(m)
        for k, pp in parts.items():
            got = (m.pose_state(k)[0].astype(np.float64) - (B1 * pm0[k]).astype(np.float64)) / C1
            want, mag = pp["sky"][0] + pp["LiDAR"][0], pp["sky"][1] + pp["LiDAR"][1]
            err = np.abs(got - want)
            print("%s: keyframe %d |got - want| %s, 2^-24 sum |term| %s, ratio %s (want vs _step_against_oracle's %.1e)" % (
                what, k, err, 2.0 ** -24 * mag, err / (2.0 ** -24 * mag), np.abs(want - ref["pose"]["float64"][k]).max()))
        sets = _row_sets(ref["vis"], m.sky_rows())
        print("%s: %d sky rows and %d LiDAR rows visible in the batch" % (what, sets["sky"].size, sets["LiDAR"].size))
        assert sets["sky"].size >= 300 and sets["LiDAR"].size >= 300, what
        hist.append((before, _recovered(before, after), ref, sets))
    (before, got, ref1, sets), (_, _, ref2, _) = hist
    _check_fresh_rots(before, got, ref1, ref2, sets, "LiDAR + sky with exposure and pose")
    m.close()


# ---- 3. raw frames end to end ----------------------------------------------------------------------------------------------
K = 2                                                  # select_every_k_frame: frames 1, 3, 5 are the training keyframes
BAND = 169                                             # keyframe 0's image is black from this row down


def _frames(seed=3):
    """Six frames in three pairs; pair j is turned by 12 j degrees about the world's vertical and moved 0.15 j sideways.  Every
    camera is pitched 25 degrees down: below row BAND its rays point more than 32 degrees below the horizon, under the sky
    (which reaches 23.6 degrees down, cos phi >= -0.4), and the scans stay above it (camera y <= 0.05 z, z >= 2)."""
    from scipy.spatial.transform import Rotation
    from gaussian_lic_b200 import synthetic as syn
    rng = np.random.default_rng(seed)
    a = np.radians(25.0)
    R0 = np.stack([[0.0, -1.0, 0.0], [-np.sin(a), 0.0, -np.cos(a)], [np.cos(a), 0.0, -np.sin(a)]], 1)   # right, down, forward
    out = []
    for i in range(6):
        j = i // 2
        R = Rotation.from_euler("z", 12.0 * j, degrees=True).as_matrix() @ R0
        t = np.array([0.0, 0.15 * j, 0.0]) + rng.normal(0, 0.01, 3)
        img = syn.make_gt_image(W, H, seed=seed + i)
        bgr = np.ascontiguousarray(np.round(img * 255).astype(np.uint8).transpose(1, 2, 0)[..., ::-1])
        if i == K - 1:
            bgr[BAND:] = 0
        n = 4000
        z = rng.uniform(2.0, 15.0, n)
        pc = np.stack([z * rng.uniform(-0.75, 0.75, n), z * rng.uniform(-0.45, 0.05, n), z], 1)
        out.append(dict(q=Rotation.from_matrix(R).as_quat(), t=t, bgr=bgr, xyz=(pc @ R.T + t).astype(np.float32),
                        rgb=rng.integers(0, 256, (n, 3), dtype=np.uint8)))
    return out


def _flip_rtol(m, batch, gts, oracles, what):
    """_compare's tolerance per group for one step: max(GRAD_RTOL, 2 y), y the f32 oracle's own distance from the f64 one
    (max |f32 - f64| / max |f64| over the visible rows of the mean over the batch's slots, through the exposure, at the
    keyframes' current cameras).  A pixel whose alpha sits on the 1/255 or T < 1e-4 threshold takes the other branch in
    float32 and moves the Gaussians it covers by a whole pixel's contribution.  On the raw frames' map the largest colour
    gradients belong to sky rows that only a few pixels reach, and an H100 run measured y = 2.2e-3 for dc on step 1 while
    the GPU was within 3e-7 of the f32 oracle."""
    raw = _raw(_state(m))
    grads, vis = {}, 0
    for o in oracles:
        acc = {g: 0.0 for g in GROUPS}
        for k in dict.fromkeys(batch):
            r = _reference_expo(raw, {k: m.pose(k, camera=True)[2]}, gts, [k], {k: m.exposure(k)}, o)
            vis = vis | r["vis"]
            for g in GROUPS:
                acc[g] = acc[g] + batch.count(k) / len(batch) * r["grads"]["float64"][g]
        grads[o.dtype.name] = acc
    rows = np.flatnonzero(vis)
    a, b = grads["float32"], grads["float64"]
    y = {g: np.abs(a[g][rows] - b[g][rows]).max() / max(np.abs(b[g][rows]).max(), 1e-30) for g in GROUPS}
    print("%s: f32 oracle vs f64 oracle, max|diff|/max|ref|: %s" % (what, {g: "%.2e" % x for g, x in y.items()}))
    return {g: max(GRAD_RTOL, 2.0 * y[g]) for g in GROUPS}


def test_raw_frames_steps_match_oracle(oracle32, oracle64):
    """enable_frames with the config's sky; after each training keyframe (the first initializes the map, the next two
    extend it) one S = 4 step with exposure and pose refinement on, checked by _step_against_oracle on the keyframes'
    8-bit images.  Before the first step, keyframe 0's black band renders black: residuals of exactly zero."""
    m = _new_mapper(3, 4)
    m.enable_exposure(EXPO_LR)
    m.enable_pose_refinement(LR_T, LR_R)
    m.enable_frames(K, SKY, RADIUS)
    frames = _frames()
    batches = [[0, 0, 0, 0], [1, 0, 1, 1], [2, 1, 0, 2]]
    hist = []
    for j, batch in enumerate(batches):
        flags = [m.add_frame(f["q"], f["t"], f["bgr"], f["xyz"], f["rgb"]) for f in frames[K * j:K * (j + 1)]]
        assert flags == [False] * (K - 1) + [True]
        st = m.stats()
        assert m.sky_rows() == SKY and (j == 0 or st.last_inserted > 0), (j, st.last_inserted)
        gts = [m.keyframe_image(k) for k in range(j + 1)]
        what = "raw frames, keyframe %d (%d rows, %d inserted), step %d" % (j, st.num_gaussians, st.last_inserted, j + 1)
        if j == 0:
            img = m.render(0)
            zero = np.all((img == 0) & (gts[0] == 0), axis=0)
            print("%s: %d pixels with an exact-zero residual, %d of them in the black band" % (what, zero.sum(), zero[BAND:].sum()))
            assert zero[BAND:].sum() >= 0.9 * zero[BAND:].size, what
        rtol = _flip_rtol(m, batch, gts, (oracle32, oracle64), what)
        before = _state(m)
        ref = _step_against_oracle(m, batch, j + 1, gts, (oracle32, oracle64), what, GROUPS[1:] if j == 0 else GROUPS, rtol)
        sets = _row_sets(ref["vis"], SKY)
        print("%s: %d sky rows and %d LiDAR rows visible in the batch" % (what, sets["sky"].size, sets["LiDAR"].size))
        assert sets["sky"].size >= 300 and sets["LiDAR"].size >= 300, what
        hist.append((before, _recovered(before, _state(m)), ref, sets))
    (before, got, ref1, sets), (_, _, ref2, _) = hist[:2]
    _check_fresh_rots(before, got, ref1, ref2, sets, "raw frames")
    assert m.stats().iterations == 3
    m.close()
