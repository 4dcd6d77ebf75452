"""glic_mapper_correct_poses on the GPU: the row update against the NumPy restatement bit for bit, a rigid motion of the whole
map and its cameras that leaves every render in place, a drifted map repaired, anchors through the map's life, keyframes,
and training after a correction."""
import numpy as np
import pytest

from helpers import small_scene
import pose_correction_oracle as O

pytestmark = pytest.mark.gpu
pytest.importorskip("torch")

W, H, F = 320, 208, 250.0
VIEWS = (0, 2, 5, 7)                         # rig views (synthetic.orbit_pose) of the training keyframes
HELD_OUT = 3
GROUPS = ("means", "dc", "sh", "opacity_logits", "log_scales", "rots")
# pixel bounds of a render before and after a rigid motion of map and cameras: float32 rounding of the moved means, rotations
# and SH moves a splat by ~1e-7 relative, which changes a pixel by far less than 1e-5 on average; a pixel whose tile or depth
# order flips at a boundary may move by up to a splat's contribution, which is rare (the 99.9th percentile) and bounded
MEAN_BOUND, P999_BOUND, MAX_BOUND = 1e-5, 1e-3, 2e-2


def _rot(axis, angle):
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * K @ K


def _moved_pose(dR, dt, R, t):
    """the pose of a camera carried along by the rigid motion x -> dR x + dt"""
    return (dR @ np.asarray(R, np.float64)).astype(np.float32), (dR @ np.asarray(t, np.float64) + dt).astype(np.float32)


def _raw(deg, P=5000, seed=21):
    g, _ = small_scene(P, W, H, seed, deg)
    raw = {k: np.array(g[k], np.float32) for k in ("means", "log_scales", "rots", "opacity_logits", "dc", "sh")}
    raw["dc"] = raw["dc"].reshape(P, 3)
    raw["degree"] = deg
    return raw


def _mapper(raw, capacity=0, held_out=True, **kw):
    from gaussian_lic_b200 import mapper, synthetic as syn
    m = mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=raw["degree"], capacity=capacity, **kw)
    m.initialize(raw)
    m._poses = []
    for i, v in enumerate(VIEWS):
        R, t = syn.orbit_pose(v, radius=2.0)
        m.add_keyframe(R, t, syn.make_gt_image(W, H, seed=7 + i))
        m._poses.append((np.asarray(R, np.float32), np.asarray(t, np.float32)))
    if held_out:
        R, t = syn.orbit_pose(HELD_OUT, radius=2.0)
        m.add_keyframe(R, t, syn.make_gt_image(W, H, seed=99), train=False)
        m._held = (np.asarray(R, np.float32), np.asarray(t, np.float32))
    return m


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same_bits(a, b, what):
    for k in a:
        assert np.array_equal(_bits(a[k]), _bits(b[k])), "%s: %s differs" % (what, k)


def _pixel_stats(a, b):
    d = np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).ravel()
    return float(d.mean()), float(np.quantile(d, 0.999)), float(d.max())


def _within(stats):
    return stats[0] <= MEAN_BOUND and stats[1] <= P999_BOUND and stats[2] <= MAX_BOUND


# ---- 1. rows bit for bit ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_rows_match_the_restatement_bit_for_bit(deg):
    from gaussian_lic_b200.mapper import pose_correction_record
    raw = _raw(deg)
    m = _mapper(raw)
    m.optimize([0, 1, 2, 3, 0, 2])                  # moments that are not zero
    P = m.stats().num_gaussians
    anchors = np.random.default_rng(deg).integers(-1, len(VIEWS), P).astype(np.int32)
    m.set_anchors(anchors)
    assert np.array_equal(m.anchors(), anchors)
    before = m.download(moments=True)
    dR, dt = _rot([0.3, -1.0, 0.5], 0.6), np.array([0.4, -1.1, 2.0])
    corr, records = [], {}
    for k in (0, 2):
        R, t = m._poses[k]
        Rn, tn = _moved_pose(dR, dt, R, t)
        corr.append((True, k, Rn, tn))
        records[k] = pose_correction_record(R, t, Rn, tn, deg)
    corr.append((False, 0, *_moved_pose(dR, dt, *m._held)))
    moved = m.correct_poses(corr)
    after = m.download(moments=True)
    want, mask = O.apply_rows({k: before[k] for k in GROUPS}, anchors, records, deg)
    assert moved == int(mask.sum()) and 0 < moved < P
    _same_bits({k: after[k] for k in GROUPS}, want, "degree %d" % deg)
    _same_bits({k: after[k][~mask] for k in GROUPS}, {k: before[k][~mask] for k in GROUPS}, "unmoved rows")
    _same_bits({k: after[k] for k in ("exp_avg", "exp_avg_sq")}, {k: before[k] for k in ("exp_avg", "exp_avg_sq")}, "moments")
    for k in ("dc", "opacity_logits", "log_scales"):
        assert np.array_equal(_bits(after[k]), _bits(before[k])), k
    assert np.array_equal(m.anchors(), anchors)
    m.close()


# ---- 2. equivariance ----------------------------------------------------------------------------------------------------------
def _renders(m):
    return [m.render(k) for k in range(len(VIEWS))] + [m.render(0, train=False)]


def test_rigid_motion_of_map_and_cameras_leaves_every_render_in_place():
    """35 degrees about a tilted axis and a 2 m translation of a trained degree-3 map, every row anchored, and of every training and
    held-out keyframe.  Observed on an H100 80GB HBM3: mean |render after - render before| <= 3.8e-7, 99.9th percentile <= 3.1e-6,
    max <= 1.2e-3 over the five keyframes; the negative control (SH rest unrotated) gave mean >= 0.034 and max >= 0.17."""
    from gaussian_lic_b200 import mapper
    raw = _raw(3, P=6000)
    m = _mapper(raw)
    m.optimize(list(range(len(VIEWS))) * 5)
    P = m.stats().num_gaussians
    m.set_anchors(np.arange(P, dtype=np.int32) % len(VIEWS))
    before, scores = _renders(m), [m.evaluate(k) for k in range(len(VIEWS))] + [m.evaluate(0, train=False)]
    g_before = m.download()
    dR, dt = _rot([0.2, 1.0, -0.4], np.radians(35.0)), np.array([1.2, -0.8, 1.4])        # 35 degrees, a 2 m translation
    corr = [(True, k, *_moved_pose(dR, dt, *m._poses[k])) for k in range(len(VIEWS))] + [(False, 0, *_moved_pose(dR, dt, *m._held))]
    assert m.correct_poses(corr) == P
    after = _renders(m)
    stats = [_pixel_stats(a, b) for a, b in zip(before, after)]
    print("render |after - before| (mean, p99.9, max) per keyframe:", stats)
    for s in stats:
        assert _within(s), stats
    for k, (p0, s0) in enumerate(scores):
        p1, s1 = m.evaluate(k) if k < len(VIEWS) else m.evaluate(0, train=False)
        assert abs(p1 - p0) < 0.01 and abs(s1 - s0) < 1e-4, (k, p0, p1, s0, s1)
    # negative control: the same moved map with its SH rest left as it was must fail the bounds
    g = m.download()
    g["sh"] = g_before["sh"]
    g["degree"] = 3
    ctrl = mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=3)
    ctrl.initialize(g)
    for k in range(len(VIEWS)):
        ctrl.add_keyframe(*corr[k][2:], np.zeros((3, H, W), np.float32))
    ctrl_stats = [_pixel_stats(before[k], ctrl.render(k)) for k in range(len(VIEWS))]
    print("negative control (SH rest unrotated):", ctrl_stats)
    assert not any(_within(s) for s in ctrl_stats), ctrl_stats
    ctrl.close()
    m.close()


# ---- 3. a drifted map repaired ------------------------------------------------------------------------------------------------
def test_a_drifted_part_of_the_map_is_moved_back():
    from gaussian_lic_b200 import mapper
    from gaussian_lic_b200.mapper import pose_correction_record
    raw = _raw(3, P=6000, seed=5)
    P = raw["means"].shape[0]
    group_b = np.arange(P) % 2 == 1                                  # anchored to training keyframe 1, the rest to keyframe 0
    truth = _mapper(raw, held_out=False)
    from gaussian_lic_b200 import synthetic as syn
    Rh, th = syn.orbit_pose(HELD_OUT, radius=2.0)
    true_view = truth.render_camera(Rh, th, outputs=("rgb",))["rgb"]
    # the drift D: 8 degrees and 0.35 m on group B's rows (rotations and SH included) and on keyframe 1's pose
    dR, dt = _rot([1.0, 0.3, 0.2], np.radians(8.0)), np.array([0.25, -0.2, 0.15])
    drift = pose_correction_record(np.eye(3), np.zeros(3), dR.astype(np.float32), dt.astype(np.float32), 3)
    drifted = {k: raw[k] for k in GROUPS}
    anchor = np.where(group_b, 1, 0).astype(np.int32)
    drifted, _ = O.apply_rows(drifted, np.where(group_b, 0, -1), {0: drift}, 3)
    drifted["degree"] = 3
    m = mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=3)
    m.initialize(drifted)
    for k, (R, t) in enumerate(truth._poses):
        pose = _moved_pose(drift["R"], drift["t"], R, t) if k == 1 else (R, t)
        m.add_keyframe(*pose, np.zeros((3, H, W), np.float32))
    m.add_keyframe(Rh, th, true_view, train=False)
    m.set_anchors(anchor)
    bad = m.render(0, train=False)
    psnr_bad, _ = m.evaluate(0, train=False)
    assert m.correct_poses([(True, 1, *truth._poses[1])]) == int(group_b.sum())
    good = m.render(0, train=False)
    psnr_good, _ = m.evaluate(0, train=False)
    stats = _pixel_stats(good, np.clip(true_view, 0, 1))
    print("held-out view after the repair (mean, p99.9, max):", stats, "PSNR %.2f -> %.2f dB" % (psnr_bad, psnr_good))
    assert not _within(_pixel_stats(bad, np.clip(true_view, 0, 1)))
    assert _within(stats), stats
    assert psnr_good - psnr_bad >= 3.0, (psnr_bad, psnr_good)
    truth.close(); m.close()


# ---- 4. anchors through the map's life ----------------------------------------------------------------------------------------
SKY, RADIUS = 40, 1000


def _points(n, seed):
    rng = np.random.default_rng(seed)
    z = rng.uniform(2.0, 10.0, n)
    xyz = np.stack([z * rng.uniform(-0.6, 0.6, n) * W / (2 * F), z * rng.uniform(-0.6, 0.6, n) * H / (2 * F), z], 1).astype(np.float32)
    return xyz, rng.integers(0, 256, (n, 3), dtype=np.uint8)


def test_anchors_follow_the_add_frame_hand_off():
    from gaussian_lic_b200 import mapper
    m = mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=3, capacity=256, seed=5)     # regrows on the way
    m.enable_frames(2, SKY, RADIUS)
    mask = np.ones((H, W), np.uint8)
    mask[:, : W // 3] = 0
    want = []
    for i in range(8):
        rng = np.random.default_rng(100 + i)
        xyz, rgb = _points(400, 200 + i)
        bgr = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        P0, ntrain = m.stats().num_gaussians, m.frames_get().train
        train = m.add_frame((0.0, 0.0, 0.0, 1.0), (0.0, 0.0, 0.01 * i), bgr, xyz, rgb, mask=mask if i == 5 else None)
        P1 = m.stats().num_gaussians
        if train:
            if P0 == 0:
                want += [-1] * SKY + [ntrain] * (P1 - SKY)
            else:
                want += [ntrain] * (P1 - P0)
        assert np.array_equal(m.anchors(), np.array(want, np.int32)), i
    assert m.frames_get().train == 4 and m.stats().capacity > 256 and m.sky_rows() == SKY
    # extend() anchors its rows to the newest training keyframe
    P0 = m.stats().num_gaussians
    xyz, rgb = _points(300, 9)
    m.extend(xyz, rgb.astype(np.float32) / 255.0, xyz[:, 2].copy())
    assert np.all(m.anchors()[P0:] == m.frames_get().train - 1) and np.array_equal(m.anchors()[:P0], np.array(want, np.int32))
    m.close()


def test_anchors_move_with_their_rows_through_every_compaction():
    """Each compaction's selection restated by the density oracles (tests/densify_oracle.py, tests/density_control_oracle.py) on
    the mapper's own statistics and activations, as test_gpu_density_control does: the column after the call is the column
    before it gathered through the oracle's source rows (clones and split children take their parent's anchor)."""
    import densify_oracle as do
    import density_control_oracle as dco
    from gaussian_lic_b200 import mapper
    from test_gpu_densify import VIEWS as DVIEWS, _activate, _pick, _trained
    from test_gpu_density_control import _child_smax
    m = _trained(3, True)                                   # sky rows, a tight capacity: the densify calls grow the arenas
    cap0 = m.stats().capacity
    rng = np.random.default_rng(8)

    def fresh():
        a = rng.integers(-1, len(DVIEWS), m.stats().num_gaussians).astype(np.int32)
        m.set_anchors(a)
        return a, m.download(moments=True), m.sky_rows()

    # densify_and_prune with all three prune tests on
    a, before, S = fresh()
    thr, extent, acc, den, smax = _pick(m, before)
    maxr = m.screen_radii()
    _, _, act = _activate(before, opacity=True)
    cls = do.classes(acc, den, smax, S, thr, mapper.PERCENT_DENSE, extent)
    args = dict(min_opacity=float(np.float32(np.quantile(act, 0.1))), max_screen_radius=int(np.quantile(maxr[maxr > 0], 0.9)),
                max_world_scale=float(np.float32(np.quantile(smax[S:], 0.9))))
    want = dco.densify_and_prune(cls, act, smax, _child_smax(before), maxr, S, **args)
    got = m.densify_and_prune(extent, grad_threshold=thr, **args)
    assert got == {k: want[k] for k in ("cloned", "split", "pruned", "rows")} and want["children"] > 0 and want["pruned"] > 0
    assert np.array_equal(m.anchors(), a[want["src"]]), "densify_and_prune"
    # densify alone, past the capacity
    m.optimize(DVIEWS)
    a, before, S = fresh()
    thr, extent, acc, den, smax = _pick(m, before)
    src, n = do.select(do.classes(acc, den, smax, S, thr, mapper.PERCENT_DENSE, extent))
    assert m.densify(extent, grad_threshold=thr) == (n["cloned"], n["split"]) and n["cloned"] > 0 and n["split"] > 0
    assert np.array_equal(m.anchors(), a[src]), "densify"
    assert m.stats().capacity > cap0
    # prune by opacity
    a, before, S = fresh()
    s, _, act = _activate(before, opacity=True)
    cut = float(np.float32(np.quantile(act, 0.3)))
    gone = dco.removed(act, s.max(1), np.zeros(act.shape[0], np.int32), np.arange(act.shape[0]) < S, cut, 0, 0.0)
    assert m.prune(cut) == int(gone.sum()) > 0
    assert np.array_equal(m.anchors(), a[~gone]), "prune"
    # prune_unseen over one view, by the mapper's own scores
    a, before, S = fresh()
    _, hits, ends = m.contribution(views=[0])
    gone = ((hits + ends) < 1) & (np.arange(hits.shape[0]) >= S)
    assert m.prune_unseen(views=[0]) == int(gone.sum()) > 0
    assert np.array_equal(m.anchors(), a[~gone]), "prune_unseen"
    m.close()


def _snapshot(m):
    s = m.download(moments=True)
    s["anchors"] = m.anchors()
    for k in range(len(VIEWS)):
        s["pose%d" % k] = m.render(k)
    return s


def test_refused_calls_change_nothing():
    from gaussian_lic_b200 import capi
    raw = _raw(2, P=2000)
    m = _mapper(raw)
    P = m.stats().num_gaussians
    a = np.arange(P, dtype=np.int32) % len(VIEWS)
    m.set_anchors(a)
    snap = _snapshot(m)
    R, t = m._poses[1]
    bad_rows = [np.where(np.arange(P) == 7, len(VIEWS), a), np.where(np.arange(P) == 9, -2, a)]
    for b in bad_rows:
        with pytest.raises(capi.GlicError):
            m.set_anchors(b.astype(np.int32))
    nan = t.copy()
    nan[1] = np.nan
    refused = [
        [(True, 1, R, t), (True, 1, R, t)],                           # listed twice
        [(True, 1, 2.0 * R, t)],                                      # not a rotation
        [(True, 1, np.diag([1.0, 1.0, -1.0]) @ R, t)],                # det -1
        [(True, 1, R, nan)],                                          # NaN
        [(True, len(VIEWS), R, t)],                                   # index out of range
        [(False, 1, R, t)],                                           # held-out index out of range
        [(True, -1, R, t)],
    ]
    for c in refused:
        with pytest.raises(capi.GlicError):
            m.correct_poses(c)
    assert m.correct_poses([]) == 0
    # a failed allocation (the record table) leaves the mapper as it was
    assert capi.lib.glic_debug_fail_allocation(1) == 0
    try:
        with pytest.raises(capi.GlicError):
            m.correct_poses([(True, 1, *_moved_pose(_rot([0, 0, 1], 0.3), np.zeros(3), R, t))])
    finally:
        capi.lib.glic_debug_fail_allocation(0)
    now = _snapshot(m)
    _same_bits(now, snap, "after refused calls")
    m.close()


# ---- 5. keyframes ---------------------------------------------------------------------------------------------------------------
def test_corrected_keyframes_draw_at_their_new_pose():
    raw = _raw(3, P=3000)
    m = _mapper(raw)
    dR, dt = _rot([1.0, -2.0, 0.5], 0.4), np.array([0.3, 0.2, -0.5])
    Rn, tn = _moved_pose(dR, dt, *m._poses[2])
    Rh, th = _moved_pose(dR, dt, *m._held)
    m.set_anchors(np.full(m.stats().num_gaussians, -1, np.int32))
    assert m.correct_poses([(True, 2, Rn, tn), (False, 0, Rh, th)]) == 0            # held-out keyframes move no row
    assert np.array_equal(_bits(m.render(2)), _bits(m.render_camera(Rn, tn, outputs=("rgb",))["rgb"]))
    assert np.array_equal(_bits(m.render(0, train=False)), _bits(m.render_camera(Rh, th, outputs=("rgb",))["rgb"]))
    m.close()


def test_refined_poses_are_composed_with_the_correction():
    raw = _raw(3, P=3000)
    m = _mapper(raw)
    m.enable_pose_refinement(1e-3, 1e-3)
    m.optimize(list(range(len(VIEWS))) * 4)
    before = [m.pose(k) for k in range(len(VIEWS))]
    states = [m.pose_state(k) for k in range(len(VIEWS))]
    assert any(not np.array_equal(before[k][1], m._poses[k][1]) for k in range(len(VIEWS)))      # refined away from the given
    dR, dt = _rot([0.0, 1.0, 0.2], 0.5), np.array([0.5, 0.0, -0.3])
    m.correct_poses([(True, k, *_moved_pose(dR, dt, *m._poses[k])) for k in (1, 3)])
    for k in range(len(VIEWS)):
        R, t = m.pose(k)
        if k in (1, 3):
            Rw, tw = dR @ before[k][0].astype(np.float64), dR @ before[k][1].astype(np.float64) + dt
            assert np.abs(R - Rw).max() < 1e-5 and np.abs(t - tw).max() < 1e-5, k
        else:
            assert np.array_equal(_bits(R), _bits(before[k][0])) and np.array_equal(_bits(t), _bits(before[k][1]))
        s = m.pose_state(k)
        assert np.array_equal(_bits(s[0]), _bits(states[k][0])) and np.array_equal(_bits(s[1]), _bits(states[k][1])) and s[2] == states[k][2]
    m.close()


# ---- 6. training continues ------------------------------------------------------------------------------------------------------
def test_deterministic_twins_stay_bit_identical():
    raw = _raw(3, P=4000)
    twins = [_mapper(raw) for _ in range(2)]
    dR, dt = _rot([0.3, 0.3, 1.0], 0.25), np.array([0.1, -0.4, 0.2])
    for m in twins:
        m.set_deterministic(True)
        m.optimize(list(range(len(VIEWS))) * 2)
        m.set_anchors(np.arange(m.stats().num_gaussians, dtype=np.int32) % len(VIEWS))
        m.correct_poses([(True, k, *_moved_pose(dR, dt, *m._poses[k])) for k in (0, 1)])
    _same_bits(twins[0].download(moments=True), twins[1].download(moments=True), "after the correction")
    for m in twins:
        m.optimize(list(range(len(VIEWS))) * 3)
    _same_bits(twins[0].download(moments=True), twins[1].download(moments=True), "after further iterations")
    assert np.isfinite(twins[0].stats().last_loss)
    for m in twins:
        m.close()


def _two_rank_run(rank, world, exchange):
    """one replica of a two-rank mapper (views_per_rank 1) with pose refinement: train, correct, train on; the downloads, anchors
    and refined poses right after the correction and after the further iterations"""
    raw = _raw(3, P=4000, seed=13)
    m = _mapper(raw, capacity=4096, rank=rank, world=world, views_per_rank=1)
    m.connect(exchange(m.export_handle()))
    m.enable_pose_refinement(1e-4, 1e-4)
    m.optimize([0, 1, 2, 3, 1, 2])
    m.set_anchors(np.arange(m.stats().num_gaussians, dtype=np.int32) % (len(VIEWS) + 1) - 1)
    dR, dt = _rot([0.5, -0.2, 1.0], 0.3), np.array([0.2, 0.1, -0.3])
    moved = m.correct_poses([(True, k, *_moved_pose(dR, dt, *m._poses[k])) for k in (1, 3)] +
                            [(False, 0, *_moved_pose(dR, dt, *m._held))])

    def snap():
        s = m.download(moments=True)
        s["anchors"] = m.anchors()
        for k in range(len(VIEWS)):
            R, t, cam = m.pose(k, camera=True)
            s["R%d" % k], s["t%d" % k], s["view%d" % k] = R, t, cam["view"]
        return s
    after = snap()
    m.optimize([2, 3, 0, 1, 3, 0])
    trained = snap()
    assert m.stats().iterations == 6 and np.isfinite(m.stats().last_loss)
    return m, moved, after, trained


def _two_rank_worker(rank, world, port, q):
    try:
        import os
        import torch
        import torch.distributed as dist
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
        torch.cuda.set_device(rank % torch.cuda.device_count())

        def exchange(mine):
            got = [None] * world
            dist.all_gather_object(got, mine)
            return got

        m, moved, after, trained = _two_rank_run(rank, world, exchange)
        dist.barrier()
        m.close()
        dist.destroy_process_group()
        q.put((rank, "ok", (moved, after, trained)))
    except Exception as e:          # noqa: BLE001 - reported to the parent
        import traceback
        q.put((rank, "%r\n%s" % (e, traceback.format_exc()), None))


@pytest.mark.timeout(300)
def test_two_ranks_stay_bit_identical_through_a_correction():
    """Two connected replicas (two GPUs when the box has them, one shared GPU otherwise, as the other two-rank tests run) with pose
    refinement make the same correct_poses call between optimize() calls: parameters, moments, anchors and refined poses are
    bit-identical across the replicas right after it and after further iterations, with no exchange for the correction itself."""
    import socket
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    q = ctx.Queue()
    procs = [ctx.Process(target=_two_rank_worker, args=(r, 2, port, q)) for r in range(2)]
    for p_ in procs:
        p_.start()
    res = sorted([q.get(timeout=240) for _ in procs], key=lambda r: r[0])
    for p_ in procs:
        p_.join(timeout=30)
    assert all(r[1] == "ok" for r in res), [r[1] for r in res]
    (ma, aa, ta), (mb, ab, tb) = res[0][2], res[1][2]
    assert ma == mb and ma == int(np.isin(aa["anchors"], (1, 3)).sum()) > 0
    for name in aa:
        assert np.array_equal(np.ascontiguousarray(aa[name]).view(np.uint8), np.ascontiguousarray(ab[name]).view(np.uint8)), \
            "replicas differ right after the correction in %s" % name
        assert np.array_equal(np.ascontiguousarray(ta[name]).view(np.uint8), np.ascontiguousarray(tb[name]).view(np.uint8)), \
            "replicas diverged after further iterations in %s" % name
    assert not np.array_equal(ta["means"], aa["means"])        # training moved the corrected map
