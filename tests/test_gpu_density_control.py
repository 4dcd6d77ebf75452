"""The native mapper's density control: the screen-radius statistic, glic_mapper_reset_opacity, glic_mapper_densify_and_prune
and the schedule inside optimize() (csrc/model_step.cu, csrc/prune.cu, csrc/mapper.cu).

Checkers: the standalone forward's radii, the NumPy restatement tests/density_control_oracle.py (on tests/densify_oracle.py)
on the mapper's own download, glic_densify_split for the children's normals, twin mappers from one initialisation, and the
replicas of a two-rank run.  Training is not bit-reproducible between two mappers (the render backward adds with float
atomics), so the twins either do not train before the compared call or train with zero learning rates and a selection that
does not depend on the gradients; the schedule's twins are compared that way.
"""
import ctypes as C
import os
import socket

import numpy as np
import pytest

import densify_oracle as do
import density_control_oracle as dco
from helpers import small_scene
from test_gpu_densify import (F, H, KEYS, SEED, VIEWS, W, _activate, _fail_until_success, _lidar_scan, _mapper, _moments, _pick, _poses,
                              _same, _split, _texture, _trained, _wall, _with_keyframes)

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

ZERO_LR = dict(position_lr=0.0, feature_lr=0.0, opacity_lr=0.0, scaling_lr=0.0, rotation_lr=0.0)


def _forward_radii(d, deg, views):
    """the elementwise max over `views` of the standalone forward's radii (0 where not visible) on the parameters d"""
    from gaussian_lic_b200 import mapper, model, ops
    dev = torch.device("cuda:0")
    mdl = model.PackedModel(dict(d, degree=deg), dev)
    mdl.activate()
    rast = ops.CRasterizer(W, H, dev)
    poses = _poses()
    out = np.zeros(d["means"].shape[0], np.int32)
    for v in views:
        _, _, radii = rast.forward(mdl.inputs, rast.make_view(mapper.camera_block(W, H, F, F, W / 2.0, H / 2.0, *poses[v])))
        torch.cuda.synchronize()
        out = np.maximum(out, np.maximum(radii.cpu().numpy().astype(np.int32), 0))
    return out


def _child_smax(d):
    """the largest activated scale of a split child of every row: the activation kernel on log-scale - log(1.6)"""
    s, _ = _activate(dict(d, log_scales=(d["log_scales"] - do.SPLIT_LOG_SCALE).astype(np.float32)))
    return s.max(1)


def _counts(res):
    return {k: res[k] for k in ("cloned", "split", "pruned", "rows")}


# ---- 1. the screen-radius statistic ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 2])
def test_screen_radii_match_the_standalone_forward(k):
    """Two batches of k views: maxr is the elementwise max of the forward's radii over the stepped views, exactly.  The
    optimiser off and an overflow-skipped iteration leave it; prune moves it, extend appends zeros across a capacity growth, a
    densify zeroes it."""
    P = 3000
    g, _ = small_scene(P, W, H, 29, 3)
    m = _mapper(3, capacity=P, views_per_rank=k)
    m.initialize(g)
    _with_keyframes(m)
    m.enable_densification()
    assert not m.screen_radii().any()
    want = np.zeros(P, np.int32)
    for b in range(2):
        views = VIEWS[b * k:(b + 1) * k]
        want = np.maximum(want, _forward_radii(m.download(), 3, views))
        m.optimize(views)
        assert np.array_equal(m.screen_radii(), want), "maxr after batch %d" % b
    assert (want > 0).sum() > P // 10
    before = m.screen_radii()
    m.set_optimizer(False)
    m.optimize(VIEWS[:k])
    m.set_optimizer(True)
    assert np.array_equal(m.screen_radii(), before), "optimiser off changed maxr"
    regrows = m.stats().overflow_regrows
    m.set_binning_pairs(1)
    m.optimize(VIEWS[:k])
    m.synchronize()
    assert m.stats().overflow_regrows > regrows
    assert np.array_equal(m.screen_radii(), before), "an overflowed iteration changed maxr"
    _, _, act = _activate(m.download(), opacity=True)
    cut = float(np.float32(np.median(act)))
    keep = act >= np.float32(cut)
    assert m.prune(cut) == int((~keep).sum()) > 0
    r1 = m.screen_radii()
    assert np.array_equal(r1, before[keep]), "maxr after prune"
    cap = m.stats().capacity
    pts, cols, dep = _lidar_scan(6000, 8, *_poses()[-1])
    n = m.extend(pts, cols.astype(np.float32), dep)
    r2 = m.screen_radii()
    assert n > 0 and r2.size == r1.size + n and m.stats().capacity > cap
    assert np.array_equal(r2[:r1.size], r1) and not r2[r1.size:].any()
    m.optimize(VIEWS)
    assert m.screen_radii()[r1.size:].any()
    m.densify(10.0, grad_threshold=1e30)
    assert not m.screen_radii().any(), "a real densify leaves maxr"
    m.close()


# ---- 2. reset_opacity -----------------------------------------------------------------------------------------------------
def test_reset_opacity_against_numpy():
    from gaussian_lic_b200 import capi
    m = _trained(3, True)
    S, M = m.sky_rows(), m.M
    before = m.download(moments=True)
    P = before["means"].shape[0]
    _, _, act = _activate(before, opacity=True)
    cut = np.float32(np.median(act[S:]))
    hit = (np.arange(P) >= S) & (act > cut)
    assert S > 0 and 0 < hit.sum() < P - S
    print("%d of %d non-sky rows above the cut, %d of %d sky rows" % (hit.sum(), P - S, (act[:S] > cut).sum(), S))
    for bad in (float("nan"), float("inf"), -float("inf"), 0.0, 1.0, -0.5, 1.5):
        assert capi.lib.glic_mapper_reset_opacity(m._h, bad) == -1, bad
    now = m.download(moments=True)
    for key in before:
        _same(now[key], before[key], "a rejected reset changed %s" % key)
    m.reset_opacity(float(cut))
    after = m.download(moments=True)
    want = before["opacity_logits"].reshape(-1).copy()
    want[hit] = dco.reset_logit(cut)
    _same(after["opacity_logits"].reshape(-1), want, "logits")
    for key in KEYS:
        if key != "opacity_logits":
            _same(after[key], before[key], "reset changed %s" % key)
    mb, ma = _moments(before, M), _moments(after, M)
    for key in mb:
        exp = mb[key].copy()
        if key[1] == "opacity_logits":
            exp[S:] = 0.0
        _same(ma[key], exp, "moments %s" % (key,))
    m.close()


# ---- 3. densify_and_prune -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("deg,sky", [(3, True), (0, False)])
def test_densify_and_prune_matches_numpy_oracle(deg, sky):
    """On a trained map: dry-run counts over consecutive-float sweeps of max_world_scale and integer sweeps of
    max_screen_radius; then every surviving row, both moments, n_sky and the restarted statistics of a real call."""
    from gaussian_lic_b200 import mapper
    m = _trained(deg, sky)
    before = m.download(moments=True)
    P, M, S = before["means"].shape[0], m.M, m.sky_rows()
    thr, extent, acc, den, smax = _pick(m, before)
    maxr = m.screen_radii()
    _, _, act = _activate(before, opacity=True)
    csmax = _child_smax(before)
    cls = do.classes(acc, den, smax, S, thr, mapper.PERCENT_DENSE, extent)
    args = dict(min_opacity=float(np.float32(np.quantile(act, 0.1))), max_screen_radius=int(np.quantile(maxr[maxr > 0], 0.9)),
                max_world_scale=float(np.float32(np.quantile(smax[S:], 0.9))))
    want = dco.densify_and_prune(cls, act, smax, csmax, maxr, S, **args)
    print("oracle counts %s, surviving children %d, sky %d of %d" % (_counts(want), want["children"], want["sky"], S))
    assert want["cloned"] > 10 and want["split"] > 10 and want["pruned"] > 10 and want["children"] > 10

    def dry(**kw):
        return m.densify_and_prune(extent, grad_threshold=thr, dry_run=True, **kw)

    nonsplit = np.nonzero((cls != 2) & (np.arange(P) >= S))[0]
    for j in nonsplit[:: max(1, nonsplit.size // 3)][:3]:
        for e in (smax[j:j + 1].view(np.int32) + np.arange(-2, 3, dtype=np.int32)).view(np.float32):
            got = dry(max_world_scale=float(e))
            assert got == _counts(dco.densify_and_prune(cls, act, smax, csmax, maxr, S, max_world_scale=e)), e
    for rv in np.unique(maxr[maxr > 0])[[0, -1]].tolist() + [int(np.median(maxr[maxr > 0]))]:
        for rr in range(max(1, rv - 2), rv + 3):
            assert dry(max_screen_radius=rr) == _counts(dco.densify_and_prune(cls, act, smax, csmax, maxr, S, max_screen_radius=rr)), rr
    assert dry(**args) == _counts(want)
    now = m.download(moments=True)
    for k in before:
        _same(now[k], before[k], "a dry run changed %s" % k)
    assert np.array_equal(m.screen_radii(), maxr)
    assert m.densify_and_prune(extent, grad_threshold=thr, **args) == _counts(want)
    after = m.download(moments=True)
    assert after["means"].shape[0] == want["rows"] and m.sky_rows() == want["sky"]
    src, kept = want["src"], want["kept"]
    kc = want["rows"] - want["children"]
    for k in KEYS:
        _same(after[k][:kc], before[k][src[:kc]], "kept / cloned rows: %s" % k)
    for k in ("rots", "dc", "sh", "opacity_logits"):
        _same(after[k][kc:], before[k][src[kc:]], "children: %s" % k)
    _same(after["log_scales"][kc:], before["log_scales"][src[kc:]] - do.SPLIT_LOG_SCALE, "children: log_scales")
    mb, ma = _moments(before, M), _moments(after, M)
    for key in mb:
        _same(ma[key][:kept], mb[key][src[:kept]], "kept rows' moments %s" % (key,))
        assert not ma[key][kept:].any(), "new rows' moments are not zero: %s" % (key,)
    # the children's xyz: every child of the unpruned densify result at its own row, then the survivors
    u = want["unpruned"]
    kc_u = u["kept"] + u["cloned"]
    parents = want["unpruned_src"][kc_u:]
    s, r = _activate(before)
    xyz, z = _split(before["means"][parents], s[parents], r[parents], 0, kc_u)
    pick = want["row"][kc:] - kc_u
    _same(after["means"][kc:], xyz[pick], "children's xyz vs glic_densify_split at their unpruned rows")
    _same(after["means"][kc:], do.split_xyz(before["means"][parents], s[parents], r[parents], z)[pick], "children's xyz vs NumPy")
    acc2, den2 = m.densify_stats()
    assert not acc2.any() and not den2.any() and not m.screen_radii().any()
    assert np.isfinite(m.optimize(VIEWS[:4]).last_loss)
    m.close()


def _twin(deg, sky, **kw):
    if sky:
        pts, cols, dep = _lidar_scan(3000, 5, *_poses([0])[0])
        m = _mapper(deg, capacity=3500, views_per_rank=2, **kw)
        m.initialize_lidar(pts, cols, dep, F, 500, 1000)
    else:
        g, _ = small_scene(3000, W, H, 31, deg)
        m = _mapper(deg, capacity=3000, views_per_rank=2, **kw)
        m.initialize(g)
    _with_keyframes(m)
    m.enable_densification()
    return m


@pytest.mark.parametrize("deg,sky,all_split", [(3, True, False), (3, False, False), (0, True, False), (0, False, False), (1, False, True)])
def test_densify_and_prune_equals_densify_then_predicate(deg, sky, all_split):
    """Twins from one initialisation (untrained: every non-sky row is selected at threshold 0): densify_and_prune on one equals
    densify() on the other followed by the predicate on its download, bit for bit in all six groups, both moments and n_sky.
    all_split: a tiny scene extent splits every row, so whole tiles of 1024 rows are split and survive."""
    a, b = _twin(deg, sky), _twin(deg, sky)
    d = a.download()
    S = a.sky_rows()
    s, _, act = _activate(d, opacity=True)
    smax = s.max(1)
    extent = 1e-6 if all_split else float(np.float32(np.median(smax[S:]) / np.float32(0.01)))
    args = dict(min_opacity=float(np.float32(np.quantile(act, 0.3))), max_world_scale=float(np.float32(np.quantile(smax[S:], 0.7))))
    got = a.densify_and_prune(extent, grad_threshold=0.0, **args)
    c, sp = b.densify(extent, grad_threshold=0.0)
    db = b.download(moments=True)
    n = db["means"].shape[0]
    sb, _, actb = _activate(db, opacity=True)
    gone = dco.removed(actb, sb.max(1), np.zeros(n, np.int32), np.arange(n) < S, args["min_opacity"], 0, args["max_world_scale"])
    keep = ~gone
    print("densify: %d cloned, %d split; the predicate removes %d of %d rows" % (c, sp, gone.sum(), n))
    assert got == dict(cloned=c, split=sp, pruned=int(gone.sum()), rows=int(keep.sum())) and (c > 10 or all_split) and sp > 10
    assert 10 < gone.sum() < n - 10
    da = a.download(moments=True)
    for k in KEYS:
        _same(da[k], db[k][keep], k)
    ma, mb = _moments(da, a.M), _moments(db, b.M)
    for key in ma:
        _same(ma[key], mb[key][keep], "moments %s" % (key,))
    assert a.sky_rows() == int(keep[:S].sum())
    a.close()
    b.close()


def test_allocation_failures_leave_everything_unchanged():
    from gaussian_lic_b200 import capi
    g, _ = small_scene(2000, W, H, 37, 3)
    m = _mapper(3, capacity=2048)
    m.initialize(g)
    _with_keyframes(m, 4)
    m.enable_densification()
    m.optimize([0, 1, 2, 3] * 2)
    p = capi.DensityParams(0.0, 0.01, 1.0, 0.001, 0, 0.0)
    k = capi.DensityCounts()
    assert capi.lib.glic_mapper_densify_and_prune(m._h, C.byref(p), 1, C.byref(k)) == 0 and k.rows > 2048
    fails = _fail_until_success(m, lambda: capi.lib.glic_mapper_densify_and_prune(m._h, C.byref(p), 0, None), "growing densify_and_prune")
    assert fails >= 2 and m.stats().num_gaussians == k.rows
    m.close()


def test_rejected_arguments_change_nothing():
    from gaussian_lic_b200 import capi
    m = _twin(1, False)
    m.optimize([0, 1])
    before, maxr = m.download(moments=True), m.screen_radii()
    nan, inf = float("nan"), float("inf")
    k = capi.DensityCounts()
    good = (0.0002, 0.01, 1.0, 0.005, 20, 0.1)
    bad = [(nan, 0.01, 1.0, 0.005, 20, 0.1), (0.0002, -1.0, 1.0, 0.005, 20, 0.1), (0.0002, 0.01, 0.0, 0.005, 20, 0.1),
           (0.0002, 0.01, 1.0, nan, 20, 0.1), (0.0002, 0.01, 1.0, -0.1, 20, 0.1), (0.0002, 0.01, 1.0, 1.5, 20, 0.1),
           (0.0002, 0.01, 1.0, 0.005, -1, 0.1), (0.0002, 0.01, 1.0, 0.005, 20, nan), (0.0002, 0.01, 1.0, 0.005, 20, inf),
           (0.0002, 0.01, 1.0, 0.005, 20, -0.1), (0.0002, 0.01, 1.0, 1.0, 0, 0.0)]       # the last removes every row
    for args in bad:
        for dry in (0, 1):
            assert capi.lib.glic_mapper_densify_and_prune(m._h, C.byref(capi.DensityParams(*args)), dry, C.byref(k)) == -1, (args, dry)
    assert capi.lib.glic_mapper_densify_and_prune(m._h, None, 0, None) == -1
    sched = capi.DensitySchedule(1, 10, 0, 0, 0.0002, 0.01, 0.005, 0.01, 20, 0.1, 0.0)                   # densify_interval 0
    assert capi.lib.glic_mapper_set_density_schedule(m._h, C.byref(sched)) == -1
    sched.densify_interval, sched.reset_opacity = 1, 1.0
    assert capi.lib.glic_mapper_set_density_schedule(m._h, C.byref(sched)) == -1
    after = m.download(moments=True)
    for key in before:
        _same(after[key], before[key], "a rejected call changed %s" % key)
    assert np.array_equal(m.screen_radii(), maxr)
    plain = _mapper(1)
    assert capi.lib.glic_mapper_densify_and_prune(plain._h, C.byref(capi.DensityParams(*good)), 1, C.byref(k)) == -1   # not enabled
    assert capi.lib.glic_mapper_set_density_schedule(plain._h, C.byref(capi.DensitySchedule(1, 10, 1, 0, 0.0002, 0.01, 0.005, 0.01, 20, 0.1, 0.0))) == -1
    assert capi.lib.glic_mapper_screen_radii(plain._h, maxr.ctypes.data_as(C.c_void_p)) == -1
    plain.close()
    m.close()


# ---- 4. the schedule ------------------------------------------------------------------------------------------------------
SCHED = dict(densify_from=1, densify_until=9, densify_interval=3, opacity_reset_interval=4, grad_threshold=0.0, min_opacity=0.005,
             reset_opacity=0.01, screen_radius=6, world_scale_factor=0.03, scene_extent=0.0)


def test_schedule_equals_host_calls():
    """A mapper with a schedule and a twin whose host calls densify_and_prune / reset_opacity after the same iterations (zero
    learning rates, threshold 0: the selection does not depend on the gradients).  Parameters, n_sky and the screen radii
    are bit-identical, the totals are the twin's counts, the derived extent is scene_extent() and NumPy's."""
    from gaussian_lic_b200 import mapper
    g, _ = small_scene(1500, W, H, 41, 3)
    ms = []
    for sched in (True, False):
        m = _mapper(3, views_per_rank=2, **ZERO_LR)
        m.initialize(g)
        _with_keyframes(m)
        m.enable_densification()
        if sched:
            m.set_density_schedule(**SCHED)
        ms.append(m)
    a, b = ms
    centres = np.stack([np.float32(t) for _, t in _poses()])
    extent = a.scene_extent()
    assert extent == b.scene_extent() == dco.scene_extent(centres) > 0
    batches = VIEWS * 2                                            # 8 iterations of 2 views
    a.optimize(batches)
    total, steps, resets = dict(cloned=0, split=0, pruned=0, rows=0), 0, 0
    for n in range(1, 9):
        b.optimize(batches[2 * (n - 1):2 * n])
        densify, sizes, reset = dco.schedule_step(n, **SCHED)
        if densify:
            ext = b.scene_extent()
            got = b.densify_and_prune(ext, grad_threshold=0.0, percent_dense=mapper.PERCENT_DENSE, min_opacity=SCHED["min_opacity"],
                                      max_screen_radius=SCHED["screen_radius"] if sizes else 0,
                                      max_world_scale=float(np.float32(SCHED["world_scale_factor"]) * np.float32(ext)) if sizes else 0.0)
            print("n = %d: %s (size tests %s)" % (n, got, sizes))
            for key in ("cloned", "split", "pruned"):
                total[key] += got[key]
            total["rows"] = got["rows"]
            steps += 1
        if reset:
            b.reset_opacity(SCHED["reset_opacity"])
            resets += 1
    assert (steps, resets) == (2, 2)
    tot = a.density_totals()
    assert tot == dict(total, steps=steps, resets=resets) and total["pruned"] > 0, (tot, total)
    da, db = a.download(), b.download()
    for k in KEYS:
        _same(da[k], db[k], k)
    assert a.sky_rows() == b.sky_rows() and a.stats().iterations == b.stats().iterations == 8
    assert np.array_equal(a.screen_radii(), b.screen_radii())
    a.clear_density_schedule()
    assert a.density_totals() == dict(cloned=0, split=0, pruned=0, rows=0, steps=0, resets=0)
    a.optimize(batches[:6])                                        # n = 9..11: no schedule, no step
    assert a.density_totals()["steps"] == 0 and a.stats().num_gaussians == tot["rows"]
    for m in ms:
        m.close()


def test_single_keyframe_skips_the_densify_step():
    g, _ = small_scene(1500, W, H, 43, 1)
    m = _mapper(1, views_per_rank=1)
    m.initialize(g)
    _with_keyframes(m, 1)
    m.enable_densification()
    m.set_density_schedule(**dict(SCHED, densify_until=7))
    assert m.scene_extent() == 0.0
    m.optimize([0] * 6)
    acc, den = m.densify_stats()
    tot = m.density_totals()
    assert tot["steps"] == 0 and tot["resets"] == 1 and m.stats().num_gaussians == 1500
    assert den.max() == 6 and m.screen_radii().any(), "a skipped step restarted the statistics"
    m.close()


# ---- 5. quality, end to end -----------------------------------------------------------------------------------------------
C0 = 0.28209479177387814
WALL_VIEWS = list(range(12))
TRAIN = [v for v in WALL_VIEWS if v % 4 != 3]


def _wall_scene():
    """the textured wall of test_gpu_densify.py rendered from the 12-view rig, and its 300-row under-seeded map"""
    from gaussian_lic_b200 import mapper, model, ops, synthetic as syn
    dev = torch.device("cuda:0")
    tm, tls, trot = _wall(0.06, 0.04, 0.004, jitter_seed=1)
    n = tm.shape[0]
    truth = dict(means=tm, log_scales=tls, rots=trot, opacity_logits=np.full(n, 4.0, np.float32),
                 dc=((_texture(tm[:, 0], tm[:, 1]) - 0.5) / C0).astype(np.float32), sh=np.zeros((n, 0, 3), np.float32), degree=0)
    mdl = model.PackedModel(truth, dev)
    mdl.activate()
    rast = ops.CRasterizer(W, H, dev)
    poses = [syn.orbit_pose(v, n_views=12, radius=1.5) for v in WALL_VIEWS]
    imgs = []
    for R, t in poses:
        color, _, _ = rast.forward(mdl.inputs, rast.make_view(mapper.camera_block(W, H, F, F, W / 2.0, H / 2.0, R, t)))
        torch.cuda.synchronize()
        imgs.append(np.clip(color.cpu().numpy(), 0, 1).astype(np.float32))
    sm, sls, srot = _wall(1.0, 0.6, 0.05)
    k = sm.shape[0]
    seed_map = dict(means=sm, log_scales=sls, rots=srot, opacity_logits=np.zeros(k, np.float32), dc=np.zeros((k, 3), np.float32),
                    sh=np.zeros((k, 3, 3), np.float32))
    return poses, imgs, seed_map


def _wall_mapper(poses, imgs, seed_map, schedule):
    from gaussian_lic_b200 import mapper
    m = mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=1, seed=SEED, views_per_rank=2)
    m.initialize(seed_map)
    for v in WALL_VIEWS:
        m.add_keyframe(*poses[v], imgs[v], train=v in TRAIN)
    if schedule is not None:
        m.enable_densification()
        m.set_density_schedule(**schedule)
    return m


def _held_out_psnr(m):
    return float(np.mean([m.evaluate(i, train=False)[0] for i in range(len(WALL_VIEWS) - len(TRAIN))]))


ROUNDS = 16                                                       # 80 iterations of 2 views each
WALL_SCHEDULE = dict(densify_from=0, densify_until=1000, densify_interval=160, opacity_reset_interval=0, scene_extent=10.0)


def _train_rounds(m):
    rng = np.random.default_rng(0)
    for it in range(ROUNDS):
        m.optimize([int(x) for x in rng.permutation(np.tile(np.arange(len(TRAIN)), 18))[:160]])


def test_schedule_adds_detail_to_an_under_seeded_wall():
    """test_gpu_densify.py's under-seeded wall: the schedule (a densify every 160 iterations) against no density control"""
    poses, imgs, seed_map = _wall_scene()
    psnr = {}
    for arm, sched in (("plain", None), ("scheduled", WALL_SCHEDULE)):
        m = _wall_mapper(poses, imgs, seed_map, sched)
        _train_rounds(m)
        psnr[arm] = _held_out_psnr(m)
        psnr[arm + "_rows"] = m.stats().num_gaussians
        if sched:
            psnr["totals"] = m.density_totals()
        m.close()
    print("held-out PSNR: %s, gap %.2f dB" % (psnr, psnr["scheduled"] - psnr["plain"]))
    assert psnr["scheduled"] > psnr["plain"] + 3.0, psnr


def test_size_tests_remove_a_floater():
    """A large opaque bar floating in front of the wall that the ground truth does not have, its largest scale 6 against
    0.1 * extent = 1.0 (a split halves it to 3.75).  The size tests switch on after the opacity-reset interval (100
    iterations; the reset value 0.99 leaves the wall alone): the scheduled run still has the floater just before its step at
    160 and none of it after, while the run that only densifies (no reset, no size tests) still has it.  The held-out PSNRs are
    printed: right after the step the scheduled run scores lower (the wall behind the floater has not trained yet), and after
    the full budget the two runs agree within run-to-run noise (gradient descent fades the floater in the other run too), so
    no PSNR order is asserted."""
    poses, imgs, seed_map = _wall_scene()
    fl = dict(means=np.float32([[0.0, -1.5, 7.0]]), log_scales=np.log(np.float32([[6.0, 0.3, 0.05]])), rots=np.float32([[1, 0, 0, 0]]),
              opacity_logits=np.float32([8.0]), dc=np.float32([[2.0, -1.5, 1.0]]), sh=np.zeros((1, 3, 3), np.float32))
    floated = {k: np.concatenate([fl[k], np.asarray(seed_map[k], np.float32)]) for k in seed_map}
    limit = np.float32(0.1) * np.float32(10.0)

    def big(m):
        s, _ = _activate(m.download())
        return int((s.max(1) > limit).sum())

    psnr = {}
    for arm, reset in (("densify only", 0), ("scheduled", 100)):
        m = _wall_mapper(poses, imgs, floated, dict(WALL_SCHEDULE, densify_interval=80, opacity_reset_interval=reset, reset_opacity=0.99))
        assert big(m) == 1
        m.optimize([i % len(TRAIN) for i in range(2 * 159)])
        assert m.stats().iterations == 159 and big(m) >= 1, "the floater is gone before the first sized step"
        m.optimize([0, 1])
        psnr[arm + " at 160"] = _held_out_psnr(m)
        psnr[arm + " floater rows at 160"] = big(m)
        _train_rounds(m)
        psnr[arm] = _held_out_psnr(m)
        psnr[arm + " totals"] = m.density_totals()
        m.close()
    print("held-out PSNR: %s" % psnr)
    assert psnr["densify only floater rows at 160"] >= 1 and psnr["scheduled floater rows at 160"] == 0, psnr


# ---- 6. two ranks on one GPU (gloo for the handles, as tests/test_gpu_densify.py) -----------------------------------------
P2 = 3000
SCHED2 = dict(densify_from=1, densify_until=6, densify_interval=2, opacity_reset_interval=3, grad_threshold=0.002, screen_radius=20)


def _run_rank(rank, world, exchange):
    from gaussian_lic_b200 import capi
    g, _ = small_scene(P2, W, H, 45, 3)
    m = _mapper(3, capacity=P2 + 512, rank=rank, world=world, views_per_rank=2 // world)
    m.initialize(g)
    _with_keyframes(m, 4)
    m.enable_densification()
    if exchange:
        m.connect(exchange(m.export_handle()))
    m.optimize([0, 1])
    res = dict(first=m.screen_radii())
    if world == 1:
        return m, res
    m.set_density_schedule(**SCHED2)
    m.optimize([2, 3, 1, 2, 0, 3, 1, 0, 2, 1])
    res.update(trained=m.download(moments=True), stats=m.densify_stats(), radii=m.screen_radii(), totals=m.density_totals())
    m.clear_density_schedule()
    m.optimize([0, 1, 2, 3])
    _, _, act = _activate(m.download(), opacity=True)
    res["over"] = capi.lib.glic_mapper_densify(m._h, 0.0, 0.01, 1e-6, 0, None, None)        # every row splits: twice the rows
    p = capi.DensityParams(0.0, 0.01, 1e-6, float(np.float32(np.median(act))), 0, 0.0)
    k = capi.DensityCounts()
    res["dry"] = capi.lib.glic_mapper_densify_and_prune(m._h, C.byref(p), 1, C.byref(k)), dict(rows=k.rows, pruned=k.pruned)
    res["fused"] = capi.lib.glic_mapper_densify_and_prune(m._h, C.byref(p), 0, C.byref(k)), dict(rows=k.rows, pruned=k.pruned)
    res["capacity"] = m.stats().capacity
    res["final"] = m.download(moments=True)
    return m, res


def _worker(rank, world, port, q):
    try:
        import torch.distributed as dist
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
        torch.cuda.set_device(rank % torch.cuda.device_count())

        def exchange(mine):
            got = [None] * world
            dist.all_gather_object(got, mine)
            return got

        m, res = _run_rank(rank, world, exchange)
        dist.barrier()
        m.close()
        dist.destroy_process_group()
        q.put((rank, "ok", res))
    except Exception as e:          # noqa: BLE001 - reported to the parent
        import traceback
        q.put((rank, "%r\n%s" % (e, traceback.format_exc()), None))


@pytest.mark.timeout(300)
def test_two_ranks_keep_identical_replicas_under_a_schedule():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p_ in procs:
        p_.start()
    res = sorted([q.get(timeout=240) for _ in procs], key=lambda r: r[0])
    for p_ in procs:
        p_.join(timeout=30)
    assert all(r[1] == "ok" for r in res), [r[1] for r in res]
    a, b = res[0][2], res[1][2]
    print("totals %s; refused densify %d, fused %s of capacity %d" % (a["totals"], a["over"], a["fused"], a["capacity"]))
    assert a["totals"] == b["totals"] and a["totals"]["steps"] == 2 and a["totals"]["resets"] == 1
    assert np.array_equal(a["first"], b["first"]) and np.array_equal(a["radii"], b["radii"])
    for i in range(2):
        _same(a["stats"][i], b["stats"][i], "replicas' statistics differ")
    for name in a["trained"]:
        _same(a["trained"][name], b["trained"][name], "replicas differ under the schedule in %s" % name)
        _same(a["final"][name], b["final"][name], "replicas differ after the fused call in %s" % name)
    assert a["over"] == b["over"] == -2
    assert a["dry"] == b["dry"] and a["dry"][0] == 0 and a["dry"][1]["rows"] <= a["capacity"]
    assert a["fused"] == b["fused"] == (0, a["dry"][1])
    # the same first batch on one rank with views_per_rank = 2: the same radii, exactly
    m, one = _run_rank(0, 1, None)
    m.close()
    assert np.array_equal(one["first"], a["first"]) and a["first"].any()
