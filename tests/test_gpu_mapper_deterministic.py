"""The native mapper's GLIC_MAPPER_OPT_DETERMINISTIC option (Mapper.set_deterministic): the deterministic render backward and the
fixed-order loss and evaluation sums inside optimize, align, evaluate and render.

* Twin mappers from one initialisation, trained with real learning rates, exposure, pose refinement, a density schedule that
  densifies, prunes and resets opacity within the run, and two views per step, return identical bits from every getter; so do
  twins fed through add_frame, and twins started from a binning capacity too small for the first frames.
* The option's growth follows the failure contract: failing each of its allocations returns GLIC_ERR_CUDA and changes nothing.
* With the option on, a step still meets the float64-oracle criteria of test_gpu_mapper_grads.py."""
import os

import numpy as np
import pytest

from test_gpu_densify import F, SEED, VIEWS, _lidar_scan, _poses, _same, _with_keyframes

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

W, H = 320, 208
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LPIPS = os.path.join(ROOT, "oracle", "_ref", "lpips_alex.bin")
SCHED = dict(densify_from=1, densify_until=20, densify_interval=5, opacity_reset_interval=12, grad_threshold=0.0002,
             min_opacity=0.005, reset_opacity=0.01, screen_radius=20, world_scale_factor=0.1, scene_extent=0.0)
STAT_FIELDS = ("num_gaussians", "capacity", "iterations", "last_inserted", "last_loss", "mean_visible", "overflow_regrows")


def _twin(binning_pairs=None, deterministic=True):
    from gaussian_lic_b200 import mapper
    pts, cols, dep = _lidar_scan(3000, 5, *_poses([0])[0])
    m = mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=3, capacity=3500, seed=SEED, views_per_rank=2)
    m.initialize_lidar(pts, cols, dep, F, 500, 1000)
    _with_keyframes(m)
    m.enable_exposure(0.001)
    m.enable_pose_refinement(1e-3, 1e-3)
    m.enable_densification()
    m.set_density_schedule(**SCHED)
    if binning_pairs:
        m.set_binning_pairs(binning_pairs)
    if deterministic:
        m.set_deterministic(True)
    if os.path.isfile(LPIPS):
        m.load_lpips(LPIPS)
    return m


def _train(m, steps=30):
    for i in range(steps):
        m.optimize([VIEWS[(2 * i) % 8], VIEWS[(2 * i + 1) % 8]])


def _getters(m):
    """every getter of the option's guarantee, as a flat dict of arrays"""
    out = {"map." + k: v for k, v in m.download(moments=True).items()}
    out["accum"], out["denom"] = m.densify_stats()
    out["maxr"] = np.asarray(m.screen_radii())
    out["sky_rows"] = np.asarray([m.sky_rows()])
    st = m.stats()
    for f in STAT_FIELDS:
        out["stats." + f] = np.asarray([getattr(st, f)], np.float64)
    for k, v in m.density_totals().items():
        out["totals." + k] = np.asarray(v, np.float64)
    n_kf = len(VIEWS)
    for i in range(n_kf):
        R, t = m.pose(i)
        out["pose%d" % i] = np.concatenate([np.ravel(R), np.ravel(t)])
        out["pose_state%d" % i] = np.concatenate([np.ravel(np.asarray(x, np.float64)) for x in m.pose_state(i)])
        out["E%d" % i] = np.ravel(m.exposure(i))
        out["E_state%d" % i] = np.concatenate([np.ravel(np.asarray(x, np.float64)) for x in m.exposure_state(i)])
    for i in (0, 5):
        out["evaluate%d" % i] = np.asarray(m.evaluate(i), np.float32)
        if os.path.isfile(LPIPS):
            out["lpips%d" % i] = np.asarray(m.evaluate_lpips(i), np.float32)
        out["render%d" % i] = np.asarray(m.render(i), np.float32)
    R, t = _poses([2])[0]
    for k, v in m.render_camera(R, t, exposure=1).items():
        out["render_camera." + k] = v
    return out


def _align(m):
    a = m.align(3, train=True, iterations=20, exposure_lr=0.01, image=True)
    return {"align." + k: np.asarray(v, np.float64 if k in ("steps", "skipped") else np.float32) for k, v in a.items()}


def _same_all(a, b, what):
    assert set(a) == set(b), what
    for k in a:
        x, y = np.asarray(a[k]), np.asarray(b[k])
        if x.dtype == np.float64:
            assert np.array_equal(x, y), "%s: %s" % (what, k)
        else:
            _same(x, y, "%s: %s" % (what, k))


def test_twins_train_bit_identically():
    a, b = _twin(), _twin()
    _train(a)
    _train(b)
    ga, gb = _getters(a), _getters(b)
    tot = a.density_totals()
    print("totals", tot, "rows", a.stats().num_gaussians)
    assert tot["steps"] >= 2 and tot["resets"] >= 1
    assert tot["cloned"] + tot["split"] > 0 and tot["pruned"] > 0, tot
    _same_all(ga, gb, "twins after 30 steps")
    _same_all(_align(a), _align(b), "align")
    a.close()
    b.close()


def test_twins_after_binning_overflow():
    """twins started from a binning capacity far below the first frame's pairs skip that frame, regrow, and stay identical"""
    a, b = _twin(binning_pairs=2000), _twin(binning_pairs=2000)
    _train(a, 12)
    _train(b, 12)
    assert a.stats().overflow_regrows > 0
    _same_all(_getters(a), _getters(b), "overflow twins")
    a.close()
    b.close()


def test_twins_fed_through_add_frame():
    from test_gpu_frames import FX, FY, RADIUS, SKY, _frames, _padded
    from gaussian_lic_b200 import mapper
    frames = _frames(10, 20_000, 2)
    ms = []
    for _ in range(2):
        m = mapper.Mapper(W, H, FX, FY, W / 2.0, H / 2.0, sh_degree=3, seed=17)
        m.enable_frames(5, SKY, RADIUS)
        m.set_deterministic(True)
        for f in frames:
            m.add_frame(f["q"], f["t"], _padded(f["bgr"]), f["xyz"], f["rgb"])
        for _ in range(10):
            m.optimize([0])
            m.optimize([1])
        ms.append(m)
    a, b = ms
    da, db = a.download(moments=True), b.download(moments=True)
    for k in da:
        _same(da[k], db[k], "add_frame twins: %s" % k)
    assert a.stats().last_loss == b.stats().last_loss
    assert a.evaluate(0) == b.evaluate(0) and a.evaluate(0, train=False) == b.evaluate(0, train=False)
    for m in ms:
        m.close()


def test_option_growth_follows_the_failure_contract():
    from gaussian_lic_b200 import capi
    m = _twin(deterministic=False)
    _train(m, 2)
    before = m.download(moments=True)
    st = m.stats()
    failed = 0
    for k in range(1, 10):
        capi.check(capi.lib.glic_debug_fail_allocation(k), "debug_fail_allocation")
        rc = capi.lib.glic_mapper_set_option(m._h, 3, 1)
        capi.check(capi.lib.glic_debug_fail_allocation(0), "debug_fail_allocation")
        if rc == 0:
            break
        assert rc == -3, (k, rc)
        failed += 1
        now = m.download(moments=True)
        for key in before:
            _same(now[key], before[key], "allocation %d: %s" % (k, key))
        assert m.stats().num_gaussians == st.num_gaussians and m.stats().capacity == st.capacity
    assert failed >= 1
    # the growth of the capacity with the option on: binning, sample and deterministic workspaces in one growth
    for k in range(1, 10):
        capi.check(capi.lib.glic_debug_fail_allocation(k), "debug_fail_allocation")
        rc = capi.lib.glic_mapper_set_option(m._h, 2, 4_000_000)
        capi.check(capi.lib.glic_debug_fail_allocation(0), "debug_fail_allocation")
        if rc == 0:
            break
        assert rc == -3, (k, rc)
        now = m.download(moments=True)
        for key in before:
            _same(now[key], before[key], "capacity growth, allocation %d: %s" % (k, key))
    assert k > 3                                             # three buffers, each failed once before the growth went through
    _train(m, 2)
    m.close()


def test_step_meets_the_oracle_criteria(oracle32, oracle64):
    from test_gpu_mapper_grads import _check_step_against_oracle, _keyframes, _mapper, _scene, _state
    raw = _scene(3)
    poses, cams, gts = _keyframes(seed=11)
    m = _mapper(raw, poses, gts, views_per_rank=2)
    m.set_deterministic(True)
    before = _state(m)
    m.optimize([0, 1])
    after = _state(m)
    _check_step_against_oracle(m, raw, before, after, cams, gts, [0, 1], (oracle64, oracle32), "deterministic, views [0, 1]")
    m.close()
