"""The density-control restatement (tests/density_control_oracle.py) on hand cases, and the C entry points' symbols and the
arguments they reject without a GPU."""
import ctypes as C

import numpy as np
import pytest

import density_control_oracle as dco

INRIA = dict(densify_from=500, densify_until=15000, densify_interval=100, opacity_reset_interval=3000)


def _fused(cls, **kw):
    P = len(cls)
    base = dict(act=np.full(P, 0.5, np.float32), smax=np.full(P, 0.1, np.float32), smax_child=np.full(P, 0.05, np.float32),
                maxr=np.zeros(P, np.int32), n_sky=0)
    base.update(kw)
    return dco.densify_and_prune(np.asarray(cls), **base)


def test_nothing_removed_is_densify():
    """min_opacity 0 and both size tests off: the densify result itself, in Inria's order"""
    r = _fused([0, 1, 2, 0, 2, 1])
    assert r["src"].tolist() == [0, 1, 3, 5, 1, 5, 2, 4, 2, 4]
    assert r["row"].tolist() == list(range(10)) and r["pruned"] == 0 and r["rows"] == 10
    assert (r["cloned"], r["split"], r["kept"], r["children"]) == (2, 2, 4, 4)


def test_predicate_keeps_result_order_and_prepruning_child_keys():
    # rows: 0 keep, 1 clone, 2 split, 3 keep (faint), 4 split (faint: both children go), 5 clone, 6 split
    cls = [0, 1, 2, 0, 2, 1, 2]
    act = np.array([0.5, 0.5, 0.5, 0.001, 0.001, 0.5, 0.5], np.float32)
    r = _fused(cls, act=act, min_opacity=0.005)
    # unpruned: kept 0 1 3 5 | clones 1 5 | first children 2 4 6 | second children 2 4 6  (rows 0..11)
    assert r["unpruned_src"].tolist() == [0, 1, 3, 5, 1, 5, 2, 4, 6, 2, 4, 6]
    assert r["src"].tolist() == [0, 1, 5, 1, 5, 2, 6, 2, 6]
    assert r["row"].tolist() == [0, 1, 3, 4, 5, 6, 8, 9, 11]       # the children keep their unpruned rows as keys
    assert (r["pruned"], r["rows"], r["kept"], r["children"]) == (3, 9, 3, 4)


def test_size_tests_judge_each_row_by_its_own_values():
    cls = [0, 0, 1, 2, 2, 0]
    smax = np.array([0.1, 2.0, 2.0, 2.0, 1.2, 2.0], np.float32)
    child = np.array([0.06, 1.25, 1.25, 1.25, 0.75, 1.25], np.float32)
    maxr = np.array([30, 5, 30, 30, 30, 50], np.int32)
    # unpruned: kept 0 1 2 5 | clone of 2 | first children 3 4 | second children 3 4; only 4's children are small enough
    r = _fused(cls, smax=smax, smax_child=child, maxr=maxr, n_sky=0, max_screen_radius=20, max_world_scale=1.0)
    assert r["src"].tolist() == [4, 4]                              # only the children of 4 (scale 0.75) survive
    r = _fused(cls, smax=smax, smax_child=child, maxr=maxr, max_screen_radius=20)
    assert r["src"].tolist() == [1, 2, 3, 4, 3, 4]                  # rows 0, 2 and 5 exceed the radius; the clone of 2 has maxr 0
    assert r["row"].tolist() == [1, 4, 5, 6, 7, 8]
    # the boundaries: strictly greater
    assert _fused([0], smax=np.float32([1.0]), max_world_scale=1.0)["rows"] == 1
    assert _fused([0], smax=np.float32([np.nextafter(np.float32(1), np.float32(2))]), max_world_scale=1.0)["rows"] == 0
    assert _fused([0], maxr=np.int32([20]), max_screen_radius=20)["rows"] == 1
    assert _fused([0], maxr=np.int32([21]), max_screen_radius=20)["rows"] == 0


def test_sky_rows_go_by_opacity_only():
    cls = [0, 0, 0, 2]
    act = np.array([0.001, 0.5, 0.5, 0.5], np.float32)
    r = _fused(cls, act=act, n_sky=3, min_opacity=0.01, maxr=np.int32([99, 99, 99, 0]), smax=np.float32([9, 9, 9, 0.1]),
               max_screen_radius=5, max_world_scale=1.0)
    assert r["src"].tolist() == [1, 2, 3, 3] and r["sky"] == 2
    nan = _fused([0], act=np.float32([np.nan]), min_opacity=1.0)
    assert nan["rows"] == 1                                         # as prune: a NaN opacity stays


def test_schedule_triggers():
    on = [n for n in range(0, 16001) if dco.schedule_step(n, **INRIA)[0]]
    assert on[0] == 600 and on[-1] == 14900 and len(on) == 144
    assert dco.schedule_step(500, **INRIA) == (False, False, False)  # densify_from < n, strictly
    assert dco.schedule_step(3000, **INRIA) == (True, False, True)   # the size tests need n > opacity_reset_interval
    assert dco.schedule_step(3100, **INRIA) == (True, True, False)
    assert dco.schedule_step(15000, **INRIA) == (False, False, False)
    assert [n for n in range(1, 16001) if dco.schedule_step(n, **INRIA)[2]] == [3000, 6000, 9000, 12000]
    never = dict(INRIA, opacity_reset_interval=0)
    assert dco.schedule_step(3100, **never) == (True, False, False) and not any(dco.schedule_step(n, **never)[2] for n in range(1, 16001))


def test_scene_extent_hand_cases():
    assert dco.scene_extent(np.zeros((0, 3))) == 0
    assert dco.scene_extent([[1.0, 2.0, 3.0]]) == 0                  # one keyframe
    assert dco.scene_extent([[1.0, 2.0, 3.0]] * 4) == 0              # all at one place
    assert dco.scene_extent([[0, 0, 0], [2, 0, 0]]) == np.float32(1.1)
    assert dco.scene_extent([[0, 0, 0], [3, 4, 0], [0, 0, 0], [0, 0, 0]]) == np.float32(1.1 * np.hypot(2.25, 3.0))
    rng = np.random.default_rng(3)
    c = rng.normal(size=(50, 3)) * 4
    want = 1.1 * np.max(np.linalg.norm(c - c.mean(0), axis=1))     # Inria's getNerfppNorm
    assert abs(float(dco.scene_extent(c)) - want) <= 1e-6 * want
    assert dco.reset_logit(0.01) == np.float32(np.log(0.01 / 0.99))


def test_new_symbols_and_rejections_without_gpu():
    from gaussian_lic_b200 import capi, mapper
    lib = capi.lib
    for name in ("glic_mapper_screen_radii", "glic_mapper_reset_opacity", "glic_mapper_densify_and_prune", "glic_mapper_set_density_schedule",
                 "glic_mapper_scene_extent", "glic_mapper_density_totals"):
        assert name in capi.SYMBOLS and hasattr(lib, name)
    assert C.sizeof(capi.DensityParams) == 24 and C.sizeof(capi.DensityCounts) == 16 and C.sizeof(capi.DensitySchedule) == 44
    out = (C.c_int32 * 4)()
    f = C.c_float()
    p = capi.DensityParams(0.0002, 0.01, 1.0, 0.005, 20, 0.1)
    k = capi.DensityCounts()
    s = capi.DensitySchedule(**mapper.DENSITY_SCHEDULE)
    assert lib.glic_mapper_screen_radii(None, out) == -1
    assert lib.glic_mapper_reset_opacity(None, 0.01) == -1
    assert lib.glic_mapper_densify_and_prune(None, C.byref(p), 0, C.byref(k)) == -1
    assert lib.glic_mapper_set_density_schedule(None, C.byref(s)) == -1
    assert lib.glic_mapper_scene_extent(None, C.byref(f)) == -1
    assert lib.glic_mapper_density_totals(None, None, None, None) == -1
    assert b"null" in lib.glic_last_error()
    assert mapper.DENSITY_SCHEDULE["min_opacity"] == float(np.float32(0.005)) and mapper.RESET_OPACITY == float(np.float32(0.01))


def test_python_schedule_rejects_unknown_fields():
    from gaussian_lic_b200 import mapper
    with pytest.raises(TypeError):
        mapper.Mapper.set_density_schedule(object(), screen_radii=20)
