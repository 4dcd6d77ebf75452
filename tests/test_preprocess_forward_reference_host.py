"""Checks of tests/preprocess_forward_reference.py itself, on the CPU: its decisions and values against the float64 C oracle's
forward (oracle64.state()), the float32 oracle's values within its bounds and its integer outputs and accept sets equal outside
the band rows, the kernel's hy above the float64 half-height, and each plausible kernel bug of
preprocess_forward_reference.MUTATIONS, applied to the restatement, moving some element of these scenes beyond its bound."""
import functools

import numpy as np
import pytest

import preprocess_forward_reference as pfr
from helpers import POSES
from preprocess_backward_reference import MAG32, MAG64
from test_preprocess_backward_reference_host import _syn, cams

FLOATS = ("depth", "xy", "conic", "rgb")
# (scene, SH degree, SH degree of the tensor, pose): small_scene at degrees 0-3, a degree-1 forward of a degree-3 tensor
# (M = 15 > 3), every stress scene
CASES = ([("small", d, d, POSES[1 + d]) for d in range(4)] + [("small", 1, 3, POSES[3])] +
         [(k, 2, 2, POSES[0]) for k in ("needles", "big", "deep", "ties", "edges")])
IDS = ["%s-d%d-m%d-v%d" % (k, d, m, p[0]) for k, d, m, p in CASES]


# Band rows of each stress case (kind, view, principal-point offset): the largest count measured over the float32 and float64
# oracles' records and an H100's (sm_90a).  These scenes are built to put rows on thresholds: the needles' 2-D covariances
# cancel, so that the float64 chain cannot decide the tile tests (hence the visibility) of up to 28% of their rows; the edges
# scene puts rows on the lim* clamps and the near cull; the deep scene's rig views stack thousands of splats on tile borders.
STRESS_BAND_ROWS = {("needles", 0, (0.0, 0.0)): 704, ("needles", 3, (0.0, 0.0)): 1101, ("needles", 5, (17.5, -9.25)): 1146,
                    ("big", 0, (0.0, 0.0)): 51, ("big", 0, (-23.0, 11.5)): 51, ("big", 1, (0.0, 0.0)): 50,
                    ("deep", 0, (0.0, 0.0)): 35, ("deep", 5, (17.5, -9.25)): 67, ("deep", 3, (0.0, 0.0)): 83,
                    ("ties", 0, (0.0, 0.0)): 12, ("ties", 0, (-23.0, 11.5)): 12,
                    ("edges", 0, (0.0, 0.0)): 125, ("edges", 0, (-23.0, 11.5)): 119, ("edges", 5, (17.5, -9.25)): 55}
# rows a pinned count may grow by: a decision quantity within a few ulp of the band's edge, where numpy's float64 log / exp /
# sqrt may round differently from one machine to the next
BAND_SLACK = 4


def band_limit(kind, P, view=0, pp=(0.0, 0.0)):
    """the band rows a case may have: a stress case its pinned count, any other scene 1% of its rows (at least 16)"""
    pinned = STRESS_BAND_ROWS.get((kind, view, tuple(float(x) for x in pp)))
    return pinned + BAND_SLACK if pinned is not None else max(16, 0.01 * P)


def scene_of(kind, deg, mdeg, view, pp):
    syn = _syn()
    if kind == "small":
        W, H, f = 320, 208, 250.0
        g = syn.make_gaussians(3000, W, H, f, f, sh_degree=mdeg, zmax=12.0, seed=11, log_scale_mean=-3.0)
        R_wc, t_wc = syn.orbit_pose(view, radius=2.0)
        cam = syn.make_camera(W, H, f, f, W / 2.0 + pp[0], H / 2.0 + pp[1], R_wc, t_wc)
    else:
        g, cam = syn.make_stress_scene(kind, view=view, pp=pp, deg=mdeg)
    g["degree"] = deg
    return g, cam


@functools.lru_cache(maxsize=None)
def scene(i):
    from oracle.oracle import Oracle
    kind, deg, mdeg, (view, pp) = CASES[i]
    g, cam = scene_of(kind, deg, mdeg, view, pp)
    out = {}
    for name, dt in (("f64", np.float64), ("f32", np.float32)):
        o = Oracle(dt)
        f = o.forward(g, cam)
        st = o.state(f)
        st["radii"] = f["radii"].copy()
        o.free(f)
        out[name] = st
    return g, cam, out


def pairs_of(st, T):
    return np.sort(st["point_list"].astype(np.int64) * T + (st["keys_sorted"] >> 32).astype(np.int64))


def run(i, A=MAG32, **kw):
    g, cam, _ = scene(i)
    c32, c64 = cams(cam)
    return pfr.forward(g, c64 if A is MAG64 else c32, A=A, **kw)


def _check(i, which, A):
    g, cam, sts = scene(i)
    st = sts[which]
    ref = run(i, A)
    got = dict(radius=st["radii"], tiles=st["tiles_touched"], clamped=st["clamped"], pairs=pairs_of(st, ref["T"]))
    rec = pfr.record_accept_sets(st["xy"], st["conic_opacity"], st["radii"], cam["W"], cam["H"], A=A)
    bad, rows = pfr.compare(ref, got, rec)
    vis = (st["tiles_touched"] > 0) & ref["vis"]
    got_f = dict(depth=st["depth"], xy=st["xy"], conic=st["conic_opacity"][:, :3], rgb=st["rgb"])
    return ref, bad, rows, vis, got_f


@pytest.mark.parametrize("i", range(len(CASES)), ids=IDS)
def test_matches_float64_oracle(i):
    ref, bad, rows, vis, got = _check(i, "f64", MAG64)
    r = {k: pfr.ratio(got[k], ref[k], 1.0, vis) * pfr.U for k in FLOATS}     # |oracle - v| / m
    print("%s: max |oracle - v| / m %s  band rows %d  paths %s" % (IDS[i], r, rows.sum(), ref["paths"]))
    assert all(len(v) == 0 for v in bad.values()), {k: v[:8] for k, v in bad.items() if len(v)}
    assert max(r.values()) <= 1e-12, r
    assert rows.sum() <= band_limit(CASES[i][0], rows.size, *CASES[i][3]), rows.sum()


@pytest.mark.parametrize("i", range(len(CASES)), ids=IDS)
def test_float32_oracle_within_bounds(i):
    """the float32 oracle (the reference's arithmetic in float32, one rounding per operation) against the bounds, and its
    integer outputs and accept sets equal to the restatement's outside the band rows"""
    ref, bad, rows, vis, got = _check(i, "f32", MAG32)
    r = {k: pfr.ratio(got[k], ref[k], pfr.BOUND[k], vis) for k in FLOATS}
    print("%s: float32 oracle, max err / bound %s  band rows %d" % (IDS[i], {k: round(v, 3) for k, v in r.items()}, rows.sum()))
    assert all(len(v) == 0 for v in bad.values()), {k: v[:8] for k, v in bad.items() if len(v)}
    assert max(r.values()) <= 1.0, r
    assert rows.sum() <= band_limit(CASES[i][0], rows.size, *CASES[i][3]), rows.sum()
    assert ref["paths"]["visible"] > 0 and (CASES[i][1] == 0 or min(ref["paths"]["clamped"]) > 0)


@pytest.mark.parametrize("i", range(len(CASES)), ids=IDS)
def test_hy_covers_half_height(i):
    """the kernel's hy (in float32, from the float32 oracle's record) is at least the float64 half-height of each splat"""
    g, cam, sts = scene(i)
    st = sts["f32"]
    ref = run(i)
    vis = st["tiles_touched"] > 0
    need = pfr.half_height(st["conic_opacity"], ref["cov"], vis)
    hy = pfr.hy_f32(st["conic_opacity"], st["radii"])
    short = vis & ~(hy >= need)
    print("%s: min hy / half-height %.6f over %d splats" % (IDS[i], float(np.min((hy / np.where(need > 0, need, 1))[vis])),
                                                           vis.sum()))
    assert not short.any(), np.flatnonzero(short)[:8]


def _caught(i, mutation):
    """max err / bound of the mutated restatement against the bound of the unmutated one, per float output"""
    if mutation == "hy_without_margin":
        g, cam, sts = scene(i)
        st = sts["f32"]
        vis = st["tiles_touched"] > 0
        need = pfr.half_height(st["conic_opacity"], run(i)["cov"], vis)
        hy = pfr.hy_f32(st["conic_opacity"], st["radii"], mutate=mutation)
        return {"hy": float((vis & (hy < need)).sum())}        # > 1 when two or more splats fall short
    ref = run(i)
    mut = run(i, mutate=mutation)
    both = ref["vis"] & mut["vis"]
    return {k: pfr.ratio(mut[k].v, ref[k], pfr.BOUND[k], both) for k in FLOATS}


@pytest.mark.parametrize("mutation", pfr.MUTATIONS)
def test_mutation_is_caught(mutation):
    best = {}
    for i in range(len(CASES)):
        for k, v in _caught(i, mutation).items():
            if v > best.get(k, (0.0, ""))[0]:
                best[k] = (v, IDS[i])
    print("%s: max err / bound per output %s" % (mutation, {k: "%.3g (%s)" % v for k, v in best.items()}))
    assert max(v for v, _ in best.values()) > 1.0, (mutation, best)
