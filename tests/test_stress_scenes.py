"""The stress scenes (synthetic.make_stress_scene) still reach the paths they were built for.

Each scene targets a path of the rasterizer that synthetic.make_gaussians never reaches: the hy fallback of the render row
cull, span-arena exhaustion in the key emission, deep tiles of many forward rounds with dead buckets, depth ties across the
sorts, and the culls and clamps at the edges of the view.  These checks read the CPU oracle's state, so a later change to a
generator that turns a stress case into an easy one fails here, without a GPU.
"""
import numpy as np
import pytest

from gaussian_lic_b200 import synthetic as syn
from helpers import big_rect_rows, hy_fallbacks, tile_rects

STRESS_POSES = [(0, (0.0, 0.0)), (0, (-23.0, 11.5))]         # the identity pose, centred and with an off-centre principal point


def _forward(oracle32, kind, view, pp, **kw):
    g, cam = syn.make_stress_scene(kind, view=view, pp=pp, **kw)
    f = oracle32.forward(g, cam)
    st = oracle32.state(f)
    return g, cam, f, st


@pytest.mark.parametrize("view,pp", STRESS_POSES)
def test_needles_reach_the_hy_fallback(oracle32, view, pp):
    g, cam, f, st = _forward(oracle32, "needles", view, pp)
    vis = f["radii"] > 0
    n = hy_fallbacks(st["conic_opacity"], vis)
    ratio = g["scales"].max(1) / g["scales"].min(1)
    print("needles: %d visible, %d take the hy fallback" % (vis.sum(), n))
    assert n >= 500, n
    assert ratio.min() >= 99.0 and ratio.max() >= 5e3
    oracle32.free(f)


@pytest.mark.parametrize("view,pp", STRESS_POSES)
def test_big_overflows_the_span_arena(oracle32, view, pp):
    g, cam, f, st = _forward(oracle32, "big", view, pp)
    P = f["P"]
    rows = big_rect_rows(st["xy"], f["radii"], cam["W"], cam["H"])
    tiles = st["tiles_touched"][f["radii"] > 0]
    print("big: rows of big rects %d, arena %d, tiles per splat max %d" % (rows, 4 * P, tiles.max()))
    assert rows > 4 * P * 1.25, (rows, 4 * P)     # overflow part-way through, not at the first CTA nor never
    assert rows < 4 * P * 4
    assert tiles.max() >= 500 and (tiles >= 32).sum() >= 1000
    oracle32.free(f)


@pytest.mark.parametrize("opaque", [False, True], ids=["low", "high"])
def test_deep_stacks_many_rounds(oracle32, opaque):
    g, cam, f, st = _forward(oracle32, "deep", 0, (0.0, 0.0), opaque=opaque)
    rg = st["ranges"].astype(np.int64)
    cnt = rg[:, 1] - rg[:, 0]
    mc = st["max_contrib"].astype(np.int64)
    live = int(((mc + 31) // 32).sum())
    print("deep(%s): max %d splats per tile (%d rounds), B %d, live buckets %d, min T %.3e" % (
        "high" if opaque else "low", cnt.max(), (cnt.max() + 255) // 256, f["B"], live, f["final_T"].min()))
    assert cnt.max() >= 2000
    if opaque:
        assert ((mc < cnt // 2) & (cnt >= 512)).any()           # pixels of a deep tile saturate early
        assert live < 0.9 * f["B"]
        assert (f["final_T"] == 0).any() or f["final_T"].min() < 1e-3
    else:
        assert f["final_T"].min() > 1e-3                         # no pixel saturates: every round is blended
        assert live == f["B"]
    oracle32.free(f)


@pytest.mark.parametrize("view,pp", STRESS_POSES)
def test_ties_share_depths(oracle32, view, pp):
    g, cam, f, st = _forward(oracle32, "ties", view, pp)
    ks = st["keys_sorted"]
    equal = int((ks[1:] == ks[:-1]).sum())
    vis = f["radii"] > 0
    # exact duplicates: same parameters at different indices
    rows = np.concatenate([g["means"], g["scales"], g["rots"], g["opacity"][:, None]], 1)
    _, first = np.unique(rows, axis=0, return_index=True)
    print("ties: %d keys equal to their predecessor, %d duplicated Gaussians" % (equal, rows.shape[0] - first.size))
    assert equal >= 100
    assert rows.shape[0] - first.size >= 256 and vis.sum() >= 0.9 * f["P"]
    # depth = z exactly under the identity pose
    np.testing.assert_array_equal(st["depth"][vis].view(np.uint32), g["means"][vis, 2].view(np.uint32))
    oracle32.free(f)


def test_edges_reach_culls_and_clamps(oracle32):
    view, pp = 0, (-23.0, 11.5)
    g, cam, f, st = _forward(oracle32, "edges", view, pp)
    W, H = cam["W"], cam["H"]
    vis = f["radii"] > 0
    z, o = g["means"][:, 2], g["opacity"]
    lims = cam["lims"]
    tx, ty = g["means"][:, 0] / z, g["means"][:, 1] / z
    x0, y0, x1, y1 = tile_rects(st["xy"], f["radii"], W, H)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    near = (z > np.float32(0.2)) & (z <= np.float32(0.25))
    outside = (tx < lims[0]) | (tx > lims[1]) | (ty < lims[2]) | (ty > lims[3])
    counts = dict(near_visible=int((near & vis).sum()), at_cull_visible=int((vis & (z <= np.float32(0.2))).sum()),
                  outside_lims_visible=int((outside & vis).sum()), x0_clamped=int((vis & (x0 == 0)).sum()),
                  y0_clamped=int((vis & (y0 == 0)).sum()), x1_clamped=int((vis & (x1 == gx)).sum()),
                  y1_clamped=int((vis & (y1 == gy)).sum()), below_1_255=int((o < np.float32(1 / 255.0)).sum()),
                  alpha_clamp_visible=int((vis & (o > 0.99)).sum()))
    print("edges:", counts)
    assert counts["at_cull_visible"] == 0
    assert counts["below_1_255"] > 0 and not vis[o < np.float32(1 / 255.0)].any()
    for k in ("near_visible", "outside_lims_visible", "x0_clamped", "y0_clamped", "x1_clamped", "y1_clamped", "alpha_clamp_visible"):
        assert counts[k] >= 20, (k, counts[k])
    oracle32.free(f)


def test_stress_scenes_are_deterministic_and_256_aligned():
    for kind in syn.STRESS:
        a, ca = syn.make_stress_scene(kind)
        b, cb = syn.make_stress_scene(kind)
        assert a["means"].shape[0] % 256 == 0
        for k in ("means", "scales", "rots", "opacity", "dc", "sh"):
            assert np.array_equal(a[k], b[k]), (kind, k)
        assert np.isfinite(a["means"]).all() and (a["scales"] > 0).all()
        assert np.allclose(np.linalg.norm(a["rots"], axis=1), 1.0, atol=1e-6)
