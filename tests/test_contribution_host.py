"""Contribution scores without a GPU: known answers of the float64 restatement (contribution_oracle), the glic_unseen_params
ctypes layout against the header (compiled with the system C compiler), and NULL / argument rejections that need no device."""
import ctypes as C

import numpy as np

from contribution_oracle import scores
from test_align_host import _c_layout


NARROW = (20.0, 0.0, 20.0)        # exp(-10) o < 1/255 one pixel away: only the centre pixel takes the splat
WIDE = (1e-4, 0.0, 1e-4)           # alpha within 0.2 % of min(0.99, o) over an 8 x 8 frame


def _stack(o, conics, W=8, H=8, c=(3.0, 3.0)):
    P = len(o)
    xy = np.array([c] * P, np.float64)
    co = np.array([[k[0], k[1], k[2], x] for x, k in zip(o, conics)])
    return scores(W, H, xy, co, np.arange(P), np.array([[0, P]]), P)


def test_one_splat_on_a_pixel_centre():
    """w = 1 * min(0.99, o) at the centre; every pixel whose alpha >= 1/255 takes the splat"""
    for o in (0.3, 0.99, 0.9999):
        mw, hits, _, T, _, _ = scores(16, 16, np.array([[7.0, 5.0]]), np.array([[0.5, 0.0, 0.5, o]]), np.array([0]),
                                   np.array([[0, 1]]), 1)
        assert mw[0] == min(0.99, o)
        ys, xs = np.mgrid[0:16, 0:16]
        a = np.minimum(0.99, o * np.exp(-0.5 * (0.5 * (xs - 7.0) ** 2 + 0.5 * (ys - 5.0) ** 2)))
        assert hits[0] == int((a >= 1.0 / 255.0).sum()) > 1
        assert np.allclose(T, np.where(a >= 1.0 / 255.0, 1.0 - a, 1.0), rtol=0, atol=1e-15)


def test_a_stack_on_one_pixel():
    """three narrow splats on one centre, front to back: weights o_0, (1 - o_0) o_1, (1 - o_0)(1 - o_1) o_2, one hit each"""
    o = [0.5, 0.25, 0.8]
    mw, hits, ends, T, _, _ = _stack(o, [NARROW] * 3)
    assert list(mw) == [0.5, 0.5 * 0.25, 0.5 * 0.75 * 0.8] and list(hits) == [1, 1, 1] and not ends.any()
    assert T[3, 3] == 0.5 * 0.75 * (1.0 - 0.8) and (np.delete(T.reshape(-1), 3 * 8 + 3) == 1.0).all()


def test_rows_that_no_pixel_takes():
    """behind wide layers of alpha 0.99 and 0.95, a third layer of alpha 0.9 would take T below 1e-4 at every pixel: it ends
    them and is not taken, and so is nothing behind it; a faint splat (o < 1/255) is taken nowhere either"""
    mw, hits, ends, T, _, _ = _stack([1.0, 0.95, 0.9, 0.9, 0.003], [WIDE, WIDE, WIDE, NARROW, (0.5, 0.0, 0.5)])
    assert list(hits) == [64, 64, 0, 0, 0] and mw[0] == 0.99 and mw[2] == mw[3] == mw[4] == 0.0
    assert list(ends) == [0, 0, 64, 0, 0]                  # the third layer ends every pixel: it is not taken, but it counts
    assert np.isclose(mw[1], 0.01 * 0.95, rtol=1e-3) and (T < 1e-3).all()
    # in front of the layers, the faint splat is still not taken; a wide splat in front of them is
    mw, hits, _, _, _, _ = _stack([0.003, 0.5, 1.0], [(0.5, 0.0, 0.5), WIDE, WIDE])
    assert list(hits) == [0, 64, 64] and mw[0] == 0.0


def test_a_splat_that_only_ends_a_pixel():
    """wide layers of alpha 0.99 and 0.95, then a narrow 0.9 splat that ends the centre pixel, then a wide 0.5 splat: the narrow
    splat takes no pixel but ends one, and without it the wide splat behind would be taken at that pixel"""
    o, k = [1.0, 0.95, 0.9, 0.5], [WIDE, WIDE, NARROW, WIDE]
    mw, hits, ends, T, _, _ = _stack(o, k)
    assert hits[2] == 0 and ends[2] == 1 and mw[2] == 0.0
    assert hits[3] == 63 and ends[3] == 0                  # every pixel but the one the narrow splat ended
    mw2, hits2, _, T2, _, _ = _stack([o[0], o[1], o[3]], [k[0], k[1], k[3]])
    assert hits2[2] == 64 and T2[3, 3] < T[3, 3]             # removing the ending splat changes the pixel


def test_flagged_pixels_mark_their_list():
    """a splat whose centre alpha is 1/255 to float64 rounding is flagged, not decided"""
    _, _, _, _, flag, marked = scores(4, 4, np.array([[2.0, 2.0]]), np.array([[0.5, 0.0, 0.5, 1.0 / 255.0]]), np.array([0]),
                                   np.array([[0, 1]]), 1)
    assert flag[2, 2] and marked[0]


def test_unseen_params_match_the_header(tmp_path):
    from gaussian_lic_b200 import capi
    py = capi.UnseenParams
    fields = [f for f, _ in py._fields_]
    assert _c_layout(tmp_path, "glic_unseen_params", fields) == [C.sizeof(py)] + [getattr(py, f).offset for f in fields]
    assert fields == ["views", "n_views", "min_weight", "min_hits", "sky"]


def test_rejections_without_a_device():
    from gaussian_lic_b200 import capi
    lib = capi.lib
    p = capi.UnseenParams(None, 0, 0.0, 1, 0)
    n = C.c_uint32(77)
    assert lib.glic_mapper_prune_unseen(None, C.byref(p), 0, C.byref(n)) == -1 and b"null" in lib.glic_last_error()
    assert n.value == 77
    mw = np.zeros(4, np.float32)
    assert lib.glic_mapper_contribution(None, None, 0, mw.ctypes.data_as(C.c_void_p), None, None) == -1
    assert b"null" in lib.glic_last_error()
    # glic_contribution: a NULL view and a frame beyond GLIC_MAX_TILES are rejected before any device work
    assert lib.glic_contribution(1, None, None, 1.0, None, None, None, None, None, 0, None, 0, None, 0, None, None, None, None,
                                 None, None) == -1
    v = capi.View(1, 1, 1, 1.0, 1.0, -1.0, 1.0, -1.0, 1.0, 16 * 5000, 16 * 5000)
    assert lib.glic_contribution(1, None, None, 1.0, None, None, C.byref(v), None, None, 0, None, 0, None, 0, None, None, None,
                                 None, None, None) == -1
    assert b"GLIC_MAX_TILES" in lib.glic_last_error()
