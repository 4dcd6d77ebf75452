"""The rasterizer entry points' argument checks without a GPU: for each check, one call that breaks exactly that check, and the
calls that break two checks where the order of the checks decides the answer.  Each call must return the check's status with
its exact text, zero the host outputs the entry point zeroes before that check and no others, and launch nothing.

The pointers are 16-byte-aligned integers that are never dereferenced: every check fires before the first CUDA call."""
import ctypes as C

import pytest

A = 0x100000                 # a 16-byte-aligned dummy device pointer
U = A + 4                    # the same, misaligned
W, H = 64, 48
JUNK = -7
BIG = 1 << 40


def _lib():
    from gaussian_lic_b200 import capi
    return capi


def _view(**over):
    capi = _lib()
    f = dict(viewmatrix=A, projmatrix=A, campos=A, tan_fovx=1.0, tan_fovy=1.0, limx_neg=-1.0, limx_pos=1.0, limy_neg=-1.0,
             limy_pos=1.0, width=W, height=H)
    f.update(over)
    return capi.View(**f)


VIEW_CASES = [
    (None, -1, "view: null pointer"),
    (dict(viewmatrix=None), -1, "view: null pointer"),
    (dict(projmatrix=None), -1, "view: null pointer"),
    (dict(campos=None), -1, "view: null pointer"),
    (dict(width=0), -1, "view: non-positive image size"),
    (dict(height=-1), -1, "view: non-positive image size"),
    (dict(width=4112, height=4096), -1, "view: 4112x4096 has 65792 tiles of 16x16, more than GLIC_MAX_TILES = 65536"),
]

ARGS = {
    "glic_forward_preprocess": ["P", "sh_degree", "M", "means3D", "scales", "scale_modifier", "rotations", "opacities", "dc", "sh",
                                "view", "no_color", "radii", "geom_ws", "geom_bytes", "image_ws", "image_bytes",
                                "num_rendered_host", "stream"],
    "glic_forward_render": ["P", "view", "no_color", "R", "geom_ws", "image_ws", "binning_ws", "binning_bytes", "sample_ws",
                            "sample_bytes", "out_color", "out_final_T", "num_buckets_host", "stream"],
    "glic_forward": ["P", "sh_degree", "M", "means3D", "scales", "scale_modifier", "rotations", "opacities", "dc", "sh", "view",
                     "no_color", "radii", "geom_ws", "geom_bytes", "image_ws", "image_bytes", "binning_ws", "binning_bytes",
                     "sample_ws", "sample_bytes", "out_color", "out_final_T", "counters_host", "stream"],
    "glic_render": ["P", "sh_degree", "M", "means3D", "scales", "scale_modifier", "rotations", "opacities", "dc", "sh", "view",
                    "radii", "geom_ws", "geom_bytes", "image_ws", "image_bytes", "binning_ws", "binning_bytes", "out_color",
                    "out_final_T", "out_depth", "out_median_depth", "counters_host", "stream"],
    "glic_contribution": ["P", "means3D", "scales", "scale_modifier", "rotations", "opacities", "view", "radii", "geom_ws",
                          "geom_bytes", "image_ws", "image_bytes", "binning_ws", "binning_bytes", "max_weight", "hits", "ends",
                          "out_final_T", "counters_host", "stream"],
    "glic_backward": ["P", "sh_degree", "M", "means3D", "scales", "scale_modifier", "rotations", "dc", "sh", "view", "radii", "R",
                      "geom_ws", "binning_ws", "image_ws", "sample_ws", "dL_dpix", "lambda_erank", "dL_dmeans2D", "dL_dconic",
                      "dL_dopacity", "dL_dcolors", "dL_dmeans3D", "dL_dcov3D", "dL_ddc", "dL_dsh", "dL_dscales", "dL_drotations",
                      "stream"],
    "glic_debug_render_backward": ["P", "view", "R", "geom_ws", "binning_ws", "image_ws", "sample_ws", "dL_dpix", "dL_dmeans2D",
                                   "dL_dconic", "dL_dopacity", "dL_dcolors", "exact", "counters", "stream"],
    "glic_debug_deterministic_entries": ["P", "view", "R", "geom_ws", "binning_ws", "image_ws", "sample_ws", "dL_dpix", "det_ws",
                                         "det_bytes", "dL_dmeans2D", "dL_dconic", "dL_dopacity", "dL_dcolors", "count_host", "gid",
                                         "tile", "values", "stream"],
    "glic_debug_pose_backward": ["P", "sh_degree", "M", "means3D", "scales", "rotations", "rot_raw", "opacity", "sh", "view",
                                 "radii", "geom_ws", "dL_dmeans2D", "dL_dconic", "dL_dopacity", "dL_dcolors", "pose_only", "g_geo",
                                 "partials", "pose6", "stream"],
}
ARGS["glic_backward_deterministic"] = ARGS["glic_backward"][:-1] + ["det_ws", "det_bytes", "stream"]

# the one host output each entry point zeroes once its first checks pass
HOST_OUT = {"glic_forward_preprocess": "num_rendered_host", "glic_forward_render": "num_buckets_host",
            "glic_debug_deterministic_entries": "count_host"}
COUNTERS = ("glic_forward", "glic_render", "glic_contribution")


def _defaults(fn):
    lib = _lib().lib
    sizes = dict(P=10, sh_degree=3, M=15, R=100, scale_modifier=1.0, lambda_erank=0.0, no_color=0, exact=0, pose_only=0,
                 geom_bytes=lib.glic_geom_bytes(10), image_bytes=lib.glic_image_bytes(W, H), binning_bytes=BIG, sample_bytes=BIG,
                 det_bytes=BIG, stream=None)
    return {a: sizes.get(a, A) for a in ARGS[fn]}


def _call(fn, over, view_over=()):
    """Calls fn with every argument valid but those in `over`; returns (status, error text, host output, counters)."""
    capi = _lib()
    lib = capi.lib
    args = _defaults(fn)
    args.update(over)
    view = None if view_over is None else _view(**dict(view_over))
    args["view"] = None if view is None else C.byref(view)
    host = C.c_int64(JUNK)
    counters = (C.c_int64 * 3)(JUNK, JUNK, JUNK)
    if fn in HOST_OUT and args[HOST_OUT[fn]] == A:
        args[HOST_OUT[fn]] = C.byref(host)
    if fn in COUNTERS and args["counters_host"] == A:
        args["counters_host"] = counters
    before = lib.glic_launch_count()
    rc = getattr(lib, fn)(*[args[a] for a in ARGS[fn]])
    assert lib.glic_launch_count() == before, "%s launched a kernel on a failed check" % fn
    return rc, lib.glic_last_error().decode(), host.value, list(counters)


def _check(fn, over, rc, msg, host=JUNK, view_over=()):
    got_rc, got_msg, got_host, got_counters = _call(fn, over, view_over)
    assert got_rc == rc, (fn, over, view_over, got_rc, got_msg)
    if rc != 0:                                        # a call that succeeds leaves the last error as it was
        assert got_msg == msg, (fn, over, view_over)
    if fn in HOST_OUT:
        assert got_host == host, (fn, over, "host output")
    assert got_counters == [JUNK] * 3, (fn, over, "counters were written")


ENTRY_POINTS = sorted(ARGS)


@pytest.mark.parametrize("fn", ENTRY_POINTS)
@pytest.mark.parametrize("view_over,rc,msg", VIEW_CASES)
def test_view_check_fires_first(fn, view_over, rc, msg):
    # the view check comes before every other: break a later check too
    over = {"P": -1} if fn != "glic_debug_pose_backward" else {"P": 0}
    _check(fn, over, rc, msg, view_over=view_over)


def _cases_forward_preprocess():
    n = "forward_preprocess: "
    bad, coef, img = n + "bad P / sh_degree / M", n + "sh has fewer coefficients than sh_degree needs", n + "image workspace too small"
    nul, rot, geom = n + "null input pointer", n + "rotations must be 16-byte aligned", n + "geometry workspace too small"
    lib = _lib().lib
    return [
        (dict(P=-1), -1, bad, JUNK), (dict(sh_degree=-1), -1, bad, JUNK), (dict(sh_degree=4), -1, bad, JUNK),
        (dict(M=-1), -1, bad, JUNK),
        (dict(num_rendered_host=None), -1, n + "num_rendered_host is NULL", JUNK),
        (dict(P=-1, num_rendered_host=None), -1, bad, JUNK),
        (dict(M=14), -1, coef, 0), (dict(sh_degree=1, M=2), -1, coef, 0),
        (dict(M=14, num_rendered_host=None), -1, n + "num_rendered_host is NULL", JUNK),
        (dict(M=14, image_ws=None), -1, coef, 0),
        (dict(no_color=1, M=0, image_ws=None), -2, img, 0),        # no_color needs no SH
        (dict(image_ws=None), -2, img, 0), (dict(image_bytes=lib.glic_image_bytes(W, H) - 1), -2, img, 0),
        (dict(P=0, image_ws=None, means3D=None), -2, img, 0),
        (dict(P=0, means3D=None, geom_ws=None), 0, "", 0),          # P = 0: nothing to check further, nothing to launch
        (dict(means3D=None), -1, nul, 0), (dict(scales=None), -1, nul, 0), (dict(rotations=None), -1, nul, 0),
        (dict(opacities=None), -1, nul, 0), (dict(radii=None), -1, nul, 0), (dict(dc=None), -1, nul, 0),
        (dict(sh=None), -1, nul, 0),
        (dict(no_color=1, dc=None, sh=None, rotations=U), -1, rot, 0),
        (dict(sh_degree=0, sh=None, rotations=U), -1, rot, 0), (dict(M=0, sh_degree=0, sh=None, rotations=U), -1, rot, 0),
        (dict(means3D=None, rotations=U), -1, nul, 0),
        (dict(rotations=U), -1, rot, 0), (dict(rotations=U, geom_ws=None), -1, rot, 0),
        (dict(geom_ws=None), -2, geom, 0), (dict(geom_bytes=lib.glic_geom_bytes(10) - 1), -2, geom, 0),
    ]


def _draw_cases(fn, n):
    """The checks glic_forward, glic_render and glic_contribution share, after their own first checks."""
    lib = _lib().lib
    img, nul = n + "image workspace too small", n + "null input pointer"
    rot, geom = n + "rotations must be 16-byte aligned", n + "geometry workspace too small"
    return [
        (dict(image_ws=None), -2, img), (dict(image_bytes=lib.glic_image_bytes(W, H) - 1), -2, img),
        (dict(P=0, image_ws=None), -2, img), (dict(image_ws=None, out_final_T=None), -2, img),
        (dict(means3D=None), -1, nul), (dict(scales=None), -1, nul), (dict(rotations=None), -1, nul),
        (dict(opacities=None), -1, nul), (dict(radii=None), -1, nul),
        (dict(means3D=None, rotations=U), -1, nul),
        (dict(rotations=U), -1, rot), (dict(rotations=U, geom_ws=None), -1, rot),
        (dict(geom_ws=None), -2, geom), (dict(geom_bytes=lib.glic_geom_bytes(10) - 1), -2, geom),
        (dict(geom_ws=None, binning_ws=None), -2, geom),
    ]


def _cases_forward():
    n = "forward: "
    bad, coef, out = n + "bad P / sh_degree / M", n + "sh has fewer coefficients than sh_degree needs", n + "null output"
    bins = n + "binning / sample workspace missing or too small"
    return _draw_cases("glic_forward", n) + [
        (dict(P=-1), -1, bad), (dict(sh_degree=-1), -1, bad), (dict(sh_degree=4), -1, bad), (dict(M=-1), -1, bad),
        (dict(P=-1, M=0), -1, bad),
        (dict(M=14), -1, coef), (dict(M=14, image_ws=None), -1, coef), (dict(no_color=1, M=0, image_ws=None), -2, n + "image workspace too small"),
        (dict(out_final_T=None), -1, out), (dict(out_color=None), -1, out), (dict(P=0, out_color=None), -1, out),
        (dict(no_color=1, out_color=None, geom_ws=None), -2, n + "geometry workspace too small"),
        (dict(dc=None), -1, n + "null input pointer"), (dict(sh=None), -1, n + "null input pointer"),
        (dict(no_color=1, dc=None, sh=None, rotations=U), -1, n + "rotations must be 16-byte aligned"),
        (dict(sh_degree=0, sh=None, rotations=U), -1, n + "rotations must be 16-byte aligned"),
        (dict(binning_ws=None), -2, bins), (dict(binning_bytes=0), -2, bins), (dict(sample_ws=None), -2, bins),
        (dict(sample_bytes=0), -2, bins), (dict(no_color=1, binning_bytes=0, sample_ws=None, sample_bytes=0), -2, bins),
        (dict(no_color=1, binning_ws=None), -2, bins),
    ]


def _cases_render():
    n = "render: "
    bad, coef, out = n + "bad P / sh_degree / M", n + "sh has fewer coefficients than sh_degree needs", n + "null output"
    bins = n + "binning workspace missing or too small"
    return _draw_cases("glic_render", n) + [
        (dict(P=-1), -1, bad), (dict(sh_degree=-1), -1, bad), (dict(sh_degree=4), -1, bad), (dict(M=-1), -1, bad),
        (dict(M=14), -1, coef), (dict(M=14, image_ws=None), -1, coef),
        (dict(out_final_T=None), -1, out), (dict(out_color=None), -1, out), (dict(P=0, out_color=None), -1, out),
        (dict(out_depth=None, out_median_depth=None, geom_ws=None), -2, n + "geometry workspace too small"),
        (dict(dc=None), -1, n + "null input pointer"), (dict(sh=None), -1, n + "null input pointer"),
        (dict(sh_degree=0, sh=None, rotations=U), -1, n + "rotations must be 16-byte aligned"),
        (dict(binning_ws=None), -2, bins), (dict(binning_bytes=0), -2, bins),
    ]


def _cases_contribution():
    n = "contribution: "
    out, bins = n + "null output", n + "binning workspace missing or too small"
    return _draw_cases("glic_contribution", n) + [
        (dict(P=-1), -1, n + "P must be >= 0"), (dict(P=-1, image_ws=None), -1, n + "P must be >= 0"),
        (dict(max_weight=None), -1, out), (dict(hits=None), -1, out), (dict(max_weight=None, means3D=None), -1, out),
        (dict(ends=None, out_final_T=None, geom_ws=None), -2, n + "geometry workspace too small"),
        (dict(binning_ws=None), -2, bins), (dict(binning_bytes=0), -2, bins),
    ]


def _cases_forward_render():
    n = "forward_render: "
    bad, bins, smp = n + "bad arguments", n + "binning workspace too small", n + "sample workspace too small"
    lib = _lib().lib
    return [
        (dict(P=-1), -1, bad, JUNK), (dict(R=-1), -1, bad, JUNK), (dict(image_ws=None), -1, bad, JUNK),
        (dict(out_final_T=None), -1, bad, JUNK), (dict(out_color=None), -1, bad, JUNK),
        (dict(P=0, out_color=None), -1, bad, JUNK),
        (dict(geom_ws=None), -2, n + "geometry workspace is NULL", 0),
        (dict(geom_ws=None, num_buckets_host=None), -2, n + "geometry workspace is NULL", JUNK),
        (dict(geom_ws=None, binning_ws=None), -2, n + "geometry workspace is NULL", 0),
        (dict(no_color=1, out_color=None, geom_ws=None), -2, n + "geometry workspace is NULL", 0),
        (dict(binning_ws=None), -2, bins, 0), (dict(binning_bytes=lib.glic_binning_bytes(100) - 1), -2, bins, 0),
        (dict(binning_ws=None, sample_ws=None), -2, bins, 0),
        (dict(sample_ws=None), -2, smp, 0), (dict(sample_bytes=lib.glic_sample_bytes(100, W, H) - 1), -2, smp, 0),
        (dict(R=0, sample_bytes=lib.glic_sample_bytes(0, W, H) - 1), -2, smp, 0),
    ]


def _cases_backward(n):
    bad, nul = n + "bad sizes", n + "null pointer"
    ali, ws = n + "rotations / dL_drotations must be 16-byte aligned", n + "missing saved workspace"
    cases = [(dict(P=-1), -1, bad), (dict(R=-1), -1, bad), (dict(sh_degree=-1), -1, bad), (dict(sh_degree=4), -1, bad),
             (dict(M=-1), -1, bad), (dict(P=-1, means3D=None), -1, bad),
             (dict(P=0, means3D=None, geom_ws=None), 0, "")]       # P = 0: nothing to do, nothing launched
    for a in ("means3D", "scales", "rotations", "radii", "dL_dpix", "dL_dmeans2D", "dL_dconic", "dL_dopacity", "dL_dcolors",
              "dL_dmeans3D", "dL_dcov3D", "dL_ddc", "dL_dscales", "dL_drotations", "sh", "dL_dsh"):
        cases.append(({a: None}, -1, nul))
    cases += [
        (dict(M=0, sh=None, dL_dsh=None, dc=None, rotations=U), -1, ali),   # dc is not read; sh only with M > 0
        (dict(means3D=None, rotations=U), -1, nul),
        (dict(rotations=U), -1, ali), (dict(dL_drotations=U), -1, ali), (dict(rotations=U, geom_ws=None), -1, ali),
        (dict(geom_ws=None), -2, ws), (dict(image_ws=None), -2, ws), (dict(binning_ws=None), -2, ws), (dict(sample_ws=None), -2, ws),
    ]
    return cases


def _cases_backward_deterministic():
    n = "backward_deterministic: "
    det = n + "deterministic workspace too small"
    lib = _lib().lib
    return _cases_backward(n) + [
        (dict(det_ws=None), -2, det), (dict(det_bytes=lib.glic_deterministic_bytes(100, W, H) - 1), -2, det),
        # the workspace check comes before the size and pointer checks when P > 0 and R > 0
        (dict(det_ws=None, sh_degree=4), -2, det), (dict(det_ws=None, means3D=None), -2, det),
        (dict(det_ws=None, P=-1), -1, n + "bad sizes"),
        (dict(R=0, det_ws=None, geom_ws=None), -2, n + "missing saved workspace"),
        (dict(R=0, det_ws=None, binning_ws=None, sample_ws=None, rotations=U), -1, n + "rotations / dL_drotations must be 16-byte aligned"),
    ]


def _cases_debug_render_backward():
    n = "debug_render_backward: "
    bad, nul, ws = n + "bad sizes", n + "null pointer", n + "missing saved workspace"
    return [
        (dict(P=-1), -1, bad), (dict(R=-1), -1, bad), (dict(P=-1, dL_dpix=None), -1, bad),
        (dict(P=0, dL_dpix=None), 0, ""), (dict(R=0, dL_dpix=None, geom_ws=None), 0, ""),
        (dict(dL_dpix=None), -1, nul), (dict(dL_dmeans2D=None), -1, nul), (dict(dL_dconic=None), -1, nul),
        (dict(dL_dopacity=None), -1, nul), (dict(dL_dcolors=None), -1, nul), (dict(dL_dpix=None, geom_ws=None), -1, nul),
        (dict(geom_ws=None), -2, ws), (dict(image_ws=None), -2, ws), (dict(binning_ws=None), -2, ws), (dict(sample_ws=None), -2, ws),
    ]


def _cases_debug_deterministic_entries():
    n = "debug_deterministic_entries: "
    bad, nul, ws, det = n + "bad arguments", n + "null pointer", n + "missing saved workspace", n + "deterministic workspace too small"
    lib = _lib().lib
    cases = [(dict(P=-1), -1, bad, JUNK), (dict(R=-1), -1, bad, JUNK), (dict(count_host=None), -1, bad, JUNK),
             (dict(P=0, dL_dpix=None, geom_ws=None), 0, "", 0)]
    for a in ("dL_dpix", "dL_dmeans2D", "dL_dconic", "dL_dopacity", "dL_dcolors", "gid", "tile", "values"):
        cases.append(({a: None}, -1, nul, 0))
    cases += [
        (dict(dL_dpix=None, geom_ws=None), -1, nul, 0),
        (dict(geom_ws=None), -2, ws, 0), (dict(image_ws=None), -2, ws, 0), (dict(binning_ws=None), -2, ws, 0),
        (dict(sample_ws=None), -2, ws, 0), (dict(geom_ws=None, det_ws=None), -2, ws, 0),
        (dict(R=0, binning_ws=None, sample_ws=None, geom_ws=None), -2, ws, 0),
        (dict(det_ws=None), -2, det, 0), (dict(det_bytes=lib.glic_deterministic_bytes(100, W, H) - 1), -2, det, 0),
    ]
    return cases


def _cases_debug_pose_backward():
    bad = "debug_pose_backward: bad arguments"
    cases = [(dict(P=0), -1, bad), (dict(P=-1), -1, bad)]
    for a in ("means3D", "scales", "rotations", "radii", "geom_ws", "dL_dmeans2D", "dL_dconic", "dL_dcolors", "partials", "pose6",
              "g_geo", "rot_raw", "opacity", "dL_dopacity"):
        cases.append(({a: None}, -1, bad))
    cases.append((dict(pose_only=1, means3D=None, g_geo=None, rot_raw=None, opacity=None, dL_dopacity=None), -1, bad))
    return cases


def _with_host(cases):
    return [c if len(c) == 4 else c + (JUNK,) for c in cases]


CASES = {
    "glic_forward_preprocess": _cases_forward_preprocess,
    "glic_forward_render": _cases_forward_render,
    "glic_forward": _cases_forward,
    "glic_render": _cases_render,
    "glic_contribution": _cases_contribution,
    "glic_backward": lambda: _cases_backward("backward: "),
    "glic_backward_deterministic": _cases_backward_deterministic,
    "glic_debug_render_backward": _cases_debug_render_backward,
    "glic_debug_deterministic_entries": _cases_debug_deterministic_entries,
    "glic_debug_pose_backward": _cases_debug_pose_backward,
}


@pytest.mark.parametrize("fn", ENTRY_POINTS)
def test_each_check(fn):
    for over, rc, msg, host in _with_host(CASES[fn]()):
        _check(fn, over, rc, msg, host)
