"""glic_render and glic_mapper_render_camera without a GPU: the ctypes camera struct against the header's layout (compiled with
the system C compiler), the NULL-mapper and NULL-camera rejections, and the frame-size checks that refuse a call before any
launch."""
import ctypes as C

import pytest

from test_align_host import _c_layout


def test_render_camera_struct_matches_the_header(tmp_path):
    from gaussian_lic_b200 import capi
    py = capi.RenderCamera
    fields = [f for f, _ in py._fields_]
    want = _c_layout(tmp_path, "glic_render_camera", fields)
    got = [C.sizeof(py)] + [getattr(py, f).offset for f in fields]
    assert got == want, (got, want)
    assert sum(getattr(py, f).size for f in fields) == C.sizeof(py) == want[0] == 4 * 18


def test_null_mapper_and_camera_are_rejected_without_a_device():
    from gaussian_lic_b200 import capi
    cam = capi.RenderCamera()
    cam.R_wc[0] = cam.R_wc[4] = cam.R_wc[8] = 1.0
    cam.fx = cam.fy = 100.0
    cam.width, cam.height = 64, 48
    out = (C.c_float * (3 * 64 * 48))()
    assert capi.lib.glic_mapper_render_camera(None, C.byref(cam), -1, 1, out, None, None, None) == -1
    assert b"null" in capi.lib.glic_last_error()
    assert capi.lib.glic_mapper_render_camera(None, None, -1, 1, out, None, None, None) == -1
    assert capi.lib.glic_mapper_render_camera(None, C.byref(cam), -1, 1, None, None, None, None) == -1
    assert out[0] == 0.0                                               # nothing written


def _view(W, H):
    from gaussian_lic_b200 import capi
    # non-NULL pointers the size checks never dereference
    return capi.View(16, 16, 16, 0.5, 0.5, -1.0, 1.0, -1.0, 1.0, W, H)


@pytest.mark.parametrize("W,H,ok", [(4096, 4096, True), (4096, 4097, False), (1, 0, False), (0, 1, False),
                                    (65536 * 16, 1, True), (65536 * 16 + 1, 1, False)])
def test_render_refuses_frames_before_any_launch(W, H, ok):
    """GLIC_MAX_TILES tiles pass the frame check (and then stop at the missing image workspace), one tile more does not"""
    from gaussian_lic_b200 import capi
    v = _view(W, H)
    st = capi.lib.glic_render(1, 0, 0, None, None, 1.0, None, None, None, None, C.byref(v), None, None, 0, None, 0, None, 0,
                              None, None, None, None, None, None)
    err = capi.lib.glic_last_error().decode()
    if ok:
        assert st == -2 and "image workspace" in err, (st, err)
    else:
        assert st == -1 and ("GLIC_MAX_TILES" in err or "image size" in err), (st, err)
