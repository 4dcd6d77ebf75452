"""LPIPS weight file and argument checks without a GPU: a weight file reads back through glic_lpips_read_weights as exactly the
floats written (the reference's weights, converted by build() into oracle/_ref/lpips_alex.bin, as exactly the converter's floats),
malformed files are refused, and frames the AlexNet trunk cannot take (under 31x31) are refused before anything is launched."""
import ctypes as C
import os
import struct

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILT = os.path.join(ROOT, "oracle", "_ref", "lpips_alex.bin")
PT = os.path.join(ROOT, "oracle", "_ref", "lpips_alex.pt")
LAYERS = [(64, 3, 11), (192, 64, 5), (384, 192, 3), (256, 384, 3), (256, 256, 3)]     # (Cout, Cin, k)


def _expected_floats():
    return 6 + sum(co * ci * k * k + co for co, ci, k in LAYERS) + sum(co for co, _, _ in LAYERS)


@pytest.fixture
def weight_file(tmp_path):
    """a well-formed weight file written by the converter's writer: header + seeded floats of every sign and magnitude"""
    from gaussian_lic_b200 import lpips_weights
    rng = np.random.default_rng(3)
    p = (rng.standard_normal(_expected_floats()) * np.exp(rng.uniform(-20, 5, _expected_floats()))).astype(np.float32)
    path = tmp_path / "w.bin"
    lpips_weights.write(path, p)
    return path, p


def _read(path):
    from gaussian_lic_b200 import capi
    out = np.full(int(capi.lib.glic_lpips_weight_floats()), np.nan, np.float32)
    rc = capi.lib.glic_lpips_read_weights(str(path).encode(), out.ctypes.data_as(C.c_void_p))
    return rc, out, capi.lib.glic_last_error().decode()


def test_weight_count_matches_the_layer_shapes():
    from gaussian_lic_b200 import capi
    assert capi.lib.glic_lpips_weight_floats() == _expected_floats() == 2470854


def test_weight_file_reads_back_exactly(weight_file):
    """the library's reader returns the written payload bit for bit, behind the header the converter writes"""
    from gaussian_lic_b200 import lpips_weights
    path, p = weight_file
    raw = open(path, "rb").read()
    magic, version, n, zero = struct.unpack("<4I", raw[:16])
    assert (magic, version, n, zero) == (lpips_weights.MAGIC, 1, _expected_floats(), 0) and raw[:4] == b"LPIP"
    assert len(raw) == 16 + 4 * n
    rc, got, err = _read(path)
    assert rc == 0, err
    assert got.tobytes() == p.tobytes()


def test_built_weights_are_the_converted_reference_module(tmp_path):
    """the weight file build() converted from the reference's lpips_alex.pt reads back as exactly the converter's floats, laid
    out as the state dict: normalisation buffers, each conv's OIHW weight and bias, the five lin weights"""
    if not (os.path.isfile(PT) and os.path.isfile(BUILT)):
        pytest.skip("oracle/_ref/lpips_alex.pt / lpips_alex.bin not built")
    pytest.importorskip("torch")
    from gaussian_lic_b200 import lpips_weights
    out = tmp_path / "w.bin"
    p = lpips_weights.convert(PT, out)
    assert open(out, "rb").read() == open(BUILT, "rb").read()
    rc, got, err = _read(BUILT)
    assert rc == 0, err
    assert got.tobytes() == p.astype(np.float32).tobytes()
    # the normalisation buffers sit first: mean (-.030, -.088, -.188), std (.458, .448, .450)
    np.testing.assert_allclose(got[:6], [-0.030, -0.088, -0.188, 0.458, 0.448, 0.450], atol=1e-6)
    st = lpips_weights.load_state(PT)
    assert np.array_equal(got[6:6 + 64 * 3 * 121].reshape(64, 3, 11, 11), st["net.layers.0.weight"].numpy())
    assert np.array_equal(got[-256:], st["lin.4.1.weight"].numpy().reshape(-1))


@pytest.mark.parametrize("case", ["truncated", "header_only", "trailing", "bad_magic", "bad_version", "bad_count", "empty", "missing"])
def test_malformed_files_are_refused(tmp_path, weight_file, case):
    raw = bytearray(open(weight_file[0], "rb").read())
    if case == "truncated":
        raw = raw[:-4]
    elif case == "header_only":
        raw = raw[:16]
    elif case == "trailing":
        raw += b"\0\0\0\0"
    elif case == "bad_magic":
        raw[:4] = b"LPIQ"
    elif case == "bad_version":
        raw[4:8] = struct.pack("<I", 2)
    elif case == "bad_count":
        raw[8:12] = struct.pack("<I", _expected_floats() - 1)
    elif case == "empty":
        raw = b""
    path = tmp_path / "bad.bin"
    if case != "missing":
        path.write_bytes(bytes(raw))
    rc, _, err = _read(path)
    assert rc == -1, case
    want = {"truncated": "truncated", "header_only": "truncated", "trailing": "trailing", "bad_magic": "magic",
            "bad_version": "version", "bad_count": "floats", "empty": "truncated", "missing": "cannot open"}[case]
    assert want in err, err


@pytest.mark.parametrize("HW", [(30, 640), (640, 30), (30, 30), (0, 0), (-31, 31), (31, 8193)])
def test_frames_outside_the_network_are_refused(HW):
    from gaussian_lic_b200 import capi
    H, W = HW
    lib = capi.lib
    assert lib.glic_lpips_scratch_bytes(H, W) == 0
    dummy = C.c_void_p(16)                # never dereferenced: the frame is checked before anything else
    before = capi.launch_count()
    assert lib.glic_lpips(H, W, dummy, dummy, dummy, dummy, dummy, 1 << 30, None) == -1
    assert b"31x31" in lib.glic_last_error()
    assert capi.launch_count() == before


def test_scratch_size_and_argument_checks():
    from gaussian_lic_b200 import capi
    lib = capi.lib
    assert lib.glic_lpips_scratch_bytes(31, 31) > 0
    # the taps of both images, fp32: at 640x512, tap 1 alone is 2 x 64 x 127 x 159 floats
    assert lib.glic_lpips_scratch_bytes(512, 640) >= 4 * 2 * 64 * 127 * 159
    assert lib.glic_lpips_scratch_bytes(1080, 1920) > lib.glic_lpips_scratch_bytes(512, 640)
    assert lib.glic_lpips(512, 640, None, None, None, None, None, 0, None) == -1
    d = C.c_void_p(16)
    assert lib.glic_lpips(512, 640, d, d, d, d, d, 16, None) == -2 and b"scratch" in lib.glic_last_error()
    assert lib.glic_lpips_read_weights(None, None) == -1
