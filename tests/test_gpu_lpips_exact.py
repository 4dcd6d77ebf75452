"""csrc/lpips.cu stage by stage against the float64 restatement of tests/lpips_reference.py, at every element: every tap
element of both images within its conv bound, every pool element bit for bit, every head CTA partial within the sum of its
pixels' bounds, and the output float bit for bit from the kernel's own partials.  Each stage is fed the kernel's own inputs,
read back from the caller's scratch.

Frames (lpips_reference.FRAMES): the smallest (31x31: taps 2-4 are 1x1; 35x35: conv0's image boundary on an M-tile edge), the
image boundary in the middle of a 64-row M tile or on its edge for each layer, W = 0..3 (mod 4) for the stride-4 right edge,
camera frames up to 2048x1536, 8192x31 and 31x8192, and one 8192x8192 frame.  Weights: the reference's (skipped when build()
did not convert them), two seeds of synthetic weights, and an adversarial payload (dead and thresholded conv0 channels that
give all-zero feature vectors on one image's dark square, so the head divides by 1e-10 alone there; zero lin entries; conv0
weights antisymmetric in x and scaled by 1e3).  Inputs: values below 0, above 1 and exactly 0 and 1; pairs that differ only
at the last pixel of image 1; identical pairs.  Every run uses scratch prefilled with 0xFF (NaN), and one run per case is
repeated on zero-filled scratch: the output and every carved region must be bit-identical.

Run with -s to see max(err / bound) per stage."""
import importlib.util
import os
import time

import numpy as np
import pytest

import lpips_reference as R

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILT = os.path.join(ROOT, "oracle", "_ref", "lpips_alex.bin")
BAND = 1 << 25                     # float64 elements of one output-row band of v, M, S
HEAD_CHUNK = 1 << 20               # pixels per head chunk (a multiple of 256)
PAYLOADS = ("reference", "synthetic1", "synthetic2", "adversarial")
# the frames the per-layer M-tile claims rest on: (W, H) -> {layer: "mid" | "edge"}
STRADDLE = {(131, 31): {0: "mid"}, (35, 35): {0: "edge"}, (71, 39): {1: "mid"}, (135, 39): {1: "edge"},
            (143, 79): {2: "mid", 3: "mid", 4: "mid"}, (143, 143): {2: "edge", 3: "edge", 4: "edge"}}


def _golden():
    spec = importlib.util.spec_from_file_location("make_lpips_golden", os.path.join(ROOT, "tests", "golden", "make_lpips_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _xn(v, mean, std):
    return (v - mean) / std


def adversarial_payload():
    p = _golden().synthetic_payload(3).copy()
    mean, std, convs, lins = R.unpack(p)
    w0, b0 = convs[0]
    b0[0:16] = -1e3                                                  # dead: zero everywhere
    w0[16:48] = np.abs(w0[16:48])                                    # thresholded: negative where the window is darker than 0.25
    thr = _xn(np.float32(0.25), mean, std).astype(np.float64)
    b0[16:48] = -(np.abs(w0[16:48]).astype(np.float64) * thr.reshape(1, 3, 1, 1)).sum((1, 2, 3))
    w0[48:64] = (w0[48:64] - w0[48:64, :, :, ::-1]) * 1e3            # x-derivative filters x1e3: cancel on x-constant input
    b0[48:64] = -1.0
    for lin in lins:
        lin[::3] = 0.0
    return p


@pytest.fixture(scope="module")
def payloads():
    from gaussian_lic_b200 import lpips_weights
    G = _golden()
    out = {"synthetic1": G.synthetic_payload(1), "synthetic2": G.synthetic_payload(2), "adversarial": adversarial_payload()}
    if os.path.isfile(BUILT):
        out["reference"] = lpips_weights.read(BUILT)
    return {k: torch.from_numpy(np.ascontiguousarray(v, np.float32)).to(DEV) for k, v in out.items()}


# ---- inputs, on the device --------------------------------------------------------------------------------------------
def _image(W, H, seed):
    rng = np.random.default_rng(seed)
    g = torch.Generator(device=DEV).manual_seed(seed)
    yy = torch.arange(H, device=DEV, dtype=torch.float32).view(H, 1) / max(W, H)
    xx = torch.arange(W, device=DEV, dtype=torch.float32).view(1, W) / max(W, H)
    img = torch.empty(3, H, W, device=DEV)
    for c in range(3):
        acc = torch.full((H, W), 0.5, device=DEV)
        for f, ph, a in zip(rng.uniform(1, 12, (4, 2)), rng.uniform(0, 2 * np.pi, 4), rng.uniform(0.05, 0.2, 4)):
            acc += float(a) * torch.sin(2 * np.pi * (float(f[0]) * xx + float(f[1]) * yy) + float(ph))
        img[c] = acc
    return img + 0.03 * torch.randn(3, H, W, device=DEV, generator=g)


def _specials(img, phase):
    """every 97th pixel (from `phase`) set to -0.3, 0, 1 or 1.4 in turn"""
    flat = img.view(3, -1)
    idx = torch.arange(phase, flat.shape[1], 97, device=DEV)
    flat[:, idx] = torch.tensor([-0.3, 0.0, 1.0, 1.4], device=DEV)[torch.arange(idx.numel(), device=DEV) % 4]
    return img


def inputs(W, H, seed):
    """(x, y, y_last): a pair with specials, a dark square in x and a saturated square in y; and x with only its last pixel
    changed (past the clamp)"""
    x = _specials(_image(W, H, seed), 0)
    g = torch.Generator(device=DEV).manual_seed(seed + 1)
    y = _specials(x + 0.25 * torch.randn(x.shape, device=DEV, generator=g), 41)
    s = min(max(min(H, W) // 3, 16), min(H, W))
    r0, c0 = (H - s) // 2, (W - s) // 2
    x[:, r0:r0 + s, c0:c0 + s] = 0.0
    y[:, :s, -s:] = 1.3
    y_last = x.clone()
    y_last[:, -1, -1] = torch.where(x[:, -1, -1].clamp(0, 1) > 0.5, 0.0, 1.0)
    return x.contiguous(), y.contiguous(), y_last.contiguous()


# ---- the kernel ------------------------------------------------------------------------------------------------------------
def run(x, y, weights, fill=0xFF):
    """glic_lpips on scratch prefilled with `fill`: (output [1], scratch)"""
    from gaussian_lic_b200 import capi, ops
    _, H, W = x.shape
    need = capi.lib.glic_lpips_scratch_bytes(H, W)
    assert need == R.layout(H, W)[1]
    scratch = torch.full((need,), fill, dtype=torch.uint8, device=DEV)
    out = ops.lpips(x, y, weights, scratch=scratch)
    torch.cuda.synchronize()
    return out, scratch


def _bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int64)


def same_bits(a, b):
    return torch.equal(_bits(a), _bits(b))


def regions_equal(sa, sb, H, W):
    ra, rb = R.carve(sa, H, W), R.carve(sb, H, W)
    return {k: same_bits(ra[k], rb[k]) for k in ra}


# ---- the stage checks ----------------------------------------------------------------------------------------------------
def check_stages(x, y, weights, out, scratch):
    """max(err / bound) per stage of one run, and what the run exercised"""
    _, H, W = x.shape
    reg = R.carve(scratch, H, W)
    mean, std, convs, lins = R.unpack(weights)
    hs, ws, _, _ = R.shapes(H, W)
    src = R.normalize(torch.stack([x, y]), mean, std)
    ratios, seen = {}, {"nx_eps": False}
    for l, (ci, co, k, s, pad) in enumerate(R.CONVS):
        w, b = convs[l]
        tap = reg["tap%d" % l]
        assert tap.shape == (2, co, hs[l], ws[l])
        rows = max(1, BAND // (2 * co * ws[l]))
        r = 0.0
        for r0 in range(0, hs[l], rows):
            band = range(r0, min(hs[l], r0 + rows))
            v, M, S = R.conv(src, w, b, s, pad, rows=band)
            r = max(r, R.conv_ratio(tap[:, :, band.start:band.stop], v, M, S))
            del v, M, S
        ratios["conv%d" % l] = r
        # head: per pixel in chunks of whole CTAs
        hw = hs[l] * ws[l]
        parts = reg["partials%d" % l]
        assert bool(torch.isfinite(parts).all())
        rh = 0.0
        for p0 in range(0, hw, HEAD_CHUNK):
            p1 = min(hw, p0 + HEAD_CHUNK)
            d, err = R.head(tap, lins[l], p0, p1)
            rh = max(rh, float(R.partial_check(parts[p0 // 256:(p1 + 255) // 256], d, err).max()))
            f = tap.view(2, co, -1)[:, :, p0:p1]
            seen["nx_eps"] |= bool(((f[0] == 0).all(0) & (f[1] != 0).any(0)).any())
        ratios["head%d" % l] = rh
        if l < 2:
            pooled = R.pool(tap)
            assert same_bits(pooled + 0.0, reg["pool%d" % l] + 0.0), "pool%d differs" % l   # +0.0: -0 and +0 alike
            src = reg["pool%d" % l]
        else:
            src = tap
    want = R.finish([reg["partials%d" % l].cpu().numpy() for l in range(5)], [h * w for h, w in zip(hs, ws)])
    assert out.cpu().numpy().view(np.int32)[0] == np.array([want], np.float32).view(np.int32)[0], (float(out), float(want))
    return ratios, seen


def _report(label, ratios):
    print("\n%s: " % label + "  ".join("%s %.3f" % kv for kv in sorted(ratios.items())))
    assert max(ratios.values()) <= 1.0, (label, ratios)


def _coverage(W, H):
    """assert the M-tile and frame-edge properties the frame is in the list for"""
    hs, ws, _, _ = R.shapes(H, W)
    for l, kind in STRADDLE.get((W, H), {}).items():
        hwo = hs[l] * ws[l]
        assert (hwo % R.BM == 0) == (kind == "edge") and hwo > 0, (W, H, l, hwo)
    if (W, H) == (31, 31):
        assert hs[2:] == [1, 1, 1] and ws[2:] == [1, 1, 1]
    if (W, H) == (35, 35):
        assert hs[0] * ws[0] == 64


def test_frames_cover_the_claimed_edges():
    for W, H in R.FRAMES:
        _coverage(W, H)
    assert {W % 4 for W, H in R.FRAMES if H == 512} == {0, 1, 2, 3}
    assert {(8192, 31), (31, 8192), (8192, 8192)} <= set(R.FRAMES)


def _reaches_last_pixel(W, H):
    """conv0 (11 wide, stride 4, pad 2, floor mode) reads input column W - 1 unless (W - 7) % 4 == 3, and likewise rows"""
    return (W - 7) % 4 != 3 and (H - 7) % 4 != 3


def check_case(W, H, name, weights, seed):
    x, y, y_last = inputs(W, H, seed)
    xs = x.view(-1)
    assert bool((xs < 0).any() and (xs > 1).any() and (xs == 0).any() and (xs == 1).any())
    # the pair, on NaN-prefilled scratch and on zero-filled scratch: bit-identical output and regions
    out, sc = run(x, y, weights, 0xFF)
    out0, sc0 = run(x, y, weights, 0x00)
    assert same_bits(out, out0)
    eq = regions_equal(sc, sc0, H, W)
    assert all(eq.values()), eq
    del sc0
    ratios, seen = check_stages(x, y, weights, out, sc)
    _report("%dx%d %s" % (W, H, name), ratios)
    if name == "adversarial":
        assert seen["nx_eps"], "no pixel of one image had an all-zero feature vector"
    del sc
    # identical pairs: the two halves of every tap are bit-identical and LPIPS is exactly 0
    out_id, sc_id = run(x, x.clone(), weights)
    reg_id = R.carve(sc_id, H, W)
    for l in range(5):
        t = reg_id["tap%d" % l]
        assert same_bits(t[0], t[1]), l
    assert float(out_id) == 0.0
    # the last pixel of image 1 changed: image 0's half of every tap and pool is the identical run's, bit for bit
    out_l, sc_l = run(x, y_last, weights)
    reg_l = R.carve(sc_l, H, W)
    for k in ["tap%d" % l for l in range(5)] + ["pool0", "pool1"]:
        assert same_bits(reg_l[k][0], reg_id[k][0]), k
    changed = not same_bits(reg_l["tap0"][1], reg_id["tap0"][1])
    if not _reaches_last_pixel(W, H):
        assert not changed and float(out_l) == 0.0               # conv0 never reads the last pixel
    elif name != "adversarial":
        assert changed
    return ratios


@pytest.mark.parametrize("name", PAYLOADS)
@pytest.mark.parametrize("WH", [f for f in R.FRAMES if f != (8192, 8192)], ids=lambda f: "%dx%d" % f)
def test_every_stage_within_its_bound(payloads, WH, name):
    if name not in payloads:
        pytest.skip("oracle/_ref/lpips_alex.bin not built (the reference's weights)")
    _coverage(*WH)
    check_case(WH[0], WH[1], name, payloads[name], seed=WH[0] * 10007 + WH[1] + PAYLOADS.index(name))


def test_largest_frame(payloads):
    """8192 x 8192, the largest side: every element of every stage, with the synthetic weights"""
    t0 = time.time()
    check_case(8192, 8192, "synthetic1", payloads["synthetic1"], seed=8192)
    print("8192x8192 checked in %.1f s on %s" % (time.time() - t0, torch.cuda.get_device_name(0)))
