"""csrc/ssim.cu against the float64 restatement of tests/loss_reference.py at every element, with each element's own bound
|got - ref| <= c * 2^-24 * M (c per output in loss_reference.BOUND, M the restatement's magnitude map): the SSIM map and its
partial maps, the SSIM backward, the L1 + D-SSIM loss and its gradient, the exposed loss with dL/dimg and dL/dE, and the
evaluation PSNR / SSIM.  Every map and gradient here is a fixed-order fmaf chain, so there is no outlier fraction and no
tolerance relative to the tensor's maximum.  The loss scalar is the one output that is not bit-reproducible: each 32x32
tile adds its partial sum with a float atomicAdd, in whatever order the CTAs finish; it is bounded, not compared bit for bit.

Shapes: the 32x32 tile edges (W, H in {1, 5, 6, 11, 31, 32, 33, 63, 65}), the bench frame 1920x1080, 2064x1040 and, for the
loss, the largest frame 4096x4096.  Inputs: random [0, 1], flat bright patches beside texture, unclamped [-0.3, 1.6], large
(25..75), exposed images that go negative, exact ties of img and gt.  Every plane has its own content, so a wrong plane
offset fails.  Run with -s to see max(err / bound) per output."""
import functools
import math
import zlib

import numpy as np
import pytest

import loss_reference as lr
from loss_reference import BOUND
from test_gpu_exposure import E_STAR, IDENTITY

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

DEV = "cuda:0"
LAM = 0.2
# W, H pairs covering every tile-edge value as a width and as a height, with the 1 and 31 (mod 32) edges against each other
EDGE_SHAPES = [(1, 1), (1, 65), (65, 1), (5, 33), (33, 5), (6, 63), (63, 6), (11, 31), (31, 11), (32, 32), (33, 65), (65, 33),
               (31, 63), (63, 31)]


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a, np.float32)).to(DEV)


def _np(t):
    return t.cpu().numpy()


def _report(name, ratios):
    print("\n%s: " % name + "  ".join("%s %.3f" % kv for kv in sorted(ratios.items())))
    assert max(ratios.values()) <= 1.0, ratios


def _seed(*key):
    """a fixed seed per case, so every case draws its own content"""
    return zlib.crc32(repr(key).encode())


# ---- the kernels through the C ABI --------------------------------------------------------------------------------------
def fused(a, b, dl):
    """glic_fused_ssim (map and partial maps) and glic_fused_ssim_backward fed those partial maps; a, b, dl [B,CH,H,W]"""
    from gaussian_lic_b200 import capi
    Bn, CH, H, W = a.shape
    ta, tb, td = _dev(a), _dev(b), _dev(dl)
    maps = [torch.empty_like(ta) for _ in range(4)]
    capi.check(capi.lib.glic_fused_ssim(Bn, CH, H, W, lr.C1, lr.C2, capi.ptr(ta), capi.ptr(tb), *[capi.ptr(t) for t in maps], None),
               "fused_ssim")
    g = torch.empty_like(ta)
    capi.check(capi.lib.glic_fused_ssim_backward(Bn, CH, H, W, lr.C1, lr.C2, capi.ptr(ta), capi.ptr(tb), capi.ptr(td),
                                                 *[capi.ptr(t) for t in maps[1:]], capi.ptr(g), None), "fused_ssim_backward")
    torch.cuda.synchronize()
    return dict(zip(("map", "dm_dmu1", "dm_dsigma1_sq", "dm_dsigma12", "dimg"), [_np(t) for t in maps + [g]]))


def loss(img, gt):
    """glic_l1_ssim_loss on [CH,H,W]: (loss, dL/dimg)"""
    from gaussian_lic_b200 import capi
    CH, H, W = img.shape
    ti, tg = _dev(img), _dev(gt)
    nb = capi.lib.glic_loss_scratch_bytes(CH, H, W)
    scratch = torch.empty(nb, dtype=torch.uint8, device=DEV)
    L = torch.empty(1, device=DEV)
    d = torch.empty_like(ti)
    capi.check(capi.lib.glic_l1_ssim_loss(CH, H, W, LAM, capi.ptr(ti), capi.ptr(tg), capi.ptr(L), capi.ptr(d), capi.ptr(scratch),
                                          nb, None), "l1_ssim_loss")
    torch.cuda.synchronize()
    return float(L.item()), _np(d)


def evaluate(img, gt):
    from gaussian_lic_b200 import capi
    CH, H, W = img.shape
    ti, tg = _dev(img), _dev(gt)
    nb = capi.lib.glic_eval_scratch_bytes(CH, H, W)
    scratch = torch.empty(nb, dtype=torch.uint8, device=DEV)
    out = torch.empty(2, device=DEV)
    capi.check(capi.lib.glic_eval_psnr_ssim(CH, H, W, capi.ptr(ti), capi.ptr(tg), capi.ptr(out), capi.ptr(scratch), nb, None),
               "eval_psnr_ssim")
    torch.cuda.synchronize()
    return [float(x) for x in _np(out)]


def n_cta(CH, H, W):
    return -(-W // 32) * -(-H // 32) * CH


# ---- the float64 references, once per case --------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def case(fam, P, H, W):
    a, b = lr.family(fam, P, H, W, seed=_seed(fam, P, H, W), E=E_STAR[0])
    dl = np.random.default_rng(_seed("dl", fam, P, H, W)).normal(size=a.shape).astype(np.float32)
    return a, b, dl


@functools.lru_cache(maxsize=None)
def ref_parts(fam, P, H, W):
    a, b, _ = case(fam, P, H, W)
    return lr.ssim_parts(a, b)


@functools.lru_cache(maxsize=None)
def ref_backward(fam, P, H, W):
    a, b, dl = case(fam, P, H, W)
    return lr.ssim_backward(a, b, dl, ref_parts(fam, P, H, W))


@functools.lru_cache(maxsize=None)
def ref_loss(fam, P, H, W):
    a, b, _ = case(fam, P, H, W)
    return lr.l1_ssim_loss(a, b, LAM, parts=ref_parts(fam, P, H, W))


def check_fused(fam, Bn, CH, H, W):
    a, b, dl = case(fam, Bn * CH, H, W)
    shape = (Bn, CH, H, W)
    got = fused(a.reshape(shape), b.reshape(shape), dl.reshape(shape))
    ref = dict(ref_parts(fam, Bn * CH, H, W), dimg=ref_backward(fam, Bn * CH, H, W))
    return {k: lr.err_ratio(got[k].reshape(a.shape), ref[k], BOUND[k]) for k in ref}


def check_loss(fam, CH, H, W, repeat=False):
    a, b, _ = case(fam, CH, H, W)
    L, d = loss(a, b)
    rL, rd = ref_loss(fam, CH, H, W)
    r = dict(loss=abs(L - rL.v) / rL.bound(n_cta(CH, H, W), BOUND["map"]), loss_dimg=lr.err_ratio(d, rd, BOUND["loss_dimg"]))
    if repeat:
        # dL/dimg has no atomics in its data path: a second call gives the same bits
        _, d2 = loss(a, b)
        assert np.array_equal(d.view(np.uint32), d2.view(np.uint32))
    return r


# ---- 1. SSIM map, partial maps and backward ---------------------------------------------------------------------------
@pytest.mark.parametrize("fam", lr.FAMILIES)
@pytest.mark.parametrize("WH", EDGE_SHAPES, ids=lambda s: "%dx%d" % s)
def test_fused_ssim_tile_edges_two_batches(WH, fam):
    """B = 2, CH = 3: six planes of different content at every tile-edge shape"""
    W, H = WH
    _report("fused B2 CH3 %dx%d %s" % (W, H, fam), check_fused(fam, 2, 3, H, W))


@pytest.mark.parametrize("fam", ["random", "flat", "exposed"])
@pytest.mark.parametrize("WH", [(1, 1), (31, 33), (65, 63), (97, 70)], ids=lambda s: "%dx%d" % s)
def test_fused_ssim_one_plane(WH, fam):
    W, H = WH
    _report("fused B1 CH1 %dx%d %s" % (W, H, fam), check_fused(fam, 1, 1, H, W))


FRAMES = [((1920, 1080), "random"), ((1920, 1080), "flat"), ((2064, 1040), "unclamped"), ((2064, 1040), "exposed")]


@pytest.mark.parametrize("WH,fam", FRAMES, ids=lambda v: "%dx%d" % v if isinstance(v, tuple) else v)
def test_fused_ssim_frames(WH, fam):
    W, H = WH
    _report("fused B1 CH3 %dx%d %s" % (W, H, fam), check_fused(fam, 1, 3, H, W))


# ---- 2. the L1 + D-SSIM loss -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fam", lr.FAMILIES)
@pytest.mark.parametrize("WH", [(1, 1), (5, 33), (63, 6), (31, 11), (33, 65), (65, 33)], ids=lambda s: "%dx%d" % s)
@pytest.mark.parametrize("CH", [1, 4])
def test_loss_tile_edges(CH, WH, fam):
    W, H = WH
    _report("loss CH%d %dx%d %s" % (CH, W, H, fam), check_loss(fam, CH, H, W, repeat=True))


@pytest.mark.parametrize("WH,fam", FRAMES + [((4096, 4096), "random")], ids=lambda v: "%dx%d" % v if isinstance(v, tuple) else v)
def test_loss_frames(WH, fam):
    """the bench frame and 2064x1040 with three channels; the largest frame with one (the float64 reference's one big case)"""
    W, H = WH
    CH = 1 if W == 4096 else 3
    _report("loss CH%d %dx%d %s" % (CH, W, H, fam), check_loss(fam, CH, H, W, repeat=W == 1920))


# ---- 3. the exposed loss --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fam", ["random", "unclamped", "large"])
@pytest.mark.parametrize("WH", [(1, 5), (33, 31), (200, 120)], ids=lambda s: "%dx%d" % s)
@pytest.mark.parametrize("e", range(3))
def test_exposed_loss(e, WH, fam):
    from gaussian_lic_b200 import ops
    W, H = WH
    img, gt = lr.family(fam, 3, H, W, seed=_seed("expo", fam, H, W, e))
    E = E_STAR[e]
    L, dimg, dE = ops.l1_ssim_loss_exposure(_dev(img), _dev(gt), _dev(E), LAM)
    torch.cuda.synchronize()
    rL, rdimg, jimg, rdE, jE = lr.l1_ssim_loss_exposure(img, gt, E, LAM)
    _report("exposed E%d %dx%d %s" % (e, W, H, fam),
            dict(loss=abs(float(L.item()) - rL.v) / rL.bound(n_cta(3, H, W), BOUND["map"]),
                 loss_dimg=lr.err_ratio(_np(dimg), rdimg, BOUND["loss_dimg"], jimg),
                 dE=lr.err_ratio(_np(dE).reshape(3, 4), rdE, BOUND["loss_dimg"], jE)))


# ---- 4. known answers -----------------------------------------------------------------------------------------------------
def test_identical_images():
    """SSIM(x, x) = 1 in exact arithmetic.  The kernel does not return exactly 1.0: nvcc contracts sigma1^2 and sigma2^2 to
    fmaf(-mu, mu, E[x^2]) but computes sigma12 as E[xy] - fl(mu1 mu2), the rounded product it shares with Cq (sm_90a SASS of
    ssim_forward_kernel), so B and Dq can differ in the last bit (Cq and A do agree: fmaf(mu1, mu1, fl(mu1^2)) rounds to
    2 fl(mu1^2)).  So the map is held to its bound around 1, as is the loss gradient, which has no L1 term (the sign is 0)."""
    a, _, dl = case("unclamped", 6, 65, 70)
    got = fused(a.reshape(2, 3, 65, 70), a.reshape(2, 3, 65, 70), dl.reshape(2, 3, 65, 70))
    ref = lr.ssim_parts(a, a)
    assert np.all(ref["map"].v == 1.0)
    r = {k: lr.err_ratio(got[k].reshape(a.shape), ref[k], BOUND[k]) for k in ref}
    L, d = loss(a[:3], a[:3])
    rL, rd = lr.l1_ssim_loss(a[:3], a[:3], LAM)
    assert abs(rL.v) < 1e-15
    r["loss"] = abs(L - rL.v) / rL.bound(n_cta(3, 65, 70), BOUND["map"])
    r["loss_dimg"] = lr.err_ratio(d, rd, BOUND["loss_dimg"])
    _report("identical", r)


@pytest.mark.parametrize("where", ["frame_corner", "far_corner", "tile_corner", "tile_edge_mid", "tile_edge_mid_y"])
def test_one_hot_backward_is_an_11x11_stencil(where):
    """dL/dmap one at a single pixel: dL/dimg is that pixel's 11x11 neighbourhood (clipped to the frame), exact zeros outside,
    and within its bound inside.  A halo or tile-seam mistake moves or loses part of the stencil."""
    H, W = 70, 100
    y, x = dict(frame_corner=(0, 0), far_corner=(H - 1, W - 1), tile_corner=(31, 32), tile_edge_mid=(16, 63),
                tile_edge_mid_y=(64, 47))[where]
    a, b, _ = case("random", 3, H, W)
    dl = np.zeros(a.shape, np.float32)
    dl[1, y, x] = 1.0                                      # the middle plane: a plane offset mistake reads another's zeros
    got = fused(a[None], b[None], dl[None])["dimg"][0]
    ref = lr.ssim_backward(a, b, dl, ref_parts("random", 3, H, W))
    inside = np.zeros(a.shape, bool)
    inside[1, max(0, y - 5):y + 6, max(0, x - 5):x + 6] = True
    assert np.all(got[~inside] == 0.0)
    assert np.all(got[inside] != 0.0)
    _report("one-hot %s" % where, dict(dimg=lr.err_ratio(got, ref, BOUND["dimg"])))


@pytest.mark.parametrize("CH", [1, 3])
def test_eval_psnr_ssim(CH):
    """identical images: PSNR +inf and SSIM within its bound of 1; otherwise both within their bounds of the float64
    scores of the clamped images"""
    r = {}
    for fam in ("random", "flat", "unclamped", "exposed", "ties"):
        for W, H in ((33, 31), (200, 120)):
            a, b, _ = case(fam, CH, H, W)
            psnr, ssim = evaluate(a, b)
            rp, rs = lr.eval_psnr_ssim(a, b)
            r["psnr"] = max(r.get("psnr", 0.0), lr.err_ratio(psnr, rp, BOUND["psnr"]))
            r["ssim"] = max(r.get("ssim", 0.0), lr.err_ratio(ssim, rs, BOUND["map"]))
            psnr, ssim = evaluate(a, a)
            rp, rs = lr.eval_psnr_ssim(a, a)
            assert psnr == math.inf and rp.v == math.inf
            r["ssim_identical"] = max(r.get("ssim_identical", 0.0), lr.err_ratio(ssim, rs, BOUND["map"]))
    _report("eval CH%d" % CH, r)


def test_evaluate_exposed_keyframe():
    """the exposed evaluation (glic_mapper_evaluate of a training keyframe with E set): PSNR and SSIM of clamp(E render)
    against the keyframe image, and the scored image itself, within their bounds of the float64 exposure of the render"""
    from gaussian_lic_b200 import mapper, synthetic as syn
    from test_gpu_exposure import F, H, W, _keyframes, _render, _scene
    raw = _scene(2)
    poses, cams, _ = _keyframes()
    img = _render(raw, cams)[1]
    gt = syn.make_gt_image(W, H, seed=3).astype(np.float32)
    m = mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=2)
    try:
        m.initialize(raw)
        m.add_keyframe(*poses[0], np.zeros_like(gt))
        m.add_keyframe(*poses[1], gt)
        m.enable_exposure(0.001)
        r = {}
        for e, E in enumerate(E_STAR + [IDENTITY]):
            m.set_exposure(1, E)
            psnr, ssim = m.evaluate(1, train=True)
            scored = m.render(1, train=True)
            rp, rs = lr.eval_psnr_ssim(img, gt, E)
            x = lr.expose(lr.Mag(img), E)
            rimg = lr.Mag(np.clip(x.v, 0.0, 1.0), x.m)
            r["psnr"] = max(r.get("psnr", 0.0), lr.err_ratio(psnr, rp, BOUND["psnr"]))
            r["ssim"] = max(r.get("ssim", 0.0), lr.err_ratio(ssim, rs, BOUND["map"]))
            # the exposure's three fmaf roundings, each at most 2^-24 of the running magnitude
            r["image"] = max(r.get("image", 0.0), lr.err_ratio(scored, rimg, 4.0))
    finally:
        m.close()
    _report("evaluate exposed", r)


# ---- 5. argument checks ---------------------------------------------------------------------------------------------------
def test_too_many_planes_refused_before_any_launch():
    """gridDim.z holds at most 65535 planes: B*CH beyond that (or beyond int) is refused before anything is enqueued, on a
    1x1 frame whose buffers are never read; 65535 planes still run"""
    from gaussian_lic_b200 import capi
    t = torch.zeros(65535 * 4, device=DEV)
    p = capi.ptr(t)
    for Bn, CH in ((1, 65536), (65536, 1), (256, 257), (2, 2 ** 30), (65536, 65536)):
        n0 = capi.launch_count()
        assert capi.lib.glic_fused_ssim(Bn, CH, 1, 1, lr.C1, lr.C2, p, p, p, None, None, None, None) != capi.GLIC_OK
        assert b"65535" in capi.lib.glic_last_error()
        assert capi.lib.glic_fused_ssim_backward(Bn, CH, 1, 1, lr.C1, lr.C2, p, p, p, p, p, p, p, None) != capi.GLIC_OK
        assert capi.launch_count() == n0
    n0 = capi.launch_count()
    assert capi.lib.glic_l1_ssim_loss(65536, 1, 1, LAM, p, p, p, p, p, 1 << 40, None) != capi.GLIC_OK
    assert capi.launch_count() == n0
    a = torch.rand(65535, device=DEV)
    b = torch.rand(65535, device=DEV)
    out = torch.empty(65535, device=DEV)
    capi.check(capi.lib.glic_fused_ssim(65535, 1, 1, 1, lr.C1, lr.C2, capi.ptr(a), capi.ptr(b), capi.ptr(out), None, None, None,
                                        None), "fused_ssim")
    torch.cuda.synchronize()
    ref = lr.ssim_parts(_np(a).reshape(-1, 1, 1), _np(b).reshape(-1, 1, 1))["map"]
    _report("65535 planes", dict(map=lr.err_ratio(_np(out).reshape(-1, 1, 1), ref, BOUND["map"])))
