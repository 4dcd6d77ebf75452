"""The masked loss and evaluation kernels of csrc/ssim.cu (glic_pack_mask, glic_l1_ssim_loss_masked, glic_eval_psnr_ssim_masked)
against the float64 restatement of tests/loss_mask_reference.py, each element within its own bound |got - ref| <= c 2^-24 M
(c from loss_reference.BOUND), and against the unmasked kernels bit for bit where the mask is all ones.

Masks: random, one valid pixel, a one-pixel valid border, a masked block on the 32x32 tile grid and one across tile seams, and
views of a wider mask with a column offset (glic_mapper_align's crops).  Forms: plain, exposed (E), fixed-order loss sum."""
import functools
import math
import zlib

import numpy as np
import pytest

import loss_mask_reference as mr
import loss_reference as lr
from loss_reference import BOUND
from test_gpu_exposure import E_STAR

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

DEV = "cuda:0"
LAM = 0.2
SHAPES = [(1, 1), (5, 33), (63, 6), (31, 11), (33, 65), (65, 33), (97, 70)]
FORMS = ["plain", "exposed", "fixed"]


def _dev(a, dtype=np.float32):
    return torch.as_tensor(np.ascontiguousarray(a, dtype)).to(DEV)


def _seed(*key):
    return zlib.crc32(repr(key).encode())


def pack(mask):
    """glic_pack_mask of a [H,W] mask -> (device words, count read back, words as numpy)"""
    from gaussian_lic_b200 import capi
    H, W = mask.shape
    wpr = capi.lib.glic_mask_words_per_row(W)
    v = _dev(np.asarray(mask, np.uint8), np.uint8)
    words = torch.empty(H * wpr, dtype=torch.int32, device=DEV)
    cnt = torch.empty(1, dtype=torch.int32, device=DEV)
    capi.check(capi.lib.glic_pack_mask(H, W, capi.ptr(v), capi.ptr(words), capi.ptr(cnt), None), "pack_mask")
    torch.cuda.synchronize()
    return words, int(cnt.item()), words.cpu().numpy().view(np.uint32).reshape(H, wpr)


def loss(img, gt, words=None, wpr=0, x0=0, count=0, E=None, fixed=False):
    """glic_l1_ssim_loss_masked on [3,H,W] -> (loss, dL/dimg, dL/dE or None); words None: the unmasked form"""
    from gaussian_lic_b200 import capi
    _, H, W = img.shape
    ti, tg = _dev(img), _dev(gt)
    nb = capi.lib.glic_loss_masked_scratch_bytes(H, W)
    scratch = torch.empty(nb, dtype=torch.uint8, device=DEV)
    L = torch.empty(1, device=DEV)
    d = torch.empty_like(ti)
    tE = _dev(E) if E is not None else None
    dE = torch.empty(12, device=DEV) if E is not None else None
    capi.check(capi.lib.glic_l1_ssim_loss_masked(H, W, LAM, capi.ptr(ti), capi.ptr(tg), capi.ptr(tE), capi.ptr(words), wpr, x0, count,
                                                 int(fixed), capi.ptr(L), capi.ptr(d), capi.ptr(dE), capi.ptr(scratch), nb, None),
               "l1_ssim_loss_masked")
    torch.cuda.synchronize()
    return float(L.item()), d.cpu().numpy(), None if dE is None else dE.cpu().numpy().reshape(3, 4)


def evaluate(img, gt, words=None, wpr=0, x0=0, count=0, E=None, fixed=False):
    from gaussian_lic_b200 import capi
    CH, H, W = img.shape
    ti, tg = _dev(img), _dev(gt)
    nb = capi.lib.glic_eval_masked_scratch_bytes(CH, H, W)
    scratch = torch.empty(nb, dtype=torch.uint8, device=DEV)
    out = torch.empty(2, device=DEV)
    tE = _dev(E) if E is not None else None
    capi.check(capi.lib.glic_eval_psnr_ssim_masked(CH, H, W, capi.ptr(ti), capi.ptr(tg), capi.ptr(tE), capi.ptr(words), wpr, x0, count,
                                                   int(fixed), capi.ptr(out), capi.ptr(scratch), nb, None), "eval_psnr_ssim_masked")
    torch.cuda.synchronize()
    return [float(x) for x in out.cpu().numpy()]


def n_cta(H, W):
    return -(-W // 32) * -(-H // 32) * 3


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _check(form, img, gt, w, words, wpr, x0, count):
    """max err / bound of the kernel against the restatement, and dL/dimg = +0 at every masked pixel"""
    E = E_STAR[0] if form == "exposed" else None
    L, d, dE = loss(img, gt, words, wpr, x0, count, E=E, fixed=form == "fixed")
    if E is None:
        rL, rd = mr.l1_ssim_loss_masked(img, gt, w, LAM)
        r = dict(loss=abs(L - rL.v) / rL.bound(n_cta(*w.shape), BOUND["map"]), loss_dimg=lr.err_ratio(d, rd, BOUND["loss_dimg"]))
        assert np.all(_bits(d)[:, ~w] == 0)                              # +0, not -0
    else:
        rL, rd, jd, rE, jE = mr.l1_ssim_loss_exposure_masked(img, gt, E, w, LAM)
        r = dict(loss=abs(L - rL.v) / rL.bound(n_cta(*w.shape), BOUND["map"]), loss_dimg=lr.err_ratio(d, rd, BOUND["loss_dimg"], jd),
                 dE=lr.err_ratio(dE, rE, BOUND["loss_dimg"], jE))
    return r


def _report(name, r):
    print("\n%s: " % name + "  ".join("%s %.3f" % kv for kv in sorted(r.items())))
    assert max(r.values()) <= 1.0, r


# ---- 1. packing ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("HW", [(1, 1), (3, 31), (7, 32), (5, 33), (9, 70), (1080, 1920), (33, 1921)], ids=lambda s: "%dx%d" % s)
def test_pack_matches_numpy(HW):
    H, W = HW
    for name in ("random", "one_pixel", "border", "ones"):
        w = mr.mask_family(name, H, W, seed=_seed("pack", H, W, name))
        _, n, got = pack(w)
        want, wn = mr.pack(w)
        assert n == wn and np.array_equal(got, want), name


# ---- 2. the masked loss against the restatement -----------------------------------------------------------------------------
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("mask", mr.MASKS)
@pytest.mark.parametrize("HW", SHAPES, ids=lambda s: "%dx%d" % s)
def test_masked_loss_matches_restatement(HW, mask, form):
    H, W = HW
    img, gt = lr.family("random", 3, H, W, seed=_seed("img", H, W, mask))
    w = mr.mask_family(mask, H, W, seed=_seed("mask", H, W, mask))
    words, n, _ = pack(w)
    _report("%s %s %dx%d" % (form, mask, W, H), _check(form, img, gt, w, words, (W + 31) // 32, 0, n))


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("x0", [1, 17, 32, 45])
def test_masked_loss_on_a_column_crop(x0, form):
    """a view of a wider frame's mask from column x0 (the crop's own mask is that frame's columns [x0, x0 + W))"""
    H, W, Wf = 70, 61, 130
    img, gt = lr.family("unclamped", 3, H, W, seed=_seed("crop", x0))
    wf = mr.mask_family("random", H, Wf, seed=_seed("cropmask", x0)) | mr.mask_family("straddle", H, Wf, seed=1)
    words, _, _ = pack(wf)
    w = wf[:, x0:x0 + W]
    _report("crop %s x0=%d" % (form, x0), _check(form, img, gt, w, words, (Wf + 31) // 32, x0, int(w.sum())))


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("mask", ["random", "straddle"])
def test_masked_loss_full_frame(mask, form):
    H, W = 1080, 1920
    img, gt = lr.family("random", 3, H, W, seed=_seed("full", mask))
    w = mr.mask_family(mask, H, W, seed=_seed("fullmask", mask))
    words, n, _ = pack(w)
    _report("full %s %s" % (form, mask), _check(form, img, gt, w, words, (W + 31) // 32, 0, n))


# ---- 3. bits -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("HW", [(1, 1), (33, 65), (1080, 1920)], ids=lambda s: "%dx%d" % s)
def test_all_ones_mask_is_the_unmasked_loss_bit_for_bit(HW, form):
    H, W = HW
    img, gt = lr.family("random", 3, H, W, seed=_seed("ones", H, W))
    words, n, _ = pack(np.ones((H, W), bool))
    E = E_STAR[1] if form == "exposed" else None
    fixed = form == "fixed"
    L0, d0, e0 = loss(img, gt, E=E, fixed=fixed)
    L1, d1, e1 = loss(img, gt, words, (W + 31) // 32, 0, n, E=E, fixed=fixed)
    assert np.array_equal(_bits(d0), _bits(d1))
    if E is not None:
        assert np.array_equal(_bits(e0), _bits(e1))
    if fixed:
        assert _bits(L0) == _bits(L1)
    p0 = evaluate(img, gt, fixed=True)
    p1 = evaluate(img, gt, words, (W + 31) // 32, 0, n, fixed=True)
    assert _bits(p0).tolist() == _bits(p1).tolist()


@pytest.mark.parametrize("form", FORMS)
def test_values_under_the_mask_leave_every_bit(form):
    """NaN, infinities and huge values in gt (and, without exposure, in img) under the mask give the bits of zeros there.  With
    exposure the rendered image under the mask still meets dL/dE through dL/dout = 0, so there it is huge but finite."""
    H, W = 100, 77
    img, gt = lr.family("random", 3, H, W, seed=_seed("nan", form))
    w = mr.mask_family("straddle", H, W, seed=2) & mr.mask_family("random", H, W, seed=3)
    words, n, _ = pack(w)
    rng = np.random.default_rng(4)
    img0, gt0 = img.copy(), gt.copy()
    img0[:, ~w] = 0
    gt0[:, ~w] = 0
    bad = rng.choice(np.array([np.nan, np.inf, -np.inf, 3e38, -3e38], np.float32), size=gt[:, ~w].shape)
    img1, gt1 = img.copy(), gt.copy()
    gt1[:, ~w] = bad
    img1[:, ~w] = rng.uniform(-3e38, 3e38, img1[:, ~w].shape) if form == "exposed" else bad
    E = E_STAR[2] if form == "exposed" else None
    fixed = form == "fixed"
    L0, d0, e0 = loss(img0, gt0, words, (W + 31) // 32, 0, n, E=E, fixed=fixed)
    L1, d1, e1 = loss(img1, gt1, words, (W + 31) // 32, 0, n, E=E, fixed=fixed)
    assert np.array_equal(_bits(d0), _bits(d1))
    if E is None:
        assert np.all(_bits(d1)[:, ~w] == 0)
    else:
        assert np.array_equal(_bits(e0), _bits(e1))
    if fixed:
        assert _bits(L0) == _bits(L1)
    assert _bits(evaluate(img0, gt0, words, (W + 31) // 32, 0, n, fixed=True)).tolist() == \
        _bits(evaluate(img1 if E is None else img0, gt1, words, (W + 31) // 32, 0, n, fixed=True)).tolist()


def test_empty_mask_refused_before_any_launch():
    from gaussian_lic_b200 import capi
    lib = capi.lib
    before = capi.launch_count()
    t = torch.zeros(3 * 8 * 8, device=DEV)
    words = torch.zeros(8, dtype=torch.int32, device=DEV)
    nb = lib.glic_loss_masked_scratch_bytes(8, 8)
    scratch = torch.empty(nb, dtype=torch.uint8, device=DEV)
    p = capi.ptr(t)
    assert lib.glic_l1_ssim_loss_masked(8, 8, LAM, p, p, None, capi.ptr(words), 1, 0, 0, 0, p, p, None, capi.ptr(scratch), nb, None) == -1
    assert b"no valid pixel" in lib.glic_last_error()
    assert lib.glic_l1_ssim_loss_masked(8, 8, LAM, p, p, None, capi.ptr(words), 1, 25, 5, 0, p, p, None, capi.ptr(scratch), nb, None) == -1
    eb = lib.glic_eval_masked_scratch_bytes(3, 8, 8)
    es = torch.empty(eb, dtype=torch.uint8, device=DEV)
    assert lib.glic_eval_psnr_ssim_masked(3, 8, 8, p, p, None, capi.ptr(words), 1, 0, 0, 0, p, capi.ptr(es), eb, None) == -1
    assert capi.launch_count() == before


# ---- 4. the masked evaluation ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fixed", [False, True])
def test_masked_evaluation_matches_restatement(fixed):
    r = {}
    for fam in ("random", "unclamped", "ties"):
        for (W, H) in ((33, 31), (200, 120)):
            for mask in mr.MASKS:
                img, gt = lr.family(fam, 3, H, W, seed=_seed("eval", fam, W, H, mask))
                w = mr.mask_family(mask, H, W, seed=_seed("evalmask", W, H, mask))
                words, n, _ = pack(w)
                for E in (None, E_STAR[0]):
                    psnr, ssim = evaluate(img, gt, words, (W + 31) // 32, 0, n, E=E, fixed=fixed)
                    rp, rs = mr.eval_psnr_ssim_masked(img, gt, w, E)
                    if math.isinf(rp.v):
                        assert psnr == math.inf
                    else:
                        r["psnr"] = max(r.get("psnr", 0.0), lr.err_ratio(psnr, rp, BOUND["psnr"]))
                    r["ssim"] = max(r.get("ssim", 0.0), lr.err_ratio(ssim, rs, BOUND["map"]))
    _report("masked eval fixed=%d" % fixed, r)
