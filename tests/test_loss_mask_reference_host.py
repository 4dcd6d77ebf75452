"""The float64 restatement of the masked loss and evaluation (tests/loss_mask_reference.py) checked on its own, without a GPU:
an all-ones mask gives the unmasked restatement, its dL/dimg is the derivative of its own loss (central differences), nothing
under the mask changes any output, and the packed layout is numpy's packbits."""
import numpy as np
import pytest

import loss_mask_reference as mr
import loss_reference as lr
from test_gpu_exposure import E_STAR

LAM = 0.2


def _case(H, W, seed, E=None):
    return lr.family("random", 3, H, W, seed=seed, E=E)


@pytest.mark.parametrize("HW", [(1, 1), (7, 9), (40, 37)], ids=lambda s: "%dx%d" % s)
def test_all_ones_mask_is_the_unmasked_restatement(HW):
    H, W = HW
    a, b = _case(H, W, 1)
    ones = np.ones((H, W), bool)
    L, d = mr.l1_ssim_loss_masked(a, b, ones, LAM)
    rL, rd = lr.l1_ssim_loss(a, b, LAM)
    assert L.v == pytest.approx(rL.v, rel=1e-14, abs=1e-15)
    np.testing.assert_allclose(d.v, rd.v, rtol=1e-12, atol=1e-18)
    np.testing.assert_allclose(d.m, rd.m, rtol=1e-12, atol=1e-18)
    eL, ed, ej, eE, eEj = mr.l1_ssim_loss_exposure_masked(a, b, E_STAR[0], ones, LAM)
    rL, red, rej, reE, reEj = lr.l1_ssim_loss_exposure(a, b, E_STAR[0], LAM)
    assert eL.v == pytest.approx(rL.v, rel=1e-14, abs=1e-15)
    np.testing.assert_allclose(ed.v, red.v, rtol=1e-12, atol=1e-18)
    np.testing.assert_allclose(eE.v, reE.v, rtol=1e-12, atol=1e-15)
    np.testing.assert_array_equal(ej, rej)
    p, s = mr.eval_psnr_ssim_masked(a, b, ones)
    rp, rs = lr.eval_psnr_ssim(a, b)
    assert p.v == pytest.approx(rp.v, rel=1e-13) and s.v == pytest.approx(rs.v, rel=1e-13)


@pytest.mark.parametrize("mask", mr.MASKS)
def test_gradient_is_the_derivative_of_the_loss(mask):
    """central differences of the float64 loss at used pixels away from an L1 kink; zero at masked pixels"""
    H, W = 12, 14
    a, b = _case(H, W, 2)
    w = mr.mask_family(mask, H, W, seed=3)
    _, d = mr.l1_ssim_loss_masked(a, b, w, LAM)
    rng = np.random.default_rng(4)
    a64 = a.astype(np.float64)
    h = 1e-6
    picks = [tuple(int(v) for v in (rng.integers(0, 3), rng.integers(0, H), rng.integers(0, W))) for _ in range(12)]
    for c, y, x in picks:
        if abs(a64[c, y, x] - b[c, y, x]) < 10 * h:
            continue
        ap, am = a64.copy(), a64.copy()
        ap[c, y, x] += h
        am[c, y, x] -= h
        fd = (mr.l1_ssim_loss_masked(ap, b, w, LAM)[0].v - mr.l1_ssim_loss_masked(am, b, w, LAM)[0].v) / (2 * h)
        if w[y, x]:
            assert d.v[c, y, x] == pytest.approx(fd, rel=1e-5, abs=1e-9), (c, y, x)
        else:
            assert d.v[c, y, x] == 0.0 and abs(fd) < 1e-12
    # the exposed form: dL/dE against differences in E (the restatement takes E as float32: a step of 2^-17 is exact there)
    E = np.asarray(E_STAR[1], np.float32)
    _, _, _, dE, _ = mr.l1_ssim_loss_exposure_masked(a, b, E, w, LAM)
    hE = 2.0 ** -17
    for k, c in ((0, 0), (1, 2), (2, 3)):
        Ep, Em = E.copy(), E.copy()
        Ep[k, c] += np.float32(hE)
        Em[k, c] -= np.float32(hE)
        fd = (mr.l1_ssim_loss_exposure_masked(a, b, Ep, w, LAM)[0].v - mr.l1_ssim_loss_exposure_masked(a, b, Em, w, LAM)[0].v) / (2 * hE)
        assert dE.v[k, c] == pytest.approx(fd, rel=1e-3, abs=1e-7), (k, c)


@pytest.mark.parametrize("mask", mr.MASKS)
def test_values_under_the_mask_change_nothing(mask):
    H, W = 20, 35
    a, b = _case(H, W, 5)
    w = mr.mask_family(mask, H, W, seed=6)
    rng = np.random.default_rng(7)
    a2, b2 = a.copy(), b.copy()
    a2[:, ~w] = rng.uniform(-1e30, 1e30, a2[:, ~w].shape)
    b2[:, ~w] = rng.uniform(-5, 5, b2[:, ~w].shape)
    L, d = mr.l1_ssim_loss_masked(a, b, w, LAM)
    L2, d2 = mr.l1_ssim_loss_masked(a2, b2, w, LAM)
    assert L.v == L2.v and L.terms == L2.terms
    np.testing.assert_array_equal(d.v, d2.v)
    np.testing.assert_array_equal(d.m, d2.m)
    out = mr.l1_ssim_loss_exposure_masked(a, b, E_STAR[2], w, LAM)
    out2 = mr.l1_ssim_loss_exposure_masked(a2, b2, E_STAR[2], w, LAM)
    assert out[0].v == out2[0].v
    for q in (1, 3):
        np.testing.assert_array_equal(out[q].v, out2[q].v)
    assert mr.eval_psnr_ssim_masked(a, b, w)[1].v == mr.eval_psnr_ssim_masked(a2, b2, w)[1].v


@pytest.mark.parametrize("W", [1, 31, 32, 33, 64, 70])
def test_pack_layout(W):
    H = 5
    w = mr.mask_family("random", H, W, seed=W)
    words, n = mr.pack(w)
    assert words.shape == (H, (W + 31) // 32) and n == int(w.sum())
    for y in range(H):
        for x in range(W):
            assert bool((int(words[y, x >> 5]) >> (x & 31)) & 1) == w[y, x]
    if W % 32:
        assert np.all(words[:, -1] >> np.uint32(W % 32) == 0)              # pad bits are 0
