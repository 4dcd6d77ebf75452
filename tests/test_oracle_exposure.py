"""The CPU restatement of the per-image exposure (exposure_oracle.py: loss, gradients and Adam step in the oracle's float32 /
float64 arithmetic) against finite differences and a plain float64 numpy statement of the formulas, and the argument checks of
the new C entry points.  No GPU needed.

Exposure: E is 3x4 row-major, out_c = E[0][c] r + E[1][c] g + E[2][c] b + E[c][3] (Inria 3DGS's matmul(img_hwc, E[:3,:3]) +
E[:3,3]).  Every E used here is asymmetric: a transposed 3x3 block would pass on a symmetric one."""
import ctypes as C

import numpy as np
import pytest

from exposure_oracle import exposure_adam, loss_exposure

H, W = 37, 53                                            # not a multiple of the 32-pixel tile
E_ASYM = np.array([[1.12, 0.05, -0.03, 0.04],
                   [-0.02, 0.91, 0.07, -0.03],
                   [0.06, -0.04, 1.05, 0.02]])
IDENTITY = np.hstack([np.eye(3), np.zeros((3, 1))])


def _images(seed=4):
    rng = np.random.default_rng(seed)
    gt = rng.uniform(0.05, 0.95, (3, H, W))
    img = np.clip(gt + 0.15 * rng.normal(size=gt.shape), 0.0, 1.2)
    return img, gt


def _expose(img, E):
    return np.einsum("khw,kc->chw", img, E[:, :3]) + E[:, 3][:, None, None]


def test_exposed_loss_is_the_loss_of_the_exposed_image(oracle64):
    img, gt = _images()
    L, _, _ = loss_exposure(oracle64, img, gt, E_ASYM, grad=False)
    L_ref, _ = oracle64.loss(_expose(img, E_ASYM), gt, grad=False)
    assert abs(L - L_ref) <= 1e-14 * L_ref, (L, L_ref)
    L_t, _, _ = loss_exposure(oracle64, img, gt, np.hstack([E_ASYM[:, :3].T, E_ASYM[:, 3:]]), grad=False)
    assert abs(L_t - L) > 1e-4 * L                       # the transposed 3x3 block is a different loss on this E


def test_gradients_match_central_differences(oracle64):
    """f64 central differences of the exposed loss against the analytic dL/dE (all 12 entries) and a sample of dL/dimg"""
    img, gt = _images()
    L0, g_img, g_E = loss_exposure(oracle64, img, gt, E_ASYM)
    h = 1e-6
    fd = np.zeros((3, 4))
    for k in range(3):
        for c in range(4):
            Ep, Em = E_ASYM.copy(), E_ASYM.copy()
            Ep[k, c] += h
            Em[k, c] -= h
            fd[k, c] = (loss_exposure(oracle64, img, gt, Ep, grad=False)[0] - loss_exposure(oracle64, img, gt, Em, grad=False)[0]) / (2 * h)
    err = np.abs(fd - g_E).max() / np.abs(g_E).max()
    print("dL/dE: analytic %s\nmax|fd - analytic| / max|analytic| = %.2e" % (g_E, err))
    assert err < 1e-5, (fd, g_E)
    rng = np.random.default_rng(1)
    idx = [(int(rng.integers(3)), int(rng.integers(H)), int(rng.integers(W))) for _ in range(24)] + [(0, 0, 0), (2, H - 1, W - 1)]
    scale = np.abs(g_img).max()
    worst = 0.0
    for k, y, x in idx:
        ip, im = img.copy(), img.copy()
        ip[k, y, x] += h
        im[k, y, x] -= h
        f = (loss_exposure(oracle64, ip, gt, E_ASYM, grad=False)[0] - loss_exposure(oracle64, im, gt, E_ASYM, grad=False)[0]) / (2 * h)
        worst = max(worst, abs(f - g_img[k, y, x]) / scale)
    print("dL/dimg: max|fd - analytic| / max|analytic| over %d entries = %.2e" % (len(idx), worst))
    assert worst < 1e-4


def test_identity_f32_equals_the_plain_loss(oracle32):
    """E = [I | 0] gives out == img exactly, so the f32 oracle's loss and dL/dimg are those of oracle.loss, value for value"""
    img, gt = (x.astype(np.float32) for x in _images(seed=9))
    L, g, _ = loss_exposure(oracle32, img, gt, IDENTITY)
    L_ref, g_ref = oracle32.loss(img, gt)
    assert L == L_ref
    assert np.array_equal(g, g_ref)                     # +0 and -0 compare equal


def _adam_numpy(E, m, v, t, g, lr, dtype):
    """float64 restatement; the betas and 1 - beta are the values the arithmetic of `dtype` holds (0.999f, 1 - 0.999f =
    0.0010000467 in float32), the bias corrections use the float64 betas as LibTorch computes them"""
    b1, b2 = (np.float64(dtype(x)) for x in (0.9, 0.999))
    c1, c2 = (np.float64(dtype(1.0) - dtype(x)) for x in (0.9, 0.999))
    t += 1
    m = b1 * m + c1 * g
    v = b2 * v + c2 * g * g
    denom = np.sqrt(v) / np.sqrt(1 - 0.999 ** t) + np.float64(dtype(1e-8))
    return E - (lr / (1 - 0.9 ** t)) * m / denom, m, v, t


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_three_adam_steps_match_numpy(oracle32, oracle64, dtype):
    o = oracle32 if dtype == "float32" else oracle64
    rng = np.random.default_rng(5)
    lr = 0.001
    E = E_ASYM.astype(o.dtype)
    m = v = np.zeros((3, 4), o.dtype)
    En, mn, vn, tn = E_ASYM.copy(), np.zeros((3, 4)), np.zeros((3, 4)), 0
    t = 0
    for step in range(3):
        g = (rng.normal(size=(3, 4)) * 10.0 ** rng.uniform(-4, -1, (3, 4))).astype(o.dtype)
        E0 = E.copy()
        E, m, v, t = exposure_adam(o, E, m, v, t, g, lr)
        En, mn, vn, tn = _adam_numpy(En, mn, vn, tn, g.astype(np.float64), lr, o.dtype.type)
        assert t == tn == step + 1
        if step == 0:                                    # bias correction: the first step moves every entry by ~lr against g
            np.testing.assert_allclose(E - E0, -lr * np.sign(g), rtol=1e-4)
        tol = 1e-6 if dtype == "float32" else 1e-13
        np.testing.assert_allclose(E, En, rtol=0, atol=tol * lr * 10 + (2e-7 if dtype == "float32" else 1e-15))
        np.testing.assert_allclose(m, mn, rtol=tol, atol=0)
        np.testing.assert_allclose(v, vn, rtol=tol, atol=0)


def test_exposure_entry_points_validate_without_gpu():
    from gaussian_lic_b200 import capi
    lib = capi.lib
    assert lib.glic_loss_exposure_scratch_bytes(0, 64) == 0 and lib.glic_loss_exposure_scratch_bytes(48, -1) == 0
    need = lib.glic_loss_exposure_scratch_bytes(48, 64)
    assert need >= 9 * 4 * 48 * 64 + 12 * 8 and lib.glic_loss_exposure_scratch_bytes(96, 64) > need
    p = C.c_void_p(256)                                  # never dereferenced: every call below fails its checks first
    call = lib.glic_l1_ssim_loss_exposure
    assert call(0, 64, 0.2, p, p, p, p, p, p, p, need, None) == -1
    assert call(48, 64, 0.2, None, p, p, p, p, p, p, need, None) == -1
    assert call(48, 64, 0.2, p, p, None, p, p, p, p, need, None) == -1 and b"bad arguments" in lib.glic_last_error()
    assert call(48, 64, 0.2, p, p, p, p, p, None, p, need, None) == -1 and b"both" in lib.glic_last_error()
    assert call(48, 64, 0.2, p, p, p, p, None, p, p, need, None) == -1 and b"both" in lib.glic_last_error()
    assert call(48, 64, 0.2, p, p, p, p, p, p, p, need - 1, None) == -2 and b"scratch" in lib.glic_last_error()
    e12 = (C.c_float * 12)()
    assert lib.glic_mapper_enable_exposure(None, 0.001) == -1
    assert lib.glic_mapper_exposure_get(None, 0, e12) == -1
    assert lib.glic_mapper_exposure_set(None, 0, e12) == -1 and b"null" in lib.glic_last_error()
