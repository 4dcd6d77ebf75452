"""CPU checks of tests/loss_reference.py, the float64 restatement the GPU loss tests compare against.

1. The restatement is the SSIM of the conv2d formulation: its map, loss and dL/dimg agree with torch float64 autograd to
   about 1e-12 relative.
2. Its bounds hold for a float32 emulation of the kernels' arithmetic order (fmaf chains of the separable passes, the
   quotients as ssim.cu writes them, the exposure's fma order), on every input family: the constants c in loss_reference.BOUND
   are fixed by the arithmetic, not fitted to a GPU run.  The max(err / bound) of each output is printed (-s)."""
import numpy as np
import pytest

import loss_reference as lr
from test_gpu_exposure import E_STAR

torch = pytest.importorskip("torch")

f32 = np.float32
G32 = lr.G.astype(np.float32)


def fma32(a, b, c):
    """fmaf: the float64 product of two floats is exact; the add rounds in float64, then to float32 (a double rounding the
    real fmaf does not make, at most 1 ulp apart and only on exact float64 midpoints)"""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)


def conv32(a):
    """the kernels' two 11-tap passes: acc = fmaf(g[k], v[k], acc), k = 0..10, horizontal then vertical, zero padding"""
    H, W = a.shape[-2:]
    lead = [(0, 0)] * (a.ndim - 2)
    p = np.pad(a, lead + [(0, 0), (5, 5)])
    acc = np.zeros(a.shape, np.float32)
    for k in range(11):
        acc = fma32(G32[k], p[..., k:k + W], acc)
    p = np.pad(acc, lead + [(5, 5), (0, 0)])
    out = np.zeros(a.shape, np.float32)
    for k in range(11):
        out = fma32(G32[k], p[..., k:k + H, :], out)
    return out


def forward32(x, y, c1=lr.C1, c2=lr.C2):
    """ssim_forward_tile's float32 arithmetic as nvcc compiles it for sm_90a: sigma1^2 and sigma2^2 contracted to
    fmaf(-mu, mu, E[x^2]), sigma12 = E[xy] - fl(mu1 mu2) (the rounded product Cq shares), A = fmaf(mu1, mu1, fl(mu2^2)) + C1;
    the quotients in source order"""
    c1, c2, two = f32(c1), f32(c2), f32(2.0)
    mu1, mu2 = conv32(x), conv32(y)
    v2, v3, v4 = conv32(x * x), conv32(y * y), conv32(x * y)
    mu2_sq, mu1_mu2 = mu2 * mu2, mu1 * mu2
    s1, s2, s12 = fma32(-mu1, mu1, v2), fma32(-mu2, mu2, v3), v4 - mu1_mu2
    Cq, Dq = two * mu1_mu2 + c1, two * s12 + c2
    A, B = fma32(mu1, mu1, mu2_sq) + c1, s1 + s2 + c2
    m = (Cq * Dq) / (A * B)
    d1 = (mu2 * two * Dq) / (A * B) - (mu2 * two * Cq) / (A * B) - (mu1 * two * Cq * Dq) / (A * A * B) + \
        (mu1 * two * Cq * Dq) / (A * B * B)
    d2 = (-Cq * Dq) / (A * B * B)
    d3 = (two * Cq) / (A * B)
    return dict(map=m, dm_dmu1=d1, dm_dsigma1_sq=d2, dm_dsigma12=d3)


def backward32(x, y, dl, parts, l1_scale=None):
    """ssim_backward_tile: out = c0 + x*2*c1 + y*c2 (+ l1_scale * sign(x - y))"""
    c = [conv32(parts[k] * dl) for k in ("dm_dmu1", "dm_dsigma1_sq", "dm_dsigma12")]
    out = c[0] + x * f32(2.0) * c[1]
    out = out + y * c[2]
    if l1_scale is not None:
        out = out + l1_scale * np.sign(x - y).astype(np.float32)
    return out


def loss32(x, y, m, lam):
    """per-pixel (1 - lambda)|x - y| - lambda m, summed per 32x32 tile in float32, scaled by 1/N and added tile by tile"""
    lam = f32(lam)
    N = x.size
    inv_n = f32(1.0 / N)
    part = (f32(1.0) - lam) * np.abs(x - y) - lam * m
    P, H, W = part.shape
    Hp, Wp = -(-H // 32) * 32, -(-W // 32) * 32
    t = np.zeros((P, Hp, Wp), np.float32)
    t[:, :H, :W] = part
    tiles = t.reshape(P, Hp // 32, 32, Wp // 32, 32).sum(axis=(2, 4), dtype=np.float32).reshape(-1)
    total = fma32(tiles[0], inv_n, lam)
    for v in tiles[1:]:
        total = f32(total + f32(v * inv_n))
    return float(total), tiles.size


def loss_consts(lam, N):
    lam = f32(lam)
    inv_n = f32(1.0 / N)
    return -lam * inv_n, (f32(1.0) - lam) * inv_n


def _ratios(out, got, ref, jumps=None):
    for k, r in ref.items():
        out[k] = max(out.get(k, 0.0), lr.err_ratio(got[k], r, lr.BOUND[k], 0.0 if jumps is None else jumps.get(k, 0.0)))


# ---- 1. the restatement against torch float64 autograd --------------------------------------------------------------
def _torch_ssim(a, b, lam):
    CH = a.shape[0]
    g = torch.tensor(lr.G)
    win = (g[:, None] @ g[None, :]).expand(CH, 1, 11, 11).contiguous()
    conv = lambda t: torch.nn.functional.conv2d(t, win, padding=5, groups=CH)
    i1 = torch.tensor(a, dtype=torch.float64, requires_grad=True)
    i2 = torch.tensor(b, dtype=torch.float64)
    u1, u2 = i1[None], i2[None]
    mu1, mu2 = conv(u1), conv(u2)
    s1, s2, s12 = conv(u1 * u1) - mu1 * mu1, conv(u2 * u2) - mu2 * mu2, conv(u1 * u2) - mu1 * mu2
    m = ((2 * mu1 * mu2 + lr.C1) * (2 * s12 + lr.C2)) / ((mu1 * mu1 + mu2 * mu2 + lr.C1) * (s1 + s2 + lr.C2))
    loss = (1 - lam) * (i1 - i2).abs().mean() + lam * (1 - m.mean())
    loss.backward()
    return m[0].detach().numpy(), float(loss.detach()), i1.grad.numpy()


@pytest.mark.parametrize("fam", ["random", "flat", "unclamped", "ties"])
def test_restatement_matches_torch_autograd(fam):
    lam = float(f32(0.2))
    a, b = lr.family(fam, 4, 37, 45, seed=3, E=E_STAR[0])
    m_t, L_t, g_t = _torch_ssim(a, b, lam)
    m = lr.ssim_parts(a, b)["map"]
    L, dimg = lr.l1_ssim_loss(a, b, lam)
    # both sides round in float64: 1e-12 of each element's magnitude (the flat family cancels in sigma^2 in float64 too)
    assert np.all(np.abs(m.v - m_t) <= 1e-12 * m.m)
    assert abs(L.v - L_t) <= 1e-12 * L.terms
    assert np.all(np.abs(dimg.v - g_t) <= 1e-12 * dimg.m)


def test_window_is_the_normalised_gaussian():
    assert lr.G.shape == (11,) and abs(lr.G.sum() - 1.0) < 1e-15
    assert np.array_equal(lr.G, lr.G[::-1]) and lr.G.argmax() == 5
    np.testing.assert_allclose(lr.G[4] / lr.G[5], np.exp(-1 / 4.5), rtol=1e-15)


def test_magnitudes_dominate_values():
    """M >= |v| for every output: each element's own rounding is inside its bound"""
    a, b = lr.family("unclamped", 2, 20, 33, seed=5)
    p = lr.ssim_parts(a, b)
    dl = np.random.default_rng(1).normal(size=a.shape).astype(np.float32)
    for k, v in dict(p, dimg=lr.ssim_backward(a, b, dl, p)).items():
        assert np.all(v.m >= np.abs(v.v)), k


# ---- 2. the bounds against the float32 emulation ----------------------------------------------------------------------
SHAPES = [(3, 33, 65), (2, 70, 90)]


@pytest.mark.parametrize("fam", lr.FAMILIES)
def test_bounds_hold_for_float32_emulation(fam):
    ratios = {}
    for i, (P, H, W) in enumerate(SHAPES):
        a, b = lr.family(fam, P, H, W, seed=10 + i, E=E_STAR[0])
        # SSIM forward and backward on a random dL/dmap
        p32 = forward32(a, b)
        ref = lr.ssim_parts(a, b)
        _ratios(ratios, p32, ref)
        dl = np.random.default_rng(20 + i).normal(size=a.shape).astype(np.float32)
        _ratios(ratios, dict(dimg=backward32(a, b, dl, p32)), dict(dimg=lr.ssim_backward(a, b, dl, ref)))
        # the loss and its gradient
        lam = 0.2
        dlc, l1 = loss_consts(lam, a.size)
        L32, n_cta = loss32(a, b, p32["map"], lam)
        L, dimg = lr.l1_ssim_loss(a, b, lam)
        ratios["loss"] = max(ratios.get("loss", 0.0), abs(L32 - L.v) / L.bound(n_cta, lr.BOUND["map"]))
        _ratios(ratios, dict(loss_dimg=backward32(a, b, dlc, p32, l1)), dict(loss_dimg=dimg))
    print("\n%-10s " % fam + "  ".join("%s %.3f" % kv for kv in sorted(ratios.items())))
    assert max(ratios.values()) <= 1.0, ratios


@pytest.mark.parametrize("fam", ["random", "unclamped", "large", "ties"])
@pytest.mark.parametrize("e", range(3))
def test_exposed_loss_bounds_hold_for_float32_emulation(fam, e):
    E = E_STAR[e]
    img, gt = lr.family(fam, 3, 45, 70, seed=30 + e)
    lam = 0.2
    out = lr.expose32(img, E)
    p32 = forward32(out, gt)
    dlc, l1 = loss_consts(lam, out.size)
    dout = backward32(out, gt, dlc, p32, l1)
    Ef = E.astype(np.float32)
    dimg = np.empty_like(dout)
    for k in range(3):
        g = Ef[k, 0] * dout[0]
        g = fma32(Ef[k, 1], dout[1], g)
        dimg[k] = fma32(Ef[k, 2], dout[2], g)
    dE = np.zeros((3, 4))
    for c in range(3):
        for k in range(3):
            dE[k, c] = (img[k].astype(np.float64) * dout[c]).sum()
        dE[c, 3] = dout[c].astype(np.float64).sum()
    L32, n_cta = loss32(out, gt, p32["map"], lam)
    L, rdimg, jimg, rdE, jE = lr.l1_ssim_loss_exposure(img, gt, E, lam)
    r = dict(loss=abs(L32 - L.v) / L.bound(n_cta, lr.BOUND["map"]),
             loss_dimg=lr.err_ratio(dimg, rdimg, lr.BOUND["loss_dimg"], jimg),
             dE=lr.err_ratio(dE, rdE, lr.BOUND["loss_dimg"], jE))
    print("\nexposed %-9s E%d " % (fam, e) + "  ".join("%s %.3f" % kv for kv in sorted(r.items())))
    assert max(r.values()) <= 1.0, r


@pytest.mark.parametrize("fam", ["random", "flat", "unclamped", "exposed"])
@pytest.mark.parametrize("expo", [False, True])
def test_eval_bounds_hold_for_float32_emulation(fam, expo):
    img, gt = lr.family(fam, 3, 50, 66, seed=40, E=E_STAR[1])
    E = E_STAR[2] if expo else None
    x = lr.expose32(img, E) if expo else img
    a, b = np.clip(x, 0, 1), np.clip(gt, 0, 1)
    d = a - b
    mse = float((d * d).astype(np.float64).mean())
    psnr32 = float(f32(10.0) * f32(np.log10(f32(1.0) / f32(mse))))
    ssim32 = float(forward32(a, b)["map"].astype(np.float64).mean())
    psnr, ssim = lr.eval_psnr_ssim(img, gt, E)
    r = dict(psnr=lr.err_ratio(psnr32, psnr, lr.BOUND["psnr"]), ssim=lr.err_ratio(ssim32, ssim, lr.BOUND["map"]))
    print("\neval %-9s expo=%d " % (fam, expo) + "  ".join("%s %.3f" % kv for kv in sorted(r.items())))
    assert max(r.values()) <= 1.0, r


def test_identical_images_known_answers():
    """the restatement itself: SSIM 1 and zero partial maps d/dmu1 at identical images; PSNR +inf"""
    a, _ = lr.family("random", 2, 21, 34, seed=50)
    p = lr.ssim_parts(a, a)
    np.testing.assert_allclose(p["map"].v, 1.0, rtol=0, atol=1e-15)
    assert np.abs(p["dm_dmu1"].v).max() <= 1e-12 * p["dm_dmu1"].m.max()
    psnr, ssim = lr.eval_psnr_ssim(a, a)
    assert psnr.v == np.inf and abs(float(ssim.v) - 1.0) < 1e-15
