"""CPU restatement of the per-image affine exposure (glic_l1_ssim_loss_exposure, glic_mapper_enable_exposure), in the float32 or
float64 arithmetic of an oracle.Oracle, whose L1 + D-SSIM loss it reuses.  Test infrastructure only.

Spec (include/glic_b200.h):
  E is 3x4 row-major (Inria 3DGS: matmul(img_hwc, E[:3,:3]) + E[:3,3]);
  out_c = E[0][c] r + E[1][c] g + E[2][c] b + E[c][3], evaluated as acc = E[c][3], then fma with r, g, b in that order;
  L = the loss of out;  dL/dimg_k = sum_c E[k][c] dL/dout_c, evaluated as E[k][0] d0, then fma with d1, d2;
  dL/dE[k][c] = sum_px img_k dL/dout_c (k < 3),  dL/dE[c][3] = sum_px dL/dout_c  (float64 sums);
  Adam (torch::optim::Adam: betas 0.9 / 0.999, eps 1e-8, no weight decay), t = step + 1:
    m = b1 m + (1-b1) g,  v = b2 v + (1-b2) g^2,  denom = sqrt(v) / sqrt(1 - b2^t) + eps,  E -= (lr / (1 - b1^t)) m / denom,
  the bias corrections and lr / (1 - b1^t) in float64 (as LibTorch computes them), every other operation rounded on its own.

float32 fma is restated as one float64 product (exact for two float32 factors) plus one float64 add, rounded to float32: that
differs from a true fmaf only where the float64 sum lands exactly halfway between two float32 values (double rounding), which
the tolerance-based comparisons absorb."""
import numpy as np


def _fma(a, b, c, dt):
    if dt is np.float64:
        return np.asarray(a, np.float64) * b + c
    return (np.asarray(a, np.float64) * np.float64(b) + np.asarray(c, np.float64)).astype(np.float32)


def expose(img, E, dt):
    img = np.asarray(img, dt)
    E = np.asarray(E, dt).reshape(3, 4)
    out = np.empty(img.shape, dt)
    for c in range(3):
        acc = np.full(img.shape[1:], E[c, 3], dt)
        for k in range(3):
            acc = _fma(img[k], E[k, c], acc, dt)
        out[c] = acc
    return out


def loss_exposure(o, img, gt, E, lambda_dssim=0.2, grad=True):
    """-> (L, dL_dimg [3,H,W] in the oracle's dtype, dL_dE [3,4] float64); the gradients are None when grad is False"""
    dt = o.dtype.type
    E = np.asarray(E, dt).reshape(3, 4)
    img = np.asarray(img, dt)
    out = expose(img, E, dt)
    L, dout = o.loss(out, gt, lambda_dssim, grad=grad)
    if not grad:
        return L, None, None
    dimg = np.empty(out.shape, dt)
    for k in range(3):
        g = (E[k, 0] * dout[0]).astype(dt)
        g = _fma(dout[1], E[k, 1], g, dt)
        dimg[k] = _fma(dout[2], E[k, 2], g, dt)
    x, d = img.astype(np.float64), dout.astype(np.float64)
    dE = np.zeros((3, 4))
    for k in range(3):
        for c in range(3):
            dE[k, c] = np.sum(x[k] * d[c])
        dE[k, 3] = np.sum(d[k])
    return L, dimg, dE


def exposure_adam(o, E, m, v, step, grad, lr):
    """one exposure step -> (E, m, v, step), new arrays in the oracle's dtype"""
    dt = o.dtype.type
    E, m, v, g = (np.asarray(x, dt) for x in (E, m, v, grad))
    t = int(step) + 1
    bc1, bc2 = 1.0 - 0.9 ** t, 1.0 - 0.999 ** t
    b1, b2, eps = dt(0.9), dt(0.999), dt(1e-8)
    m1 = _fma(g, dt(1.0) - b1, b1 * m, dt)
    v1 = _fma(g * g, dt(1.0) - b2, b2 * v, dt)
    denom = np.sqrt(v1) / dt(np.sqrt(bc2)) + eps
    step_size = dt(float(dt(lr)) / bc1)
    return E + (-step_size) * (m1 / denom), m1, v1, t
