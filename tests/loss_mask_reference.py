"""Float64 restatement of the masked loss and evaluation of csrc/ssim.cu (glic_l1_ssim_loss_masked, glic_eval_psnr_ssim_masked),
built on tests/loss_reference.py's Mag values and magnitudes.

With w the [H,W] valid-pixel mask (1 = used), a the image (exposed by E first when given) and b the ground truth:
    a' = w ? a : 0,  b' = w ? b : 0                     (a select: what lies under the mask never enters)
    L  = (1 - lambda) sum_used |a' - b'| / Nw + lambda (1 - sum_used SSIM(a', b') / Nw),   Nw = 3 count(w)
    dL/da = w ? dL/da' : 0
The SSIM map of (a', b') is the unmasked one of the selected planes: masked pixels act like the zero padding at the frame
border.  dL/da' is the unmasked backward of the SSIM term with dL/dmap = -lambda/Nw at used pixels and 0 at masked ones, plus
the L1 sign term at used pixels.  The evaluation clamps a and b to [0, 1], selects them the same way and takes MSE and the SSIM
mean over the 3 count(w) used elements (CH count(w) for CH planes).
"""
import math

import numpy as np

import loss_reference as lr
from loss_reference import Mag


def _select(x, w):
    """x' = w ? x : 0 for Mag x [..., H, W] and a boolean mask [H, W]"""
    return Mag(np.where(w, x.v, 0.0), np.where(w, x.m, 0.0))


def _masked_loss_value(lam, x, y, ssim_map, w, Nw):
    """the loss value over the used pixels of the selected planes x, y"""
    d = np.where(w, np.abs(x.v - y.v), 0.0)
    s = np.where(w, ssim_map.v, 0.0)
    v = lam + ((1.0 - lam) * d - lam * s).sum() / Nw
    terms = lam + ((1.0 - lam) * d + lam * np.abs(s)).sum() / Nw
    return lr.Loss(v, terms, lam * np.where(w, ssim_map.m, 0.0).sum() / Nw)


def _masked_dout(x, y, w, lam, p, Nw):
    """dL/da of the selected planes: the SSIM term's backward with dL/dmap = -lambda/Nw at used pixels, the L1 sign there, and
    0 at masked pixels"""
    _, dl, l1 = lr._loss_constants(lam, Nw)
    dmap = Mag(np.where(w, dl.v, 0.0) * np.ones(x.v.shape), np.where(w, dl.m, 0.0) * np.ones(x.v.shape))
    d = lr.ssim_backward(x, y, dmap, p) + l1 * Mag(np.where(w, np.sign(x.v - y.v), 0.0), 0.0)
    return _select(d, w), l1


def l1_ssim_loss_masked(img, gt, mask, lam=0.2):
    """glic_l1_ssim_loss_masked without exposure on [3,H,W] planes: (loss, dL/dimg)"""
    w = np.asarray(mask, bool)
    x, y = _select(Mag(np.asarray(img, np.float64)), w), _select(Mag(np.asarray(gt, np.float64)), w)
    Nw = x.v.shape[0] * int(w.sum())
    p = lr.ssim_parts(x, y)
    dimg, _ = _masked_dout(x, y, w, float(np.float32(lam)), p, Nw)
    return _masked_loss_value(float(np.float32(lam)), x, y, p["map"], w, Nw), dimg


def l1_ssim_loss_exposure_masked(img, gt, E, mask, lam=0.2):
    """glic_l1_ssim_loss_masked with E: (loss, dimg, dimg_jump, dE, dE_jump) as lr.l1_ssim_loss_exposure returns them"""
    w = np.asarray(mask, bool)
    img64 = np.asarray(img, np.float64)
    E64 = np.asarray(E, np.float32).astype(np.float64)
    x = _select(lr.expose(Mag(img64), E), w)
    y = _select(Mag(np.asarray(gt, np.float64)), w)
    Nw = 3 * int(w.sum())
    lam = float(np.float32(lam))
    p = lr.ssim_parts(x, y)
    dout, l1 = _masked_dout(x, y, w, lam, p, Nw)
    diff = x.v - y.v
    jump = np.where(w & (np.abs(diff) <= 4.0 * lr.U * x.m), 2.0 * abs(float(l1.v)), 0.0)
    dimg_v, dimg_m, dimg_j = [], [], []
    for k in range(3):
        acc = Mag(0.0, 0.0)
        for c in range(3):
            acc = acc + dout[c] * Mag(E64[k, c])
        dimg_v.append(acc.v); dimg_m.append(acc.m)
        dimg_j.append(sum(abs(E64[k, c]) * jump[c] for c in range(3)))
    dE_v, dE_m, dE_j = np.zeros((3, 4)), np.zeros((3, 4)), np.zeros((3, 4))
    absimg = np.where(w, np.abs(img64), 0.0)
    img_used = np.where(w, img64, 0.0)                # dL/dout is 0 under the mask: the image there adds nothing
    for c in range(3):
        for k in range(3):
            dE_v[k, c] = (img_used[k] * dout.v[c]).sum()
            dE_m[k, c] = (absimg[k] * dout.m[c]).sum()
            dE_j[k, c] = (absimg[k] * jump[c]).sum()
        dE_v[c, 3], dE_m[c, 3], dE_j[c, 3] = dout.v[c].sum(), dout.m[c].sum(), jump[c].sum()
    return (_masked_loss_value(lam, x, y, p["map"], w, Nw), Mag(np.stack(dimg_v), np.stack(dimg_m)), np.stack(dimg_j),
            Mag(dE_v, dE_m), dE_j)


def eval_psnr_ssim_masked(img, gt, mask, E=None):
    """glic_eval_psnr_ssim_masked: (psnr, ssim) as Mag scalars; PSNR is +inf when the used elements agree"""
    w = np.asarray(mask, bool)
    x = lr.expose(Mag(img), E) if E is not None else Mag(np.asarray(img, np.float64))
    x = _select(Mag(np.clip(x.v, 0.0, 1.0), x.m), w)
    y = _select(Mag(np.clip(np.asarray(gt, np.float64), 0.0, 1.0)), w)
    Nw = x.v.shape[0] * int(w.sum())
    d = x - y
    se = d * d
    mse = Mag(se.v.sum() / Nw, se.m.sum() / Nw)
    if mse.v == 0.0:
        psnr = Mag(np.inf, 0.0)
    else:
        v = 10.0 * math.log10(1.0 / float(mse.v))
        psnr = Mag(v, 10.0 / math.log(10.0) * float(mse.m) / float(mse.v) + abs(v))
    smap = lr.ssim_parts(x, y)["map"]
    ssim = Mag(np.where(w, smap.v, 0.0).sum() / Nw, np.where(w, smap.m, 0.0).sum() / Nw)
    return psnr, ssim


def pack(mask):
    """the device layout of glic_pack_mask: [H][ceil(W/32)] uint32 words, pixel x at bit x & 31 of word x >> 5"""
    w = np.asarray(mask, bool)
    H, W = w.shape
    wpr = (W + 31) // 32
    padded = np.zeros((H, 32 * wpr), bool)
    padded[:, :W] = w
    bits = np.packbits(padded.reshape(H, wpr, 32), axis=-1, bitorder="little")      # 4 bytes per word, little-endian
    return np.ascontiguousarray(bits).view("<u4").reshape(H, wpr), int(w.sum())


# ---- mask families ----------------------------------------------------------------------------------------------------
def mask_family(name, H, W, seed):
    """[H,W] bool masks with at least one used pixel"""
    rng = np.random.default_rng(seed)
    w = np.zeros((H, W), bool)
    if name == "random":
        w = rng.uniform(0, 1, (H, W)) < 0.6
    elif name == "one_pixel":
        w[rng.integers(0, H), rng.integers(0, W)] = True
    elif name == "border":                          # a one-pixel used border around a masked interior
        w[0, :] = w[-1, :] = True
        w[:, 0] = w[:, -1] = True
    elif name == "tile_block":                      # a masked block on the 32x32 tile grid
        w[:] = True
        w[32:min(H, 96), 32:min(W, 64)] = False
    elif name == "straddle":                        # a masked block across tile seams
        w[:] = True
        w[H // 4:H // 4 + max(1, H // 2), W // 3:W // 3 + max(1, W // 3) + 17] = False
    elif name == "ones":
        w[:] = True
    else:
        raise ValueError(name)
    if not w.any():
        w[H // 2, W // 2] = True
    return w


MASKS = ("random", "one_pixel", "border", "tile_block", "straddle")
