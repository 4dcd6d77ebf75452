"""Float64 restatement of csrc/ssim.cu (SSIM map and partial maps, the SSIM backward, the L1 + D-SSIM loss, the exposed loss
and the evaluation PSNR / SSIM), with a magnitude map beside every output.

Each output is a `Mag`: its float64 value `v` and its magnitude `m`.  `m` is the same computation with every sum replaced
by the sum of the operands' magnitudes (a cancellation such as sigma1^2 = conv(x^2) - mu1^2 costs conv(x^2) + mu1^2, not
their difference) and products and quotients propagated to first order.  The inputs are float32 values, taken as exact,
with magnitude |x| so that the first rounding made from them is counted.  A float32 computation of the same arithmetic in
any fixed order then differs from `v` by a small multiple of 2^-24 * m at every element: each rounding contributes at most
2^-24 times the magnitude of its result, and `m` dominates every intermediate result's contribution to the output.  The
tests check `|got - v| <= c * 2^-24 * m` per element with one constant c per output (see tests/test_gpu_loss_exact.py).

The window is the 11-tap Gaussian with sigma 1.5 built here from its definition; the convolutions are separable with zero
("same") padding, as the kernels pad at the frame border.
"""
import math

import numpy as np
from scipy.ndimage import correlate1d

U = 2.0 ** -24                             # unit roundoff of float32 round-to-nearest


def f32(x):
    return float(np.float32(x))


C1 = f32(np.float32(0.01) * np.float32(0.01))       # the float32 constants the loss and evaluation pass (0.01^2, 0.03^2)
C2 = f32(np.float32(0.03) * np.float32(0.03))


def window():
    x = np.arange(11, dtype=np.float64) - 5.0
    g = np.exp(-(x * x) / (2.0 * 1.5 * 1.5))
    return g / g.sum()


G = window()


def _is_pow2(c):
    return isinstance(c, (int, float)) and c != 0 and math.frexp(abs(c))[0] == 0.5


class Mag:
    """A float64 value with its magnitude (see the module docstring).  Python numbers combine as float32 constants: a power
    of two scales exactly, any other constant counts as rounded once."""
    __slots__ = ("v", "m")

    def __init__(self, v, m=None):
        self.v = np.asarray(v, np.float64)
        self.m = np.abs(self.v) if m is None else np.asarray(m, np.float64)

    @staticmethod
    def of(x):
        return x if isinstance(x, Mag) else Mag(x)

    def __add__(self, o):
        o = Mag.of(o)
        return Mag(self.v + o.v, self.m + o.m)

    __radd__ = __add__

    def __sub__(self, o):
        o = Mag.of(o)
        return Mag(self.v - o.v, self.m + o.m)

    def __rsub__(self, o):
        return Mag.of(o) - self

    def __neg__(self):
        return Mag(-self.v, self.m)

    def __mul__(self, o):
        if _is_pow2(o):
            return Mag(self.v * o, self.m * abs(o))
        o = Mag.of(o)
        return Mag(self.v * o.v, self.m * np.abs(o.v) + np.abs(self.v) * o.m)

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = Mag.of(o)
        q = self.v / o.v
        return Mag(q, (self.m + np.abs(q) * o.m) / np.abs(o.v))

    def __getitem__(self, k):
        return Mag(self.v[k], self.m[k])

    def sum(self, axis=None):
        return Mag(self.v.sum(axis), self.m.sum(axis))

    def mean(self, axis=None):
        return Mag(self.v.mean(axis), self.m.mean(axis))

    # The functions below carry the argument's magnitude through to first order and add their own error, counted in
    # units of their result so that m >= |v| holds after them as it does after the operators above.
    def sqrt(self):
        """sqrtf is correctly rounded: d sqrt(x) = dx / (2 sqrt x), plus half the result for its own rounding"""
        r = np.sqrt(self.v)
        with np.errstate(divide="ignore", invalid="ignore"):
            m = np.where(r > 0.0, self.m / (2.0 * r), 0.0)
        return Mag(r, m + 0.5 * np.abs(r))

    def exp(self, ulps=2.0):
        """expf is not correctly rounded (CUDA: at most 2 ulp): |e^x| dx, plus `ulps` units of the result"""
        r = np.exp(self.v)
        return Mag(r, np.abs(r) * self.m + ulps * np.abs(r))

    def log(self, ulps=2.0):
        """logf is not correctly rounded (CUDA: at most 1 ulp): dx / |x|, plus `ulps` units of the result"""
        r = np.log(self.v)
        return Mag(r, self.m / np.abs(self.v) + ulps * np.abs(r))

    def rcp(self, ulps=1.0):
        """1 / x by an approximate reciprocal (rcp.approx.f32: at most 1 ulp): dx / x^2, plus `ulps` units of the result"""
        r = 1.0 / self.v
        return Mag(r, self.m * r * r + ulps * np.abs(r))

    def fma(self, b, c):
        """fmaf(self, b, c): the exact product and sum, rounded once"""
        return self * b + c

    def minimum(self, o):
        """fminf: the smaller value, with the larger of the two magnitudes (the operands may be within rounding of each other,
        so the float32 evaluation may select either)"""
        o = Mag.of(o)
        return Mag(np.minimum(self.v, o.v), np.maximum(self.m, o.m))

    @staticmethod
    def where(cond, a, b):
        a, b = Mag.of(a), Mag.of(b)
        return Mag(np.where(cond, a.v, b.v), np.where(cond, a.m, b.m))


def conv_array(a):
    """11x11 separable Gaussian over the last two axes, zero padding"""
    a = correlate1d(np.asarray(a, np.float64), G, axis=-1, mode="constant", cval=0.0)
    return correlate1d(a, G, axis=-2, mode="constant", cval=0.0)


def conv(x):
    x = Mag.of(x)
    return Mag(conv_array(x.v), conv_array(x.m))       # the weights are positive: the magnitude is the convolved magnitude


def ssim_parts(x, y, c1=C1, c2=C2):
    """SSIM map and its three partial maps of planes x, y ([..., H, W] arrays or Mag), as ssim_forward_tile defines them"""
    x, y = Mag.of(x), Mag.of(y)
    mu1, mu2 = conv(x), conv(y)
    s1 = conv(x * x) - mu1 * mu1
    s2 = conv(y * y) - mu2 * mu2
    s12 = conv(x * y) - mu1 * mu2
    Cq = mu1 * mu2 * 2.0 + c1
    Dq = s12 * 2.0 + c2
    A = mu1 * mu1 + mu2 * mu2 + c1
    B = s1 + s2 + c2
    AB = A * B
    CD = Cq * Dq
    out = dict(map=CD / AB)
    out["dm_dmu1"] = ((mu2 * 2.0 * Dq) / AB - (mu2 * 2.0 * Cq) / AB - (mu1 * 2.0 * CD) / (A * A * B) +
                      (mu1 * 2.0 * CD) / (A * B * B))
    out["dm_dsigma1_sq"] = -CD / (A * B * B)
    out["dm_dsigma12"] = (Cq * 2.0) / AB
    return out


def ssim_backward(x, y, dL_dmap, parts):
    """dL/dx = conv(dL * dm_dmu1) + 2 x conv(dL * dm_dsigma1_sq) + y conv(dL * dm_dsigma12); the partial maps carry their own
    magnitudes into the result"""
    x, y, d = Mag.of(x), Mag.of(y), Mag.of(dL_dmap)
    a = conv(d * parts["dm_dmu1"])
    b = conv(d * parts["dm_dsigma1_sq"])
    c = conv(d * parts["dm_dsigma12"])
    return a + x * 2.0 * b + y * c


def expose(img, E):
    """out_c = E[0][c] r + E[1][c] g + E[2][c] b + E[c][3] of a [3,H,W] image; E a 3x4 float32 matrix"""
    img = Mag.of(img)
    E = np.asarray(E, np.float32).astype(np.float64)
    planes = []
    for c in range(3):
        acc = Mag(E[c, 3])
        for k in range(3):
            acc = acc + img[k] * Mag(E[k, c])
        planes.append(acc)
    return Mag(np.stack([p.v for p in planes]), np.stack([p.m for p in planes]))


def _loss_constants(lam, N):
    """dL/dmap of the SSIM term and the L1 scale: -lambda/N and (1 - lambda)/N, each rounded once to float32 by the caller"""
    lam = float(np.float32(lam))
    return lam, Mag(-lam / N), Mag((1.0 - lam) / N)


class Loss:
    """A loss value with what bounds the float32 kernel's result: `terms` = lambda + mean((1 - lambda)|x - y| + lambda |m|),
    the magnitude of the per-CTA and atomic sums, and `map_m` = lambda * mean(M(map)), the SSIM map's own error carried in."""

    def __init__(self, v, terms, map_m):
        self.v, self.terms, self.map_m = float(v), float(terms), float(map_m)

    def bound(self, n_cta, c_map):
        """|got - v| allowed to the kernel's loss scalar: each of the n_cta atomicAdds and the 1024-pixel CTA sums rounds at
        most once per level, 2^-24 of the running total; the map's error is bounded by c_map (the SSIM map's constant)"""
        return (n_cta + 1024) * U * self.terms + c_map * U * self.map_m


def _loss_value(lam, x, y, ssim_map):
    d = np.abs(x.v - y.v)
    N = d.size
    v = lam + ((1.0 - lam) * d - lam * ssim_map.v).sum() / N
    terms = lam + ((1.0 - lam) * d + lam * np.abs(ssim_map.v)).sum() / N
    return Loss(v, terms, lam * ssim_map.m.sum() / N)


def l1_ssim_loss(img, gt, lam=0.2, parts=None):
    """glic_l1_ssim_loss on [CH,H,W] planes: loss = (1 - lambda) mean|img - gt| + lambda (1 - mean SSIM) and dL/dimg.
    The L1 sign is exact here: img and gt are the float32 inputs, so sign(img - gt) is what the kernel sees.  parts: the
    ssim_parts of the same planes, when already computed."""
    x, y = Mag(img), Mag(gt)
    lam, dl, l1 = _loss_constants(lam, x.v.size)
    p = ssim_parts(x, y) if parts is None else parts
    dimg = ssim_backward(x, y, dl, p) + l1 * Mag(np.sign(x.v - y.v), 0.0)
    return _loss_value(lam, x, y, p["map"]), dimg


def l1_ssim_loss_exposure(img, gt, E, lam=0.2):
    """glic_l1_ssim_loss_exposure: the loss of the exposed image out = expose(img, E) against gt ([3,H,W]), dL/dimg and dL/dE.
    Returns (loss, dimg, dimg_jump, dE, dE_jump).  The exposed image is rounded in float32 by the kernel, so where out is
    within its rounding of gt the L1 sign the kernel sees is not decided here: there the step's full height 2 (1 - lambda)/N
    is allowed as `jump` (zero almost everywhere), and carried through to dL/dimg and dL/dE."""
    img64 = np.asarray(img, np.float64)
    E64 = np.asarray(E, np.float32).astype(np.float64)
    x = expose(Mag(img64), E)
    y = Mag(gt)
    lam, dl, l1 = _loss_constants(lam, x.v.size)
    p = ssim_parts(x, y)
    diff = x.v - y.v
    dout = ssim_backward(x, y, dl, p) + l1 * Mag(np.sign(diff), 0.0)
    jump = np.where(np.abs(diff) <= 4.0 * U * x.m, 2.0 * abs(float(l1.v)), 0.0)
    dimg_v, dimg_m, dimg_j = [], [], []
    for k in range(3):
        acc = Mag(0.0, 0.0)
        for c in range(3):
            acc = acc + dout[c] * Mag(E64[k, c])
        dimg_v.append(acc.v); dimg_m.append(acc.m)
        dimg_j.append(sum(abs(E64[k, c]) * jump[c] for c in range(3)))
    dimg = Mag(np.stack(dimg_v), np.stack(dimg_m))
    dE_v, dE_m, dE_j = np.zeros((3, 4)), np.zeros((3, 4)), np.zeros((3, 4))
    absimg = np.abs(img64)
    for c in range(3):
        for k in range(3):
            dE_v[k, c] = (img64[k] * dout.v[c]).sum()
            dE_m[k, c] = (absimg[k] * dout.m[c]).sum()
            dE_j[k, c] = (absimg[k] * jump[c]).sum()
        dE_v[c, 3], dE_m[c, 3], dE_j[c, 3] = dout.v[c].sum(), dout.m[c].sum(), jump[c].sum()
    return _loss_value(lam, x, y, p["map"]), dimg, np.stack(dimg_j), Mag(dE_v, dE_m), dE_j


def eval_psnr_ssim(img, gt, E=None):
    """glic_eval_psnr_ssim (and, with E, the mapper's exposed evaluation): PSNR and mean SSIM of img (exposed by E first)
    and gt, both clamped to [0, 1].  Returns (psnr, ssim) as Mag scalars; PSNR is +inf for identical clamped images."""
    x = expose(Mag(img), E) if E is not None else Mag(img)
    x = Mag(np.clip(x.v, 0.0, 1.0), x.m)                 # the clamp is 1-Lipschitz: it carries the magnitude as it is
    y = Mag(np.clip(np.asarray(gt, np.float64), 0.0, 1.0))
    d = x - y
    se = d * d
    mse = Mag(se.v.mean(), se.m.mean())
    if mse.v == 0.0:
        psnr = Mag(np.inf, 0.0)
    else:
        v = 10.0 * math.log10(1.0 / float(mse.v))
        # first order through the log, plus the float32 mse, log10f and product on the value itself
        psnr = Mag(v, 10.0 / math.log(10.0) * float(mse.m) / float(mse.v) + abs(v))
    return psnr, ssim_parts(x, y)["map"].mean()


def err_ratio(got, ref, c, jump=0.0):
    """max over elements of |got - ref.v| / (c 2^-24 ref.m + jump): at most 1 when every element is within its bound"""
    got = np.asarray(got, np.float64)
    err = np.abs(got - ref.v)
    bound = c * U * ref.m + jump
    if not np.all(np.isfinite(got)):
        return math.inf
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0.0, 0.0, err / bound)
    return float(r.max()) if r.size else 0.0


# ---- input families -------------------------------------------------------------------------------------------------
# Each returns (a, b) float32 [P, H, W]: every plane drawn separately, so a wrong plane offset reads different content.
def expose32(img, E):
    """the kernels' float32 exposure of a [3,H,W] image (acc = E[c][3], then one fma per channel)"""
    img = np.asarray(img, np.float32).astype(np.float64)
    E = np.asarray(E, np.float32).astype(np.float64)
    out = np.empty(img.shape, np.float32)
    for c in range(3):
        acc = np.full(img.shape[1:], np.float32(E[c, 3]))
        for k in range(3):
            acc = (img[k] * E[k, c] + acc.astype(np.float64)).astype(np.float32)
        out[c] = acc
    return out


def family(name, P, H, W, seed, E=None):
    """E: the 3x4 exposure of the \"exposed\" family"""
    rng = np.random.default_rng(seed)
    shape = (P, H, W)
    if name == "random":
        a, b = rng.uniform(0, 1, shape), rng.uniform(0, 1, shape)
    elif name == "flat":
        # flat bright halves (values 0.93-0.95 with 1e-3 texture) beside textured halves, split per plane at its own column
        a, b = rng.uniform(0, 1, shape), rng.uniform(0, 1, shape)
        for p in range(P):
            cut = int(rng.integers(0, W + 1)) if W > 1 else 1
            lvl = rng.uniform(0.93, 0.95, 2)
            a[p, :, :cut] = lvl[0] + 1e-3 * rng.uniform(-1, 1, (H, cut))
            b[p, :, :cut] = lvl[1] + 1e-3 * rng.uniform(-1, 1, (H, cut))
    elif name == "unclamped":
        a, b = rng.uniform(-0.3, 1.6, shape), rng.uniform(-0.3, 1.6, shape)
    elif name == "large":
        a, b = rng.uniform(25, 75, shape), rng.uniform(25, 75, shape)
    elif name == "exposed":
        # exposed renders of dark-to-bright images: E's offsets push the dark pixels below zero
        a = np.concatenate([expose32(rng.uniform(0, 1, (3, H, W)), E) for _ in range((P + 2) // 3)])[:P]
        b = rng.uniform(0, 1, shape)
    elif name == "ties":
        a = rng.uniform(0, 1, shape)
        b = np.where(rng.uniform(0, 1, shape) < 0.5, a.astype(np.float32), rng.uniform(0, 1, shape))
    else:
        raise ValueError(name)
    return np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)


FAMILIES = ("random", "flat", "unclamped", "large", "exposed", "ties")


# c of each output: |float32 - float64| <= c * 2^-24 * M at every element.  M sums the magnitude of every rounded
# intermediate, so a worst case in which all ~35 roundings on the longest path (two 11-tap fmaf chains, the moment products,
# the cancellations, the quotients) err at their full half-ulp in the same direction would need c near that depth.  Rounding
# errors of these fixed-order chains are not aligned like that: the float32 emulation of the kernels' order in
# test_loss_reference_host.py stays below c = 1.9 for the map and its partial maps on every family at 33x65 and 70x90, and
# below 2.4 over a full 1920x1080x3 frame (the largest of millions of pixels); 1.3 for the loss gradient on the large-value
# family at that size, under 0.3 elsewhere; 0.7 for PSNR.  The constants leave a factor of 2.5 to 3 above those maxima.
#   map, dm_*: the SSIM map and its three partial maps (glic_fused_ssim)
#   dimg: glic_fused_ssim_backward for a given dL/dmap, fed the kernel's own partial maps (their M carried in)
#   loss_dimg: dL/dimg of glic_l1_ssim_loss and dL/dout of the exposed loss; dL/dimg and dL/dE of the exposed loss take the
#     same c (the 3x3 mix adds two roundings of its own, and dL/dE is summed in float64)
#   psnr: evaluation PSNR (the SSIM score takes the map's c: it is the float64 mean of the map)
BOUND = dict(map=6.0, dm_dmu1=6.0, dm_dsigma1_sq=6.0, dm_dsigma12=6.0, dimg=2.0, loss_dimg=4.0, psnr=2.0)
