"""Float64 restatement of csrc/lpips.cu, stage by stage, with an error bound beside every element.

Every stage takes the kernel's own inputs, read back from the caller's scratch (`layout` restates carve()):
  conv0 input   (clamp(x, 0, 1) - mean) / std, restated in float32 (`normalize`): exact, so no error term.
  conv l        v = b + sum_k a_k w_k in float64 (`conv`), from the kernel's own pool or tap, in the kernel's K order
                (ci, ky, kx) with zero padding.  Bound: see SPLIT and GAMMA below.  ReLU is 1-Lipschitz, so relu(v) takes the
                same bound.
  max pools     exact (`pool`): compared bit for bit.
  head          per pixel in float64 from the kernel's own tap (`head`), with a first-order bound from magnitudes; each CTA's
                float64 partial (256 pixels) is compared with the sum of its pixels' values within the sum of their bounds.
  finish        restated in float64 from the kernel's own partials (`finish`): the output float matches bit for bit.

The same functions run on the CPU (tests/test_lpips_reference_host.py) and on the GPU (tests/test_gpu_lpips_exact.py); they work
on torch float64 tensors and chunk the large ones, so an 8192 x 8192 frame stays within a few GB of device memory.

`emulate_conv` is a host emulation of the kernel's split-TF32 arithmetic (cvt.rna.tf32 rounding, exact products, fp32
accumulation in the kernel's order) under two accumulation models, and with the controlled faults of `FAULTS`.
"""
import math

import numpy as np

U = 2.0 ** -24                                     # unit roundoff of float32 round-to-nearest

# (Cin, Cout, k, stride, pad), as CONVS in lpips.cu
CONVS = [(3, 64, 11, 4, 2), (64, 192, 5, 1, 2), (192, 384, 3, 1, 1), (384, 256, 3, 1, 1), (256, 256, 3, 1, 1)]
BM, BK, K8 = 64, 32, 8                             # the conv kernel's M tile, K block and mma k
HEAD_THREADS = 256
EPS = float(np.float32(1e-10))                     # the head's 1e-10f

# (W, H) of every frame the tests run: the smallest, the image boundary in the middle of an M tile or on its edge per layer,
# W = 0..3 (mod 4) for the stride-4 right edge, camera frames, and the largest side
FRAMES = [(31, 31), (35, 35), (131, 31), (71, 39), (135, 39), (143, 79), (143, 143), (640, 512), (641, 512), (642, 512),
          (643, 512), (1280, 720), (1280, 1024), (1920, 1080), (2048, 1536), (8192, 31), (31, 8192), (8192, 8192)]

# ---- the conv bound -----------------------------------------------------------------------------------------------------
# |tap - relu(v)| <= SPLIT * M + GAMMA * (S + M) + U * (|v| + that), per element, where
#   M = sum_k |a_k w_k|, S = sum_j |s_j| with s_j the exact partial sum after k8 step j (bias not included: the accumulator
#   starts at zero and the bias is added in the epilogue), and the last term is the epilogue's acc + bias rounding.
# SPLIT: a = hi + lo exactly in fp32, hi and the rounded lo are TF32 (cvt.rna: relative error <= 2^-11 each), so
#   a b - (hi_a hi_b + hi_a lo_b + lo_a hi_b) = hi_a (lo_b* - lo_b) + (lo_a* - lo_a) hi_b + lo_a* lo_b*  (lo* the exact residual)
#   and each of the three terms is at most 2^-22 (1 + 2^-11) |a b|.
# GAMMA: each k8 step issues three mma.sync m16n8k8, each adding 8 exact products to the fp32 accumulator.  NVIDIA does not
#   document how the tensor cores round that sum.  Two host models of it are emulated below (`emulate_conv`): "rn", the nine
#   addends summed one at a time in fp32 round-to-nearest, and "rz", the nine addends aligned to the largest one's exponent
#   and truncated there with no extra bits, summed, and the sum truncated to fp32 (round toward zero) -- the least accurate
#   accumulation reported for NVIDIA tensor cores.  Truncation loses a fraction of an ulp of the running sum per mma, always
#   toward zero, so the error grows with the number of steps, and fastest when every product has the same sign (nothing
#   cancels the bias).  On the layers of tests/test_lpips_reference_host.py the rz model reaches err / (S + M) = 6.1 U on
#   all-positive conv0 inputs and weights, 0.3 U on random and cancellation-heavy ones; rn stays under 0.8 U.  GAMMA = 8 U
#   covers both models with a margin of 1.3, and stays tight enough that a single TF32 pass (products of TF32-rounded
#   operands, relative error up to 2^-10) exceeds the bound 14- to 52-fold on every layer on random inputs at the frames the
#   tests use, and a dropped cross term 9- to 40-fold (the negative controls).
SPLIT = 3.0 * 2.0 ** -22 * (1.0 + 2.0 ** -11)
GAMMA = 8.0 * U


# ---- shapes and the scratch layout ---------------------------------------------------------------------------------------
def shapes(H, W):
    """(h[5], w[5], ph[2], pw[2]) as shapes() in lpips.cu"""
    h0, w0 = (H + 4 - 11) // 4 + 1, (W + 4 - 11) // 4 + 1
    ph0, pw0 = (h0 - 3) // 2 + 1, (w0 - 3) // 2 + 1
    ph1, pw1 = (ph0 - 3) // 2 + 1, (pw0 - 3) // 2 + 1
    return [h0, ph0, ph1, ph1, ph1], [w0, pw0, pw1, pw1, pw1], [ph0, ph1], [pw0, pw1]


def head_blocks(hw):
    return (hw + HEAD_THREADS - 1) // HEAD_THREADS


def layout(H, W):
    """carve(): taps 0-4, pools 0-1, then the float64 partials of taps 0-4, each region 128-byte aligned (Carver).
    Returns ({name: (byte offset, element count, dtype, shape)}, total bytes)."""
    h, w, ph, pw = shapes(H, W)
    regions = [("tap%d" % l, "f4", (2, CONVS[l][1], h[l], w[l])) for l in range(5)]
    regions += [("pool%d" % p, "f4", (2, CONVS[p][1], ph[p], pw[p])) for p in range(2)]
    regions += [("partials%d" % l, "f8", (head_blocks(h[l] * w[l]),)) for l in range(5)]
    out, off = {}, 0
    for name, dt, shape in regions:
        off = (off + 127) & ~127
        n = int(np.prod(shape))
        out[name] = (off, n, dt, shape)
        off += n * (4 if dt == "f4" else 8)
    return out, (off + 127) & ~127


def carve(scratch, H, W):
    """views of a uint8 torch scratch tensor as the kernel's regions ({name: tensor of the region's shape})"""
    import torch
    regions, _ = layout(H, W)
    out = {}
    for name, (off, n, dt, shape) in regions.items():
        size = 4 if dt == "f4" else 8
        out[name] = scratch[off:off + n * size].view(torch.float32 if dt == "f4" else torch.float64).view(shape)
    return out


# ---- the weight payload ---------------------------------------------------------------------------------------------------
def unpack(payload):
    """(mean[3], std[3], [(w [Cout,Cin,k,k], b [Cout])] x 5, [lin [Cout]] x 5) views of a flat float32 payload"""
    off, convs = 6, []
    for ci, co, k, _, _ in CONVS:
        w = payload[off:off + co * ci * k * k].reshape(co, ci, k, k)
        off += co * ci * k * k
        convs.append((w, payload[off:off + co]))
        off += co
    lins = []
    for _, co, _, _, _ in CONVS:
        lins.append(payload[off:off + co])
        off += co
    assert off == payload.shape[0]
    return payload[0:3], payload[3:6], convs, lins


# ---- conv0's input -------------------------------------------------------------------------------------------------------
def normalize(img, mean, std):
    """__fdiv_rn(__fsub_rn(clamp(x, 0, 1), mean), std) per channel of [..., 3, H, W] float32: every operation correctly
    rounded float32, so this is the kernel's value exactly (torch tensors; float32 in, float32 out).  Computed in float64:
    the difference of two floats in [-1, 1] is exact there, and a float64 quotient of two floats rounded to float32 is the
    correctly rounded float32 quotient (53 >= 2 * 24 + 2)."""
    import torch
    x = img.clamp(0.0, 1.0).to(torch.float64)
    d = (x - mean.to(torch.float64).view(3, 1, 1)).to(torch.float32).to(torch.float64)
    return (d / std.to(torch.float64).view(3, 1, 1)).to(torch.float32)


# ---- conv ----------------------------------------------------------------------------------------------------------------
def _k8_pad(K):
    return (K + K8 - 1) // K8 * K8


def conv(inp, w, b, stride, pad, rows=None, budget=1 << 28):
    """v, M, S of the convolution of inp [2, Cin, Hi, Wi] (either dtype; taken as exact) by w [Cout, Cin, k, k] and b [Cout],
    for output rows `rows` (a range; all by default), as float64 [2, Cout, len(rows), Wo] tensors on inp's device.
      v: b + sum_k a_k w_k;  M: sum_k |a_k w_k|;  S: sum over k8 steps j of |s_j|, s_j = sum_{k < 8(j+1)} a_k w_k.
    budget: float64 elements of the largest temporary (the per-step partial sums of one chunk)."""
    import torch
    import torch.nn.functional as F
    n_img, Cin, Hi, Wi = inp.shape
    Cout, _, k, _ = w.shape
    Ho, Wo = (Hi + 2 * pad - k) // stride + 1, (Wi + 2 * pad - k) // stride + 1
    rows = range(Ho) if rows is None else rows
    K = Cin * k * k
    Kp = _k8_pad(K)
    steps = Kp // K8
    dev = inp.device
    W64 = torch.zeros(Cout, Kp, dtype=torch.float64, device=dev)
    W64[:, :K] = w.reshape(Cout, K).to(torch.float64)
    b64 = b.to(torch.float64)
    Wst = W64.view(Cout, steps, K8).permute(1, 2, 0)               # [steps, 8, Cout]
    Wabs = W64.abs().t()
    nr = len(rows)
    out = [torch.empty(n_img, Cout, nr, Wo, dtype=torch.float64, device=dev) for _ in range(3)]
    band = max(1, min(nr, budget // max(1, Wo * steps * Cout)))
    for i0 in range(0, nr, band):
        sub = rows[i0:i0 + band]
        r0, r1 = sub[0], sub[-1] + 1
        y0, y1 = r0 * stride - pad, (r1 - 1) * stride - pad + k        # the padded input rows this band reads
        src = inp[:, :, max(y0, 0):min(y1, Hi)].to(torch.float64)
        src = F.pad(src, (pad, pad, max(0, -y0), max(0, y1 - Hi)))
        for n in range(n_img):
            A = F.unfold(src[n:n + 1], k, stride=stride)[0].t()           # [pixels, K] in (ci, ky, kx) order
            A = F.pad(A, (0, Kp - K))
            v = A @ W64.t() + b64
            m = A.abs() @ Wabs
            part = torch.bmm(A.view(-1, steps, K8).permute(1, 0, 2), Wst)  # [steps, pixels, Cout]
            S = part.cumsum_(0).abs_().sum(0)
            for o, t in zip(out, (v, m, S)):
                o[n, :, i0:i0 + len(sub)] = t.t().reshape(Cout, len(sub), Wo)
    return out


def conv_bound(v, M, S):
    rest = SPLIT * M + GAMMA * (S + M)
    return rest + U * (v.abs() + rest)


# ---- pools ---------------------------------------------------------------------------------------------------------------
def pool(tap):
    """3x3 / stride 2 max pool, floor mode, of [2, C, h, w]: exact (the kernel's fmaxf chain over the same nine floats)"""
    import torch.nn.functional as F
    return F.max_pool2d(tap, 3, 2)


# ---- head ----------------------------------------------------------------------------------------------------------------
def head(tap, lin, p0=0, p1=None):
    """per-pixel LPIPS term of tap [2, C, h, w] (float32, the kernel's own) for flat pixels [p0, p1), in float64, and its
    bound.  The kernel's float32 arithmetic, with u = 2^-24:
      sx = sum_c fmaf(x, x, sx)       C sequential roundings of a sum of non-negative terms: relative error <= C u
      nx = sqrtf(sx) + 1e-10f         sqrt halves the relative error and rounds once, the add rounds once
      e_c = x_c / nx - y_c / ny       two correctly rounded quotients and a difference
      d = sum_c fmaf(lin_c, e_c^2, d) the square rounds once; C sequential roundings of a sum of |lin_c| e_c^2 terms
    The bound is these first-order terms, doubled to cover the second-order ones."""
    import torch
    C = tap.shape[1]
    f = tap.reshape(2, C, -1)[:, :, p0:p1].to(torch.float64)
    x, y = f[0], f[1]
    lin = lin.to(torch.float64).view(C, 1)
    nx = torch.sqrt((x * x).sum(0)) + EPS
    ny = torch.sqrt((y * y).sum(0)) + EPS
    dn_x = (C / 2.0 + 2.0) * U                                      # relative error of the kernel's nx
    dn_y = dn_x
    qx, qy = x / nx, y / ny
    e = qx - qy
    err_e = qx.abs() * (dn_x + U) + qy.abs() * (dn_y + U) + U * e.abs()
    e2 = e * e
    err_e2 = 2.0 * e.abs() * err_e + U * e2
    d = (lin * e2).sum(0)
    err_d = (lin.abs() * err_e2).sum(0) + C * U * (lin.abs() * e2).sum(0)
    return d, 2.0 * err_d


def partial_check(partials, d, err):
    """ratio of |partial_b - sum_p d_p| to the sum of the pixels' bounds plus the float64 sums' own rounding, per CTA
    (d, err: the head's values and bounds of every pixel in order)"""
    import torch
    n = partials.shape[0]
    pad = n * HEAD_THREADS - d.shape[0]
    d = torch.nn.functional.pad(d, (0, pad)).view(n, HEAD_THREADS)
    err = torch.nn.functional.pad(err, (0, pad)).view(n, HEAD_THREADS)
    want = d.sum(1)
    bound = err.sum(1) + 2.0 ** -52 * HEAD_THREADS * d.abs().sum(1) + 1e-300
    return ((partials.to(torch.float64) - want).abs() / bound)


# ---- finish --------------------------------------------------------------------------------------------------------------
def finish(partials, hws):
    """lpips_finish_kernel from the kernel's own partials (float64 numpy arrays): lane-strided sums, the xor butterfly,
    / hw, the five taps added in order, rounded to float32"""
    taps = []
    for p, hw in zip(partials, hws):
        p = [float(x) for x in np.asarray(p, np.float64)]
        s = [0.0] * 32
        for lane in range(32):
            for b in range(lane, len(p), 32):
                s[lane] += p[b]
        for o in (16, 8, 4, 2, 1):
            s = [s[lane] + s[lane ^ o] for lane in range(32)]
        taps.append(s[0] / float(hw))
    return np.float32((((taps[0] + taps[1]) + taps[2]) + taps[3]) + taps[4])


# ---- host emulation of the split-TF32 kernel arithmetic ----------------------------------------------------------------
def tf32(x):
    """cvt.rna.tf32.f32: round to 10 fraction bits, ties away from zero (float32 in, float32 out)"""
    b = np.ascontiguousarray(x, np.float32).view(np.uint32)
    return ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def _rz32(x):
    """float64 -> the float32 value nearest toward zero"""
    f = x.astype(np.float32)
    over = np.abs(f.astype(np.float64)) > np.abs(x)
    return np.where(over, np.nextafter(f, np.float32(0)), f)


def _mma(acc, prods, model):
    """acc [M, N] float32 plus eight exact products [M, N, 8] float64, rounded by an accumulation model"""
    if model == "rn":
        for i in range(prods.shape[-1]):
            acc = (acc.astype(np.float64) + prods[..., i]).astype(np.float32)
        return acc
    add = np.concatenate([acc.astype(np.float64)[..., None], prods], -1)
    _, e = np.frexp(np.abs(add).max(-1, keepdims=True))
    q = np.ldexp(1.0, e - 24)                                         # one ulp of the largest addend in fp32
    return _rz32(np.trunc(add / q).sum(-1) * q[..., 0])


# controlled faults of the emulation; each must exceed the bound
FAULTS = ("single_tf32", "no_lo_hi", "pad_off_by_one", "swap_images")


def im2col(inp, k, stride, pad, shift=0):
    """[2 * Ho * Wo, Cin*k*k] float32 rows of inp [2, Cin, Hi, Wi] in the kernel's M order (image, oy, ox) and K order;
    shift moves the window one column right (a padding fault)"""
    import torch
    import torch.nn.functional as F
    t = torch.from_numpy(np.ascontiguousarray(inp, np.float32))
    t = F.pad(t, (pad - shift, pad + shift, pad, pad))
    A = F.unfold(t, k, stride=stride)                                 # [2, K, L]
    return A.permute(0, 2, 1).reshape(-1, A.shape[1]).numpy()


def emulate_conv(inp, w, b, stride, pad, model="rz", fault=None, cols=None):
    """the kernel's output relu(acc + b) [2, Cout', Ho, Wo] float32 of inp [2, Cin, Hi, Wi] (float32, already normalised for
    conv0), w [Cout, Cin, k, k], b: K blocks of 32 in k8 steps, three mma per step (lo*hi, hi*lo, hi*hi) accumulated by
    `model`.  cols: the output channels to emulate (all by default)."""
    Cout, Cin, k, _ = w.shape
    Hi, Wi = inp.shape[2:]
    Ho, Wo = (Hi + 2 * pad - k) // stride + 1, (Wi + 2 * pad - k) // stride + 1
    cols = np.arange(Cout) if cols is None else np.asarray(cols)
    A = im2col(inp, k, stride, pad, shift=1 if fault == "pad_off_by_one" else 0)
    if fault == "swap_images":
        HWo = Ho * Wo
        t0 = HWo // BM * BM                                           # the M tile that holds the image boundary
        rows = np.arange(t0, min(t0 + BM, 2 * HWo))
        other = np.where(rows < HWo, rows + HWo, rows - HWo)
        A = A.copy()
        A[rows] = A[np.clip(other, 0, 2 * HWo - 1)]
    K = A.shape[1]
    Kp = (K + BK - 1) // BK * BK
    A = np.pad(A, ((0, 0), (0, Kp - K)))
    B = np.pad(np.asarray(w, np.float32).reshape(Cout, K)[cols], ((0, 0), (0, Kp - K)))
    ahi, bhi = tf32(A), tf32(B)
    alo, blo = tf32(A - ahi), tf32(B - bhi)
    f64 = lambda t: t.astype(np.float64)
    ahi, alo, bhi, blo = f64(ahi), f64(alo), f64(bhi), f64(blo)
    if fault == "single_tf32":
        terms = [(ahi, bhi)]
    elif fault == "no_lo_hi":
        terms = [(ahi, blo), (ahi, bhi)]
    else:
        terms = [(alo, bhi), (ahi, blo), (ahi, bhi)]
    acc = np.zeros((A.shape[0], len(cols)), np.float32)
    for k0 in range(0, Kp, K8):
        s = slice(k0, k0 + K8)
        for x, y in terms:
            acc = _mma(acc, x[:, None, s] * y[None, :, s], model)
    out = np.maximum((acc + np.asarray(b, np.float32)[cols]).astype(np.float32), np.float32(0))
    return out.reshape(2, Ho, Wo, len(cols)).transpose(0, 3, 1, 2)


def conv_ratio(got, v, M, S):
    """max over elements of |got - relu(v)| / conv_bound (float64 torch tensors or arrays)"""
    import torch
    got, v, M, S = (torch.as_tensor(np.asarray(t) if not isinstance(t, torch.Tensor) else t).to(torch.float64)
                    for t in (got, v, M, S))
    err = (got - v.clamp_min(0.0)).abs()
    if not bool(torch.isfinite(got).all()):
        return math.inf
    r = err / conv_bound(v, M, S)
    r = torch.where(err == 0.0, torch.zeros_like(r), r)
    return float(r.max()) if r.numel() else 0.0
