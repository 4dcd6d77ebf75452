"""Float64 restatement of csrc/preprocess_backward.cu (preprocess_backward_kernel), both output forms, with a magnitude
beside every output.

The kernel maps one Gaussian's 2-D gradients (dL/dmean2D, dL/dconic, the clamp-masked dL/dcolour) to the gradients of its
3-D parameters with a fixed float32 computation per row.  This module restates each stage of it: the forward quantities it
recomputes (cov3D from scale and quaternion, T = J W, the clamped ratios, the dilated 2-D covariance), the EWA backward,
the projection term, the SH adjoint of degrees 0..3 with the adjoint of the direction normalisation, the cov3D adjoint to
scale and quaternion, the effective-rank regulariser; for the compact form the sigmoid / exp / normalize chain rule on the
raw parameters; with `pose` each row's six camera-pose terms.

Values and magnitudes are loss_reference.Mag, with the same meaning as there: the float32 inputs are exact, every sum
costs the sum of its operands' magnitudes, so |float32 kernel - v| <= c * 2^-24 * m per element with one constant c per
output (BOUND below).  On well-conditioned rows m is within a small factor of |v|; where the float32 chain cancels (the
needle-shaped Gaussians split densification makes) m grows exactly as far as that cancellation goes.

The same code also runs in float32 (F32): numpy float32 arithmetic, one rounding per operation, branches decided on the
float32 values.  That is a float32 evaluation of the kernel's arithmetic in its order (without the fma contractions nvcc
chooses), used on the CPU to see how much of the bound such an evaluation uses.

Branches are decided in float64.  The kernel decides them on its float32 values, so a row whose branch quantity lies
within BAND * 2^-24 * m of a threshold may take either side; `band` marks those rows, and the caller evaluates them a
second time with `flip` and accepts either value.  The thresholds: txtz / tytz against the four lim* clamps (the frustum
masks of the EWA backward), the effective rank against 1 - 1e-5 and 2 - 1e-5 (the regulariser acts when
0 <= erank - 1 + 1e-5 < 1), the raw rotation's norm against 1e-12 (normalize's guard).

Two quirks of the reference are restated as the kernel keeps them: dL/dscale is the gradient with respect to mod * s
without the factor mod, and the regulariser adds 1 to dL/dscale.z whenever lambda_erank > 0.

`mutate` applies one of MUTATIONS, a plausible kernel bug, to the restatement; tests/test_preprocess_backward_reference_host.py
checks that each moves some element of its scenes beyond the bound.
"""
import numpy as np

from loss_reference import U, Mag

# |float32 kernel - v| <= c * 2^-24 * m per element.  The longest paths are about 40 roundings deep (forward recomputation,
# EWA backward, the SH contraction, the cov3D adjoint), but their errors do not align: over every case of
# tests/test_gpu_preprocess_backward_exact.py on an H100 (sm_90a) the largest err / bound with these constants was 0.27
# (dmeans3D), 0.08 (dcov3D), 0.50 (ddc), 0.63 (dsh), 0.25 (dscales), 0.07 (drots), 0.20 (g_xyz), 0.08 (g_scale),
# 0.07 (g_rot), 0.31 (g_opacity) and 0.70 (pose, the sum of the rows' bounds); the float32 evaluation of
# test_preprocess_backward_reference_host.py stays within the same ranges.  ddc and dsh are one or two roundings of exact
# inputs, so c = 2 there is already close to the worst case.
BOUND = dict(dmeans3D=4.0, dcov3D=4.0, ddc=2.0, dsh=2.0, dscales=4.0, drots=4.0,
             g_xyz=4.0, g_scale=4.0, g_rot=4.0, g_opacity=2.0, pose=4.0)
# half-width of the band around a branch threshold, in units of 2^-24 * m of the branch quantity
BAND = 4.0

MUTATIONS = ("swapped_limx", "db_without_2", "pose_unclamped_J", "quat_unscaled", "sh3_sign", "clamp_unmasked",
             "normalize_without_projection")

SH0 = 0.28209479177387814
SH1 = 0.4886025119029199
SH2a, SH2b, SH2c = 1.0925484305920792, 0.31539156525252005, 0.5462742152960396
SH3a, SH3b, SH3c, SH3d, SH3e = 0.5900435899266435, 2.890611442640554, 0.4570457994644658, 0.3731763325901154, 1.445305721320277
NORM_EPS = float(np.float32(1e-12))


class _Mag:
    """float64 with magnitudes; kernel constants as their float32 values (f64_constants: as the float64 oracle's)"""
    mag = True

    def __init__(self, f64_constants=False):
        self.f64 = f64_constants

    def k(self, c):
        """a constant factor: exact, so a product with it keeps the other operand's magnitude scaled"""
        return Mag(c if self.f64 else float(np.float32(c)), 0.0)

    def ka(self, c):
        """a constant term of a sum: the sum's rounding is relative to the result, so the constant brings its own |c|"""
        return Mag(c if self.f64 else float(np.float32(c)))

    def x(self, a):
        return Mag(np.asarray(a, np.float64))

    @staticmethod
    def val(a):
        return a.v

    @staticmethod
    def sqrt(a):
        return a.sqrt()

    @staticmethod
    def exp(a):
        return a.exp()

    @staticmethod
    def log(a):
        return a.log()

    @staticmethod
    def where(c, a, b):
        a, b = Mag.of(a), Mag.of(b)
        return Mag(np.where(c, a.v, b.v), np.where(c, a.m, b.m))

    @staticmethod
    def clip(a, lo, hi):
        """fminf(hi, fmaxf(lo, a)): a clamped value is the exact float32 limit"""
        v = np.clip(a.v, lo, hi)
        return Mag(v, np.where(v == a.v, a.m, np.abs(v)))

    @staticmethod
    def erank_ratio(e):
        """(float)(erank / ((double)erank - 1 + 1e-5)): the denominator is formed in double, exactly enough that it keeps
        the magnitude of erank"""
        return e / Mag(e.v - 1.0 + 1e-5, e.m)

    @staticmethod
    def zeros(shape):
        return Mag(np.zeros(shape), np.zeros(shape))

    @staticmethod
    def stack(parts, n):
        parts = [Mag.of(p) for p in parts]
        return Mag(np.stack([np.broadcast_to(p.v, (n,)) for p in parts], 1), np.stack([np.broadcast_to(p.m, (n,)) for p in parts], 1))


class _F32:
    """numpy float32: one rounding per operation"""
    mag = False
    f64 = False

    @staticmethod
    def k(c):
        return np.float32(c)

    ka = k

    @staticmethod
    def x(a):
        return np.asarray(a, np.float32)

    @staticmethod
    def val(a):
        return np.asarray(a, np.float64)

    @staticmethod
    def sqrt(a):
        return np.sqrt(a)

    @staticmethod
    def exp(a):
        return np.exp(a)

    @staticmethod
    def log(a):
        return np.log(a)

    @staticmethod
    def where(c, a, b):
        return np.where(c, a, b).astype(np.float32)

    @staticmethod
    def clip(a, lo, hi):
        return np.minimum(np.float32(hi), np.maximum(np.float32(lo), a))

    @staticmethod
    def erank_ratio(e):
        e = np.asarray(e, np.float64)
        return (e / (e - 1.0 + 1e-5)).astype(np.float32)

    @staticmethod
    def zeros(shape):
        return np.zeros(shape, np.float32)

    @staticmethod
    def stack(parts, n):
        return np.stack([np.broadcast_to(np.asarray(p, np.float32), (n,)) for p in parts], 1)


MAG32 = _Mag()                 # the kernel's float32 constants (what the GPU evaluates)
MAG64 = _Mag(f64_constants=True)   # the float64 oracle's constants (glic_oracle_preprocess_backward in double)
F32 = _F32()


def _sh_basis(A, D, x, y, z):
    k = A.k
    b = [k(-SH1) * y, k(SH1) * z, k(-SH1) * x]
    if D < 2:
        return b
    xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
    b += [k(SH2a) * xy, k(-SH2a) * yz, k(SH2b) * (zz * 2 - xx - yy), k(-SH2a) * xz, k(SH2c) * (xx - yy)]
    if D < 3:
        return b
    b += [k(-SH3a) * y * (xx * k(3) - yy), k(SH3b) * xy * z, k(-SH3c) * y * (zz * 4 - xx - yy),
          k(SH3d) * z * (zz * 2 - xx * k(3) - yy * k(3)), k(-SH3c) * x * (zz * 4 - xx - yy), k(SH3e) * z * (xx - yy),
          k(-SH3a) * x * (xx - yy * k(3))]
    return b


def _sh_dir_gradient(A, D, x, y, z, w, mutate):
    """dL/ddir = sum_k w_k grad b_k, in sh_math.cuh's grouping"""
    k = A.k
    gx, gy, gz = k(-SH1) * w[2], k(-SH1) * w[0], k(SH1) * w[1]
    if D < 2:
        return gx, gy, gz
    a3, a4, a5, a6, a7 = k(SH2a) * w[3], k(-SH2a) * w[4], k(SH2b) * w[5], k(-SH2a) * w[6], k(SH2c) * w[7]
    gx = gx + (a3 * y - a5 * 2 * x + a6 * z + a7 * 2 * x)
    gy = gy + (a3 * x + a4 * z - a5 * 2 * y - a7 * 2 * y)
    gz = gz + (a4 * y + a5 * 4 * z + a6 * x)
    if D < 3:
        return gx, gy, gz
    xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
    c8, c9, c10, c11 = k(-SH3a) * w[8], k(SH3b) * w[9], k(-SH3c) * w[10], k(SH3d) * w[11]
    c12, c13, c14 = k(-SH3c) * w[12], k(SH3e) * w[13], k(-SH3a) * w[14]
    t9 = -(c9 * yz) if mutate == "sh3_sign" else c9 * yz
    gx = gx + (c8 * k(6) * xy + t9 - c10 * 2 * xy - c11 * k(6) * xz + c12 * (zz * 4 - xx * k(3) - yy) + c13 * 2 * xz +
               c14 * k(3) * (xx - yy))
    gy = gy + (c8 * k(3) * (xx - yy) + c9 * xz + c10 * (zz * 4 - xx - yy * k(3)) - c11 * k(6) * yz - c12 * 2 * xy -
               c13 * 2 * yz - c14 * k(6) * xy)
    gz = gz + (c9 * xy + c10 * 8 * yz + c11 * k(3) * (zz * 2 - xx - yy) + c12 * 8 * xz + c13 * (xx - yy))
    return gx, gy, gz


def _quat_gradient(q, G):
    r, x, y, z = q
    s01, s02, s12 = G[1] + G[3], G[2] + G[6], G[5] + G[7]
    a10, a02, a21 = G[3] - G[1], G[2] - G[6], G[7] - G[5]
    return [(z * a10 + y * a02 + x * a21) * 2,
            (y * s01 + z * s02 + r * a21) * 2 - x * 4 * (G[4] + G[8]),
            (x * s01 + r * a02 + z * s12) * 2 - y * 4 * (G[0] + G[8]),
            (r * a10 + x * s02 + y * s12) * 2 - z * 4 * (G[0] + G[4])]


def _xform_row(m, r, x, y, z):
    """m[12 + r] + fma(z, m[8 + r], fma(x, m[r], y * m[4 + r]))"""
    return m[12 + r] + (z * m[8 + r] + (x * m[r] + y * m[4 + r]))


def ewa_forward(A, v, lims, fx, fy, mod_, px, py, pz, sraw, q, dilation=True):
    """geom_math.cuh cov3d_from_scale_rot and cov2d_project: the activated scale times mod, R(q), M = S R, the cov3D V =
    M^T M, the view-space position, the clamped ratios, T = J W and the 2-D covariance (a, b, c), with its 0.3 dilation"""
    s = [mod_ * si for si in sraw]
    r, x, y, z = q
    yy, zz, xz, rx, rz = y * y, z * z, x * z, r * x, r * z
    R = [A.ka(1) - (yy + zz) * 2, (x * y - rz) * 2, (r * y + xz) * 2,
         (x * y + rz) * 2, A.ka(1) - (x * x + zz) * 2, (y * z - rx) * 2,
         (xz - r * y) * 2, (y * z + rx) * 2, A.ka(1) - (x * x + yy) * 2]
    Mm = [s[i % 3] * R[i] for i in range(9)]
    V = [Mm[0] * Mm[0] + Mm[1] * Mm[1] + Mm[2] * Mm[2], Mm[3] * Mm[0] + Mm[4] * Mm[1] + Mm[5] * Mm[2],
         Mm[6] * Mm[0] + Mm[7] * Mm[1] + Mm[8] * Mm[2], Mm[3] * Mm[3] + Mm[4] * Mm[4] + Mm[5] * Mm[5],
         Mm[6] * Mm[3] + Mm[7] * Mm[4] + Mm[8] * Mm[5], Mm[6] * Mm[6] + Mm[7] * Mm[7] + Mm[8] * Mm[8]]
    tx, ty, tz = (_xform_row(v, j, px, py, pz) for j in range(3))
    txtz, tytz = tx / tz, ty / tz
    lx, ly = A.clip(txtz, lims[0], lims[1]), A.clip(tytz, lims[2], lims[3])
    tz2 = tz * tz
    J00, J11 = fx / tz, fy / tz
    J02, J12 = (fx * (lx * -tz)) / tz2, (fy * (ly * -tz)) / tz2
    T00, T01, T02 = v[2] * J02 + v[0] * J00, v[6] * J02 + v[4] * J00, v[10] * J02 + v[8] * J00
    T10, T11, T12 = v[2] * J12 + v[1] * J11, v[6] * J12 + v[5] * J11, v[10] * J12 + v[9] * J11
    A00, A01 = T00 * V[0] + T01 * V[1] + T02 * V[2], T10 * V[0] + T11 * V[1] + T12 * V[2]
    A10, A11 = T00 * V[1] + T01 * V[3] + T02 * V[4], T10 * V[1] + T11 * V[3] + T12 * V[4]
    A20, A21 = T00 * V[2] + T01 * V[4] + T02 * V[5], T10 * V[2] + T11 * V[4] + T12 * V[5]
    a = A00 * T00 + A10 * T01 + A20 * T02
    b = A01 * T00 + A11 * T01 + A21 * T02
    c = A01 * T10 + A11 * T11 + A21 * T12
    if dilation:
        a, c = a + A.ka(0.3), c + A.ka(0.3)
    return dict(s=s, R=R, Mm=Mm, V=V, tz=tz, txtz=txtz, tytz=tytz, lx=lx, ly=ly, T=(T00, T01, T02, T10, T11, T12), a=a, b=b,
                c=c)


def _band(A, q, thresholds):
    """rows whose float64 branch quantity q lies within BAND * 2^-24 * m of a threshold"""
    if not A.mag:
        return np.zeros(np.shape(q), bool)
    out = np.zeros(q.v.shape, bool)
    for t in thresholds:
        out |= np.abs(q.v - t) <= BAND * U * q.m
    return out


def backward(*args, **kw):
    with np.errstate(all="ignore"):
        return _backward(*args, **kw)


def _backward(g, cam, radii, clamped, dmean2D, dconic, dcolors, mod=1.0, lambda_erank=0.0, compact=None, pose=False, A=MAG32,
              flip=None, mutate=None):
    """preprocess_backward_kernel on P rows.

    g: dict(means [P,3], scales [P,3] (activated), rots [P,4] (as handed to the kernel), sh [P,M,3] or None (M = 0: no colour
       backward, as the kernel skips it), degree D).
    cam: dict(view [16], proj [16] (column-major), campos [3], lims [4], fx, fy): the focal lengths the kernel uses (float32
       W / (2 tan fovx) for the GPU, the oracle's float64 value against it).
    radii [P] (rows with radii <= 0 are exact zeros), clamped [P,3] (the forward's clamp bits), dmean2D [P,>=2],
    dconic [P,4] as (xx, xy, -, yy) or [P,3] as (xx, xy, yy), dcolors [P,3].
    compact: dict(opacity [P] (activated), dL_dopacity [P], rot_raw [P,4]) for the compact form's chain rule.
    pose: also each row's six pose terms (per row [P,6] and their sum).
    flip: dict(x, y, erank, nn) of bool [P]: rows that take the other side of that branch.

    Returns a dict of outputs ([P, ...] Mag, or float32 arrays with A = F32): dmeans3D, dcov3D, ddc, dsh, dscales, drots;
    with compact g_rot, g_xyz, g_scale, g_opacity; with pose pose_rows and pose; and band (dict of bool [P] per branch) and
    paths (counts of the rows that took each path)."""
    flip = flip or {}
    means, scales, rots = (np.asarray(g[k], np.float32) for k in ("means", "scales", "rots"))
    P = means.shape[0]
    sh = g.get("sh")
    sh = None if sh is None or np.asarray(sh).size == 0 else np.asarray(sh, np.float32).reshape(P, -1, 3)
    M = 0 if sh is None else sh.shape[1]
    D = int(g["degree"])
    vis = np.flatnonzero(np.asarray(radii).reshape(-1)[:P] > 0)
    n = vis.size
    k, X = A.k, A.x
    dconic = np.asarray(dconic, np.float32).reshape(P, -1)
    gc = dconic[:, [0, 1, 3]] if dconic.shape[1] == 4 else dconic
    v = [X(a) for a in np.asarray(cam["view"], np.float32)]
    pr = [X(a) for a in np.asarray(cam["proj"], np.float32)]
    cp = [X(a) for a in np.asarray(cam["campos"], np.float32)]
    lims = [float(a) for a in np.asarray(cam["lims"], np.float32)]
    fx, fy = X(cam["fx"]), X(cam["fy"])
    mod_ = X(np.float32(mod))
    px, py, pz = (X(means[vis, j]) for j in range(3))
    sraw = [X(scales[vis, j]) for j in range(3)]
    q = [X(rots[vis, j]) for j in range(4)]

    def flipped(name, cond):
        f = flip.get(name)
        return cond if f is None else cond ^ np.asarray(f, bool)[vis]

    band = {}

    # ---- forward quantities, recomputed (geom_math.cuh cov3d_from_scale_rot, cov2d_project) ---------------------------------
    e = ewa_forward(A, v, lims, fx, fy, mod_, px, py, pz, sraw, q)
    s, R, Mm, V, tz, txtz, tytz, lx, ly = (e[kk] for kk in ("s", "R", "Mm", "V", "tz", "txtz", "tytz", "lx", "ly"))
    T00, T01, T02, T10, T11, T12 = e["T"]
    a, b, c = e["a"], e["b"], e["c"]

    # ---- EWA backward --------------------------------------------------------------------------------------------------------
    tv = A.val(txtz)
    if mutate == "swapped_limx":
        xin = ~((tv < lims[1]) | (tv > lims[0]))
    else:
        xin = ~((tv < lims[0]) | (tv > lims[1]))
    yin = ~((A.val(tytz) < lims[2]) | (A.val(tytz) > lims[3]))
    band["x"], band["y"] = _band(A, txtz, lims[:2]), _band(A, tytz, lims[2:])
    xin, yin = flipped("x", xin), flipped("y", yin)
    gxx, gxy, gyy = (X(gc[vis, j]) for j in range(3))
    denom = a * c - b * b
    d2i = k(1) / (denom * denom + A.ka(1e-7))
    dLa = d2i * (-(c * c) * gxx + b * 2 * c * gxy + (denom - a * c) * gyy)
    dLc = d2i * (-(a * a) * gyy + a * 2 * b * gxy + (denom - a * c) * gxx)
    dLb = d2i * (b * c * gxx - (denom + b * 2 * b) * gxy + a * b * gyy)
    if mutate != "db_without_2":
        dLb = dLb * 2
    dcov = [T00 * T00 * dLa + T00 * T10 * dLb + T10 * T10 * dLc,
            T00 * 2 * T01 * dLa + (T00 * T11 + T01 * T10) * dLb + T10 * 2 * T11 * dLc,
            T00 * 2 * T02 * dLa + (T00 * T12 + T02 * T10) * dLb + T10 * 2 * T12 * dLc,
            T01 * T01 * dLa + T01 * T11 * dLb + T11 * T11 * dLc,
            T02 * 2 * T01 * dLa + (T01 * T12 + T02 * T11) * dLb + T11 * 2 * T12 * dLc,
            T02 * T02 * dLa + T02 * T12 * dLb + T12 * T12 * dLc]
    r00, r10 = T00 * V[0] + T01 * V[1] + T02 * V[2], T10 * V[0] + T11 * V[1] + T12 * V[2]
    r01, r11 = T00 * V[1] + T01 * V[3] + T02 * V[4], T10 * V[1] + T11 * V[3] + T12 * V[4]
    r02, r12 = T00 * V[2] + T01 * V[4] + T02 * V[5], T10 * V[2] + T11 * V[4] + T12 * V[5]
    dT = [[r00 * 2 * dLa + r10 * dLb, r01 * 2 * dLa + r11 * dLb, r02 * 2 * dLa + r12 * dLb],
          [r10 * 2 * dLc + r00 * dLb, r11 * 2 * dLc + r01 * dLb, r12 * 2 * dLc + r02 * dLb]]
    dJ00 = v[0] * dT[0][0] + v[4] * dT[0][1] + v[8] * dT[0][2]
    dJ02 = v[2] * dT[0][0] + v[6] * dT[0][1] + v[10] * dT[0][2]
    dJ11 = v[1] * dT[1][0] + v[5] * dT[1][1] + v[9] * dT[1][2]
    dJ12 = v[2] * dT[1][0] + v[6] * dT[1][1] + v[10] * dT[1][2]
    itz = k(1) / tz
    itz2 = itz * itz
    itz3 = itz2 * itz
    dtx = A.where(xin, -fx * itz2 * dJ02, k(0))
    dty = A.where(yin, -fy * itz2 * dJ12, k(0))
    dtz = -fx * itz2 * dJ00 - fy * itz2 * dJ11 + fx * 2 * (lx * tz) * itz3 * dJ02 + fy * 2 * (ly * tz) * itz3 * dJ12
    dm = [v[0] * dtx + v[1] * dty + v[2] * dtz, v[4] * dtx + v[5] * dty + v[6] * dtz, v[8] * dtx + v[9] * dty + v[10] * dtz]

    # ---- projection term -----------------------------------------------------------------------------------------------------
    hx, hy, hw = _xform_row(pr, 0, px, py, pz), _xform_row(pr, 1, px, py, pz), _xform_row(pr, 3, px, py, pz)
    m_w = k(1) / (hw + A.ka(1e-7))
    mul1, mul2 = hx * m_w * m_w, hy * m_w * m_w
    g2x, g2y = X(np.asarray(dmean2D, np.float32).reshape(P, -1)[vis, 0]), X(np.asarray(dmean2D, np.float32).reshape(P, -1)[vis, 1])
    pj = [(pr[0] * m_w - pr[3] * mul1) * g2x + (pr[1] * m_w - pr[3] * mul2) * g2y,
          (pr[4] * m_w - pr[7] * mul1) * g2x + (pr[5] * m_w - pr[7] * mul2) * g2y,
          (pr[8] * m_w - pr[11] * mul1) * g2x + (pr[9] * m_w - pr[11] * mul2) * g2y]
    dm = [dm[j] + pj[j] for j in range(3)]

    # ---- SH backward and the adjoint of dir = o / |o| -----------------------------------------------------------------------
    cl = np.asarray(clamped).reshape(P, 3)[vis].astype(bool)
    if mutate == "clamp_unmasked":
        cl[:, 1] = False
    dcol = np.asarray(dcolors, np.float32).reshape(P, 3)[vis]
    ddc = [k(0)] * 3
    dsh = []
    dsv = [k(0)] * 3
    if sh is not None:
        o = [px - cp[0], py - cp[1], pz - cp[2]]
        sum2 = o[0] * o[0] + o[1] * o[1] + o[2] * o[2]
        inv = k(1) / A.sqrt(sum2)
        dx_, dy_, dz_ = o[0] * inv, o[1] * inv, o[2] * inv
        dRGB = [X(np.where(cl[:, ch], np.float32(0), dcol[:, ch])) for ch in range(3)]
        ddc = [k(SH0) * dRGB[ch] for ch in range(3)]
        dd = [k(0)] * 3
        if D > 0:
            nb = (D + 1) ** 2 - 1
            bs = _sh_basis(A, D, dx_, dy_, dz_)
            rows = sh[vis]
            w = []
            for kk in range(nb):
                sv = [X(rows[:, kk, ch]) if kk < M else k(0) for ch in range(3)]
                w.append(sv[0] * dRGB[0] + sv[1] * dRGB[1] + sv[2] * dRGB[2])
                if kk < M:
                    dsh += [bs[kk] * dRGB[ch] for ch in range(3)]
            dd = _sh_dir_gradient(A, D, dx_, dy_, dz_, w, mutate)
        dsh += [k(0)] * (3 * M - len(dsh))
        invsum32 = k(1) / A.sqrt(sum2 * sum2 * sum2)
        dsv = [((sum2 - o[0] * o[0]) * dd[0] - o[1] * o[0] * dd[1] - o[2] * o[0] * dd[2]) * invsum32,
               (-(o[0] * o[1]) * dd[0] + (sum2 - o[1] * o[1]) * dd[1] - o[2] * o[1] * dd[2]) * invsum32,
               (-(o[0] * o[2]) * dd[0] - o[1] * o[2] * dd[1] + (sum2 - o[2] * o[2]) * dd[2]) * invsum32]
        dm = [dm[j] + dsv[j] for j in range(3)]

    # ---- cov3D backward: Sigma = M^T M, M = S R --------------------------------------------------------------------------------
    dS = [dcov[0], dcov[1] * 0.5, dcov[2] * 0.5, dcov[1] * 0.5, dcov[3], dcov[4] * 0.5, dcov[2] * 0.5, dcov[4] * 0.5, dcov[5]]
    dMt = [None] * 9
    for kk in range(3):
        for j in range(3):
            dMt[3 * j + kk] = Mm[j] * 2 * dS[3 * kk] + Mm[3 + j] * 2 * dS[3 * kk + 1] + Mm[6 + j] * 2 * dS[3 * kk + 2]
    ds = [R[j] * dMt[3 * j] + R[3 + j] * dMt[3 * j + 1] + R[6 + j] * dMt[3 * j + 2] for j in range(3)]
    sg = sraw if mutate == "quat_unscaled" else s
    G = [None] * 9
    for j in range(3):
        for kk in range(3):
            G[3 * kk + j] = dMt[3 * j + kk] * sg[j]
    dq = _quat_gradient(q, G)
    paths = dict(rows=n, xmask0=int((~xin & ~band["x"]).sum()), ymask0=int((~yin & ~band["y"]).sum()))
    if sh is not None:
        for ch in range(3):
            paths["clamped_%d" % ch] = int(cl[:, ch].sum())
    band["erank"] = np.zeros(n, bool)
    if lambda_erank > 0:
        s1s1, s2s2, s3s3 = sraw[0] * sraw[0], sraw[1] * sraw[1], sraw[2] * sraw[2]
        ssum = s1s1 + s2s2 + s3s3
        qq = [sraw[j] / ssum for j in range(3)]
        lq = [A.log(qj) for qj in qq]
        er = A.exp(-qq[0] * lq[0] - qq[1] * lq[1] - qq[2] * lq[2])
        ev = A.val(er) - 1.0 + 1e-5
        take = flipped("erank", (ev >= 0.0) & (ev < 1.0))
        band["erank"] = _band(A, er, (1.0 - 1e-5, 2.0 - 1e-5))
        paths["erank_in"], paths["erank_out"] = int((take & ~band["erank"]).sum()), int((~take & ~band["erank"]).sum())
        f = A.erank_ratio(er)
        e = [f * (-lq[j] - A.ka(1)) for j in range(3)]
        le = X(np.float32(np.float32(lambda_erank) * np.float32(2))) / (ssum * ssum)
        add = [le * sraw[0] * (e[0] * (s2s2 + s3s3) - e[1] * s2s2 - e[2] * s3s3),
               le * sraw[1] * (-e[0] * s1s1 + e[1] * (s1s1 + s3s3) - e[2] * s3s3),
               le * sraw[2] * (-e[0] * s1s1 - e[1] * s2s2 + e[2] * (s1s1 + s2s2))]
        ds = [A.where(take, ds[j] + add[j], ds[j]) for j in range(3)]
        ds[2] = ds[2] + A.ka(1)

    def full(parts):
        return _scatter(A, P, vis, A.stack(parts, n) if parts else None, len(parts))

    out = dict(dmeans3D=full(dm), dcov3D=full(dcov), ddc=full(ddc), dsh=full(dsh), dscales=full(ds), drots=full(dq))
    out["dsh"] = _reshape(out["dsh"], (P, M, 3))

    # ---- compact form: sigmoid / exp / normalize chain rule on the raw parameters -------------------------------------------
    band["nn"] = np.zeros(n, bool)
    if compact is not None:
        op = X(np.asarray(compact["opacity"], np.float32).reshape(-1)[vis])
        gop = X(np.asarray(compact["dL_dopacity"], np.float32).reshape(-1)[vis])
        rr = [X(np.asarray(compact["rot_raw"], np.float32).reshape(P, 4)[vis, j]) for j in range(4)]
        g_o = gop * (op * (A.ka(1) - op))
        g_s = [ds[j] * sraw[j] for j in range(3)]
        nn = A.sqrt(rr[0] * rr[0] + rr[1] * rr[1] + rr[2] * rr[2] + rr[3] * rr[3])
        big = flipped("nn", A.val(nn) > NORM_EPS)
        band["nn"] = _band(A, nn, (NORM_EPS,))
        paths["nn_small"] = int((~big & ~band["nn"]).sum())
        inv = k(1) / A.where(big, nn, k(1))
        qn = [rr[j] * inv for j in range(4)]
        qg = qn[0] * dq[0] + qn[1] * dq[1] + qn[2] * dq[2] + qn[3] * dq[3]
        if mutate == "normalize_without_projection":
            g_big = [dq[j] * inv for j in range(4)]
        else:
            g_big = [(dq[j] - qn[j] * qg) * inv for j in range(4)]
        g_r = [A.where(big, g_big[j], dq[j] * k(1.0 / NORM_EPS)) for j in range(4)]
        out.update(g_rot=full(g_r), g_xyz=full(dm), g_scale=full(g_s), g_opacity=_reshape(full([g_o]), (P,)))

    # ---- pose terms ----------------------------------------------------------------------------------------------------------
    if pose:
        u = [pj[j] + dsv[j] for j in range(3)]
        gv = [dtx + (v[0] * pj[0] + v[4] * pj[1] + v[8] * pj[2]),
              dty + (v[1] * pj[0] + v[5] * pj[1] + v[9] * pj[2]),
              dtz + (v[2] * pj[0] + v[6] * pj[1] + v[10] * pj[2])]
        p6 = [dtx + (v[0] * u[0] + v[4] * u[1] + v[8] * u[2]),
              dty + (v[1] * u[0] + v[5] * u[1] + v[9] * u[2]),
              dtz + (v[2] * u[0] + v[6] * u[1] + v[10] * u[2])]
        vx, vy, vz = _xform_row(v, 0, px, py, pz), _xform_row(v, 1, px, py, pz), tz
        rxr, ryr = (txtz, tytz) if mutate == "pose_unclamped_J" else (lx, ly)
        PJ00, PJ11, PJ02, PJ12 = fx * itz, fy * itz, -fx * rxr * itz, -fy * ryr * itz
        wx, wy, wz = vy * gv[2] - vz * gv[1], vz * gv[0] - vx * gv[2], vx * gv[1] - vy * gv[0]
        for cc in range(3):
            G0, G1, G2 = PJ00 * dT[0][cc], PJ11 * dT[1][cc], PJ02 * dT[0][cc] + PJ12 * dT[1][cc]
            a0, a1, a2 = v[4 * cc], v[4 * cc + 1], v[4 * cc + 2]
            wx = wx + (a1 * G2 - a2 * G1)
            wy = wy + (a2 * G0 - a0 * G2)
            wz = wz + (a0 * G1 - a1 * G0)
        rows6 = full(p6 + [wx, wy, wz])
        out["pose_rows"] = rows6
        out["pose"] = rows6.sum(0) if A.mag else rows6.astype(np.float64).sum(0)
    out["band"] = {kk: _scatter_mask(P, vis, bb) for kk, bb in band.items()}
    out["flip_rows"] = int(np.any([bb for bb in band.values()], 0).sum()) if band else 0
    out["paths"] = paths
    return out


def _scatter(A, P, vis, rows, width):
    if A.mag:
        v, m = np.zeros((P, width)), np.zeros((P, width))
        if rows is not None:
            v[vis], m[vis] = rows.v, rows.m
        return Mag(v, m)
    out = np.zeros((P, width), np.float32)
    if rows is not None:
        out[vis] = rows
    return out


def _scatter_mask(P, vis, b):
    out = np.zeros(P, bool)
    out[vis] = b
    return out


def _reshape(a, shape):
    return Mag(a.v.reshape(shape), a.m.reshape(shape)) if isinstance(a, Mag) else a.reshape(shape)


def either_ratio(got, ref, alt, c, rows_band):
    """max over elements of |got - ref| / (c 2^-24 m); on the rows in rows_band (bool [P]) the smaller of that and the same
    ratio against alt (the restatement with those rows' branches flipped).  Non-finite values fail."""
    got = np.asarray(got, np.float64)
    if not np.all(np.isfinite(got)):
        return np.inf
    r = _ratios(got, ref, c)
    if alt is not None and rows_band.any():
        ra = _ratios(got, alt, c)
        sel = rows_band.reshape((-1,) + (1,) * (got.ndim - 1)) & np.ones(got.shape, bool)
        r = np.where(sel, np.minimum(r, ra), r)
    return float(r.max()) if r.size else 0.0


def _ratios(got, ref, c):
    got = np.asarray(got, np.float64).reshape(ref.v.shape)
    err = np.abs(got - ref.v)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(err == 0.0, 0.0, err / (c * U * ref.m))
