"""Shared helpers of the parity tests (test infrastructure)."""
import numpy as np

from gaussian_lic_b200 import synthetic as syn

# Tolerances (north_star): RGB / transmittance within 1e-4 abs, tile/key indexing bit-exact.
COLOR_ATOL = 1e-4
# expf differs between glibc and the GPU's ex2.approx path by <= 2 ulp; a pixel whose alpha sits within
# that distance of the 1/255 or T<1e-4 thresholds may take the other branch on the CPU oracle (SURVEY 7.3).
# Such flips move a pixel by <= alpha*T*c ~ 4e-3; we allow a vanishing fraction of them, bounded in size.
FLIP_FRACTION = 2e-5
FLIP_MAX = 2e-2
GRAD_RTOL = 2e-3       # relative to the max |grad| of the tensor (fp32 atomics reorder sums)


def small_scene(P=3000, W=320, H=208, seed=11, deg=3, zmax=12.0, f=250.0, log_scale_mean=-3.0, view=0, pp=(0.0, 0.0),
                radius=2.0):
    """Gaussians in the world (= view-0 camera) frame + the camera of rig view `view` (synthetic.orbit_pose: view 0 is
    the identity pose, v >= 1 sits on a circle of `radius` around (0,0,10) and looks at it => R != I, t != 0).
    pp = principal-point offset in pixels from the image centre (cx = W/2 + pp[0], cy = H/2 + pp[1]): a non-zero offset
    makes all four lim* clamps of camera.h:63-66 differ and P02 / P12 of the projection non-zero."""
    g = syn.make_gaussians(P, W, H, f, f, sh_degree=deg, zmax=zmax, seed=seed, log_scale_mean=log_scale_mean)
    R_wc, t_wc = syn.orbit_pose(view, radius=radius)
    cam = syn.make_camera(W, H, f, f, W / 2.0 + pp[0], H / 2.0 + pp[1], R_wc, t_wc)
    return g, cam


# (view, principal-point offset): the identity pose, rotated + translated rig views, and an off-centre principal point
POSES = [(0, (0.0, 0.0)), (1, (0.0, 0.0)), (3, (0.0, 0.0)), (5, (17.5, -9.25)), (0, (-23.0, 11.5))]


def image_close(a, b, what):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    err = np.abs(a - b)
    bad = err > COLOR_ATOL
    frac = bad.mean()
    msg = "%s: max err %.3e, frac>1e-4 = %.3e (%d px)" % (what, err.max(), frac, bad.sum())
    print(msg)
    assert frac <= FLIP_FRACTION, msg
    assert err.max() <= FLIP_MAX, msg


def max_abs_close(a, b, what, atol=COLOR_ATOL):
    """every element within atol (the CUDA path against the reference's own CUDA: no threshold flips are allowed)"""
    err = float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max())
    print("%s: max err %.3e" % (what, err))
    assert err <= atol, (what, err)


# Element-wise criterion on top of the norm-relative one: |a-b| <= EL_RTOL*|b| + EL_ATOL*max|b| for every entry, so that
# small-magnitude entries (most of dL_dsh, dL_drots) are constrained too.  A gradient entry is a sum of up to thousands of
# fp32 terms of both signs, so its rounding noise scales with the tensor (the EL_ATOL term: the f32 oracle differs from
# the f64 oracle by <= 5e-6*max|b| there); EL_FRAC entries may miss it (a pixel whose alpha sits on the 1/255 or T<1e-4
# threshold takes the other branch and moves the Gaussians it touches by a whole pixel contribution).
EL_RTOL = 5e-3
EL_ATOL = 5e-5
EL_FRAC = 1e-3


def grad_close(a, b, what, rtol=GRAD_RTOL, el_rtol=EL_RTOL, el_atol=EL_ATOL, el_frac=EL_FRAC, scale=None):
    """scale: max |ref| of the whole tensor when a and b are a sample of it (defaults to the max over b)"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    assert np.isfinite(a).all(), what + " has non-finite values"
    sampled = scale is not None
    scale = max(np.abs(b).max() if scale is None else scale, 1e-12)
    diff = np.abs(a - b)
    err = diff.max() / scale
    bad = diff > el_rtol * np.abs(b) + el_atol * scale
    frac = float(bad.mean()) if bad.size else 0.0
    if sampled and bad.size:
        frac = max(0.0, float(bad.sum()) - 1.0) / bad.size          # a sample may hold one of the el_frac outliers
    big = np.abs(b) > 1e-3 * scale
    rel_big = float((diff[big] / np.abs(b)[big]).max()) if big.any() else 0.0
    print("%s: max|diff|/max|ref| = %.3e (scale %.3e); element-wise: %.3e of %d entries beyond %.0e*|ref| + %.0e*max, "
          "max rel err over entries > 1e-3*max = %.3e" % (what, err, scale, frac, bad.size, el_rtol, el_atol, rel_big))
    assert err <= rtol, "%s rel err %.3e > %.1e" % (what, err, rtol)
    assert frac <= el_frac, "%s: %.3e of the entries fail the element-wise bound (allowed %.1e)" % (what, frac, el_frac)


# ---- path predicates of the stress scenes (tests/test_stress_scenes.py, tests/test_gpu_stress.py) ------------------------------
def hy_fallbacks(conic_opacity, vis):
    """Visible Gaussians whose render row cull takes the 1.11 * radius + 1 fallback: the conic's determinant cancels,
    dcon <= 1e-3 * prod (preprocess.cu, where hy is computed; f32 as there)."""
    co = np.asarray(conic_opacity, np.float32)
    prod = (co[:, 0] * co[:, 2]).astype(np.float32)
    dcon = (prod - (co[:, 1] * co[:, 1]).astype(np.float32)).astype(np.float32)
    return int((vis & ~(dcon > np.float32(1e-3) * prod)).sum())


def tile_rects(xy, radii, W, H):
    """getRect of every Gaussian: (x0, y0, x1, y1) in tiles, clamped to the grid (f32 arithmetic, truncation)"""
    gx, gy = (W + 15) // 16, (H + 15) // 16
    x, y = np.asarray(xy, np.float32)[:, 0], np.asarray(xy, np.float32)[:, 1]
    r = np.asarray(radii).astype(np.float32)
    q = np.float32(0.0625)

    def cl(v, hi):
        return np.clip(np.trunc(v).astype(np.int64), 0, hi)
    return (cl((x - r) * q, gx), cl((y - r) * q, gy), cl((x + r + np.float32(16) - np.float32(1)) * q, gx),
            cl((y + r + np.float32(16) - np.float32(1)) * q, gy))


def big_rect_rows(xy, radii, W, H):
    """rows of the rects of more than 32 tiles: what the counting walk asks of the 4P-entry span arena"""
    x0, y0, x1, y1 = tile_rects(xy, radii, W, H)
    n = (x1 - x0) * (y1 - y0)
    vis = np.asarray(radii) > 0
    return int((y1 - y0)[vis & (n > 32)].sum())



# ---- golden vectors of the reference itself (tests/golden/make_reference_pins.py) ------------------------------------------
# The reference's outputs at the sizes of the reference-pin tests are stored compactly: integer outputs as SHA-256 digests,
# images and gradients as a seeded sample plus whole-tensor statistics.
PIN_SCENES = [(4096, 320, 208, 3, 11), (10240, 640, 480, 0, 42), (25600, 800, 450, 3, 8)]     # (P, W, H, degree, seed)
ITER_ORDER = ("means", "dc", "sh", "op", "log_s", "rot")                 # trainingSetup order, gaussian.cpp:399-424
ITER_LRS = [1.6e-4, 2.5e-3, 2.5e-3 / 20.0, 0.05, 0.005, 0.001]           # config/fastlivo.yaml:18-22
ITER_CASES = [s + (v, pp) for s in PIN_SCENES[:2] for v, pp in POSES[:4]]  # (P, W, H, degree, seed, view, pp)
# the benchmark workload (synthetic.make_scene("cfg2")) trimmed to a multiple of 256, identity / rig views, off-centre principal point
CFG2_P = 499_968
CFG2_CASES = [(0, (0.0, 0.0)), (1, (0.0, 0.0)), (3, (0.0, 0.0)), (5, (41.5, -27.25))]
N_PIX = 1024
N_ROWS = 64
STAT_RTOL = 1e-3       # least tolerance of sum |x| and max |x| over a whole tensor (fp32 atomics reorder sums)


def pin_key(P, seed, view, pp):
    return "P%d_s%d_v%d_pp%g_%g" % (P, seed, view, pp[0], pp[1])


def golden_dL(H, W, seed):
    """dL/dpixel of the backward pins (numpy: identical on every machine)"""
    return np.random.default_rng(1000 + seed).normal(size=(3, H, W)).astype(np.float32)


def digest(a):
    """SHA-256 of an integer / float array's bits in canonical little-endian unsigned form"""
    import hashlib
    a = np.ascontiguousarray(np.asarray(a))
    a = a.view({1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[a.dtype.itemsize]).astype(
        {1: "<u1", 2: "<u2", 4: "<u4", 8: "<u8"}[a.dtype.itemsize])
    return hashlib.sha256(a.tobytes()).hexdigest()


def sample_pixels(H, W, seed):
    return np.sort(np.random.default_rng(2000 + seed).choice(H * W, size=min(N_PIX, H * W), replace=False))


def sample_rows(vis, seed):
    idx = np.flatnonzero(vis)
    return np.sort(np.random.default_rng(3000 + seed).choice(idx, size=min(N_ROWS, idx.size), replace=False))


def tensor_stats(a):
    a = np.abs(np.asarray(a, np.float64))
    return np.array([a.max() if a.size else 0.0, a.sum()], np.float64)


class Golden:
    """One case of a golden file: gold.sha(name, array), gold.image(name, img), gold.grad(name, tensor, vis)."""

    def __init__(self, name, key):
        import os
        import pytest
        path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", name + ".npz")
        if not os.path.isfile(path):
            pytest.skip("golden vector %s not generated yet" % name)
        self.z, self.key = np.load(path), key
        self.stored = {k[len(key) + 1:] for k in self.z.files if k.startswith(key + "/")}
        assert self.stored, "no golden case " + key

    def __getitem__(self, n):
        return self.z[self.key + "/" + n]

    def has(self, n):
        return n + "/stats" in self.stored

    def sha(self, n, a):
        assert digest(a) == bytes(self["sha/" + n]).hex(), "%s differs from the reference (bit-exact)" % n

    def stats_close(self, n, a, what, rtol=STAT_RTOL, max_atol=0.0):
        mx, s = tensor_stats(a)
        gmx, gs = self[n + "/stats"]
        print("%s: max|x| %.6e vs %.6e, sum|x| %.6e vs %.6e" % (what, mx, gmx, s, gs))
        assert abs(mx - gmx) <= rtol * max(gmx, 1e-12) + max_atol, (what, "max |x|", mx, gmx)
        assert abs(s - gs) <= rtol * max(gs, 1e-12), (what, "sum |x|", s, gs)

    def image(self, n, img, pix, what, check=None):
        """img [C,H,W] or [H,W]: the stored pixel sample through `check` (default image_close) + whole-image statistics"""
        img = np.asarray(img, np.float32)
        mine = img.reshape(-1, img.shape[-2] * img.shape[-1])[:, pix] if img.ndim == 3 else img.reshape(-1)[pix]
        (check or image_close)(mine, self[n + "/pix"], what)
        self.stats_close(n, img, what, max_atol=FLIP_MAX)

    def grad(self, n, a, rows, what, rtol=GRAD_RTOL):
        a = np.asarray(a, np.float32)
        ref = self[n + "/rows"]
        grad_close(a.reshape(a.shape[0], -1)[rows], ref, what, rtol=rtol, scale=float(self[n + "/stats"][0]))
        self.stats_close(n, a, what, rtol=max(rtol, STAT_RTOL))
