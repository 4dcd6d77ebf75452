"""Deterministic synthetic scenes for parity tests and benchmarks (SURVEY.md 8(d)).

Pure numpy (host side); the same arrays feed the CUDA path, the CPU oracle and the
reference build, so every implementation sees identical bits.

Camera math restates /root/reference/src/camera.h:38-110 (FoV, view / projection matrices
in the column-major layout the kernels receive, asymmetric lim clamps) in closed form.
"""
import math

import numpy as np

CONFIGS = {
    # name: (P, W, H, fx, fy, cx, cy, sh_degree, zmax)
    "cfg1": (10_000, 640, 480, 400.0, 400.0, 320.0, 240.0, 0, 20.0),
    "cfg2": (500_000, 1920, 1080, 1000.0, 1000.0, 960.0, 540.0, 3, 20.0),
    "cfg3": (2_000_000, 1920, 1080, 1000.0, 1000.0, 960.0, 540.0, 3, 20.0),
    "cfg4": (5_000_000, 1920, 1080, 1000.0, 1000.0, 960.0, 540.0, 3, 60.0),
}


def make_camera(W, H, fx, fy, cx, cy, R_wc=None, t_wc=None):
    """Pinhole camera -> the 16+16+3 floats + scalars handed to the rasterizer.

    view[4c+r] = Rt[r][c] and proj[4c+r] = (P*Rt)[r][c] (column-major, see SURVEY App. A.1).
    """
    R_wc = np.eye(3) if R_wc is None else np.asarray(R_wc, np.float64)
    t_wc = np.zeros(3) if t_wc is None else np.asarray(t_wc, np.float64)
    R_cw = R_wc.T
    t_cw = -R_wc.T @ t_wc
    Rt = np.eye(4, dtype=np.float32)
    Rt[:3, :3] = R_cw.astype(np.float32)
    Rt[:3, 3] = t_cw.astype(np.float32)
    fovx = np.float32(2.0 * math.atan(W / (2.0 * fx)))
    fovy = np.float32(2.0 * math.atan(H / (2.0 * fy)))
    znear, zfar = np.float32(0.01), np.float32(100.0)
    Pm = np.zeros((4, 4), np.float32)
    Pm[0, 0] = np.float32(1.0 / math.tan(float(fovx) / 2))
    Pm[1, 1] = np.float32(1.0 / math.tan(float(fovy) / 2))
    Pm[0, 2] = (np.float32(2) * np.float32(cx) - np.float32(W)) / np.float32(W)
    Pm[1, 2] = (np.float32(2) * np.float32(cy) - np.float32(H)) / np.float32(H)
    Pm[3, 2] = 1.0
    Pm[2, 2] = zfar / (zfar - znear)
    Pm[2, 3] = -(zfar * znear) / (zfar - znear)
    full = (Pm @ Rt).astype(np.float32)
    campos = (-(R_cw.T @ t_cw)).astype(np.float32)
    ffx, ffy, fcx, fcy = np.float32(fx), np.float32(fy), np.float32(cx), np.float32(cy)
    lims = np.array([-0.15 * W / ffx - fcx / ffx, 1.15 * W / ffx - fcx / ffx,
                     -0.15 * H / ffy - fcy / ffy, 1.15 * H / ffy - fcy / ffy], np.float32)
    return dict(W=int(W), H=int(H), view=np.ascontiguousarray(Rt.T).reshape(16).copy(),
                proj=np.ascontiguousarray(full.T).reshape(16).copy(), campos=campos,
                tanfovx=float(np.tan(np.float32(fovx * np.float32(0.5)))),
                tanfovy=float(np.tan(np.float32(fovy * np.float32(0.5)))), lims=lims)


def orbit_pose(v, n_views=8, radius=2.0, target=(0.0, 0.0, 10.0)):
    """View v of the closed-form multi-view rig (SURVEY 8(d)); view 0 is the identity pose."""
    if v == 0:
        return np.eye(3), np.zeros(3)
    ang = 2.0 * math.pi * v / n_views
    tgt = np.asarray(target, np.float64)
    pos = np.array([radius * math.sin(ang), 0.0, radius * (1.0 - math.cos(ang))])
    fwd = tgt - pos
    fwd /= np.linalg.norm(fwd)
    up = np.array([0.0, -1.0, 0.0])
    right = np.cross(fwd, up)
    right /= np.linalg.norm(right)
    down = np.cross(fwd, right)
    R_wc = np.stack([right, down, fwd], axis=1)  # camera axes (x right, y down, z forward) in world
    return R_wc, pos


def make_gaussians(P, W, H, fx, fy, sh_degree=3, zmax=20.0, seed=42, log_scale_mean=-4.0):
    """Activated Gaussian parameters in the view-0 (= world) frame."""
    rng = np.random.Generator(np.random.Philox(seed))
    z = rng.uniform(-1.0, zmax, P)
    x = np.abs(z) * rng.uniform(-1.1 * W / (2 * fx), 1.1 * W / (2 * fx), P)
    y = np.abs(z) * rng.uniform(-1.1 * H / (2 * fy), 1.1 * H / (2 * fy), P)
    means = np.stack([x, y, z], 1).astype(np.float32)
    log_scales = rng.normal(log_scale_mean, 0.6, (P, 3)).astype(np.float32)
    q = rng.normal(0.0, 1.0, (P, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    logits = rng.normal(0.0, 2.0, P)
    logits[rng.random(P) < 0.02] = -7.0
    dc = rng.normal(0.0, 1.0, (P, 3)).astype(np.float32)
    M = (sh_degree + 1) ** 2 - 1
    sh = rng.normal(0.0, 0.1, (P, M, 3)).astype(np.float32)
    return dict(means=means, scales=np.exp(log_scales).astype(np.float32), rots=q.astype(np.float32),
                opacity=(1.0 / (1.0 + np.exp(-logits))).astype(np.float32), dc=dc, sh=sh, degree=int(sh_degree),
                log_scales=log_scales, opacity_logits=logits.astype(np.float32))


# ---- stress scenes: the splat shapes, depth stacks and frame positions make_gaussians never produces ---------------------
# kind: (P, W, H, f).  Every P is a multiple of 256.
STRESS = {
    "needles": (4096, 320, 208, 250.0),   # long / short scale ratio 1e2 .. 1e4: conics whose determinant cancels
    "big": (4096, 480, 320, 300.0),       # rects of tens to all 600 tiles: big-rect rows overflow the 4P span arena
    "deep": (4096, 160, 112, 200.0),      # >= 2000 splats over a few tiles: >= 8 forward rounds of 256 splats
    "ties": (4096, 320, 208, 250.0),      # groups of bit-identical depth and exact duplicates (identity pose: depth = z)
    "edges": (2048, 256, 176, 220.0),     # the z = 0.2 cull, the four lim* clamps, rects clamped at every border, alpha clamps
}


def _quat_z(phi):
    """rotation by phi about the optical axis: the splat's local x axis lies at angle phi in the image"""
    return np.stack([np.cos(phi / 2), np.zeros_like(phi), np.zeros_like(phi), np.sin(phi / 2)], 1)


def _random_quat(rng, n):
    q = rng.normal(0.0, 1.0, (n, 4))
    return q / np.linalg.norm(q, axis=1, keepdims=True)


def _finish(means, scales, q, opacity, rng, deg):
    P = means.shape[0]
    M = (deg + 1) ** 2 - 1
    opacity = np.asarray(opacity, np.float64)
    return dict(means=np.asarray(means, np.float32), scales=np.asarray(scales, np.float32),
                rots=(q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32),
                opacity=opacity.astype(np.float32), dc=rng.normal(0.0, 1.0, (P, 3)).astype(np.float32),
                sh=rng.normal(0.0, 0.1, (P, M, 3)).astype(np.float32), degree=int(deg),
                log_scales=np.log(np.asarray(scales, np.float32)).astype(np.float32),
                opacity_logits=np.log(opacity / (1.0 - np.minimum(opacity, 1.0 - 1e-7))).astype(np.float32))


def make_stress_scene(kind, view=0, pp=(0.0, 0.0), seed=0, opaque=False, deg=2):
    """(g, cam) of stress scene `kind` (STRESS) in the format of make_gaussians / make_camera, for rig view `view` and
    principal-point offset `pp`.  Deterministic.  `opaque` selects the high-opacity variant of "deep": its pixels cross
    T < 1e-4 at different points of a 256-splat round, so most of their tiles' buckets are never reached."""
    P, W, H, f = STRESS[kind]
    rng = np.random.Generator(np.random.Philox(1000 + 17 * seed + list(STRESS).index(kind)))
    cx, cy = W / 2.0, H / 2.0

    def at_pixels(u, v, z):      # world (= view-0 camera) points seen by the identity pose at pixel (u, v), depth z
        return np.stack([(u - cx) / f * z, (v - cy) / f * z, z], 1)

    def sigma_px_to_world(s_px, z):
        return s_px * z / f

    if kind == "needles":
        z = rng.uniform(2.0, 14.0, P)
        means = at_pixels(rng.uniform(-0.1 * W, 1.1 * W, P), rng.uniform(-0.1 * H, 1.1 * H, P), z)
        long_px = np.exp(rng.uniform(np.log(4.0), np.log(160.0), P))
        ratio = np.exp(rng.uniform(np.log(1e2), np.log(1e4), P))
        s_long = sigma_px_to_world(long_px, z)
        scales = np.stack([s_long, s_long / ratio, s_long / np.exp(rng.uniform(np.log(1e2), np.log(1e4), P))], 1)
        # a quarter nearly axis-aligned, a quarter nearly diagonal (both in the image plane), half at random 3-D orientations
        k = rng.integers(0, 4, P)
        phi = np.where(k == 0, rng.integers(0, 2, P) * (np.pi / 2) + rng.normal(0.0, 1e-3, P),
                       rng.integers(0, 4, P) * (np.pi / 2) + np.pi / 4 + rng.normal(0.0, 2e-2, P))
        q = np.where((k <= 1)[:, None], _quat_z(phi), _random_quat(rng, P))
        opacity = rng.uniform(0.02, 0.95, P)
    elif kind == "big":
        # half of the splats close to the camera with screen radii of 40 .. 400 px, the rest ordinary background;
        # shuffled so that the span arena runs out part-way through the CTAs
        big = rng.random(P) < 0.5
        z = np.where(big, rng.uniform(1.5, 5.0, P), rng.uniform(4.0, 20.0, P))
        means = at_pixels(rng.uniform(-0.2 * W, 1.2 * W, P), rng.uniform(-0.2 * H, 1.2 * H, P), z)
        s_px = np.where(big, np.exp(rng.uniform(np.log(14.0), np.log(130.0), P)), np.exp(rng.uniform(np.log(0.5), np.log(4.0), P)))
        aniso = np.exp(rng.normal(0.0, 0.4, (P, 3)))
        scales = sigma_px_to_world(s_px, z)[:, None] * aniso
        q = _random_quat(rng, P)
        opacity = np.where(big, rng.uniform(0.01, 0.25, P), rng.uniform(0.05, 0.95, P))
    elif kind == "deep":
        # 15/16 of the splats over a 24 x 24 px patch in the middle of the frame, the rest scattered
        stack = rng.random(P) < 15.0 / 16.0
        z = rng.uniform(2.0, 12.0, P)
        u = np.where(stack, cx - 12.0 + rng.uniform(0.0, 24.0, P), rng.uniform(0.0, W, P))
        v = np.where(stack, cy - 12.0 + rng.uniform(0.0, 24.0, P), rng.uniform(0.0, H, P))
        means = at_pixels(u, v, z)
        scales = sigma_px_to_world(rng.uniform(3.0, 9.0, P), z)[:, None] * np.exp(rng.normal(0.0, 0.2, (P, 3)))
        q = _random_quat(rng, P)
        # low: alpha never far above 1/255, so no pixel saturates through ~3500 splats; high: T < 1e-4 after tens to hundreds
        opacity = rng.uniform(0.02, 0.3, P) if opaque else rng.uniform(0.0045, 0.0075, P)
    elif kind == "ties":
        # 24 depths shared by groups of ~150 splats each, the last quarter exact copies of earlier ones
        n = P - P // 4
        depths = np.sort(rng.uniform(2.0, 12.0, 24)).astype(np.float32)
        z = depths[rng.integers(0, 24, n)].astype(np.float64)
        means = at_pixels(rng.uniform(0.0, W, n), rng.uniform(0.0, H, n), z)
        means[:, 2] = z                                                   # exactly the float32 depth
        scales = sigma_px_to_world(np.exp(rng.uniform(np.log(1.0), np.log(12.0), n)), z)[:, None] * np.exp(rng.normal(0.0, 0.3, (n, 3)))
        q = _random_quat(rng, n)
        opacity = rng.uniform(0.05, 0.9, n)
        src = rng.integers(0, n, P - n)
        means, scales, q, opacity = (np.concatenate([a, a[src]]) for a in (means, scales, q, opacity))
        g = _finish(means, scales, q, opacity, rng, deg)
        for k in ("dc", "sh"):
            g[k][n:] = g[k][src]
        R_wc, t_wc = orbit_pose(view)
        return g, make_camera(W, H, f, f, cx + pp[0], cy + pp[1], R_wc, t_wc)
    elif kind == "edges":
        n4 = P // 4
        parts_m, parts_s = [], []
        # 1. just past the near cull: z in (0.2, 0.25] (plus a few exactly at 0.2 and one float32 ulp above it)
        z = rng.uniform(0.2, 0.25, n4)
        z[:16] = 0.2
        z[16:32] = np.nextafter(np.float32(0.2), np.float32(1.0))
        parts_m.append(at_pixels(rng.uniform(0.0, W, n4), rng.uniform(0.0, H, n4), z))
        parts_s.append(sigma_px_to_world(rng.uniform(1.0, 25.0, n4), z))
        # 2. on and just outside the four lim* clamps (1.15 / -0.15 of the frame, measured from the principal point)
        ccx, ccy = cx + pp[0], cy + pp[1]
        lim = np.array([(-0.15 * W - ccx) / f, (1.15 * W - ccx) / f, (-0.15 * H - ccy) / f, (1.15 * H - ccy) / f])
        z = rng.uniform(1.0, 10.0, n4)
        side = rng.integers(0, 4, n4)
        over = np.choose(rng.integers(0, 4, n4), [np.ones(n4), np.full(n4, 1.0 + 1e-6), np.full(n4, 1.01), np.full(n4, 1.2)])
        tx = rng.uniform(lim[0], lim[1], n4)
        ty = rng.uniform(lim[2], lim[3], n4)
        tx = np.where(side == 0, lim[0] * over, np.where(side == 1, lim[1] * over, tx))
        ty = np.where(side == 2, lim[2] * over, np.where(side == 3, lim[3] * over, ty))
        parts_m.append(np.stack([tx * z, ty * z, z], 1))
        parts_s.append(sigma_px_to_world(rng.uniform(2.0, 40.0, n4), z))
        # 3. big rects clamped at every border: centres on or beyond the border, radii of 20 .. 120 px
        z = rng.uniform(1.5, 8.0, n4)
        b = rng.integers(0, 4, n4)
        u = np.where(b == 0, rng.uniform(-60.0, 2.0, n4), np.where(b == 1, rng.uniform(W - 2.0, W + 60.0, n4), rng.uniform(0.0, W, n4)))
        v = np.where(b == 2, rng.uniform(-60.0, 2.0, n4), np.where(b == 3, rng.uniform(H - 2.0, H + 60.0, n4), rng.uniform(0.0, H, n4)))
        parts_m.append(at_pixels(u, v, z))
        parts_s.append(sigma_px_to_world(rng.uniform(7.0, 40.0, n4), z))
        # 4. ordinary splats carrying the opacity edge cases
        n = P - 3 * n4
        z = rng.uniform(2.0, 12.0, n)
        parts_m.append(at_pixels(rng.uniform(0.0, W, n), rng.uniform(0.0, H, n), z))
        parts_s.append(sigma_px_to_world(rng.uniform(1.0, 10.0, n), z))
        means = np.concatenate(parts_m)
        scales = np.concatenate(parts_s)[:, None] * np.exp(rng.normal(0.0, 0.3, (P, 3)))
        q = _random_quat(rng, P)
        t = np.float32(1.0 / 255.0)
        edge_op = np.array([np.nextafter(t, np.float32(0)), t, np.nextafter(t, np.float32(1)), 0.0040, 0.0045, 0.99,
                            0.995, 0.999, np.nextafter(np.float32(1), np.float32(0)), 1.0], np.float64)
        opacity = np.where(rng.random(P) < 0.5, edge_op[rng.integers(0, edge_op.size, P)], rng.uniform(0.05, 0.95, P))
        perm = rng.permutation(P)                           # mix the cases across CTAs
        means, scales, q, opacity = means[perm], scales[perm], q[perm], opacity[perm]
    else:
        raise ValueError("unknown stress scene %r" % (kind,))
    g = _finish(means, scales, q, opacity, rng, deg)
    R_wc, t_wc = orbit_pose(view)
    return g, make_camera(W, H, f, f, cx + pp[0], cy + pp[1], R_wc, t_wc)


def make_frame_scene(W, H, P=2048, seed=0, deg=1):
    """A few thousand ordinary Gaussians seen by the identity pose of a W x H frame of any shape: focal length and splat
    size scale with the frame, so that splats cover a few pixels at every size (from 1 x 1 to 4096 x 4096)."""
    f = 0.8 * max(W, H)
    g = make_gaussians(P, W, H, f, f, sh_degree=deg, zmax=12.0, seed=seed, log_scale_mean=float(np.log(3.0 * 6.0 / f)))
    return g, make_camera(W, H, f, f, W / 2.0, H / 2.0)


def make_gt_image(W, H, seed=7):
    """Low-frequency random RGB image in [0,1]: sum of 16 random 2-D cosines per channel."""
    rng = np.random.Generator(np.random.Philox(seed))
    yy, xx = np.meshgrid(np.arange(H, dtype=np.float64) / H, np.arange(W, dtype=np.float64) / W, indexing="ij")
    img = np.zeros((3, H, W))
    for ch in range(3):
        for _ in range(16):
            kx, ky = rng.uniform(-6, 6, 2)
            ph = rng.uniform(0, 2 * math.pi)
            img[ch] += rng.uniform(0.2, 1.0) * np.cos(2 * math.pi * (kx * xx + ky * yy) + ph)
        img[ch] = (img[ch] - img[ch].min()) / (img[ch].max() - img[ch].min())
    return img.astype(np.float32)


def make_scene(name="cfg1", P=None, seed=42, view=0, pp=(0.0, 0.0), radius=2.0, **overrides):
    """Gaussians of config `name` + the camera of rig view `view`; pp = principal-point offset (pixels) from the config's."""
    Pn, W, H, fx, fy, cx, cy, deg, zmax = CONFIGS[name]
    P = Pn if P is None else P
    deg = overrides.pop("sh_degree", deg)
    g = make_gaussians(P, W, H, fx, fy, sh_degree=deg, zmax=zmax, seed=seed, **overrides)
    R_wc, t_wc = orbit_pose(view, radius=radius)
    cam = make_camera(W, H, fx, fy, cx + pp[0], cy + pp[1], R_wc, t_wc)
    return g, cam


def make_sort_pairs(n, seed=99, tiles=8160):
    """cfg5: key = (tile << 32) | float_bits(depth in [0.2, 100)), value = index."""
    rng = np.random.Generator(np.random.Philox(seed))
    tile = rng.integers(0, tiles, n, dtype=np.uint64)
    depth = rng.uniform(0.2, 100.0, n).astype(np.float32)
    keys = (tile << np.uint64(32)) | depth.view(np.uint32).astype(np.uint64)
    vals = np.arange(n, dtype=np.uint32)
    return keys, vals
