"""Vectorised NumPy restatement of extend()'s point selection (csrc/extend.cu, gaussian.cpp:499-607) -- test infrastructure.

Every float32 step is one NumPy float32 operation, rounded once like the device's _rn intrinsics, so the camera and pixel
coordinates are the kernel's bit for bit.  select() reproduces the whole selection in O(n log n): the per-pixel winner by np.lexsort on
(pixel key, camera depth with -0.0 folded onto +0.0, index), then the survivors (in the image, depth_rsp > 0, 1 - T < 0.99f) in
ascending index order.  It takes the camera coordinates from the caller when given, so the selection the reference's own
tensor arithmetic implies can be formed from coordinates torch computed.
"""
import numpy as np

F32 = np.float32
ALPHA_MAX = F32(0.99)


def camera_coords(points, R_cw, t_cw):
    """R_cw p + t_cw in extend_pixel's order: ((p0 r0 + p1 r1) + p2 r2) + t per row, every step rounded to float32"""
    p = np.asarray(points, F32).reshape(-1, 3)
    R = np.asarray(R_cw, F32).reshape(3, 3)
    t = np.asarray(t_cw, F32).reshape(3)
    with np.errstate(all="ignore"):
        return ((p[:, 0:1] * R[:, 0] + p[:, 1:2] * R[:, 1]) + p[:, 2:3] * R[:, 2]) + t


def pixel_coords(cam, fx, fy, cx, cy):
    """(x * fx) / z + cx and the same for y, each step rounded to float32 (not yet floored)"""
    cam = np.asarray(cam, F32).reshape(-1, 3)
    with np.errstate(all="ignore"):
        xf = (cam[:, 0] * F32(fx)) / cam[:, 2] + F32(cx)
        yf = (cam[:, 1] * F32(fy)) / cam[:, 2] + F32(cy)
    return xf, yf


def select(points, depth_rsp, R_cw, t_cw, fx, fy, cx, cy, W, H, final_T, cam=None):
    """The selection of extend() -> dict(cam, xf, yf (float32 pixel coordinates), px, py (floored, int64; -1 where not in
    the image), in_image, winner (bool per point), keep (ascending int32 indices of the survivors)).

    A point takes part when floor(xf) is in [0, W) and floor(yf) in [0, H); NaN and infinite coordinates never are.  The
    winner of a pixel has the smallest camera depth, -0.0 and +0.0 being equal, and the smallest index among equal depths."""
    if cam is None:
        cam = camera_coords(points, R_cw, t_cw)
    cam = np.asarray(cam, F32).reshape(-1, 3)
    n = cam.shape[0]
    xf, yf = pixel_coords(cam, fx, fy, cx, cy)
    with np.errstate(invalid="ignore"):
        fxp, fyp = np.floor(xf), np.floor(yf)
        inside = (fxp >= 0) & (fxp < W) & (fyp >= 0) & (fyp < H)
    px = np.where(inside, fxp, -1).astype(np.int64)
    py = np.where(inside, fyp, -1).astype(np.int64)
    idx = np.flatnonzero(inside)
    winner = np.zeros(n, bool)
    if idx.size:
        key = py[idx] * W + px[idx]
        depth = cam[idx, 2] + F32(0.0)                        # -0.0 -> +0.0
        order = np.lexsort((idx, depth, key))                  # last key is the primary one
        k_sorted = key[order]
        first = np.ones(order.size, bool)
        first[1:] = k_sorted[1:] != k_sorted[:-1]
        winner[idx[order[first]]] = True
    T = np.asarray(final_T, F32).reshape(H, W)
    rsp = np.asarray(depth_rsp, F32).reshape(-1)
    alpha = np.ones(n, F32)
    alpha[inside] = F32(1.0) - T[py[inside], px[inside]]
    keep = np.flatnonzero(winner & (rsp > 0) & (alpha < ALPHA_MAX)).astype(np.int32)
    return dict(cam=cam, xf=xf, yf=yf, px=px, py=py, in_image=inside, winner=winner, keep=keep)
