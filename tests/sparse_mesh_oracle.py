"""NumPy restatement of the sparse grid's definitions (include/glic_b200.h "Sparse meshing"): the allocation rule of one view in
float64, one rounding per operation in the order the header writes them, and the sparse grid as the dense restatement of
mesh_oracle.py restricted to the allocated blocks.  Written from the definitions, not from the kernels."""
import numpy as np

import mesh_oracle as mo

LAT = 1 << 19            # lattice indices in [-LAT, LAT)
BLK = LAT // 8


def block_key(bi, bj, bk):
    bi, bj, bk = (np.asarray(x, np.int64) for x in (bi, bj, bk))
    return ((bk + BLK) << 34) | ((bj + BLK) << 17) | (bi + BLK)


def key_blocks(keys):
    keys = np.asarray(keys, np.int64)
    return (keys & 0x1FFFF) - BLK, ((keys >> 17) & 0x1FFFF) - BLK, (keys >> 34) - BLK


def pixel_ranges(view, W, H, fx, fy, cx, cy, depth, mask, trunc, max_depth, origin, s):
    """per used pixel: (lattice lo [n,3], lattice hi [n,3], clipped [n]) after clipping to the lattice; empty ranges have lo > hi"""
    m = np.asarray(view, np.float32).astype(np.float64)
    R = [[m[4 * a + r] for a in range(3)] for r in range(3)]
    t = [m[12 + r] for r in range(3)]
    f64 = lambda v: np.float64(np.float32(v))
    fx, fy, cx, cy, trunc, s = (f64(v) for v in (fx, fy, cx, cy, trunc, s))
    o = np.asarray(origin, np.float32).astype(np.float64)
    d32 = np.asarray(depth, np.float32)
    with np.errstate(invalid="ignore"):
        used = (d32 > 0) & ((np.float32(max_depth) == 0) | (d32 <= np.float32(max_depth)))
    if mask is not None:
        used &= np.asarray(mask, bool)
    py, px = np.nonzero(used)
    d = d32[py, px].astype(np.float64)
    lo = np.full((d.size, 3), np.inf)
    hi = np.full((d.size, 3), -np.inf)
    finite = np.ones(d.size, bool)
    with np.errstate(all="ignore"):
        for q in range(8):
            u = (px + (q & 1)).astype(np.float64)
            v = (py + ((q >> 1) & 1)).astype(np.float64)
            z = d + trunc if q >> 2 else d
            c = (((u - cx) * z) / fx, ((v - cy) * z) / fy, z)
            for a in range(3):
                X = (R[0][a] * (c[0] - t[0]) + R[1][a] * (c[1] - t[1])) + R[2][a] * (c[2] - t[2])
                finite &= np.isfinite(X)
                lo[:, a] = np.minimum(lo[:, a], X)
                hi[:, a] = np.maximum(hi[:, a], X)
        L = np.floor((lo - o) / s) - 2
        Hh = np.ceil((hi - o) / s) + 2
    clipped = ~finite | (~(L >= -LAT)).any(1) | (~(Hh <= LAT - 1)).any(1)
    L = np.where(L >= -LAT, L, -LAT)
    Hh = np.where(Hh <= LAT - 1, Hh, LAT - 1)
    L[~finite] = 0
    Hh[~finite] = -1
    return L.astype(np.int64), Hh.astype(np.int64), clipped


def block_set(view, W, H, fx, fy, cx, cy, depth, mask=None, trunc=0.1, max_depth=0.0, origin=(0, 0, 0), s=0.05):
    """(sorted unique block keys int64, clipped pixel count) of one view"""
    L, Hh, clipped = pixel_ranges(view, W, H, fx, fy, cx, cy, depth, mask, trunc, max_depth, origin, s)
    keys = []
    for lo, hi in zip(L >> 3, Hh >> 3):
        if (hi < lo).any():
            continue
        bi, bj, bk = np.meshgrid(np.arange(lo[0], hi[0] + 1), np.arange(lo[1], hi[1] + 1), np.arange(lo[2], hi[2] + 1), indexing="ij")
        keys.append(block_key(bi.ravel(), bj.ravel(), bk.ravel()))
    keys = np.unique(np.concatenate(keys)) if keys else np.zeros(0, np.int64)
    return keys, int(clipped.sum())


def allocated(g, keys, shift=(0, 0, 0)):
    """bool [N]: the dense grid g's lattice points that lie in a block of keys; dense point (i, j, k) is sparse lattice point
    (i, j, k) + shift"""
    (i, j, k), _ = mo.lattice(g)
    return np.isin(block_key((i + shift[0]) >> 3, (j + shift[1]) >> 3, (k + shift[2]) >> 3), keys)


def restrict(g, keep):
    """a copy of the dense grid g with every point outside `keep` unobserved: the sparse grid's content on g's box"""
    r = dict(g)
    r["tsdf"] = np.where(keep, g["tsdf"], np.float32(0))
    r["weight"] = np.where(keep, g["weight"], np.float32(0))
    r["col"] = np.where(keep[None], g["col"], np.float32(0))
    return r


def negative_points(g, view, W, H, fx, fy, cx, cy, depth, mask, trunc, max_depth):
    """bool [N]: the lattice points of g's box that one view gives t < 0"""
    h = mo.new_grid(g["origin"], g["s"], g["dims"])
    ok = mo.integrate(h, view, W, H, fx, fy, cx, cy, depth, None, mask, trunc, max_depth)
    return ok & (h["tsdf"] < 0)


def dilate(flags, dims):
    """the +-1 (26-)neighbourhood of the set points of a flat [N] bool array over a box of dims, clipped to the box"""
    nx, ny, nz = dims
    a = flags.reshape(nz, ny, nx)
    out = a.copy()
    for dz in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                sh = np.zeros_like(a)
                src = a[max(dz, 0):nz + min(dz, 0), max(dy, 0):ny + min(dy, 0), max(dx, 0):nx + min(dx, 0)]
                sh[max(-dz, 0):nz + min(-dz, 0), max(-dy, 0):ny + min(-dy, 0), max(-dx, 0):nx + min(-dx, 0)] = src
                out |= sh
    return out.reshape(-1)
