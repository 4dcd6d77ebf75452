"""NumPy restatement of glic_mapper_densify (include/glic_b200.h "Densification") -- test infrastructure.

select() gives the classes and the result rows' sources, rows() the expected parameters and moments except the children's
xyz, split_xyz() the children's xyz from their normals, normals() the generator in float64 (its uniforms exactly).
Every float32 step is one NumPy float32 operation, rounded once like the device's _rn intrinsics.
"""
import numpy as np

MASK = (1 << 64) - 1
GOLDEN = 0x9E3779B97F4A7C15
SPLIT_LOG_SCALE = np.float32(np.log(1.6))


def mix64(z):
    """the SplitMix64 finaliser on uint64 arrays (wrapping arithmetic)"""
    z = np.asarray(z, np.uint64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def mix64_int(z):
    """the same on one Python int (the restatement's own check)"""
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9 & MASK
    z = (z ^ (z >> 27)) * 0x94D049BB133111EB & MASK
    return z ^ (z >> 31)


def uniforms(seed, call, rows):
    """u1, u2 [n, 3] (float32, exact multiples of 2^-24) of the children at result rows `rows`"""
    rows = np.asarray(rows, np.uint64).reshape(-1, 1)
    a = np.arange(3, dtype=np.uint64).reshape(1, 3)
    with np.errstate(over="ignore"):
        k = ((np.uint64(call + 1) << np.uint64(32)) + rows) * np.uint64(3) + a
        r = mix64(np.uint64(seed) + (k + np.uint64(1)) * np.uint64(GOLDEN))
    u1 = (r >> np.uint64(40)).astype(np.float32) * np.float32(2.0 ** -24)
    u2 = ((r >> np.uint64(16)) & np.uint64(0xFFFFFF)).astype(np.float32) * np.float32(2.0 ** -24)
    return u1, u2


def normals(seed, call, rows):
    """Box-Muller of the uniforms in float64: what the device's float32 evaluation approximates"""
    u1, u2 = uniforms(seed, call, rows)
    return np.sqrt(-2.0 * np.log(1.0 - u1.astype(np.float64))) * np.cos(2.0 * np.pi * u2.astype(np.float64))


def build_rotation(q):
    """Inria's build_rotation of normalised q = (r, x, y, z), in the header's float32 operation order -> [n, 3, 3]"""
    q = np.asarray(q, np.float32)
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    one, two = np.float32(1.0), np.float32(2.0)
    R = np.empty((q.shape[0], 3, 3), np.float32)
    R[:, 0, 0] = one - two * (y * y + z * z)
    R[:, 0, 1] = two * (x * y - r * z)
    R[:, 0, 2] = two * (x * z + r * y)
    R[:, 1, 0] = two * (x * y + r * z)
    R[:, 1, 1] = one - two * (x * x + z * z)
    R[:, 1, 2] = two * (y * z - r * x)
    R[:, 2, 0] = two * (x * z - r * y)
    R[:, 2, 1] = two * (y * z + r * x)
    R[:, 2, 2] = one - two * (x * x + y * y)
    return R


def split_xyz(p, s, q, z):
    """p + R(q) (s * z), each product and sum rounded once, in the header's order"""
    p, s, z = (np.asarray(a, np.float32) for a in (p, s, z))
    R = build_rotation(q)
    v = s * z
    out = np.empty_like(p)
    for i in range(3):
        out[:, i] = p[:, i] + ((R[:, i, 0] * v[:, 0] + R[:, i, 1] * v[:, 1]) + R[:, i, 2] * v[:, 2])
    return out


def classes(accum, denom, smax, n_sky, grad_threshold, percent_dense, scene_extent):
    """0 keep, 1 clone, 2 split per row; smax = the largest activated scale (expf on the device: pass the device's values)"""
    accum, denom, smax = (np.asarray(a, np.float32) for a in (accum, denom, smax))
    with np.errstate(divide="ignore", invalid="ignore"):
        grad = np.where(denom > 0, accum / np.where(denom > 0, denom, np.float32(1)), np.float32(0)).astype(np.float32)
    sel = grad >= np.float32(grad_threshold)
    sel[:n_sky] = False
    clone_max = np.float32(percent_dense) * np.float32(scene_extent)
    cls = np.zeros(accum.shape[0], np.int64)
    cls[sel & (smax <= clone_max)] = 1
    cls[sel & ~(smax <= clone_max)] = 2
    return cls


def select(cls):
    """source row of every result row, and the counts: kept rows (not split), clones, first children, second children"""
    P = cls.shape[0]
    kept, clones, splits = np.nonzero(cls != 2)[0], np.nonzero(cls == 1)[0], np.nonzero(cls == 2)[0]
    src = np.concatenate([kept, clones, splits, splits])
    return src, dict(kept=kept.size, cloned=clones.size, split=splits.size, total=P + clones.size + splits.size)
