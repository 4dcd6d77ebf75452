"""NumPy float32 restatement of the meshing definitions (include/glic_b200.h "Meshing"): TSDF integration of one view and naive
surface-nets extraction.  numpy's float32 operations round once each, as the kernels' _rn intrinsics do; the one fused operation
of the definitions (xform_row's fma) is restated exactly through a float64 sum rounded to odd.  Written from the definitions, not
from the kernels, so that a match bit for bit checks both."""
import numpy as np

f32 = np.float32
# corner A (a + 2 b + 4 c) of each of a cell's 12 edges, in the fixed edge order; edge e's other end is A + (1 << (e // 4))
EDGE_A = (0, 2, 4, 6, 0, 1, 4, 5, 0, 1, 2, 3)


def fma32(a, b, c):
    """Correctly rounded float32 fma(a, b, c): a b is exact in float64, the sum is rounded to odd in float64 (a TwoSum gives the
    sign of what was lost), and a float64 value rounded to odd rounds to float32 as the exact value would (53 >= 24 + 2)."""
    a, b, c = (np.asarray(v, np.float32).astype(np.float64) for v in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    odd = (s.view(np.int64) & 1) == 1
    fix = np.isfinite(s) & (e != 0) & ~odd
    s = np.where(fix, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


def new_grid(origin, voxel_size, dims):
    """a cleared grid: dict of flat float32 planes tsdf [N], weight [N], col [3,N] and its geometry"""
    nx, ny, nz = (int(d) for d in dims)
    N = nx * ny * nz
    return dict(origin=np.asarray(origin, np.float32).reshape(3), s=f32(voxel_size), dims=(nx, ny, nz),
                tsdf=np.zeros(N, np.float32), weight=np.zeros(N, np.float32), col=np.zeros((3, N), np.float32))


def lattice(g):
    """(i, j, k) int arrays and world positions (X, Y, Z) float32 of every lattice point, in index order"""
    nx, ny, nz = g["dims"]
    L = np.arange(nx * ny * nz, dtype=np.int64)
    ijk = (L % nx, (L // nx) % ny, L // (nx * ny))
    pos = tuple(g["origin"][a] + g["s"] * ijk[a].astype(np.float32) for a in range(3))
    return ijk, pos


def view_of(R_cw, t_cw):
    """the 16 column-major floats of the world -> camera matrix [R_cw | t_cw]"""
    Rt = np.eye(4, dtype=np.float32)
    Rt[:3, :3] = np.asarray(R_cw, np.float32)
    Rt[:3, 3] = np.asarray(t_cw, np.float32).reshape(3)
    return np.ascontiguousarray(Rt.T).reshape(16)


def integrate(g, view, W, H, fx, fy, cx, cy, depth, rgb=None, mask=None, trunc=0.1, max_depth=0.0):
    """glic_tsdf_integrate in place on g; view: 16 column-major float32; depth [H,W]; rgb [3,H,W] or None; mask [H,W] bool
    (True = used) or None.  Returns the bool array of updated points."""
    m = np.asarray(view, np.float32).reshape(16)
    _, (X, Y, Z) = lattice(g)
    fx, fy, cx, cy, trunc, max_depth = (f32(v) for v in (fx, fy, cx, cy, trunc, max_depth))

    def row(r):
        return m[12 + r] + fma32(Z, m[8 + r], fma32(X, m[r], Y * m[4 + r]))

    x, y, z = row(0), row(1), row(2)
    with np.errstate(all="ignore"):
        ok = z > 0
        u = fx * (x / z) + cx
        v = fy * (y / z) + cy
        ok &= (u >= 0) & (u < f32(W)) & (v >= 0) & (v < f32(H))
        px = np.where(ok, np.floor(np.where(ok, u, 0)), 0).astype(np.int64)
        py = np.where(ok, np.floor(np.where(ok, v, 0)), 0).astype(np.int64)
        if mask is not None:
            ok &= np.asarray(mask, bool)[py, px]
        d = np.asarray(depth, np.float32)[py, px]
        ok &= (d > 0) & ((max_depth == 0) | (d <= max_depth))
        sdf = d - z
        ok &= sdf >= -trunc
        t = np.fmin(f32(1), sdf / trunc)
    w = g["weight"][ok]
    w1 = w + f32(1)
    g["tsdf"][ok] = (g["tsdf"][ok] * w + t[ok]) / w1
    if rgb is not None:
        c = np.asarray(rgb, np.float32)[:, py[ok], px[ok]]
        g["col"][:, ok] = (g["col"][:, ok] * w + c) / w1
    g["weight"][ok] = w1
    return ok


def active_cells(g):
    """bool [N]: the cell with lower corner L exists and is active"""
    nx, ny, nz = g["dims"]
    t = g["tsdf"].reshape(nz, ny, nx)
    w = g["weight"].reshape(nz, ny, nx)
    allobs = np.ones((nz - 1, ny - 1, nx - 1), bool)
    nin = np.zeros((nz - 1, ny - 1, nx - 1), np.int32)
    for q in range(8):
        a, b, c = q & 1, (q >> 1) & 1, q >> 2
        sl = (slice(c, nz - 1 + c), slice(b, ny - 1 + b), slice(a, nx - 1 + a))
        allobs &= w[sl] > 0
        nin += t[sl] < 0
    act = np.zeros((nz, ny, nx), bool)
    act[:-1, :-1, :-1] = allobs & (nin > 0) & (nin < 8)
    return act.reshape(-1)


def extract(g):
    """Naive surface nets of g -> (xyz [V,3] float32, rgb [V,3] uint8, faces [F,3] int32)"""
    nx, ny, nz = g["dims"]
    N = nx * ny * nz
    tsdf, weight, col = g["tsdf"], g["weight"], g["col"]
    act = active_cells(g)
    cells = np.flatnonzero(act)
    V = cells.size
    vid = np.full(N, -1, np.int64)
    vid[cells] = np.arange(V)
    st = (1, nx, nx * ny)
    corner = [cells + (q & 1) * st[0] + ((q >> 1) & 1) * st[1] + (q >> 2) * st[2] for q in range(8)]
    sp = np.zeros((3, V), np.float32)
    sc = np.zeros((3, V), np.float32)
    n = np.zeros(V, np.int32)
    with np.errstate(all="ignore"):
        for e in range(12):
            ax, A = e >> 2, EDGE_A[e]
            B = A + (1 << ax)
            tA, tB = tsdf[corner[A]], tsdf[corner[B]]
            cr = (tA < 0) != (tB < 0)
            f = tA / (tA - tB)
            p = [np.full(V, f32(A & 1)), np.full(V, f32((A >> 1) & 1)), np.full(V, f32(A >> 2))]
            p[ax] = f
            for a in range(3):
                cA, cB = col[a][corner[A]], col[a][corner[B]]
                cc = cA + f * (cB - cA)
                sp[a] = np.where(cr, np.where(n == 0, p[a], sp[a] + p[a]), sp[a])
                sc[a] = np.where(cr, np.where(n == 0, cc, sc[a] + cc), sc[a])
            n += cr
        fn = n.astype(np.float32)
        ijk = (cells % nx, (cells // nx) % ny, cells // (nx * ny))
        xyz = np.stack([g["origin"][a] + g["s"] * (ijk[a].astype(np.float32) + sp[a] / fn) for a in range(3)], axis=1)
        c = np.fmin(np.fmax(sc / fn, f32(0)), f32(1))
        rgb = np.rint(c * f32(255)).astype(np.uint8).T.copy()
    # faces: every lattice edge of axis a from L whose two ends are observed, exactly one inside, and whose four cells are active
    L = np.arange(N, dtype=np.int64)
    lijk = (L % nx, (L // nx) % ny, L // (nx * ny))
    dims = (nx, ny, nz)
    keys, quads, inside = [], [], []
    for a in range(3):
        b, c_ = (a + 1) % 3, (a + 2) % 3
        ok = (lijk[a] < dims[a] - 1) & (lijk[b] >= 1) & (lijk[c_] >= 1)
        Ls = L[ok]
        Bs = Ls + st[a]
        ok2 = (weight[Ls] > 0) & (weight[Bs] > 0) & ((tsdf[Ls] < 0) != (tsdf[Bs] < 0))
        Ls = Ls[ok2]
        q = np.stack([Ls - st[b] - st[c_], Ls - st[c_], Ls, Ls - st[b]], axis=1)
        ok3 = act[q].all(axis=1)
        Ls, q = Ls[ok3], q[ok3]
        keys.append(3 * Ls + a)
        quads.append(vid[q])
        inside.append(tsdf[Ls] < 0)
    keys, quads, inside = np.concatenate(keys), np.concatenate(quads), np.concatenate(inside)
    order = np.argsort(keys, kind="stable")
    quads, inside = quads[order], inside[order]
    quads = np.where(inside[:, None], quads, quads[:, ::-1])
    faces = np.empty((2 * quads.shape[0], 3), np.int32)
    faces[0::2] = quads[:, [0, 1, 2]]
    faces[1::2] = quads[:, [0, 2, 3]]
    return xyz, rgb, faces


# ---- geometry of a mesh ---------------------------------------------------------------------------------------------------
def edge_counts(faces):
    """(undirected edge -> number of faces, directed edge -> number of faces) as count arrays over unique edges"""
    d = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]]).astype(np.int64)
    _, dir_counts = np.unique(d, axis=0, return_counts=True)
    _, und_counts = np.unique(np.sort(d, axis=1), axis=0, return_counts=True)
    return und_counts, dir_counts


def euler_characteristic(xyz, faces):
    und, _ = edge_counts(faces)
    used = np.unique(faces).size
    return used - und.size + faces.shape[0]


def signed_volume(xyz, faces):
    p = xyz.astype(np.float64)[faces]
    return float(np.einsum("ij,ij->i", p[:, 0], np.cross(p[:, 1], p[:, 2])).sum() / 6.0)


# ---- analytic depth maps ------------------------------------------------------------------------------------------------------
def look_at(pos, target, up=(0.0, -1.0, 0.0)):
    """R_cw, t_cw (float64) of a camera at pos looking at target (z forward, y down)"""
    pos, target = np.asarray(pos, np.float64), np.asarray(target, np.float64)
    fwd = target - pos
    fwd /= np.linalg.norm(fwd)
    right = np.cross(fwd, np.asarray(up, np.float64))
    if np.linalg.norm(right) < 1e-9:
        right = np.cross(fwd, np.array([1.0, 0.0, 0.0]))
    right /= np.linalg.norm(right)
    down = np.cross(fwd, right)
    R_cw = np.stack([right, down, fwd])
    return R_cw, -R_cw @ pos


def sphere_depth(R_cw, t_cw, W, H, fx, fy, cx, cy, centre, radius):
    """z-depth [H,W] float32 of a sphere along the ray through each pixel centre u = px + 0.5 (float64, 0 where the ray misses)"""
    C = np.asarray(R_cw, np.float64) @ np.asarray(centre, np.float64) + np.asarray(t_cw, np.float64)
    u = (np.arange(W) + 0.5 - cx) / fx
    v = (np.arange(H) + 0.5 - cy) / fy
    dx, dy = np.meshgrid(u, v)
    dd = dx * dx + dy * dy + 1.0
    b = dx * C[0] + dy * C[1] + C[2]
    disc = b * b - dd * (C @ C - radius * radius)
    s = (b - np.sqrt(np.maximum(disc, 0.0))) / dd
    return np.where((disc > 0) & (s > 0), s, 0.0).astype(np.float32)
