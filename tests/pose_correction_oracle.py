"""NumPy float64 restatement of glic_mapper_correct_poses (include/glic_b200.h, "Pose corrections").

record_rt / record_q restate the record's R, t and q operation for operation (NumPy's float64 ops round once, as the host code
does); sh_fit builds the SH band rotation matrices independently, by a least-squares fit on random directions of the sh_basis
polynomials restated here; apply_rows restates the row kernel's update on a mapper download.
"""
import numpy as np

# sh_math.cuh's constants, at the float64 values its floats round
B1 = 0.4886025119029199
B2 = (1.0925484305920792, 0.31539156525252005, 0.5462742152960396)
B3 = (0.5900435899266435, 2.890611442640554, 0.4570457994644658, 0.3731763325901154, 1.445305721320277)
OFFSET = {1: 0, 2: 9, 3: 34}


def band_basis(l, d):
    """[N, 2l+1] basis values of band l at unit directions d [N, 3] (sh_basis's polynomials and order)"""
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    if l == 1:
        return np.stack([-B1 * y, B1 * z, -B1 * x], 1)
    xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
    if l == 2:
        a, b, c = B2
        return np.stack([a * xy, -a * yz, b * (2 * zz - xx - yy), -a * xz, c * (xx - yy)], 1)
    a, b, c, e, f = B3
    return np.stack([-a * y * (3 * xx - yy), b * xy * z, -c * y * (4 * zz - xx - yy), e * z * (2 * zz - 3 * xx - 3 * yy),
                     -c * x * (4 * zz - xx - yy), f * z * (xx - yy), -a * x * (xx - 3 * yy)], 1)


def quat_matrix(q):
    """R(q) of sh_math.cuh for q = (r, x, y, z)"""
    r, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)],
                     [2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)],
                     [2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)]])


def quat_mul(a, b):
    """Hamilton product a (x) b, (r, x, y, z)"""
    r1, x1, y1, z1 = a
    r2, x2, y2, z2 = b
    return np.array([r1 * r2 - x1 * x2 - y1 * y2 - z1 * z2, r1 * x2 + x1 * r2 + y1 * z2 - z1 * y2,
                     r1 * y2 - x1 * z2 + y1 * r2 + z1 * x2, r1 * z2 + x1 * y2 - y1 * x2 + z1 * r2])


def record_rt(R_old, t_old, R_new, t_new):
    """the record's R (dR = R_new R_old^T) and t (t_new - dR t_old), in the header's order, from float32 poses"""
    Ro, Rn = np.asarray(R_old, np.float32).reshape(9).astype(np.float64), np.asarray(R_new, np.float32).reshape(9).astype(np.float64)
    to, tn = np.asarray(t_old, np.float32).astype(np.float64), np.asarray(t_new, np.float32).astype(np.float64)
    R = np.zeros(9)
    for i in range(3):
        for j in range(3):
            R[3 * i + j] = (Rn[3 * i] * Ro[3 * j] + Rn[3 * i + 1] * Ro[3 * j + 1]) + Rn[3 * i + 2] * Ro[3 * j + 2]
    t = np.array([tn[i] - ((R[3 * i] * to[0] + R[3 * i + 1] * to[1]) + R[3 * i + 2] * to[2]) for i in range(3)])
    return R, t


def record_q(R):
    """the header's branch-by-largest-diagonal unit quaternion of R [9], with its sign rule"""
    R = [np.float64(v) for v in np.asarray(R, np.float64).reshape(9)]
    tr = (R[0] + R[4]) + R[8]
    branch, best = 0, tr
    for b in range(1, 4):
        if R[4 * (b - 1)] > best:
            best, branch = R[4 * (b - 1)], b
    if branch == 0:
        r = 0.5 * np.sqrt(1.0 + tr); s = 0.25 / r
        x, y, z = (R[7] - R[5]) * s, (R[2] - R[6]) * s, (R[3] - R[1]) * s
    elif branch == 1:
        x = 0.5 * np.sqrt(((1.0 + R[0]) - R[4]) - R[8]); s = 0.25 / x
        r, y, z = (R[7] - R[5]) * s, (R[1] + R[3]) * s, (R[2] + R[6]) * s
    elif branch == 2:
        y = 0.5 * np.sqrt(((1.0 - R[0]) + R[4]) - R[8]); s = 0.25 / y
        r, x, z = (R[2] - R[6]) * s, (R[1] + R[3]) * s, (R[5] + R[7]) * s
    else:
        z = 0.5 * np.sqrt(((1.0 - R[0]) - R[4]) + R[8]); s = 0.25 / z
        r, x, y = (R[3] - R[1]) * s, (R[2] + R[6]) * s, (R[5] + R[7]) * s
    n = np.sqrt(((r * r + x * x) + y * y) + z * z)
    q = np.array([r / n, x / n, y / n, z / n])
    lead = next((v for v in q[1:] if v != 0.0), 0.0)
    if q[0] < 0.0 or (q[0] == 0.0 and lead < 0.0):
        q = -q
    q[0] = q[0] + 0.0
    return q


def sh_fit(q, degree, n_dirs=400, seed=0):
    """the band matrices of R(q) by least squares: sum_m A[m][n] b_m(d) = b_n(R(q)^T d) on random unit directions"""
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(n_dirs, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    e = d @ quat_matrix(q)                                   # rows (R^T d_i)^T = d_i^T R
    return [np.linalg.lstsq(band_basis(l, d), band_basis(l, e), rcond=None)[0] for l in range(1, degree + 1)]


def apply_rows(g, anchor, records, degree):
    """the row kernel on a download g (means, rots, sh [P,M,3], ...): rows whose anchor has a record (dict keyframe -> record of
    gaussian_lic_b200.mapper.pose_correction_record) move; returns (new download, moved rows mask)"""
    out = {k: np.array(v, copy=True) for k, v in g.items()}
    anchor = np.asarray(anchor)
    moved = np.zeros(anchor.shape[0], bool)
    for k, rec in records.items():
        sel = anchor == k
        moved |= sel
        if not sel.any():
            continue
        R, t, q = rec["R"].reshape(9), rec["t"], rec["q"]
        p = g["means"][sel].astype(np.float64)
        out["means"][sel] = np.stack([((R[3 * i] * p[:, 0] + R[3 * i + 1] * p[:, 1]) + R[3 * i + 2] * p[:, 2]) + t[i]
                                      for i in range(3)], 1).astype(np.float32)
        o = g["rots"][sel].astype(np.float64)
        rr, rx, ry, rz = o[:, 0], o[:, 1], o[:, 2], o[:, 3]
        qr, qx, qy, qz = q
        out["rots"][sel] = np.stack([((qr * rr - qx * rx) - qy * ry) - qz * rz, ((qr * rx + qx * rr) + qy * rz) - qz * ry,
                                     ((qr * ry - qx * rz) + qy * rr) + qz * rx, ((qr * rz + qx * ry) - qy * rx) + qz * rr],
                                    1).astype(np.float32)
        sh = g["sh"][sel].astype(np.float64)                 # [n, M, 3]
        new = sh.copy()
        for l in range(1, degree + 1):
            A, k0, n = rec["sh"][l - 1], l * l - 1, 2 * l + 1
            for m in range(n):
                acc = A[m, 0] * sh[:, k0]
                for j in range(1, n):
                    acc = acc + A[m, j] * sh[:, k0 + j]
                new[:, k0 + m] = acc
        out["sh"][sel] = new.astype(np.float32)
    return out, moved
