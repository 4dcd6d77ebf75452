"""CPU restatement of the native mapper's pose refinement (glic_mapper_enable_pose_refinement) in float64, on top of an
oracle.Oracle's forward and backward.  Test infrastructure only.

Spec (include/glic_b200.h, csrc/preprocess_backward.cu):
  T_cw = [R_cw | t_cw], R_cw = R_wc^T, t_cw = -R_wc^T t_wc;  T_cw(delta) = Exp(delta) T_cw, delta = (rho, omega) in the camera
  frame, translation first;  g = dL/ddelta at delta = 0.  With W = R_cw (the rotation block of the view), per visible Gaussian i
      g_view,i = dL/dp_view through J + W * (the projection adjoint),  G_i = J_i^T dL/dT_i,  d_i = the SH-direction adjoint,
      dL/drho = sum_i g_view,i + W d_i,   dL/domega = sum_i p_view,i x g_view,i + sum_c W[:,c] x G_i[:,c].
  Only the projection and EWA adjoints are restated here; d_i falls out of the oracle's own dL_dmeans3D = W^T g_view,i + d_i.
  Adam: exposure_adam_kernel's float32 arithmetic (betas 0.9 / 0.999, eps 1e-8, bias correction from the keyframe's step count)
  with lr_translation on rho and lr_rotation on omega; then T_cw <- Exp(u) T_cw in float64 and the float pose re-derived."""
import numpy as np

from exposure_oracle import _fma


# ---- SE(3) --------------------------------------------------------------------------------------------------------------
def hat(w):
    return np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])


def se3_exp(u):
    """4x4 float64 Exp(u), u = (rho, omega): the Taylor series below theta = 1e-2, as the kernel evaluates it"""
    u = np.asarray(u, np.float64)
    w = u[3:]
    th2 = float(w @ w)
    if th2 < 1e-4:
        A = 1.0 - th2 / 6.0 * (1.0 - th2 / 20.0 * (1.0 - th2 / 42.0))
        B = 0.5 * (1.0 - th2 / 12.0 * (1.0 - th2 / 30.0 * (1.0 - th2 / 56.0)))
        C = (1.0 / 6.0) * (1.0 - th2 / 20.0 * (1.0 - th2 / 42.0 * (1.0 - th2 / 72.0)))
    else:
        th = np.sqrt(th2)
        A, B, C = np.sin(th) / th, 2.0 * np.sin(0.5 * th) ** 2 / th2, (th - np.sin(th)) / (th2 * th)
    K = hat(w)
    K2 = K @ K
    T = np.eye(4)
    T[:3, :3] = np.eye(3) + A * K + B * K2
    T[:3, 3] = (np.eye(3) + B * K + C * K2) @ u[:3]
    return T


def T_cw_of(R_wc, t_wc):
    """float64 T_cw of a float pose, as the mapper initialises its master pose"""
    R = np.asarray(R_wc, np.float32).astype(np.float64).reshape(3, 3)
    t = np.asarray(t_wc, np.float32).astype(np.float64).reshape(3)
    T = np.eye(4)
    T[:3, :3] = R.T
    T[:3, 3] = -(R.T @ t)
    return T


def float_pose(T):
    """(R_wc, t_wc) float32 re-derived from a float64 T_cw"""
    R, t = T[:3, :3], T[:3, 3]
    return R.T.astype(np.float32), (-(R.T @ t)).astype(np.float32)


# ---- cameras in float64 ---------------------------------------------------------------------------------------------------
def camera64(o, W, H, fx, fy, cx, cy, T):
    """the camera block of pose T_cw with its pose-dependent part (view, proj, campos) in float64; the projection P and the
    FoV / clamp limits are the oracle's (they do not depend on the pose)"""
    base = o.camera(W, H, fx, fy, cx, cy)                          # identity pose: proj = P
    Pm = np.asarray(base["proj"], np.float64).reshape(4, 4).T      # column-major -> row-major
    Rt = np.eye(4)
    Rt[:3, :] = T[:3, :]
    cam = dict(base)
    cam["view"] = Rt.T.reshape(16).copy()                          # column-major
    cam["proj"] = (Pm @ Rt).T.reshape(16).copy()
    cam["campos"] = -(T[:3, :3].T @ T[:3, 3])
    return cam


# ---- the gradient ---------------------------------------------------------------------------------------------------------
def _cov3d(scales, rots):
    q = np.asarray(rots, np.float64)
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)], -1),
                  np.stack([2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)], -1),
                  np.stack([2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1)], 1)
    s2 = np.asarray(scales, np.float64) ** 2
    return np.einsum("pij,pj,pkj->pik", R, s2, R)


def pose_gradient(g, cam, fwd, bwd, parts=False, rows=None, magnitude=False):
    """dL/d(rho, omega) [6] float64 of one view, from the oracle's forward (radii) and backward (dL_dmeans2D, dL_dconic,
    dL_dmeans3D).  g: the activated Gaussians handed to Oracle.forward.  parts=True also returns the translation identity's
    right-hand side W * sum_i dL_dmeans3D_i.  rows: sum only over these Gaussians (indices; default all), e.g. the sky rows
    alone.  magnitude=True returns [2, 6] instead: the gradient and sum_i |term_i| over its per-Gaussian terms, the scale of
    the rounding error of a float32 evaluation of each term."""
    vis = np.flatnonzero(np.asarray(fwd["radii"])[:int(np.asarray(g["means"]).shape[0])] > 0)
    if rows is not None:
        vis = np.intersect1d(vis, np.asarray(rows))
    view = np.asarray(cam["view"], np.float64).reshape(4, 4).T       # row-major Rt
    Wm, tv = view[:3, :3], view[:3, 3]
    pr = np.asarray(cam["proj"], np.float64)                         # column-major
    W_, H_ = cam["W"], cam["H"]
    fx = W_ / (2.0 * np.float64(np.float32(cam["tanfovx"])))
    fy = H_ / (2.0 * np.float64(np.float32(cam["tanfovy"])))
    lim = np.asarray(cam["lims"], np.float64)
    p = np.asarray(g["means"], np.float64)[vis]
    Sig = _cov3d(np.asarray(g["scales"], np.float64)[vis], np.asarray(g["rots"], np.float64)[vis])
    g2 = np.asarray(bwd["dL_dmeans2D"], np.float64).reshape(-1, 3)[vis]
    gc = np.asarray(bwd["dL_dconic"], np.float64).reshape(-1, 4)[vis]
    dm3 = np.asarray(bwd["dL_dmeans3D"], np.float64).reshape(-1, 3)[vis]
    pv = p @ Wm.T + tv
    tz = pv[:, 2]
    txtz, tytz = pv[:, 0] / tz, pv[:, 1] / tz
    lx, ly = np.clip(txtz, lim[0], lim[1]), np.clip(tytz, lim[2], lim[3])
    xm = ((txtz >= lim[0]) & (txtz <= lim[1])).astype(np.float64)
    ym = ((tytz >= lim[2]) & (tytz <= lim[3])).astype(np.float64)
    n = vis.size
    J = np.zeros((n, 2, 3))
    J[:, 0, 0], J[:, 0, 2] = fx / tz, -fx * lx / tz
    J[:, 1, 1], J[:, 1, 2] = fy / tz, -fy * ly / tz
    T = J @ Wm                                                       # [n,2,3]
    cov = T @ Sig @ T.transpose(0, 2, 1)
    a, b, c = cov[:, 0, 0] + 0.3, cov[:, 0, 1], cov[:, 1, 1] + 0.3
    gxx, gxy, gyy = gc[:, 0], gc[:, 1], gc[:, 3]
    denom = a * c - b * b
    d2 = 1.0 / (denom * denom + 1e-7)
    dLa = d2 * (-c * c * gxx + 2 * b * c * gxy + (denom - a * c) * gyy)
    dLc = d2 * (-a * a * gyy + 2 * a * b * gxy + (denom - a * c) * gxx)
    dLb = d2 * 2 * (b * c * gxx - (denom + 2 * b * b) * gxy + a * b * gyy)
    r = T @ Sig                                                      # r[i][m] = sum_k T_ik Sigma_km
    dT = np.stack([2 * r[:, 0] * dLa[:, None] + r[:, 1] * dLb[:, None], 2 * r[:, 1] * dLc[:, None] + r[:, 0] * dLb[:, None]], 1)
    dJ = dT @ Wm.T                                                   # dJ[i][k] = sum_m dT[i][m] W[k][m]
    tcx, tcy = lx * tz, ly * tz
    dt = np.stack([xm * -fx / tz ** 2 * dJ[:, 0, 2], ym * -fy / tz ** 2 * dJ[:, 1, 2],
                   -fx / tz ** 2 * dJ[:, 0, 0] - fy / tz ** 2 * dJ[:, 1, 1] + 2 * fx * tcx / tz ** 3 * dJ[:, 0, 2]
                   + 2 * fy * tcy / tz ** 3 * dJ[:, 1, 2]], 1)
    hx = p @ pr[[0, 4, 8]] + pr[12]
    hy = p @ pr[[1, 5, 9]] + pr[13]
    hw = p @ pr[[3, 7, 11]] + pr[15]
    mw = 1.0 / (hw + 1e-7)
    m1, m2 = hx * mw * mw, hy * mw * mw
    pj = np.stack([(pr[0] * mw - pr[3] * m1) * g2[:, 0] + (pr[1] * mw - pr[3] * m2) * g2[:, 1],
                   (pr[4] * mw - pr[7] * m1) * g2[:, 0] + (pr[5] * mw - pr[7] * m2) * g2[:, 1],
                   (pr[8] * mw - pr[11] * m1) * g2[:, 0] + (pr[9] * mw - pr[11] * m2) * g2[:, 1]], 1)
    gview = dt + pj @ Wm.T
    d = dm3 - gview @ Wm                                             # the SH-direction adjoint (world frame)
    G = J.transpose(0, 2, 1) @ dT                                    # dL/dW through T = J W
    rho = gview.sum(0) + Wm @ d.sum(0)
    omega = np.cross(pv, gview).sum(0) + np.cross(np.broadcast_to(Wm.T[None], G.shape), G.transpose(0, 2, 1)).sum((0, 1))
    out = np.concatenate([rho, omega])
    if magnitude:
        terms = np.concatenate([gview + d @ Wm.T, np.cross(pv, gview)
                                + np.cross(np.broadcast_to(Wm.T[None], G.shape), G.transpose(0, 2, 1)).sum(1)], 1)
        return np.stack([out, np.abs(terms).sum(0)])
    if parts:
        return out, Wm @ dm3.sum(0)
    return out


def view_loss_and_grad(o, g, cam, gt, lambda_dssim=0.2):
    """(L, dL/d(rho, omega)) of one view's L1 + D-SSIM loss, by the oracle's forward and backward"""
    f = o.forward(g, cam)
    L, dpix = o.loss(f["color"], gt, lambda_dssim)
    b = o.backward(f, dpix)
    gr = pose_gradient(g, cam, f, b)
    o.free(f)
    return L, gr


# ---- Adam + composition ---------------------------------------------------------------------------------------------------
def pose_adam(m, v, step, grad, lr_t, lr_r):
    """the kernel's float32 Adam on the 6-vector -> (update u [6] float32, m, v, step)"""
    dt = np.float32
    m, v, g = (np.asarray(x, dt) for x in (m, v, grad))
    t = int(step) + 1
    bc1, bc2 = 1.0 - 0.9 ** t, 1.0 - 0.999 ** t
    b1, b2, eps = dt(0.9), dt(0.999), dt(1e-8)
    m1 = _fma(g, dt(1.0) - b1, b1 * m, dt)
    v1 = _fma(g * g, dt(1.0) - b2, b2 * v, dt)
    denom = np.sqrt(v1) / dt(np.sqrt(bc2)) + eps
    lr = np.array([lr_t] * 3 + [lr_r] * 3, np.float32)
    step_size = np.array([dt(float(x) / bc1) for x in lr], dt)
    return ((-step_size) * (m1 / denom)).astype(dt), m1, v1, t


def pose_step(T, m, v, step, grad, lr_t, lr_r):
    """one pose step -> (T_cw float64, m, v, step); an all-zero update leaves T as it is"""
    u, m1, v1, t = pose_adam(m, v, step, grad, lr_t, lr_r)
    if not np.any(u != 0):
        return T.copy(), m1, v1, t
    return se3_exp(u.astype(np.float64)) @ T, m1, v1, t
