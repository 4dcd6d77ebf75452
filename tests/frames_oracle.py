"""CPU restatement of Dataset::addFrame (gaussian.cpp:41-111) as glic_mapper_add_frame computes it (test infrastructure).

Every float64 operation is a single numpy scalar or element-wise operation, so each rounds once, as the reference's
Eigen code does on x86-64 without FMA.
"""
import numpy as np


def quat_rotation(q_wc):
    """Eigen::Quaterniond(w, x, y, z).toRotationMatrix() in Eigen's operation order, no normalisation; q = (x, y, z, w)."""
    x, y, z, w = (np.float64(v) for v in q_wc)
    tx, ty, tz = 2.0 * x, 2.0 * y, 2.0 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return np.array([[1.0 - (tyy + tzz), txy - twz, txz + twy],
                     [txy + twz, 1.0 - (txx + tzz), tyz - twx],
                     [txz - twy, tyz + twx, 1.0 - (txx + tyy)]], np.float64)


def depth_rsp64(q_wc, t_wc, xyz):
    """gaussian.cpp:66-70 in double: ((Rcw20 p0 + Rcw21 p1) + Rcw22 p2) + tcw2, R_cw = R^T, t_cw = -R_cw t_wc, p = (double)xyz."""
    R = quat_rotation(q_wc)
    t = np.asarray(t_wc, np.float64)
    tcw2 = -((R[0, 2] * t[0] + R[1, 2] * t[1]) + R[2, 2] * t[2])
    p = np.asarray(xyz, np.float32).astype(np.float64).reshape(-1, 3)
    return ((R[0, 2] * p[:, 0] + R[1, 2] * p[:, 1]) + R[2, 2] * p[:, 2]) + tcw2


def depth_rsp(q_wc, t_wc, xyz):
    """The stored depth: float of depth_rsp64."""
    return depth_rsp64(q_wc, t_wc, xyz).astype(np.float32)


def float_pose(q_wc, t_wc):
    """The keyframe's float pose: (float)R (row-major [3,3]) and (float)t."""
    return quat_rotation(q_wc).astype(np.float32), np.asarray(t_wc, np.float64).astype(np.float32)


def is_train(frame_index, k):
    """gaussian.cpp:75: the frame with all_frame_num_ == frame_index before it is a training keyframe."""
    return (frame_index + 1) % k == 0


DECODE = np.arange(256, dtype=np.float32) * np.float32(1.0 / 255.0)   # convertTo(CV_32F, 1.0f / 255.0f) of each byte value


def decode(bgr):
    """[H,W,3] BGR8 -> [3,H,W] float32 RGB: cvtColor(BGR2RGB) + convertTo(CV_32FC3, 1.0f / 255.0f) (gaussian.cpp:48-49)."""
    return np.ascontiguousarray(DECODE[np.asarray(bgr, np.uint8)[..., ::-1]].transpose(2, 0, 1))


def colours_init(rgb):
    """initialize()'s colours: the Dataset's doubles rgb / 255.0 (gaussian.cpp:65)."""
    return np.asarray(rgb, np.uint8).astype(np.float64) / 255.0


def colours_extend(rgb):
    """extend()'s colours: floats of those doubles (gaussian.cpp:517-519)."""
    return colours_init(rgb).astype(np.float32)
