"""CPU restatement of initialize() (/root/reference/src/gaussian.cpp:212-304) for the tests: the sky generator's uniforms bit
for bit, the LiDAR rows as the reference's host loop computes them (double arithmetic, glibc's log, stored as float), and the
sky formula (float32, numpy's trigonometry: within an ulp or two of the device's, not bit-equal).  TEST INFRASTRUCTURE ONLY."""
import math

import numpy as np

C0 = 0.28209479177387814                                   # gaussian.h:46


def sky_uniforms(n, seed):
    """[n,2] float32 (u1, u2) of rows 0..n-1: row i takes the i-th SplitMix64 output started at seed (include/glic_b200.h,
    glic_skybox_init), u1 = its top 24 bits * 2^-24, u2 = bits 16..39 * 2^-24."""
    z = np.uint64(int(seed) & (2 ** 64 - 1)) + (np.arange(int(n), dtype=np.uint64) + np.uint64(1)) * np.uint64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    z = z ^ (z >> np.uint64(31))
    u1 = (z >> np.uint64(40)).astype(np.float32) * np.float32(2.0 ** -24)
    u2 = ((z >> np.uint64(16)) & np.uint64(0xFFFFFF)).astype(np.float32) * np.float32(2.0 ** -24)
    return np.stack([u1, u2], 1)


def logit32(o):
    """inverse_sigmoid of a float32 opacity (general_utils.h:26-29): the ratio in float32, its log correctly rounded to float32
    (as the device's logf and torch's are for 0.1 and 0.7; numpy's float32 log is one ulp low at 0.7 / 0.3)"""
    o = np.float32(o)
    return np.float32(math.log(float(o / (np.float32(1.0) - o))))


def _rows(n):
    return dict(xyz=np.zeros((n, 3), np.float32), f_dc=np.zeros((n, 3), np.float32), log_scale=np.zeros((n, 3), np.float32),
                rot=np.tile(np.array([1, 0, 0, 0], np.float32), (n, 1)), opacity_logit=np.zeros(n, np.float32))


def lidar_init(points, colors, depth_rsp, scaling_scale, focal):
    """gaussian.cpp:214-240: xyz = point; f_dc = RGB2SH(colour) = (c - 0.5) / C0 in double (gaussian.h:46-47), colours being the
    Dataset's rgb / 255.0 doubles; log-scale = log(scaling_scale * d / f) in double on all three axes, f = (fx + fy) / 2;
    rotation (1, 0, 0, 0); opacity inverse_sigmoid(0.1f)."""
    p = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
    c = np.ascontiguousarray(colors, np.float64).reshape(-1, 3)
    d = np.ascontiguousarray(depth_rsp, np.float32).reshape(-1)
    out = _rows(p.shape[0])
    out["xyz"][:] = p
    out["f_dc"][:] = ((c - 0.5) / C0).astype(np.float32)
    ss, f = float(scaling_scale), float(focal)
    ls = np.array([math.log(ss * float(x) / f) for x in d], np.float64).astype(np.float32)
    out["log_scale"][:] = ls[:, None]
    out["opacity_logit"][:] = logit32(0.1)
    return out


def sky_init(n, radius, seed=None, uv=None):
    """gaussian.cpp:243-266 on uv (default sky_uniforms(n, seed)): theta = (2 pi) u1, phi = acos(1 - 1.4 u2),
    x = ((10 R) cos theta) sin phi, y likewise with sin theta, z = (10 R) cos phi; f_dc = (0.7, 0.8, 0.95) raw; log-scale =
    log(sqrt(max(d2, 1e-7))) with d2 the simple-knn mean over the sky points alone (brute force in float64: small n);
    rotation (1, 0, 0, 0); opacity inverse_sigmoid(0.7f)."""
    uv = sky_uniforms(n, seed) if uv is None else np.ascontiguousarray(uv, np.float32).reshape(-1, 2)
    n = uv.shape[0]
    out = _rows(n)
    f = np.float32
    r10, pi = f(float(radius) * 10.0), np.arccos(f(-1.0))
    theta = (f(2.0) * pi) * uv[:, 0]
    phi = np.arccos(f(1.0) - f(1.4) * uv[:, 1])
    out["xyz"][:, 0] = r10 * np.cos(theta) * np.sin(phi)
    out["xyz"][:, 1] = r10 * np.sin(theta) * np.sin(phi)
    out["xyz"][:, 2] = r10 * np.cos(phi)
    x = out["xyz"].astype(np.float64)
    d2 = np.full(n, np.inf)
    if n > 3:
        dd = ((x[:, None, :] - x[None, :, :]) ** 2).sum(-1)
        np.fill_diagonal(dd, np.inf)
        d2 = np.sort(dd, 1)[:, :3].mean(1)
    out["log_scale"][:] = np.log(np.sqrt(np.maximum(d2, 1e-7))).astype(np.float32)[:, None]
    out["f_dc"][:] = np.array([0.7, 0.8, 0.95], np.float32)
    out["opacity_logit"][:] = logit32(0.7)
    out["uv"] = uv
    return out
