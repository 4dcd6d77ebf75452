"""Float64 restatement of the inference blend's two depth planes (glic_render) on the GPU's own sorted lists and splat records.

Per pixel, front to back over its tile's list: power = -0.5 (cx dx^2 + cz dy^2) - cy dx dy, alpha = min(0.99, o exp(power)); a
splat is taken when power <= 0, alpha >= 1/255 and T (1 - alpha) >= 1e-4 (the last test ends the pixel without taking it);
depth += T alpha z; the median depth is z of the first taken splat after which T < 0.5.  Everything is float64, so a pixel
whose take / skip or median decision lies within float32 rounding of a threshold is flagged rather than decided."""
import numpy as np

ALPHA_MIN, T_MIN, ALPHA_MAX = 1.0 / 255.0, 1e-4, 0.99
ALPHA_RTOL = 1e-5            # float32 power / expf against float64: a few ulp of |power| <= ln 255
T_RTOL = 2e-4                # float32 T after hundreds of products against float64


def depth_planes(W, H, xy, conic_opacity, depth, point_list, ranges, tile=16):
    """xy [P,2], conic_opacity [P,4] (cx, cy, cz, o), depth [P] as float32 from the GPU; point_list [R] and ranges [T,2] of the
    forward's sorted lists.  Returns float64 (T, depth, median [H,W]) and a bool [H,W] mask of the pixels whose decisions lie
    within rounding of a threshold."""
    xy, co, z = (np.asarray(a, np.float64) for a in (xy, conic_opacity, depth))
    gx = (W + tile - 1) // tile
    T_out = np.ones((H, W))
    D_out = np.zeros((H, W))
    med_out = np.zeros((H, W))
    flag = np.zeros((H, W), bool)
    for t, (a, b) in enumerate(np.asarray(ranges, np.int64)):
        if b <= a:
            continue
        ty, tx = divmod(t, gx)
        ys, xs = np.mgrid[ty * tile:ty * tile + tile, tx * tile:tx * tile + tile]
        inside = (xs < W) & (ys < H)
        px, py = xs[inside].astype(np.float64), ys[inside].astype(np.float64)
        n = px.size
        T = np.ones(n)
        D = np.zeros(n)
        med = np.zeros(n)
        done = np.zeros(n, bool)
        fl = np.zeros(n, bool)
        for gid in np.asarray(point_list[a:b], np.int64):
            dx, dy = xy[gid, 0] - px, xy[gid, 1] - py
            cx, cy, cz, o = co[gid]
            power = -0.5 * (cx * dx * dx + cz * dy * dy) - cy * dx * dy
            alpha = np.minimum(ALPHA_MAX, o * np.exp(np.minimum(power, 0.0)))
            live = ~done & (power <= 0.0)
            fl |= ~done & (np.abs(power) <= 1e-6)
            fl |= live & (np.abs(alpha - ALPHA_MIN) <= ALPHA_RTOL * ALPHA_MIN)
            take = live & (alpha >= ALPHA_MIN)
            test_T = T * (1.0 - alpha)
            fl |= take & (np.abs(test_T - T_MIN) <= T_RTOL * T_MIN)
            end = take & (test_T < T_MIN)
            done |= end
            take &= ~end
            D = np.where(take, D + T * alpha * z[gid], D)
            fl |= take & (med == 0.0) & (np.abs(test_T - 0.5) <= T_RTOL * 0.5)
            med = np.where(take & (med == 0.0) & (test_T < 0.5), z[gid], med)
            T = np.where(take, test_T, T)
            if done.all():
                break
        T_out[ys[inside], xs[inside]] = T
        D_out[ys[inside], xs[inside]] = D
        med_out[ys[inside], xs[inside]] = med
        flag[ys[inside], xs[inside]] = fl
    return T_out, D_out, med_out, flag
