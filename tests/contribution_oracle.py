"""Float64 restatement of the contribution scores (glic_contribution) on the GPU's own sorted lists and splat records.

Per pixel, front to back over its tile's list, as render_camera_oracle walks it: power = -0.5 (cx dx^2 + cz dy^2) - cy dx dy,
alpha = min(0.99, o exp(power)); a splat is taken when power <= 0, alpha >= 1/255 and T (1 - alpha) >= 1e-4 (the last test ends
the pixel without taking it).  A taken pair has weight T alpha (T before the splat); a row's scores are the largest weight of
its taken pairs (0 if none), their number, and the number of pixels it ends.  A pixel whose take / skip decision lies within float32 rounding of a threshold
is flagged rather than decided, and every row of its tile's list is marked, since the pixel's later decisions may move too."""
import numpy as np

from render_camera_oracle import ALPHA_MAX, ALPHA_MIN, ALPHA_RTOL, T_MIN, T_RTOL


def scores(W, H, xy, conic_opacity, point_list, ranges, P, tile=16):
    """xy [P,2], conic_opacity [P,4] (cx, cy, cz, o) as float32 from the GPU; point_list [R] and ranges [T,2] of the forward's
    sorted lists.  Returns float64 max_weight [P], int64 hits [P], int64 ends [P], float64 final T [H,W], the bool [H,W] mask of flagged pixels
    and the bool [P] mask of rows a flagged pixel's list holds."""
    xy, co = (np.asarray(a, np.float64) for a in (xy, conic_opacity))
    gx = (W + tile - 1) // tile
    max_w = np.zeros(P)
    hits = np.zeros(P, np.int64)
    ends = np.zeros(P, np.int64)
    T_out = np.ones((H, W))
    flag = np.zeros((H, W), bool)
    marked = np.zeros(P, bool)
    for t, (a, b) in enumerate(np.asarray(ranges, np.int64)):
        if b <= a:
            continue
        ty, tx = divmod(t, gx)
        ys, xs = np.mgrid[ty * tile:ty * tile + tile, tx * tile:tx * tile + tile]
        inside = (xs < W) & (ys < H)
        px, py = xs[inside].astype(np.float64), ys[inside].astype(np.float64)
        n = px.size
        T = np.ones(n)
        done = np.zeros(n, bool)
        fl = np.zeros(n, bool)
        lst = np.asarray(point_list[a:b], np.int64)
        for gid in lst:
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
            ends[gid] += int(end.sum())
            take &= ~end
            if take.any():
                max_w[gid] = max(max_w[gid], float((T * alpha)[take].max()))
                hits[gid] += int(take.sum())
            T = np.where(take, test_T, T)
            if done.all():
                break
        T_out[ys[inside], xs[inside]] = T
        flag[ys[inside], xs[inside]] = fl
        if fl.any():
            marked[lst] = True
    return max_w, hits, ends, T_out, flag, marked
