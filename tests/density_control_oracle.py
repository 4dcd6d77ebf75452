"""NumPy restatement of the native mapper's density control (include/glic_b200.h: glic_mapper_densify_and_prune,
glic_mapper_set_density_schedule, glic_mapper_scene_extent) -- test infrastructure.

densify_and_prune() is the header's two-step definition: densify_oracle.select() gives the densify result, then the prune
predicate removes rows of it.  The activated values (opacity, largest scale) are inputs: pass the device's own (the activation
kernel's expf), as tests/densify_oracle.py does for the scales.
"""
import math

import numpy as np

import densify_oracle as do


def removed(act, smax, maxr, sky, min_opacity, max_screen_radius, max_world_scale):
    """the prune predicate per row: act(logit) < min_opacity, or (non-sky) maxr > max_screen_radius > 0, or (non-sky) largest
    activated scale > max_world_scale > 0.  A NaN opacity or scale never removes a row."""
    act, smax = np.asarray(act, np.float32), np.asarray(smax, np.float32)
    gone = act < np.float32(min_opacity)
    other = ~np.asarray(sky, bool)
    if max_screen_radius > 0:
        gone |= other & (np.asarray(maxr) > int(max_screen_radius))
    if max_world_scale > 0:
        gone |= other & (smax > np.float32(max_world_scale))
    return gone


def densify_and_prune(cls, act, smax, smax_child, maxr, n_sky, min_opacity=0.0, max_screen_radius=0, max_world_scale=0.0):
    """cls: densify_oracle.classes(); act, smax, maxr: per existing row; smax_child: the largest activated scale of a child of
    each row (its log-scale - log(1.6)).  Returns the surviving rows' sources (`src`), their rows in the unpruned densify result
    (`row`: a child's generator key), the unpruned result (`unpruned_src`) and the counts the call reports."""
    src, n = do.select(cls)
    rows = np.arange(src.size)
    kc = n["kept"] + n["cloned"]
    new, child = rows >= n["kept"], rows >= kc
    sky = ~new & (src < n_sky)
    mr = np.where(new, 0, np.asarray(maxr)[src])
    sm = np.where(child, np.asarray(smax_child, np.float32)[src], np.asarray(smax, np.float32)[src])
    keep = np.nonzero(~removed(np.asarray(act, np.float32)[src], sm, mr, sky, min_opacity, max_screen_radius, max_world_scale))[0]
    return dict(src=src[keep], row=keep, unpruned_src=src, sky=int(np.count_nonzero(sky[keep])),
                kept=int(np.count_nonzero(keep < n["kept"])), cloned=n["cloned"], split=n["split"],
                children=int(np.count_nonzero(keep >= kc)), pruned=int(src.size - keep.size), rows=int(keep.size), unpruned=n)


def schedule_step(n, densify_from=500, densify_until=15000, densify_interval=100, opacity_reset_interval=3000, **_):
    """what the schedule does after the iteration that made stats.iterations = n: (densify, size tests on, opacity reset)"""
    densify = densify_from < n < densify_until and n % densify_interval == 0
    sizes = densify and opacity_reset_interval > 0 and n > opacity_reset_interval
    reset = opacity_reset_interval > 0 and n < densify_until and n % opacity_reset_interval == 0
    return densify, sizes, reset


def scene_extent(centres):
    """getNerfppNorm's radius, 1.1 * max_k |c_k - mean(c)|, in double in the mapper's order, rounded to float32"""
    c = [[float(x) for x in row] for row in np.asarray(centres, np.float64).reshape(-1, 3)]
    if not c:
        return np.float32(0.0)
    mean = [0.0, 0.0, 0.0]
    for row in c:
        for i in range(3):
            mean[i] += row[i]
    mean = [m / len(c) for m in mean]
    far = 0.0
    for row in c:
        dx, dy, dz = row[0] - mean[0], row[1] - mean[1], row[2] - mean[2]
        far = max(far, math.sqrt(dx * dx + dy * dy + dz * dz))
    return np.float32(1.1 * far)


def reset_logit(max_opacity):
    """the logit glic_mapper_reset_opacity writes: log(r / (1 - r)) in double, r = (double)max_opacity, rounded to float32"""
    r = float(np.float32(max_opacity))
    return np.float32(math.log(r / (1.0 - r)))
