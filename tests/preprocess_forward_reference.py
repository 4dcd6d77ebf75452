"""Float64 restatement of csrc/preprocess.cu's per-Gaussian forward (preprocess_forward_kernel), with a magnitude beside every
float output and every discrete decision made in float64.

Per Gaussian the kernel computes, in float32: the view-space depth and the near cull (tz <= 0.2); cov3D from scale, modifier
and quaternion; the EWA 2-D covariance with the lim* clamps and the 0.3 dilation (preprocess_backward_reference.ewa_forward,
which the backward restatement shares); det and the conic, with the det == 0 and opacity < 1/255 culls; lambda1 and
radius = ceil(3 sqrt(lambda1)); the pixel centre (ndc2Pix, in double); the tile rect (getRect); the accept set, every tile of
the rect whose tile_max_power (geom_math.cuh, StopThePop's rectangle test) is <= log(255 o), and the cull of rows with no
accepted tile; the SH colour of degree D from an [P, M, 3] tensor with M >= (D + 1)^2 - 1, + 0.5, the clamp at 0 and the three
clamp bits; and the render row cull's half-extent hy.

Values and magnitudes are loss_reference.Mag, as in preprocess_backward_reference: |float32 kernel - v| <= c * 2^-24 * m per
element, one constant c per float output (BOUND).  Every decision is taken on the float64 value; a row whose decision quantity
lies within BAND * 2^-24 * m of its threshold is put in a band and may take either side: the near cull, det == 0, the 0.1
floor of lambda1, the ceil of the radius, the four truncations of the rect, each tile test (one such tile is `unsure`), and
each clamp.  A clamp's band changes only the clamp bit: the clamped and unclamped colour are both within the bound there.

hy is not bounded against a restated value but checked as the property the render needs (half_height): it is at least the
float64 half-height of {alpha >= 1/255}.

`mutate` applies one of MUTATIONS, a plausible kernel bug, to the restatement; tests/test_preprocess_forward_reference_host.py
checks that each moves some element of its scenes beyond its bound (hy_without_margin: below the half-height).

"""
import numpy as np

from loss_reference import U, Mag
from preprocess_backward_reference import (MAG32, MAG64, SH0, _sh_basis, _xform_row, ewa_forward)

# |float32 kernel - v| <= c * 2^-24 * m per element.  Geometry is a fixed float32 order of at most ~30 roundings, the colour
# a sum of up to 16 products contracted as nvcc chooses.  Over every case of tests/test_gpu_preprocess_forward_exact.py on an
# H100 80GB HBM3 (sm_90a, 700 W limit) the largest err / bound with these constants was 0.43 (depth), 0.28 (xy), 0.08 (conic)
# and 0.68 (rgb); the float32 oracle of test_preprocess_forward_reference_host.py stays within the same ranges.  The kernel's
# hy exceeded the float64 half-height by a factor of at least 1.001 on every visible splat.
BOUND = dict(depth=2.0, xy=4.0, conic=4.0, rgb=4.0)
# half-width of the band around a threshold, in units of 2^-24 * m of the decision quantity
BAND = 8.0
TILE = 16

MUTATIONS = ("sh2_sign", "clamp_at_1", "no_dilation", "dc_without_C0", "unnormalised_dir", "sh_row_stride_count",
             "hy_without_margin")


def sh_count(D):
    return (D + 1) ** 2 - 1


def _near(A, q, t):
    return np.abs(q.v - t) <= BAND * U * q.m


def _ndc2pix(A, ndc, S):
    """(float)(fma((double)ndc + 1, S, -1) * 0.5): one float32 rounding of a double result"""
    return ((ndc + A.ka(1.0)) * A.k(float(S)) - A.ka(1.0)) * 0.5


def _trunc_band(A, q, hi):
    """(int)q clamped to [0, hi]: which integers the float32 q may straddle (k = 0 decides nothing: both sides give 0)"""
    k = np.round(q.v)
    return (np.abs(q.v - k) <= BAND * U * q.m) & (k >= 1) & (k <= hi)


def _clip_trunc(v, hi):
    return np.clip(np.floor(v), 0, hi).astype(np.int64)


def tile_power(A, cox, coy, coz, mx, my, tx, ty):
    """geom_math.cuh tile_max_power on candidate pairs (Mag arrays cox.. mx, my; int arrays tx, ty), with `unsure`: pairs
    whose side tests of the mean against the tile's pixel-centre rectangle lie within the band"""
    tminx, tminy = (tx * TILE).astype(np.float64), (ty * TILE).astype(np.float64)
    tmaxx, tmaxy = tminx + (TILE - 1), tminy + (TILE - 1)
    xmd, ymd = A.k(0) + tminx - mx, A.k(0) + tminy - my          # tminx - mx: the kernel's fsub
    x_left, y_above = xmd.v > 0, ymd.v > 0
    right, below = mx.v > tmaxx, my.v > tmaxy
    unsure = (_near(A, xmd, 0.0) | _near(A, ymd, 0.0) | _near(A, mx - tmaxx, 0.0) | _near(A, my - tmaxy, 0.0))
    not_in_x = x_left.astype(np.float64) + right
    not_in_y = y_above.astype(np.float64) + below
    inside = not_in_x + not_in_y == 0
    sx = sy = float(TILE - 1)
    px, py = np.where(x_left, tminx, tmaxx), np.where(y_above, tminy, tmaxy)
    dx, dy = np.where(xmd.v < 0, -sx, sx), np.where(ymd.v < 0, -sy, sy)
    diffx, diffy = mx - px, my - py
    rcpx, rcpy = A.k(1) / (cox * (sx * sx)), A.k(1) / (coz * (sy * sy))
    ux = ((coy * dx) * diffy + (cox * dx) * diffx) * rcpx
    uy = ((coz * dy) * diffy + (coy * dy) * diffx) * rcpy
    tx_ = A.clip(ux, 0.0, 1.0) * Mag(not_in_y, 0.0)
    ty_ = A.clip(uy, 0.0, 1.0) * Mag(not_in_x, 0.0)
    ex, ey = mx - (tx_ * dx + px), my - (ty_ * dy + py)
    h = (ex * (cox * ex) + ey * (coz * ey)) * 0.5
    pw = (coy * ex) * ey + h
    return A.where(inside, A.k(0), pw), unsure & ~inside


def _accept(A, cox, coy, coz, mx, my, thr, rect, n, T, gx, chunk):
    """every candidate tile of every rect (n [P] candidates, rect [P,4]) through tile_power <= thr, about `chunk` pairs at a
    time: sure pairs, unsure pairs (tile test or side test within the band), and their counts per row"""
    P = n.size
    rw = rect[:, 2] - rect[:, 0]
    sure_cnt, unsure_cnt = np.zeros(P, np.int64), np.zeros(P, np.int64)
    pairs, upairs = [np.zeros(0, np.int64)], [np.zeros(0, np.int64)]
    rows = np.flatnonzero(n > 0)
    csum = np.cumsum(n[rows])
    start = 0
    while start < rows.size:
        stop = max(int(np.searchsorted(csum, (csum[start - 1] if start else 0) + chunk, side="right")), start + 1)
        sel = rows[start:stop]
        cnt = n[sel]
        gid = np.repeat(sel, cnt)
        j = np.arange(gid.size) - np.repeat(np.cumsum(cnt) - cnt, cnt)
        tx = rect[gid, 0] + j % rw[gid]
        ty = rect[gid, 1] + j // rw[gid]
        pwr, uns = tile_power(A, cox[gid], coy[gid], coz[gid], mx[gid], my[gid], tx, ty)
        t = thr[gid]
        acc = pwr.v <= t.v
        uns |= np.abs(pwr.v - t.v) <= BAND * U * (pwr.m + t.m)
        key = gid.astype(np.int64) * T + ty * gx + tx
        pairs.append(key[acc & ~uns])
        upairs.append(key[uns])
        sure_cnt += np.bincount(gid[acc & ~uns], minlength=P)
        unsure_cnt += np.bincount(gid[uns], minlength=P)
        start = stop
    return dict(pairs=np.sort(np.concatenate(pairs)), unsure_pairs=np.sort(np.concatenate(upairs)), tiles=sure_cnt,
                unsure=unsure_cnt)


def tile_rect_f32(xy, radius, W, H):
    """geom_math.cuh tile_rect in float32 (numpy float32 arithmetic rounds as the kernel's intrinsics do): [P,4] x0, y0, x1, y1"""
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    x, y = (np.asarray(xy, np.float32)[:, j] for j in range(2))
    r = np.asarray(radius).astype(np.float32)
    q, f16, m1 = np.float32(0.0625), np.float32(16.0), np.float32(-1.0)

    def cl(val, hi):
        with np.errstate(invalid="ignore"):
            return np.clip(np.trunc(np.nan_to_num(val)).astype(np.int64), 0, hi)
    return np.stack([cl((x - r) * q, gx), cl((y - r) * q, gy), cl((((x + r) + f16) + m1) * q, gx),
                     cl((((y + r) + f16) + m1) * q, gy)], 1)


def record_accept_sets(xy, conic_opacity, radius, W, H, A=MAG32, chunk=1 << 21):
    """the accept sets of a forward's own record (xy [P,2], conic_opacity [P,4], radius [P], float32), the record's values
    taken as exact: what the tile walk of preprocess_forward_kernel and emit_keys_kernel must produce from them.  Rows with
    radius <= 0 have none."""
    with np.errstate(all="ignore"):
        xy, co = np.asarray(xy, np.float32), np.asarray(conic_opacity, np.float32)
        P = xy.shape[0]
        gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
        rect = tile_rect_f32(xy, radius, W, H)
        n = np.where(np.asarray(radius) > 0, (rect[:, 2] - rect[:, 0]) * (rect[:, 3] - rect[:, 1]), 0)
        X = A.x
        thr = A.log(X(co[:, 3]) / A.k(1.0 / 255.0))
        return _accept(A, X(co[:, 0]), X(co[:, 1]), X(co[:, 2]), X(xy[:, 0]), X(xy[:, 1]), thr, rect, n, gx * gy, gx, chunk)


def forward(g, cam, mod=1.0, A=MAG32, no_color=False, mutate=None, chunk=1 << 21):
    """preprocess_forward_kernel on P rows.

    g: dict(means [P,3], scales [P,3] (activated), rots [P,4] (normalised), opacity [P], dc [P,3], sh [P,M,3], degree).
    cam: dict(view, proj, campos, lims, W, H, fx, fy): fx, fy as the kernel forms them (float32 W / (2 tan fovx)) with MAG32,
    as the float64 oracle does with MAG64 (preprocess_backward_reference's cams() gives both).

    Returns a dict: vis [P] (the float64 decisions), radius [P], rect [P,4] (x0, y0, x1, y1), tiles [P] (accepted tiles
    outside the band), unsure [P] (tiles in the band), pairs / unsure_pairs (int64 gid * T + tile, sorted), clamped [P,3] (u8);
    Mags depth [P], xy [P,2], conic [P,3], opacity-scaled thr [P], rgb [P,3], cov [P,3] (a, b, c); band: dict of bool [P] per
    decision (skip: the row's rect or visibility is undecided; tile: some tile test is; clamp_c: channel c's clamp);
    and paths: counts of the rows that took each path."""
    with np.errstate(all="ignore"):
        return _forward(g, cam, mod, A, no_color, mutate, chunk)


def _forward(g, cam, mod, A, no_color, mutate, chunk):
    means, scales, rots = (np.asarray(g[k], np.float32) for k in ("means", "scales", "rots"))
    P = means.shape[0]
    opac = np.asarray(g["opacity"], np.float32).reshape(P)
    D = int(g["degree"])
    W, H = int(cam["W"]), int(cam["H"])
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    T = gx * gy
    k, X = A.k, A.x
    v = [X(a) for a in np.asarray(cam["view"], np.float32)]
    pr = [X(a) for a in np.asarray(cam["proj"], np.float32)]
    cp = [X(a) for a in np.asarray(cam["campos"], np.float32)]
    lims = [float(a) for a in np.asarray(cam["lims"], np.float32)]
    fx, fy = X(cam["fx"]), X(cam["fy"])
    px, py, pz = (X(means[:, j]) for j in range(3))
    sraw = [X(scales[:, j]) for j in range(3)]
    q = [X(rots[:, j]) for j in range(4)]
    e = ewa_forward(A, v, lims, fx, fy, X(np.float32(mod)), px, py, pz, sraw, q, dilation=mutate != "no_dilation")
    a, b, c, tz = e["a"], e["b"], e["c"], e["tz"]
    band = {}
    f32 = (lambda x: float(np.float32(x))) if not A.f64 else float

    # ---- culls, conic, radius, pixel centre, rect -----------------------------------------------------------------------------
    near_t = f32(0.2)
    active = ~(tz.v <= near_t)
    near_band = _near(A, tz, near_t)
    skip = np.zeros(P, bool)                      # the other undecided decisions, counted on rows past the near cull
    hx, hy, hw = (_xform_row(pr, j, px, py, pz) for j in (0, 1, 3))
    pw = k(1) / (hw + A.ka(1e-7))
    ndcx, ndcy = hx * pw, hy * pw
    det = a * c - b * b
    active &= det.v != 0.0
    skip |= _near(A, det, 0.0)
    det_inv = k(1) / det
    cox, coy, coz = c * det_inv, det_inv * -b, a * det_inv
    o = X(opac)
    low_op = opac < np.float32(1.0 / 255.0) if not A.f64 else opac < 1.0 / 255.0
    active &= ~low_op
    mid = (a + c) * 0.5
    disc = mid * mid - det
    floor_ = f32(0.1)
    skip |= _near(A, disc, floor_)
    lam1 = mid + A.sqrt(A.where(disc.v > floor_, disc, A.ka(0.1)))
    s3 = A.sqrt(lam1) * k(3)
    rad_f = np.ceil(s3.v)
    skip |= _near(A, s3, np.round(s3.v))
    mx, my = _ndc2pix(A, ndcx, W), _ndc2pix(A, ndcy, H)
    irad = np.where(active, np.nan_to_num(rad_f, nan=0.0, posinf=2.0 ** 31, neginf=0.0), 0.0).clip(0, 2.0 ** 31).astype(np.int64)
    r_ = irad.astype(np.float64)
    q0 = [(mx - r_) * 0.0625, (my - r_) * 0.0625]
    q1 = [(mx + r_ + A.ka(16.0) - A.ka(1.0)) * 0.0625, (my + r_ + A.ka(16.0) - A.ka(1.0)) * 0.0625]
    rect = np.stack([_clip_trunc(q0[0].v, gx), _clip_trunc(q0[1].v, gy), _clip_trunc(q1[0].v, gx), _clip_trunc(q1[1].v, gy)], 1)
    for qq, hi in ((q0[0], gx), (q0[1], gy), (q1[0], gx), (q1[1], gy)):
        skip |= _trunc_band(A, qq, hi)
    thr = A.log(o / k(1.0 / 255.0))
    rect[~active] = 0
    rw, rh = rect[:, 2] - rect[:, 0], rect[:, 3] - rect[:, 1]
    n = np.where(active, np.maximum(rw, 0) * np.maximum(rh, 0), 0)

    # ---- the accept set, from the restated record -----------------------------------------------------------------------------
    sets = _accept(A, cox, coy, coz, mx, my, thr, rect, n, T, gx, chunk)
    sure_cnt, unsure_cnt = sets["tiles"], sets["unsure"]
    vis = active & (sure_cnt + unsure_cnt > 0)
    band["skip"] = (near_band | (skip & ~(tz.v <= near_t))) & ~low_op
    band["visible"] = active & (sure_cnt == 0) & (unsure_cnt > 0) & ~band["skip"]

    # ---- colour ----------------------------------------------------------------------------------------------------------------
    rgb = A.zeros((P, 3)) if A.mag else None
    clamped = np.zeros((P, 3), np.uint8)
    nclamp = [0, 0, 0]
    if not no_color:
        od = [px - cp[0], py - cp[1], pz - cp[2]]
        inv = k(1) / A.sqrt(od[0] * od[0] + od[1] * od[1] + od[2] * od[2])
        x_, y_, z_ = (od if mutate == "unnormalised_dir" else [oj * inv for oj in od])
        dc = np.asarray(g["dc"], np.float32).reshape(P, 3)
        res = [(X(dc[:, ch]) if mutate == "dc_without_C0" else k(SH0) * X(dc[:, ch])) for ch in range(3)]
        if D > 0:
            nb = sh_count(D)
            sh = np.asarray(g["sh"], np.float32).reshape(P, -1, 3)
            M = sh.shape[1]
            assert M >= nb, (M, nb)
            if mutate == "sh_row_stride_count":        # row idx * count(D) of the flat tensor instead of row idx * M
                flat = sh.reshape(-1, 3)
                sh = flat[np.clip(np.arange(P)[:, None] * nb + np.arange(nb)[None, :], 0, flat.shape[0] - 1)]
            bs = _sh_basis(A, D, x_, y_, z_)
            if mutate == "sh2_sign" and D > 1:
                bs[4] = -bs[4]
            for kk in range(nb):
                for ch in range(3):
                    res[ch] = res[ch] + bs[kk] * X(sh[:, kk, ch])
        res = [r_c + A.ka(0.5) for r_c in res]
        parts = []
        for ch in range(3):
            cl = res[ch].v < 0.0
            band["clamp_%d" % ch] = _near(A, res[ch], 0.0) & vis
            clamped[:, ch] = cl & vis
            nclamp[ch] = int((cl & vis & ~band["clamp_%d" % ch]).sum())
            val = A.where(cl, A.k(0), res[ch])
            val = Mag(val.v, np.where(cl, res[ch].m, val.m))     # a clamp within the band: 0 and res both within the bound
            if mutate == "clamp_at_1":
                val = A.where(val.v > 1.0, A.ka(1.0), val)
            parts.append(val)
        rgb = A.stack(parts, P)

    def keep(m_):
        return Mag(np.where(vis.reshape((-1,) + (1,) * (m_.v.ndim - 1)), m_.v, 0.0),
                   np.where(vis.reshape((-1,) + (1,) * (m_.v.ndim - 1)), m_.m, 0.0))

    out = dict(vis=vis, radius=np.where(vis, irad, 0), rect=np.where(vis[:, None], rect, 0), tiles=np.where(vis, sure_cnt, 0),
               unsure=np.where(vis, unsure_cnt, 0), pairs=sets["pairs"], unsure_pairs=sets["unsure_pairs"], clamped=clamped, T=T,
               gx=gx,
               depth=keep(tz), xy=keep(A.stack([mx, my], P)), conic=keep(A.stack([cox, coy, coz], P)), thr=thr,
               rgb=keep(rgb) if rgb is not None else None, cov=A.stack([a, b, c], P), band=band)
    band_rows = np.any([bb for bb in band.values()], 0)
    out["band_rows"] = band_rows
    out["paths"] = dict(rows=P, visible=int(vis.sum()), near=int(((tz.v <= near_t) & ~band_rows).sum()),
                        low_opacity=int(low_op.sum()),
                        no_tile=int((active & ~vis & ~band_rows).sum()), lam_floor=int((active & ~(disc.v > floor_)).sum()),
                        clamped=nclamp, band=int(band_rows.sum()))
    return out


def hy_f32(co, radii, mutate=None):
    """the kernel's hy in float32 (preprocess.cu, where the record's .w is written; __logf as logf).  hy_without_margin drops
    the three safety terms: + 1e-3 on the threshold, * 1.001 and + 0.01"""
    co = np.asarray(co, np.float32)
    cx, cy, cz, o = co[:, 0], co[:, 1], co[:, 2], co[:, 3]
    bare = mutate == "hy_without_margin"
    with np.errstate(all="ignore"):
        thr2 = np.log(np.float32(255.0) * o) + (np.float32(0.0) if bare else np.float32(1e-3))
        prod = cx * cz
        dcon = prod - cy * cy
        hy = np.float32(1.11) * np.asarray(radii).astype(np.float32) + np.float32(1.0)
        fine = np.sqrt(np.float32(2.0) * thr2 * cx / dcon)
        if not bare:
            fine = fine * np.float32(1.001) + np.float32(0.01)
        return np.where(dcon > np.float32(1e-3) * prod, np.minimum(hy, fine), hy).astype(np.float32)


def half_height(co, cov, vis):
    """float64 half-height of {alpha >= 1/255} = {q <= 2 ln(255 o)} per visible splat: of the splat's own float32 conic (when
    its float64 determinant is not cancelled: > 1e-3 cox coz) and of the restatement's 2-D covariance, sqrt(2 ln(255 o) c);
    the larger of the two"""
    co = np.asarray(co, np.float64)
    cx, cy, cz, o = co[:, 0], co[:, 1], co[:, 2], co[:, 3]
    with np.errstate(all="ignore"):
        t = 2.0 * np.log(255.0 * o)
        dcon = cx * cz - cy * cy
        h_conic = np.where(dcon > 1e-3 * cx * cz, np.sqrt(np.maximum(t, 0.0) * cx / dcon), 0.0)
        h_cov = np.sqrt(np.maximum(t, 0.0) * np.asarray(cov.v if isinstance(cov, Mag) else cov, np.float64)[:, 2])
        return np.where(vis, np.maximum(np.nan_to_num(h_conic), h_cov), 0.0)


def ratio(got, ref, c, rows):
    """max over rows (bool [P]) of |got - v| / (c 2^-24 m); non-finite values fail"""
    got = np.asarray(got, np.float64).reshape(ref.v.shape)[rows]
    if not np.all(np.isfinite(got)):
        return np.inf
    err = np.abs(got - ref.v[rows])
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0.0, 0.0, err / (c * U * ref.m[rows]))
    return float(r.max()) if r.size else 0.0


def compare(ref, got, rec):
    """one forward's integer outputs against the restatement.  got: dict(radius [P], tiles [P], clamped [P,3], pairs (sorted
    int64 gid * T + tile)); rec: record_accept_sets of the same forward's record.  Visibility, radius and clamp bits are held to
    the restated chain, except on the rows in its band for that decision.  The accept set of every row is held to rec (it may
    hold any of rec's unsure pairs), and where the chain decides every tile of a row, to the chain's.  Returns (rows that
    disagree, per output; band rows [P])."""
    T = ref["T"]
    P = ref["vis"].size
    band = ref["band"]
    tiles = np.asarray(got["tiles"], np.int64)
    gvis = tiles > 0
    gp = np.asarray(got["pairs"], np.int64)
    bad = {}
    bad["visible"] = np.flatnonzero((gvis != ref["vis"]) & ~band["skip"] & ~band["visible"])
    both = gvis & ref["vis"] & ~band["skip"]
    bad["radius"] = np.flatnonzero(both & (np.asarray(got["radius"]) != ref["radius"]))
    cl = np.asarray(got["clamped"]).reshape(P, 3).astype(bool)
    cb = np.stack([band.get("clamp_%d" % ch, np.zeros(P, bool)) for ch in range(3)], 1)
    bad["clamped"] = np.flatnonzero((both[:, None] & (cl != ref["clamped"].astype(bool)) & ~cb).any(1))
    bad["tiles"] = np.flatnonzero(tiles != np.bincount(gp // T, minlength=P)[:P])
    # the record's accept sets: every sure pair is there, every pair there is sure or unsure
    missing = rec["pairs"][gvis[rec["pairs"] // T]]
    missing = missing[~np.isin(missing, gp, assume_unique=True)]
    extra = gp[~np.isin(gp, rec["pairs"], assume_unique=True) & ~np.isin(gp, rec["unsure_pairs"], assume_unique=True)]
    # the chain's, on the rows it decides
    decided = both & (ref["unsure"] == 0)
    cs = ref["pairs"][decided[ref["pairs"] // T]]
    gsel = gp[decided[gp // T]]
    chain = np.setxor1d(cs, gsel)
    bad["pairs"] = np.unique(np.concatenate([missing, extra]) // T)
    bad["chain_pairs"] = np.unique(chain // T)
    rows = band["skip"] | band["visible"] | cb.any(1) | (gvis & (rec["unsure"] > 0))
    return bad, rows
