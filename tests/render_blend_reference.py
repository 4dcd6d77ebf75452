"""Float64 restatement of the training blend of csrc/render.cu -- render_forward_kernel<FWD_TRAIN> and render_backward_kernel
-- with a magnitude beside every output.

Inputs are the GPU's own: xy, conic_opacity and rgb of every Gaussian, the sorted point_list and the tile ranges (from
CRasterizer.debug_state()), and dL/dpix; all are taken as exact float32 values.  `walk` visits every pair of every tile list
at every pixel of the tile, with no row cull, and applies the reference's semantics (glic_oracle_render and
glic_oracle_render_backward): power > 0 skips the pair, alpha = min(0.99, o G), alpha < 1/255 skips the pair, T (1 - alpha)
< 1e-4 ends the pixel without taking the splat, and dL/dG = o dL/dalpha also where the 0.99 clamp is active.  It returns:

- per pixel: the colour C, the final T and n_contrib (the 1-based list position of the last splat taken); per tile
  max_contrib;
- per pair (list entry e = one (Gaussian, tile)) with dL/dpix given: the nine values the kernel adds for that Gaussian and
  tile -- mean.x, mean.y, conic.x, conic.y, conic.w, colour r, g, b, opacity -- scaled as the kernel scales them (mean by
  -0.5 W o and -0.5 H o, conic by -0.5 o).  Summed over the tiles they are the four 2-D gradients.

Values and magnitudes are loss_reference.Mag (see there): |float32 kernel - v| <= c * 2^-24 * m per element, c per output
in BOUND.  The magnitudes follow the kernels' formulation, not the textbook one: the colour suffix of dL/dalpha is
C_final - C_prefix, a cancellation costing the sum of both magnitudes; the five geometric values are formed from the
per-column moments S0 = sum w, S1 = sum w dy, S2 = sum w dy^2 of w = G dL/dalpha; T is a product chain whose magnitude grows
with every splat taken.

Each pixel gets a flag when one of its decisions lies within FLAG * 2^-24 * m of a threshold: power = 0, o G = 1/255, and
T (1 - alpha) = 1e-4.  The float32 kernel may decide such a pixel either way, so its colour, T and n_contrib are not
compared; the tests give it dL/dpix = 0, which makes every backward term it produces an exact zero in the kernel and here.

The walk goes down the lists one position at a time for all tiles at once, dropping tiles whose list has ended or whose
pixels have all ended, so its cost is about (pairs in the lists) x 256 pixel evaluations.

The same walk also runs in float32 (F32): numpy float32, one rounding per operation, in the kernels' order -- the forward's
warp-band row cull from each splat's half-extent hy (preprocess.cu), restarts of T and the colour suffix from the checkpoint
at each 32-splat bucket, the FAST body (MUFU.EX2 exponent with the expf fallback near 1/255, one colour suffix) or the
former exact body (expf, three suffixes), per-lane sums over the lane's pixel pairs, the reduce-scatter across the 32
lanes, and RP = 8 or 4 row pairs per warp.  ex2.approx and rcp.approx are emulated with their stated errors (2 and 1 ulp).
numpy has no fma; it is a float64 product and sum rounded to float32.  `mutant` applies one of MUTATIONS, a plausible kernel
bug, to that evaluation; tests/test_render_blend_reference_host.py checks that each pushes some element beyond its bound.
"""
import numpy as np

from loss_reference import U, Mag

TILE = 16
BUCKET = 32


def _f32(x):
    return float(np.float32(x))


# the thresholds as the kernels compare them (float32 constants) and as the float64 oracle does
KERNEL = dict(amin=_f32(np.float32(1.0) / np.float32(255.0)), tmin=_f32(1e-4), amax=_f32(0.99))
EXACT = dict(amin=1.0 / 255.0, tmin=1e-4, amax=0.99)

# |float32 kernel - v| <= c * 2^-24 * m per element.  Over every case of tests/test_gpu_render_blend_exact.py on an H100
# (sm_90a) the largest err / bound with these constants was 0.39 (C), 0.15 (T), and per (Gaussian, tile) entry 0.044 (mean),
# 0.047 (conic), 0.12 (colour) and 0.047 (opacity); the per-Gaussian sums of every atomic and deterministic form stayed
# below 0.04 of their bound.  The float32 evaluation of test_render_blend_reference_host.py stays within the same ranges.
BOUND = dict(C=4.0, T=4.0, mean=8.0, conic=8.0, opacity=8.0, color=4.0)
PAIR_KEYS = ("mean", "mean", "conic", "conic", "conic", "color", "color", "color", "opacity")
# half-width of the band around a decision threshold, in units of 2^-24 * m of the quantity decided on
FLAG = 4.0

MUTATIONS = ("hy_short", "bucket_last_dropped", "T_after", "ckpt_neighbour", "WH_swapped", "suffix_late", "my_cy_sign",
             "clamp_zero", "rp4_row15")


class _M:
    """float64 values with magnitudes"""
    mag = True

    @staticmethod
    def inp(x):
        return Mag(np.asarray(x, np.float64))

    @staticmethod
    def diff(a, b):
        """a - b of two exact inputs: one rounding of the exact difference"""
        d = np.asarray(a, np.float64) - np.asarray(b, np.float64)
        return Mag(d, np.abs(d))

    @staticmethod
    def full(shape, x, m):
        return Mag(np.full(shape, x, np.float64), np.full(shape, m, np.float64))

    @staticmethod
    def fma(a, b, c):
        return Mag.of(a) * b + c

    @staticmethod
    def exp(x, ulps):
        return x.exp(ulps)

    @staticmethod
    def ex2(x):
        return x.exp(4.0)

    @staticmethod
    def rcp(x):
        return x.rcp(1.0)

    @staticmethod
    def one_minus(x):
        """fl(1 - x): the constant 1 is exact, so the rounding is relative to the result"""
        return Mag(1.0 - x.v, np.abs(1.0 - x.v) + x.m)

    minimum = staticmethod(lambda a, c: a.minimum(c))
    where = staticmethod(Mag.where)
    v = staticmethod(lambda x: x.v)
    m = staticmethod(lambda x: x.m)

    @staticmethod
    def seq(x, axis):
        return x.sum(axis)

    tree = seq

    @staticmethod
    def scaled(o, c):
        """fl(c * o) for a float32 constant c: one rounding"""
        v = c * np.asarray(o, np.float64)
        return Mag(v, np.abs(v))

    @staticmethod
    def take(x, idx):
        return x[idx]


def _pert(x, salt):
    """a deterministic value in [-1, 1] per element: where in its error budget an approximate instruction lands"""
    b = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    return ((b * np.uint64(2654435761) + np.uint64(salt)) % np.uint64(2001)).astype(np.float64) / 1000.0 - 1.0


class _F32:
    """numpy float32, one rounding per operation"""
    mag = False
    LOG2E = np.float32(1.44269504088896341)

    @staticmethod
    def inp(x):
        return np.asarray(x, np.float32)

    @staticmethod
    def diff(a, b):
        return np.asarray(a, np.float32) - np.asarray(b, np.float32)

    @staticmethod
    def full(shape, x, m):
        return np.full(shape, x, np.float32)

    @staticmethod
    def fma(a, b, c):
        return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)

    @staticmethod
    def exp(x, ulps):
        return np.exp(np.asarray(x, np.float32))

    @staticmethod
    def ex2(p):
        """ex2.approx.ftz.f32(fl(p * fl(log2 e))): at most 2 ulp off 2^y; subnormal results flush to zero"""
        y = (np.asarray(p, np.float32) * _F32.LOG2E).astype(np.float32)
        e = np.exp2(y.astype(np.float64))
        e = (e * (1.0 + 2.0 ** -22 * _pert(y, 17))).astype(np.float32)
        return np.where(np.abs(e) < np.float32(2.0 ** -126), np.float32(0.0), e)

    @staticmethod
    def one_minus(x):
        return np.float32(1.0) - x

    @staticmethod
    def rcp(x):
        """rcp.approx.ftz.f32: at most 1 ulp"""
        r = 1.0 / np.asarray(x, np.float64)
        return (r * (1.0 + 2.0 ** -23 * _pert(x, 5))).astype(np.float32)

    @staticmethod
    def minimum(a, c):
        return np.minimum(a, np.float32(c))

    where = staticmethod(lambda c, a, b: np.where(c, a, b).astype(np.float32))
    v = staticmethod(lambda x: np.asarray(x, np.float64))
    m = staticmethod(lambda x: np.zeros(np.shape(x)))

    @staticmethod
    def seq(x, axis):
        """left fold from 0 along `axis`"""
        x = np.moveaxis(np.asarray(x, np.float32), axis, 0)
        acc = np.zeros(x.shape[1:], np.float32)
        for t in x:
            acc = acc + t
        return acc

    @staticmethod
    def tree(x, axis):
        """the butterfly over a power-of-two axis: element i meets i ^ (n/2) first, then i ^ (n/4), ..."""
        x = np.moveaxis(np.asarray(x, np.float32), axis, 0)
        while x.shape[0] > 1:
            h = x.shape[0] // 2
            x = x[:h] + x[h:]
        return x[0]

    @staticmethod
    def scaled(o, c):
        return np.float32(c) * np.asarray(o, np.float32)

    @staticmethod
    def take(x, idx):
        return x[idx]


M, F32 = _M, _F32


def half_extent(co, radii):
    """the per-splat vertical half-extent hy of preprocess.cu (float32, as there; __logf as logf)"""
    co = np.asarray(co, np.float32)
    cx, cy, cz, o = co[:, 0], co[:, 1], co[:, 2], co[:, 3]
    with np.errstate(all="ignore"):
        thr2 = np.log(np.float32(255.0) * o) + np.float32(1e-3)
        prod = cx * cz
        dcon = prod - cy * cy
        hy = np.float32(1.11) * np.asarray(radii).astype(np.float32) + np.float32(1.0)
        fine = np.sqrt(np.float32(2.0) * thr2 * cx / dcon) * np.float32(1.001) + np.float32(0.01)
        return np.where(dcon > np.float32(1e-3) * prod, np.minimum(hy, fine), hy).astype(np.float32)


def _gather_pix(img, px, py, inside):
    """[C,H,W] or [H,W] image -> [C, nt, 256] / [nt, 256] at the tiles' pixels (0 outside the frame)"""
    img = np.asarray(img)
    qy, qx = np.minimum(py, img.shape[-2] - 1), np.minimum(px, img.shape[-1] - 1)
    return np.where(inside, img[..., qy, qx], 0)


def walk(st, W, H, A=M, tiles=None, dL=None, Cf=None, consts=KERNEL, hy=None, fast=True, rp=8, mutant=None):
    """One walk over the lists of `tiles` (default: all).  st: xy [P,2], conic_opacity [P,4], rgb [P,3], point_list [R],
    ranges [T,2].  A = M (float64 + magnitudes, no row cull) or F32 (the kernels' float32 arithmetic; hy [P] enables their
    row culls).  Without dL: the forward.  With dL [3,H,W] and Cf (the forward's `C` of the same tiles): the forward again
    and the backward's per-pair values.  Returns a dict of per-tile-pixel arrays ([nt, 256], pixel = row * 16 + column):
    C (3 values), T, last (n_contrib), flag; max_contrib [nt]; pair_v / pair_m [R, 9] (backward only); paths."""
    xy = np.asarray(st["xy"], np.float64)
    co = np.asarray(st["conic_opacity"], np.float64)
    rgb = np.asarray(st["rgb"], np.float64)
    pl = np.asarray(st["point_list"]).astype(np.int64)
    rg = np.asarray(st["ranges"]).reshape(-1, 2).astype(np.int64)
    gx = (W + TILE - 1) // TILE
    tiles = np.arange(rg.shape[0]) if tiles is None else np.asarray(tiles, np.int64)
    nt = tiles.size
    start, n = rg[tiles, 0], rg[tiles, 1] - rg[tiles, 0]
    col, row = np.arange(256) % TILE, np.arange(256) // TILE
    px = (tiles % gx)[:, None] * TILE + col
    py = (tiles // gx)[:, None] * TILE + row
    inside = (px < W) & (py < H)
    amin, tmin, amax = consts["amin"], consts["tmin"], consts["amax"]
    bwd = dL is not None
    mutant = mutant or ""
    if mutant == "rp4_row15":
        rp = 4
    hy_eff = None
    if hy is not None:
        hy_eff = np.asarray(hy, np.float32) - (np.float32(0.5) if mutant == "hy_short" else np.float32(0.0))

    # output per tile pixel
    out = dict(C_v=np.zeros((3, nt, 256)), C_m=np.zeros((3, nt, 256)), T_v=np.ones((nt, 256)), T_m=np.ones((nt, 256)),
               last=np.zeros((nt, 256), np.int64), flag=np.zeros((nt, 256), bool))
    R = pl.size
    pair_v = np.zeros((R, 9)) if bwd else None
    pair_m = np.zeros((R, 9)) if bwd else None
    paths = dict(pairs=int(n.sum()), taken=0, ended=0, clamped=0, flag_power=0, flag_alpha=0, flag_T=0,
                 max_list=int(n.max()) if nt else 0, buckets=int(((n + BUCKET - 1) // BUCKET).sum()))

    S = dict(act=inside.copy(), T=A.full((nt, 256), 1.0, 1.0), last=np.zeros((nt, 256), np.int64),
             flag=np.zeros((nt, 256), bool))
    for c in range(3):
        S["C%d" % c] = A.full((nt, 256), 0.0, 0.0)
    if bwd:
        g = _gather_pix(dL, px, py, inside).astype(np.float64)
        for c in range(3):
            S["g%d" % c] = A.inp(g[c])
            S["f%d" % c] = Cf[c]
        for k in ("Tb", "Ab", "a0", "a1", "a2", "pT", "p0", "p1", "p2"):
            S[k] = A.full((nt, 256), 0.0, 0.0)
    cur = np.arange(nt)

    def flush(rows, Sx):
        idx = cur[rows]
        for c in range(3):
            out["C_v"][c, idx] = A.v(Sx["C%d" % c][rows])
            out["C_m"][c, idx] = A.m(Sx["C%d" % c][rows])
        out["T_v"][idx] = A.v(Sx["T"][rows])
        out["T_m"][idx] = A.m(Sx["T"][rows])
        out["last"][idx] = Sx["last"][rows]
        out["flag"][idx] = Sx["flag"][rows]

    Q = 8 // rp                   # parts per tile
    NP = rp // 2                  # pixel pairs per lane
    for j in range(paths["max_list"]):
        keep = (n[cur] > j) & S["act"].any(1)
        if not keep.all():
            flush(~keep, S)
            S = {k: x[keep] for k, x in S.items()}
            cur = cur[keep]
        if not cur.size:
            break
        e = start[cur] + j
        gid = pl[e]
        x, y = xy[gid, 0][:, None], xy[gid, 1][:, None]
        cxi, cyi, czi, oi = (co[gid, k][:, None] for k in range(4))
        cols = [A.inp(rgb[gid, k][:, None]) for k in range(3)]
        fx, fy = px[cur].astype(np.float64), py[cur].astype(np.float64)
        dx, dy = A.diff(x, fx), A.diff(y, fy)
        cx, cy, cz, o = A.inp(cxi), A.inp(cyi), A.inp(czi), A.inp(oi)
        power = A.fma(dx, dx * cx, dy * (dy * cz)) * (-0.5) - dy * (dx * cy)
        pv = A.v(power)
        act = S["act"]
        reach_f = reach_b = np.ones_like(act)
        if hy_eff is not None:
            h = hy_eff[gid][:, None]
            yf = np.float32(1.0) * xy[gid, 1][:, None].astype(np.float32)
            band_mid = (py[cur] - row + 4 * (row // 4)).astype(np.float32) + np.float32(1.5)
            reach_f = ~(np.abs(band_mid - yf) > h + np.float32(1.5))
            row_mid = (py[cur] - row + 2 * (row // 2)).astype(np.float32) + np.float32(0.5)
            reach_b = ~(np.abs(row_mid - yf) > h + np.float32(0.5))
        cand = act & reach_f & (pv <= 0.0)
        pneg = A.minimum(power, 0.0)
        G = A.exp(pneg, 2.0)
        oG = G * o
        alpha = A.minimum(oG, amax)
        av = A.v(alpha)
        tk = cand & (av >= amin)
        T = S["T"]
        one_m = A.one_minus(alpha)
        tT = T * one_m
        tTv = A.v(tT)
        end = tk & (tTv < tmin)
        if A.mag:
            fp = act & (np.abs(pv) < FLAG * U * power.m)
            fa = cand & (np.abs(oG.v - amin) < FLAG * U * oG.m)
            ft = tk & (np.abs(tTv - tmin) < FLAG * U * tT.m)
            S["flag"] = S["flag"] | fp | fa | ft
            paths["flag_power"] += int(fp.sum())
            paths["flag_alpha"] += int(fa.sum())
            paths["flag_T"] += int(ft.sum())
        tk = tk & ~end
        paths["taken"] += int(tk.sum())
        paths["ended"] += int(end.sum())
        paths["clamped"] += int((tk & (A.v(oG) > amax)).sum())

        if bwd:
            if j % BUCKET == 0:
                # restart from the bucket's checkpoint (T, C) -- the neighbouring bucket's under the mutant
                ck = (S["pT"], S["p0"], S["p1"], S["p2"]) if mutant == "ckpt_neighbour" and j >= BUCKET else \
                     (T, S["C0"], S["C1"], S["C2"])
                S["pT"], S["p0"], S["p1"], S["p2"] = T, S["C0"], S["C1"], S["C2"]
                S["Tb"] = ck[0]
                a = [ck[1 + c] - S["f%d" % c] for c in range(3)]
                S["a0"], S["a1"], S["a2"] = a
                S["Ab"] = A.fma(a[2], S["g2"], A.fma(a[1], S["g1"], a[0] * S["g0"]))
            tkb = tk & reach_b
            if mutant == "bucket_last_dropped":
                tkb = tkb & ~((j % BUCKET == BUCKET - 1) | (j == n[cur] - 1))[:, None]
            if mutant == "rp4_row15":
                tkb = tkb & (row != 15)[None, :]
            if fast:
                Gb = A.ex2(pneg)
                if not A.mag:
                    xb = Gb * o
                    near = np.abs(xb - np.float32(amin)) <= np.float32(amin / 65536.0)
                    Gb = np.where(near, G, Gb)
            else:
                Gb = G
            ab = A.minimum(Gb * o, amax)
            Gz = A.where(tkb, Gb, 0.0)
            al = A.where(tkb, ab, 0.0)
            one_mb = A.one_minus(al)
            Tb = S["Tb"]
            Tn = A.where(tkb, Tb * one_mb, Tb)
            dch = al * (Tn if mutant == "T_after" else Tb)
            ainv = A.rcp(one_mb)
            gs = [S["g%d" % c] for c in range(3)]
            csum = [dch * gs[c] for c in range(3)]
            if fast:
                cg = A.fma(gs[2], cols[2], A.fma(gs[1], cols[1], gs[0] * cols[0]))
                if mutant == "suffix_late":
                    dLa = A.fma(ainv, S["Ab"], Tb * cg)
                    S["Ab"] = A.where(tkb, A.fma(dch, cg, S["Ab"]), S["Ab"])
                else:
                    S["Ab"] = A.where(tkb, A.fma(dch, cg, S["Ab"]), S["Ab"])
                    dLa = A.fma(ainv, S["Ab"], Tb * cg)
            else:
                dLa = None
                for c in range(3):
                    S["a%d" % c] = A.where(tkb, A.fma(dch, cols[c], S["a%d" % c]), S["a%d" % c])
                    t = A.fma(ainv, S["a%d" % c], Tb * cols[c])
                    dLa = t * gs[c] if dLa is None else A.fma(t, gs[c], dLa)
            S["Tb"] = Tn
            w = Gz * dLa
            if mutant == "clamp_zero":
                w = A.where(A.v(oG) > amax, 0.0, w)
            w = A.where(tkb, w, 0.0)
            wy = w * dy
            wyy = wy * dy

            # per-lane sums: pixel (row 8q + 4p + 2s + h, column) of part q is pair p, half s of lane (h, column)
            def lanes(z):
                if A.mag:
                    zz = Mag(z.v.reshape(-1, Q, NP, 2, 2, 16), z.m.reshape(-1, Q, NP, 2, 2, 16))
                    s = zz.sum(2)
                    return Mag(s.v.sum(2).reshape(-1, Q, 32), s.m.sum(2).reshape(-1, Q, 32))
                zz = np.asarray(z, np.float32).reshape(-1, Q, NP, 2, 2, 16)
                s = A.seq(zz, 2)
                return (s[:, :, 0] + s[:, :, 1]).reshape(-1, Q, 32)
            v_o, s1, s2 = lanes(w), lanes(wy), lanes(wyy)
            v_c = [lanes(z) for z in csum]
            dxl = A.take(dx, (slice(None), slice(0, 32)))       # row 0 and 1 of the tile: the lane's column
            dxl = dxl[:, None, :] if not A.mag else Mag(dxl.v[:, None, :], dxl.m[:, None, :])
            c3 = [A.take(z, (slice(None), slice(None), None)) for z in (cx, cy, cz)]
            cxl, cyl, czl = c3
            sx = dxl * v_o
            v_mx = A.fma(sx, cxl, s1 * cyl)
            cyt = sx * cyl
            v_my = A.fma(s1, czl, -cyt if mutant == "my_cy_sign" else cyt)
            v_cx, v_cy, v_cw = sx * dxl, s1 * dxl, s2
            vals = [A.tree(z, 2) for z in (v_mx, v_my, v_cx, v_cy, v_cw, v_c[0], v_c[1], v_c[2], v_o)]   # [L, Q]
            sW, sH = (-0.5 * H, -0.5 * W) if mutant == "WH_swapped" else (-0.5 * W, -0.5 * H)
            o1 = oi[:, 0][:, None]
            fac = [A.scaled(o1, sW), A.scaled(o1, sH)] + [A.inp(o1) * (-0.5)] * 3 + [None] * 4
            for k in range(9):
                z = vals[k] if fac[k] is None else vals[k] * fac[k]
                z = A.seq(z, 1) if Q > 1 else A.take(z, (slice(None), 0))
                pair_v[e, k] = A.v(z)
                pair_m[e, k] = A.m(z)

        for c in range(3):
            Cc = S["C%d" % c]
            S["C%d" % c] = A.where(tk, A.fma(T, alpha * cols[c], Cc), Cc)
        S["T"] = A.where(tk, tT, T)
        S["last"] = np.where(tk, j + 1, S["last"])
        S["act"] = act & ~end
    if cur.size:
        flush(np.ones(cur.size, bool), S)
    out["max_contrib"] = out["last"].max(1) if nt else np.zeros(0, np.int64)
    out.update(pair_v=pair_v, pair_m=pair_m, paths=paths, px=px, py=py, inside=inside, tiles=tiles)
    out["C"] = [Mag(out["C_v"][c], out["C_m"][c]) if A.mag else out["C_v"][c].astype(np.float32) for c in range(3)]
    return out


def frame(x, w, H, W, fill=np.nan):
    """a per-tile-pixel array of walk `w` ([nt, 256] or [C, nt, 256]) as a frame [H, W] / [C, H, W]"""
    x = np.asarray(x)
    ins = w["inside"]
    lead = x.shape[:-2]
    f = np.full(lead + (H, W), fill, np.float64 if x.dtype.kind == "f" else x.dtype)
    f[..., w["py"][ins], w["px"][ins]] = x[..., ins]
    return f


def per_gaussian(w, point_list, P):
    """the walk's per-pair values summed per Gaussian: v [P, 9], m [P, 9], and the number of pairs of each Gaussian"""
    pl = np.asarray(point_list).astype(np.int64)
    v, m = np.zeros((P, 9)), np.zeros((P, 9))
    np.add.at(v, pl, w["pair_v"])
    np.add.at(m, pl, w["pair_m"])
    return v, m, np.bincount(pl, minlength=P)


def pair_bound(m, extra=0.0):
    """c * 2^-24 * m per column of a [*, 9] magnitude array (extra: additional roundings per element, e.g. a summation's)"""
    c = np.array([BOUND[k] for k in PAIR_KEYS])
    e = np.asarray(extra, np.float64)
    return (c + (e[:, None] if e.ndim else e)) * U * m


def ratio(got, v, bound):
    """|got - v| / bound elementwise (0 where both the error and the bound are 0); non-finite values give inf"""
    got = np.asarray(got, np.float64)
    err = np.abs(got - v)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0.0, 0.0, err / bound)
    return np.where(np.isfinite(got), r, np.inf)
