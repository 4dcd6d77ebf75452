"""render_forward_kernel<FWD_TRAIN> and render_backward_kernel (csrc/render.cu) against the float64 restatement of
tests/render_blend_reference.py at every pixel and every (Gaussian, tile) contribution, each element against its own bound
|got - v| <= c * 2^-24 * m (c in render_blend_reference.BOUND, m the restatement's magnitude).  There is no outlier fraction
and no tolerance relative to a tensor's maximum: a bug confined to a few pixels or pairs fails.

The restatement takes the kernels' own inputs (xy, conic_opacity, rgb, point_list and ranges from debug_state(), and
dL/dpix) and walks every pair of every tile list without the row cull, so a cull that drops a pair the blend takes is seen.
Pixels whose decisions lie within rounding of a threshold are flagged; their colour, T and n_contrib are not compared and
they get dL/dpix = 0, which makes every backward term they produce an exact zero in the kernel and in the restatement.
Each case asserts that only a few pixels are flagged (see FLAG_SHARE in test_render_blend_reference_host.py) and prints
the count.

- Forward: C and T at every unflagged pixel within the bound, n_contrib equal there, and max_contrib equal to the maximum
  of the kernel's own n_contrib over each tile.
- Backward per (Gaussian, tile): CRasterizer.deterministic_entries gives, bit for bit, what the atomic form adds for each
  bucket; every entry is held to the restated tile contribution.  A pair that one side has and the other lacks counts as zero
  on the lacking side.  A large frame (cfg2) is checked on a sample of tiles this way.
- Backward per Gaussian, for render_backward(exact=False) (production), render_backward(exact=True) and the 2-D outputs of
  backward() and of backward(deterministic=True): the summed bound plus (5 + adds) * 2^-24 * sum m, where 5 is the depth of
  the in-warp sum and adds = tiles touched (the deterministic fold adds fewer).

Run with -s to see max(err / bound) per output and form, the flagged pixels and the paths each case reached.
"""
import time

import numpy as np
import pytest

import render_blend_reference as rb
from helpers import POSES, hy_fallbacks, small_scene
from test_gpu_stress import CASES as STRESS_CASES
from test_render_blend_reference_host import flag_limit

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

DEV = "cuda:0"
FOLD = 5.0                       # roundings of the in-warp sum (32 lanes) before an entry leaves the warp
TWO_D = ("dL_dmeans2D", "dL_dconic", "dL_dopacity", "dL_dcolors")


def _two_d(grads):
    g = {k: grads[k].cpu().numpy().astype(np.float64) for k in TWO_D}
    return np.concatenate([g["dL_dmeans2D"][:, :2], g["dL_dconic"][:, [0, 1, 3]], g["dL_dcolors"], g["dL_dopacity"]], 1)


def _max_by_key(r):
    """[.., 9] ratios -> max per output kind"""
    r = np.asarray(r).reshape(-1, 9)
    return {k: float(max(r[:, i].max() if r.size else 0.0 for i, kk in enumerate(rb.PAIR_KEYS) if kk == k))
            for k in ("mean", "conic", "color", "opacity")}


class Case:
    """one forward on the GPU with the restatement's forward of the same lists"""

    def __init__(self, g, cam, tiles=None, kind=""):
        from gaussian_lic_b200 import ops
        self.W, self.H, self.kind = cam["W"], cam["H"], kind
        self.r = ops.CRasterizer(self.W, self.H)
        self.gd = ops.scene_to_device(g)
        self.view = self.r.make_view(cam)
        color, T, self.radii = self.r.forward(self.gd, self.view)
        torch.cuda.synchronize()
        d = self.r.debug_state()
        self.d = d
        self.st = dict(xy=d["xy"].cpu().numpy(), conic_opacity=d["conic_opacity"].cpu().numpy(), rgb=d["rgb"].cpu().numpy(),
                       point_list=d["point_list"].cpu().numpy().view(np.uint32),
                       ranges=d["ranges"].cpu().numpy().view(np.uint32))
        self.P = self.st["xy"].shape[0]
        self.color, self.T = color.cpu().numpy(), T.cpu().numpy()
        self.nc = d["n_contrib"].cpu().numpy().view(np.uint32).reshape(self.H, self.W)
        self.mc = d["max_contrib"].cpu().numpy().view(np.uint32)
        self.tiles = tiles(self.st["ranges"]) if callable(tiles) else tiles
        t0 = time.time()
        self.fw = rb.walk(self.st, self.W, self.H, tiles=self.tiles)
        self.t_walk = time.time() - t0
        fw = self.fw
        self.flagged = rb.frame(fw["flag"], fw, self.H, self.W, False)
        self.nflag = int(self.flagged.sum())

    def check_forward(self):
        fw, H, W = self.fw, self.H, self.W
        ok = fw["inside"] & ~fw["flag"]
        gx = lambda a: rb._gather_pix(a, fw["px"], fw["py"], fw["inside"])
        col, T, nc = gx(self.color), gx(self.T), gx(self.nc).astype(np.int64)
        r = dict(C=max(float(rb.ratio(col[c][ok], fw["C_v"][c][ok], rb.BOUND["C"] * rb.U * fw["C_m"][c][ok]).max(initial=0))
                       for c in range(3)),
                 T=float(rb.ratio(T[ok], fw["T_v"][ok], rb.BOUND["T"] * rb.U * fw["T_m"][ok]).max(initial=0)))
        bad = ok & (nc != fw["last"])
        assert not bad.any(), ("n_contrib differs at %d unflagged pixels" % bad.sum(), nc[bad][:8], fw["last"][bad][:8])
        np.testing.assert_array_equal(self.mc[fw["tiles"]].astype(np.int64), nc.max(1), err_msg="max_contrib")
        assert self.nflag <= flag_limit(self.kind, W * H), (self.nflag, W * H)
        return r

    def dL(self, kind="normal", seed=0, pixel=None):
        """dL/dpix of a pattern, exactly zero at the flagged pixels"""
        H, W = self.H, self.W
        if kind == "normal":
            dL = np.random.default_rng(seed).normal(size=(3, H, W)).astype(np.float32)
        elif kind == "onehot":
            dL = np.zeros((3, H, W), np.float32)
            dL[:, pixel[0], pixel[1]] = np.float32([1.0, -0.75, 0.5])
        else:                                     # the fused loss's own dL/dimg against a random target
            gt = np.random.default_rng(seed).random((3, H, W), dtype=np.float32)
            _, dl = self.r.loss(torch.as_tensor(self.color).to(DEV), torch.as_tensor(gt).to(DEV))
            torch.cuda.synchronize()
            dL = dl.cpu().numpy().copy()
        dL[:, self.flagged] = 0.0
        return dL

    def check_backward(self, dL, forms=True):
        fw = self.fw
        dLt = torch.as_tensor(dL).to(DEV)
        t0 = time.time()
        bw = rb.walk(self.st, self.W, self.H, tiles=self.tiles, dL=dL, Cf=fw["C"])
        t_bwd = time.time() - t0
        ratios = {}
        # per (Gaussian, tile): the deterministic form's entries
        grads = self.r.alloc_grads()
        gid, tile, vals = self.r.deterministic_entries(self.view, dLt, grads)
        torch.cuda.synchronize()
        gid, tile, vals = gid.cpu().numpy().astype(np.int64), tile.cpu().numpy().astype(np.int64), vals.cpu().numpy()
        rg = self.st["ranges"].astype(np.int64)
        pl = self.st["point_list"].astype(np.int64)
        cnt = rg[:, 1] - rg[:, 0]
        t_of = np.repeat(np.arange(rg.shape[0]), cnt)
        e_of = rg[t_of, 0] + np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt)
        key = t_of * self.P + pl[e_of]
        order = np.argsort(key, kind="stable")
        ks = key[order]
        q = tile * self.P + gid
        pos = np.minimum(np.searchsorted(ks, q), ks.size - 1)
        assert ks.size == 0 and q.size == 0 or (ks[pos] == q).all(), "an entry whose (Gaussian, tile) is in no list"
        e = e_of[order[pos]]
        assert np.unique(e).size == e.size, "two entries for one (Gaussian, tile)"
        got = np.zeros((pl.size, 9))
        got[e] = vals
        tile_e = np.zeros(pl.size, np.int64)
        tile_e[e_of] = t_of
        sel = np.isin(tile_e, fw["tiles"])
        ratios["entry"] = _max_by_key(rb.ratio(got[sel], bw["pair_v"][sel], rb.pair_bound(bw["pair_m"][sel])))
        info = dict(entries=int(np.isin(tile, fw["tiles"]).sum()), restated_nonzero=int(((bw["pair_v"] != 0).any(1) & sel).sum()),
                    walk_s=round(self.t_walk + t_bwd, 1))
        if forms:
            v, m, n = rb.per_gaussian(bw, pl, self.P)

            def per_gaussian(grads):
                return _max_by_key(rb.ratio(_two_d(grads), v, rb.pair_bound(m, FOLD + n)))
            for name, exact in (("atomic", False), ("exact", True)):
                grads = self.r.alloc_grads()
                for k in TWO_D:
                    grads[k].zero_()
                self.r.render_backward(self.view, dLt, grads, exact=exact)
                torch.cuda.synchronize()
                ratios[name] = per_gaussian(grads)
            grads = self.r.backward(self.gd, self.view, self.radii, dLt)
            torch.cuda.synchronize()
            ratios["backward"] = per_gaussian(grads)
            grads = self.r.backward(self.gd, self.view, self.radii, dLt, deterministic=True)
            torch.cuda.synchronize()
            ratios["deterministic"] = per_gaussian(grads)
        return ratios, info

    def paths(self):
        rg = self.st["ranges"].astype(np.int64)
        n = rg[:, 1] - rg[:, 0]
        return dict(self.fw["paths"], flagged=self.nflag, rounds=int((n.max() + 255) // 256) if n.size else 0,
                    span_count=self.d["span_count"], span_cap=self.d["span_cap"],
                    hy_fallback=hy_fallbacks(self.st["conic_opacity"], self.radii.cpu().numpy() > 0))


def _report(name, fwd, bwd, info, paths):
    print("\n%s\n    forward %s\n    %s\n    %s\n    paths %s" % (
        name, "  ".join("%s %.3f" % kv for kv in fwd.items()),
        "\n    ".join("%-13s %s" % (f, "  ".join("%s %.3f" % kv for kv in r.items())) for f, r in bwd.items()), info, paths))
    worst = max([max(fwd.values())] + [max(r.values()) for r in bwd.values()])
    assert worst <= 1.0, (name, fwd, bwd)


def run_case(name, g, cam, dL_kind="normal", seed=0, kind="", tiles=None, forms=True, pixel=None):
    c = Case(g, cam, tiles=tiles, kind=kind)
    fwd = c.check_forward()
    if dL_kind == "onehot" and pixel is None:
        return c
    bwd, info = c.check_backward(c.dL(dL_kind, seed, pixel), forms=forms)
    _report(name, fwd, bwd, info, c.paths())
    return c


@pytest.mark.parametrize("deg", [0, 1, 2, 3])
@pytest.mark.parametrize("view,pp", POSES, ids=["v%d-pp%g_%g" % (v, p[0], p[1]) for v, p in POSES])
def test_small_scene(deg, view, pp):
    g, cam = small_scene(deg=deg, view=view, pp=pp)
    run_case("small deg %d view %d pp %s" % (deg, view, pp), g, cam, seed=view)


PARITY = [((10000, 640, 480, 0, 42), POSES[0]), ((20000, 500, 300, 2, 7), POSES[3]), ((8000, 333, 211, 1, 5), POSES[4])]


@pytest.mark.parametrize("size,pose", PARITY, ids=["P%d-%dx%d" % s[0][:3] for s in PARITY])
def test_parity_sizes(size, pose):
    P, W, H, deg, seed = size
    g, cam = small_scene(P, W, H, seed, deg, view=pose[0], pp=pose[1])
    run_case("P %d %dx%d" % (P, W, H), g, cam, seed=seed)


@pytest.mark.parametrize("kind,opaque,view,pp", STRESS_CASES,
                         ids=["%s%s-v%d-pp%g_%g" % (k, "-high" if o else "", v, p[0], p[1]) for k, o, v, p in STRESS_CASES])
def test_stress_scene(kind, opaque, view, pp):
    from gaussian_lic_b200 import synthetic as syn
    g, cam = syn.make_stress_scene(kind, view=view, pp=pp, opaque=opaque)
    c = run_case("stress %s%s view %d pp %s" % (kind, "-high" if opaque else "", view, pp), g, cam, seed=view, kind=kind)
    p = c.paths()
    if kind == "big" and view == 0:
        assert p["span_count"] > p["span_cap"]
    if kind == "deep" and view == 0:
        assert p["rounds"] >= 8
    if kind == "needles":
        assert p["hy_fallback"] > 0
    if opaque or kind in ("big", "edges"):
        assert p["ended"] > 0


def test_opacity_at_threshold():
    """opacities just above 1/255: o G straddles 1/255 over most of every footprint, where the production backward decides
    from the exact expf"""
    g, cam = small_scene(P=20000, seed=5)
    rng = np.random.default_rng(5)
    g["opacity"] = (rng.uniform(1.0, 1.25, g["opacity"].shape) / 255.0).astype(np.float32)
    run_case("opacity at 1/255", g, cam, seed=5)


@pytest.mark.parametrize("W,H", [(1, 1), (7, 5), (17, 1), (1, 300), (333, 211), (2064, 1040)])
def test_frame_shapes(W, H):
    """driven by the fused loss's own dL/dimg"""
    from gaussian_lic_b200 import synthetic as syn
    g, cam = syn.make_frame_scene(W, H)
    run_case("frame %dx%d" % (W, H), g, cam, dL_kind="loss", seed=W + H)


@pytest.mark.parametrize("where", ["frame_corner", "tile_corner", "bucket_boundary"])
def test_one_hot(where):
    """dL/dpix one-hot at a single pixel, every other entry exactly zero: only the pairs of that pixel contribute"""
    g, cam = small_scene(view=1)
    c = Case(g, cam)
    c.check_forward()
    nc, ok = c.nc, ~c.flagged
    if where == "frame_corner":
        pix = (c.H - 1, c.W - 1) if ok[c.H - 1, c.W - 1] else (0, 0)
    elif where == "tile_corner":
        cand = [(y, x) for y in range(15, c.H, 16) for x in range(15, c.W, 16) if ok[y, x] and nc[y, x] > 0]
        pix = max(cand, key=lambda q: nc[q])
    else:       # the pixel's last taken splat closes a bucket: n_contrib a multiple of 32
        ys, xs = np.nonzero(ok & (nc > 0) & (nc % 32 == 0))
        assert ys.size > 0
        pix = (ys[0], xs[0])
    bwd, info = c.check_backward(c.dL("onehot", pixel=pix))
    info["pixel"], info["n_contrib"] = pix, int(nc[pix])
    _report("one-hot at %s" % where, c.check_forward(), bwd, info, c.paths())


def test_cfg2_sampled_tiles():
    """one cfg2 view (1920 x 1080, 500 k Gaussians) on the deepest tile, the four corners, edge tiles and 64 random tiles:
    the forward and the per-(Gaussian, tile) entries there"""
    from gaussian_lic_b200 import mapper as gmapper, synthetic as syn
    P, W, H, fx, fy, cx, cy, deg, _ = syn.CONFIGS["cfg2"]
    g, _ = syn.make_scene("cfg2")
    cam = gmapper.camera_block(W, H, fx, fy, cx, cy, *syn.orbit_pose(1, radius=0.25))
    gx, gy = (W + 15) // 16, (H + 15) // 16
    T = gx * gy

    def sample(ranges):
        rg = ranges.astype(np.int64)
        tiles = {int(np.argmax(rg[:, 1] - rg[:, 0])), 0, gx - 1, T - gx, T - 1, gx // 2, T - gx // 2 - 1, (gy // 2) * gx,
                 (gy // 2) * gx + gx - 1}
        tiles |= set(np.random.default_rng(0).choice(T, 64, replace=False).tolist())
        return np.array(sorted(tiles))
    c = run_case("cfg2 view 1, sampled tiles", g, cam, tiles=sample, forms=False)
    assert c.fw["tiles"].size >= 64
