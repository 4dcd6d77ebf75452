"""csrc/preprocess_backward.cu against the float64 restatement of tests/preprocess_backward_reference.py at every row of
every output, each element against its own bound |got - v| <= c * 2^-24 * m (c per output in
preprocess_backward_reference.BOUND, m the restatement's magnitude).

Given its 2-D inputs the per-Gaussian backward is a fixed float32 computation per row, so the restatement takes the
kernel's own inputs -- the render backward's dL/dmean2D, dL/dconic and dL/dcolour, the forward's radii and clamp bits --
and the render backward's float atomics are out of the comparison.  There is no outlier fraction and no tolerance relative
to the tensor's maximum: a bug confined to a few rows fails.  Rows whose branch quantity lies within its rounding of a
threshold (the frustum masks, the effective-rank branch, normalize's guard) may take either side and are held to either
value; each case asserts that only a few rows are there.

1. The reference-facing nine-tensor form through glic_backward (ops.CRasterizer.backward): dL_dmeans3D, dL_dcov3D, dL_ddc,
   dL_dsh, dL_dscales, dL_drots; culled rows exact zeros.  small_scene at SH degrees 0-3 x POSES; every stress scene at the
   poses test_gpu_stress.py uses, the needles included (whose four 3-D gradients no float32 evaluation can pin to another,
   but which hold to the restatement's bound); P in {1, 31, 33, 127, 129, 4097} for the warp and CTA tails of the SH slab;
   a cfg2 view; SH degree D below the SH tensor's (D in {0, 1, 2}, M = 15); M = 0; lambda_erank = 0.25 on both sides of its
   branch; scale_modifier 0.5 and 1.7.
2. The mapper's compact + pose form through glic_debug_pose_backward: the 11 floats of every row with respect to the raw
   parameters and the six pose floats, driven by the render backward's outputs and by synthetic 2-D gradients of 1e-6 .. 1e3
   with exact zeros, with raw rotations of norm 1e-13 .. 1e3 and opacities at 0 and 1.  The pose bound is the sum of the
   rows' bounds.

Each case prints the rows that took each path it is there for and asserts they are not zero.  Run with -s to see
max(err / bound) per output.
"""
import ctypes as C

import numpy as np
import pytest

import preprocess_backward_reference as pbr
from helpers import CFG2_P, POSES, small_scene
from preprocess_backward_reference import BOUND
from test_gpu_stress import CASES as STRESS_CASES
from test_preprocess_backward_reference_host import cams, erank_scales, grads2d, outside_rows

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

DEV = "cuda:0"
NINE = ("dmeans3D", "dcov3D", "ddc", "dsh", "dscales", "drots")
COMPACT = ("g_xyz", "g_scale", "g_rot", "g_opacity")


def _report(name, ratios, paths):
    print("\n%s: %s\n    paths %s" % (name, "  ".join("%s %.3f" % kv for kv in sorted(ratios.items())), paths))
    assert max(ratios.values()) <= 1.0, ratios


def _band_rows(ref, on_clamps):
    """rows within rounding of a branch threshold: a handful, except in the edges scene, which puts about 1/20 of its rows
    exactly on the lim* clamps (on_clamps)"""
    rows = np.any(list(ref["band"].values()), 0)
    assert rows.sum() <= max(8, (0.06 if on_clamps else 0.0) * ref["paths"]["rows"]), (rows.sum(), ref["paths"])
    return rows


def _forward(g, cam, mod=1.0):
    from gaussian_lic_b200 import ops
    r = ops.CRasterizer(cam["W"], cam["H"])
    gd = ops.scene_to_device(g)
    view = r.make_view(cam)
    _, _, radii = r.forward(gd, view, scale_modifier=mod)
    torch.cuda.synchronize()
    clamped = r.debug_state()["clamped"].cpu().numpy()
    return r, gd, view, radii, clamped


# ---- 1. the nine-tensor form ------------------------------------------------------------------------------------------------
def check_nine(g, cam, mod=1.0, lam=0.0, seed=0, on_clamps=False):
    r, gd, view, radii, clamped = _forward(g, cam, mod)
    dL = np.random.default_rng(seed).normal(size=(3, cam["H"], cam["W"])).astype(np.float32)
    grads = r.backward(gd, view, radii, torch.as_tensor(dL).to(DEV), scale_modifier=mod, lambda_erank=lam)
    torch.cuda.synchronize()
    got = {k: grads["dL_" + k].cpu().numpy() for k in NINE}
    d2 = [grads[k].cpu().numpy() for k in ("dL_dmeans2D", "dL_dconic", "dL_dcolors")]
    radii = radii.cpu().numpy()
    c32, _ = cams(cam)
    ref = pbr.backward(g, c32, radii, clamped, *d2, mod=mod, lambda_erank=lam)
    alt = pbr.backward(g, c32, radii, clamped, *d2, mod=mod, lambda_erank=lam, flip=ref["band"])
    band = _band_rows(ref, on_clamps)
    culled = radii <= 0
    for k in NINE:
        a = got[k].reshape(ref[k].v.shape)
        assert not a[culled].any(), k                                  # culled rows: exact zeros
    ratios = {k: pbr.either_ratio(got[k], ref[k], alt[k], BOUND[k], band) for k in NINE}
    paths = dict(ref["paths"], band=int(band.sum()), culled=int(culled.sum()), partial_warp=len(radii) % 32)
    return ratios, paths


@pytest.mark.parametrize("deg", [0, 1, 2, 3])
@pytest.mark.parametrize("view,pp", POSES, ids=["v%d-pp%g_%g" % (v, p[0], p[1]) for v, p in POSES])
def test_small_scene(deg, view, pp):
    g, cam = small_scene(deg=deg, view=view, pp=pp)
    ratios, paths = check_nine(g, cam, seed=view)
    _report("small deg %d view %d pp %s" % (deg, view, pp), ratios, paths)
    if deg > 0:
        assert min(paths["clamped_%d" % ch] for ch in range(3)) > 0


@pytest.mark.parametrize("kind,opaque,view,pp", STRESS_CASES)
def test_stress_scene(kind, opaque, view, pp):
    from gaussian_lic_b200 import synthetic as syn
    g, cam = syn.make_stress_scene(kind, view=view, pp=pp, opaque=opaque)
    ratios, paths = check_nine(g, cam, seed=view, on_clamps=kind == "edges")
    _report("stress %s%s view %d pp %s" % (kind, "-high" if opaque else "", view, pp), ratios, paths)
    assert min(paths["clamped_%d" % ch] for ch in range(3)) > 0


@pytest.mark.parametrize("P", [1, 31, 33, 127, 129, 4097])
def test_warp_and_cta_tails(P):
    """the SH slab of a last, partial warp (wcnt < 32) and of a last, partial CTA, at degree 3 (K = 45 floats a row)"""
    g, cam = small_scene(P=P, deg=3, zmax=6.0, log_scale_mean=-2.0)
    ratios, paths = check_nine(g, cam, seed=P)
    _report("P %d" % P, ratios, paths)
    assert paths["rows"] > 0 and paths["partial_warp"] == P % 32


def test_cfg2_view():
    from gaussian_lic_b200 import synthetic as syn
    g, cam = syn.make_scene("cfg2", P=CFG2_P, view=5, pp=(41.5, -27.25))
    ratios, paths = check_nine(g, cam, seed=2)
    _report("cfg2 view 5", ratios, paths)
    assert min(paths["clamped_%d" % ch] for ch in range(3)) > 0


@pytest.mark.parametrize("D", [0, 1, 2])
def test_sh_degree_below_the_tensor(D):
    """sh_rest_count(D) < M = 15: the rows of dL_dsh past the degree are zeros, and only the first coefficients enter"""
    g, cam = small_scene(deg=3, view=1)
    g["degree"] = D
    ratios, paths = check_nine(g, cam, seed=D)
    _report("degree %d of M = 15" % D, ratios, paths)


def test_no_sh_rest():
    """M = 0: no colour backward, dL_ddc zero (the reference's `if (shs)`)"""
    g, cam = small_scene(deg=0, view=3)
    assert g["sh"].shape[1] == 0
    ratios, paths = check_nine(g, cam, seed=3)
    _report("M = 0", ratios, paths)


@pytest.mark.parametrize("kind", ["small", "needles", "edges"])
def test_effective_rank_regulariser(kind):
    from gaussian_lic_b200 import synthetic as syn
    g, cam = small_scene(deg=2, view=1) if kind == "small" else syn.make_stress_scene(kind, view=0)
    erank_scales(g, 7)
    ratios, paths = check_nine(g, cam, lam=0.25, seed=7, on_clamps=kind == "edges")
    _report("lambda_erank 0.25 %s" % kind, ratios, paths)
    assert paths["erank_in"] > 0 and paths["erank_out"] > 0


@pytest.mark.parametrize("mod", [0.5, 1.7])
@pytest.mark.parametrize("kind", ["small", "needles"])
def test_scale_modifier(kind, mod):
    from gaussian_lic_b200 import synthetic as syn
    g, cam = small_scene(deg=3, view=5, pp=(17.5, -9.25)) if kind == "small" else syn.make_stress_scene(kind, view=3, deg=3)
    ratios, paths = check_nine(g, cam, mod=mod, seed=11)
    _report("scale_modifier %g %s" % (mod, kind), ratios, paths)


# ---- 2. the compact + pose form ------------------------------------------------------------------------------------------------
def check_compact(g, cam, synthetic, seed, on_clamps=False):
    from gaussian_lic_b200 import capi
    rng = np.random.default_rng(seed)
    P = g["means"].shape[0]
    g = dict(g)
    op = g["opacity"].astype(np.float32).copy()
    pick = rng.random(P)
    op[pick < 0.05] = np.float32(1e-7)                                  # opacities at 0 and 1
    op[(pick >= 0.05) & (pick < 0.1)] = np.nextafter(np.float32(1), np.float32(0))
    op[(pick >= 0.1) & (pick < 0.12)] = np.float32(1)
    g["opacity"] = op
    r, gd, view, radii, clamped = _forward(g, cam)
    if synthetic:
        d2 = list(grads2d(P, seed))
        d2[1] = np.stack([d2[1][:, 0], d2[1][:, 1], np.zeros(P, np.float32), d2[1][:, 2]], 1)
        dop = (rng.normal(size=P) * 10.0 ** rng.uniform(-6.0, 3.0, P)).astype(np.float32)
        dev = [torch.as_tensor(a).to(DEV).contiguous() for a in d2 + [dop]]
    else:
        dL = torch.as_tensor(rng.normal(size=(3, cam["H"], cam["W"])).astype(np.float32)).to(DEV)
        grads = r.alloc_grads()
        for k in ("dL_dmeans2D", "dL_dconic", "dL_dopacity", "dL_dcolors"):
            grads[k].zero_()
        r.render_backward(view, dL, grads)
        torch.cuda.synchronize()
        dev = [grads[k] for k in ("dL_dmeans2D", "dL_dconic", "dL_dcolors", "dL_dopacity")]
    norms = 10.0 ** rng.uniform(-13.0, 3.0, P)
    rot_raw = (g["rots"] * norms[:, None]).astype(np.float32)
    tr = torch.as_tensor(rot_raw).to(DEV)
    M = r.M
    part = torch.empty((P + 127) // 128 * 6, dtype=torch.float64, device=DEV)
    geo = torch.full((11 * P,), float("nan"), dtype=torch.float32, device=DEV)
    pose6 = torch.full((6,), float("nan"), dtype=torch.float32, device=DEV)
    capi.check(capi.lib.glic_debug_pose_backward(
        P, int(g["degree"]), M, capi.ptr(gd["means"]), capi.ptr(gd["scales"]), capi.ptr(gd["rots"]), capi.ptr(tr),
        capi.ptr(gd["opacity"]), capi.ptr(gd["sh"]) if M else None, C.byref(view), capi.ptr(radii), capi.ptr(r.geom_ws),
        capi.ptr(dev[0]), capi.ptr(dev[1]), capi.ptr(dev[3]), capi.ptr(dev[2]), 0, capi.ptr(geo), capi.ptr(part),
        capi.ptr(pose6), None), "debug_pose_backward")
    torch.cuda.synchronize()
    geo = geo.cpu().numpy()
    got = dict(g_rot=geo[:4 * P].reshape(P, 4), g_xyz=geo[4 * P:7 * P].reshape(P, 3), g_scale=geo[7 * P:10 * P].reshape(P, 3),
               g_opacity=geo[10 * P:])
    d2 = [t.cpu().numpy() for t in dev]
    radii = radii.cpu().numpy()
    c32, _ = cams(cam)
    compact = dict(opacity=op, dL_dopacity=d2[3], rot_raw=rot_raw)
    kw = dict(compact=compact, pose=True)
    ref = pbr.backward(g, c32, radii, clamped, *d2[:3], **kw)
    alt = pbr.backward(g, c32, radii, clamped, *d2[:3], flip=ref["band"], **kw)
    band = _band_rows(ref, on_clamps)
    culled = radii <= 0
    for k in COMPACT:
        assert not got[k].reshape(P, -1)[culled].any(), k
    ratios = {k: pbr.either_ratio(got[k], ref[k], alt[k], BOUND[k], band) for k in COMPACT}
    # the pose floats: the sum of the rows' float32 terms, added in float64; the bound is the sum of the rows' bounds, and a
    # row in a band may contribute either of its values
    jump = np.abs(alt["pose_rows"].v - ref["pose_rows"].v)[band].sum(0)
    p6 = pose6.cpu().numpy().astype(np.float64)
    ratios["pose"] = float(np.max(np.abs(p6 - ref["pose"].v) / (BOUND["pose"] * pbr.U * ref["pose"].m + jump)))
    assert np.isfinite(p6).all()
    paths = dict(ref["paths"], band=int(band.sum()), culled=int(culled.sum()),
                 opacity_0_1=int(((op <= 1e-7) | (op >= np.nextafter(np.float32(1), np.float32(0))))[~culled].sum()))
    return ratios, paths


COMPACT_CASES = [("small", 3, 1, POSES[1]), ("small", 0, 0, POSES[3]), ("small", 1, 0, POSES[4]), ("needles", 2, 0, POSES[2]),
                 ("edges", 3, 1, POSES[0]), ("outside", 3, 0, POSES[0]), ("outside", 2, 1, POSES[3])]


@pytest.mark.parametrize("synthetic", [False, True], ids=["render", "synthetic"])
@pytest.mark.parametrize("kind,deg,seed,pose", COMPACT_CASES,
                         ids=["%s-d%d-v%d" % (k, d, p[0]) for k, d, s, p in COMPACT_CASES])
def test_compact_and_pose(kind, deg, seed, pose, synthetic):
    from gaussian_lic_b200 import synthetic as syn
    view, pp = pose
    if kind == "small":
        g, cam = small_scene(deg=deg, view=view, pp=pp)
    else:
        g, cam = syn.make_stress_scene("edges" if kind == "outside" else kind, view=view, pp=pp, deg=deg)
        if kind == "outside":
            g = outside_rows(g, cam)
    ratios, paths = check_compact(g, cam, synthetic, seed=17 * seed + view + (100 if synthetic else 0), on_clamps=kind == "edges")
    _report("compact + pose %s deg %d view %d %s" % (kind, deg, view, "synthetic" if synthetic else "render"), ratios, paths)
    assert paths["nn_small"] > 0 and paths["opacity_0_1"] > 0
    if kind != "small":
        assert paths["xmask0"] > 0 and paths["ymask0"] > 0
