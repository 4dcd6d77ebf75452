"""GPU parity on the stress scenes and on a sweep of frame shapes: CUDA path vs the CPU oracle.

Same checks and tolerances as test_gpu_parity.py (integer state bit-exact, images through image_close, gradients through
grad_close), on the scenes of synthetic.make_stress_scene -- needle-shaped splats, span-arena overflow, tiles of thousands
of splats, depth ties, view-edge culls and clamps (tests/test_stress_scenes.py checks that each reaches its path) -- and on
frames from 1 x 1 to the largest the library accepts, GLIC_MAX_TILES = 65 536 tiles.

The tensor-scale tolerances here absorb errors confined to a few pixels or pairs.  test_gpu_render_blend_exact.py pins the
same scenes per element: colour, T and n_contrib at every pixel, and the 2-D gradients per (Gaussian, tile) entry and per
Gaussian for every backward form, against a float64 restatement that walks every pair without the row cull.
"""
import numpy as np
import pytest

from helpers import GRAD_RTOL, POSES, big_rect_rows, grad_close, hy_fallbacks, image_close

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

GRADS = ("dL_dmeans2D", "dL_dconic", "dL_dopacity", "dL_dcolors", "dL_dmeans3D", "dL_dcov3D", "dL_ddc", "dL_dsh", "dL_dscales",
         "dL_drots")

# (kind, opaque, view, pp): every kind at the identity pose plus rotated / off-centre rig views where the scene stays meaningful
# (ties needs the identity pose, where depth = z exactly)
CASES = ([("needles", False) + p for p in (POSES[0], POSES[2], POSES[3])] +
         [("big", False) + p for p in (POSES[0], POSES[4], POSES[1])] +
         [("deep", False) + p for p in (POSES[0], POSES[3])] +
         [("deep", True) + p for p in (POSES[0], POSES[2])] +
         [("ties", False) + p for p in (POSES[0], POSES[4])] +
         [("edges", False) + p for p in (POSES[4], POSES[0], POSES[3])])
IDS = ["%s%s-v%d-pp%g_%g" % (k, "-high" if o else ("-low" if k == "deep" else ""), v, pp[0], pp[1]) for k, o, v, pp in CASES]


def render(g, cam):
    from gaussian_lic_b200 import ops
    r = ops.CRasterizer(cam["W"], cam["H"])
    gd = ops.scene_to_device(g)
    view = r.make_view(cam)
    color, T, radii = r.forward(gd, view)
    torch.cuda.synchronize()
    return r, gd, view, color, T, radii


def check_forward(r, color, T, radii, f, st, what=""):
    d = r.debug_state()
    assert r.R == f["R"] and d["R"] == f["R"], (r.R, d["R"], f["R"])
    assert r.B == f["B"] and d["B"] == f["B"], (r.B, d["B"], f["B"])
    np.testing.assert_array_equal(radii.cpu().numpy(), f["radii"])
    np.testing.assert_array_equal(d["tiles_touched"].cpu().numpy().astype(np.uint32), st["tiles_touched"])
    vis = f["radii"] > 0
    for k in ("depth", "xy", "conic_opacity"):
        np.testing.assert_array_equal(d[k].cpu().numpy().view(np.uint32)[vis], st[k].view(np.uint32)[vis], err_msg=k)
    np.testing.assert_array_equal(d["keys_sorted"].cpu().numpy().view(np.uint64), st["keys_sorted"])
    np.testing.assert_array_equal(d["point_list"].cpu().numpy().view(np.uint32), st["point_list"])
    np.testing.assert_array_equal(d["ranges"].cpu().numpy().view(np.uint32), st["ranges"])
    np.testing.assert_array_equal(d["bucket_offsets"].cpu().numpy().view(np.uint32), st["bucket_offsets"])
    np.testing.assert_allclose(d["rgb"].cpu().numpy()[vis], st["rgb"][vis], atol=2e-6, rtol=1e-5)
    image_close(color.cpu().numpy(), f["color"], what + "color")
    image_close(T.cpu().numpy(), f["final_T"], what + "final_T")
    nc = d["n_contrib"].cpu().numpy().view(np.uint32)
    assert (nc != st["n_contrib"]).mean() < 1e-4
    return d


NEEDLE_UNSTABLE = ("dL_dmeans3D", "dL_dcov3D", "dL_dscales", "dL_drots")


def f32_formula_unstable(b32, b64):
    """True when the f32 oracle's dL_dmeans3D misses the f64 oracle's by more than GRAD_RTOL of the tensor's scale.  For
    needle-shaped splats the reference's f32 chain from dL/dcov2D back to the 3-D parameters (terms ~ s_long^2 against a
    result ~ 1) cancels catastrophically: measured on the needle scene, the f32 oracle misses the f64 dL_dmeans3D by 2e-2
    (identity pose) to 10 (rig view 3) times the tensor's scale, and the CUDA path by as much with its own rounding; dL_dcov3D,
    dL_dscales and dL_drots inherit the same cancellation.  Neither f32 evaluation can pin the other there, so those four are
    not compared with the f32 oracle on this scene; the 2-D gradients (where the render kernels and the hy fallback act),
    opacity and colour gradients still are.  test_gpu_preprocess_backward_exact.py pins those four at every row instead:
    against a float64 restatement fed the kernel's own 2-D gradients, each element within a bound that grows exactly as
    far as the f32 cancellation can go."""
    a, r = b32["dL_dmeans3D"].astype(np.float64), b64["dL_dmeans3D"].astype(np.float64)
    return np.abs(a - r).max() > GRAD_RTOL * np.abs(r).max()


def check_backward(grads, b, f, what="", skip=()):
    for k in GRADS:
        a = grads[k].cpu().numpy()
        if a.size and k not in skip:
            grad_close(a.reshape(b[k].shape), b[k], what + k)
    inv = f["radii"] <= 0          # culled Gaussians get exact zeros (rasterize_points.cu:192-201 semantics)
    for k in ("dL_dmeans3D", "dL_dscales", "dL_drots", "dL_dsh", "dL_ddc", "dL_dcov3D", "dL_dopacity"):
        a = grads[k].cpu().numpy()
        if a.size:
            assert not a[inv].any(), k


def path_counters(d, f, st):
    """what the stress scene exercised on the GPU (printed; the PR / run log records them)"""
    rg = st["ranges"].astype(np.int64)
    per_tile = rg[:, 1] - rg[:, 0]
    mc = d["max_contrib"].cpu().numpy().astype(np.int64)
    return dict(span_count=d["span_count"], span_cap=d["span_cap"], max_splats_per_tile=int(per_tile.max()),
                rounds=int((per_tile.max() + 255) // 256), B=f["B"], live_buckets=int(((mc + 31) // 32).sum()),
                hy_fallback=hy_fallbacks(d["conic_opacity"].cpu().numpy(), f["radii"] > 0))


@pytest.mark.parametrize("kind,opaque,view,pp", CASES, ids=IDS)
def test_stress_matches_oracle(oracle32, oracle64, kind, opaque, view, pp):
    from gaussian_lic_b200 import synthetic as syn
    g, cam = syn.make_stress_scene(kind, view=view, pp=pp, opaque=opaque)
    r, gd, v, color, T, radii = render(g, cam)
    f = oracle32.forward(g, cam)
    st = oracle32.state(f)
    d = check_forward(r, color, T, radii, f, st)
    c = path_counters(d, f, st)
    print("path counters %s: %s" % (kind + ("-high" if opaque else ""), c))
    if kind == "big" and view == 0:
        # the arena overflowed part-way through: some rects stored spans, the later ones had their rows recomputed
        assert c["span_count"] > c["span_cap"] and big_rect_rows(st["xy"], f["radii"], cam["W"], cam["H"]) > c["span_cap"]
    if kind == "deep" and view == 0:
        assert c["rounds"] >= 8
    dL = np.random.default_rng(view).normal(size=(3, cam["H"], cam["W"])).astype(np.float32)
    grads = r.backward(gd, v, radii, torch.as_tensor(dL).cuda())
    torch.cuda.synchronize()
    b = oracle32.backward(f, dL)
    skip = ()
    if kind == "needles":
        f64 = oracle64.forward(g, cam)
        assert f32_formula_unstable(b, oracle64.backward(f64, dL))    # still true, else compare dL_dmeans3D again
        oracle64.free(f64)
        skip = NEEDLE_UNSTABLE
    check_backward(grads, b, f, skip=skip)
    oracle32.free(f)


@pytest.mark.parametrize("kind,view,pp", [("needles", 0, (0.0, 0.0)), ("big", 0, (0.0, 0.0)), ("big", 5, (17.5, -9.25))])
def test_stress_torch_shim_matches_oracle(oracle32, oracle64, kind, view, pp):
    """the reference-facing LibTorch shim (RasterizeGaussiansCUDA / RasterizeGaussiansBackwardCUDA through autograd)"""
    from gaussian_lic_b200 import ops, synthetic as syn
    g, cam = syn.make_stress_scene(kind, view=view, pp=pp)
    t = lambda a: torch.as_tensor(a, dtype=torch.float32).cuda()
    leaves = dict(means=t(g["means"]), op=t(g["opacity"]).view(-1, 1), dc=t(g["dc"]).view(-1, 1, 3), sh=t(g["sh"]),
                  scales=t(g["scales"]), rots=t(g["rots"]))
    for x in leaves.values():
        x.requires_grad_(True)
    rs = ops.GaussianRasterizationSettings(cam["H"], cam["W"], cam["tanfovx"], cam["tanfovy"], *[float(x) for x in cam["lims"]],
                                           torch.zeros(3, device="cuda"), 1.0, t(cam["view"]).view(4, 4), t(cam["proj"]).view(4, 4),
                                           g["degree"], t(cam["campos"]))
    means2D = torch.zeros_like(leaves["means"], requires_grad=True)
    color, radii, final_T = ops.GaussianRasterizer(rs)(leaves["means"], means2D, leaves["op"], leaves["dc"], leaves["sh"],
                                                       leaves["scales"], leaves["rots"])
    dL = np.random.default_rng(5).normal(size=(3, cam["H"], cam["W"])).astype(np.float32)
    (color * t(dL)).sum().backward()
    torch.cuda.synchronize()
    f = oracle32.forward(g, cam)
    b = oracle32.backward(f, dL)
    np.testing.assert_array_equal(radii.cpu().numpy(), f["radii"])
    image_close(color.detach().cpu().numpy(), f["color"], "shim color")
    image_close(final_T.cpu().numpy(), f["final_T"], "shim final_T")
    skip = ()
    if kind == "needles":
        f64 = oracle64.forward(g, cam)
        assert f32_formula_unstable(b, oracle64.backward(f64, dL))
        oracle64.free(f64)
        skip = NEEDLE_UNSTABLE
    for name, k in (("means", "dL_dmeans3D"), ("op", "dL_dopacity"), ("dc", "dL_ddc"), ("sh", "dL_dsh"), ("scales", "dL_dscales"),
                    ("rots", "dL_drots")):
        if k not in skip:
            grad_close(leaves[name].grad.cpu().numpy().reshape(b[k].shape), b[k], "shim " + k)
    oracle32.free(f)


# ---- frame shapes -----------------------------------------------------------------------------------------------------------
# narrower / shorter than a tile, 1 pixel wide or tall, odd sizes, T = 8192 (one full sweep of the tile scans, 14 key bits),
# T = 8385 (a second sweep), T = 32 400 (15 bits) and T = 65 536 (16 bits: the largest frame)
FRAMES = [(1, 1), (7, 5), (16, 16), (17, 1), (1, 300), (333, 211), (2048, 1024), (2064, 1040), (3840, 2160), (4096, 4096)]


def _gt(W, H):
    return np.random.default_rng(W * 7919 + H).random((3, H, W), dtype=np.float32)


@pytest.mark.parametrize("W,H", FRAMES, ids=["%dx%d" % s for s in FRAMES])
def test_frame_shapes_match_oracle(oracle32, W, H):
    from gaussian_lic_b200 import ops, synthetic as syn
    g, cam = syn.make_frame_scene(W, H)
    r, gd, v, color, T, radii = render(g, cam)
    f = oracle32.forward(g, cam)
    st = oracle32.state(f)
    check_forward(r, color, T, radii, f, st, "%dx%d " % (W, H))
    # the fused L1 + SSIM loss of the rendered frame (also frames smaller than the 11-tap window)
    gt = _gt(W, H)
    loss, dl = r.loss(color, torch.as_tensor(gt).cuda())
    torch.cuda.synchronize()
    L, dl_ref = oracle32.loss(f["color"], gt)
    assert abs(float(loss.item()) - L) < 2e-5, (float(loss.item()), L)
    grad_close(dl.cpu().numpy(), dl_ref, "dL_dimg (fused loss)", rtol=1e-4)
    # the backward, driven by the loss gradient of the CUDA path (the same input for both sides)
    dL = dl.cpu().numpy()
    grads = r.backward(gd, v, radii, dl)
    torch.cuda.synchronize()
    check_backward(grads, oracle32.backward(f, dL), f, "%dx%d " % (W, H))
    oracle32.free(f)


@pytest.mark.parametrize("W,H", [(1, 1), (7, 5), (17, 1), (1, 300), (333, 211), (2064, 1040)])
def test_fused_ssim_frame_shapes(oracle32, W, H):
    from gaussian_lic_b200 import ops
    rng = np.random.default_rng(W + 3 * H)
    a = rng.random((1, 3, H, W), dtype=np.float32)
    b = np.clip(a + 0.1 * rng.normal(size=a.shape).astype(np.float32), 0, 1)
    ta, tb = torch.as_tensor(a).cuda(), torch.as_tensor(b).cuda()
    m, d1, d2, d3 = ops.fusedssim(ops.SSIM_C1, ops.SSIM_C2, ta, tb, True)
    om, o1, o2, o3 = oracle32.ssim(a[0], b[0])
    np.testing.assert_allclose(m.cpu().numpy()[0], om, atol=2e-5)
    for x, y, n in ((d1, o1, "dm_dmu1"), (d2, o2, "dm_dsigma1_sq"), (d3, o3, "dm_dsigma12")):
        grad_close(x.cpu().numpy()[0], y, n, rtol=1e-4)
    dmap = rng.normal(size=a.shape).astype(np.float32)
    gi = ops.fusedssim_backward(ops.SSIM_C1, ops.SSIM_C2, ta, tb, torch.as_tensor(dmap).cuda(), d1, d2, d3)
    og = oracle32.ssim_backward(a[0], b[0], dmap[0], o1, o2, o3)
    grad_close(gi.cpu().numpy()[0], og, "dL_dimg1", rtol=1e-4)


def test_frame_size_limit_refused_before_any_launch(oracle32):
    """More than GLIC_MAX_TILES tiles is refused by the view check, before anything is enqueued; the same rasterizer then
    renders a valid frame exactly."""
    from gaussian_lic_b200 import capi, ops, synthetic as syn
    g, cam = syn.make_frame_scene(333, 211)
    r = ops.CRasterizer(cam["W"], cam["H"])
    gd = ops.scene_to_device(g)
    good = r.make_view(cam)
    for W, H in ((4112, 4112), (4097, 4096), (65536 * 16 + 1, 16)):
        bad = capi.View(good.viewmatrix, good.projmatrix, good.campos, good.tan_fovx, good.tan_fovy, good.limx_neg,
                        good.limx_pos, good.limy_neg, good.limy_pos, W, H)
        n0 = capi.launch_count()
        with pytest.raises(capi.GlicError, match="GLIC_MAX_TILES"):
            r.forward(gd, bad)
        assert capi.launch_count() == n0
    color, T, radii = r.forward(gd, good)
    f = oracle32.forward(g, cam)
    assert (r.R, r.B) == (f["R"], f["B"])
    np.testing.assert_array_equal(radii.cpu().numpy(), f["radii"])
    image_close(color.cpu().numpy(), f["color"], "color after a refused frame")
    image_close(T.cpu().numpy(), f["final_T"], "final_T after a refused frame")
    oracle32.free(f)
