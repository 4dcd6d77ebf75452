"""GPU parity tests: CUDA path (through the C ABI and through the LibTorch shim) vs the CPU oracle.

Bit-exact: radii, tiles_touched, R, B, sorted (tile|depth) list, tile ranges, bucket offsets.
Tolerance (1e-4 abs, see helpers.py): colour, transmittance; gradients relative to tensor scale.
"""
import numpy as np
import pytest

from helpers import POSES, grad_close, image_close, small_scene

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


def _run_cuda(g, cam, no_color=False):
    from gaussian_lic_b200 import ops
    r = ops.CRasterizer(cam["W"], cam["H"])
    gd = ops.scene_to_device(g)
    view = r.make_view(cam)
    color, T, radii = r.forward(gd, view, no_color=no_color)
    torch.cuda.synchronize()
    return r, gd, view, color, T, radii


@pytest.mark.parametrize("view,pp", POSES)
@pytest.mark.parametrize("P,W,H,deg,seed", [(3000, 320, 208, 3, 11), (10000, 640, 480, 0, 42), (20000, 500, 300, 2, 7)])
def test_forward_matches_oracle(oracle32, P, W, H, deg, seed, view, pp):
    g, cam = small_scene(P, W, H, seed, deg, view=view, pp=pp)
    r, gd, view, color, T, radii = _run_cuda(g, cam)
    f = oracle32.forward(g, cam)
    st = oracle32.state(f)
    d = r.debug_state()
    assert r.R == f["R"], (r.R, f["R"])
    assert d["R"] == f["R"] and d["B"] == f["B"] and r.B == f["B"], (d["R"], d["B"], f["R"], f["B"])
    np.testing.assert_array_equal(radii.cpu().numpy(), f["radii"])
    np.testing.assert_array_equal(d["tiles_touched"].cpu().numpy().astype(np.uint32), st["tiles_touched"])
    vis = f["radii"] > 0
    np.testing.assert_array_equal(d["depth"].cpu().numpy().view(np.uint32)[vis], st["depth"].view(np.uint32)[vis])
    np.testing.assert_array_equal(d["xy"].cpu().numpy().view(np.uint32)[vis], st["xy"].view(np.uint32)[vis])
    np.testing.assert_array_equal(d["conic_opacity"].cpu().numpy().view(np.uint32)[vis], st["conic_opacity"].view(np.uint32)[vis])
    np.testing.assert_array_equal(d["keys_sorted"].cpu().numpy().view(np.uint64), st["keys_sorted"])
    np.testing.assert_array_equal(d["point_list"].cpu().numpy().view(np.uint32), st["point_list"])
    np.testing.assert_array_equal(d["ranges"].cpu().numpy().view(np.uint32), st["ranges"])
    np.testing.assert_array_equal(d["bucket_offsets"].cpu().numpy().view(np.uint32), st["bucket_offsets"])
    np.testing.assert_allclose(d["rgb"].cpu().numpy()[vis], st["rgb"][vis], atol=2e-6, rtol=1e-5)
    image_close(color.cpu().numpy(), f["color"], "color")
    image_close(T.cpu().numpy(), f["final_T"], "final_T")
    nc = d["n_contrib"].cpu().numpy().view(np.uint32)
    assert (nc != st["n_contrib"]).mean() < 1e-4
    oracle32.free(f)


def test_forward_no_color(oracle32):
    g, cam = small_scene(4000, 320, 208, 3, 3)
    r, gd, view, color, T, radii = _run_cuda(g, cam, no_color=True)
    f = oracle32.forward(g, cam, no_color=True)
    assert r.R == f["R"] and r.B == 0 and f["B"] == 0
    np.testing.assert_array_equal(radii.cpu().numpy(), f["radii"])
    image_close(T.cpu().numpy(), f["final_T"], "final_T(no_color)")
    oracle32.free(f)


@pytest.mark.parametrize("view,pp", POSES)
@pytest.mark.parametrize("P,W,H,deg,seed", [(3000, 320, 208, 3, 11), (10000, 640, 480, 0, 42), (8000, 333, 211, 1, 5)])
def test_backward_matches_oracle(oracle32, P, W, H, deg, seed, view, pp):
    g, cam = small_scene(P, W, H, seed, deg, view=view, pp=pp)
    r, gd, view, color, T, radii = _run_cuda(g, cam)
    rng = np.random.default_rng(seed)
    dL = rng.normal(size=(3, H, W)).astype(np.float32)
    grads = r.backward(gd, view, radii, torch.as_tensor(dL).cuda())
    torch.cuda.synchronize()
    f = oracle32.forward(g, cam)
    b = oracle32.backward(f, dL)
    for k_cuda, k_or in [("dL_dmeans2D", "dL_dmeans2D"), ("dL_dconic", "dL_dconic"), ("dL_dopacity", "dL_dopacity"),
                         ("dL_dcolors", "dL_dcolors"), ("dL_dmeans3D", "dL_dmeans3D"), ("dL_dcov3D", "dL_dcov3D"),
                         ("dL_ddc", "dL_ddc"), ("dL_dsh", "dL_dsh"), ("dL_dscales", "dL_dscales"), ("dL_drots", "dL_drots")]:
        a = grads[k_cuda].cpu().numpy()
        if a.size == 0:
            continue
        grad_close(a.reshape(b[k_or].shape), b[k_or], k_cuda)
    # culled Gaussians get exact zeros in every output (rasterize_points.cu:192-201 semantics)
    inv = f["radii"] <= 0
    for k in ("dL_dmeans3D", "dL_dscales", "dL_drots", "dL_dsh", "dL_ddc", "dL_dcov3D", "dL_dopacity"):
        a = grads[k].cpu().numpy()
        if a.size:
            assert not a[inv].any(), k
    oracle32.free(f)


def test_empty_and_tiny_inputs():
    from gaussian_lic_b200 import ops
    W, H = 64, 48
    g, cam = small_scene(1, W, H, 1, 3)
    r, gd, view, color, T, radii = _run_cuda(g, cam)
    assert torch.isfinite(color).all() and torch.isfinite(T).all()
    # P = 0 through the LibTorch shim (rasterize_points.cu:110: zero outputs, R = B = 0)
    z = lambda *s: torch.zeros(*s, device="cuda")
    out = ops.RasterizeGaussiansCUDA(z(3), z(0, 3), z(0), z(0, 1), z(0, 3), z(0, 4), 1.0, z(0),
                                     torch.as_tensor(cam["view"]).cuda().view(4, 4), torch.as_tensor(cam["proj"]).cuda().view(4, 4),
                                     cam["tanfovx"], cam["tanfovy"], H, W, *[float(x) for x in cam["lims"]],
                                     z(0, 1, 3), z(0, 15, 3), 3, torch.as_tensor(cam["campos"]).cuda(), False, False, False)
    assert out[0] == 0 and out[1] == 0 and not out[2].any() and not out[3].any()
    with pytest.raises(RuntimeError):
        ops.RasterizeGaussiansCUDA(z(3), z(5, 2), z(0), z(5, 1), z(5, 3), z(5, 4), 1.0, z(0),
                                   torch.as_tensor(cam["view"]).cuda(), torch.as_tensor(cam["proj"]).cuda(),
                                   cam["tanfovx"], cam["tanfovy"], H, W, *[float(x) for x in cam["lims"]],
                                   z(5, 1, 3), z(5, 15, 3), 3, torch.as_tensor(cam["campos"]).cuda(), False, False, False)


def test_empty_scene_outputs_of_every_draw():
    """P = 0 through the five draw entry points of the C ABI: every output plane, the host counters, the image header and the
    launches, starting from NaN planes, junk counters and a junk header.  glic_render writes T = 1 (nothing covers a pixel); the
    others write T = 0 as rasterize_points.cu:110 does."""
    import ctypes as C
    from gaussian_lic_b200 import capi
    lib = capi.lib
    W, H = 64, 48
    _, cam = small_scene(1, W, H, 1, 3)
    dev = "cuda"
    t = lambda a: torch.as_tensor(a, dtype=torch.float32).to(dev)
    vm, pm, cp = t(cam["view"]), t(cam["proj"]), t(cam["campos"])
    lims = [float(x) for x in cam["lims"]]
    view = capi.View(vm.data_ptr(), pm.data_ptr(), cp.data_ptr(), cam["tanfovx"], cam["tanfovy"], *lims, W, H)
    ws = lambda n: torch.empty(max(int(n), 16), dtype=torch.uint8, device=dev)
    geom, image = ws(lib.glic_geom_bytes(0)), ws(lib.glic_image_bytes(W, H))
    binning, sample = ws(lib.glic_binning_bytes(64)), ws(lib.glic_sample_bytes(64, W, H))
    nan = lambda *s: torch.full(s, float("nan"), device=dev)
    JUNK = -7

    def run(call):
        image.fill_(0xFF)                                 # the header reads num_rendered = -1, num_buckets = 2^32 - 1
        counters = (C.c_int64 * 3)(JUNK, JUNK, JUNK)
        host = C.c_int64(JUNK)
        torch.cuda.synchronize()
        before = lib.glic_launch_count()
        assert call(counters, host) == 0, lib.glic_last_error()
        torch.cuda.synchronize()
        hdr = (C.c_int64 * 2)()
        assert lib.glic_debug_image(W, H, image.data_ptr(), None, None, None, None, hdr, None) == 0
        torch.cuda.synchronize()
        return lib.glic_launch_count() - before, list(counters), host.value, list(hdr)

    ptr = lambda x: None if x is None else x.data_ptr()
    JUNK_HDR = [-1, 2 ** 32 - 1]
    zero, ones = torch.zeros(H, W, device=dev), torch.ones(H, W, device=dev)
    for no_color in (0, 1):
        # glic_forward_preprocess: nothing to launch; R = 0 and the header untouched
        launches, counters, host, hdr = run(lambda c, h: lib.glic_forward_preprocess(
            0, 3, 15, None, None, 1.0, None, None, None, None, C.byref(view), no_color, None, None, 0, image.data_ptr(),
            image.numel(), C.byref(h), None))
        assert (launches, host, hdr) == (0, 0, JUNK_HDR)
        # glic_forward_render: T and colour zeroed, B = 0, the header untouched
        color, T = nan(3, H, W), nan(H, W)
        launches, counters, host, hdr = run(lambda c, h: lib.glic_forward_render(
            0, C.byref(view), no_color, 0, geom.data_ptr(), image.data_ptr(), binning.data_ptr(), binning.numel(), sample.data_ptr(),
            sample.numel(), color.data_ptr(), T.data_ptr(), C.byref(h), None))
        assert (launches, host, hdr) == (0, 0, JUNK_HDR)
        assert torch.equal(T, zero) and not color.any()
        # glic_forward: T and colour zeroed, the counters and the header zero; with no_color a missing colour plane is allowed
        for color in ((nan(3, H, W), None) if no_color else (nan(3, H, W),)):
            T = nan(H, W)
            launches, counters, host, hdr = run(lambda c, h: lib.glic_forward(
                0, 3, 15, None, None, 1.0, None, None, None, None, C.byref(view), no_color, None, geom.data_ptr(), geom.numel(),
                image.data_ptr(), image.numel(), binning.data_ptr(), binning.numel(), sample.data_ptr(), sample.numel(), ptr(color),
                T.data_ptr(), c, None))
            assert (launches, counters, hdr) == (0, [0, 0, 0], [0, 0])
            assert torch.equal(T, zero) and (color is None or not color.any())
    # glic_render: T = 1 by one fill launch, colour and the optional depth planes zeroed, the counters and the header zero
    for depths in (True, False):
        color, T = nan(3, H, W), nan(H, W)
        depth, median = (nan(H, W), nan(H, W)) if depths else (None, None)
        launches, counters, host, hdr = run(lambda c, h: lib.glic_render(
            0, 3, 15, None, None, 1.0, None, None, None, None, C.byref(view), None, geom.data_ptr(), geom.numel(), image.data_ptr(),
            image.numel(), binning.data_ptr(), binning.numel(), color.data_ptr(), T.data_ptr(), ptr(depth), ptr(median), c, None))
        assert (launches, counters, hdr) == (1, [0, 0, 0], [0, 0])
        assert torch.equal(T, ones) and not color.any()
        assert depth is None or (not depth.any() and not median.any())
    # glic_contribution: T zeroed when asked for, the scores untouched, the counters and the header zero
    for with_T in (True, False):
        mw, hits, ends = nan(4), torch.full((4,), 5, dtype=torch.int64, device=dev), torch.full((H * W,), 6, dtype=torch.int64, device=dev)
        T = nan(H, W) if with_T else None
        launches, counters, host, hdr = run(lambda c, h: lib.glic_contribution(
            0, None, None, 1.0, None, None, C.byref(view), None, geom.data_ptr(), geom.numel(), image.data_ptr(), image.numel(),
            binning.data_ptr(), binning.numel(), mw.data_ptr(), hits.data_ptr(), ends.data_ptr(), ptr(T), c, None))
        assert (launches, counters, hdr) == (0, [0, 0, 0], [0, 0])
        assert T is None or torch.equal(T, zero)
        assert torch.isnan(mw).all() and (hits == 5).all() and (ends == 6).all()


def test_torch_shim_autograd_matches_capi(oracle32):
    """The reference-facing symbols (LibTorch shim) driven like rasterizer.cpp / renderer.cpp."""
    from gaussian_lic_b200 import ops
    g, cam = small_scene(5000, 320, 208, 9, 3)
    dev = "cuda"
    t = lambda a: torch.as_tensor(a, dtype=torch.float32).to(dev)
    means = t(g["means"]).requires_grad_(True)
    log_s = t(g["log_scales"]).requires_grad_(True)
    rot_raw = t(g["rots"] * 1.7).requires_grad_(True)
    op_logit = t(g["opacity_logits"]).view(-1, 1).requires_grad_(True)
    dc = t(g["dc"]).view(-1, 1, 3).requires_grad_(True)
    sh = t(g["sh"]).requires_grad_(True)
    rs = ops.GaussianRasterizationSettings(cam["H"], cam["W"], cam["tanfovx"], cam["tanfovy"], *[float(x) for x in cam["lims"]],
                                           torch.zeros(3, device=dev), 1.0, t(cam["view"]).view(4, 4), t(cam["proj"]).view(4, 4),
                                           3, t(cam["campos"]))
    rast = ops.GaussianRasterizer(rs)
    means2D = torch.zeros_like(means, requires_grad=True)
    color, radii, final_T = rast(means, means2D, torch.sigmoid(op_logit), dc, sh, torch.exp(log_s),
                                 torch.nn.functional.normalize(rot_raw))
    gt = t(__import__("gaussian_lic_b200").synthetic.make_gt_image(cam["W"], cam["H"]))
    loss = 0.8 * ops.l1_loss(color, gt) + 0.2 * (1.0 - ops.fused_ssim(color.unsqueeze(0), gt.unsqueeze(0)))
    loss.backward()
    torch.cuda.synchronize()
    # oracle: same activations in numpy
    g2 = dict(g)
    g2["rots"] = (g["rots"] * 1.7) / np.linalg.norm(g["rots"] * 1.7, axis=1, keepdims=True)
    f = oracle32.forward(g2, cam)
    L, dl = oracle32.loss(f["color"], gt.cpu().numpy())
    b = oracle32.backward(f, dl)
    assert abs(float(loss.item()) - L) < 2e-5, (float(loss.item()), L)
    image_close(color.detach().cpu().numpy(), f["color"], "shim color")
    np.testing.assert_array_equal(radii.cpu().numpy(), f["radii"])
    grad_close(means.grad.cpu().numpy(), b["dL_dmeans3D"], "d means (shim)")
    grad_close(dc.grad.cpu().numpy(), b["dL_ddc"], "d dc (shim)")
    grad_close(sh.grad.cpu().numpy(), b["dL_dsh"], "d sh (shim)")
    grad_close(log_s.grad.cpu().numpy(), b["dL_dscales"] * g["scales"], "d log-scale (shim)")
    o = g["opacity"].reshape(-1, 1)
    grad_close(op_logit.grad.cpu().numpy(), b["dL_dopacity"] * o * (1 - o), "d opacity-logit (shim)")
    oracle32.free(f)


def test_capacity_overflow_recovers(oracle32):
    """glic_forward sizes the pair list by a caller capacity; an undersized one must be flagged (empty frame, no
    out-of-bounds access) and a retry with the reported R must reproduce the exact result."""
    from gaussian_lic_b200 import ops
    g, cam = small_scene(6000, 320, 208, 13, 3)
    r = ops.CRasterizer(cam["W"], cam["H"])
    gd = ops.scene_to_device(g)
    view = r.make_view(cam)
    r.cap_target = 1500                                   # far below R
    color, T, radii = r.forward(gd, view, sync=False)
    assert r.finish() is True and r.R > 1500              # overflow reported together with the true R
    assert float(color.abs().max()) == 0.0 and float((T - 1.0).abs().max()) == 0.0   # empty frame, nothing read
    color, T, radii = r.forward(gd, view)                 # sync=True retries until it fits
    f = oracle32.forward(g, cam)
    assert (r.R, r.B) == (f["R"], f["B"]) and r.cap >= r.R
    image_close(color.cpu().numpy(), f["color"], "color after capacity growth")
    oracle32.free(f)
