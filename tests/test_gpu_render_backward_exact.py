"""The production render backward (fast exponent, exact-expf fallback near alpha = 1/255) against the former kernel body
(exact expf for every pixel), on the same saved forward state.

Both forms must take the same (pixel, splat) decisions -- the forward's -- so their gradients may differ only by fp32
reassociation: every entry within 1e-5 of the tensor's max |grad|, no outliers.  The counting forms of the two kernels must
walk the same visits and take exactly the same pixel-splat pairs."""
import numpy as np
import pytest

from helpers import POSES, small_scene

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

TWO_D = ("dL_dmeans2D", "dL_dconic", "dL_dopacity", "dL_dcolors")
ATOL = 1e-5        # of max |grad| per tensor


def _run(g, cam, seed):
    from gaussian_lic_b200 import ops
    r = ops.CRasterizer(cam["W"], cam["H"])
    gd = ops.scene_to_device(g)
    view = r.make_view(cam)
    r.forward(gd, view)
    dL = torch.as_tensor(np.random.default_rng(seed).normal(size=(3, cam["H"], cam["W"])).astype(np.float32)).cuda()
    out = {}
    for exact in (True, False):
        grads = r.alloc_grads()
        for k in TWO_D:
            grads[k].zero_()
        r.render_backward(view, dL, grads, exact=exact)
        ctr = torch.zeros(8, dtype=torch.int64, device="cuda")
        scratch = r.alloc_grads()
        for k in TWO_D:
            scratch[k].zero_()
        r.render_backward(view, dL, scratch, exact=exact, counters=ctr)
        torch.cuda.synchronize()
        out[exact] = ({k: grads[k].cpu().numpy().astype(np.float64) for k in TWO_D},
                      dict(zip(ops.CRasterizer.BWD_COUNTERS, (int(x) for x in ctr.tolist()))))
    return out


def _check(out):
    (g_old, c_old), (g_new, c_new) = out[True], out[False]
    print("counters exact %s\ncounters fast  %s" % (c_old, c_new))
    for k in ("live_buckets", "splats", "visits", "visits_taken", "candidate_pixels", "taken_pixels"):
        assert c_new[k] == c_old[k], (k, c_new[k], c_old[k])
    assert c_old["fallback_pixels"] == 0
    assert c_new["taken_pixels"] > 0
    for k in TWO_D:
        scale = max(np.abs(g_old[k]).max(), 1e-30)
        err = np.abs(g_new[k] - g_old[k]).max() / scale
        print("%s: max |fast - exact| / max |exact| = %.3e" % (k, err))
        assert err <= ATOL, (k, err)
    return c_new


@pytest.mark.parametrize("view,pp", POSES, ids=["v%d_pp%g_%g" % (v, pp[0], pp[1]) for v, pp in POSES])
def test_fast_backward_matches_exact_body(view, pp):
    g, cam = small_scene(view=view, pp=pp)
    _check(_run(g, cam, view))


def test_fast_backward_matches_exact_body_at_the_threshold():
    """opacities just above 1/255: o G straddles 1/255 over most of every splat's footprint, so the fast alpha of many
    pixels falls into the guard band and is decided by the exact expf"""
    g, cam = small_scene(P=20000, seed=5)
    rng = np.random.default_rng(5)
    g["opacity"] = (rng.uniform(1.0, 1.25, g["opacity"].shape) / 255.0).astype(np.float32)
    c = _check(_run(g, cam, 5))
    assert c["fallback_pixels"] > 0
    assert c["visits_taken"] < c["visits"]


def test_fast_backward_matches_exact_body_cfg2():
    from gaussian_lic_b200 import mapper as gmapper, synthetic as syn
    P, W, H, fx, fy, cx, cy, deg, _ = syn.CONFIGS["cfg2"]
    g, _ = syn.make_scene("cfg2")
    cam = gmapper.camera_block(W, H, fx, fy, cx, cy, *syn.orbit_pose(0, radius=0.25))
    _check(_run(g, cam, 0))
