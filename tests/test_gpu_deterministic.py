"""The deterministic render backward (glic_backward_deterministic) on the GPU.

* Restatement: the ordered entry list of glic_debug_deterministic_entries, folded on the host in the documented association
  (deterministic_oracle.py), equals the four 2-D gradient arrays bit for bit -- on rotated views, an off-centre principal point,
  a splat that covers a whole 1920x1080 frame (one run of thousands of tiles), P = 1, P = 2^16 +- 1 and a scene with every
  Gaussian culled.
* Repeatability: five calls on one saved state give the same bits for every output.
* Agreement with the atomic glic_backward: per Gaussian with n contributions v_i, |det - atomic| <= 2 gamma_{n-1} sum |v_i|.
* torch: under torch.use_deterministic_algorithms(True) RasterizeGaussiansBackwardCUDA takes the deterministic path."""
import numpy as np
import pytest

from deterministic_oracle import fold_entries, gamma, scatter
from helpers import POSES, small_scene

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

TWO_D = ("dL_dmeans2D", "dL_dconic", "dL_dopacity", "dL_dcolors")
ALL = TWO_D + ("dL_dmeans3D", "dL_dcov3D", "dL_ddc", "dL_dsh", "dL_dscales", "dL_drots")


def _setup(g, cam, seed=0):
    from gaussian_lic_b200 import ops
    r = ops.CRasterizer(cam["W"], cam["H"])
    gd = ops.scene_to_device(g)
    view = r.make_view(cam)
    _, _, radii = r.forward(gd, view)
    dL = torch.as_tensor(np.random.default_rng(seed).normal(size=(3, cam["H"], cam["W"])).astype(np.float32)).cuda()
    return r, gd, view, radii, dL


def _np(grads, keys=ALL):
    torch.cuda.synchronize()
    return {k: grads[k].cpu().numpy() for k in keys if grads[k].numel()}


def _restated(r, view, dL):
    grads = r.alloc_grads()
    gid, tile, values = r.deterministic_entries(view, dL, grads)
    got = _np(grads, TWO_D)
    gid, tile, values = gid.cpu().numpy(), tile.cpu().numpy(), values.cpu().numpy()
    # the list is ordered by gid, then by ascending tile, one entry per (tile, Gaussian)
    if gid.size:
        assert np.all(np.diff(gid) >= 0)
        same = np.diff(gid) == 0
        assert np.all(np.diff(tile)[same] > 0)
        assert gid.min() >= 0 and gid.max() < r.P
    gids, sums, counts, abs_sums = fold_entries(gid, values)
    want = scatter(r.P, gids, sums)
    for k in TWO_D:
        assert got[k].reshape(r.P, -1).tobytes() == want[k].tobytes(), k
    return got, gids, counts, abs_sums


def _check_scene(g, cam, seed=0):
    r, gd, view, radii, dL = _setup(g, cam, seed)
    got, gids, counts, abs_sums = _restated(r, view, dL)
    det = _np(r.backward(gd, view, radii, dL, deterministic=True))
    atomic = _np(r.backward(gd, view, radii, dL))
    for k in TWO_D:
        assert det[k].tobytes() == got[k].tobytes(), k
    # agreement with the atomic form, bound from the entries: 2 gamma_{n-1} sum |v| per Gaussian and value
    bound = 2.0 * gamma(counts - 1)[:, None] * abs_sums
    d = {k: np.abs(det[k].astype(np.float64) - atomic[k].astype(np.float64)).reshape(r.P, -1) for k in TWO_D}
    diff = np.concatenate([d["dL_dmeans2D"][gids][:, 0:2], d["dL_dconic"][gids][:, [0, 1, 3]], d["dL_dcolors"][gids],
                           d["dL_dopacity"][gids]], axis=1)
    assert np.all(diff <= bound), float((diff - bound).max())
    rows = np.setdiff1d(np.arange(r.P), gids)
    for k in TWO_D:
        assert not det[k].reshape(r.P, -1)[rows].any() and not atomic[k].reshape(r.P, -1)[rows].any(), k
    return r, counts


@pytest.mark.parametrize("view,pp", POSES, ids=["v%d_pp%g_%g" % (v, pp[0], pp[1]) for v, pp in POSES])
def test_restatement_and_agreement(view, pp):
    g, cam = small_scene(view=view, pp=pp)
    _, counts = _check_scene(g, cam, seed=view)
    assert counts.size > 100 and counts.max() > 1


def test_whole_frame_splat_1080p():
    """one splat in front of the camera covering all 8160 tiles of a 1920x1080 frame, behind it a few thousand small ones"""
    g, cam = small_scene(P=4000, W=1920, H=1080, f=1000.0, seed=3)
    g["means"][0] = (0.0, 0.0, 2.0)
    g["scales"][0] = (40.0, 40.0, 0.01)
    g["rots"][0] = (1.0, 0.0, 0.0, 0.0)
    g["opacity"][0] = 0.3
    r, counts = _check_scene(g, cam, seed=3)
    assert counts.max() >= 4000, counts.max()


@pytest.mark.parametrize("P", [1, (1 << 16) - 1, 1 << 16, (1 << 16) + 1])
def test_restatement_at_key_bit_boundaries(P):
    g, cam = small_scene(P=P, seed=P % 97, log_scale_mean=-3.0 if P > 1 else -1.0)
    if P == 1:
        g["means"][0] = (0.0, 0.0, 5.0)
    _check_scene(g, cam, seed=1)


def test_all_culled():
    g, cam = small_scene(P=500)
    g["means"][:, 2] = -5.0                                   # behind the camera
    r, gd, view, radii, dL = _setup(g, cam)
    assert int(radii.max()) == 0
    got, gids, _, _ = _restated(r, view, dL)
    assert gids.size == 0
    det = _np(r.backward(gd, view, radii, dL, deterministic=True))
    for k, v in det.items():
        assert not v.any(), k


def test_repeatable_bits():
    g, cam = small_scene(P=20000, seed=7, view=1)
    r, gd, view, radii, dL = _setup(g, cam, seed=7)
    first = _np(r.backward(gd, view, radii, dL, deterministic=True))
    for _ in range(4):
        again = _np(r.backward(gd, view, radii, dL, deterministic=True))
        for k in first:
            assert again[k].tobytes() == first[k].tobytes(), k


def test_short_workspace_is_refused():
    from gaussian_lic_b200 import capi
    import ctypes as C
    g, cam = small_scene(P=2000)
    r, gd, view, radii, dL = _setup(g, cam)
    gr = r.alloc_grads()
    need = capi.lib.glic_deterministic_bytes(r.cap, r.W, r.H)
    ws = torch.empty(need - 1, dtype=torch.uint8, device="cuda")
    st = capi.lib.glic_backward_deterministic(
        r.P, r.D, r.M, capi.ptr(gd["means"]), capi.ptr(gd["scales"]), 1.0, capi.ptr(gd["rots"]), capi.ptr(gd["dc"]),
        capi.ptr(gd["sh"]), C.byref(view), capi.ptr(radii), r.cap, capi.ptr(r.geom_ws), capi.ptr(r.binning_ws),
        capi.ptr(r.image_ws), capi.ptr(r.sample_ws), capi.ptr(dL), 0.0, *[capi.ptr(gr[k]) for k in ALL], capi.ptr(ws), ws.numel(),
        None)
    assert st == -2                                           # GLIC_ERR_WORKSPACE


@pytest.fixture
def deterministic_torch():
    before = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(before)


def _torch_grads(g, cam, dL):
    from gaussian_lic_b200 import ops
    t = lambda a: torch.as_tensor(a, dtype=torch.float32).cuda()
    leaves = dict(means=t(g["means"]), op=t(g["opacity"]).view(-1, 1), dc=t(g["dc"]).view(-1, 1, 3), sh=t(g["sh"]),
                  scales=t(g["scales"]), rots=t(g["rots"]))
    for x in leaves.values():
        x.requires_grad_(True)
    rs = ops.GaussianRasterizationSettings(cam["H"], cam["W"], cam["tanfovx"], cam["tanfovy"], *[float(x) for x in cam["lims"]],
                                           torch.zeros(3, device="cuda"), 1.0, t(cam["view"]).view(4, 4), t(cam["proj"]).view(4, 4),
                                           g["degree"], t(cam["campos"]))
    means2D = torch.zeros_like(leaves["means"], requires_grad=True)
    color, _, _ = ops.GaussianRasterizer(rs)(leaves["means"], means2D, leaves["op"], leaves["dc"], leaves["sh"], leaves["scales"],
                                             leaves["rots"])
    (color * dL).sum().backward()
    torch.cuda.synchronize()
    out = {k: v.grad.cpu().numpy() for k, v in leaves.items()}
    out["means2D"] = means2D.grad.cpu().numpy()
    return out


def _c_grads(r, gd, view, radii, dL, deterministic):
    gr = _np(r.backward(gd, view, radii, dL, deterministic=deterministic))
    return dict(means=gr["dL_dmeans3D"], op=gr["dL_dopacity"], dc=gr["dL_ddc"], sh=gr["dL_dsh"], scales=gr["dL_dscales"],
                rots=gr["dL_drots"], means2D=gr["dL_dmeans2D"])


def test_torch_deterministic_flag(deterministic_torch):
    g, cam = small_scene(P=5000, view=3, seed=4)
    r, gd, view, radii, dL = _setup(g, cam, seed=4)
    a, b = _torch_grads(g, cam, dL), _torch_grads(g, cam, dL)
    want = _c_grads(r, gd, view, radii, dL, True)
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k
        assert a[k].reshape(-1).tobytes() == want[k].reshape(-1).tobytes(), k


def test_torch_default_is_atomic_within_reassociation():
    """flag off: the atomic backward.  The 2-D gradients (means2D, opacity) within 2 gamma_{n-1} sum |v| of the deterministic
    ones per Gaussian (bound from the entry list); the 3-D gradients, which the per-Gaussian backward derives from them, within
    1e-5 of the tensor's max |grad| of glic_backward's"""
    assert not torch.are_deterministic_algorithms_enabled()
    g, cam = small_scene(P=5000, view=3, seed=4)
    r, gd, view, radii, dL = _setup(g, cam, seed=4)
    got = _torch_grads(g, cam, dL)
    _, gids, counts, abs_sums = _restated(r, view, dL)
    bound = 2.0 * gamma(counts - 1)[:, None] * abs_sums
    det = _c_grads(r, gd, view, radii, dL, True)
    d_m2 = np.abs(got["means2D"].astype(np.float64) - det["means2D"].astype(np.float64))[gids][:, 0:2]
    d_op = np.abs(got["op"].astype(np.float64) - det["op"].astype(np.float64)).reshape(-1)[gids]
    assert np.all(d_m2 <= bound[:, 0:2]) and np.all(d_op <= bound[:, 8])
    want = _c_grads(r, gd, view, radii, dL, False)
    for k in got:
        a, w = got[k].reshape(-1).astype(np.float64), want[k].reshape(-1).astype(np.float64)
        scale = max(np.abs(w).max(), 1e-30)
        assert np.abs(a - w).max() <= 1e-5 * scale, k
