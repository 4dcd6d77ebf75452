"""LPIPS (AlexNet) on the GPU: glic_lpips against the reference's own TorchScript module run in float64 on cuda:0 -- its values
pinned in tests/golden/lpips_pins.npz and, where build() copied the module to oracle/_ref/, run live -- and the native mapper's
evaluate_lpips / render.  (Why float64: see tests/golden/make_lpips_golden.py; the module's own float32 run is not accurate
enough to be the yardstick.)

The pinned image pairs are regenerated from their seeds by tests/golden/make_lpips_golden.py's make_pair().  The reference's
weights are converted by build() into oracle/_ref/lpips_alex.bin; the tests that need them skip without it.  Seeded synthetic
weights of the same layout, checked against a float64 torch.nn.functional restatement, cover the kernels without them."""
import importlib.util
import os

import numpy as np
import pytest

from test_gpu_exposure import _expose32
from test_gpu_mapper_grads import H, W, _keyframes, _mapper, _scene

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
BUILT = os.path.join(ROOT, "oracle", "_ref", "lpips_alex.bin")
PT = os.path.join(ROOT, "oracle", "_ref", "lpips_alex.pt")
TOL = 2e-5


def _golden_module():
    spec = importlib.util.spec_from_file_location("make_lpips_golden", os.path.join(GOLD, "make_lpips_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


G = _golden_module()


@pytest.fixture(scope="module")
def weights():
    """the reference's weights on the device"""
    if not os.path.isfile(BUILT):
        pytest.skip("oracle/_ref/lpips_alex.bin not built (the reference's weights)")
    from gaussian_lic_b200 import lpips_weights
    return torch.from_numpy(lpips_weights.read(BUILT)).cuda()


@pytest.fixture(scope="module")
def synthetic():
    """(payload, device copy) of seeded synthetic weights"""
    p = G.synthetic_payload(1)
    return p, torch.from_numpy(p).cuda()


@pytest.fixture(scope="module")
def weight_path(tmp_path_factory):
    """a weight file for the mapper: the reference's if built, else the synthetic one written through the converter's writer"""
    if os.path.isfile(BUILT):
        return BUILT
    from gaussian_lic_b200 import lpips_weights
    path = tmp_path_factory.mktemp("lpips") / "synthetic.bin"
    lpips_weights.write(path, G.synthetic_payload(1))
    return str(path)


@pytest.fixture(scope="module")
def pins():
    z = np.load(os.path.join(GOLD, "lpips_pins.npz"))
    return {(int(w), int(h), int(s), str(k)): float(v) for w, h, s, k, v in zip(z["W"], z["H"], z["seed"], z["kind"], z["lpips"])}


def _lpips(x, y, weights):
    from gaussian_lic_b200 import ops
    out = ops.lpips(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), weights)
    torch.cuda.synchronize()
    return out.cpu().numpy()[0]


@pytest.mark.parametrize("pair", G.PAIRS, ids=["%dx%d-%s" % (p[0], p[1], p[3]) for p in G.PAIRS])
def test_lpips_matches_reference_pins(weights, pins, pair):
    W_, H_, seed, kind = pair
    got = _lpips(*G.make_pair(W_, H_, seed, kind), weights)
    want = pins[pair]
    if kind == "identical":
        assert got == 0.0 and abs(want) <= TOL
    else:
        assert abs(float(got) - want) <= TOL, (got, want, float(got) - want)


@pytest.mark.parametrize("WH,kind", [((640, 512), "light"), ((640, 512), "unrelated"), ((333, 197), "heavy"), ((31, 31), "heavy"),
                                     ((1920, 1080), "light")])
def test_lpips_synthetic_weights_match_float64_restatement(synthetic, WH, kind):
    """every layer, the pools and the heads with weights that are not the reference's, against the network restated in float64"""
    p, dev = synthetic
    x, y = G.make_pair(WH[0], WH[1], 50 + WH[1], kind)
    want = G.lpips64(p, x, y)
    got = _lpips(x, y, dev)
    assert abs(float(got) - want) <= TOL * max(1.0, abs(want)), (got, want)


def test_identical_images_give_exactly_zero(synthetic):
    weights = synthetic[1]
    for W_, H_ in ((1920, 1080), (333, 197), (31, 31)):
        x, _ = G.make_pair(W_, H_, 7, "heavy")
        assert _lpips(x, x.copy(), weights) == 0.0
        # values outside [0,1] are clamped first: identical after the clamp is identical
        assert _lpips(x * 1.5 - 0.25, np.clip(x * 1.5 - 0.25, 0, 1), weights) == 0.0


def test_two_calls_give_identical_bits(synthetic):
    from gaussian_lic_b200 import ops
    weights = synthetic[1]
    x, y = (torch.from_numpy(a).cuda() for a in G.make_pair(1920, 1080, 11, "heavy"))
    a = ops.lpips(x, y, weights)
    b = ops.lpips(x, y, weights)
    torch.cuda.synchronize()
    assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()
    assert float(a) > 0.0


def test_lpips_matches_the_torchscript_module_live(weights):
    if not os.path.isfile(PT):
        pytest.skip("oracle/_ref/lpips_alex.pt not built")
    m = G.reference_module64(PT)
    for W_, H_, seed, kind in ((640, 512, 101, "light"), (640, 512, 102, "heavy"), (333, 197, 103, "unrelated"), (64, 48, 104, "heavy"),
                               (1920, 1080, 105, "light")):
        x, y = G.make_pair(W_, H_, seed, kind)
        want = G.reference_lpips(m, x, y, dtype=torch.float64)
        got = _lpips(x, y, weights)
        assert abs(float(got) - want) <= TOL, ((W_, H_, kind), got, want)


# ---- the native mapper ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def scene():
    raw = _scene(3)
    poses, _, gts = _keyframes()
    return raw, poses, gts


def _trained_mapper(scene, expo=False):
    raw, poses, gts = scene
    m = _mapper(raw, poses[:-1], gts[:-1])
    m.add_keyframe(*poses[-1], gts[-1], train=False)          # one held-out view
    if expo:
        m.enable_exposure(0.001)
    m.optimize([0, 1, 0])
    return m


def test_mapper_lpips_needs_weights(scene):
    from gaussian_lic_b200 import capi
    m = _trained_mapper(scene)
    with pytest.raises(capi.GlicError, match="no LPIPS weights loaded"):
        m.evaluate_lpips(0)
    m.close()


@pytest.mark.parametrize("train,index", [(True, 0), (True, 1), (False, 0)])
def test_mapper_evaluate_lpips(scene, weight_path, train, index):
    from gaussian_lic_b200 import lpips_weights
    weights = torch.from_numpy(lpips_weights.read(weight_path)).cuda()
    raw, poses, gts = scene
    m = _trained_mapper(scene)
    m.load_lpips(weight_path)
    psnr, ssim = m.evaluate(index, train)
    p2, s2, lp = m.evaluate_lpips(index, train)
    assert np.float32(p2).tobytes() == np.float32(psnr).tobytes() and np.float32(s2).tobytes() == np.float32(ssim).tobytes()
    img = m.render(index, train)
    gt = gts[index] if train else gts[-1]
    assert img.shape == (3, H, W) and img.dtype == np.float32 and img.min() >= 0.0 and img.max() <= 1.0
    # the LPIPS of the rendered image against the keyframe's image, through glic_lpips directly
    assert np.float32(lp).tobytes() == np.float32(_lpips(img, np.ascontiguousarray(gt, np.float32), weights)).tobytes()
    assert lp > 0.0
    # the image reproduces the PSNR the mapper reported
    mse = np.mean((img.astype(np.float64) - np.clip(np.asarray(gt, np.float64), 0, 1)) ** 2)
    assert abs(10 * np.log10(1 / mse) - psnr) < 1e-3
    # a second call scores the same render with the same bits
    assert m.evaluate_lpips(index, train) == (p2, s2, lp)
    m.close()


def test_mapper_render_applies_the_training_exposure(scene):
    m = _trained_mapper(scene, expo=True)
    E0 = m.exposure(0)
    ident = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)
    m.set_exposure(0, ident)
    base = m.render(0)                                         # E = [I | 0]: the rendered image itself, clamped
    held = m.render(0, train=False)
    E = np.array([[0.9, 0.05, -0.02, 0.03], [0.04, 1.1, 0.03, -0.02], [-0.03, 0.02, 0.8, 0.01]], np.float32)
    m.set_exposure(0, E)
    out = m.render(0)
    inside = np.all((base > 0) & (base < 1), axis=0)         # pixels the clamp did not touch: base is the raw render there
    assert inside.mean() > 0.3
    want = np.clip(_expose32(base, E), 0, 1)
    assert np.abs(out - want)[:, inside].max() <= 1e-6
    assert np.abs(out - base)[:, inside].max() > 1e-2
    # held-out views are drawn with the identity whatever the training keyframes' exposures are
    assert np.array_equal(m.render(0, train=False), held)
    # the trained exposure (not the identity) is what render applies after optimize()
    m.set_exposure(0, E0)
    assert not np.array_equal(E0, ident) and np.abs(m.render(0) - np.clip(_expose32(base, E0), 0, 1))[:, inside].max() <= 1e-6
    m.close()


def test_mapper_refuses_frames_under_31(scene, weight_path):
    from gaussian_lic_b200 import capi, mapper
    raw, _, _ = scene
    m = mapper.Mapper(30, 40, 30.0, 30.0, 15.0, 20.0, sh_degree=3)
    m.initialize(raw)
    m.add_keyframe(np.eye(3), np.zeros(3), np.full((3, 40, 30), 0.5, np.float32))
    m.load_lpips(weight_path)
    with pytest.raises(capi.GlicError, match="31x31"):
        m.evaluate_lpips(0)
    assert m.render(0).shape == (3, 40, 30)
    m.close()
