"""tests/lpips_reference.py without a GPU: the restatement against torch.nn.functional and the float64 network of
tests/golden/make_lpips_golden.py, the scratch layout against glic_lpips_scratch_bytes, and the conv bound against a host
emulation of the kernel's split-TF32 arithmetic -- within it under both accumulation models, and exceeded by each controlled
fault (a single TF32 pass, a dropped cross term, padding off by one, the two images swapped in the M tile that straddles
them).  Run with -s to see the ratios."""
import importlib.util
import os

import numpy as np
import pytest

import lpips_reference as R

torch = pytest.importorskip("torch")
F = torch.nn.functional

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _golden_module():
    spec = importlib.util.spec_from_file_location("make_lpips_golden", os.path.join(ROOT, "tests", "golden", "make_lpips_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


G = _golden_module()


def test_scratch_layout_matches_the_library():
    from gaussian_lic_b200 import capi
    for W, H in R.FRAMES:
        regions, total = R.layout(H, W)
        assert total == capi.lib.glic_lpips_scratch_bytes(H, W), (W, H)
        assert all(off % 128 == 0 for off, _, _, _ in regions.values())


@pytest.mark.parametrize("WH", [(31, 31), (35, 35), (64, 48), (131, 31)])
def test_restatement_matches_torch_float64(WH):
    """every stage of the restatement, chained in float64, against conv2d / max_pool2d and the float64 network itself"""
    W, H = WH
    p = G.synthetic_payload(1)
    x, y = G.make_pair(W, H, 7 + W, "heavy")
    x[0, 0, :3] = [-0.5, 1.5, 1.0]
    pt = torch.from_numpy(p)
    mean, std, convs, lins = R.unpack(pt)
    inp = R.normalize(torch.from_numpy(np.stack([x, y])), mean, std)
    # the float32 normalisation is the float32 arithmetic itself
    want = (np.clip(np.stack([x, y]), 0, 1) - p[:3].reshape(3, 1, 1)) / p[3:6].reshape(3, 1, 1)
    assert want.dtype == np.float32 and np.array_equal(inp.numpy(), want)
    # the chain starts from the float64 normalisation, as the float64 network does
    t = (torch.from_numpy(np.stack([x, y])).double().clamp(0, 1) - mean.double().view(3, 1, 1)) / std.double().view(3, 1, 1)
    hs, ws, _, _ = R.shapes(H, W)
    total = 0.0
    for l, (ci, co, k, s, pad) in enumerate(R.CONVS):
        w, b = convs[l]
        v, M, S = R.conv(t, w, b, s, pad)
        ref = F.conv2d(t, w.to(torch.float64), b.to(torch.float64), stride=s, padding=pad)
        assert v.shape == ref.shape == (2, co, hs[l], ws[l])
        assert float((v - ref).abs().max()) <= 1e-12 * float(M.max())
        assert bool((M >= v.abs() - 1e-12 * M).all()) and bool((S >= 0).all())
        t = v.clamp_min(0.0)
        d, err = R.head(t, lins[l])
        assert bool((err >= 0).all())
        total += float(d.sum()) / (hs[l] * ws[l])
        if l < 2:
            pooled = R.pool(t)
            assert torch.equal(pooled, F.max_pool2d(t, 3, 2))
            t = pooled
    assert abs(total - G.lpips64(p, x, y, device="cpu")) <= 1e-12


def test_conv_chunking_and_rows():
    """a band-chunked and a row-restricted conv give the same values as one pass"""
    rng = np.random.default_rng(5)
    inp = torch.from_numpy(rng.standard_normal((2, 3, 45, 37)).astype(np.float32))
    w = torch.from_numpy(rng.standard_normal((8, 3, 11, 11)).astype(np.float32))
    b = torch.from_numpy(rng.standard_normal(8).astype(np.float32))
    whole = R.conv(inp, w, b, 4, 2)
    chunked = R.conv(inp, w, b, 4, 2, budget=1)
    rows = R.conv(inp, w, b, 4, 2, rows=range(3, 7))
    for a, c, r in zip(whole, chunked, rows):
        assert torch.equal(a, c) and torch.equal(a[:, :, 3:7], r)


def test_finish_and_partials():
    """the finish restatement is the float64 mean of the partials per tap, added in order; the partial check accepts the
    exact per-CTA sums and refuses a partial one pixel's value off"""
    rng = np.random.default_rng(2)
    hws = [1000, 37, 1, 513, 256 * 40 + 3]
    parts = [rng.uniform(0, 1e-2, R.head_blocks(hw)) for hw in hws]
    want = np.float32(sum(p.sum() / hw for p, hw in zip(parts, hws)))
    got = R.finish(parts, hws)
    assert abs(float(got) - float(want)) <= 2.0 ** -23 * abs(float(want))
    d = torch.from_numpy(rng.uniform(0, 1, 1000))
    err = torch.full((1000,), 1e-9, dtype=torch.float64)
    good = torch.stack([d[i:i + 256].sum() for i in range(0, 1000, 256)])
    assert float(R.partial_check(good, d, err).max()) <= 1.0
    bad = good.clone()
    bad[3] += d[800]
    assert float(R.partial_check(bad, d, err).max()) > 1.0


def test_tf32_rounding():
    x = np.array([1.0, 1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, -(1.0 + 2.0 ** -11), 1.0 + 2.0 ** -12, 3.0e-39], np.float32)
    got = R.tf32(x)
    # ties go away from zero; anything under half an ulp (2^-10 at 1) goes down
    assert list(got[:5]) == [1.0, 1.0 + 2.0 ** -10, 1.0 + 2 * 2.0 ** -10, -(1.0 + 2.0 ** -10), 1.0]
    for v in rng_values():
        hi = R.tf32(v)
        assert np.all(np.abs(hi.astype(np.float64) - v) <= 2.0 ** -11 * np.abs(v.astype(np.float64)))
        assert np.all(hi.view(np.uint32) & 0x1FFF == 0)


def rng_values():
    rng = np.random.default_rng(9)
    yield (rng.standard_normal(10000) * np.exp(rng.uniform(-30, 30, 10000))).astype(np.float32)


# ---- the bound against the emulated kernel ---------------------------------------------------------------------------
def _layer_case(l, kind, seed=0):
    """(inp [2, Cin, h, w] float32, w, b, output channels to emulate) for conv l at the M-tile straddling frame of its layer:
    conv0 (131, 31), conv1 (71, 39), conv2-4 (143, 79); 'random': He weights over random inputs (conv0: the normalised range;
    later layers: ReLU-like, half zeros); 'positive': the same with every weight and input made non-negative, so the
    truncation of an rz accumulation never cancels; 'cancel': the weights made antisymmetric in kx and scaled by 1e3, over inputs constant
    along x, so every output's exact partial sums cancel to the bias"""
    W, H = {0: (131, 31), 1: (71, 39)}.get(l, (143, 79))
    hs, ws, phs, pws = R.shapes(H, W)
    hi, wi = {0: (H, W), 1: (phs[0], pws[0])}.get(l, (phs[1], pws[1]))
    ci, co, k, _, _ = R.CONVS[l]
    rng = np.random.default_rng(100 * l + seed)
    w = (rng.standard_normal((co, ci, k, k)) * np.sqrt(2.0 / (ci * k * k))).astype(np.float32)
    b = (0.05 * rng.standard_normal(co)).astype(np.float32)
    if l == 0:
        inp = ((rng.uniform(0, 1, (2, 3, hi, wi)) + 0.1) / 0.45).astype(np.float32)
    else:
        inp = np.maximum(rng.standard_normal((2, ci, hi, wi)), 0).astype(np.float32)
    if kind == "positive":
        w, inp = np.abs(w), np.abs(inp)
    if kind == "cancel":
        w = ((w - w[..., ::-1]) * 1e3).astype(np.float32)
        inp = np.ascontiguousarray(np.repeat(inp[..., :1], wi, axis=-1))
    cols = np.arange(co) if l == 0 else np.arange(0, co, 4)
    return inp, w, b, cols


_REF = {}


def _reference(l, kind):
    if (l, kind) not in _REF:
        inp, w, b, cols = _layer_case(l, kind)
        _, _, k, s, pad = R.CONVS[l]
        v, M, S = R.conv(torch.from_numpy(inp), torch.from_numpy(w), torch.from_numpy(b), s, pad)
        _REF[(l, kind)] = (inp, w, b, cols, s, pad, [t[:, cols] for t in (v, M, S)])
    return _REF[(l, kind)]


@pytest.mark.parametrize("model", ["rn", "rz"])
@pytest.mark.parametrize("kind", ["random", "positive", "cancel"])
@pytest.mark.parametrize("l", range(5))
def test_split_tf32_emulation_within_bound(l, kind, model):
    inp, w, b, cols, s, pad, (v, M, S) = _reference(l, kind)
    got = R.emulate_conv(inp, w, b, s, pad, model, cols=cols)
    r = R.conv_ratio(got, v, M, S)
    print("\nconv%d %s %s: max err/bound %.3f" % (l, kind, model, r))
    assert r <= 1.0


@pytest.mark.parametrize("fault", R.FAULTS)
@pytest.mark.parametrize("l", range(5))
def test_negative_controls_exceed_bound(l, fault):
    """each controlled fault of the emulation exceeds the bound somewhere at the layer's straddling frame, on random inputs"""
    inp, w, b, cols, s, pad, (v, M, S) = _reference(l, "random")
    got = R.emulate_conv(inp, w, b, s, pad, "rn", fault=fault, cols=cols)
    r = R.conv_ratio(got, v, M, S)
    print("\nconv%d %s: max err/bound %.1f" % (l, fault, r))
    assert r > 1.0
