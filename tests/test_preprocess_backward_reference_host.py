"""Checks of tests/preprocess_backward_reference.py itself, on the CPU: its values against the float64 C oracle's per-Gaussian
backward (glic_oracle_preprocess_backward, checked against finite differences in test_oracle_gradients.py), its compact
chain rule against torch float64 autograd, its pose sum against tests/pose_oracle.py; a float32 evaluation of the same
arithmetic stays inside the bounds; and each plausible kernel bug of preprocess_backward_reference.MUTATIONS, applied to
the restatement, moves some element beyond them."""
import functools

import numpy as np
import pytest

import preprocess_backward_reference as pbr
from helpers import POSES

# (scene, SH degree, scale modifier, lambda_erank, pose): every stress kind, each SH degree, scale_modifier != 1, the
# effective-rank regulariser on scales chosen to land on both sides of its branch
CASES = [("needles", 2, 1.0, 0.0, POSES[2]), ("edges", 3, 1.7, 0.25, POSES[3]), ("big", 1, 0.5, 0.0, POSES[1]),
         ("deep", 0, 1.0, 0.0, POSES[0]), ("ties", 3, 1.0, 0.25, POSES[4]), ("edges", 2, 1.0, 0.0, POSES[0]),
         ("needles", 3, 1.7, 0.0, POSES[3]), ("outside", 3, 1.0, 0.0, POSES[0])]
IDS = ["%s-d%d-mod%g-erank%g-v%d" % (k, d, m, l, p[0]) for k, d, m, l, p in CASES]


def _syn():
    import importlib.util
    import os
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gaussian_lic_b200", "synthetic.py")
    spec = importlib.util.spec_from_file_location("_synthetic", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def grads2d(P, seed):
    """2-D gradients spanning 1e-6 .. 1e3 with both signs and exact zeros in every component"""
    rng = np.random.default_rng(seed)

    def one(k):
        a = rng.normal(size=(P, k)) * 10.0 ** rng.uniform(-6.0, 3.0, (P, k))
        a[rng.random((P, k)) < 0.1] = 0.0
        return a.astype(np.float32)
    return one(3), one(3), one(3)


def erank_scales(g, seed):
    """a third of the rows turned into needles (two scales 1e-2 of the third) so that the effective rank falls below 2 there;
    the rest keep an effective rank far from the branch"""
    rng = np.random.default_rng(seed)
    s = g["scales"].astype(np.float64)
    sel = rng.random(s.shape[0]) < 1.0 / 3.0
    s[sel] = np.stack([np.full(sel.sum(), 1.0), np.full(sel.sum(), 1e-2), np.full(sel.sum(), 1e-2)], 1) * rng.uniform(0.5, 1.5, (sel.sum(), 1))
    g["scales"] = s.astype(np.float32)


def cams(cam):
    """the focal lengths as the kernel forms them (float32 W / (2 tan fov)) and as the float64 oracle does"""
    W, H = cam["W"], cam["H"]
    f32 = lambda n, t: float(np.float32(n) / (np.float32(2.0) * np.float32(t)))
    return (dict(cam, fx=f32(W, cam["tanfovx"]), fy=f32(H, cam["tanfovy"])),
            dict(cam, fx=W / (2.0 * cam["tanfovx"]), fy=H / (2.0 * cam["tanfovy"])))


def outside_rows(g, cam):
    """the rows of a scene whose txtz or tytz lies beyond a lim* clamp by more than 1e-3 (both frustum masks at 0 for some)"""
    v = np.asarray(cam["view"], np.float64).reshape(4, 4).T
    p = g["means"].astype(np.float64) @ v[:3, :3].T + v[:3, 3]
    t = p[:, :2] / p[:, 2:]
    lim = np.asarray(cam["lims"], np.float64)
    out = (t[:, 0] < lim[0] - 1e-3) | (t[:, 0] > lim[1] + 1e-3) | (t[:, 1] < lim[2] - 1e-3) | (t[:, 1] > lim[3] + 1e-3)
    return {k: (a[out] if isinstance(a, np.ndarray) else a) for k, a in g.items()}


def make_scene(kind, view, pp, deg):
    """a stress scene; "outside": the edges scene's rows beyond the clamps alone, where the pose path's J uses the clamped
    ratios (every row's pose terms count in their sum)"""
    g, cam = _syn().make_stress_scene("edges" if kind == "outside" else kind, view=view, pp=pp, deg=deg)
    return (outside_rows(g, cam), cam) if kind == "outside" else (g, cam)


@functools.lru_cache(maxsize=None)
def scene(i):
    from oracle.oracle import Oracle
    kind, deg, mod, lam, (view, pp) = CASES[i]
    g, cam = make_scene(kind, view, pp, deg)
    if lam:
        erank_scales(g, i)
    o = Oracle(np.float32)
    f = o.forward(g, cam, scale_modifier=float(np.float32(mod)))
    clamped = o.state(f)["clamped"]
    radii = f["radii"].copy()
    o.free(f)
    P = g["means"].shape[0]
    dm2, dco, dcol = grads2d(P, 100 + i)
    rng = np.random.default_rng(200 + i)
    norms = 10.0 ** rng.uniform(-13.0, 3.0, P)
    compact = dict(opacity=g["opacity"], dL_dopacity=rng.normal(size=P).astype(np.float32),
                   rot_raw=(g["rots"] * norms[:, None]).astype(np.float32))
    return g, cam, radii, clamped, (dm2, dco, dcol), mod, lam, compact


def run(i, A=pbr.MAG32, **kw):
    g, cam, radii, clamped, d2, mod, lam, compact = scene(i)
    c32, c64 = cams(cam)
    pose = mod == 1.0 and lam == 0.0          # the compact + pose form runs with scale_modifier 1 and no regulariser
    return pbr.backward(g, c64 if A is pbr.MAG64 else c32, radii, clamped, *d2, mod=mod, lambda_erank=lam,
                        compact=compact if pose else None, pose=pose, A=A, **kw)


NINE = ("dmeans3D", "dcov3D", "ddc", "dsh", "dscales", "drots")
COMPACT = ("g_xyz", "g_scale", "g_rot", "g_opacity")


@pytest.mark.parametrize("i", range(len(CASES)), ids=IDS)
def test_matches_float64_oracle(oracle64, i):
    g, cam, radii, clamped, (dm2, dco, dcol), mod, lam, _ = scene(i)
    ref = oracle64.preprocess_backward(g, cam, radii, clamped, dm2, dco, dcol, float(np.float32(mod)), lam)
    got = run(i, pbr.MAG64)
    r = {}
    for k in NINE:
        a = ref["dL_" + k].reshape(got[k].v.shape)
        err = np.abs(a - got[k].v)
        r[k] = float(np.where(err == 0.0, 0.0, err / np.maximum(got[k].m, 1e-300)).max()) if err.size else 0.0
    print("%s: max |oracle - v| / m: %s  paths %s" % (IDS[i], r, got["paths"]))
    assert max(r.values()) <= 1e-12, r
    # the regulariser's cases reach both sides of its branch
    if lam:
        assert got["paths"]["erank_in"] > 0 and got["paths"]["erank_out"] > 0


@pytest.mark.parametrize("i", range(len(CASES)), ids=IDS)
def test_float32_evaluation_within_bounds(i):
    """the same arithmetic in numpy float32 (one rounding per operation, branches on its own values) against the bounds:
    the constants hold for a float32 evaluation in the kernel's order"""
    ref = run(i)
    alt = run(i, flip=ref["band"])
    f32 = run(i, pbr.F32)
    band = np.any(list(ref["band"].values()), 0)
    r = {k: pbr.either_ratio(f32[k], ref[k], alt[k], pbr.BOUND[k], band) for k in NINE + (COMPACT if "g_xyz" in ref else ())}
    if "pose" in ref:
        r["pose"] = float(np.abs(f32["pose"] - ref["pose"].v).max() / (pbr.BOUND["pose"] * pbr.U * ref["pose"].m).max())
    print("%s: float32 evaluation, max err / bound: %s  band rows %d" % (IDS[i], {k: round(v, 3) for k, v in r.items()}, band.sum()))
    assert max(r.values()) <= 1.0, r


def test_compact_chain_matches_autograd():
    """g_opacity, g_scale, g_rot of the compact form against torch float64 autograd of sigmoid, exp and normalize (eps = the
    kernel's float32 1e-12) with the restatement's dL/d(opacity, scale, rotation) upstream; raw rotation norms 1e-13 .. 1e3"""
    torch = pytest.importorskip("torch")
    tot = 0
    for i in range(len(CASES)):
        out = run(i, pbr.MAG64)
        if "g_rot" not in out:
            continue
        g, cam, radii, clamped, d2, mod, lam, compact = scene(i)
        vis = np.asarray(radii) > 0
        rr = torch.tensor(compact["rot_raw"][vis], dtype=torch.float64, requires_grad=True)
        ls = torch.tensor(np.log(g["scales"][vis].astype(np.float64)), requires_grad=True)
        o = g["opacity"][vis].astype(np.float64)
        with np.errstate(divide="ignore"):
            lg = torch.tensor(np.log(o) - np.log1p(-o), requires_grad=True)     # opacity 1: logit +inf, the gradient 0
        q = torch.nn.functional.normalize(rr, dim=1, eps=pbr.NORM_EPS)
        L = ((q * torch.tensor(out["drots"].v[vis])).sum() + (torch.exp(ls) * torch.tensor(out["dscales"].v[vis])).sum() +
             (torch.sigmoid(lg) * torch.tensor(compact["dL_dopacity"][vis].astype(np.float64))).sum())
        L.backward()
        nb = ~out["band"]["nn"][vis]
        for name, ref in (("g_rot", rr.grad.numpy()), ("g_scale", ls.grad.numpy()), ("g_opacity", lg.grad.numpy())):
            got = out[name]
            v, m = got.v[vis], got.m[vis]
            err = np.abs(v - ref)[nb]
            r = float(np.where(err == 0.0, 0.0, err / np.maximum(m[nb], 1e-300)).max())
            print("%s %s: max |autograd - v| / m = %.3e" % (IDS[i], name, r))
            assert r <= 1e-12, (IDS[i], name, r)
        tot += int((np.linalg.norm(compact["rot_raw"][vis].astype(np.float64), axis=1) <= pbr.NORM_EPS).sum())
    assert tot > 0                                               # the normalize guard was reached


def test_pose_sum_matches_pose_oracle():
    """the six pose floats (the sum of every row's terms) against pose_oracle.pose_gradient on the restatement's own
    dL/dmeans3D and the same 2-D gradients"""
    import pose_oracle
    n = 0
    for i in range(len(CASES)):
        out = run(i, pbr.MAG64)
        if "pose" not in out:
            continue
        g, cam, radii, clamped, (dm2, dco, dcol), *_ = scene(i)
        conic4 = np.stack([dco[:, 0], dco[:, 1], np.zeros_like(dco[:, 0]), dco[:, 2]], 1)
        ref = pose_oracle.pose_gradient(g, cam, dict(radii=radii), dict(dL_dmeans2D=dm2, dL_dconic=conic4,
                                                                         dL_dmeans3D=out["dmeans3D"].v))
        r = float((np.abs(ref - out["pose"].v) / out["pose"].m).max())
        print("%s: pose |pose_oracle - v| / m = %.3e" % (IDS[i], r))
        assert r <= 1e-12, (IDS[i], ref, out["pose"].v)
        n += 1
    assert n >= 3


def _caught(i, mutation):
    """max err / bound of the mutated restatement against the bound of the unmutated one, per output"""
    ref = run(i)
    mut = run(i, mutate=mutation)
    r = {k: pbr.either_ratio(mut[k].v, ref[k], None, pbr.BOUND[k], None) for k in NINE + COMPACT if k in ref}
    if "pose" in ref:
        r["pose"] = float((np.abs(mut["pose"].v - ref["pose"].v) / (pbr.BOUND["pose"] * pbr.U * ref["pose"].m)).max())
    return r


@pytest.mark.parametrize("mutation", pbr.MUTATIONS)
def test_mutation_is_caught(mutation):
    best = {}
    for i in range(len(CASES)):
        for k, v in _caught(i, mutation).items():
            if v > best.get(k, (0.0, ""))[0]:
                best[k] = (v, IDS[i])
    print("%s: max err / bound per output %s" % (mutation, {k: "%.3g (%s)" % v for k, v in best.items()}))
    assert max(v for v, _ in best.values()) > 1.0, (mutation, best)
