"""Checks of tests/render_blend_reference.py itself, on the CPU: its values against the float64 C oracle's render forward and
backward (glic_oracle_render / glic_oracle_render_backward, fed the same float64 state) and against torch float64 autograd;
a float32 evaluation in the kernels' order (render_blend_reference.F32) stays inside the bounds; and each plausible kernel bug
of render_blend_reference.MUTATIONS, applied to that evaluation, pushes some element beyond them."""
import functools
import time

import numpy as np
import pytest

import render_blend_reference as rb
from helpers import POSES, small_scene
from loss_reference import U

STRESS = [("needles", False), ("big", False), ("deep", False), ("deep", True), ("ties", False), ("edges", False)]
# share of a frame's pixels whose decisions may lie within rounding of a threshold: a handful in ordinary scenes; the needles
# put many pixels of their footprint's rim within rounding of 1/255 (the power of a needle conic cancels), and the big splats
# end many pixels after chains of hundreds of splats, whose T is uncertain by as many roundings
FLAG_SHARE = dict(needles=0.08, big=0.01)


def flag_limit(kind, pixels):
    return max(64, int(FLAG_SHARE.get(kind, 2e-3) * pixels))


def stress_scene(kind, opaque, view=0, pp=(0.0, 0.0)):
    from gaussian_lic_b200 import synthetic as syn
    return syn.make_stress_scene(kind, view=view, pp=pp, opaque=opaque)


def normal_dL(fw, H, W, seed):
    """dL/dpix ~ N(0, 1), exactly zero at the flagged pixels"""
    dL = np.random.default_rng(seed).normal(size=(3, H, W)).astype(np.float32)
    dL[:, rb.frame(fw["flag"], fw, H, W, False)] = 0.0
    return dL


def _grads(o):
    return np.concatenate([o["dmean2D"], o["dconic"], o["dcolor"], o["dopacity"][:, None]], 1)


# ---- agreement with the float64 C oracle --------------------------------------------------------------------------------------
CASES64 = [("small", False) + p for p in POSES] + [s + POSES[0] for s in STRESS]


@pytest.mark.parametrize("kind,opaque,view,pp", CASES64, ids=["%s%s-v%d-pp%g_%g" % (k, "-high" if o else "", v, p[0], p[1])
                                                              for k, o, v, p in CASES64])
def test_agrees_with_float64_oracle(oracle64, kind, opaque, view, pp):
    g, cam = small_scene(view=view, pp=pp) if kind == "small" else stress_scene(kind, opaque, view, pp)
    W, H = cam["W"], cam["H"]
    f = oracle64.forward(g, cam)
    st = oracle64.state(f)
    t0 = time.time()
    fw = rb.walk(st, W, H, consts=rb.EXACT)
    t1 = time.time()
    col, fT, nc, mc = oracle64.render(W, H, st["ranges"], st["point_list"], st["xy"], st["conic_opacity"], st["rgb"])
    ok = fw["inside"] & ~fw["flag"]
    nflag = int((fw["flag"] & fw["inside"]).sum())
    gcol = rb._gather_pix(col, fw["px"], fw["py"], fw["inside"])
    gT = rb._gather_pix(fT, fw["px"], fw["py"], fw["inside"])
    gnc = rb._gather_pix(nc.reshape(H, W), fw["px"], fw["py"], fw["inside"])
    rc = max(rb.ratio(gcol[c][ok], fw["C_v"][c][ok], 1e-12 * fw["C_m"][c][ok]).max() for c in range(3))
    rt = rb.ratio(gT[ok], fw["T_v"][ok], 1e-12 * fw["T_m"][ok]).max()
    assert (gnc[ok] == fw["last"][ok]).all()
    clean = ~(fw["flag"] & fw["inside"]).any(1)
    assert (mc[fw["tiles"]][clean] == fw["max_contrib"][clean]).all()
    dL = normal_dL(fw, H, W, view)
    bw = rb.walk(st, W, H, dL=dL, Cf=fw["C"], consts=rb.EXACT)
    t2 = time.time()
    v, m, _ = rb.per_gaussian(bw, st["point_list"], st["xy"].shape[0])
    ref = _grads(oracle64.render_backward(W, H, st["ranges"], st["point_list"], st["xy"], st["conic_opacity"], st["rgb"], nc, col, dL))
    rg = rb.ratio(ref, v, 1e-12 * m).max(0)
    print("\n%s: flagged %d px, C %.2e T %.2e grads %s (of 1e-12 m); walk %.1f s forward, %.1f s forward + backward; %s"
          % (kind, nflag, rc, rt, np.array2string(rg, precision=2), t1 - t0, t2 - t1, fw["paths"]))
    assert rc <= 1.0 and rt <= 1.0 and rg.max() <= 1.0
    assert nflag <= flag_limit(kind, W * H), nflag
    oracle64.free(f)


# ---- agreement with torch float64 autograd ------------------------------------------------------------------------------------
def _tiny_state(seed, W=40, H=24, P=30):
    """P splats over a W x H frame, every tile's list holding all of them in index order; opaque ones so that the 0.99 clamp
    acts and pixels end"""
    rng = np.random.default_rng(seed)
    xy = np.stack([rng.uniform(-4, W + 4, P), rng.uniform(-4, H + 4, P)], 1)
    s = rng.uniform(1.5, 8.0, (P, 2))
    th = rng.uniform(0, np.pi, P)
    c, sn = np.cos(th), np.sin(th)
    cov = np.zeros((P, 2, 2))
    for i in range(P):
        Rm = np.array([[c[i], -sn[i]], [sn[i], c[i]]])
        cov[i] = Rm @ np.diag(s[i] ** 2) @ Rm.T
    inv = np.linalg.inv(cov)
    op = rng.uniform(0.02, 0.9, P)
    op[rng.random(P) < 0.5] = 1.0
    xy[:4] = [W / 2, H / 2] + rng.uniform(-2, 2, (4, 2))         # four opaque splats over the middle: pixels there end
    op[:4] = 1.0
    co = np.stack([inv[:, 0, 0], inv[:, 0, 1], inv[:, 1, 1], op], 1)
    T = ((W + 15) // 16) * ((H + 15) // 16)
    st = dict(xy=xy.astype(np.float32), conic_opacity=co.astype(np.float32), rgb=rng.random((P, 3)).astype(np.float32),
              point_list=np.tile(np.arange(P, dtype=np.uint32), T),
              ranges=np.stack([np.arange(T) * P, np.arange(T) * P + P], 1).astype(np.uint32))
    return st, W, H


def _torch_grads(st, W, H, dL):
    torch = pytest.importorskip("torch")
    d = lambda a: torch.tensor(np.asarray(a, np.float64), requires_grad=True)
    xy, co, rgb = d(st["xy"]), d(st["conic_opacity"]), d(st["rgb"])
    py, px = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    px, py = torch.tensor(px.reshape(-1)), torch.tensor(py.reshape(-1))
    T = torch.ones(H * W, dtype=torch.float64)
    C = torch.zeros(3, H * W, dtype=torch.float64)
    live = torch.ones(H * W, dtype=torch.bool)
    for i in range(xy.shape[0]):                      # every tile lists all splats in index order
        dx, dy = xy[i, 0] - px, xy[i, 1] - py
        power = -0.5 * (co[i, 0] * dx * dx + co[i, 2] * dy * dy) - co[i, 1] * dx * dy
        oG = co[i, 3] * torch.exp(power)
        a = oG - (oG - 0.99).clamp(min=0).detach()    # the clamp, straight-through: dL/dG = o dL/dalpha
        take = live & (power.detach() <= 0) & (a.detach() >= 1.0 / 255.0)
        end = take & (T.detach() * (1 - a.detach()) < 1e-4)
        take = take & ~end
        live = live & ~end
        C = C + torch.where(take, T * a, torch.zeros_like(T))[None] * rgb[i][:, None]
        T = torch.where(take, T * (1 - a), T)
    (C * torch.tensor(np.asarray(dL, np.float64).reshape(3, -1))).sum().backward()
    gxy, gco = xy.grad.numpy(), co.grad.numpy()
    # the kernel's convention: dL/dmean2D in NDC (0.5 W, 0.5 H), dL/dconic.y half the derivative by the off-diagonal entry
    return np.concatenate([gxy * [0.5 * W, 0.5 * H], gco[:, :1], 0.5 * gco[:, 1:2], gco[:, 2:3], rgb.grad.numpy(), gco[:, 3:4]], 1)


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_agrees_with_torch_autograd(seed):
    st, W, H = _tiny_state(seed)
    fw = rb.walk(st, W, H, consts=rb.EXACT)
    dL = normal_dL(fw, H, W, seed)
    bw = rb.walk(st, W, H, dL=dL, Cf=fw["C"], consts=rb.EXACT)
    v, m, _ = rb.per_gaussian(bw, st["point_list"], st["xy"].shape[0])
    ref = _torch_grads(st, W, H, dL)
    r = rb.ratio(ref, v, 1e-12 * m).max(0)
    print("\nseed %d: %s (of 1e-12 m), paths %s" % (seed, np.array2string(r, precision=2), fw["paths"]))
    assert r.max() <= 1.0
    assert fw["paths"]["clamped"] > 0 and fw["paths"]["ended"] > 0


# ---- the float32 evaluation in the kernels' order stays inside the bounds; each mutant leaves them -----------------------------
@functools.lru_cache(maxsize=None)
def _f32_case(name):
    """(state, W, H, hy, restatement forward, restatement backward, dL) of a scene in its float32 oracle state"""
    from oracle.oracle import Oracle
    o32 = Oracle(np.float32)
    if name == "small":
        g, cam = small_scene(view=1)
    else:
        kind, _, opaque = name.partition("-")
        g, cam = stress_scene(kind, opaque == "high")
    W, H = cam["W"], cam["H"]
    f = o32.forward(g, cam)
    st = o32.state(f)
    hy = rb.half_extent(st["conic_opacity"], f["radii"])
    o32.free(f)
    fw = rb.walk(st, W, H)
    dL = normal_dL(fw, H, W, 7)
    bw = rb.walk(st, W, H, dL=dL, Cf=fw["C"])
    return st, W, H, hy, fw, bw, dL


def _f32_ratios(name, fast=True, rp=8, mutant=None):
    st, W, H, hy, fw, bw, dL = _f32_case(name)
    e = rb.walk(st, W, H, A=rb.F32, hy=hy, fast=fast, rp=rp, mutant=mutant)
    eb = rb.walk(st, W, H, A=rb.F32, dL=dL, Cf=e["C"], hy=hy, fast=fast, rp=rp, mutant=mutant)
    ok = fw["inside"] & ~fw["flag"]
    r = dict(C=max(rb.ratio(e["C_v"][c][ok], fw["C_v"][c][ok], rb.BOUND["C"] * U * fw["C_m"][c][ok]).max() for c in range(3)),
             T=rb.ratio(e["T_v"][ok], fw["T_v"][ok], rb.BOUND["T"] * U * fw["T_m"][ok]).max(),
             n_contrib=float((e["last"][ok] != fw["last"][ok]).sum()))
    rp_ = rb.ratio(eb["pair_v"], bw["pair_v"], rb.pair_bound(bw["pair_m"])).max(0)
    for k in ("mean", "conic", "color", "opacity"):
        r["pair_" + k] = float(max(x for x, kk in zip(rp_, rb.PAIR_KEYS) if kk == k))
    # the per-Gaussian sums of the emulated entries, added in float32 as atomics would (a fixed order stands for any)
    P = st["xy"].shape[0]
    v, m, cnt = rb.per_gaussian(bw, st["point_list"], P)
    s = np.zeros((P, 9), np.float32)
    pl = np.asarray(st["point_list"]).astype(np.int64)
    for k in range(9):
        np.add.at(s[:, k], pl, eb["pair_v"][:, k].astype(np.float32))
    r["gaussian"] = float(rb.ratio(s, v, rb.pair_bound(m, 5.0 + cnt * (8 // rp))).max())
    return r


F32_CASES = [("small", True, 8), ("small", False, 8), ("small", True, 4), ("deep-high", True, 8), ("deep-high", False, 8),
             ("needles", True, 8), ("edges", True, 4), ("ties", True, 8)]


@pytest.mark.parametrize("name,fast,rp", F32_CASES, ids=["%s-%s-rp%d" % (n, "fast" if f else "exact", r) for n, f, r in F32_CASES])
def test_float32_evaluation_within_bounds(name, fast, rp):
    r = _f32_ratios(name, fast, rp)
    print("\n%s fast=%s rp=%d: %s" % (name, fast, rp, "  ".join("%s %.3f" % kv for kv in r.items())))
    assert r.pop("n_contrib") == 0
    assert max(r.values()) <= 1.0, r


@pytest.mark.parametrize("mutant", rb.MUTATIONS)
def test_mutant_leaves_the_bounds(mutant):
    r = _f32_ratios("small", mutant=mutant)
    print("\n%s: %s" % (mutant, "  ".join("%s %.3g" % kv for kv in r.items())))
    assert r["n_contrib"] > 0 or max(v for k, v in r.items() if k != "n_contrib") > 1.0, r
