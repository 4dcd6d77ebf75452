"""csrc/preprocess.cu's per-Gaussian forward against the float64 restatement of tests/preprocess_forward_reference.py at every
Gaussian: depth, xy and conic within |got - v| <= c * 2^-24 * m (c in preprocess_forward_reference.BOUND), rgb likewise,
radius, tiles_touched and the clamp bits equal, and each row's accept set (read back from the sorted pair list) equal to the
float64 tile tests of its own record.  Rows whose decision lies within rounding of its threshold may take either side; each
case asserts that only a few rows are there and prints the count.  The render row cull's half-extent hy (read from the splat
records) must be at least the float64 half-height of {alpha >= 1/255}: the cull may be loose, never tight.

1. Every Gaussian of glic_forward: small_scene at SH degrees 0-3 x POSES, the stress scenes of test_gpu_stress.py, a cfg2 view.
2. The SH row layouts: the forward stages the CTA's SH rows into shared memory by one TMA bulk copy (preprocess.cu, when the
   run is 16-byte aligned and a multiple of 16 bytes), else by warp copies of 128-bit loads plus a scalar tail (warp_rows.cuh,
   aligned rows) or of scalar loads (unaligned rows), and reads rows of more than 45 floats (M >= 16) from global memory
   unstaged; the backward loads and stores its warp's SH slab with the same two warp copies, or works unstaged.  The C ABI
   accepts any M >= (D + 1)^2 - 1 and requires alignment of the rotations only, so each of these paths takes legal inputs.
   LAYOUTS offsets sh, dc, means, scales and opacity by 0-12 bytes inside larger buffers and pads the SH rows with NaN
   coefficients past the degree; the forward's records, radii, image, final_T and sorted keys and all ten backward outputs
   (glic_backward_deterministic, whose render backward adds the tile contributions in a fixed order, so that the 2-D gradients
   fed to the per-Gaussian backward are bit-reproducible) must be bit-identical to those of the same scene in aligned, unpadded
   tensors, and dL_dsh's rows past the degree exact zeros.  dL_dsh is NaN before the call (glic_backward clears only the 2-D
   gradients), so every element the test reads was written by the kernel, and the NaN floats around it must stay NaN.
   staging_paths() counts which path each forward CTA and backward warp takes, by the kernels' own rules; every one is reached.
3. glic_render, the no_color forward and glic_contribution share the forward: the same radii (and tile lists) on a subset,
   the no_color forward and glic_render each on workspaces cleared before the call, glic_contribution into a fresh radii.

Run with -s to see max(err / bound) per output, the band rows and the path counts.
"""
import numpy as np
import pytest

import preprocess_backward_reference as pbr
import preprocess_forward_reference as pfr
from helpers import CFG2_P, POSES, small_scene
from test_gpu_stress import CASES as STRESS_CASES
from test_preprocess_backward_reference_host import cams
from test_preprocess_forward_reference_host import band_limit

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

DEV = "cuda:0"
FLOATS = ("depth", "xy", "conic", "rgb")
SH_ROW_MAX = 45                 # warp_rows.cuh: the largest staged row, in floats
PRE_THREADS, PB_THREADS = 256, 128
GEOM_HDR = 128                  # common.cuh: GeomState::carve puts the splat records after the 128-byte header


def records(r, P):
    """the 48-byte splat records of the last forward: [P, 12] float32 (x, y, conic.x, conic.y | conic.z, o, r, g | b, depth,
    radius bits, hy)"""
    raw = r.geom_ws[GEOM_HDR:GEOM_HDR + 48 * P].cpu().numpy()
    return raw.view(np.float32).reshape(P, 12)


def gpu_state(r, P):
    d = r.debug_state()
    st = {k: d[k].cpu().numpy() for k in ("depth", "xy", "conic_opacity", "rgb", "tiles_touched", "clamped")}
    T = ((r.W + 15) // 16) * ((r.H + 15) // 16)
    st["pairs"] = np.sort(d["point_list"].cpu().numpy().astype(np.int64) * T +
                          (d["keys_sorted"].cpu().numpy().view(np.uint64) >> 32).astype(np.int64))
    st["keys_sorted"] = d["keys_sorted"].cpu().numpy()
    rec = records(r, P)
    # the record read-back sits where debug_geom reads: the same xy and conic bits
    np.testing.assert_array_equal(rec[:, :2].view(np.uint32), st["xy"].view(np.uint32))
    np.testing.assert_array_equal(rec[:, 2:5].view(np.uint32), st["conic_opacity"][:, :3].view(np.uint32))
    st["hy"] = rec[:, 11]
    return st


def check_exact(g, cam, st, radii, what, kind="small", view=0, pp=(0.0, 0.0), mod=1.0):
    """one forward's state against the restatement; returns (ratios, paths)"""
    c32, _ = cams(cam)
    ref = pfr.forward(g, c32, mod=mod)
    got = dict(radius=radii, tiles=st["tiles_touched"], clamped=st["clamped"], pairs=st["pairs"])
    rec = pfr.record_accept_sets(st["xy"], st["conic_opacity"], radii, cam["W"], cam["H"])
    bad, rows = pfr.compare(ref, got, rec)
    vis = (np.asarray(st["tiles_touched"]) > 0) & ref["vis"]
    fl = dict(depth=st["depth"], xy=st["xy"], conic=st["conic_opacity"][:, :3], rgb=st["rgb"])
    ratios = {k: pfr.ratio(fl[k], ref[k], pfr.BOUND[k], vis) for k in FLOATS}
    gvis = np.asarray(st["tiles_touched"]) > 0
    need = pfr.half_height(st["conic_opacity"], ref["cov"], gvis)
    short = gvis & ~(st["hy"] >= need)
    ratios["hy_short"] = float(short.sum())
    paths = dict(ref["paths"], band_rows=int(rows.sum()), unsure_pairs=int(rec["unsure_pairs"].size),
                 pairs=int(st["pairs"].size), min_hy_over_need=float(np.min((st["hy"] / np.where(need > 0, need, 1))[gvis]))
                 if gvis.any() else 0.0)
    print("\n%s: %s  band rows %d\n    paths %s" % (what, "  ".join("%s %.3f" % kv for kv in sorted(ratios.items())),
                                                   rows.sum(), paths))
    assert all(len(v) == 0 for v in bad.values()), {k: v[:8] for k, v in bad.items() if len(v)}
    assert not short.any(), ("hy below the half-height", np.flatnonzero(short)[:8], st["hy"][short][:8], need[short][:8])
    assert max(ratios[k] for k in FLOATS) <= 1.0, ratios
    assert rows.sum() <= band_limit(kind, rows.size, view, pp), (rows.sum(), rows.size)
    return ratios, paths


def forward_on_gpu(g, cam, gd=None, mod=1.0):
    from gaussian_lic_b200 import ops
    r = ops.CRasterizer(cam["W"], cam["H"])
    gd = ops.scene_to_device(g) if gd is None else gd
    view = r.make_view(cam)
    color, T, radii = r.forward(gd, view, scale_modifier=mod)
    torch.cuda.synchronize()
    P = int(gd["means"].shape[0])
    return r, gd, view, color, T, radii, gpu_state(r, P)


# ---- 1. every Gaussian of glic_forward ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("deg", [0, 1, 2, 3])
@pytest.mark.parametrize("view,pp", POSES, ids=["v%d-pp%g_%g" % (v, p[0], p[1]) for v, p in POSES])
def test_small_scene(deg, view, pp):
    g, cam = small_scene(deg=deg, view=view, pp=pp)
    r, gd, v, color, T, radii, st = forward_on_gpu(g, cam)
    _, paths = check_exact(g, cam, st, radii.cpu().numpy(), "small deg %d view %d pp %s" % (deg, view, pp))
    assert paths["visible"] > 0 and (deg == 0 or min(paths["clamped"]) > 0)


@pytest.mark.parametrize("kind,opaque,view,pp", STRESS_CASES)
def test_stress_scene(kind, opaque, view, pp):
    from gaussian_lic_b200 import synthetic as syn
    g, cam = syn.make_stress_scene(kind, view=view, pp=pp, opaque=opaque)
    r, gd, v, color, T, radii, st = forward_on_gpu(g, cam)
    check_exact(g, cam, st, radii.cpu().numpy(), "stress %s%s view %d pp %s" % (kind, "-high" if opaque else "", view, pp), kind,
                view, pp)


def test_cfg2_view():
    from gaussian_lic_b200 import synthetic as syn
    g, cam = syn.make_scene("cfg2", P=CFG2_P, view=5, pp=(41.5, -27.25))
    r, gd, v, color, T, radii, st = forward_on_gpu(g, cam)
    check_exact(g, cam, st, radii.cpu().numpy(), "cfg2 view 5")


# ---- 2. the SH row layouts -------------------------------------------------------------------------------------------------------
def _aligned16(byte_offset):
    return byte_offset % 16 == 0


def staging_paths(P, D, M, sh_off, dsh_off, no_color=False):
    """which SH staging path each forward CTA and each backward warp takes, by the kernels' rules (byte offsets of sh and dL_dsh
    from a 16-byte aligned base):
      forward (preprocess.cu, preprocess_forward_kernel, where sh_tma / sh_staged are set): nothing staged unless !no_color,
        D > 0 and K = 3M <= SH_ROW_MAX ("unstaged": rows read from global memory where the colour is evaluated); TMA when the
        CTA's run of bcnt * K floats is a multiple of 16 bytes and starts 16-byte aligned; else warp_load_rows per warp,
        whose 128-bit loop plus scalar tail runs when the warp's run starts aligned ("warp_vec"; "warp_vec_tail" when the run
        is not a multiple of 4 floats, so the tail loop has work) and the scalar loop when it does not ("warp_scalar");
      backward (preprocess_backward.cu, preprocess_backward_kernel: `staged`, warp_load_rows, warp_store_rows): warps with no
        row return; staged when 0 < K <= SH_ROW_MAX, the load (D > 0) and the store each 128-bit + tail or scalar by the
        alignment of the warp's run; "unstaged" when K > SH_ROW_MAX."""
    K = 3 * M
    c = dict(f_tma=0, f_warp_vec=0, f_warp_vec_tail=0, f_warp_scalar=0, f_unstaged=0, b_load_vec=0, b_load_scalar=0,
             b_store_vec=0, b_store_scalar=0, b_unstaged=0)
    for b in range((P + PRE_THREADS - 1) // PRE_THREADS):
        if no_color or D == 0:
            continue
        if K > SH_ROW_MAX:
            c["f_unstaged"] += 1
            continue
        bfirst = b * PRE_THREADS
        bcnt = min(PRE_THREADS, P - bfirst)
        src = sh_off + 4 * bfirst * K
        if (bcnt * K * 4) % 16 == 0 and _aligned16(src):
            c["f_tma"] += 1
            continue
        for w in range(PRE_THREADS // 32):
            wfirst = bfirst + 32 * w
            wcnt = min(32, P - wfirst)
            if wcnt <= 0:
                continue
            if _aligned16(sh_off + 4 * wfirst * K):
                c["f_warp_vec_tail" if (wcnt * K) % 4 else "f_warp_vec"] += 1
            else:
                c["f_warp_scalar"] += 1
    for w in range((P + 31) // 32):
        wfirst = 32 * w
        if K == 0:
            continue
        if K > SH_ROW_MAX:
            c["b_unstaged"] += 1
            continue
        if D > 0:
            c["b_load_vec" if _aligned16(sh_off + 4 * wfirst * K) else "b_load_scalar"] += 1
        c["b_store_vec" if _aligned16(dsh_off + 4 * wfirst * K) else "b_store_scalar"] += 1
    return c


# (D, P, byte offset, M): every degree, P, offset and M of the issue's ranges, chosen so that every staging path is reached
LAYOUTS = [(3, 4099, 0, 15), (3, 4097, 4, 15), (1, 257, 8, 3), (1, 33, 0, 3), (2, 259, 12, 8), (2, 31, 0, 15),
           (3, 255, 0, 16), (1, 4099, 4, 24), (2, 1, 8, 16), (3, 1, 12, 15), (2, 4097, 0, 8), (1, 255, 12, 15),
           (3, 259, 8, 24), (2, 33, 4, 24), (1, 31, 0, 16), (3, 257, 0, 15)]
LAYOUT_IDS = ["d%d-P%d-off%d-M%d" % c for c in LAYOUTS]


GUARD = 4                       # NaN floats after each placed tensor (and the offset's floats before it)


def _placed(a, off_bytes, with_buffer=False):
    """a float32 numpy array as a device tensor starting `off_bytes` past a 512-byte aligned allocation (a view into it); the
    floats of the allocation around it are NaN"""
    a = np.ascontiguousarray(a, np.float32)
    o = off_bytes // 4
    buf = torch.full((a.size + o + GUARD,), float("nan"), dtype=torch.float32, device=DEV)
    t = buf[o:o + a.size].view(a.shape)
    t.copy_(torch.as_tensor(a))
    assert t.data_ptr() % 16 == off_bytes % 16
    return (t, buf, o) if with_buffer else t


def _layout_scene(D, P):
    g, cam = small_scene(P=P, deg=D, zmax=6.0, log_scale_mean=-2.0)
    return g, cam


def _padded(g, M):
    """g with SH rows of M coefficients: the degree's coefficients, then NaN"""
    P, nb = g["means"].shape[0], pfr.sh_count(int(g["degree"]))
    sh = np.full((P, M, 3), np.nan, np.float32)
    sh[:, :nb] = g["sh"][:, :nb]
    return dict(g, sh=sh)


def _run_both(gd, cam, dL, dsh_off=0):
    from gaussian_lic_b200 import ops
    r = ops.CRasterizer(cam["W"], cam["H"])
    view = r.make_view(cam)
    color, T, radii = r.forward(gd, view)
    torch.cuda.synchronize()
    P = int(gd["means"].shape[0])
    st = gpu_state(r, P)
    st["rec"] = records(r, P)
    grads = r.alloc_grads()
    M = r.M
    if M:
        # NaN everywhere: every element of dL_dsh must be written by the kernel (glic_backward does not clear it), and the
        # guard floats around it must stay NaN
        grads["dL_dsh"], buf, o = _placed(np.full((P, M, 3), np.nan, np.float32), dsh_off, with_buffer=True)
    grads = r.backward(gd, view, radii, dL, grads=grads, deterministic=True)
    torch.cuda.synchronize()
    out = {k: t.cpu().numpy() for k, t in grads.items()}
    if M:
        b = buf.cpu().numpy()
        n = P * M * 3
        assert np.isnan(b[:o]).all() and np.isnan(b[o + n:]).all(), "dL_dsh written outside its rows"
        assert not np.isnan(out["dL_dsh"]).any(), "dL_dsh elements left unwritten: %d" % int(np.isnan(out["dL_dsh"]).sum())
    return r, view, color.cpu().numpy(), T.cpu().numpy(), radii.cpu().numpy(), st, out


NINE = ("dL_dmeans2D", "dL_dconic", "dL_dopacity", "dL_dcolors", "dL_dmeans3D", "dL_dcov3D", "dL_ddc", "dL_dsh", "dL_dscales",
        "dL_drots")


@pytest.mark.parametrize("D,P,off,M", LAYOUTS, ids=LAYOUT_IDS)
def test_sh_row_layouts(D, P, off, M):
    from gaussian_lic_b200 import ops
    g, cam = _layout_scene(D, P)
    nb = pfr.sh_count(D)
    dL = torch.as_tensor(np.random.default_rng(P + D).normal(size=(3, cam["H"], cam["W"])).astype(np.float32)).to(DEV)
    base = _run_both(ops.scene_to_device(g), cam, dL)
    gp = _padded(g, M)
    gd = dict(degree=D, rots=torch.as_tensor(gp["rots"]).to(DEV).contiguous())
    for k in ("means", "scales", "opacity", "dc", "sh"):
        gd[k] = _placed(gp[k], off)
    lay = _run_both(gd, cam, dL, dsh_off=off)
    _, _, c0, T0, r0, s0, b0 = base
    r, view, c1, T1, r1, s1, b1 = lay
    same = lambda a, b_, what: np.testing.assert_array_equal(np.asarray(a).view(np.uint32), np.asarray(b_).view(np.uint32),
                                                             err_msg=what)
    np.testing.assert_array_equal(r1, r0)
    same(s1["rec"], s0["rec"], "splat records")
    same(c1, c0, "image")
    same(T1, T0, "final_T")
    np.testing.assert_array_equal(s1["keys_sorted"], s0["keys_sorted"])
    np.testing.assert_array_equal(s1["pairs"], s0["pairs"])
    np.testing.assert_array_equal(s1["clamped"], s0["clamped"])
    for k in NINE:
        a, b_ = b1[k], b0[k]
        if k == "dL_dsh":
            assert np.all(a[:, nb:] == 0.0), "dL_dsh rows past the degree are not exact zeros"     # (NaN before the call)
            a = a[:, :nb]
        same(a, b_.reshape(a.shape), k)
    # rgb against its bound, and the visible rows
    ratios, paths = check_exact(gp, cam, s1, r1, "layout D %d P %d offset %d M %d" % (D, P, off, M))
    assert paths["visible"] > 0
    # the backward's bounds on every other case (check_nine's restatement, on the offset and padded tensors)
    if LAYOUTS.index((D, P, off, M)) % 2 == 0:
        d2 = [b1[k] for k in ("dL_dmeans2D", "dL_dconic", "dL_dcolors")]
        c32, _ = cams(cam)
        ref = pbr.backward(gp, c32, r1, s1["clamped"], *d2)
        alt = pbr.backward(gp, c32, r1, s1["clamped"], *d2, flip=ref["band"])
        band = np.any(list(ref["band"].values()), 0)
        got = {k: b1["dL_" + k] for k in ("dmeans3D", "dcov3D", "ddc", "dsh", "dscales", "drots")}
        got["dsh"] = got["dsh"].reshape(P, M, 3)
        br = {k: pbr.either_ratio(got[k], ref[k], alt[k], pbr.BOUND[k], band) for k in got}
        print("    backward max err / bound %s" % {k: round(v, 3) for k, v in br.items()})
        assert max(br.values()) <= 1.0, br
    print("    staging paths %s" % staging_paths(P, D, M, off, off))


def test_layouts_reach_every_staging_path():
    tot = {}
    for D, P, off, M in LAYOUTS:
        for k, v in staging_paths(P, D, M, off, off).items():
            tot[k] = tot.get(k, 0) + v
    print("\nstaging paths over LAYOUTS: %s" % tot)
    assert all(v > 0 for v in tot.values()), tot


# ---- 3. entry points that share the forward ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,P,off,M", LAYOUTS[::3], ids=LAYOUT_IDS[::3])
def test_entry_points_share_the_forward(D, P, off, M):
    from gaussian_lic_b200 import ops
    g, cam = _layout_scene(D, P)
    gp = _padded(g, M)
    gd = dict(degree=D, rots=torch.as_tensor(gp["rots"]).to(DEV).contiguous())
    for k in ("means", "scales", "opacity", "dc", "sh"):
        gd[k] = _placed(gp[k], off)
    r = ops.CRasterizer(cam["W"], cam["H"])
    view = r.make_view(cam)
    _, _, radii = r.forward(gd, view)
    torch.cuda.synchronize()
    ref_radii, ref_pairs = radii.cpu().numpy(), gpu_state(r, P)["pairs"]
    # the no_color forward, then glic_render, each on cleared workspaces: the lists read back are the call's own
    for ws in (r.geom_ws, r.binning_ws):
        ws.zero_()
    _, _, rn = r.forward(gd, view, no_color=True)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(rn.cpu().numpy(), ref_radii)
    np.testing.assert_array_equal(gpu_state(r, P)["pairs"], ref_pairs)
    for ws in (r.geom_ws, r.binning_ws):
        ws.zero_()
    out = r.render(gd, view)
    np.testing.assert_array_equal(out["radii"].cpu().numpy(), ref_radii)
    d = r.debug_render_state(out["counters"][0])
    pairs = np.sort(d["point_list"].cpu().numpy().astype(np.int64) * ((r.W + 15) // 16) * ((r.H + 15) // 16) +
                    (d["keys_sorted"].cpu().numpy().view(np.uint64) >> 32).astype(np.int64))
    np.testing.assert_array_equal(pairs, ref_pairs)
    # glic_contribution
    rc = torch.empty(P, dtype=torch.int32, device=DEV)
    mw = torch.zeros(P, dtype=torch.float32, device=DEV)
    hits = torch.zeros(P, dtype=torch.int64, device=DEV)
    r.contribution(gd, view, mw, hits, radii=rc)
    np.testing.assert_array_equal(rc.cpu().numpy(), ref_radii)
    print("\nentry points D %d P %d offset %d M %d: %d visible, %d pairs" % (D, P, off, M, (ref_radii > 0).sum(), ref_pairs.size))
