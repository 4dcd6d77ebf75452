"""The native mapper's gradients (csrc/mapper.cu) against the float64 CPU oracle, recovered exactly from its Adam moments.

The other mapper tests compare parameters after Adam, and this project's Adam (adam_math.cuh: no bias correction,
eps = 1e-15) takes the same step when every gradient element is multiplied by a positive factor that stays constant over
the steps: on a first step every visible entry moves by +-lr * 0.1 / sqrt(0.001), whatever the gradient's size.  A wrong
mean over views or ranks, a missing chain-rule factor or a stale accumulator would pass them.

Adam's first moment gives the gradient back: m' = fma(1 - b1, g, fl(b1 m)) rounds once, so in float64
    g = (m' - fl(b1 m)) / fl(1 - b1)
is the gradient the step used, for every parameter of every Gaussian that stepped, within 0.5 ulp(m') / 0.1.  Each test
downloads the parameters and moments before and after one step and compares that gradient, group by group, with the mean
over the batch's views of the f64 oracle's dL/d(raw parameter).  The oracle runs on the image and dL/dpixel the mapper
itself produced: the same kernels (activations, forward, fused L1 + SSIM loss) on the same inputs.
"""
import os
import socket

import numpy as np
import pytest

from helpers import grad_close, small_scene

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

W, H, F = 320, 208, 250.0
P = 6000                                     # not a multiple of 32: the last warp of adam_compact_kernel is partial
VIEWS = (0, 2, 5)                            # rig views (synthetic.orbit_pose) of the keyframes
GROUPS = ("rots", "means", "log_scales", "opacity_logits", "dc", "sh")      # arena order (glic_packed_offsets)
B1, B2, EPS = np.float32(0.9), np.float32(0.999), np.float32(1e-15)
C1 = np.float64(np.float32(1.0) - B1)        # 0.10000002384185791: 1 - b1 as the kernel rounds it (exact in f32)
C2 = np.float64(np.float32(1.0) - B2)
ZERO_Q, TINY_Q, LAST = 17, 18, P - 1         # edge rows: zero raw quaternion, |q| < 1e-12, a visible row in the last warp
EDGE = (ZERO_Q, TINY_Q)


def _lr6():
    """per-group learning rates as mapper.cu builds them from the float config (sh-rest: feature_lr / 20.0f)"""
    from gaussian_lic_b200.mapper import FASTLIVO
    f = {k: np.float32(v) for k, v in FASTLIVO.items()}
    return (f["rotation_lr"], f["position_lr"], f["scaling_lr"], f["opacity_lr"], f["feature_lr"], f["feature_lr"] / np.float32(20.0))


def _widths(M):
    return (4, 3, 3, 1, 3, 3 * M)


def _scene(deg, P_=P, seed=21):
    """small_scene's Gaussians plus the edge rows: a zero raw quaternion (normalize's 1e-12 branch, exact zero rotation
    gradient), one of norm 3.9e-13 (the same branch with a gradient scaled by 1e12), and a row of the partial last warp
    placed where every rig view sees it."""
    g, _ = small_scene(P_, W, H, seed, deg)
    raw = {k: np.array(g[k], np.float32) for k in ("means", "log_scales", "rots", "opacity_logits", "dc", "sh")}
    for i, xyz, q in ((ZERO_Q, (0.1, -0.1, 9.0), (0.0, 0.0, 0.0, 0.0)), (TINY_Q, (-0.3, 0.2, 9.5), (3e-13, -1e-13, 2e-13, 1e-13)),
                      (P_ - 1, (0.2, 0.3, 8.5), (0.9, 0.1, -0.3, 0.2))):
        raw["means"][i] = xyz
        raw["log_scales"][i] = np.log([0.08, 0.05, 0.11])
        raw["opacity_logits"][i] = 2.0
        raw["rots"][i] = q
    raw["degree"] = deg
    return raw


def _keyframes(seed=7):
    from gaussian_lic_b200 import mapper, synthetic as syn
    poses = [syn.orbit_pose(v, radius=2.0) for v in VIEWS]
    cams = [mapper.camera_block(W, H, F, F, W / 2.0, H / 2.0, R, t) for R, t in poses]
    gts = [syn.make_gt_image(W, H, seed=seed + i) for i in range(len(VIEWS))]
    return poses, cams, gts


def _mapper(raw, poses, gts, capacity=0, **kw):
    from gaussian_lic_b200 import mapper
    m = mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=raw["degree"], capacity=capacity, **kw)
    m.initialize(raw)
    for (R, t), img in zip(poses, gts):
        m.add_keyframe(R, t, img)
    return m


def _state(m):
    """parameters (p), exp_avg (m) and exp_avg_sq (v) of every group as [P, k] float32 arrays"""
    d = m.download(moments=True)
    n = d["means"].shape[0]
    out = dict(p={}, m={}, v={}, P=n, degree=int(m.cfg.sh_degree))
    for key, name in (("m", "exp_avg"), ("v", "exp_avg_sq")):
        o = 0
        for grp, k in zip(GROUPS, _widths(m.M)):
            out[key][grp] = d[name][o:o + n * k].reshape(n, k)
            o += n * k
    for grp, k in zip(GROUPS, _widths(m.M)):
        out["p"][grp] = d[grp].reshape(n, k)
    return out


def _raw(st):
    p, n = st["p"], st["P"]
    return dict(means=p["means"], log_scales=p["log_scales"], rots=p["rots"], opacity_logits=p["opacity_logits"].reshape(n),
                dc=p["dc"], sh=p["sh"].reshape(n, -1, 3) if p["sh"].size else np.zeros((n, 0, 3), np.float32), degree=st["degree"])


def _recovered(before, after):
    """the gradient each entry's step used: (m' - fl(b1 m)) / fl(1 - b1), in float64 (meaningful on the rows that stepped)"""
    return {g: (after["m"][g].astype(np.float64) - (B1 * before["m"][g]).astype(np.float64)) / C1 for g in GROUPS}


def _reference(raw, cams, gts, batch, oracles):
    """Mean over the batch's views of dL/d(raw parameters), per oracle, on the image and dL/dpixel the mapper rendered."""
    from gaussian_lic_b200 import model, ops
    dev = torch.device("cuda:0")
    n = raw["means"].shape[0]
    mdl = model.PackedModel(raw, dev)
    mdl.activate()
    rast = ops.CRasterizer(W, H, dev)
    out = dict(radii=[], clamped=[], loss=None, grads={})
    sums = {o.dtype.name: {g: 0.0 for g in GROUPS} for o in oracles}
    for v in batch:
        color, _, radii = rast.forward(mdl.inputs, rast.make_view(cams[v]))
        loss, dL = rast.loss(color, torch.as_tensor(gts[v]).to(dev), 0.2)
        torch.cuda.synchronize()
        dL = dL.cpu().numpy()
        out["loss"] = float(loss.item())
        out["radii"].append(radii.cpu().numpy().copy())
        for o in oracles:
            op, sc, rot = o.activations(raw["opacity_logits"], raw["log_scales"], raw["rots"])
            f = o.forward(dict(means=raw["means"], scales=sc, rots=rot, opacity=op, dc=raw["dc"], sh=raw["sh"], degree=raw["degree"]),
                          cams[v])
            b = o.backward(f, dL)
            if o.dtype == np.float64:
                out["clamped"].append(o.state(f)["clamped"].copy())
                out.setdefault("oracle_radii", []).append(f["radii"].copy())
            g_op, g_s, g_r = o.activations_backward(op, sc, raw["rots"], b["dL_dopacity"], b["dL_dscales"], b["dL_drots"])
            o.free(f)
            per = dict(rots=g_r, means=b["dL_dmeans3D"], log_scales=g_s, opacity_logits=g_op, dc=b["dL_ddc"], sh=b["dL_dsh"])
            acc = sums[o.dtype.name]
            for g in GROUPS:
                acc[g] = acc[g] + np.asarray(per[g], np.float64).reshape(n, -1)
    for name, acc in sums.items():
        out["grads"][name] = {g: acc[g] / len(batch) for g in GROUPS}
    out["vis"] = np.any([r > 0 for r in out["radii"]], axis=0)
    return out


def _yardstick(ref, rows, what):
    """how far the f32 oracle (the reference's own arithmetic) is from the f64 one on the same rows"""
    a, b = ref["grads"]["float32"], ref["grads"]["float64"]
    d = {}
    for g in GROUPS:
        r = np.setdiff1d(rows, EDGE) if g == "rots" else rows
        if b[g][r].size:
            d[g] = np.abs(a[g][r] - b[g][r]).max() / max(np.abs(b[g][r]).max(), 1e-12)
    print("%s: f32 oracle vs f64 oracle, max|diff|/max|ref|: %s" % (what, {g: "%.2e" % x for g, x in d.items()}))


def _compare(got, ref, rows, what, groups=GROUPS, rtol=None):
    """grad_close (test_gpu_parity.py's tolerances) on every group over the rows that stepped; the edge rows are kept out of
    the rotation group, whose scale the 1e12 factor of the tiny quaternion would set.  rtol: {group: norm tolerance} where a
    caller has measured that the f32 oracle itself is further than GRAD_RTOL from the f64 one (default GRAD_RTOL)."""
    want = ref["grads"]["float64"]
    n_or = int((np.any([r > 0 for r in ref["oracle_radii"]], axis=0) != ref["vis"]).sum())
    print("%s: %d Gaussians stepped, %d differ in visibility between the GPU and the f64 oracle" % (what, rows.size, n_or))
    _yardstick(ref, rows, what)
    for g in groups:
        r = np.setdiff1d(rows, EDGE) if g == "rots" else rows
        if want[g][r].size:
            grad_close(got[g][r], want[g][r], "%s: d %s" % (what, g), **({} if rtol is None else dict(rtol=rtol[g])))


def _recovery_bound(after):
    """per-entry bound of the recovery error, 0.5 ulp(m') / (1 - b1): a gradient far below the moment it is added to (a row
    whose gradient shrank by orders of magnitude since the last step) is lost in m''s rounding"""
    return {g: 0.5 * np.spacing(np.abs(after["m"][g])).astype(np.float64) / C1 for g in GROUPS}


def _check_edge_rows(got, ref, before, after, what):
    """The edge rows' rotation gradients on their own, within a relative 1e-5 of the oracle (plus the recovery bound).
    Returns whether the tiny quaternion took normalize's |r| <= 1e-12 branch in this step (its first step does; the step
    moves it by ~3 lr per component, out of that branch)."""
    want = ref["grads"]["float64"]["rots"]
    bound = _recovery_bound(after)["rots"]
    for i in EDGE:
        assert ref["vis"][i], "%s: edge row %d is not visible" % (what, i)
        err = np.abs(got["rots"][i] - want[i])
        scale = np.abs(want[i]).max()
        print("%s: edge row %d (|r| = %.2e): d rots %s vs oracle %s (max|diff|/max|ref| %.2e)" % (
            what, i, np.linalg.norm(before["p"]["rots"][i]), got["rots"][i], want[i], err.max() / max(scale, 1e-300)))
        assert np.all(err <= 1e-5 * scale + bound[i]), (what, i, got["rots"][i], want[i])
    assert not before["p"]["rots"][ZERO_Q].any() and not got["rots"][ZERO_Q].any()   # dR/dq is linear in q: zero at q = 0
    tiny = np.linalg.norm(before["p"]["rots"][TINY_Q].astype(np.float64)) < 1e-12
    if tiny:
        assert np.abs(want[TINY_Q]).max() > 1e5, what   # the 1e12 factor of the clamped branch
    return tiny


def _check_step(before, after, got, rows, lr6, what):
    """Adam itself, bit for bit: p' = p + (-lr m') / (sqrt(v') + eps) in float32; v' = b2 v + (1 - b2) g^2 to 1e-6"""
    for g, lr in zip(GROUPS, lr6):
        p, v = before["p"][g][rows], before["v"][g][rows].astype(np.float64)
        p1, m1, v1 = after["p"][g][rows], after["m"][g][rows], after["v"][g][rows]
        if p.size == 0:
            continue
        want = p + (-lr * m1) / (np.sqrt(v1) + EPS)
        assert want.dtype == np.float32
        bad = p1 != want
        assert not bad.any(), "%s: %d %s entries off the float32 Adam step (first %s vs %s)" % (what, bad.sum(), g, p1[bad][:4], want[bad][:4])
        vw = np.float64(B2) * v + C2 * got[g][rows] ** 2
        # + a few subnormal ulps: the gradient of an isotropic Gaussian's rotation is rounding noise whose square is subnormal
        assert np.all(np.abs(v1 - vw) <= 1e-6 * vw + 1e-44), "%s: exp_avg_sq of %s" % (what, g)


def _check_untouched(before, after, idle, what):
    """Gaussians visible in no view of the batch keep their parameters and both moments bit for bit"""
    assert idle.any(), what
    for key in ("p", "m", "v"):
        for g in GROUPS:
            a, b = before[key][g][idle], after[key][g][idle]
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), "%s: an idle row's %s / %s changed" % (what, key, g)


def _check_step_against_oracle(m, raw_before, before, after, cams, gts, batch, oracles, what):
    """everything one optimiser step must satisfy; returns the reference, the recovered gradient and whether the tiny
    quaternion took normalize's clamped branch"""
    ref = _reference(_raw(before), cams, gts, batch, oracles)
    st = m.stats()
    assert abs(st.last_loss - ref["loss"]) <= 1e-5 * ref["loss"], (what, st.last_loss, ref["loss"])   # atomic sum order only
    vis = ref["vis"]
    rows = np.flatnonzero(vis)
    got = _recovered(before, after)
    _compare(got, ref, rows, what)
    tiny = _check_edge_rows(got, ref, before, after, what)
    _check_step(before, after, got, rows, _lr6(), what)
    _check_untouched(before, after, ~vis, what)
    if raw_before["degree"] == 0:                          # reference quirk: no SH-rest tensor => no colour backward at all
        assert not got["dc"][rows].any() and not ref["grads"]["float64"]["dc"].any(), what
    else:                                                  # clamped channels reached the rebuilt colour gradient
        n_cl = sum(int(((c != 0).any(1) & (r > 0)).sum()) for c, r in zip(ref["clamped"], ref["radii"]))
        print("%s: %d (view, visible Gaussian) pairs with a clamped colour channel" % (what, n_cl))
        assert n_cl > 0, what
    return ref, got, tiny


# ---- 1. one view per step, two steps, all SH degrees, both zeroing branches of the 2-D accumulators --------------------
@pytest.mark.parametrize("capacity", [0, 6144])
@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_single_view_steps_match_oracle(oracle32, oracle64, deg, capacity):
    """Two steps on different views: the second runs on the other parity's colour and flag slots, takes the SH directions
    from the xyz the first step moved, and needs the accumulators the first step filled to be zeroed again.  Capacity
    6144 (7 * 6144 + P <= 10 P) zeroes the three 2-D accumulators with one memset over their span, the default capacity
    with three."""
    raw = _scene(deg)
    poses, cams, gts = _keyframes()
    m = _mapper(raw, poses, gts, capacity=capacity)
    cap = m.stats().capacity
    single_span = 7 * cap + P <= 10 * P                   # glic_backward_compact_internal's choice
    assert single_span == (capacity == 6144), cap
    assert P % 32 != 0
    for step, v in enumerate((1, 2)):
        what = "degree %d, capacity %d, step %d (view %d)" % (deg, cap, step + 1, VIEWS[v])
        before = _state(m)
        m.optimize([v])
        after = _state(m)
        ref, _, tiny = _check_step_against_oracle(m, raw, before, after, cams, gts, [v], (oracle64, oracle32), what)
        assert ref["vis"][LAST], what                      # a row of the partial last warp stepped (and was compared)
        assert tiny == (step == 0), what
    assert m.stats().iterations == 2
    m.close()


# ---- 2. several views per step (gradient accumulation over a rank's views) --------------------------------------------
@pytest.mark.parametrize("batch", [[0, 1], [2, 0, 1], [1, 1]], ids=["2views", "3views", "same_view_twice"])
def test_views_per_rank_mean_matches_oracle(oracle32, oracle64, batch):
    """views_per_rank = len(batch): the geometric gradients are accumulated over the views (cg.accumulate) and scaled by
    1 / k, the colour gradients are summed over the view slots and scaled by 1 / S; the reference is the mean over views."""
    raw = _scene(2 if len(batch) == 3 else 3)
    poses, cams, gts = _keyframes(seed=11)
    m = _mapper(raw, poses, gts, views_per_rank=len(batch))
    before = _state(m)
    m.optimize(batch)
    after = _state(m)
    assert m.stats().iterations == 1
    what = "views %s per step" % batch
    ref, _, tiny = _check_step_against_oracle(m, raw, before, after, cams, gts, batch, (oracle64, oracle32), what)
    assert tiny, what
    n_vis = np.sum([r > 0 for r in ref["radii"]], axis=0)
    if len(set(batch)) > 1:
        print("%s: %d Gaussians visible in exactly one view of the batch" % (what, int((n_vis == 1).sum())))
        assert (n_vis == 1).sum() > 100 and (n_vis == len(batch)).sum() > 100, what
    m.close()


# ---- 5. after extend(): a regrown arena, old rows with moments, new rows from zero moments ------------------------------
def test_step_after_extend_matches_oracle(oracle32, oracle64):
    """extend() forces a regrow (capacity 3072 < P0 + inserted), as test_gpu_mapper's extend test does; one step later the
    old rows' gradient comes out of the moment recursion and the new rows' from their zero moments."""
    from gaussian_lic_b200 import mapper
    P0 = 3000
    raw = _scene(3, P_=P0, seed=5)
    poses, cams, gts = _keyframes(seed=3)
    m = mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=3, capacity=3072, scaling_scale=1.0)
    m.initialize(raw)
    m.add_keyframe(*poses[0], gts[0])
    m.optimize([0, 0, 0])
    m.add_keyframe(*poses[1], gts[1])
    rng = np.random.default_rng(9)
    n = 8000
    z = rng.uniform(0.5, 15.0, n)
    pts_cam = np.stack([z * rng.uniform(-0.8, 0.8, n), z * rng.uniform(-0.6, 0.6, n), z], 1)
    R_wc, t_wc = poses[1]
    pts = (pts_cam @ np.asarray(R_wc).T + np.asarray(t_wc)).astype(np.float32)
    cols = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    inserted = m.extend(pts, cols, z.astype(np.float32))
    st = m.stats()
    assert inserted > 0 and st.num_gaussians == P0 + inserted and st.capacity > 3072, (inserted, st.capacity)
    before = _state(m)
    assert np.abs(before["m"]["means"][:P0]).max() > 0 and not before["m"]["means"][P0:].any()
    m.optimize([1])
    after = _state(m)
    what = "after extend (+%d, capacity %d)" % (inserted, st.capacity)
    ref = _reference(_raw(before), cams, gts, [1], (oracle64, oracle32))
    assert abs(m.stats().last_loss - ref["loss"]) <= 1e-5 * ref["loss"]
    got = _recovered(before, after)
    vis = ref["vis"]
    old, new = np.flatnonzero(vis[:P0]), P0 + np.flatnonzero(vis[P0:])
    assert old.size > 100 and new.size > 100, (old.size, new.size)
    _compare(got, ref, old, what + ", old rows")
    # the new rows are isotropic (three equal log-scales) with the identity rotation: their covariance does not depend on
    # the rotation, whose gradient is zero up to rounding; it is held against the scale of the old rows' rotation gradient
    _compare(got, ref, new, what + ", new rows", groups=GROUPS[1:])
    iso = np.all(before["p"]["log_scales"][new] == before["p"]["log_scales"][new][:, :1], axis=1)
    ident = np.all(before["p"]["rots"][new] == np.float32([1, 0, 0, 0]), axis=1)
    rot_scale = np.abs(ref["grads"]["float64"]["rots"][np.setdiff1d(old, EDGE)]).max()
    noise = np.abs(got["rots"][new]).max(1)
    print("%s, new rows: %d / %d isotropic with the identity rotation; max |d rots| = %.3e (row %d) = %.2e of the old rows' "
          "max, f64 oracle max %.3e" % (what, int((iso & ident).sum()), new.size, noise.max(), new[noise.argmax()],
                                        noise.max() / rot_scale, np.abs(ref["grads"]["float64"]["rots"][new]).max()))
    assert (iso & ident).all() and noise.max() <= 1e-6 * rot_scale, what
    _check_step(before, after, got, np.flatnonzero(vis), _lr6(), what)
    _check_untouched(before, after, ~vis, what)
    m.close()


# ---- 6. two ranks, one view each: the geometric mean-reduce and the colour push -------------------------------------------
def _rank_worker(rank, world, port, q):
    try:
        import torch.distributed as dist
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
        torch.cuda.set_device(rank % torch.cuda.device_count())
        raw = _scene(3)
        poses, cams, gts = _keyframes(seed=31)
        m = _mapper(raw, poses, gts, capacity=P, rank=rank, world=world)
        got = [None] * world
        dist.all_gather_object(got, m.export_handle())
        m.connect(got)
        before = _state(m)
        m.optimize([1, 2])                                 # one step: rank r renders slot r
        after = _state(m)
        st = m.stats()
        dist.barrier()
        m.close()
        dist.destroy_process_group()
        q.put((rank, "ok", before, after, (st.iterations, st.last_loss)))
    except Exception as e:          # noqa: BLE001 - reported to the parent
        import traceback
        q.put((rank, "%r\n%s" % (e, traceback.format_exc()), None, None, None))


@pytest.mark.timeout(300)
def test_two_ranks_mean_matches_oracle(oracle32, oracle64):
    """world = 2, views_per_rank = 1 (one GPU shared by both ranks when the machine has one): the 11 geometric floats are
    mean-reduced by p2p.cu, the colour gradients and flags pushed to the peer; rank 0's step must use the mean of the two
    views' gradients, and both replicas must be bit-identical."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    q = ctx.Queue()
    procs = [ctx.Process(target=_rank_worker, args=(r, 2, port, q)) for r in range(2)]
    for p_ in procs:
        p_.start()
    res = sorted([q.get(timeout=240) for _ in procs], key=lambda r: r[0])
    for p_ in procs:
        p_.join(timeout=30)
    assert all(r[1] == "ok" for r in res), [r[1] for r in res]
    (_, _, before, after, (iters, last_loss)), (_, _, _, after1, _) = res
    assert iters == 1
    for key in ("p", "m", "v"):
        for g in GROUPS:
            assert np.array_equal(after[key][g], after1[key][g]), "replicas diverged in %s / %s" % (key, g)
    _, cams, gts = _keyframes(seed=31)
    what = "2 ranks x 1 view"
    ref = _reference(_raw(before), cams, gts, [1, 2], (oracle64, oracle32))
    n_vis = np.sum([r > 0 for r in ref["radii"]], axis=0)
    assert (n_vis == 1).sum() > 100, what
    vis = ref["vis"]
    got = _recovered(before, after)
    _compare(got, ref, np.flatnonzero(vis), what)
    assert _check_edge_rows(got, ref, before, after, what)
    _check_step(before, after, got, np.flatnonzero(vis), _lr6(), what)
    _check_untouched(before, after, ~vis, what)
    ref0 = _reference(_raw(before), cams, gts, [1], ())     # rank 0's pinned loss is that of its own view
    assert abs(last_loss - ref0["loss"]) <= 1e-5 * ref0["loss"], (last_loss, ref0["loss"])
