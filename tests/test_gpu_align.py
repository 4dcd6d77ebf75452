"""Test-time alignment in the native mapper (glic_mapper_align) on the GPU: the map stays frozen, no fit is evaluate(), the pose
and exposure gradients against the f64 restatements (recovered from the result's first Adam moments, g = m' / fl(1 - b1)), the
second step at the moved pose, the recovery of a perturbed pose and a known exposure, the overflow skip, argument validation, and
one rank aligning between the optimize() calls of two; plus the pose-only per-Gaussian backward against the COMPACT + POSE form
on the same render-backward outputs, bit for bit."""
import math
import os
import socket

import numpy as np
import pytest

from exposure_oracle import loss_exposure
from pose_oracle import T_cw_of, float_pose, pose_gradient, pose_step
from test_gpu_exposure import E_STAR, IDENTITY, _render
from test_gpu_mapper_grads import C1, F, GROUPS, H, W, _keyframes, _mapper, _scene, _state
from test_gpu_pose import _check_pose_grad, _rot_angle

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

LR_T, LR_R, EXPO_LR = 1e-3, 1e-3, 1e-3
B1 = np.float32(0.9)


@pytest.fixture(scope="module")
def weight_path(tmp_path_factory):
    """the reference's LPIPS weights if built, else seeded synthetic ones through the converter's writer"""
    from test_gpu_lpips import BUILT, G
    if os.path.isfile(BUILT):
        return BUILT
    from gaussian_lic_b200 import lpips_weights
    path = tmp_path_factory.mktemp("lpips") / "synthetic.bin"
    lpips_weights.write(path, G.synthetic_payload(1))
    return str(path)


def _bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def _snapshot(m, n_train):
    """every getter the frozen-map contract covers (stats without overflow_regrows)"""
    st = m.stats()
    out = dict(state=_state(m), dens=m.densify_stats(), maxr=m.screen_radii(), sky=m.sky_rows(),
               stats=tuple(getattr(st, k) for k, _ in st._fields_ if k != "overflow_regrows"))
    for k in range(n_train):
        out["pose%d" % k] = m.pose(k, camera=True)
        out["pose_state%d" % k] = m.pose_state(k)
        out["expo%d" % k] = m.exposure_state(k)
    return out


def _same(a, b):
    for g in GROUPS:
        for key in ("p", "m", "v"):
            assert np.array_equal(_bits(a["state"][key][g]), _bits(b["state"][key][g])), (key, g)
    assert all(np.array_equal(_bits(x), _bits(y)) for x, y in zip(a["dens"], b["dens"]))
    assert np.array_equal(a["maxr"], b["maxr"]) and a["sky"] == b["sky"] and a["stats"] == b["stats"]
    for key in a:
        if key.startswith("pose") or key.startswith("expo"):
            for x, y in zip(a[key], b[key]):
                if isinstance(x, dict):
                    assert all(np.array_equal(_bits(x[f]), _bits(y[f])) for f in ("view", "proj", "campos")), key
                elif isinstance(x, np.ndarray):
                    assert np.array_equal(_bits(x), _bits(y)), key
                else:
                    assert x == y, key


def _trained(raw, poses, gts, **kw):
    """a mapper with pose refinement, exposure and densification on, trained a few batches; keyframe 3 is held out"""
    m = _mapper(raw, poses, gts, **kw)
    m.add_keyframe(*poses[1], gts[1], train=False)
    m.enable_exposure(EXPO_LR)
    m.enable_pose_refinement(LR_T, LR_R)
    m.enable_densification()
    for i in range(3):
        m.set_exposure(i, E_STAR[i])
    m.optimize([0, 1, 2, 1])
    return m


# ---- 1. the map is frozen --------------------------------------------------------------------------------------------------
def test_align_leaves_the_mapper_unchanged():
    raw = _scene(3)
    poses, cams, gts = _keyframes(seed=41)
    m, twin = _trained(raw, poses, gts), _trained(raw, poses, gts)
    assert m.sample_views() == twin.sample_views()
    before = _snapshot(m, 3)
    assert before["pose_state0"][2] > 0 and before["expo0"][3] > 0 and before["dens"][1].any()
    for train, index in ((False, 0), (True, 1), (True, 2)):
        for split in (False, True):
            r = m.align(index, train=train, iterations=4, lr_translation=LR_T, lr_rotation=LR_R, exposure_lr=EXPO_LR, split=split)
            assert r["steps"] == 4 and r["skipped"] == 0
    _same(before, _snapshot(m, 3))
    assert m.sample_views() == twin.sample_views()
    m.close()
    twin.close()


# ---- 2. no fit is evaluate() -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("how", ["zero_iterations", "zero_rates"])
def test_no_fit_scores_like_evaluate(weight_path, how):
    raw = _scene(2)
    poses, cams, gts = _keyframes(seed=43)
    m = _trained(raw, poses, gts)
    m.load_lpips(weight_path)
    kw = dict(iterations=0) if how == "zero_iterations" else dict(iterations=3, lr_translation=0.0, lr_rotation=0.0, exposure_lr=0.0)
    for train, index in ((False, 0), (True, 0), (True, 2)):
        r = m.align(index, train=train, image=True, **kw)
        want = m.evaluate_lpips(index, train)
        assert _bits([r["psnr"], r["ssim"], r["lpips"]]).tolist() == _bits(want).tolist(), (train, index, r["psnr"], want)
        assert np.array_equal(_bits(r["image"]), _bits(m.render(index, train)))
        if train:
            R, t = m.pose(index)
            E = m.exposure(index)
        else:
            R, t = np.asarray(poses[1][0], np.float32), np.asarray(poses[1][1], np.float32)
            E = IDENTITY
        assert np.array_equal(r["R_wc"], R) and np.array_equal(r["t_wc"], t) and np.array_equal(r["E"], E)
        assert r["steps"] == kw["iterations"] and not r["expo_exp_avg"].any()
    m.close()


# ---- 3. gradients against the f64 restatements -----------------------------------------------------------------------------
def _align_reference(raw, cam, gt, E, split, oracles):
    """dL/d(rho, omega) per oracle dtype and the f64 dL/dE of one view, on the image and (exposed, cropped) dL/dpixel the
    mapper's kernels produce; with split the loss is taken on the left-half planes and dL/dpixel padded with zeros"""
    from gaussian_lic_b200 import model, ops
    dev = torch.device("cuda:0")
    mdl = model.PackedModel(raw, dev)
    mdl.activate()
    rast = ops.CRasterizer(W, H, dev)
    color, _, _ = rast.forward(mdl.inputs, rast.make_view(cam))
    wf = W // 2 if split else W
    img = color[:, :, :wf].contiguous()
    g_t = torch.as_tensor(np.ascontiguousarray(gt[:, :, :wf])).to(dev)
    loss, dL, _ = ops.l1_ssim_loss_exposure(img, g_t, torch.as_tensor(E).to(dev))
    torch.cuda.synchronize()
    dpix = np.zeros((3, H, W), np.float32)
    dpix[:, :, :wf] = dL.cpu().numpy()
    _, _, dE = loss_exposure(oracles[-1], img.cpu().numpy(), gt[:, :, :wf], E)
    out = {}
    for o in oracles:
        op, sc, rot = o.activations(raw["opacity_logits"], raw["log_scales"], raw["rots"])
        g = dict(means=raw["means"], scales=sc, rots=rot, opacity=op, dc=raw["dc"], sh=raw["sh"], degree=raw["degree"])
        f = o.forward(g, cam)
        out[o.dtype.name] = {0: pose_gradient(g, cam, f, o.backward(f, dpix))}
        o.free(f)
    return out, dE, float(loss.item())


@pytest.mark.parametrize("deg", [0, 3])
@pytest.mark.parametrize("split,expo", [(False, False), (True, True)], ids=["whole_frame", "split_with_exposure"])
def test_align_gradients_match_restatement(oracle32, oracle64, deg, split, expo):
    from test_gpu_mapper_grads import _raw
    raw = _scene(deg)
    poses, cams, gts = _keyframes(seed=47)
    m = _mapper(raw, poses, gts)
    m.add_keyframe(*poses[1], gts[2], train=False)
    r = m.align(0, iterations=1, exposure_lr=EXPO_LR if expo else 0.0, split=split)
    assert r["steps"] == 1
    what = "align, degree %d, split %s, exposure %s" % (deg, split, expo)
    ref, dE, loss = _align_reference(_raw(_state(m)), cams[1], gts[2], IDENTITY, split, [oracle32, oracle64])
    assert abs(r["first_loss"] - loss) <= 1e-5 * loss, (r["first_loss"], loss)
    _check_pose_grad({0: r["pose_exp_avg"].astype(np.float64) / C1}, ref, what)
    if expo:
        g = r["expo_exp_avg"].astype(np.float64) / C1
        err = np.linalg.norm(g - dE) / np.linalg.norm(dE)
        print("%s: dL/dE recovered %s\n  f64 oracle %s\n  |diff| / |ref| = %.2e" % (what, g.ravel(), dE.ravel(), err))
        assert err <= 1e-4
    else:
        assert not r["expo_exp_avg"].any() and np.array_equal(r["E"], IDENTITY)
    m.close()


# ---- 4. the second step at the moved pose -------------------------------------------------------------------------------------
def test_second_step_at_the_moved_pose(oracle32, oracle64):
    from gaussian_lic_b200 import mapper
    from test_gpu_mapper_grads import _raw
    raw = _scene(3)
    poses, cams, gts = _keyframes(seed=53)
    m = _mapper(raw, poses, gts)
    m.add_keyframe(*poses[2], gts[0], train=False)
    one = m.align(0, iterations=1)
    two = m.align(0, iterations=2)
    T0 = T_cw_of(*poses[2])
    g1 = one["pose_exp_avg"].astype(np.float64) / C1
    T1, m1, v1, t1 = pose_step(T0, np.zeros(6), np.zeros(6), 0, g1, LR_T, LR_R)
    R1, tt1 = float_pose(T1)
    assert np.abs(R1 - one["R_wc"]).max() <= 1e-6 and np.abs(tt1 - one["t_wc"]).max() <= 1e-6
    # step 2's gradient (the render backward's float atomics make the two calls' first steps agree to rounding only)
    g2 = (two["pose_exp_avg"].astype(np.float64) - (B1 * one["pose_exp_avg"]).astype(np.float64)) / C1
    cam1 = mapper.camera_block(W, H, F, F, W / 2.0, H / 2.0, one["R_wc"], one["t_wc"])
    ref, _, _ = _align_reference(_raw(_state(m)), cam1, gts[0], IDENTITY, False, [oracle32, oracle64])
    _check_pose_grad({0: g2}, ref, "align, second step")
    T2, _, _, _ = pose_step(T1, m1, v1, t1, g2, LR_T, LR_R)
    R2, tt2 = float_pose(T2)
    dr, dt = np.abs(R2 - two["R_wc"]).max(), np.abs(tt2 - two["t_wc"]).max()
    print("second step: |R - restated| %.2e, |t - restated| %.2e" % (dr, dt))
    assert dr <= 1e-5 and dt <= 1e-5
    m.close()


# ---- 5. recovery --------------------------------------------------------------------------------------------------------------
REC_ITERS = 300
# H100 80GB HBM3 run: 0.0158 rad -> 2.2e-4 / 2.0e-4, 0.021 -> 3.0e-5 / 2.8e-5, |E - E*| 1.1e-3 / 9.2e-4, PSNR 16.2 -> 56.1 /
# 16.0 -> 60.0 dB (whole frame / split); the bounds leave a margin of 4 or more
REC_ROT, REC_TRANS, REC_E = 1e-3, 3e-4, 5e-3


@pytest.mark.parametrize("split", [False, True], ids=["whole_frame", "split"])
def test_align_recovers_pose_and_exposure(split):
    from scipy.spatial.transform import Rotation
    from gaussian_lic_b200 import capi, mapper
    raw = _scene(3)
    poses, cams, _ = _keyframes()
    gts = _render(raw, cams)
    E_true = E_STAR[1]
    gt = np.einsum("khw,kc->chw", gts[1].astype(np.float64), E_true[:, :3].astype(np.float64)) + E_true[:, 3][:, None, None]
    gt = gt.astype(np.float32)
    m = mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=3)
    m.initialize(raw)
    for (R, t), img in zip(poses, gts):
        m.add_keyframe(R, t, img)
    rng = np.random.default_rng(5)
    R_true, t_true = poses[1]
    dR = Rotation.from_rotvec(rng.normal(size=3) * np.deg2rad(1.0) / np.sqrt(3)).as_matrix()
    m.add_keyframe(dR @ R_true, t_true + rng.normal(size=3) * 0.03 / np.sqrt(3), gt, train=False)
    start = m.align(0, iterations=0, split=split)
    r = m.align(0, iterations=REC_ITERS, lr_translation=LR_T, lr_rotation=LR_R, exposure_lr=0.01, split=split, image=True)
    e0 = (_rot_angle(start["R_wc"], R_true), float(np.linalg.norm(start["t_wc"] - t_true)))
    e1 = (_rot_angle(r["R_wc"], R_true), float(np.linalg.norm(r["t_wc"] - t_true)))
    de = float(np.abs(r["E"] - E_true).max())
    print("align recovery (split %s): rotation %.2e -> %.2e rad, translation %.2e -> %.2e, |E - E*| %.2e, PSNR %.2f -> %.2f, "
          "loss %.5f -> %.5f" % (split, e0[0], e1[0], e0[1], e1[1], de, start["psnr"], r["psnr"], r["first_loss"], r["last_loss"]))
    assert e1[0] <= REC_ROT and e1[1] <= REC_TRANS and de <= REC_E
    assert r["psnr"] > start["psnr"] + 5 and r["last_loss"] < 0.5 * r["first_loss"]
    assert r["steps"] == REC_ITERS and r["skipped"] == 0
    if split:                                            # the scores are glic_eval_psnr_ssim of the right-half crops
        ws = W - W // 2
        crop = lambda x: np.ascontiguousarray(x[:, :, W // 2:], np.float32)
        a, b = torch.as_tensor(crop(r["image"])).cuda(), torch.as_tensor(crop(gt)).cuda()
        scratch = torch.empty(capi.lib.glic_eval_scratch_bytes(3, H, ws), dtype=torch.uint8, device="cuda")
        out = torch.empty(2, dtype=torch.float32, device="cuda")
        capi.check(capi.lib.glic_eval_psnr_ssim(3, H, ws, capi.ptr(a), capi.ptr(b), capi.ptr(out), capi.ptr(scratch),
                                                scratch.numel(), None), "eval_psnr_ssim")
        torch.cuda.synchronize()
        assert _bits(out.cpu().numpy()).tolist() == _bits([r["psnr"], r["ssim"]]).tolist()
    m.close()


# ---- 6. overflow ----------------------------------------------------------------------------------------------------------
def test_overflowed_iterations_are_skipped():
    raw = _scene(1)
    poses, cams, gts = _keyframes()
    m = _mapper(raw, poses, gts)
    m.add_keyframe(*poses[0], gts[1], train=False)
    m.set_binning_pairs(1000)
    regrows = m.stats().overflow_regrows
    r = m.align(0, iterations=5, exposure_lr=EXPO_LR)
    assert r["skipped"] == 5 and r["steps"] == 0 and math.isnan(r["first_loss"]) and math.isnan(r["last_loss"])
    assert np.array_equal(r["R_wc"], np.asarray(poses[0][0], np.float32)) and np.array_equal(r["t_wc"], np.asarray(poses[0][1], np.float32))
    assert np.array_equal(r["E"], IDENTITY) and not r["pose_exp_avg"].any() and not r["expo_exp_avg"].any()
    assert _bits([r["psnr"], r["ssim"]]).tolist() == _bits(m.evaluate(0, False)).tolist()
    assert m.stats().overflow_regrows > regrows
    r2 = m.align(0, iterations=5, exposure_lr=EXPO_LR)
    assert r2["skipped"] == 0 and r2["steps"] == 5
    m.close()


# ---- 7. validation --------------------------------------------------------------------------------------------------------
def test_rejected_arguments_change_nothing(weight_path):
    import ctypes as C
    from gaussian_lic_b200 import capi
    raw = _scene(0)
    poses, cams, gts = _keyframes()
    m = _trained(raw, poses, gts)
    before = _snapshot(m, 3)
    bad = [dict(index=1), dict(index=-1), dict(index=3, train=True), dict(iterations=-1), dict(lr_translation=-1e-3),
           dict(lr_rotation=float("nan")), dict(exposure_lr=float("inf"))]
    for kw in bad:
        with pytest.raises(capi.GlicError):
            m.align(**dict(dict(index=0), **kw))
    p, r = capi.AlignParams(1, LR_T, LR_R, 0.0, 2), capi.AlignResult()
    assert capi.lib.glic_mapper_align(m._h, 0, 0, C.byref(p), C.byref(r), None) == -1            # split not 0 or 1
    p.split = 0
    assert capi.lib.glic_mapper_align(m._h, 0, 0, None, C.byref(r), None) == -1
    assert capi.lib.glic_mapper_align(m._h, 0, 0, C.byref(p), None, None) == -1
    _same(before, _snapshot(m, 3))
    m.close()
    # a score region under 31x31 with LPIPS weights loaded; a mapper without rows
    from gaussian_lic_b200 import mapper
    small = mapper.Mapper(60, 40, 50.0, 50.0, 30.0, 20.0, sh_degree=0)
    small.initialize(dict((k, v[:100]) for k, v in raw.items() if k != "degree"))
    small.add_keyframe(*poses[0], np.zeros((3, 40, 60), np.float32), train=False)
    small.load_lpips(weight_path)
    small.align(0, iterations=1)
    with pytest.raises(capi.GlicError, match="31x31"):
        small.align(0, iterations=1, split=True)
    small.close()
    empty = mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=0)
    empty.add_keyframe(*poses[0], gts[0], train=False)
    with pytest.raises(capi.GlicError, match="no rows"):
        empty.align(0)
    empty.close()


# ---- the pose-only backward against COMPACT + POSE --------------------------------------------------------------------------
@pytest.mark.parametrize("deg", [0, 1, 3])
def test_pose_only_backward_equals_the_pose_form(deg):
    import ctypes as C
    from gaussian_lic_b200 import capi, model, ops
    raw = _scene(deg)
    poses, cams, gts = _keyframes(seed=59)
    dev = torch.device("cuda:0")
    mdl = model.PackedModel(raw, dev)
    mdl.activate()
    g = mdl.inputs
    rast = ops.CRasterizer(W, H, dev)
    view = rast.make_view(cams[1])
    color, _, radii = rast.forward(g, view)
    _, dL = rast.loss(color, torch.as_tensor(gts[1]).to(dev), 0.2)
    grads = rast.alloc_grads()
    for k in ("dL_dmeans2D", "dL_dconic", "dL_dopacity", "dL_dcolors"):
        grads[k].zero_()
    rast.render_backward(view, dL, grads)
    P, M = rast.P, rast.M
    rot_raw = torch.as_tensor(raw["rots"]).to(dev)
    part = torch.empty((P + 127) // 128 * 6, dtype=torch.float64, device=dev)
    geo = torch.full((11 * P,), float("nan"), dtype=torch.float32, device=dev)
    out = {}
    for only in (0, 1):
        pose6 = torch.full((6,), float("nan"), dtype=torch.float32, device=dev)
        capi.check(capi.lib.glic_debug_pose_backward(
            P, deg, M, capi.ptr(g["means"]), capi.ptr(g["scales"]), capi.ptr(g["rots"]), capi.ptr(rot_raw), capi.ptr(g["opacity"]),
            capi.ptr(g["sh"]) if M else None, C.byref(view), capi.ptr(radii), capi.ptr(rast.geom_ws), capi.ptr(grads["dL_dmeans2D"]),
            capi.ptr(grads["dL_dconic"]), capi.ptr(grads["dL_dopacity"]), capi.ptr(grads["dL_dcolors"]), only,
            None if only else capi.ptr(geo), capi.ptr(part), capi.ptr(pose6), None), "debug_pose_backward")
        torch.cuda.synchronize()
        out[only] = pose6.cpu().numpy()
    print("degree %d: POSE %s\n          POSE_ONLY %s" % (deg, out[0], out[1]))
    assert np.isfinite(out[0]).all() and np.abs(out[0]).max() > 0
    assert np.array_equal(_bits(out[0]), _bits(out[1]))
    assert np.isfinite(geo.cpu().numpy()).all()                     # the POSE form wrote every row


# ---- 8. two ranks -----------------------------------------------------------------------------------------------------------
BATCHES_2R = [1, 2, 0, 1, 2, 2]


def _align_rank_worker(rank, world, port, q):
    try:
        import torch.distributed as dist
        from test_gpu_mapper_grads import P
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
        torch.cuda.set_device(rank % torch.cuda.device_count())
        raw = _scene(3)
        poses, cams, gts = _keyframes(seed=31)
        m = _mapper(raw, poses, gts, capacity=P, rank=rank, world=world, views_per_rank=1)
        m.add_keyframe(*poses[1], gts[0], train=False)
        got = [None] * world
        dist.all_gather_object(got, m.export_handle())
        m.connect(got)
        m.enable_pose_refinement(LR_T, LR_R)
        m.enable_exposure(EXPO_LR)
        steps = []
        for i in range(3):
            m.optimize(BATCHES_2R[2 * i:2 * i + 2])
            if rank == 0:
                steps.append(m.align(0, iterations=5, exposure_lr=EXPO_LR, split=bool(i % 2))["steps"])
                steps.append(m.align(1, train=True, iterations=3, exposure_lr=EXPO_LR)["steps"])
        out = dict(state=_state(m), pose=[m.pose(i, camera=True) for i in range(3)], expo=[m.exposure_state(i) for i in range(3)],
                   steps=steps)
        dist.barrier()
        m.close()
        dist.destroy_process_group()
        q.put((rank, "ok", out))
    except Exception as e:          # noqa: BLE001 - reported to the parent
        import traceback
        q.put((rank, "%r\n%s" % (e, traceback.format_exc()), None))


@pytest.mark.timeout(300)
def test_two_ranks_stay_identical_when_one_aligns():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    q = ctx.Queue()
    procs = [ctx.Process(target=_align_rank_worker, args=(r, 2, port, q)) for r in range(2)]
    for p_ in procs:
        p_.start()
    res = sorted([q.get(timeout=240) for _ in procs], key=lambda r: r[0])
    for p_ in procs:
        p_.join(timeout=30)
    assert all(r[1] == "ok" for r in res), [r[1] for r in res]
    a, b = res[0][2], res[1][2]
    assert a["steps"] == [5, 3] * 3 and b["steps"] == []
    for key in ("p", "m", "v"):
        for g in GROUPS:
            assert np.array_equal(_bits(a["state"][key][g]), _bits(b["state"][key][g])), "replicas diverged in %s / %s" % (key, g)
    for k in range(3):
        for x, y in zip(a["pose"][k][:2] + a["expo"][k][:3], b["pose"][k][:2] + b["expo"][k][:3]):
            assert np.array_equal(_bits(x), _bits(y)), "replicas diverged in keyframe %d" % k
        assert np.array_equal(a["pose"][k][2]["view"], b["pose"][k][2]["view"])
