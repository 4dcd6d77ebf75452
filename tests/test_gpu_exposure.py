"""Per-keyframe affine exposure on the GPU: the exposed L1 + D-SSIM loss (glic_l1_ssim_loss_exposure) against the CPU oracle,
and the native mapper's exposure (glic_mapper_enable_exposure) -- its gradients recovered from the Adam moments, the fit of
known exposures, the overflow skip, the two-rank exchange and evaluation.

E is 3x4 row-major, out_c = E[0][c] r + E[1][c] g + E[2][c] b + E[c][3].  Every E used here is asymmetric, so a transposed
3x3 block fails."""
import os
import socket

import numpy as np
import pytest

from exposure_oracle import loss_exposure
from helpers import grad_close
from test_gpu_mapper_grads import (C1, F, GROUPS, H, W, _compare, _keyframes, _mapper, _raw, _recovered, _scene, _state)

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

EXPO_LR = 0.001                      # config/fastlivo.yaml:26
E_STAR = [np.array([[1.21, 0.04, -0.03, 0.05], [-0.05, 0.83, 0.02, -0.04], [0.03, 0.06, 0.95, 0.02]], np.float32),
          np.array([[0.74, -0.03, 0.05, -0.05], [0.06, 1.12, -0.04, 0.03], [-0.02, 0.05, 1.28, -0.02]], np.float32),
          np.array([[1.05, 0.05, 0.02, 0.04], [-0.04, 0.96, 0.06, 0.01], [0.05, -0.02, 0.71, -0.03]], np.float32)]
IDENTITY = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)


def _expose(img, E):
    """float64 exposure of a [3,H,W] image"""
    E = np.asarray(E, np.float64)
    return np.einsum("khw,kc->chw", np.asarray(img, np.float64), E[:, :3]) + E[:, 3][:, None, None]


def _expose32(img, E):
    """the kernels' float32 evaluation: acc = E[c][3], then fmaf with r, g, b (each fma as one float64 product, exact, plus
    one add, rounded to float32)"""
    img = np.asarray(img, np.float32).astype(np.float64)
    E = np.asarray(E, np.float32).astype(np.float64)
    out = np.empty(img.shape, np.float32)
    for c in range(3):
        acc = np.full(img.shape[1:], np.float32(E[c, 3]))
        for k in range(3):
            acc = (img[k] * E[k, c] + acc.astype(np.float64)).astype(np.float32)
        out[c] = acc
    return out


def _op(img, gt, E):
    from gaussian_lic_b200 import ops
    dev = torch.device("cuda:0")
    t = [torch.as_tensor(np.ascontiguousarray(x, np.float32)).to(dev) for x in (img, gt, E)]
    loss, dimg, dE = ops.l1_ssim_loss_exposure(*t)
    torch.cuda.synchronize()
    return float(loss.item()), dimg.cpu().numpy(), dE.cpu().numpy()


# ---- 1-3. the standalone op ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("HW", [(37, 53), (120, 200), (1080, 1920)])
def test_exposed_loss_matches_oracle(oracle32, oracle64, HW):
    from gaussian_lic_b200 import synthetic as syn
    h, w = HW
    rng = np.random.default_rng(h)
    gt = syn.make_gt_image(w, h, seed=3)
    img = np.clip(gt + 0.2 * rng.normal(size=gt.shape), 0, 1.5).astype(np.float32)
    E = E_STAR[0]
    loss, dimg, dE = _op(img, gt, E)
    L32, g32, _ = loss_exposure(oracle32, img, gt, E)
    L64, _, dE64 = loss_exposure(oracle64, img, gt, E)
    print("%dx%d: loss %.7f (f32 oracle %.7f, f64 %.7f)" % (h, w, loss, L32, L64))
    assert abs(loss - L32) < 1e-5
    grad_close(dimg, g32, "dL_dimg (exposed loss %dx%d)" % (h, w), rtol=1e-4)
    err = np.linalg.norm(dE - dE64) / np.linalg.norm(dE64)
    print("dL_dE %s\n  vs f64 oracle: |diff| / |ref| = %.2e" % (dE, err))
    assert err <= 1e-4
    _, _, dE_t = loss_exposure(oracle64, img, gt, np.hstack([E[:, :3].T, E[:, 3:]]))
    assert np.linalg.norm(dE - dE_t) / np.linalg.norm(dE64) > 1e-3                # the transposed block is told apart


def test_identity_exposure_equals_the_plain_loss():
    from gaussian_lic_b200 import ops, synthetic as syn
    Hh, Ww = 120, 200
    rng = np.random.default_rng(8)
    gt = syn.make_gt_image(Ww, Hh, seed=4)
    img = np.clip(gt + 0.2 * rng.normal(size=gt.shape), 0, 1.5).astype(np.float32)
    loss, dimg, _ = _op(img, gt, IDENTITY)
    r = ops.CRasterizer(Ww, Hh)
    l0, d0 = r.loss(torch.as_tensor(img).cuda(), torch.as_tensor(gt).cuda())
    torch.cuda.synchronize()
    assert np.array_equal(dimg, d0.cpu().numpy())                                   # values: +0 == -0
    assert abs(loss - float(l0.item())) <= 1e-6 * loss                              # atomic order of the loss sum only


def test_exposure_gradient_is_deterministic():
    from gaussian_lic_b200 import synthetic as syn
    Hh, Ww = 1080, 1920
    rng = np.random.default_rng(9)
    gt = syn.make_gt_image(Ww, Hh, seed=5)
    img = np.clip(gt + 0.2 * rng.normal(size=gt.shape), 0, 1.5).astype(np.float32)
    _, d1, e1 = _op(img, gt, E_STAR[1])
    _, d2, e2 = _op(img, gt, E_STAR[1])
    assert np.array_equal(e1.view(np.uint32), e2.view(np.uint32))
    assert np.array_equal(d1.view(np.uint32), d2.view(np.uint32))


# ---- mapper helpers ---------------------------------------------------------------------------------------------------------
def _render(raw, cams):
    """the model's image from every camera, by the kernels the mapper runs"""
    from gaussian_lic_b200 import model, ops
    mdl = model.PackedModel(raw, torch.device("cuda:0"))
    mdl.activate()
    rast = ops.CRasterizer(W, H)
    out = []
    for cam in cams:
        color, _, _ = rast.forward(mdl.inputs, rast.make_view(cam))
        torch.cuda.synchronize()
        out.append(color.cpu().numpy().copy())
    return out


def _expo_states(m, n):
    return [m.exposure_state(i) for i in range(n)]


def _reference_expo(raw, cams, gts, batch, Es, oracle64):
    """Mean over the batch's slots of the f64 oracle's dL/d(raw parameters) through the exposure backward, and of dL/dE per
    keyframe, on the image and exposed-loss dL/dpixel the mapper's own kernels produce."""
    from gaussian_lic_b200 import model, ops
    dev = torch.device("cuda:0")
    n = raw["means"].shape[0]
    mdl = model.PackedModel(raw, dev)
    mdl.activate()
    rast = ops.CRasterizer(W, H, dev)
    out = dict(radii=[], oracle_radii=[], loss=None, dE={}, grads={"float64": {g: 0.0 for g in GROUPS}})
    for v in batch:
        color, _, radii = rast.forward(mdl.inputs, rast.make_view(cams[v]))
        loss, dL, _ = ops.l1_ssim_loss_exposure(color, torch.as_tensor(gts[v]).to(dev), torch.as_tensor(Es[v]).to(dev))
        torch.cuda.synchronize()
        out["loss"] = float(loss.item())
        out["radii"].append(radii.cpu().numpy().copy())
        col = color.cpu().numpy()
        _, _, dE = loss_exposure(oracle64, col, gts[v], Es[v])
        out["dE"][v] = out["dE"].get(v, 0.0) + dE / len(batch)
        o = oracle64
        op, sc, rot = o.activations(raw["opacity_logits"], raw["log_scales"], raw["rots"])
        f = o.forward(dict(means=raw["means"], scales=sc, rots=rot, opacity=op, dc=raw["dc"], sh=raw["sh"], degree=raw["degree"]), cams[v])
        b = o.backward(f, dL.cpu().numpy())
        out["oracle_radii"].append(f["radii"].copy())
        g_op, g_s, g_r = o.activations_backward(op, sc, raw["rots"], b["dL_dopacity"], b["dL_dscales"], b["dL_drots"])
        o.free(f)
        per = dict(rots=g_r, means=b["dL_dmeans3D"], log_scales=g_s, opacity_logits=g_op, dc=b["dL_ddc"], sh=b["dL_dsh"])
        acc = out["grads"]["float64"]
        for g in GROUPS:
            acc[g] = acc[g] + np.asarray(per[g], np.float64).reshape(n, -1) / len(batch)
    out["grads"]["float32"] = out["grads"]["float64"]            # _compare's yardstick line: not measured here
    out["vis"] = np.any([r > 0 for r in out["radii"]], axis=0)
    return out


# ---- 5. gradients recovered from the moments ------------------------------------------------------------------------------
@pytest.mark.parametrize("batch", [[0, 1], [1, 1]], ids=["two_views", "same_view_twice"])
def test_mapper_gradients_through_exposure_match_oracle(oracle64, batch):
    raw = _scene(3)
    poses, cams, gts = _keyframes(seed=13)
    m = _mapper(raw, poses, gts, views_per_rank=len(batch))
    m.enable_exposure(EXPO_LR)
    Es = [E_STAR[i] for i in range(len(poses))]
    for i, E in enumerate(Es):
        m.set_exposure(i, E)
    assert all(np.array_equal(m.exposure(i), Es[i]) for i in range(len(poses)))
    before, ex0 = _state(m), _expo_states(m, len(poses))
    assert all(t == 0 and not mm.any() and not vv.any() for _, mm, vv, t in ex0)
    m.optimize(batch)
    after, ex1 = _state(m), _expo_states(m, len(poses))
    what = "exposure, views %s per step" % batch
    ref = _reference_expo(_raw(before), cams, gts, batch, Es, oracle64)
    assert abs(m.stats().last_loss - ref["loss"]) <= 1e-5 * ref["loss"], (m.stats().last_loss, ref["loss"])
    got = _recovered(before, after)
    _compare(got, ref, np.flatnonzero(ref["vis"]), what)
    for k in range(len(poses)):
        E1, m1, v1, t1 = ex1[k]
        if k not in batch:                                                     # not in the batch: not stepped
            assert t1 == 0 and np.array_equal(E1, Es[k]) and not m1.any() and not v1.any(), (what, k)
            continue
        assert t1 == 1, (what, k, t1)                                          # [1, 1]: one step for the two slots
        g = m1.astype(np.float64) / C1
        want = ref["dE"][k]
        err = np.linalg.norm(g - want) / np.linalg.norm(want)
        print("%s: keyframe %d dL/dE recovered %s\n  f64 oracle %s\n  |diff| / |ref| = %.2e" % (what, k, g, want, err))
        assert err <= 1e-4, (what, k)
        assert np.all(np.abs(E1 - Es[k]) <= 1.01 * EXPO_LR) and np.abs(E1 - Es[k]).min() >= 0.5 * EXPO_LR   # first step: ~lr each
    m.close()


# ---- 4 + 8. the fit of known exposures, and evaluation ------------------------------------------------------------------------
FIT_PASSES = (300, 100)      # passes at FIT_LR, then at FIT_LR / 10
FIT_LR = 0.01
FIT_BOUND = 0.01             # max |E - E*| after the fit: 4.9e-3 in a recorded run (H100, keyframe 0; 1-5e-4 for the others)


def test_mapper_recovers_known_exposures():
    """Gaussians frozen (all five learning rates 0); keyframe k's ground truth is the model's own image under E*_k.  After
    FIT_PASSES passes over the three keyframes at exposure_lr = FIT_LR and FIT_LR / 10, every fitted E_k is within FIT_BOUND of E*_k (one
    recorded run on an H100: see the printed error), the loss has fallen, and a held-out keyframe with the same pose and
    ground truth evaluates with the identity."""
    from gaussian_lic_b200 import mapper
    raw = _scene(3)
    poses, cams, _ = _keyframes()
    imgs = _render(raw, cams)
    gts = [_expose(im, E).astype(np.float32) for im, E in zip(imgs, E_STAR)]
    frozen = dict(position_lr=0.0, feature_lr=0.0, opacity_lr=0.0, scaling_lr=0.0, rotation_lr=0.0)
    m = mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=3, **frozen)
    m.initialize(raw)
    m.enable_exposure(FIT_LR)                                   # before the keyframes: they start at the identity too
    for (R, t), img in zip(poses, gts):
        m.add_keyframe(R, t, img)
    m.add_keyframe(*poses[0], gts[0], train=False)
    assert np.array_equal(m.exposure(2), IDENTITY)
    first = m.optimize([0, 1, 2]).last_loss
    m.optimize([0, 1, 2] * (FIT_PASSES[0] - 1))
    m.enable_exposure(FIT_LR / 10)                              # a second call changes the learning rate only
    m.optimize([0, 1, 2] * FIT_PASSES[1])
    last = m.stats().last_loss
    errs = [np.abs(m.exposure(k) - E_STAR[k]).max() for k in range(3)]
    print("exposure fit: loss %.5f -> %.5f; max |E - E*| per keyframe %s; steps %s" % (
        first, last, ["%.2e" % e for e in errs], [m.exposure_state(k)[3] for k in range(3)]))
    assert last < 0.25 * first
    assert max(errs) <= FIT_BOUND
    assert all(m.exposure_state(k)[3] == sum(FIT_PASSES) for k in range(3))
    # held-out view, identity exposure: PSNR of the clamped raw render against the clamped gt
    psnr_test, _ = m.evaluate(0, train=False)
    want = 10 * np.log10(1.0 / np.mean((np.clip(imgs[0], 0, 1) - np.clip(gts[0], 0, 1)) ** 2))
    psnr_train, _ = m.evaluate(0, train=True)
    print("keyframe 0: PSNR trained %.2f dB, held-out (identity) %.3f dB, numpy identity %.3f dB" % (psnr_train, psnr_test, want))
    assert abs(psnr_test - want) <= 0.01
    assert psnr_train > psnr_test + 10
    m.close()


def test_evaluate_applies_the_training_exposure():
    """With E* set, a training keyframe whose gt is clamp(E* render) scores at least the PSNR the identity case reaches on
    the untransformed gt (both infinite when the renders agree bit for bit), and far more than the identity on that gt."""
    from gaussian_lic_b200 import mapper
    raw = _scene(2)
    poses, cams, _ = _keyframes()
    imgs = _render(raw, cams)
    scores = {}
    for name, E in (("identity", None), ("exposed", E_STAR[1])):
        gt = imgs[1] if E is None else np.clip(_expose32(imgs[1], E), 0, 1)
        m = mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=2)
        m.initialize(raw)
        m.add_keyframe(*poses[0], np.zeros_like(imgs[0]))
        m.add_keyframe(*poses[1], gt.astype(np.float32))
        if E is not None:
            m.enable_exposure(EXPO_LR)
            m.set_exposure(1, E)
        scores[name] = m.evaluate(1, train=True)
        if E is not None:
            m.set_exposure(1, IDENTITY)
            scores["exposed gt, identity E"] = m.evaluate(1, train=True)
        m.close()
    print("evaluate: PSNR / SSIM %s" % scores)
    assert scores["exposed"][0] >= min(scores["identity"][0], 100.0) - 0.05
    assert scores["exposed"][0] > scores["exposed gt, identity E"][0] + 5


# ---- 6. overflow --------------------------------------------------------------------------------------------------------------
def test_overflowed_iteration_leaves_exposure_unchanged():
    raw = _scene(1)
    poses, cams, gts = _keyframes()
    m = _mapper(raw, poses, gts)
    m.enable_exposure(EXPO_LR)
    m.set_exposure(0, E_STAR[0])
    m.optimize([0])                                              # one real step: non-zero moments, t = 1
    s0 = _expo_states(m, 3)
    m.set_binning_pairs(1000)                                    # far fewer pairs than the frame needs
    st = m.optimize([0])
    assert st.overflow_regrows >= 1 and st.iterations == 2
    s1 = _expo_states(m, 3)
    for a, b in zip(s0, s1):
        for x, y in zip(a[:3], b[:3]):
            assert np.array_equal(x.view(np.uint32), y.view(np.uint32))
        assert a[3] == b[3]
    assert s1[0][3] == 1
    m.optimize([0])                                              # the regrown workspace steps again
    assert m.exposure_state(0)[3] == 2
    m.close()


# ---- 7. two ranks -------------------------------------------------------------------------------------------------------------
BATCHES_2R = [1, 2, 0, 1, 2, 2]                                   # three batches of two slots


def _expo_run(rank, world, k, exchange=None):
    raw = _scene(3)
    poses, cams, gts = _keyframes(seed=31)
    from test_gpu_mapper_grads import P
    m = _mapper(raw, poses, gts, capacity=P, rank=rank, world=world, views_per_rank=k)
    if world > 1:
        m.connect(exchange(m.export_handle()))
    m.enable_exposure(EXPO_LR)
    for i in (1, 2):
        m.set_exposure(i, E_STAR[i])
    m.optimize(BATCHES_2R)
    st = m.stats()
    out = dict(state=_state(m), expo=_expo_states(m, 3), iters=st.iterations)
    return m, out


def _expo_rank_worker(rank, world, port, q):
    try:
        import torch.distributed as dist
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
        torch.cuda.set_device(rank % torch.cuda.device_count())

        def exchange(mine):
            got = [None] * world
            dist.all_gather_object(got, mine)
            return got

        m, out = _expo_run(rank, world, 1, exchange)
        dist.barrier()
        m.close()
        dist.destroy_process_group()
        q.put((rank, "ok", out))
    except Exception as e:          # noqa: BLE001 - reported to the parent
        import traceback
        q.put((rank, "%r\n%s" % (e, traceback.format_exc()), None))


@pytest.mark.timeout(300)
def test_two_ranks_exposure_replicas_and_one_rank_accumulation():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    q = ctx.Queue()
    procs = [ctx.Process(target=_expo_rank_worker, args=(r, 2, port, q)) for r in range(2)]
    for p_ in procs:
        p_.start()
    res = sorted([q.get(timeout=240) for _ in procs], key=lambda r: r[0])
    for p_ in procs:
        p_.join(timeout=30)
    assert all(r[1] == "ok" for r in res), [r[1] for r in res]
    a, b = res[0][2], res[1][2]
    assert a["iters"] == b["iters"] == len(BATCHES_2R) // 2
    for key in ("p", "m", "v"):
        for g in GROUPS:
            assert np.array_equal(a["state"][key][g], b["state"][key][g]), "replicas diverged in %s / %s" % (key, g)
    for k in range(3):
        for x, y in zip(a["expo"][k][:3], b["expo"][k][:3]):
            assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), "replicas diverged in keyframe %d's exposure" % k
        assert a["expo"][k][3] == b["expo"][k][3]
    assert [a["expo"][k][3] for k in range(3)] == [1, 2, 2]                       # [2, 2] steps keyframe 2 once
    m, one = _expo_run(0, 1, 2)
    m.close()
    worst = max(np.abs(a["expo"][k][0].astype(np.float64) - one["expo"][k][0]).max() for k in range(3))
    print("2 ranks vs 1 rank x 2 views: max |E diff| = %.3e (%.3g lr)" % (worst, worst / EXPO_LR))
    for k in range(3):
        assert one["expo"][k][3] == a["expo"][k][3]
    # the first batch's exposure gradients are bit-identical in both arms; later ones see Gaussians that differ by the render
    # backward's atomic order only
    assert worst <= 0.02 * EXPO_LR
