"""The native mapper (csrc/mapper.cu) at full batch width and across the growth of its per-keyframe state, against the
float64 CPU oracle.

test_gpu_mapper_grads.py, test_gpu_exposure.py and test_gpu_pose.py check the gradients of a step with at most three view
slots and three keyframes.  A real run takes up to 32 slots per step (world * views_per_rank), fills the last batch of a
list by wrapping around it, and keeps adding training keyframes while exposure and pose refinement are on, so the
per-keyframe arrays are regrown (64 rows first, then doubling; a late enable sizes them to the keyframes present).  Here:

  1. S = 8 and 32 slots, exposure and pose refinement on, two consecutive steps (both parities of the exchange block's
     slot regions).  Step 1 holds one keyframe in slots 0, 13 * S / 32 and S - 1; step 2 holds one keyframe only in slot 0,
     another only in slot S - 1 and the first again in three slots.  Every step is checked as the narrow tests check one:
     the Gaussians' gradients recovered from the Adam moments against the mean over the S slots of the f64 oracle, Adam
     bit for bit, idle rows untouched, and per batch keyframe dL/dE and dL/d(rho, omega) against (1/S) * the sum over the
     slots holding it -- divided by S, not by the keyframe's multiplicity -- with one Adam step per keyframe;
  2. a list of 11 views at S = 8 steps as the two batches the wrap-around spells out: bit for bit wherever the render
     backward's float atomics do not enter, at the gradient tests' tolerance where they do;
  3. exposure on from the start, keyframes added up to 141 with pose refinement enabled at 70: every row regrow keeps
     the older keyframes' E, pose, camera block and Adam state bit for bit, and a batch across the boundaries matches the
     oracle;
  4. the bounds of the slot count and of the view indices.

The oracle side uses that every slot holding a keyframe renders the same image: the mean over the S slots is evaluated
once per distinct keyframe of the batch, weighted by the number of slots holding it.
"""
import itertools

import numpy as np
import pytest

from helpers import grad_close
from test_gpu_exposure import E_STAR, EXPO_LR, IDENTITY, _reference_expo
from test_gpu_mapper_grads import (B1, C1, F, GROUPS, H, P, W, _check_step, _check_untouched, _compare, _lr6, _mapper, _raw,
                                   _recovered, _scene, _state)
from test_gpu_pose import LR_R, LR_T, _check_pose_grad, _pose_reference

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

N_KF = 12                                    # training keyframes of tests 1, 2 and 4
N_IMG = 4                                    # ground-truth images, shared round-robin by the keyframes
A, B, C = 5, 8, 9                            # test 1: A in three slots per step; B only in slot 0, C only in slot S - 1


def _orbit(n, seed=41):
    """n keyframes on the rig circle (synthetic.orbit_pose with n views), N_IMG ground truths shared between them.  The
    mapper keeps a pointer to each image: the returned list keeps the arrays alive as long as the test holds it."""
    from gaussian_lic_b200 import synthetic as syn
    poses = [syn.orbit_pose(v, n_views=n) for v in range(n)]
    imgs = [syn.make_gt_image(W, H, seed=seed + i) for i in range(N_IMG)]
    return poses, [imgs[k % N_IMG] for k in range(n)]


def _exposures(n):
    """distinct, asymmetric, non-identity E per keyframe"""
    rng = np.random.default_rng(5)
    return [(E_STAR[k % 3] + rng.uniform(-0.03, 0.03, (3, 4))).astype(np.float32) for k in range(n)]


def _flat(x):
    if isinstance(x, dict):
        return [a for k in sorted(x) for a in _flat(x[k])]
    if isinstance(x, (tuple, list)):
        return [a for v in x for a in _flat(v)]
    return [np.atleast_1d(np.asarray(x))]


def _same(x, y):
    """bit-identical, element by element, through nested tuples / lists / dicts"""
    a, b = _flat(x), _flat(y)
    return len(a) == len(b) and all(p.dtype == q.dtype and p.shape == q.shape and p.tobytes() == q.tobytes() for p, q in zip(a, b))


def _kf_state(m, k, pose=True):
    """(E, exposure exp_avg, exp_avg_sq, steps), (R_wc, t_wc, camera block), (pose exp_avg, exp_avg_sq, steps) of keyframe k"""
    return m.exposure_state(k), m.pose(k, camera=True) if pose else None, m.pose_state(k) if pose else None


def _batch_reference(raw, cams, gts, Es, batch, oracles):
    """The mean over the S slots of `batch` of the f64 oracle's dL/d(raw parameters) through the exposure (_reference_expo),
    and per keyframe (1/S) * the sum over its slots of dL/dE and of dL/d(rho, omega) (_pose_reference, with the f32 oracle's
    value as the yardstick); the loss of each keyframe's view.  oracles = (f32, f64)."""
    oracle32, oracle64 = oracles
    S = len(batch)
    mult = {k: batch.count(k) for k in dict.fromkeys(batch)}
    out = dict(radii=[], oracle_radii=[], dE={}, pose={"float32": {}, "float64": {}}, loss={},
               grads={"float64": {g: 0.0 for g in GROUPS}})
    for k, n in mult.items():
        r = _reference_expo(raw, cams, gts, [k], Es, oracle64)
        acc = out["grads"]["float64"]
        for g in GROUPS:
            acc[g] = acc[g] + (n / S) * r["grads"]["float64"][g]
        out["radii"] += r["radii"]
        out["oracle_radii"] += r["oracle_radii"]
        out["loss"][k] = r["loss"]
        out["dE"][k] = (n / S) * r["dE"][k]
        pr, _ = _pose_reference(raw, cams, gts, [k], [oracle32, oracle64], Es=Es)
        for dt in ("float32", "float64"):
            out["pose"][dt][k] = (n / S) * pr[dt][k]
    out["grads"]["float32"] = out["grads"]["float64"]              # _compare's yardstick line: not measured here
    out["vis"] = np.any([r > 0 for r in out["radii"]], axis=0)
    return out


def _step_against_oracle(m, batch, n_train, gts, oracles, what, groups=GROUPS, rtol=None):
    """One optimiser step over `batch` (S slots, exposure and pose refinement on), checked against the f64 oracle at the
    cameras and exposures the keyframes had before it.  groups: the Gaussians' parameter groups compared with _compare (a
    map of isotropic, unrotated rows only has a rotation gradient of rounding noise, which the caller bounds itself);
    rtol: _compare's per-group tolerances"""
    before, it0 = _state(m), m.stats().iterations
    pre = [_kf_state(m, k) for k in range(n_train)]
    kfs = list(dict.fromkeys(batch))
    cams = {k: pre[k][1][2] for k in kfs}                          # the (refined) device camera block
    Es = {k: pre[k][0][0] for k in kfs}
    st = m.optimize(batch)
    assert st.iterations == it0 + 1, what
    after = _state(m)
    post = [_kf_state(m, k) for k in range(n_train)]
    ref = _batch_reference(_raw(before), cams, gts, Es, batch, oracles)
    want_loss = ref["loss"][batch[-1]]                             # the statistics keep the loss of the last slot
    assert abs(st.last_loss - want_loss) <= 1e-5 * want_loss, (what, st.last_loss, want_loss)
    got = _recovered(before, after)
    rows = np.flatnonzero(ref["vis"])
    _compare(got, ref, rows, what, groups, rtol)
    _check_step(before, after, got, rows, _lr6(), what)
    _check_untouched(before, after, ~ref["vis"], what)
    got_pose = {}
    for k in range(n_train):
        if k not in kfs:                                           # outside the batch: E, pose, camera block, Adam state kept
            assert _same(pre[k], post[k]), "%s: keyframe %d is not in the batch but changed" % (what, k)
            continue
        (_, em0, _, et0), _, (pm0, _, pt0) = pre[k]
        (E1, em1, _, et1), _, (pm1, _, pt1) = post[k]
        assert et1 == et0 + 1 and pt1 == pt0 + 1, (what, k, et0, et1, pt0, pt1)   # one step, whatever the multiplicity
        assert not np.array_equal(E1, pre[k][0][0]), (what, k)
        gE = (em1.astype(np.float64) - (B1 * em0).astype(np.float64)) / C1
        err = np.linalg.norm(gE - ref["dE"][k]) / np.linalg.norm(ref["dE"][k])
        print("%s: keyframe %d in slots %s: dL/dE |diff|/|ref| = %.2e against the f64 oracle" % (
            what, k, [s for s, v in enumerate(batch) if v == k], err))
        assert err <= 1e-4, (what, k, err)
        got_pose[k] = (pm1.astype(np.float64) - (B1 * pm0).astype(np.float64)) / C1
    _check_pose_grad(got_pose, ref["pose"], what)
    return ref


def _wide_mapper(raw, poses, gts, S, **kw):
    m = _mapper(raw, poses, gts, capacity=P, views_per_rank=S, **kw)
    m.enable_exposure(EXPO_LR)
    m.enable_pose_refinement(LR_T, LR_R)
    for k, E in enumerate(_exposures(len(poses))):
        m.set_exposure(k, E)
    return m


def _wide_batches(S):
    """step 1: A in slots 0, 13 S / 32 and S - 1; step 2: B only in slot 0, C only in slot S - 1, A in slots 1, 13 S / 32
    and S - 2; the other slots cycle over a few keyframes, so that some keyframes are in neither batch"""
    mid = 13 * S // 32
    fill = itertools.cycle([1, 2, 3, 4, 6, 7])
    b1 = [A if s in (0, mid, S - 1) else next(fill) for s in range(S)]
    fill = itertools.cycle([2, 3, 6, 10])
    b2 = [B if s == 0 else C if s == S - 1 else A if s in (1, mid, S - 2) else next(fill) for s in range(S)]
    return b1, b2


# ---- 1. full-width batches, exposure and pose refinement on ------------------------------------------------------------
@pytest.mark.parametrize("S,deg", [(8, 3), (8, 1), (32, 3)], ids=["S8-deg3", "S8-deg1", "S32-deg3"])
def test_wide_batch_steps_match_oracle(oracle32, oracle64, S, deg):
    raw = _scene(deg)
    poses, gts = _orbit(N_KF)
    m = _wide_mapper(raw, poses, gts, S)
    b1, b2 = _wide_batches(S)
    assert {B, C}.isdisjoint(b1) and b2.count(B) == b2.count(C) == 1 and b1.count(A) == b2.count(A) == 3
    for step, batch in enumerate((b1, b2)):
        what = "S = %d, degree %d, step %d" % (S, deg, step + 1)
        assert set(range(N_KF)) - set(batch), what                  # some keyframes sit out
        _step_against_oracle(m, batch, N_KF, gts, (oracle32, oracle64), what)
    assert m.stats().iterations == 2
    m.close()


# ---- 2. the wrapped last batch -------------------------------------------------------------------------------------------
WRAP_LIST = [3, 7, 1, 10, 0, 5, 11, 2, 8, 4, 9]                  # 11 views at S = 8: the second batch wraps around


def test_wrapped_last_batch_equals_explicit_batches():
    """optimize(list) at S = 8 over 11 views against a twin mapper given the two batches it spells out: list[:8], then
    list[8:] + list[:5].  The render backward sums with float atomics, so two runs agree bit for bit only where that order
    does not enter.  With the Gaussians and the poses frozen (all their rates zero: every update is an exact zero) each
    render, each dL/dE and so each exposure and its Adam state are bit-identical, as are the parameters, the poses and the
    camera blocks; the Gaussians' and the poses' moments, which hold gradients summed by the atomics, are compared at the
    mapper gradient tests' tolerance.  The step counts are exact."""
    raw = _scene(3)
    poses, gts = _orbit(N_KF, seed=51)
    frozen = dict(position_lr=0.0, feature_lr=0.0, opacity_lr=0.0, scaling_lr=0.0, rotation_lr=0.0)
    lst = WRAP_LIST
    batches = [lst[:8], lst[8:] + lst[:5]]
    out = []
    for explicit in (False, True):
        m = _mapper(raw, poses, gts, capacity=P, views_per_rank=8, **frozen)
        m.enable_exposure(EXPO_LR)
        m.enable_pose_refinement(0.0, 0.0)
        for k, E in enumerate(_exposures(N_KF)):
            m.set_exposure(k, E)
        if explicit:
            for b in batches:
                m.optimize(b)
        else:
            m.optimize(lst)
        st = m.stats()
        out.append(dict(iters=st.iterations, loss=st.last_loss, state=_state(m), kf=[_kf_state(m, k) for k in range(N_KF)]))
        m.close()
    a, b = out
    assert a["iters"] == b["iters"] == 2
    print("wrapped list %s at S = 8: last loss %.7f, twin %.7f" % (lst, a["loss"], b["loss"]))
    assert abs(a["loss"] - b["loss"]) <= 1e-6 * b["loss"]          # the loss of list[4]: atomic sum order only
    for key in ("p", "m", "v"):
        for g in GROUPS:
            x, y = a["state"][key][g], b["state"][key][g]
            if key == "p":
                assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), g
            elif y.size:
                grad_close(x, y, "wrapped vs explicit batches: %s of %s" % ({"m": "exp_avg", "v": "exp_avg_sq"}[key], g))
    assert a["state"]["m"]["means"].any()
    for k in range(N_KF):
        steps = sum(k in bb for bb in batches)
        (ea, pa, sa), (eb, pb, sb) = a["kf"][k], b["kf"][k]
        assert ea[3] == eb[3] == steps and sa[2] == sb[2] == steps, (k, ea[3], eb[3], sa[2], sb[2], steps)
        assert _same(ea, eb), "keyframe %d: exposure state differs from the twin's" % k
        assert _same(pa, pb), "keyframe %d: pose differs from the twin's" % k
        if steps:
            assert not np.array_equal(ea[0], _exposures(N_KF)[k])
            for x, y in zip(sa[:2], sb[:2]):
                err = np.abs(x.astype(np.float64) - y).max() / np.abs(y).max()
                assert err <= 1e-4, (k, x, y)
    print("step counts per keyframe: %s" % [a["kf"][k][0][3] for k in range(N_KF)])


# ---- 3. per-keyframe state across the row regrows ------------------------------------------------------------------------
N_GROW = 141


def test_keyframe_state_survives_row_growth(oracle32, oracle64):
    """Exposure on from the start (rows for 64 keyframes, then 128, 256), pose refinement enabled with 70 keyframes present
    (rows for 70, then 140, 280).  Each add_keyframe that crosses one of those sizes must leave every older training
    keyframe's E, pose, camera block and Adam state bit-identical and start the new one at the identity E and its given pose
    with zero state; held-out keyframes are added in between.  S = 8 steps between the stages keep the state non-trivial,
    and a last batch across all four boundaries is checked against the oracle."""
    from gaussian_lic_b200 import mapper
    raw = _scene(3)
    poses, gts = _orbit(N_GROW, seed=61)
    m = mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=3, capacity=P, views_per_rank=8)
    m.initialize(raw)
    m.enable_exposure(EXPO_LR)
    pose_on = False
    n_test = 0

    def add(k):
        nonlocal n_test
        m.add_keyframe(*poses[k], gts[k])
        if k % 16 == 7:                                            # a held-out keyframe between the training ones
            m.add_keyframe(*poses[k], gts[k + 1], train=False)
            n_test += 1

    def check_new(k):
        E, em, ev, et = m.exposure_state(k)
        assert np.array_equal(E, IDENTITY) and not em.any() and not ev.any() and et == 0, k
        if pose_on:
            R, t, cam = m.pose(k, camera=True)
            pm, pv, pt = m.pose_state(k)
            assert np.array_equal(R, poses[k][0].astype(np.float32)) and np.array_equal(t, poses[k][1].astype(np.float32)), k
            want = mapper.camera_block(W, H, F, F, W / 2.0, H / 2.0, *poses[k])
            assert all(np.array_equal(cam[key], want[key]) for key in ("view", "proj", "campos")), k
            assert not pm.any() and not pv.any() and pt == 0, k

    def add_across(k, what):
        snap = [_kf_state(m, i, pose_on) for i in range(k)]
        add(k)
        kept = [_same(s, _kf_state(m, i, pose_on)) for i, s in enumerate(snap)]
        stepped = sum(s[0][3] > 0 for s in snap)
        moved = sum(s[2][2] > 0 for s in snap) if pose_on else 0
        print("add training keyframe %d (%s): %d / %d older keyframes bit-identical before and after (%d with exposure "
              "steps, %d with pose steps); %d held-out keyframes so far" % (k, what, sum(kept), k, stepped, moved, n_test))
        assert all(kept), "%s: keyframes %s changed" % (what, [i for i, ok in enumerate(kept) if not ok])
        assert stepped > 0 and (moved > 0 or not pose_on), what
        check_new(k)

    for k in range(64):
        add(k)
    m.optimize([0, 1, 5, 17, 33, 50, 62, 63])
    add_across(64, "exposure rows 64 -> 128")
    for k in range(65, 70):
        add(k)
    m.optimize([0, 5, 63, 64, 2, 3, 40, 69])
    m.enable_pose_refinement(LR_T, LR_R)                           # 70 training keyframes: pose rows for exactly 70
    pose_on = True
    for k in range(70):                                            # every keyframe starts at its given pose
        R, _ = m.pose(k)
        assert np.array_equal(R, poses[k][0].astype(np.float32)) and m.pose_state(k)[2] == 0, k
    m.optimize([1, 5, 30, 63, 64, 69, 0, 12])
    add_across(70, "pose rows 70 -> 140")
    for k in range(71, 128):
        add(k)
    m.optimize([5, 63, 64, 69, 70, 100, 127, 2])
    add_across(128, "exposure rows 128 -> 256")
    for k in range(129, 140):
        add(k)
    m.optimize([5, 63, 64, 69, 70, 127, 128, 139])
    add_across(140, "pose rows 140 -> 280")
    _step_against_oracle(m, [5, 63, 64, 69, 70, 127, 128, 140], N_GROW, gts, (oracle32, oracle64), "after the regrows, S = 8")
    m.close()


# ---- 4. slot bounds ----------------------------------------------------------------------------------------------------------
def test_slot_count_and_view_index_bounds():
    """32 slots per step are accepted, 33 (one rank or two ranks x 17) refused with GLIC_ERR_INVALID_ARGUMENT; a view index
    out of range in slot 31 -- of the only batch, or of the second batch of a list -- is refused before anything is
    enqueued: parameters, moments, per-keyframe state and the iteration count stay as they were."""
    from gaussian_lic_b200 import capi, mapper
    for world, k in ((1, 33), (2, 17)):
        with pytest.raises(capi.GlicError, match=r"mapper_create failed \(-1\)"):
            mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=1, world=world, views_per_rank=k)
    raw = _scene(1)
    poses, gts = _orbit(N_KF, seed=71)
    m = _wide_mapper(raw, poses, gts, 32)
    ok = [k % N_KF for k in range(32)]
    m.optimize(ok)                                                 # one real step: non-zero moments and per-keyframe state
    assert m.stats().iterations == 1
    before, kf0 = _state(m), [_kf_state(m, k) for k in range(N_KF)]
    for bad in (ok[:31] + [N_KF], ok[:31] + [-1], ok + ok[:31] + [N_KF]):
        with pytest.raises(capi.GlicError, match=r"mapper_optimize failed \(-1\): .*out of range"):
            m.optimize(bad)
        assert m.stats().iterations == 1, len(bad)
        after = _state(m)
        for key in ("p", "m", "v"):
            for g in GROUPS:
                assert np.array_equal(before[key][g].view(np.uint32), after[key][g].view(np.uint32)), (len(bad), key, g)
        assert all(_same(kf0[k], _kf_state(m, k)) for k in range(N_KF)), len(bad)
    m.optimize(ok)                                                 # the mapper still steps
    assert m.stats().iterations == 2
    m.close()
