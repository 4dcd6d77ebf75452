"""glic_mapper_prune (csrc/prune.cu): stable compaction of the native mapper's arenas by activated opacity.

Checkers: a NumPy oracle on the mapper's own download (rows[act >= min_opacity], act from glic_activations_forward, the
activation kernel the decision shares), a second mapper built from the same initialisation and never pruned (renders,
evaluation, extend() and training), glic_ply_write of the surviving rows for save_map, and the two replicas of a two-rank run.
"""
import ctypes as C
import os
import socket

import numpy as np
import pytest

from helpers import small_scene

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

W, H, F = 320, 208, 250.0
KEYS = ("means", "dc", "sh", "opacity_logits", "log_scales", "rots")
LR = dict(rots=0.001, means=1.6e-4, log_scales=0.005, opacity_logits=0.05, dc=2.5e-3, sh=2.5e-3 / 20)   # config/fastlivo.yaml:18-22


def _mapper(deg=3, capacity=0, **kw):
    from gaussian_lic_b200 import mapper
    return mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=deg, capacity=capacity, **kw)


def _poses(views):
    from gaussian_lic_b200 import synthetic as syn
    return [syn.orbit_pose(v, radius=2.0) for v in views]


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same(a, b, what):
    assert a.shape == b.shape and np.array_equal(_bits(a), _bits(b)), what


def _act(logits):
    """glic_activations_forward of the logits: the exact float the prune decides on"""
    from gaussian_lic_b200 import capi
    n = int(logits.size)
    dev = torch.device("cuda:0")
    f32 = dict(dtype=torch.float32, device=dev)
    lg = torch.as_tensor(np.ascontiguousarray(logits, np.float32).reshape(n)).to(dev)
    ls, rot = torch.zeros(n, 3, **f32), torch.ones(n, 4, **f32)
    o, s, r = torch.empty(n, **f32), torch.empty(n, 3, **f32), torch.empty(n, 4, **f32)
    torch.cuda.synchronize()
    capi.check(capi.lib.glic_activations_forward(n, capi.ptr(lg), capi.ptr(ls), capi.ptr(rot), capi.ptr(o), capi.ptr(s), capi.ptr(r), None),
               "activations_forward")
    torch.cuda.synchronize()
    return o.cpu().numpy()


def _moment_rows(mom, P, M, rows):
    """rows of a packed moment download (glic_packed_offsets(P, M) layout), repacked for len(rows) rows"""
    out, off = [], 0
    for k in (4, 3, 3, 1, 3, 3 * M):
        out.append(mom[off:off + P * k].reshape(P, k)[rows].reshape(-1))
        off += P * k
    return np.concatenate(out)


def _expect_rows(dl, M, rows):
    P = dl["means"].shape[0]
    out = {k: dl[k][rows] for k in KEYS}
    for k in ("exp_avg", "exp_avg_sq"):
        if k in dl:
            out[k] = _moment_rows(dl[k], P, M, rows)
    return out


def _check_download(got, want, what):
    for k in want:
        _same(got[k], want[k], "%s: %s" % (what, k))


def _compare(a, b, steps, what):
    """test_gpu_mapper.py's atomic-order criterion: two runs of the same training differ only through the render backward's
    float-atomic order; per group 99.9 % of the entries within 2 % of one learning rate, none beyond the sign-flip bound."""
    worst = {}
    for k, lr in LR.items():
        x, y = np.asarray(a[k], np.float64).reshape(-1), np.asarray(b[k], np.float64).reshape(-1)
        assert x.shape == y.shape, (what, k)
        if x.size == 0:
            continue
        d = np.abs(x - y)
        worst[k] = (np.quantile(d, 0.999) / lr, d.max() / lr)
    msg = "%s: |param diff| / lr (q99.9, max): %s" % (what, {k: "%.2g, %.2g" % v for k, v in worst.items()})
    print(msg)
    for k, (q, mx) in worst.items():
        assert q <= 0.02 + 1e-7 / LR[k], msg
        assert mx <= 6.4 * steps + 1e-7 / LR[k], msg


def _logit(p):
    return np.float32(np.log(p / (1.0 - p)))


def _sweep(center, n):
    """n consecutive float32 values around `center`"""
    b = np.float32(center).view(np.int32).astype(np.int64)
    return (b + np.arange(-(n // 2), n - n // 2)).astype(np.int32).view(np.float32)


@pytest.mark.parametrize("deg,thr", [(3, None), (0, None), (3, 0.3), (0, 0.62)])
def test_prune_matches_numpy_oracle(deg, thr):
    """A third of the rows carry consecutive floats around logit(min_opacity), behind every camera (never trained, so the sweep
    is intact at prune time); the others train a few steps.  prune == rows[act >= min_opacity] of the download before it, for
    every group and both moments, bit for bit; a dry run changes nothing and returns the same count."""
    from gaussian_lic_b200 import mapper, synthetic as syn
    thr = mapper.DEAD_OPACITY if thr is None else float(np.float32(thr))
    P = 6000
    g, _ = small_scene(P, W, H, 23, deg)
    rng = np.random.default_rng(5)
    sweep_rows = np.sort(rng.choice(P, P // 3, replace=False))
    sweep = _sweep(_logit(thr), sweep_rows.size)
    act_sweep = _act(sweep)
    # the activation crosses the threshold inside the sweep: rows on both sides of the cut differ by single ulps of the logit
    below = act_sweep < np.float32(thr)
    cross = int(below.sum())
    assert 0 < cross < sweep.size, cross
    print("threshold %.9g: largest logit removed %.9g (act %.9g), smallest kept %.9g (act %.9g)"
          % (thr, sweep[below].max(), act_sweep[below][np.argmax(sweep[below])], sweep[~below].min(),
             act_sweep[~below][np.argmin(sweep[~below])]))
    g = dict(g)
    g["opacity_logits"] = np.asarray(g["opacity_logits"], np.float32).copy()
    g["opacity_logits"][sweep_rows] = rng.permutation(sweep)
    g["means"] = np.asarray(g["means"], np.float32).copy()
    g["means"][sweep_rows, 2] = -5.0                                       # behind both cameras: culled, never stepped
    poses = _poses([0, 3])
    m = _mapper(deg)
    m.initialize(g)
    for i, (R, t) in enumerate(poses):
        m.add_keyframe(R, t, syn.make_gt_image(W, H, seed=30 + i))
    m.optimize([0, 1, 1, 0])
    before = m.download(moments=True)
    _same(before["opacity_logits"][sweep_rows], g["opacity_logits"][sweep_rows], "the sweep rows were stepped")
    assert np.count_nonzero(before["exp_avg"]) > 0 and np.count_nonzero(before["exp_avg_sq"]) > 0
    keep = _act(before["opacity_logits"]) >= np.float32(thr)
    n_removed = int((~keep).sum())
    assert 0 < n_removed < P and (~keep[sweep_rows]).sum() == cross
    st0 = m.stats()
    assert m.prune(thr, dry_run=True) == n_removed
    _check_download(m.download(moments=True), before, "dry run")
    assert m.stats().num_gaussians == P and m.stats().capacity == st0.capacity
    assert m.prune(thr) == n_removed
    st = m.stats()
    assert st.num_gaussians == P - n_removed and st.capacity == st0.capacity and m.sky_rows() == 0
    _check_download(m.download(moments=True), _expect_rows(before, m.M, keep), "prune")
    assert m.prune(thr) == 0                                               # nothing left below the threshold
    st = m.optimize([0, 1])                                                # training continues on the compacted arena
    assert np.isfinite(st.last_loss) and st.num_gaussians == P - n_removed
    m.close()


@pytest.mark.parametrize("deg", [1, 2])
def test_prune_large_map(deg):
    """1.2 M rows (1172 tiles of the selection: the tile scan runs over more than one 1024-wide chunk), SH degrees 1 and 2,
    rows removed in runs and singly, the first and the last row among them."""
    from gaussian_lic_b200 import synthetic as syn
    P = 1_200_000
    g = syn.make_gaussians(P, W, H, F, F, sh_degree=deg, zmax=12.0, seed=3, log_scale_mean=-3.0)
    rng = np.random.default_rng(11)
    lg = rng.uniform(-9.0, 3.0, P).astype(np.float32)
    lg[:5000] = -20.0                                                      # a run of removed rows at the front ...
    lg[-3] = -20.0                                                         # ... and near the end
    lg[0], lg[P - 1] = -20.0, -20.0
    g = dict(g, opacity_logits=lg)
    m = _mapper(deg)
    m.initialize(g)
    before = m.download(moments=True)
    for thr in (1.0 / 255.0, 0.25):
        thr = float(np.float32(thr))
        keep = _act(before["opacity_logits"]) >= np.float32(thr)
        assert m.prune(thr, dry_run=True) == int((~keep).sum())
        assert m.prune(thr) == int((~keep).sum())
        after = m.download(moments=True)
        _check_download(after, _expect_rows(before, m.M, keep), "large map, threshold %g" % thr)
        before = after
    m.close()


def _scene_with_dead_rows(P, seed, deg=3):
    """small_scene with a third of the rows below the 1/255 cut (in front of the cameras: alive they would be drawn) and some
    rows just above it"""
    g, _ = small_scene(P, W, H, seed, deg)
    rng = np.random.default_rng(seed)
    lg = np.asarray(g["opacity_logits"], np.float32).copy()
    rows = rng.permutation(P)
    dead, faint = rows[:P // 3], rows[P // 3:P // 3 + P // 10]
    lg[dead] = rng.uniform(-12.0, -5.55, dead.size)
    lg[faint] = rng.uniform(-5.52, -4.5, faint.size)
    lg[rows[-40:]] = _sweep(_logit(1.0 / 255.0), 40)                       # on the cut itself
    return dict(g, opacity_logits=lg)


def _scan(n, seed, R_wc, t_wc):
    rng = np.random.default_rng(seed)
    z = rng.uniform(0.5, 15.0, n)
    pts_cam = np.stack([z * rng.uniform(-0.8, 0.8, n), z * rng.uniform(-0.6, 0.6, n), z], 1)
    pts = (pts_cam @ np.asarray(R_wc).T + np.asarray(t_wc)).astype(np.float32)
    cols = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    return pts, cols, z.astype(np.float32)


def _pruned_pair(g, poses, gts):
    """mappers A and B from one initialisation with three training keyframes and a held-out one; A pruned at 1/255"""
    from gaussian_lic_b200 import mapper
    P = g["means"].shape[0]
    ms = []
    for _ in range(2):
        m = _mapper(3, capacity=P)
        m.initialize(g)
        for i in range(3):
            m.add_keyframe(*poses[i], gts[i])
        m.add_keyframe(*poses[3], gts[3], train=False)
        ms.append(m)
    A, B = ms
    init = B.download(moments=True)
    dead = _act(init["opacity_logits"]) < np.float32(mapper.DEAD_OPACITY)
    cap = A.stats().capacity
    assert A.prune() == int(dead.sum()) and dead.sum() > P // 3 - 50
    assert A.stats().num_gaussians == P - dead.sum() and A.stats().capacity == cap
    _check_download(A.download(moments=True), _expect_rows(init, 15, ~dead), "A after prune")
    return A, B, init, dead


def test_pruning_dead_rows_changes_nothing_else():
    """A and B from one initialisation, A pruned at 1/255: the same renders, metrics and extend() rows bit for bit; on a second
    such pair, the same training up to the render backward's atomic order, and B's dead rows never move."""
    from gaussian_lic_b200 import synthetic as syn
    P = 6000
    g = _scene_with_dead_rows(P, 41)
    poses = _poses([0, 2, 5, 1])
    gts = [syn.make_gt_image(W, H, seed=50 + i) for i in range(4)]
    A, B, init, dead = _pruned_pair(g, poses, gts)
    alive = np.nonzero(~dead)[0]
    cap = A.stats().capacity
    # right after the prune: every keyframe renders and scores the same, bit for bit
    for train, idx in [(1, 0), (1, 1), (1, 2), (0, 0)]:
        _same(A.render(idx, train=bool(train)), B.render(idx, train=bool(train)), "render %d/%d" % (train, idx))
        assert A.evaluate(idx, train=bool(train)) == B.evaluate(idx, train=bool(train)), (train, idx)
    # extend() on the newest training keyframe appends the same rows to both, across a capacity regrow of both arenas
    pts, cols, dep = _scan(20000, 9, *poses[2])
    na, nb = A.extend(pts, cols, dep), B.extend(pts, cols, dep)
    assert na == nb > 0
    assert A.stats().capacity > cap and B.stats().capacity > cap, (cap, A.stats().capacity, B.stats().capacity)
    da, db = A.download(moments=True), B.download(moments=True)
    new_a = _expect_rows(da, 15, np.arange(alive.size, alive.size + na))
    new_b = _expect_rows(db, 15, np.arange(P, P + nb))
    _check_download(new_a, new_b, "extend() rows")
    _check_download(_expect_rows(da, 15, np.arange(alive.size)), _expect_rows(db, 15, alive), "old rows after extend()")
    A.close(); B.close()
    # training on fixed views (a fresh pair: the rows extend() appends start isotropic with the identity rotation, so their
    # rotation gradient is rounding noise that Adam's normalisation turns into steps of either sign): A's rows follow B's
    # surviving rows; B's dead rows stay as they were at the prune
    A, B, init, dead = _pruned_pair(g, poses, gts)
    steps = 0
    for _ in range(3):
        sa, sb = A.optimize([0, 1, 2]), B.optimize([0, 1, 2])
        steps += 3
        assert np.isfinite(sa.last_loss) and np.isfinite(sb.last_loss)
    da, db = A.download(), B.download(moments=True)
    _compare(da, {k: db[k][alive] for k in KEYS}, steps, "A vs B's survivors after %d steps" % steps)
    _check_download(_expect_rows(db, 15, dead), _expect_rows(init, 15, dead), "B's dead rows")
    A.close(); B.close()


def _lidar_scan(n, seed, R_wc=None, t_wc=None):
    """test_gpu_initialize.py's scan: n points in front of a camera, 8-bit colours as the Dataset's doubles"""
    rng = np.random.default_rng(seed)
    z = rng.uniform(0.5, 15.0, n)
    pts = np.stack([z * rng.uniform(-0.6, 0.6, n), z * rng.uniform(-0.4, 0.4, n), z], 1)
    if R_wc is not None:
        pts = pts @ np.asarray(R_wc, np.float64).T + np.asarray(t_wc, np.float64)
    cols = rng.integers(0, 256, (n, 3)) / 255.0
    dep = np.exp(rng.uniform(np.log(0.1), np.log(200.0), n)).astype(np.float32)
    return pts.astype(np.float32), cols, dep


def _ply_write(path, d, rows):
    from gaussian_lic_b200 import capi
    a = {k: np.ascontiguousarray(d[k][rows], np.float32) for k in KEYS}
    p = lambda x: x.ctypes.data_as(C.c_void_p) if x.size else None
    capi.check(capi.lib.glic_ply_write(str(path).encode(), len(rows), a["sh"].shape[1], p(a["means"]), p(a["dc"]), p(a["sh"]),
                                       p(a["opacity_logits"]), p(a["log_scales"]), p(a["rots"])), "ply_write")


def _split(vals):
    """a threshold with rows of `vals` on both sides"""
    u = np.unique(vals)
    assert u.size >= 2, "nothing to split"
    return float(u[u.size // 2])


def test_sky_rows_and_save_map(tmp_path):
    """initialize_lidar with a sky, some training, then a prune splitting the LiDAR rows (the sky survives) and one splitting the
    sky: sky_rows() counts the surviving sky rows and save_map writes exactly the surviving non-sky rows."""
    from gaussian_lic_b200 import synthetic as syn
    n, S = 6000, 4000
    FOCAL = 250.0
    poses = _poses([0, 1])
    pts, cols, dep = _lidar_scan(n, 5, *poses[0])
    m = _mapper(3, seed=3)
    m.initialize_lidar(pts, cols, dep, FOCAL, S, 1000)
    for i, (R, t) in enumerate(poses):
        m.add_keyframe(R, t, syn.make_gt_image(W, H, seed=3 + i))
    m.optimize([0, 1] * 4)
    sky = S
    for part in ("lidar", "sky"):
        before = m.download(moments=True)
        P = before["means"].shape[0]
        act = _act(before["opacity_logits"])
        thr = _split(act[sky:]) if part == "lidar" else _split(act[:sky])
        thr = float(np.float32(thr))
        keep = act >= np.float32(thr)
        sky_new = int(keep[:sky].sum())
        assert (sky_new == sky) if part == "lidar" else (0 < sky_new < sky), (part, sky_new, sky)
        assert m.prune(thr) == int((~keep).sum())
        assert m.sky_rows() == sky_new
        after = m.download(moments=True)
        _check_download(after, _expect_rows(before, m.M, keep), "sky test, %s split" % part)
        sky = sky_new
        P = after["means"].shape[0]
        m.save_map(tmp_path / ("mine_%s.ply" % part))
        _ply_write(tmp_path / ("want_%s.ply" % part), after, np.arange(sky, P))
        assert (tmp_path / ("mine_%s.ply" % part)).read_bytes() == (tmp_path / ("want_%s.ply" % part)).read_bytes(), part
        print("%s split at %.6g: %d rows kept, %d of them sky" % (part, thr, P, sky))
    st = m.optimize([0, 1])
    assert np.isfinite(st.last_loss)
    m.close()


def test_rejected_arguments_leave_the_model_untouched():
    from gaussian_lic_b200 import capi, synthetic as syn
    pts, cols, dep = _lidar_scan(2000, 7)
    m = _mapper(3, seed=9)
    m.initialize_lidar(pts, cols, dep, 250.0, 500, 1000)
    m.add_keyframe(*_poses([0])[0], syn.make_gt_image(W, H, seed=2))
    m.optimize([0, 0])
    before, st0, sky0 = m.download(moments=True), m.stats(), m.sky_rows()
    assert np.all(_act(before["opacity_logits"]) < np.float32(1.0))
    out = C.c_uint32(12345)
    for thr, dry in [(float("nan"), 0), (float("nan"), 1), (-0.1, 0), (-1e-30, 0), (1.5, 0), (float("inf"), 0), (float("-inf"), 0),
                     (1.0, 0), (1.0, 1)]:                                  # 1.0 removes every row here
        assert capi.lib.glic_mapper_prune(m._h, thr, dry, C.byref(out)) == -1, (thr, dry)
        _check_download(m.download(moments=True), before, "rejected prune(%r, %d)" % (thr, dry))
        assert m.sky_rows() == sky0 and m.stats().num_gaussians == st0.num_gaussians and m.stats().capacity == st0.capacity
    assert capi.lib.glic_mapper_prune(None, 0.5, 0, C.byref(out)) == -1
    assert capi.lib.glic_mapper_prune(m._h, 0.0, 0, None) == 0             # removes nothing; the count pointer may be NULL
    _check_download(m.download(moments=True), before, "prune(0)")
    m.close()
    empty = _mapper(0)                                                     # no rows: OK, 0 removed
    assert capi.lib.glic_mapper_prune(empty._h, 0.5, 0, C.byref(out)) == 0 and out.value == 0
    empty.close()


# ---- two ranks, spawned as tests/test_gpu_mapper_multi.py spawns them ------------------------------------------------------
P2 = 5000
BATCHES = [[0, 1], [2, 0], [1, 2], [0, 2]]


def _run_rank(rank, world, exchange):
    from gaussian_lic_b200 import mapper, synthetic as syn
    g = _scene_with_dead_rows(P2, 44)
    poses = _poses([0, 2, 5])
    m = mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=3, capacity=P2, rank=rank, world=world, views_per_rank=1)
    m.initialize(g)
    for i, (R, t) in enumerate(poses):
        m.add_keyframe(R, t, syn.make_gt_image(W, H, seed=21 + i))
    m.connect(exchange(m.export_handle()))
    m.optimize([v for b in BATCHES[:2] for v in b])
    removed = [m.prune(), m.prune(0.2)]                                   # the dead rows, then a threshold through live ones
    pruned = m.download(moments=True)
    st = m.optimize([v for b in BATCHES[2:] for v in b])
    assert st.iterations == len(BATCHES) and st.overflow_regrows == 0 and np.isfinite(st.last_loss)
    final = m.download(moments=True)
    return m, removed, pruned, final


def _worker(rank, world, port, q):
    try:
        import torch.distributed as dist
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
        torch.cuda.set_device(rank % torch.cuda.device_count())

        def exchange(mine):
            got = [None] * world
            dist.all_gather_object(got, mine)
            return got

        m, removed, pruned, final = _run_rank(rank, world, exchange)
        dist.barrier()
        m.close()
        dist.destroy_process_group()
        q.put((rank, "ok", (removed, pruned, final)))
    except Exception as e:          # noqa: BLE001 - reported to the parent
        import traceback
        q.put((rank, "%r\n%s" % (e, traceback.format_exc()), None))


@pytest.mark.timeout(300)
def test_two_ranks_prune_identically():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p_ in procs:
        p_.start()
    res = sorted([q.get(timeout=240) for _ in procs], key=lambda r: r[0])
    for p_ in procs:
        p_.join(timeout=30)
    assert all(r[1] == "ok" for r in res), [r[1] for r in res]
    (ra, pa, fa), (rb, pb, fb) = res[0][2], res[1][2]
    assert ra == rb and ra[0] > P2 // 3 - 50 and ra[1] > 0, (ra, rb)
    for name in pa:                                            # replicas: bit-identical after the prune and after training on
        _same(pa[name], pb[name], "replicas differ after the prune in %s" % name)
        _same(fa[name], fb[name], "replicas diverged after the prune in %s" % name)
    assert fa["means"].shape[0] == P2 - sum(ra)
    assert not np.array_equal(fa["means"], pa["means"])        # training moved the compacted map
