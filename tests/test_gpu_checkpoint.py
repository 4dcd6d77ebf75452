"""Mapper checkpoints (include/glic_b200.h "Checkpoints"; Mapper.save_checkpoint / Mapper.from_checkpoint).

* A restored mapper returns every getter's bits, the same PLY, masks, images and view-sampler draws as the one that saved.
* Under the deterministic option, a run interrupted by a save, a new process-like restore and a resume ends bit-identical to the
  uninterrupted run: through density events, for add_frame mappers with a pending scan, and for two connected ranks; and saving
  mid-run changes nothing.
* Float keyframe images keep their memory class and no longer need the caller's arrays.
* Malformed files and non-fresh targets are refused with the target still fresh; failed allocations follow the failure contract.
* tests/checkpoint_format.py, the documented format restated in numpy, reads a GPU-written file to the getters' values."""
import os

import numpy as np
import pytest

import checkpoint_format as CF
from test_gpu_densify import F, SEED, VIEWS, _lidar_scan, _poses, _same, _with_keyframes
from test_gpu_mapper_deterministic import LPIPS, SCHED, W, H, _align, _getters, _same_all, _train, _twin

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

N_STEPS, M_STEPS = 8, 22          # schedule events at iterations 5, 10, 15 (densify) and 12 (opacity reset): the save falls between


def _lpips():
    return LPIPS if os.path.isfile(LPIPS) else None


def _steps(m, first, count):
    """_train's view sequence from step `first` on"""
    for i in range(first, first + count):
        m.optimize([VIEWS[(2 * i) % 8], VIEWS[(2 * i + 1) % 8]])


def _rot(axis, angle):
    a = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * K @ K


def _count(m, train):
    """the number of keyframes in the training (held-out) list"""
    from gaussian_lic_b200 import capi
    n = 0
    while True:
        try:
            m.mask(train, n)
        except capi.GlicError:
            return n
        n += 1


def _extras(m):
    """what _getters leaves out: anchors, every keyframe's mask and image"""
    out = {"anchors": np.asarray(m.anchors())}
    for train in (True, False):
        out["count%d" % train] = np.asarray([_count(m, train)], np.float64)
        for i in range(_count(m, train)):
            mk, cnt = m.mask(train, i)
            out["mask%d_%d" % (train, i)] = np.zeros(1, np.uint8) if mk is None else mk
            out["mask_count%d_%d" % (train, i)] = np.asarray([cnt], np.float64)
            out["image%d_%d" % (train, i)] = m.keyframe_image(i, train)
    return out


def _state(m):
    """every getter whose value does not depend on float atomics: the restored state of a mapper trained without the option"""
    out = {"map." + k: v for k, v in m.download(moments=True).items()}
    out["accum"], out["denom"] = m.densify_stats()
    out["maxr"] = np.asarray(m.screen_radii())
    st = m.stats()
    for f in ("num_gaussians", "capacity", "iterations", "last_inserted", "last_loss", "mean_visible", "overflow_regrows"):
        out["stats." + f] = np.asarray([getattr(st, f)], np.float64)
    for k, v in m.density_totals().items():
        out["totals." + k] = np.asarray(v, np.float64)
    for i in range(len(VIEWS)):
        R, t, cam = m.pose(i, camera=True)
        out["pose%d" % i] = np.concatenate([np.ravel(R), np.ravel(t), cam["view"], cam["proj"], cam["campos"]])
        out["pose_state%d" % i] = np.concatenate([np.ravel(np.asarray(x, np.float64)) for x in m.pose_state(i)])
        out["E_state%d" % i] = np.concatenate([np.ravel(np.asarray(x, np.float64)) for x in m.exposure_state(i)])
    out.update(_extras(m))
    return out


def _restore(m, path):
    from gaussian_lic_b200 import mapper
    m.save_checkpoint(path)
    return mapper.Mapper.from_checkpoint(path, lpips=_lpips())


def _rich_twin(steps=N_STEPS):
    """_twin with a ninth, masked training keyframe, non-trivial anchors and a pose correction, trained `steps` steps"""
    from gaussian_lic_b200 import synthetic as syn
    m = _twin()
    R, t = syn.orbit_pose(2.5, radius=2.0)
    m.add_keyframe(R, t, syn.make_gt_image(W, H, seed=77), train=True)
    yy, xx = np.mgrid[0:H, 0:W]
    m.set_mask(True, len(VIEWS), (xx + yy) % 7 != 0)
    m.set_mask(True, 2, xx > W // 3)
    P = m.stats().num_gaussians
    m.set_anchors(np.arange(P, dtype=np.int32) % (len(VIEWS) + 2) - 1)
    _steps(m, 0, steps // 2)
    R1, t1 = _poses([VIEWS[1]])[0]
    dR, dt = _rot([0.2, 1.0, -0.3], 0.02), np.array([0.01, -0.02, 0.005])
    assert m.correct_poses([(True, 1, (dR @ np.asarray(R1, np.float64)).astype(np.float32),
                             (dR @ np.asarray(t1, np.float64) + dt).astype(np.float32))]) > 0
    _steps(m, steps // 2, steps - steps // 2)
    return m


def _check_format(path, m):
    """the numpy reader of the documented format against the getters of the mapper that wrote the file"""
    f = CF.read(path)
    assert f["order"] == ["MAP ", "CNTR", "KEYF", "EXPO", "POSE", "DENS", "SCHD"]
    mp, d = f["map"], m.download(moments=True)
    st = m.stats()
    assert (mp["P"], mp["Pcap"], mp["n_sky"]) == (st.num_gaussians, st.capacity, m.sky_rows())
    P = mp["P"]
    for k in ("means", "dc", "opacity_logits", "log_scales", "rots"):
        _same(mp["params"][k].reshape(d[k].shape), d[k], "format: " + k)
    _same(mp["params"]["sh"].reshape(d["sh"].shape), d["sh"], "format: sh")
    _same(CF.packed_moments(mp["exp_avg"], m.M), d["exp_avg"], "format: exp_avg")
    _same(CF.packed_moments(mp["exp_avg_sq"], m.M), d["exp_avg_sq"], "format: exp_avg_sq")
    assert np.array_equal(mp["anchor"], m.anchors())
    c = f["counters"]
    assert c["stats"]["iterations"] == st.iterations and c["stats"]["num_gaussians"] == P
    assert c["deterministic"] == 1 and c["optimizer"] == 1
    assert c["flags"] == CF.FLAGS["initialized"] | CF.FLAGS["exposure"] | CF.FLAGS["pose"] | CF.FLAGS["densification"]
    kf = f["keyframes"]
    assert kf["n_test"] == 0 and kf["n_train"] == len(VIEWS) + 1
    for i, k in enumerate(kf["list"]):
        assert k["kind"] == 1 and k["frame"] == 0xFFFFFFFF
        _same(k["image"], m.keyframe_image(i), "format: image %d" % i)
        mk, cnt = m.mask(True, i)
        assert k["mask_valid"] == cnt
        if cnt:
            assert np.array_equal(k["mask"], mk)
        R, t, cam = m.pose(i, camera=True)
        _same(k["cam_dev"][:35], np.concatenate([cam["view"], cam["proj"], cam["campos"]]), "format: device camera %d" % i)
        E, m1, m2, t_e = m.exposure_state(i)
        ex = f["exposure"]
        _same(ex["E"][i], E, "E"); _same(ex["m"][i], m1, "E m"); _same(ex["v"][i], m2, "E v")
        assert ex["t"][i] == t_e
        pm1, pm2, t_p = m.pose_state(i)
        po = f["pose"]
        _same(po["f"][i][:9].reshape(3, 3), R, "pose R"); _same(po["f"][i][9:], t, "pose t")
        _same(po["m"][i], pm1, "pose m"); _same(po["v"][i], pm2, "pose v")
        assert po["t"][i] == t_p
    acc, den = m.densify_stats()
    _same(f["densification"]["accum"], acc, "accum")
    _same(f["densification"]["denom"], den, "denom")
    assert np.array_equal(f["densification"]["maxr"], m.screen_radii())
    tot = m.density_totals()
    s = f["schedule"]
    assert s["on"] == 1 and s["steps"] == tot["steps"] and s["resets"] == tot["resets"]
    assert s["schedule"]["densify_interval"] == SCHED["densify_interval"]


def test_round_trip_restores_every_getter(tmp_path):
    a = _rich_twin()
    path = tmp_path / "a.ckpt"
    b = _restore(a, path)
    _check_format(path, a)
    _same_all(_getters(a), _getters(b), "restored getters")
    _same_all(_extras(a), _extras(b), "restored anchors, masks and images")
    a.save_map(tmp_path / "a.ply")
    b.save_map(tmp_path / "b.ply")
    assert (tmp_path / "a.ply").read_bytes() == (tmp_path / "b.ply").read_bytes()
    for _ in range(3):
        assert a.sample_views() == b.sample_views()
    a.close()
    b.close()


def test_resume_trains_on_bit_identically(tmp_path):
    """twin A trains N + M steps; twin B trains N, saves and is closed; a restored mapper trains the M steps on"""
    a = _rich_twin(N_STEPS)
    _steps(a, N_STEPS, M_STEPS)
    b = _rich_twin(N_STEPS)
    b.save_checkpoint(tmp_path / "b.ckpt")
    b.close()
    from gaussian_lic_b200 import mapper
    c = mapper.Mapper.from_checkpoint(tmp_path / "b.ckpt", lpips=_lpips())
    _steps(c, N_STEPS, M_STEPS)
    tot = a.density_totals()
    assert tot["steps"] >= 3 and tot["resets"] >= 1 and a.stats().iterations == N_STEPS + M_STEPS
    _same_all(_getters(a), _getters(c), "resumed getters")
    _same_all(_extras(a), _extras(c), "resumed anchors, masks and images")
    _same_all(_align(a), _align(c), "resumed align")
    a.close()
    c.close()


def test_saving_mid_run_changes_nothing(tmp_path):
    a, b = _twin(), _twin()
    _train(a, N_STEPS + M_STEPS)
    _steps(b, 0, N_STEPS)
    b.save_checkpoint(tmp_path / "b.ckpt")
    _steps(b, N_STEPS, M_STEPS)
    _same_all(_getters(a), _getters(b), "a twin that saved")
    a.close()
    b.close()


def test_resume_through_add_frame_with_a_pending_scan(tmp_path):
    from test_gpu_frames import FX, FY, RADIUS, SKY, _frames, _padded
    from gaussian_lic_b200 import mapper
    frames = _frames(10, 20_000, 2)

    def start():
        m = mapper.Mapper(W, H, FX, FY, W / 2.0, H / 2.0, sh_degree=3, seed=17)
        m.enable_frames(5, SKY, RADIUS)
        m.set_deterministic(True)
        yy, xx = np.mgrid[0:H, 0:W]
        for i, f in enumerate(frames[:7]):
            m.add_frame(f["q"], f["t"], _padded(f["bgr"]), f["xyz"], f["rgb"], mask=(xx + 2 * yy) % 5 != 0 if i == 2 else None)
        for _ in range(5):
            m.optimize([0])
        return m

    def finish(m):
        for f in frames[7:]:
            m.add_frame(f["q"], f["t"], _padded(f["bgr"]), f["xyz"], f["rgb"])
        for _ in range(5):
            m.optimize([0])
            m.optimize([1])

    a, b = start(), start()
    assert b.frames_get().pending_points > 0
    b.save_checkpoint(tmp_path / "f.ckpt")
    f = CF.read(tmp_path / "f.ckpt")
    assert f["frames"]["stats"]["pending_points"] == b.frames_get().pending_points
    assert [k["kind"] for k in f["keyframes"]["list"]] == [0] * 7
    assert sorted(k["frame"] for k in f["keyframes"]["list"]) == list(range(7))
    b.close()
    c = mapper.Mapper.from_checkpoint(tmp_path / "f.ckpt")
    finish(a)
    finish(c)
    da, dc = a.download(moments=True), c.download(moments=True)
    for k in da:
        _same(da[k], dc[k], "add_frame resume: %s" % k)
    sa, sc = a.stats(), c.stats()
    assert (sa.last_loss, sa.num_gaussians, sa.iterations, sa.last_inserted) == (sc.last_loss, sc.num_gaussians, sc.iterations, sc.last_inserted)
    fa, fc = a.frames_get(), c.frames_get()
    assert [getattr(fa, k) for k, _ in fa._fields_] == [getattr(fc, k) for k, _ in fc._fields_]
    assert np.array_equal(a.anchors(), c.anchors()) and a.sky_rows() == c.sky_rows()
    _same_all(_extras(a), _extras(c), "add_frame resume: masks and images")
    for i in range(2):
        assert a.evaluate(i) == c.evaluate(i)
    assert a.evaluate(0, train=False) == c.evaluate(0, train=False)
    a.close()
    c.close()


def test_without_the_deterministic_option_the_restored_state_is_exact(tmp_path):
    a = _twin(deterministic=False)
    _train(a, 10)
    b = _restore(a, tmp_path / "a.ckpt")
    _same_all(_state(a), _state(b), "restored state without the option")
    _train(b, 3)                                         # it trains on (not compared bitwise: float atomics)
    assert np.isfinite(b.stats().last_loss) and b.stats().iterations == 13
    a.close()
    b.close()


def test_float_keyframes_in_both_memory_classes(tmp_path):
    from gaussian_lic_b200 import mapper, synthetic as syn

    def make():
        pts, cols, dep = _lidar_scan(3000, 5, *_poses([0])[0])
        m = mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=3, capacity=3500, seed=SEED, views_per_rank=2)
        m.initialize_lidar(pts, cols, dep, F, 500, 1000)
        for i, (R, t) in enumerate(_poses()):
            img = torch.from_numpy(syn.make_gt_image(W, H, seed=40 + i))
            m.add_keyframe(R, t, img.pin_memory() if i % 2 else img.cuda(), train=i != 7)
        m.enable_exposure(0.001)
        m.set_deterministic(True)
        return m

    def steps(m, first, count):
        for i in range(first, first + count):
            m.optimize([(2 * i) % 7, (2 * i + 1) % 7])

    a, b = make(), make()
    steps(a, 0, 6)
    steps(b, 0, 6)
    b.save_checkpoint(tmp_path / "b.ckpt")
    kinds = [k["kind"] for k in CF.read(tmp_path / "b.ckpt")["keyframes"]["list"]]
    assert kinds == [2, 1, 2, 1, 2, 1, 2, 1]               # training 0..6 then the held-out one; kind 2 = device, 1 = host
    images = [b.keyframe_image(i) for i in range(7)] + [b.keyframe_image(0, train=False)]
    b.close()
    b._keep.clear()                                      # the caller's images are gone
    del b
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    c = mapper.Mapper.from_checkpoint(tmp_path / "b.ckpt")
    assert c._keep == []
    for i in range(7):
        _same(c.keyframe_image(i), images[i], "image %d" % i)
    _same(c.keyframe_image(0, train=False), images[7], "held-out image")
    steps(a, 6, 8)
    steps(c, 6, 8)
    da, dc = a.download(moments=True), c.download(moments=True)
    for k in da:
        _same(da[k], dc[k], "float keyframes: %s" % k)
    assert a.evaluate(0, train=False) == c.evaluate(0, train=False)
    a.close()
    c.close()


def _rank_mapper(rank, world):
    from gaussian_lic_b200 import mapper
    pts, cols, dep = _lidar_scan(3000, 5, *_poses([0])[0])
    m = mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=3, capacity=4096, seed=SEED, rank=rank, world=world, views_per_rank=1)
    m.initialize_lidar(pts, cols, dep, F, 500, 1000)
    _with_keyframes(m)
    m.enable_exposure(0.001)
    m.enable_pose_refinement(1e-3, 1e-3)
    m.enable_densification()
    m.set_density_schedule(**dict(SCHED, densify_from=1000))     # statistics only: a connected mapper's capacity is fixed
    m.set_deterministic(True)
    return m


def _rank_worker(rank, world, port, q, phase, paths):
    try:
        import torch
        import torch.distributed as dist
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
        torch.cuda.set_device(rank % torch.cuda.device_count())

        def exchange(mine):
            got = [None] * world
            dist.all_gather_object(got, mine)
            return got

        def snap(m):
            s = m.download(moments=True)
            s["accum"], s["denom"] = m.densify_stats()
            for k in range(len(VIEWS)):
                s["pose%d" % k] = np.concatenate([np.ravel(x) for x in m.pose(k)])
                s["E%d" % k] = m.exposure(k)
            s["loss"] = np.asarray([m.stats().last_loss], np.float32)
            return s

        out = {}
        if phase == 0:
            u = _rank_mapper(rank, world)                 # the uninterrupted run
            u.connect(exchange(u.export_handle()))
            _steps(u, 0, N_STEPS + M_STEPS)
            out["uninterrupted"] = snap(u)
            dist.barrier()
            u.close()
            s = _rank_mapper(rank, world)                 # the run that saves after N steps
            s.connect(exchange(s.export_handle()))
            _steps(s, 0, N_STEPS)
            s.save_checkpoint(paths[rank])
            dist.barrier()
            s.close()
        else:
            from gaussian_lic_b200 import mapper
            r = mapper.Mapper.from_checkpoint(paths[rank])
            r.connect(exchange(r.export_handle()))
            _steps(r, N_STEPS, M_STEPS)
            out["resumed"] = snap(r)
            dist.barrier()
            r.close()
        dist.destroy_process_group()
        q.put((rank, "ok", out))
    except Exception as e:          # noqa: BLE001 - reported to the parent
        import traceback
        q.put((rank, "%r\n%s" % (e, traceback.format_exc()), None))


def _spawn(phase, paths):
    import socket
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    q = ctx.Queue()
    procs = [ctx.Process(target=_rank_worker, args=(r, 2, port, q, phase, paths)) for r in range(2)]
    for p_ in procs:
        p_.start()
    res = sorted([q.get(timeout=400) for _ in procs], key=lambda r: r[0])
    for p_ in procs:
        p_.join(timeout=30)
    assert all(r[1] == "ok" for r in res), [r[1] for r in res]
    return [r[2] for r in res]


@pytest.mark.timeout(900)
def test_two_ranks_save_and_resume_in_fresh_processes(tmp_path):
    """each rank of a connected pair saves its own file; fresh processes restore, export, connect and continue: the replicas are
    bit-identical to each other and to an uninterrupted two-rank run"""
    paths = [str(tmp_path / ("rank%d.ckpt" % r)) for r in range(2)]
    first = _spawn(0, paths)
    second = _spawn(1, paths)
    for r in range(2):
        assert CF.read(paths[r])["config"]["rank"] == r
    def bits(a):
        return np.ascontiguousarray(a).view(np.uint8)

    for name in first[0]["uninterrupted"]:
        for r in range(2):
            # the loss is of the rank's own last view; everything else is replicated
            want = first[r if name == "loss" else 0]["uninterrupted"][name]
            assert np.array_equal(bits(first[r]["uninterrupted"][name]), bits(want)), "uninterrupted replicas differ in %s" % name
            assert np.array_equal(bits(second[r]["resumed"][name]), bits(want)), "rank %d resumed differs in %s" % (r, name)


def _small(tmp_path):
    """a small trained mapper with a masked held-out keyframe, and its checkpoint"""
    from gaussian_lic_b200 import synthetic as syn
    m = _twin()
    R, t = syn.orbit_pose(3.5, radius=2.0)
    m.add_keyframe(R, t, syn.make_gt_image(W, H, seed=91), train=False)
    m.set_mask(False, 0, np.mgrid[0:H, 0:W][1] > 20)
    _steps(m, 0, 6)
    path = tmp_path / "good.ckpt"
    m.save_checkpoint(path)
    return m, path


def test_refusals_leave_the_target_fresh(tmp_path):
    from gaussian_lic_b200 import capi, mapper
    src, path = _small(tmp_path)
    good = path.read_bytes()
    cfg = mapper.checkpoint_config(path)
    target = mapper.Mapper.__new__(mapper.Mapper)
    target._create(cfg)

    def refused(data, what, m=target):
        p = tmp_path / "bad.ckpt"
        p.write_bytes(data)
        rc = capi.lib.glic_mapper_load_checkpoint(m._h, str(p).encode())
        assert rc == -1, (what, rc)
        if m is target:
            assert target.stats().num_gaussians == 0 and target.stats().iterations == 0, what

    # targets that are not fresh
    pts, cols, dep = _lidar_scan(500, 5, *_poses([0])[0])
    for how in ("initialized", "keyframe", "frames", "exported"):
        m = mapper.Mapper.__new__(mapper.Mapper)
        m._create(mapper.checkpoint_config(path))
        if how == "initialized":
            m.initialize_lidar(pts, cols, dep, F, 0, 0)
        elif how == "keyframe":
            _with_keyframes(m, 1)
        elif how == "frames":
            m.enable_frames(5, 0, 0)
        else:
            m.export_handle()
        before = m.stats()
        refused(good, how, m)
        assert (m.stats().num_gaussians, m.stats().capacity) == (before.num_gaussians, before.capacity), how
        m.close()
    # a configuration that differs in one field
    for field, value in (("fx", cfg.fx * 1.0001), ("seed", cfg.seed + 1), ("max_iters", cfg.max_iters + 1), ("views_per_rank", 1),
                         ("lambda_dssim", 0.3)):
        c2 = mapper.checkpoint_config(path)
        setattr(c2, field, value)
        m = mapper.Mapper.__new__(mapper.Mapper)
        m._create(c2)
        refused(good, "config " + field, m)
        m.close()
    # malformed files, into the one fresh target
    _, secs = CF.sections(good)
    end = len(good) - 16
    for tag, off, n in secs:
        for cut in (off - 16, off - 8, off, off + n // 2, off + n - 1):
            refused(good[:cut], "cut in %s at %d" % (tag, cut))
        blob = bytearray(good)
        for delta in (-4, 4):
            blob[off - 8:off] = np.uint64(n + delta).tobytes()
            refused(bytes(blob), "%s length %+d" % (tag, delta))
        refused(good[:end] + good[off - 16:off + n] + good[end:], "duplicated " + tag)
    refused(good[:end], "no end marker")
    refused(good[:-1], "end marker cut")
    refused(good + b"\0\0\0\0", "trailing bytes")
    refused(good[:8] + np.uint32(2).tobytes() + good[12:], "version 2")
    refused(b"GLICCKPU" + good[8:], "magic")
    refused(good[:end] + CF.section("XTRA", b"1234") + good[end:], "unknown section")
    # the same target still loads the good file
    target.load_checkpoint(path)
    _same_all(_state(src), _state(target), "after the refusals")
    src.close()
    target.close()


def test_failed_allocations_leave_the_target_fresh(tmp_path):
    from gaussian_lic_b200 import capi, mapper
    src, path = _small(tmp_path)
    target = mapper.Mapper.__new__(mapper.Mapper)
    target._create(mapper.checkpoint_config(path))
    live = capi.lib.glic_debug_mapper_allocations()
    failed = 0
    for k in range(1, 200):
        capi.check(capi.lib.glic_debug_fail_allocation(k), "debug_fail_allocation")
        rc = capi.lib.glic_mapper_load_checkpoint(target._h, str(path).encode())
        capi.check(capi.lib.glic_debug_fail_allocation(0), "debug_fail_allocation")
        if rc == 0:
            break
        assert rc == -3, (k, rc)
        failed += 1
        st = target.stats()
        assert st.num_gaussians == 0 and st.iterations == 0, k
        assert capi.lib.glic_debug_mapper_allocations() == live, k       # nothing of the failed load is kept
    assert failed > 20                                    # keyframes, masks, then every buffer of the growth
    _same_all(_state(src), _state(target), "after the failed loads")
    # a failed staging allocation of the save leaves an existing file as it was, and no temporary file
    out = tmp_path / "existing.ckpt"
    out.write_bytes(b"previous contents")
    capi.check(capi.lib.glic_debug_fail_allocation(1), "debug_fail_allocation")
    rc = capi.lib.glic_mapper_save_checkpoint(src._h, str(out).encode())
    capi.check(capi.lib.glic_debug_fail_allocation(0), "debug_fail_allocation")
    assert rc == -3
    assert out.read_bytes() == b"previous contents" and not (tmp_path / "existing.ckpt.tmp").exists()
    # a save into a directory that does not exist fails before anything is written
    with pytest.raises(capi.GlicError):
        src.save_checkpoint(tmp_path / "absent" / "x.ckpt")
    src.close()
    target.close()


def test_empty_mapper_round_trips_and_then_trains(tmp_path):
    from gaussian_lic_b200 import mapper

    def grow(m):
        pts, cols, dep = _lidar_scan(3000, 5, *_poses([0])[0])
        m.initialize_lidar(pts, cols, dep, F, 500, 1000)
        _with_keyframes(m)
        _steps(m, 0, 6)

    a = mapper.Mapper(W, H, F, F, W / 2.0, H / 2.0, sh_degree=3, capacity=3500, seed=SEED, views_per_rank=2)
    a.set_deterministic(True)
    b = _restore(a, tmp_path / "empty.ckpt")
    assert b.stats().num_gaussians == 0 and b.stats().capacity == a.stats().capacity
    assert a.sample_views() == b.sample_views() == []
    grow(a)
    grow(b)
    da, db = a.download(moments=True), b.download(moments=True)
    for k in da:
        _same(da[k], db[k], "empty round trip: %s" % k)
    assert a.stats().last_loss == b.stats().last_loss
    a.close()
    b.close()
