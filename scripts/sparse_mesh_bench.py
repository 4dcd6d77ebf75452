"""Cost of the sparse block TSDF on the GPU (include/glic_b200.h "Sparse meshing"), against the dense grid where one fits.

  - mesh_bench.py's scene (one 1920x1080 view of a sphere in front of a wall, 512^3 lattice points of 1 cm; only the pixels whose
    truncation band stays in the dense box have a depth): dense and sparse,
    glic_block_set_insert per view, integration per view (CUDA events around `--calls` back-to-back calls per window, median over
    the windows), count + extract (host clock around the synchronising pair), the device bytes of each grid, and whether the
    two meshes are identical;
  - an outdoor-extent map no dense grid holds: opaque flat Gaussians on a ground plane and two facades along a 300 m straight
    street, 100 keyframes along it, 5 cm voxels: glic_mapper_extract_mesh_sparse (host clock around the synchronising call),
    its blocks and the bytes of its grid.

    python scripts/sparse_mesh_bench.py [--windows 7] [--calls 10]

Prints one JSON line with the medians, every window, and the card name and power limit.  Needs a GPU; writes nothing."""
import argparse
import ctypes as C
import json
import math
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _timed(fn, windows, calls, torch):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    out = []
    for _ in range(windows):
        torch.cuda.synchronize()
        ev[0].record()
        for _ in range(calls):
            fn()
        ev[1].record()
        torch.cuda.synchronize()
        out.append(ev[0].elapsed_time(ev[1]) / calls)
    return statistics.median(out), out


def _host_timed(fn, windows, torch):
    out = []
    for _ in range(windows):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(out), out, r


def street_map(length=300.0, width=16.0, height=6.0, step=0.12, sigma=0.1):
    """opaque flat Gaussians on the ground y = 1.5 (y points down) and on the facades z = +-width / 2, x in [-5, length + 20]"""
    import numpy as np
    xs = np.arange(-5.0, length + 20.0, step)
    zs = np.arange(-width / 2, width / 2 + 1e-9, step)
    ys = np.arange(1.5 - height, 1.5 + 1e-9, step)
    gx, gz = np.meshgrid(xs, zs)
    ground = np.stack([gx.ravel(), np.full(gx.size, 1.5), gz.ravel()], 1)
    fx, fy = np.meshgrid(xs, ys)
    walls = [np.stack([fx.ravel(), fy.ravel(), np.full(fx.size, z)], 1) for z in (-width / 2, width / 2)]
    means = np.concatenate([ground] + walls).astype(np.float32)
    scales = np.concatenate([np.tile([sigma, 0.002, sigma], (ground.shape[0], 1))] +
                            [np.tile([sigma, sigma, 0.002], (w.shape[0], 1)) for w in walls])
    P = means.shape[0]
    rng = np.random.default_rng(0)
    return dict(means=means, log_scales=np.log(scales).astype(np.float32), rots=np.tile([1.0, 0.0, 0.0, 0.0], (P, 1)).astype(np.float32),
                opacity_logits=np.full(P, 6.0, np.float32), dc=rng.random((P, 3)).astype(np.float32), sh=np.zeros((P, 0, 3), np.float32),
                degree=0)


def street_pose(k, n, length):
    """keyframe k of n along the street: at x = k length / (n - 1), eye height, looking ahead and swaying left and right"""
    import numpy as np
    pos = np.array([k * length / (n - 1), 0.0, 0.0])
    fwd = np.array([1.0, 0.15, 0.35 * math.sin(0.7 * k)])
    fwd /= np.linalg.norm(fwd)
    right = np.cross(fwd, np.array([0.0, -1.0, 0.0]))
    right /= np.linalg.norm(right)
    down = np.cross(fwd, right)
    return np.stack([right, down, fwd], axis=1), pos


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--keyframes", type=int, default=100)
    ap.add_argument("--length", type=float, default=300.0)
    args = ap.parse_args()
    import numpy as np
    import torch
    import mesh_oracle as mo
    from gaussian_lic_b200 import capi, mapper as gmapper, ops
    from pose_bench import card
    assert torch.cuda.is_available(), "sparse_mesh_bench.py needs a GPU"
    dev = torch.device("cuda:0")
    out = {"card": card()}

    # ---- mesh_bench.py's 512^3 scene, dense and sparse ----
    W, H, f, n = 1920, 1080, 1000.0, 512
    s = 5.12 / n
    origin = (-2.56, -2.0, 1.0)
    R, t = np.eye(3), np.zeros(3)
    depth = mo.sphere_depth(R, t, W, H, f, f, W / 2.0, H / 2.0, (0.0, 0.4, 3.5), 1.2)
    depth = np.where(depth > 0, depth, np.float32(5.5)).astype(np.float32)
    # only the pixels whose truncation band stays inside the dense box, so that it holds every block and the meshes compare
    u, v = np.meshgrid(np.arange(W) - W / 2.0, np.arange(H) - H / 2.0)
    depth[(np.abs(u) > 430) | (v < -340)] = 0.0
    depth_d = torch.from_numpy(depth).to(dev)
    rgb_d = torch.rand(3, H, W, device=dev)
    view_d = torch.from_numpy(mo.view_of(R, t)).to(dev)
    trunc = 3 * s
    cam = (W, H, f, f, W / 2.0, H / 2.0)

    st, st_data = ops.block_set(1 << 22, dev)
    blocks, clipped, over = ops.block_set_insert(st, origin, s, view_d, *cam, depth_d, trunc=trunc)
    assert not over
    cnt = (C.c_int64 * 3)()
    o3 = (C.c_float * 3)(*origin)

    def insert():                                                     # the set already holds the view: the timed calls add nothing
        capi.lib.glic_block_set_insert(C.byref(st), o3, s, capi.ptr(view_d), W, H, f, f, W / 2.0, H / 2.0,
                                       capi.ptr(depth_d), None, 0, trunc, 0.0, cnt, None)
    ins_ms, ins_w = _timed(insert, args.windows, args.calls, torch)
    sgrid, sdata = ops.sparse_tsdf(origin, s, st, blocks, dev)
    ops.sparse_tsdf_integrate(sgrid, view_d, *cam, depth_d, rgb_d, trunc=trunc)
    s_int_ms, s_int_w = _timed(lambda: ops.sparse_tsdf_integrate(sgrid, view_d, *cam, depth_d, rgb_d, trunc=trunc), args.windows, args.calls, torch)
    s_ext_ms, s_ext_w, smesh = _host_timed(lambda: ops.sparse_mesh_extract(sgrid, dev), args.windows, torch)
    sparse_bytes = capi.lib.glic_block_set_bytes(st.capacity) + capi.lib.glic_sparse_tsdf_bytes(blocks)
    # the same number of integrations into both grids, so the meshes compare
    calls_done = 1 + args.windows * args.calls
    dgrid, ddata = ops.tsdf_grid(origin, s, (n, n, n), dev)
    for _ in range(calls_done):
        ops.tsdf_integrate(dgrid, view_d, *cam, depth_d, rgb_d, trunc=trunc)
    d_int_ms, d_int_w = _timed(lambda: ops.tsdf_integrate(dgrid, view_d, *cam, depth_d, rgb_d, trunc=trunc), args.windows, args.calls, torch)
    for _ in range(args.windows * args.calls):
        ops.sparse_tsdf_integrate(sgrid, view_d, *cam, depth_d, rgb_d, trunc=trunc)
    d_ext_ms, d_ext_w, dmesh = _host_timed(lambda: ops.mesh_extract(dgrid, dev), args.windows, torch)
    smesh = ops.sparse_mesh_extract(sgrid, dev)
    same = all(torch.equal(a.view(torch.uint8), b.view(torch.uint8)) for a, b in zip(smesh[:3], dmesh))
    out["scene_512"] = dict(frame=[W, H], voxel=s, blocks=blocks, clipped_pixels=clipped,
                            dense=dict(bytes=capi.lib.glic_tsdf_bytes((C.c_int * 3)(n, n, n)), integrate_ms=d_int_ms,
                                       integrate_windows=d_int_w, count_extract_ms=d_ext_ms, count_extract_windows=d_ext_w),
                            sparse=dict(bytes=sparse_bytes, insert_ms=ins_ms, insert_windows=ins_w, integrate_ms=s_int_ms,
                                        integrate_windows=s_int_w, count_extract_ms=s_ext_ms, count_extract_windows=s_ext_w),
                            vertices=int(smesh[0].shape[0]), faces=int(smesh[2].shape[0]), meshes_identical=bool(same))
    del sgrid, sdata, dgrid, ddata, st, st_data, smesh, dmesh
    torch.cuda.empty_cache()

    # ---- an outdoor-extent street ----
    Wm, Hm, fm = 1280, 720, 640.0
    raw = street_map(args.length)
    m = gmapper.Mapper(Wm, Hm, fm, fm, Wm / 2.0, Hm / 2.0, sh_degree=0, capacity=raw["means"].shape[0])
    m.initialize(raw)
    img = np.zeros((3, Hm, Wm), np.float32)
    for k in range(args.keyframes):
        m.add_keyframe(*street_pose(k, args.keyframes, args.length), img)
    p = dict(origin=(-10.0, -6.0, -12.0), voxel_size=0.05, trunc=0.15, max_depth=40.0)
    c = m.extract_mesh_sparse(**p)
    calls = []
    for _ in range(3):
        t0 = time.perf_counter()
        c = m.extract_mesh_sparse(**p)
        calls.append((time.perf_counter() - t0) * 1e3)
    ext = [hi - lo + 1 for lo, hi in zip(c["lattice_lo"], c["lattice_hi"])]
    out["street"] = dict(gaussians=int(raw["means"].shape[0]), length_m=args.length, keyframes=args.keyframes, frame=[Wm, Hm],
                         voxel=p["voxel_size"], counts=c, lattice_extent=ext, dense_points_needed=int(np.prod(ext, dtype=np.int64)),
                         grid_bytes=capi.lib.glic_sparse_tsdf_bytes(c["blocks"]), ms_median=statistics.median(calls), ms_calls=calls,
                         ms_per_keyframe=statistics.median(calls) / args.keyframes)
    m.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
