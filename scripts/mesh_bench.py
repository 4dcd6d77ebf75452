"""Cost of meshing on the GPU (include/glic_b200.h "Meshing").

  - glic_tsdf_integrate of one 1920x1080 view into a 512^3 grid (2.7 GB): CUDA events around `--calls` back-to-back calls per
    window, median over the windows;
  - glic_mesh_count + glic_mesh_extract of that grid: host clock around the pair (the count synchronises, the extract is
    followed by a synchronise);
  - glic_mapper_extract_mesh over 100 training keyframes of a cfg2-sized map (500 k Gaussians, SH degree 3, 1920x1080): host
    clock around the synchronising call.

Each time comes with the bytes a traffic model says it moves and that rate's share of the H100 SXM data-sheet HBM3 bandwidth
(3.35 TB/s).  Integration: 20 B read + 20 B written per updated lattice point (tsdf, weight, colour) and 4 B per point that
skips (its depth sample), counted from the weights the call changed.  Extraction: its three grid passes read the tsdf and
weight of every lattice point (24 B per point), plus the mesh it writes (15 B per vertex, 12 B per face).

    python scripts/mesh_bench.py [--windows 7] [--calls 10] [--dim 512]

Prints one JSON line with the medians, every window, and the card name and power limit.  Needs a GPU; writes nothing."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_BYTES_PER_S = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--calls", type=int, default=10, help="integrate calls per timed window")
    ap.add_argument("--dim", type=int, default=512)
    ap.add_argument("--keyframes", type=int, default=100)
    args = ap.parse_args()
    import numpy as np
    import torch
    import mesh_oracle as mo
    from gaussian_lic_b200 import mapper as gmapper, ops, synthetic as syn
    from pose_bench import card
    assert torch.cuda.is_available(), "mesh_bench.py needs a GPU"
    dev = torch.device("cuda:0")
    out = {"card": card()}

    # ---- integration at 1920x1080 into dim^3 ----
    W, H, f = 1920, 1080, 1000.0
    n = args.dim
    s = 5.12 / n
    dims = (n, n, n)
    N = n ** 3
    R, t = np.eye(3), np.zeros(3)
    depth = mo.sphere_depth(R, t, W, H, f, f, W / 2.0, H / 2.0, (0.0, 0.4, 3.5), 1.2)
    depth = np.where(depth > 0, depth, np.float32(5.5)).astype(np.float32)        # the sphere in front of a wall
    depth_d = torch.from_numpy(depth).to(dev)
    rgb_d = torch.rand(3, H, W, device=dev)
    view_d = torch.from_numpy(mo.view_of(R, t)).to(dev)
    grid, data = ops.tsdf_grid((-2.56, -2.0, 1.0), s, dims, dev)

    def integrate():
        ops.tsdf_integrate(grid, view_d, W, H, f, f, W / 2.0, H / 2.0, depth_d, rgb_d, trunc=3 * s)

    integrate()
    torch.cuda.synchronize()
    updated = int((data[N:2 * N] > 0).sum())
    int_bytes = 40 * updated + 4 * (N - updated)
    for _ in range(3):
        integrate()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    int_ms = []
    for _ in range(args.windows):
        torch.cuda.synchronize()
        ev[0].record()
        for _ in range(args.calls):
            integrate()
        ev[1].record()
        torch.cuda.synchronize()
        int_ms.append(ev[0].elapsed_time(ev[1]) / args.calls)
    med = statistics.median(int_ms)
    out["integrate"] = dict(frame=[W, H], grid=list(dims), grid_bytes=20 * N, lattice_points=N, updated_points=updated,
                            model_bytes=int_bytes, ms_median=med, ms_windows=int_ms,
                            tb_per_s=int_bytes / (med * 1e-3) / 1e12, hbm_share=int_bytes / (med * 1e-3) / HBM_BYTES_PER_S)

    # ---- count + extract of that grid ----
    ops.mesh_extract(grid, dev)
    torch.cuda.synchronize()
    ext_ms = []
    for _ in range(args.windows):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        xyz, col, faces = ops.mesh_extract(grid, dev)
        torch.cuda.synchronize()
        ext_ms.append((time.perf_counter() - t0) * 1e3)
    V, F = int(xyz.shape[0]), int(faces.shape[0])
    ext_bytes = 24 * N + 15 * V + 12 * F
    med = statistics.median(ext_ms)
    out["count_extract"] = dict(vertices=V, faces=F, model_bytes=ext_bytes, ms_median=med, ms_windows=ext_ms,
                                tb_per_s=ext_bytes / (med * 1e-3) / 1e12, hbm_share=ext_bytes / (med * 1e-3) / HBM_BYTES_PER_S)
    del grid, data, xyz, col, faces
    torch.cuda.empty_cache()

    # ---- extract_mesh over the keyframes of a cfg2-sized map ----
    P, W, H, fx, fy, cx, cy, deg, _ = syn.CONFIGS["cfg2"]
    g, _ = syn.make_scene("cfg2")
    m = gmapper.Mapper(W, H, fx, fy, cx, cy, sh_degree=deg, capacity=P)
    m.initialize(g)
    img = np.zeros((3, H, W), np.float32)
    for k in range(args.keyframes):
        m.add_keyframe(*syn.orbit_pose(k, n_views=args.keyframes, radius=0.5), img)
    p = dict(origin=(-12.8, -7.2, 0.5), voxel_size=0.05, dims=(512, 288, 400), trunc=0.15)
    Nm = int(np.prod(p["dims"]))
    got = m.extract_mesh(**p)
    map_ms = []
    for _ in range(3):
        t0 = time.perf_counter()
        got = m.extract_mesh(**p)
        map_ms.append((time.perf_counter() - t0) * 1e3)
    med = statistics.median(map_ms)
    out["mapper_extract_mesh"] = dict(config="cfg2", keyframes=args.keyframes, grid=list(p["dims"]), grid_bytes=20 * Nm,
                                      vertices=got["n_vertices"], faces=got["n_faces"], observed_voxels=got["observed_voxels"],
                                      ms_median=med, ms_calls=map_ms, ms_per_keyframe=med / args.keyframes,
                                      overflow_regrows=int(m.stats().overflow_regrows))
    m.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
