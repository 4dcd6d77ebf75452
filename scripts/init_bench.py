"""Cost of initialize() in the native mapper (glic_mapper_initialize_lidar): 100 k sky points plus the first LiDAR scan, at
20 k and 200 k points, on a 640x512 mapper.

Each timed call is the whole C ABI call as a host sees it: H2D of the scan (pinned-free numpy arrays), the arena reset, the
sky kernels (positions, simple-knn over the sky, the remaining fields), the LiDAR kernel and the final synchronise.  A host
clock around a call that ends in a device synchronise; every size is warmed up first.

    python scripts/init_bench.py [--reps 10] [--sky 100000]

Prints one JSON line: the median and min ms per call at each LiDAR size, every repetition, and the card name and power
limit.  Needs a GPU; writes nothing."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power, clock = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--sky", type=int, default=100_000, help="skybox_points_num (config/fastlivo.yaml:27)")
    ap.add_argument("--radius", type=int, default=1000, help="skybox_radius (config/fastlivo.yaml:28)")
    args = ap.parse_args()
    import numpy as np
    import torch
    from gaussian_lic_b200 import mapper as gmapper

    assert torch.cuda.is_available(), "init_bench needs a GPU"
    W, H, fx, fy = 640, 512, 431.795259219, 431.550090267              # config/fastlivo.yaml:1-4
    out = {"sky_points": args.sky, "width": W, "height": H, "card": card()}
    for n in (20_000, 200_000):
        rng = np.random.default_rng(n)
        z = rng.uniform(0.5, 60.0, n)
        pts = np.stack([z * rng.uniform(-0.7, 0.7, n), z * rng.uniform(-0.5, 0.5, n), z], 1).astype(np.float32)
        cols = rng.integers(0, 256, (n, 3)) / 255.0
        dep = z.astype(np.float32)
        m = gmapper.Mapper(W, H, fx, fy, W / 2.0, H / 2.0, sh_degree=3, seed=1)
        m.initialize_lidar(pts, cols, dep, (fx + fy) / 2, args.sky, args.radius)          # warm-up (modules, arena size)
        ms = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            m.initialize_lidar(pts, cols, dep, (fx + fy) / 2, args.sky, args.radius)      # ends in a stream synchronise
            ms.append((time.perf_counter() - t0) * 1e3)
        assert m.stats().num_gaussians == args.sky + n
        m.close()
        out["lidar_%d" % n] = {"median_ms": float(np.median(ms)), "min_ms": float(np.min(ms)), "ms": [round(x, 4) for x in ms]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
