"""Cost of the contribution scores (glic_contribution, glic_mapper_contribution, glic_mapper_prune_unseen) at cfg2, and what
pruning the unseen rows does to the iteration.

  1. blend: the scoring form of the blend against the no_color and colour training blends, on bench.py's scene and the eight rig
     views, each timed by the library's GLIC_STAGE_RENDER_FWD events; the three forms alternate window by window.
  2. mapper: one glic_mapper_contribution over the eight rig keyframes, by the host clock (the call synchronises).
  3. prune: glic_mapper_prune_unseen at 500 k and 2 M rows with 10 % and 50 % of the rows hidden behind an opaque layer (two walls
     of large flat opaque Gaussians beyond the scene), by the host clock; the rows removed are reported with the rows
     built hidden and the rows a dry run finds unseen in the same scene without walls or hidden rows.
  4. iteration: cfg2 iterations (glic_mapper_optimize over the rig views) of a mapper pruned of its hidden rows and of its unpruned
     twin from the same initialisation, alternating window by window, by the host clock.
The card's name and power limit are read in the same call.

    python scripts/contribution_bench.py [--windows 5] [--iters 20]

Prints one JSON line.  Needs a GPU; writes nothing."""
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


def median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def hidden_map(P, frac, seed=1):
    """bench.py's cfg2 scene with frac * P of its rows moved behind two opaque walls at z = 22 and 22.5 (the scene ends at 20)"""
    import numpy as np
    from gaussian_lic_b200 import synthetic as syn
    _, W, H, fx, fy, _, _, deg, zmax = syn.CONFIGS["cfg2"]
    g = syn.make_gaussians(P, W, H, fx, fy, sh_degree=deg, zmax=zmax, seed=seed)
    g = {k: (np.array(v) if isinstance(v, np.ndarray) else v) for k, v in g.items()}
    rng = np.random.default_rng(seed)
    grid = np.arange(-16.0, 16.01, 0.5)
    gx, gy = np.meshgrid(grid, grid)
    walls = np.concatenate([np.stack([gx.ravel(), gy.ravel(), z + rng.uniform(0.0, 0.05, gx.size)], 1) for z in (22.0, 22.5)]).astype(np.float32)
    if frac == 0.0:
        return g
    nw, nh = walls.shape[0], int(frac * P) - walls.shape[0]
    rows = rng.permutation(P)
    w_rows, h_rows = rows[:nw], rows[nw:nw + nh]
    g["means"][w_rows] = walls
    g["log_scales"][w_rows] = np.log([0.5, 0.5, 0.02]).astype(np.float32)
    g["rots"][w_rows] = np.array([1.0, 0.0, 0.0, 0.0], np.float32)
    g["opacity_logits"].reshape(P)[w_rows] = 7.0
    g["means"][h_rows] = np.stack([rng.uniform(-8, 8, nh), rng.uniform(-5, 5, nh), rng.uniform(24, 30, nh)], 1)
    return g


def mapper_of(g, n_views=8):
    from gaussian_lic_b200 import mapper as gmapper, synthetic as syn
    _, W, H, fx, fy, cx, cy, deg, _ = syn.CONFIGS["cfg2"]
    m = gmapper.Mapper(W, H, fx, fy, cx, cy, sh_degree=deg, capacity=int(g["means"].shape[0]), max_iters=8)
    m.initialize(g)
    for v in range(n_views):
        m.add_keyframe(*syn.orbit_pose(v, radius=0.25), syn.make_gt_image(W, H, seed=v))
    return m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=5, help="timed windows per arm (alternating)")
    ap.add_argument("--iters", type=int, default=20, help="iterations per window of part 4")
    args = ap.parse_args()
    import numpy as np
    import torch
    from gaussian_lic_b200 import capi, mapper as gmapper, ops, synthetic as syn
    assert torch.cuda.is_available(), "contribution_bench.py needs a GPU"
    out = {"card": card()}
    P, W, H, fx, fy, cx, cy, deg, _ = syn.CONFIGS["cfg2"]
    g, _ = syn.make_scene("cfg2")
    r = ops.CRasterizer(W, H)
    gd = ops.scene_to_device(g)
    views = [r.make_view(gmapper.camera_block(W, H, fx, fy, cx, cy, *syn.orbit_pose(v, radius=0.25))) for v in range(8)]
    mw = torch.zeros(P, dtype=torch.float32, device="cuda")
    hits = torch.zeros(P, dtype=torch.int64, device="cuda")
    for v in views:                                        # warm up and size the workspaces for every view
        r.forward(gd, v)
        r.forward(gd, v, no_color=True)
        r.contribution(gd, v, mw, hits)
    arms = {"score": lambda v: r.contribution(gd, v, mw, hits), "no_color": lambda v: r.forward(gd, v, no_color=True),
            "colour": lambda v: r.forward(gd, v)}
    res = {k: [] for k in arms}
    for _ in range(args.windows):
        for k, fn in arms.items():
            capi.profile_enable(True)
            for v in views:
                fn(v)
            torch.cuda.synchronize()
            ms, n = capi.profile_read()["render_fwd"]
            capi.profile_enable(False)
            res[k].append(ms / n)
    out["blend_ms_per_view"] = {k: round(median(x), 4) for k, x in res.items()}
    out["blend_spread_ms"] = {k: round(max(x) - min(x), 4) for k, x in res.items()}
    out["taken_pairs_per_view"] = int(hits.sum().item()) // (len(views) * (1 + args.windows))      # warm-up + score windows
    del r, gd, mw, hits
    torch.cuda.empty_cache()
    # 2. the mapper's eight-view call
    m = mapper_of(g)
    m.contribution()
    t = []
    for _ in range(args.windows):
        t0 = time.perf_counter()
        m.contribution()
        t.append(1e3 * (time.perf_counter() - t0))
    out["mapper_contribution_ms_8_views"] = round(median(t), 3)
    m.close()
    # 3. prune_unseen, and 4. iterations of a pruned mapper and its unpruned twin
    out["prune"] = {}
    for Pn in (500_000, 2_000_000):
        for frac in (0.1, 0.5):
            gh = hidden_map(Pn, frac)
            base = mapper_of(hidden_map(Pn, 0.0))            # the same scene without walls or hidden rows
            natural = base.prune_unseen(dry_run=True)       # the rows no view sees anyway
            base.close()
            m = mapper_of(gh)
            m.prune_unseen(dry_run=True)                    # sizes the score buffers and the binning workspace
            t0 = time.perf_counter()
            n = m.prune_unseen()
            host_ms = 1e3 * (time.perf_counter() - t0)
            out["prune"]["%dk_%d%%" % (Pn // 1000, int(100 * frac))] = {
                "ms": round(host_ms, 3), "removed": n, "built_hidden": int(frac * Pn) - 2 * 65 * 65, "unseen_without_walls": natural}
            if Pn == 500_000 and frac == 0.5:
                twin = mapper_of(gh)
                its = {"pruned": [], "unpruned": []}
                batch = list(range(8)) * ((args.iters + 7) // 8)
                for mm in (m, twin):
                    mm.optimize(batch[:8])
                    mm.synchronize()
                for _ in range(args.windows):
                    for k, mm in (("pruned", m), ("unpruned", twin)):
                        t0 = time.perf_counter()
                        mm.optimize(batch[:args.iters])
                        mm.synchronize()
                        its[k].append(1e3 * (time.perf_counter() - t0) / args.iters)
                out["iteration_ms_500k_50%_hidden"] = {k: round(median(x), 4) for k, x in its.items()}
                out["iteration_spread_ms"] = {k: round(max(x) - min(x), 4) for k, x in its.items()}
                twin.close()
            m.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
