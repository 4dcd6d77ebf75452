"""Cost of glic_mapper_prune, and what it buys the native mapping iteration.

1. The call: a mapper of P rows at SH degree 3 (cfg2's P = 500 000 and 2 000 000), a fraction of its rows below the 1/255 cut
   (logit -10), capacity = P.  Each timed call starts from a freshly initialised arena (untimed) and is timed by a host clock
   around the synchronising call: selection, spare-arena allocation and zeroing, three gathers, frees.  The dry run (selection
   only) is timed the same way.  One more call runs under torch.profiler (CUDA activities): the device time of each kernel,
   memset and copy it issues, and the bytes the three gathers move over their kernel time.
2. The iteration: two cfg2 mappers from one initialisation with the same fraction of dead rows; one is pruned at 1/255, the
   other is not.  Their timed windows alternate in this one call (bench.py's mapping_iter_native step: one view per iteration
   from eight pinned-host keyframes, optimiser on); each window is device time on the mapper's stream.

    python scripts/prune_bench.py [--reps 5] [--steps 56] [--windows 9]

Prints one JSON line with every figure, and the card name and power limit.  Needs a GPU; writes nothing."""
import argparse
import json
import os
import re
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DEAD_LOGIT = -10.0


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power, clock = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def with_dead_rows(g, frac, seed=7):
    import numpy as np
    rng = np.random.default_rng(seed)
    P = g["means"].shape[0]
    lg = np.asarray(g["opacity_logits"], np.float32).copy()
    lg[rng.random(P) < frac] = DEAD_LOGIT
    return dict(g, opacity_logits=lg)


def time_call(P, frac, reps):
    """median / min host ms of prune(1/255) and of its dry run on a P-row degree-3 map"""
    import numpy as np
    from gaussian_lic_b200 import mapper as gmapper, synthetic as syn
    _, W, H, fx, fy, cx, cy, deg, zmax = syn.CONFIGS["cfg2"]
    g = with_dead_rows(syn.make_gaussians(P, W, H, fx, fy, sh_degree=deg, zmax=zmax, seed=42), frac)
    m = gmapper.Mapper(W, H, fx, fy, cx, cy, sh_degree=deg, capacity=P)
    M = m.M
    cap = m.stats().capacity
    dry, real, removed = [], [], None
    for r in range(reps + 1):                                              # the first call of each kind warms up
        m.initialize(g)
        m.synchronize()
        t0 = time.perf_counter()
        n_dry = m.prune(dry_run=True)
        t1 = time.perf_counter()
        n = m.prune()
        t2 = time.perf_counter()
        assert n == n_dry and m.stats().num_gaussians == P - n
        removed = n
        if r:
            dry.append((t1 - t0) * 1e3)
            real.append((t2 - t1) * 1e3)
    m.initialize(g)
    device = device_times(m)
    m.close()
    row = 4 * (14 + 3 * M)
    gathered = 3 * ((P - removed) * row + P * row)                       # three gathers: read the kept rows, write rows [0, P)
    med = float(np.median(real))
    gather_us = sum(v for k, v in device.items() if "prune_gather_kernel" in k)
    return {"P": P, "capacity": cap, "dead_fraction": frac, "removed": removed, "ms_prune_median": round(med, 4),
            "ms_prune_min": round(float(np.min(real)), 4), "ms_dry_run_median": round(float(np.median(dry)), 4),
            "ms_prune_all": [round(x, 4) for x in real], "device_us": device,
            "device_us_total": round(sum(device.values()), 1), "gather_bytes": gathered,
            "gather_TBps": round(gathered / (gather_us * 1e-6) / 1e12, 2) if gather_us else None}


def device_times(m):
    """device time (us) of every kernel, memset and copy of one prune(1/255) call, from torch.profiler's trace"""
    import tempfile
    import torch
    from torch.profiler import ProfilerActivity, profile
    m.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.prune()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        trace = json.load(open(path))
    out = {}
    for e in trace["traceEvents"]:
        if e.get("ph") != "X" or e.get("cat") not in ("kernel", "gpu_memset", "gpu_memcpy"):
            continue
        name = re.search(r"(\w+)(?:<[^()]*>)?\(", e["name"]).group(1) if e["cat"] == "kernel" else e["cat"]
        out[name] = round(out.get(name, 0.0) + float(e["dur"]), 1)
    return out


def time_iterations(frac, steps, windows):
    import numpy as np
    import torch
    from gaussian_lic_b200 import mapper as gmapper, synthetic as syn
    P, W, H, fx, fy, cx, cy, deg, _ = syn.CONFIGS["cfg2"]
    g, _ = syn.make_scene("cfg2")
    g = with_dead_rows(g, frac)
    poses = [syn.orbit_pose(v, radius=0.25) for v in range(8)]               # bench.py's rig
    gt_host = torch.as_tensor(syn.make_gt_image(W, H)).pin_memory()
    arms, removed = {}, None
    for name in ("unpruned", "pruned"):
        m = gmapper.Mapper(W, H, fx, fy, cx, cy, sh_degree=deg, capacity=P)
        m.initialize(g)
        for R_wc, t_wc in poses:
            m.add_keyframe(R_wc, t_wc, gt_host)
        if name == "pruned":
            removed = m.prune()
        m.optimize(list(range(8)) * 2)                                       # warm-up; settles the binning capacity
        arms[name] = m
    batch = list(range(8))
    reps = (steps + 7) // 8
    wins = {k: [] for k in arms}
    for _ in range(windows):
        for name, m in arms.items():
            torch.cuda.synchronize()
            st = m.optimize(batch * reps)                                    # ms_optimize: device time of the whole window
            wins[name].append(st.ms_optimize / (8 * reps))
    med = {k: float(np.median(v)) for k, v in wins.items()}
    out = {"P": P, "dead_fraction": frac, "removed": removed, "iterations_per_window": 8 * reps, "windows": windows,
           "ms_per_iter_unpruned": round(med["unpruned"], 4), "ms_per_iter_pruned": round(med["pruned"], 4),
           "delta_ms": round(med["pruned"] - med["unpruned"], 4),
           "spread_ms": {k: round(float(np.max(v) - np.min(v)), 4) for k, v in wins.items()},
           "window_ms": {k: [round(x, 4) for x in v] for k, v in wins.items()}}
    for m in arms.values():
        m.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="timed prune calls per case")
    ap.add_argument("--steps", type=int, default=56, help="iterations per timed window")
    ap.add_argument("--windows", type=int, default=9, help="timed windows per arm (alternating)")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "prune_bench.py needs a GPU"
    calls = [time_call(P, frac, args.reps) for P in (500_000, 2_000_000) for frac in (0.1, 0.5)]
    iters = [time_iterations(frac, args.steps, args.windows) for frac in (0.1, 0.5)]
    print(json.dumps({"prune_call": calls, "iteration": iters, "card": card()}))


if __name__ == "__main__":
    main()
