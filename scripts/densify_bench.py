"""Cost of densification in the native mapper: the statistics on the iteration, and the glic_mapper_densify call.

1. The iteration: two cfg2 mappers from one initialisation, one with densification enabled (statistics gathered every
   iteration, densify never called), the other without.  Their timed windows alternate in this one call (bench.py's
   mapping_iter_native step: one view per iteration from eight pinned-host keyframes, optimiser on); each window is device
   time on the mapper's stream.
2. The call: a mapper of P rows at SH degree 3 (cfg2's 500 000 and 2 000 000), capacity = 2 P, statistics from one pass over
   the eight keyframes, a threshold that selects the given fraction of the rows and a scene extent that clones about half of
   them.  Only the rows with a nonzero statistic can be selected (grad_i = 0 < threshold for the others), and at cfg2 the rig's
   eight views give few rows one: when the requested fraction exceeds them, every such row is selected, and `selected` /
   `selected_fraction_actual` report what the call did.  Each timed call starts from a freshly initialised and trained map (untimed) and is timed by a host clock around the
   synchronising call: selection, spare-arena allocation and zeroing, three gathers, the children, frees.  One more call runs
   under torch.profiler (CUDA activities): the device time of each kernel, memset and copy it issues, and the bytes the three
   gathers move over their kernel time.

    python scripts/densify_bench.py [--reps 5] [--steps 56] [--windows 9]

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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power, clock = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def rig(W, H):
    import torch
    from gaussian_lic_b200 import synthetic as syn
    poses = [syn.orbit_pose(v, radius=0.25) for v in range(8)]               # bench.py's rig
    return poses, torch.as_tensor(syn.make_gt_image(W, H)).pin_memory()


def device_times(fn):
    """device time (us) of every kernel, memset and copy fn() issues, from torch.profiler's trace"""
    import tempfile
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        fn()
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


def time_call(P, frac, reps):
    import numpy as np
    from gaussian_lic_b200 import mapper as gmapper, synthetic as syn
    _, W, H, fx, fy, cx, cy, deg, zmax = syn.CONFIGS["cfg2"]
    g = syn.make_gaussians(P, W, H, fx, fy, sh_degree=deg, zmax=zmax, seed=42)
    poses, gt = rig(W, H)
    m = gmapper.Mapper(W, H, fx, fy, cx, cy, sh_degree=deg, capacity=2 * P)
    for R_wc, t_wc in poses:
        m.add_keyframe(R_wc, t_wc, gt)
    m.enable_densification()

    def fresh():
        m.initialize(g)
        m.optimize(list(range(8)))
        m.synchronize()

    fresh()
    acc, den = m.densify_stats()
    grad = np.where(den > 0, acc / np.where(den > 0, den, 1), 0).astype(np.float32)
    thr = float(max(np.float32(np.quantile(grad, 1.0 - frac)), np.float32(np.min(grad[grad > 0]))))
    smax = np.exp(m.download()["log_scales"].astype(np.float64)).max(axis=1)
    extent = float(np.median(smax[grad >= thr]) / 0.01)
    real, dry, counts = [], [], None
    for r in range(reps + 1):                                              # the first call warms up
        fresh()
        t0 = time.perf_counter()
        c_dry = m.densify(extent, grad_threshold=thr, dry_run=True)
        t1 = time.perf_counter()
        counts = m.densify(extent, grad_threshold=thr)
        t2 = time.perf_counter()
        assert counts == c_dry and m.stats().num_gaussians == P + sum(counts)
        if r:
            dry.append((t1 - t0) * 1e3)
            real.append((t2 - t1) * 1e3)
    fresh()
    device = device_times(lambda: m.densify(extent, grad_threshold=thr))
    cap = m.stats().capacity
    m.close()
    row = 4 * (14 + 3 * 15)
    total, kept = P + sum(counts), P - counts[1]
    gathered = (total * row + total * row) + 2 * (kept * row + total * row)   # parameters: every result row; moments: the kept rows
    gather_us = sum(v for k, v in device.items() if "prune_gather_kernel" in k)
    return {"P": P, "capacity": cap, "selected_fraction": frac, "nonzero_rows": int((grad > 0).sum()), "selected": sum(counts),
            "selected_fraction_actual": round(sum(counts) / P, 5), "cloned": counts[0], "split": counts[1],
            "ms_densify_median": round(float(np.median(real)), 4), "ms_densify_min": round(float(np.min(real)), 4),
            "ms_dry_run_median": round(float(np.median(dry)), 4), "ms_densify_all": [round(x, 4) for x in real],
            "device_us": device, "device_us_total": round(sum(device.values()), 1), "gather_bytes": gathered,
            "gather_TBps": round(gathered / (gather_us * 1e-6) / 1e12, 2) if gather_us else None}


def time_iterations(steps, windows):
    import numpy as np
    import torch
    from gaussian_lic_b200 import mapper as gmapper, synthetic as syn
    P, W, H, fx, fy, cx, cy, deg, _ = syn.CONFIGS["cfg2"]
    g, _ = syn.make_scene("cfg2")
    poses, gt = rig(W, H)
    arms = {}
    for name in ("off", "on"):
        m = gmapper.Mapper(W, H, fx, fy, cx, cy, sh_degree=deg, capacity=P)
        m.initialize(g)
        for R_wc, t_wc in poses:
            m.add_keyframe(R_wc, t_wc, gt)
        if name == "on":
            m.enable_densification()
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
    out = {"P": P, "iterations_per_window": 8 * reps, "windows": windows,
           "ms_per_iter_off": round(med["off"], 4), "ms_per_iter_on": round(med["on"], 4), "delta_ms": round(med["on"] - med["off"], 4),
           "spread_ms": {k: round(float(np.max(v) - np.min(v)), 4) for k, v in wins.items()},
           "window_ms": {k: [round(x, 4) for x in v] for k, v in wins.items()}}
    for m in arms.values():
        m.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="timed densify calls per case")
    ap.add_argument("--steps", type=int, default=56, help="iterations per timed window")
    ap.add_argument("--windows", type=int, default=9, help="timed windows per arm (alternating)")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "densify_bench.py needs a GPU"
    iters = time_iterations(args.steps, args.windows)
    calls = [time_call(P, frac, args.reps) for P in (500_000, 2_000_000) for frac in (0.01, 0.1)]
    print(json.dumps({"iteration": iters, "densify_call": calls, "card": card()}))


if __name__ == "__main__":
    main()
