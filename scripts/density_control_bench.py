"""Cost of the native mapper's density control: the screen-radius statistic on the iteration, densify_and_prune against
densify then prune, and reset_opacity.

1. The iteration: densify_bench.py's measurement, two cfg2 mappers from one initialisation with densification off and on
   (now the view-space statistics and the screen-radius slot), in alternating windows of device time.
2. Fused vs sequential: a mapper of P rows at SH degree 3 (500 000 and 2 000 000), capacity 2 P, statistics from one pass
   over the eight keyframes, a threshold that selects about 1 % of the rows (at most the rows with a nonzero statistic), a
   scene extent that clones about half of them and a min_opacity that removes about 5 % of the densify result.  Each timed
   call starts from a freshly initialised and trained map (untimed); the arms alternate: glic_mapper_densify_and_prune, and
   glic_mapper_densify followed by glic_mapper_prune with the same min_opacity.  Host time around the synchronising calls,
   for real calls and dry runs; one more call of each arm under torch.profiler (CUDA activities) gives the device time of
   every kernel, memset and copy, and the bytes the gathers move (reads of the source rows, writes of the output rows, per
   arena) over their kernel time.
3. reset_opacity on the same maps: host time around the synchronising call and its device time.

    python scripts/density_control_bench.py [--reps 5] [--steps 56] [--windows 9]

Prints one JSON line with every figure, and the card name and power limit.  Needs a GPU; writes nothing."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from densify_bench import ROOT, card, device_times, rig, time_iterations  # noqa: E402

sys.path.insert(0, ROOT)
ROW = 4 * (14 + 3 * 15)                                                  # bytes of one row of an arena at SH degree 3


def gather_bytes(P_in, P_out, kept):
    """bytes the three gathers of one compaction move: the parameters read P_out rows, each moment arena `kept` rows, and all
    three write max(P_in, P_out) rows (a prune zeroes the rows it vacates)"""
    written = max(P_in, P_out)
    return (P_out + written) * ROW + 2 * (kept + written) * ROW


def time_calls(P, reps):
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
    thr = float(max(np.float32(np.quantile(grad, 0.99)), np.float32(np.min(grad[grad > 0]))))
    d = m.download()
    smax = np.exp(d["log_scales"].astype(np.float64)).max(axis=1)
    extent = float(np.median(smax[grad >= thr]) / 0.01)
    act = 1.0 / (1.0 + np.exp(-d["opacity_logits"].astype(np.float64)))
    min_op = float(np.float32(np.quantile(act, 0.05)))

    def fused(dry=False):
        return m.densify_and_prune(extent, grad_threshold=thr, min_opacity=min_op, dry_run=dry)

    def sequential():
        c = m.densify(extent, grad_threshold=thr)
        return c, m.prune(min_op)

    t = {k: [] for k in ("fused", "fused_dry", "sequential", "sequential_dry", "reset")}
    counts = seq = None
    for r in range(reps + 1):                                              # the first round warms up
        fresh()
        t0 = time.perf_counter()
        dry = fused(True)
        t1 = time.perf_counter()
        counts = fused()
        t2 = time.perf_counter()
        m.reset_opacity()
        t3 = time.perf_counter()
        assert counts == dry
        fresh()
        t4 = time.perf_counter()
        m.densify(extent, grad_threshold=thr, dry_run=True)
        m.prune(min_op, dry_run=True)                                    # counts the map before the densify: the time, not the result
        t5 = time.perf_counter()
        seq = sequential()
        t6 = time.perf_counter()
        if r:
            for k, v in (("fused_dry", t1 - t0), ("fused", t2 - t1), ("reset", t3 - t2), ("sequential_dry", t5 - t4), ("sequential", t6 - t5)):
                t[k].append(v * 1e3)
    fresh()
    dev_fused = device_times(lambda: fused())
    dev_reset = device_times(lambda: m.reset_opacity())
    fresh()
    dev_seq = device_times(sequential)
    cap = m.stats().capacity
    m.close()
    unpruned = P + counts["cloned"] + counts["split"]
    kept = P - counts["split"]
    bytes_fused = gather_bytes(P, counts["rows"], kept)
    bytes_seq = gather_bytes(P, unpruned, kept) + gather_bytes(unpruned, unpruned - seq[1], unpruned - seq[1])
    us = lambda dev: sum(v for k, v in dev.items() if "prune_gather_kernel" in k)       # noqa: E731
    stat = lambda v: {"median": round(float(np.median(v)), 4), "min": round(float(np.min(v)), 4)}  # noqa: E731
    return {"P": P, "capacity": cap, "nonzero_rows": int((grad > 0).sum()), "counts_fused": counts,
            "counts_sequential": {"cloned": seq[0][0], "split": seq[0][1], "pruned": seq[1]},
            "selected_fraction": round((counts["cloned"] + counts["split"]) / P, 5), "pruned_fraction": round(counts["pruned"] / unpruned, 5),
            "host_ms": {k: stat(v) for k, v in t.items()},
            "device_us_fused": dev_fused, "device_us_fused_total": round(sum(dev_fused.values()), 1),
            "device_us_sequential": dev_seq, "device_us_sequential_total": round(sum(dev_seq.values()), 1),
            "device_us_reset": dev_reset,
            "gather_bytes_fused": bytes_fused, "gather_bytes_sequential": bytes_seq,
            "gather_TBps_fused": round(bytes_fused / (us(dev_fused) * 1e-6) / 1e12, 2) if us(dev_fused) else None,
            "gather_TBps_sequential": round(bytes_seq / (us(dev_seq) * 1e-6) / 1e12, 2) if us(dev_seq) else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="timed calls per case and arm")
    ap.add_argument("--steps", type=int, default=56, help="iterations per timed window")
    ap.add_argument("--windows", type=int, default=9, help="timed windows per arm (alternating)")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "density_control_bench.py needs a GPU"
    iters = time_iterations(args.steps, args.windows)
    calls = [time_calls(P, args.reps) for P in (500_000, 2_000_000)]
    print(json.dumps({"iteration": iters, "calls": calls, "card": card()}))


if __name__ == "__main__":
    main()
