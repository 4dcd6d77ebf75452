"""Where the device time of bench.py's cfg2 `value` step goes between its stream operations: the native mapper (resident
keyframes, optimiser off, one view per step) under torch.profiler (CUDA activities) in a run of its own.  For one
steady-state step it lists every kernel, memset and memcpy on the mapper's stream with its start (relative to the step's
first operation) and duration, then the number of stream operations, the sum of kernel durations, the step's device span
(first start -> last end) and the total of the idle gaps between consecutive operations; the same figures as medians over
the profiled steps; the card name and power limit.  One JSON line at the end.
Usage: python scripts/step_gaps_bench.py [steps] [chrome_trace.json]"""
import json
import os
import statistics
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from gaussian_lic_b200 import mapper as gmapper, synthetic as syn  # noqa: E402
from sort_stage_bench import card, short  # noqa: E402

STEPS = int(sys.argv[1]) if len(sys.argv) > 1 else 10
FIRST = "activations_forward_kernel"          # the first kernel of every step


def ops_of(trace):
    ev = [e for e in trace["traceEvents"] if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy")]
    out = []
    for e in ev:
        if e["cat"] == "kernel":
            nm = short(e["name"])
        else:
            nm = "memset" if e["cat"] == "gpu_memset" else "memcpy " + e.get("name", "").replace("Memcpy ", "")
        out.append({"name": nm, "kind": e["cat"], "ts": float(e["ts"]), "dur": float(e["dur"]),
                    "stream": e.get("args", {}).get("stream", e.get("tid"))})
    return sorted(out, key=lambda r: r["ts"])


def split_steps(ops):
    """Steps on the mapper's stream: each starts at the memsets right before FIRST (or at FIRST) and ends where the next begins."""
    heads = [i for i, r in enumerate(ops) if r["name"].startswith(FIRST)]
    if len(heads) < 3:
        raise SystemExit("fewer than 3 steps found in the trace")
    stream = ops[heads[0]]["stream"]
    mine = [r for r in ops if r["stream"] == stream]
    heads = [i for i, r in enumerate(mine) if r["name"].startswith(FIRST)]
    starts = []
    for h in heads:
        i = h
        while i > 0 and mine[i - 1]["kind"] == "gpu_memset":     # the previous step ends with its loss D2H copy
            i -= 1
        starts.append(i)
    # the step before the last head ends where the last head's step starts; the last step may be cut by the optimize() call's tail
    steps = [mine[a:b] for a, b in zip(starts[:-1], starts[1:])]
    return stream, steps


def figures(step):
    kern = sum(r["dur"] for r in step if r["kind"] == "kernel")
    gaps, end, overlap = 0.0, step[0]["ts"] + step[0]["dur"], 0.0
    for r in step[1:]:
        d = r["ts"] - end
        if d > 0:
            gaps += d
        else:
            overlap -= d
        end = max(end, r["ts"] + r["dur"])
    span = end - step[0]["ts"]
    one_cta = sum(r["dur"] for r in step if any(k in r["name"] for k in ("sort_scan_hist_kernel", "bucket_scan_kernel", "live_scan_kernel",
                                                                           "overflow_word_kernel")))
    return {"ops": len(step), "kernels": sum(r["kind"] == "kernel" for r in step), "kernel_us": kern, "span_us": span,
            "gap_us": gaps, "overlap_us": overlap, "one_cta_us": one_cta}


def main():
    P, W, H, fx, fy, cx, cy, deg, zmax = syn.CONFIGS["cfg2"]
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    g, _ = syn.make_scene("cfg2")
    gt = torch.as_tensor(syn.make_gt_image(W, H)).to(dev)
    mp = gmapper.Mapper(W, H, fx, fy, cx, cy, sh_degree=deg, capacity=P)
    mp.initialize(g)
    for v in range(8):
        mp.add_keyframe(*syn.orbit_pose(v, radius=0.25), gt)  # resident keyframes, as bench.py's `value` leg
    batch = [0]                                              # bench.py --gpus 1: one resident view per step
    mp.set_optimizer(False)
    mp.optimize(batch * 5)
    torch.cuda.synchronize()
    step_ms = mp.optimize(batch * 20).ms_optimize / 20       # device time of the whole step, profiler off

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        mp.optimize(batch * (STEPS + 1))
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as td:
        path = sys.argv[2] if len(sys.argv) > 2 else os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        trace = json.load(open(path))
    mp.close()

    ops = ops_of(trace)
    stream, steps = split_steps(ops)
    steps = steps[1:] if len(steps) > 2 else steps          # the first profiled step follows the profiler's start
    figs = [figures(s) for s in steps]
    med = {k: statistics.median(f[k] for f in figs) for k in figs[0]}
    one = steps[len(steps) // 2]
    others = [r for r in ops if r["stream"] != stream and one[0]["ts"] <= r["ts"] <= one[-1]["ts"] + one[-1]["dur"]]

    name, q = card()
    print("card: %s | power.limit, clocks.max.sm: %s" % (name, q))
    print("one steady-state step on the mapper's stream (%d operations):" % len(one))
    print("%4s %-58s %10s %9s %9s" % ("#", "operation", "start_us", "dur_us", "gap_us"))
    end = one[0]["ts"]
    for i, r in enumerate(one):
        print("%4d %-58s %10.2f %9.2f %9.2f" % (i + 1, r["name"][:58], r["ts"] - one[0]["ts"], r["dur"], r["ts"] - end if i else 0.0))
        end = max(end, r["ts"] + r["dur"])
    for r in others:
        print("     [other stream] %-47s %10.2f %9.2f" % (r["name"][:47], r["ts"] - one[0]["ts"], r["dur"]))
    f = figures(one)
    print("stream operations %d (kernels %d) | kernels %.1f us | span %.1f us | gaps %.1f us | overlap %.1f us | one-CTA kernels %.1f us"
          % (f["ops"], f["kernels"], f["kernel_us"], f["span_us"], f["gap_us"], f["overlap_us"], f["one_cta_us"]))
    print("median of %d steps: operations %d | kernels %.1f us | span %.1f us | gaps %.1f us | one-CTA kernels %.1f us"
          % (len(figs), med["ops"], med["kernel_us"], med["span_us"], med["gap_us"], med["one_cta_us"]))
    print("step time with the profiler off: %.4f ms" % step_ms)
    print(json.dumps({"card": name, "power_limit_max_sm": q, "steps_profiled": len(figs), "step_ms_profiler_off": round(step_ms, 4),
                      "median": {k: round(v, 2) for k, v in med.items()}, "other_stream_ops": len(others),
                      "step": [[r["name"], round(r["dur"], 2)] for r in one]}))


if __name__ == "__main__":
    main()
