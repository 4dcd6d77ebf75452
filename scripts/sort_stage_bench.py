"""Per-kernel device time of the binning span of bench.py's cfg2 `value` step (native mapper, resident keyframes, optimiser
off): every kernel and memset from the depth sort's preparation through tile_ranges_kernel, averaged over the profiled
steps, captured with torch.profiler (CUDA activities) in a run of its own.  Prints the card name, its power limit, a table
and one JSON line.  Usage: python scripts/sort_stage_bench.py [steps] [chrome_trace.json]"""
import collections
import json
import os
import re
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gaussian_lic_b200 import mapper as gmapper, synthetic as syn  # noqa: E402

STEPS = int(sys.argv[1]) if len(sys.argv) > 1 else 10
SORT_KERNELS = ("onesweep_pass_kernel", "sort_scan_hist_kernel", "depth_scan_kernel")


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = "nvidia-smi unavailable (%r)" % (e,)
    return name, q


def short(name):
    """'void glic::(anonymous namespace)::onesweep_pass_kernel<unsigned int, 16>(...)' -> 'onesweep_pass_kernel<unsigned int, 16>'"""
    n = re.sub(r"^void\s+", "", name).replace("(anonymous namespace)::", "")
    depth, cut, ns = 0, len(n), 0
    for i, ch in enumerate(n):
        depth += (ch == "<") - (ch == ">")
        if depth == 0 and ch == "(":
            cut = i
            break
        if depth == 0 and n.startswith("::", i):
            ns = i + 2
    return n[ns:cut]


def main():
    P, W, H, fx, fy, cx, cy, deg, zmax = syn.CONFIGS["cfg2"]
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    g, _ = syn.make_scene("cfg2")
    gt = torch.as_tensor(syn.make_gt_image(W, H)).to(dev)
    mp = gmapper.Mapper(W, H, fx, fy, cx, cy, sh_degree=deg, capacity=P)
    mp.initialize(g)
    for v in range(8):
        mp.add_keyframe(*syn.orbit_pose(v, radius=0.25), gt)
    batch = list(range(1))                                  # bench.py --gpus 1: one resident view per step
    mp.set_optimizer(False)
    mp.optimize(batch * 5)
    torch.cuda.synchronize()
    step_ms = mp.optimize(batch * 20).ms_optimize / 20      # device time of the whole step, profiler off

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        mp.optimize(batch * STEPS)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as td:
        path = sys.argv[2] if len(sys.argv) > 2 else os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        trace = json.load(open(path))
    mp.close()

    ev = sorted((e for e in trace["traceEvents"] if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy")),
                key=lambda e: e["ts"])
    # one span per step: the memsets right before preprocess_forward_kernel (header, scan status, depth-sort histograms)
    # through tile_ranges_kernel
    spans, cur, pending = [], None, []
    for e in ev:
        nm = e["name"] if e["cat"] == "kernel" else ("memset" if e["cat"] == "gpu_memset" else "memcpy")
        rec = (short(nm) if e["cat"] == "kernel" else nm, float(e["ts"]), float(e["dur"]))
        if cur is None:
            if "preprocess_forward_kernel" in nm:
                cur = pending + [rec]
            else:
                pending = pending + [rec] if e["cat"] != "kernel" else []
            continue
        cur.append(rec)
        if "tile_ranges_kernel" in nm:
            spans.append(cur)
            cur, pending = None, []
    if not spans:
        raise SystemExit("no preprocess -> ranges span found in the trace")
    # label repeated launches of one kernel within a span (the sort passes) by their order
    per = collections.OrderedDict()
    for sp in spans:
        seen = collections.Counter()
        for nm, _, dur in sp:
            seen[nm] += 1
            key = "%s #%d" % (nm, seen[nm])
            per.setdefault(key, []).append(dur)
    n = len(spans)
    rows = [(k, sum(v) / n, len(v) / n) for k, v in per.items()]
    sort_us = sum(us for k, us, _ in rows if any(s in k for s in SORT_KERNELS))
    span_us = sum(us for _, us, _ in rows)
    wall_us = sum(sp[-1][1] + sp[-1][2] - sp[0][1] for sp in spans) / n
    name, q = card()
    print("card: %s | power.limit, clocks.max.sm: %s" % (name, q))
    print("%-60s %10s %8s" % ("kernel (order within the span)", "us/step", "calls"))
    for k, us, c in rows:
        print("%-60s %10.2f %8.2f" % (k[:60], us, c))
    print("%-60s %10.2f" % ("sum of the sort kernels (passes, scan, depth scan)", sort_us))
    print("%-60s %10.2f" % ("sum of every kernel and memset in the span", span_us))
    print("%-60s %10.2f" % ("span wall time (first start -> last end)", wall_us))
    print(json.dumps({"card": name, "power_limit_max_sm": q, "steps_profiled": n, "step_ms_profiler_off": round(step_ms, 4),
                      "sort_kernels_us": round(sort_us, 2), "span_kernels_us": round(span_us, 2), "span_wall_us": round(wall_us, 2),
                      "kernels_us": {k: round(us, 2) for k, us, _ in rows}}))


if __name__ == "__main__":
    main()
