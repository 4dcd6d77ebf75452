#!/usr/bin/env python
"""glic_lpips at 640x512 and 1920x1080: device time per call (CUDA events, median of timed windows) and the FLOP/s it achieves
on the five convolutions (2 * M * N * K per layer, batch of 2; ~9.2 GFLOP per image at 640x512, ~59 at 1920x1080).  Where
build() copied the reference's TorchScript module to oracle/_ref/lpips_alex.pt, the module is timed on the same card with
TF32 off (its traced convolutions' allow_tf32 argument rewritten, see tests/golden/make_lpips_golden.py) and as traced (TF32
convolutions); the module's float64 value is printed beside glic_lpips's as the accuracy yardstick.  Prints the card name and
its power limit beside the numbers.

    python scripts/lpips_bench.py [--iters N] [--windows K]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LAYERS = [(64, 3, 11, 4, 2), (192, 64, 5, 1, 2), (384, 192, 3, 1, 1), (256, 384, 3, 1, 1), (256, 256, 3, 1, 1)]  # Cout Cin k s p


def conv_flops(H, W):
    """multiply-adds x 2 of the five convolutions for ONE image"""
    h, w = (H + 4 - 11) // 4 + 1, (W + 4 - 11) // 4 + 1
    sizes = [(h, w)]
    h, w = (h - 3) // 2 + 1, (w - 3) // 2 + 1
    sizes.append((h, w))
    h, w = (h - 3) // 2 + 1, (w - 3) // 2 + 1
    sizes += [(h, w)] * 3
    return sum(2 * hh * ww * co * ci * k * k for (hh, ww), (co, ci, k, _, _) in zip(sizes, LAYERS))


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=20).stdout.strip()
        return out or "unknown"
    except Exception:
        return "unknown"


def time_fn(fn, iters, windows):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(windows):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b) / iters)
    return float(np.median(ms)), float(max(ms) - min(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--windows", type=int, default=7)
    args = ap.parse_args()
    from gaussian_lic_b200 import lpips_weights, ops
    import importlib.util
    spec = importlib.util.spec_from_file_location("g", os.path.join(ROOT, "tests", "golden", "make_lpips_golden.py"))
    G = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(G)
    pt = os.path.join(ROOT, "oracle", "_ref", "lpips_alex.pt")
    if os.path.isfile(G.WEIGHTS):
        w = torch.from_numpy(lpips_weights.read(G.WEIGHTS)).cuda()
    else:                                                            # timing does not depend on the weights' values
        print("oracle/_ref/lpips_alex.bin not built: timing seeded synthetic weights", file=sys.stderr)
        w = torch.from_numpy(G.synthetic_payload(0)).cuda()
    res = dict(device=torch.cuda.get_device_name(0), power_limit=power_limit(), rows=[])
    for W, H in ((640, 512), (1920, 1080)):
        x, y = (torch.from_numpy(a).cuda() for a in G.make_pair(W, H, 5, "heavy"))
        scratch = torch.empty(ops.capi.lib.glic_lpips_scratch_bytes(H, W), dtype=torch.uint8, device="cuda")
        ms, spread = time_fn(lambda: ops.lpips(x, y, w, scratch=scratch), args.iters, args.windows)
        flop = 2 * conv_flops(H, W)
        row = dict(size="%dx%d" % (W, H), gflop_per_call=flop / 1e9, glic_ms=ms, glic_spread_ms=spread, glic_tflops=flop / ms / 1e9,
                   value=float(ops.lpips(x, y, w)))
        if os.path.isfile(pt):
            with torch.no_grad():
                for tag, tf32 in (("ref_tf32_off", False), ("ref_as_traced", None)):
                    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
                    m = G.reference_module(pt, allow_tf32=tf32)
                    xb, yb = x[None], y[None]
                    row[tag + "_ms"], row[tag + "_spread_ms"] = time_fn(lambda: m(xb, yb), args.iters, args.windows)
                    row[tag + "_value"] = float(m(xb, yb))
                    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved
            row["ref_float64_value"] = G.reference_lpips(G.reference_module64(pt), x.cpu().numpy(), y.cpu().numpy(), dtype=torch.float64)
        res["rows"].append(row)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
