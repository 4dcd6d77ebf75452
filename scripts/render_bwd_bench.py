"""Time the render backward alone at cfg2 and count the work it does.

Builds bench.py's scene and view 0 through ops.CRasterizer, runs one forward and the fused L1 + D-SSIM loss, then launches
only the render backward (glic_debug_render_backward: the live-bucket scan + render_backward_kernel) many times.  Each launch
is timed by its own pair of CUDA events; the four 2-D gradient buffers are re-zeroed between launches, outside the events.
The production kernel and the former body (exact expf for every pixel) alternate window by window, so both see the same
machine state.  The counting form of each kernel reports what one launch walks:

  live_buckets       buckets some pixel reached (one warp each)
  splats             (live bucket, splat) pairs whose row mask is not empty
  splats_taken       of these, splats some pixel took (they pay the reduce-scatter and the 9 RED)
  visits             (splat, two row pairs) visits that pass the warp-uniform row test
  visits_taken       of these, visits in which some pixel takes the splat
  candidate_pixels   pixels of visits with the pixel's rows in range, k < rel and power <= 0
  taken_pixels       pixel-splat pairs taken (alpha >= 1/255): identical for both forms
  fallback_pixels    pixels the production kernel decided from the exact expf (fast alpha within the guard band)

    python scripts/render_bwd_bench.py [--launches 50] [--windows 7] [--config cfg2]

Prints one JSON line with the median us per launch of each form, every window, the counters and the card's name and power
limit.  Needs a GPU; writes nothing."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power, clock = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="cfg2")
    ap.add_argument("--launches", type=int, default=50, help="timed launches per window")
    ap.add_argument("--windows", type=int, default=7, help="timed windows per form (alternating)")
    args = ap.parse_args()
    import numpy as np
    import torch
    from gaussian_lic_b200 import mapper as gmapper, ops, synthetic as syn
    assert torch.cuda.is_available(), "render_bwd_bench.py needs a GPU"
    P, W, H, fx, fy, cx, cy, deg, _ = syn.CONFIGS[args.config]
    g, _ = syn.make_scene(args.config)
    cam = gmapper.camera_block(W, H, fx, fy, cx, cy, *syn.orbit_pose(0, radius=0.25))      # bench.py's view 0
    r = ops.CRasterizer(W, H)
    gd = ops.scene_to_device(g)
    view = r.make_view(cam)
    img, _, _ = r.forward(gd, view)
    gt = torch.as_tensor(syn.make_gt_image(W, H)).cuda()
    _, dL = r.loss(img, gt)
    grads = r.alloc_grads()
    two_d = [grads[k] for k in ("dL_dmeans2D", "dL_dconic", "dL_dopacity", "dL_dcolors")]
    forms = {"fast": False, "exact": True}

    counts = {}
    for name, exact in forms.items():
        ctr = torch.zeros(8, dtype=torch.int64, device="cuda")
        for t in two_d:
            t.zero_()
        r.render_backward(view, dL, grads, exact=exact, counters=ctr)
        counts[name] = dict(zip(ops.CRasterizer.BWD_COUNTERS, (int(x) for x in ctr.tolist())))

    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.launches)]

    def window(exact):
        for a, b in ev:
            for t in two_d:
                t.zero_()
            a.record()
            r.render_backward(view, dL, grads, exact=exact)
            b.record()
        torch.cuda.synchronize()
        return 1e3 * sum(a.elapsed_time(b) for a, b in ev) / len(ev)

    for exact in forms.values():
        window(exact)                                                       # warm-up
    wins = {k: [] for k in forms}
    for _ in range(args.windows):
        for name, exact in forms.items():
            wins[name].append(window(exact))
    med = {k: float(np.median(v)) for k, v in wins.items()}
    out = {"config": args.config, "P": P, "W": W, "H": H, "R": r.R, "launches_per_window": args.launches, "windows": args.windows,
           "us_per_launch": {k: round(v, 2) for k, v in med.items()},
           "spread_us": {k: round(float(np.max(v) - np.min(v)), 2) for k, v in wins.items()},
           "window_us": {k: [round(x, 2) for x in v] for k, v in wins.items()},
           "counters": counts, "card": card()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
