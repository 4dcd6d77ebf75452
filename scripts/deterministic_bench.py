"""Cost of the deterministic render backward (glic_backward_deterministic) against the atomic one (glic_backward) at cfg2.

Builds bench.py's scene and view 0 through ops.CRasterizer, runs one forward and the fused L1 + D-SSIM loss, then times whole
backward calls (render backward + per-Gaussian backward), each by its own pair of CUDA events.  The atomic and deterministic
forms alternate window by window, so both see the same machine state; the median window is reported with the spread.  A
second pair of arms times the native mapping iteration (glic_mapper_optimize on view 0, synchronised) with
GLIC_MAPPER_OPT_DETERMINISTIC off and on, alternated window by window.  A separate torch.profiler run attributes the deterministic form's device time to its kernels (the render backward that stores
the entries, the entry sort's passes, the per-Gaussian fold).  Also reports the workspace bytes and the card's name and power
limit, read in the same call.

    python scripts/deterministic_bench.py [--calls 30] [--windows 7] [--config cfg2]

Prints one JSON line.  Needs a GPU; writes nothing."""
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
    ap.add_argument("--calls", type=int, default=30, help="timed backward calls per window")
    ap.add_argument("--windows", type=int, default=7, help="timed windows per form (alternating)")
    args = ap.parse_args()
    import numpy as np
    import torch
    from gaussian_lic_b200 import mapper as gmapper, ops, synthetic as syn
    assert torch.cuda.is_available(), "deterministic_bench.py needs a GPU"
    P, W, H, fx, fy, cx, cy, deg, _ = syn.CONFIGS[args.config]
    g, _ = syn.make_scene(args.config)
    cam = gmapper.camera_block(W, H, fx, fy, cx, cy, *syn.orbit_pose(0, radius=0.25))      # bench.py's view 0
    r = ops.CRasterizer(W, H)
    gd = ops.scene_to_device(g)
    view = r.make_view(cam)
    img, _, radii = r.forward(gd, view)
    gt = torch.as_tensor(syn.make_gt_image(W, H)).cuda()
    _, dL = r.loss(img, gt)
    grads = r.alloc_grads()
    forms = {"atomic": False, "deterministic": True}
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.calls)]

    def window(det):
        for a, b in ev:
            a.record()
            r.backward(gd, view, radii, dL, grads=grads, deterministic=det)
            b.record()
        torch.cuda.synchronize()
        return 1e3 * sum(a.elapsed_time(b) for a, b in ev) / len(ev)

    for det in forms.values():
        window(det)                                                         # warm-up (and the workspace's first allocation)
    wins = {k: [] for k in forms}
    for _ in range(args.windows):
        for name, det in forms.items():
            wins[name].append(window(det))
    med = {k: float(np.median(v)) for k, v in wins.items()}

    # the native mapping iteration (glic_mapper_optimize on view 0, host clock around synchronised calls), option off and on
    # alternated window by window; each switch drains the pipeline
    import time
    m = gmapper.Mapper(W, H, fx, fy, cx, cy, sh_degree=deg, capacity=P)
    m.initialize(g)
    m.add_keyframe(*syn.orbit_pose(0, radius=0.25), syn.make_gt_image(W, H))

    def mwindow(det):
        m.set_deterministic(det)
        m.optimize([0])
        m.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.calls):
            m.optimize([0])
        m.synchronize()
        return 1e6 * (time.perf_counter() - t0) / args.calls

    for det in forms.values():
        mwindow(det)
    mwins = {k: [] for k in forms}
    for _ in range(args.windows):
        for name, det in forms.items():
            mwins[name].append(mwindow(det))
    mloss = {}
    for name, det in forms.items():
        m.set_deterministic(det)
        mloss[name] = float(m.optimize([0]).last_loss)
    m.close()

    # per-kernel device time of the deterministic form, in a run of its own
    from torch.profiler import ProfilerActivity, profile
    n_prof = 10
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n_prof):
            r.backward(gd, view, radii, dL, grads=grads, deterministic=True)
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = getattr(e, "cuda_time_total", 0.0)
        for tag in ("render_backward_kernel", "onesweep_pass_kernel", "sort_histogram_kernel", "sort_scan_hist_kernel",
                    "det_reduce_kernel", "live_scan_kernel", "preprocess_backward"):
            if tag in e.key:
                kernels[tag] = round(kernels.get(tag, 0.0) + t / n_prof, 2)
    out = {"config": args.config, "P": P, "W": W, "H": H, "R": r.R, "capacity": r.cap, "calls_per_window": args.calls,
           "windows": args.windows, "us_per_backward": {k: round(v, 2) for k, v in med.items()},
           "spread_us": {k: round(float(np.max(v) - np.min(v)), 2) for k, v in wins.items()},
           "window_us": {k: [round(x, 2) for x in v] for k, v in wins.items()},
           "deterministic_kernel_us_per_call": kernels,
           "mapper_us_per_iteration": {k: round(float(np.median(v)), 2) for k, v in mwins.items()},
           "mapper_spread_us": {k: round(float(np.max(v) - np.min(v)), 2) for k, v in mwins.items()},
           "mapper_last_loss": mloss,
           "workspace_bytes": {"deterministic": int(r.lib.glic_deterministic_bytes(r.cap, W, H)),
                               "sample": int(r.lib.glic_sample_bytes(r.cap, W, H)),
                               "binning": int(r.lib.glic_binning_bytes(r.cap))},
           "card": card()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
