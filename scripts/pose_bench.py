"""Cost of the per-keyframe pose refinement (glic_mapper_enable_pose_refinement) in the native mapping iteration at cfg2.

Two native mappers on the same scene and keyframes run bench.py's mapping_iter_native step: one view per iteration from eight
pinned-host keyframes (image H2D, activations, forward, fused L1 + D-SSIM loss, backward, Gaussian Adam).  One mapper never
enables pose refinement; the other trains the keyframe poses (the pose gradient fused into the per-Gaussian backward, its
finish kernel, the pose Adam step and camera rebuild).  Their timed windows alternate in this one call, so
both see the same machine state; each window is device time on the mapper's stream over `--steps` iterations.

    python scripts/pose_bench.py [--steps 50] [--windows 9] [--config cfg2]

Prints one JSON line: the median ms per iteration of each arm, every window, the delta, and the card name and power limit.
Needs a GPU; writes nothing."""
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
    ap.add_argument("--steps", type=int, default=50, help="iterations per timed window")
    ap.add_argument("--windows", type=int, default=9, help="timed windows per arm (alternating)")
    ap.add_argument("--lr-translation", type=float, default=1e-4)
    ap.add_argument("--lr-rotation", type=float, default=1e-4)
    args = ap.parse_args()
    import numpy as np
    import torch
    from gaussian_lic_b200 import mapper as gmapper, synthetic as syn
    assert torch.cuda.is_available(), "pose_bench.py needs a GPU"
    P, W, H, fx, fy, cx, cy, deg, _ = syn.CONFIGS[args.config]
    g, _ = syn.make_scene(args.config)
    poses = [syn.orbit_pose(v, radius=0.25) for v in range(8)]               # bench.py's rig
    gt_host = torch.as_tensor(syn.make_gt_image(W, H)).pin_memory()
    arms = {}
    for name in ("off", "on"):
        m = gmapper.Mapper(W, H, fx, fy, cx, cy, sh_degree=deg, capacity=P)
        m.initialize(g)
        for R_wc, t_wc in poses:
            m.add_keyframe(R_wc, t_wc, gt_host)
        if name == "on":
            m.enable_pose_refinement(args.lr_translation, args.lr_rotation)
        m.optimize(list(range(8)) * 2)                                       # warm-up; settles the binning capacity
        arms[name] = m
    batch = list(range(8))
    reps = (args.steps + 7) // 8
    wins = {"off": [], "on": []}
    for _ in range(args.windows):
        for name in ("off", "on"):
            torch.cuda.synchronize()
            st = arms[name].optimize(batch * reps)                           # ms_optimize: device time of the whole window
            wins[name].append(st.ms_optimize / (8 * reps))
    med = {k: float(np.median(v)) for k, v in wins.items()}
    spread = {k: float(np.max(v) - np.min(v)) for k, v in wins.items()}
    moved = [float(np.abs(arms["on"].pose(k)[1] - poses[k][1]).max()) for k in range(8)]
    out = {"config": args.config, "P": P, "W": W, "H": H, "iterations_per_window": 8 * reps, "windows": args.windows,
           "ms_per_iter_off": round(med["off"], 4), "ms_per_iter_on": round(med["on"], 4),
           "delta_ms": round(med["on"] - med["off"], 4), "spread_ms": {k: round(v, 4) for k, v in spread.items()},
           "window_ms": {k: [round(x, 4) for x in v] for k, v in wins.items()},
           "pose_moved": max(moved),
           "card": card()}
    for m in arms.values():
        m.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
