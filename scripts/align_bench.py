"""Cost of test-time alignment (glic_mapper_align) at cfg2.

One native mapper (pose refinement on) with eight pinned-host training keyframes (bench.py's rig) and one held-out keyframe.
  - per-iteration device-bound time: an alignment iteration ((t(align N) - t(align 0)) / N, host clock around calls that end
    in a synchronise; the loop is enqueued without one) and a training iteration (ms_optimize / iterations, optimiser on),
    their timed windows alternating in this one call;
  - the per-Gaussian backward alone on the same render-backward outputs (glic_debug_pose_backward), the POSE_ONLY form
    against the COMPACT + POSE form: CUDA events over `--launches` launches per window, windows alternating, with the bytes
    each form needs (computed from the shapes and the view's visible rows);
  - a whole glic_mapper_align call at 100 iterations by a host clock (it ends in a synchronise).

    python scripts/align_bench.py [--config cfg2] [--iters 100] [--windows 7] [--launches 200]

Prints one JSON line with the medians, every window, and the card name and power limit.  Needs a GPU; writes nothing."""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def backward_bytes(P, vis, M):
    """bytes each form of the per-Gaussian backward reads and writes: radii of every row; per visible row means, scales,
    rotations (12 + 12 + 16), the clamp byte, the 2-D gradients (12 + 16), dL/dcolour (12) and the SH rest (12 M); the POSE
    form also reads opacity, dL/dopacity and the raw rotation (4 + 4 + 16) per visible row and writes 44 B for every row"""
    only = 4 * P + vis * (12 + 12 + 16 + 1 + 12 + 16 + 12 + 12 * M)
    return only, only + vis * 24 + 44 * P


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="cfg2")
    ap.add_argument("--iters", type=int, default=100, help="alignment iterations per call, and training iterations per window")
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--launches", type=int, default=200, help="backward launches per timed window")
    args = ap.parse_args()
    import numpy as np
    import torch
    from gaussian_lic_b200 import capi, mapper as gmapper, model, ops, synthetic as syn
    from pose_bench import card
    assert torch.cuda.is_available(), "align_bench.py needs a GPU"
    P, W, H, fx, fy, cx, cy, deg, _ = syn.CONFIGS[args.config]
    g, _ = syn.make_scene(args.config)
    poses = [syn.orbit_pose(v, radius=0.25) for v in range(8)]
    gt_host = torch.as_tensor(syn.make_gt_image(W, H)).pin_memory()
    m = gmapper.Mapper(W, H, fx, fy, cx, cy, sh_degree=deg, capacity=P)
    m.initialize(g)
    for R_wc, t_wc in poses:
        m.add_keyframe(R_wc, t_wc, gt_host)
    m.add_keyframe(*syn.orbit_pose(3, radius=0.3), gt_host, train=False)
    m.enable_pose_refinement(1e-4, 1e-4)
    m.optimize(list(range(8)) * 2)                                          # warm-up; settles the binning capacity
    m.align(0, iterations=args.iters)
    batch = list(range(8))
    reps = (args.iters + 7) // 8

    def align_s(n):
        t = time.perf_counter()
        r = m.align(0, iterations=n, lr_translation=1e-4, lr_rotation=1e-4)
        dt = time.perf_counter() - t
        assert r["steps"] == n
        return dt

    wins = {"align_iter": [], "train_iter": [], "align_call": []}
    for _ in range(args.windows):
        torch.cuda.synchronize()
        t0 = align_s(0)
        tn = align_s(args.iters)
        wins["align_iter"].append(1e3 * (tn - t0) / args.iters)
        wins["align_call"].append(1e3 * tn)
        st = m.optimize(batch * reps)
        wins["train_iter"].append(st.ms_optimize / (8 * reps))

    # the per-Gaussian backward alone, both forms on the same render-backward outputs
    dev = torch.device("cuda:0")
    raw = dict(g, degree=deg)
    mdl = model.PackedModel(raw, dev)
    mdl.activate()
    gi = mdl.inputs
    rast = ops.CRasterizer(W, H, dev)
    cam = gmapper.camera_block(W, H, fx, fy, cx, cy, *poses[0])
    view = rast.make_view(cam)
    color, _, radii = rast.forward(gi, view)
    _, dL = rast.loss(color, gt_host.to(dev), 0.2)
    grads = rast.alloc_grads()
    for k in ("dL_dmeans2D", "dL_dconic", "dL_dopacity", "dL_dcolors"):
        grads[k].zero_()
    rast.render_backward(view, dL, grads)
    M = rast.M
    rot_raw = torch.as_tensor(np.asarray(g["rots"], np.float32)).to(dev)
    part = torch.empty((P + 127) // 128 * 6, dtype=torch.float64, device=dev)
    geo = torch.empty(11 * P, dtype=torch.float32, device=dev)
    pose6 = {k: torch.empty(6, dtype=torch.float32, device=dev) for k in (0, 1)}

    def launch(only):
        capi.check(capi.lib.glic_debug_pose_backward(
            P, deg, M, capi.ptr(gi["means"]), capi.ptr(gi["scales"]), capi.ptr(gi["rots"]), capi.ptr(rot_raw), capi.ptr(gi["opacity"]),
            capi.ptr(gi["sh"]) if M else None, C.byref(view), capi.ptr(radii), capi.ptr(rast.geom_ws), capi.ptr(grads["dL_dmeans2D"]),
            capi.ptr(grads["dL_dconic"]), capi.ptr(grads["dL_dopacity"]), capi.ptr(grads["dL_dcolors"]), only,
            None if only else capi.ptr(geo), capi.ptr(part), capi.ptr(pose6[only]), None), "debug_pose_backward")

    for only in (0, 1):
        for _ in range(20):
            launch(only)
    bwd = {0: [], 1: []}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for _ in range(args.windows):
        for only in (0, 1):
            torch.cuda.synchronize()
            ev[0].record()
            for _ in range(args.launches):
                launch(only)
            ev[1].record()
            torch.cuda.synchronize()
            bwd[only].append(1e3 * ev[0].elapsed_time(ev[1]) / args.launches)
    same = bool(torch.equal(pose6[0].view(torch.int32), pose6[1].view(torch.int32)))
    vis = int((radii > 0).sum().item())
    b_only, b_pose = backward_bytes(P, vis, M)
    med = {k: float(np.median(v)) for k, v in wins.items()}
    us = {"pose_only": float(np.median(bwd[1])), "compact_pose": float(np.median(bwd[0]))}
    out = {"config": args.config, "P": P, "W": W, "H": H, "visible": vis, "iterations": args.iters, "windows": args.windows,
           "ms_per_align_iter": round(med["align_iter"], 4), "ms_per_train_iter": round(med["train_iter"], 4),
           "ms_align_call": round(med["align_call"], 3),
           "backward_us": {k: round(v, 2) for k, v in us.items()},
           "backward_bytes": {"pose_only": b_only, "compact_pose": b_pose},
           "backward_TBps": {"pose_only": round(b_only / us["pose_only"] / 1e6, 3), "compact_pose": round(b_pose / us["compact_pose"] / 1e6, 3)},
           "pose6_bit_identical": same,
           "window_ms": {k: [round(x, 4) for x in v] for k, v in wins.items()},
           "window_backward_us": {("pose_only" if k else "compact_pose"): [round(x, 2) for x in v] for k, v in bwd.items()},
           "card": card()}
    m.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
