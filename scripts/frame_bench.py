"""Cost of 8-bit frame keyframes (glic_mapper_add_frame) against float pinned-host keyframes (glic_mapper_add_keyframe) in
the native mapping iteration at cfg2.

Two native mappers on the same scene run bench.py's mapping_iter_native step: one view per iteration over eight keyframes
at bench.py's rig, optimiser on.  One takes the keyframes as [3,H,W] float32 pinned host images (image H2D on the copy
stream each iteration); the other takes the same images as BGR8 frames through add_frame (select_every_k_frame = 1, no
scan: the map is already initialized), kept in HBM and decoded on the copy stream each iteration.  Their timed windows
alternate in this one call; each window is device time on the mapper's stream over `--steps` iterations.  Also: the
decode kernel alone (CUDA events over `--decode-launches` launches at 1920x1080), the image bytes an iteration moves
host-to-device in each arm, and the device bytes the frame store holds per frame.

    python scripts/frame_bench.py [--steps 50] [--windows 9] [--config cfg2]

Prints one JSON line with the card name and power limit.  Needs a GPU; writes nothing."""
import argparse
import ctypes as C
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


def quat(R):
    """(x, y, z, w) of a rotation matrix"""
    from scipy.spatial.transform import Rotation
    return Rotation.from_matrix(R).as_quat()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="cfg2")
    ap.add_argument("--steps", type=int, default=50, help="iterations per timed window")
    ap.add_argument("--windows", type=int, default=9, help="timed windows per arm (alternating)")
    ap.add_argument("--decode-launches", type=int, default=500)
    args = ap.parse_args()
    import numpy as np
    import torch
    from gaussian_lic_b200 import capi, mapper as gmapper, synthetic as syn
    assert torch.cuda.is_available(), "frame_bench.py needs a GPU"
    P, W, H, fx, fy, cx, cy, deg, _ = syn.CONFIGS[args.config]
    g, _ = syn.make_scene(args.config)
    poses = [syn.orbit_pose(v, radius=0.25) for v in range(8)]               # bench.py's rig
    bgr = np.ascontiguousarray(np.round(syn.make_gt_image(W, H) * 255).astype(np.uint8).transpose(1, 2, 0)[..., ::-1])
    table = np.arange(256, dtype=np.float32) * np.float32(1.0 / 255.0)
    gt_host = torch.as_tensor(np.ascontiguousarray(table[bgr[..., ::-1]].transpose(2, 0, 1))).pin_memory()   # the same image as floats
    no_pts, no_rgb = np.zeros((0, 3), np.float32), np.zeros((0, 3), np.uint8)
    arms = {}
    for name in ("float", "frames"):
        m = gmapper.Mapper(W, H, fx, fy, cx, cy, sh_degree=deg, capacity=P)
        m.initialize(g)
        if name == "float":
            for R_wc, t_wc in poses:
                m.add_keyframe(R_wc, t_wc, gt_host)
        else:
            m.enable_frames(1, 0, 0)
            for R_wc, t_wc in poses:
                assert m.add_frame(quat(R_wc), t_wc, bgr, no_pts, no_rgb)
        m.optimize(list(range(8)) * 2)                                       # warm-up; settles the binning capacity
        arms[name] = m
    same_image = bool(np.array_equal(arms["frames"].keyframe_image(0), gt_host.numpy()))
    batch = list(range(8))
    reps = (args.steps + 7) // 8
    wins = {"float": [], "frames": []}
    for _ in range(args.windows):
        for name in ("float", "frames"):
            torch.cuda.synchronize()
            st = arms[name].optimize(batch * reps)                           # ms_optimize: device time of the whole window
            wins[name].append(st.ms_optimize / (8 * reps))
    med = {k: float(np.median(v)) for k, v in wins.items()}
    spread = {k: float(np.max(v) - np.min(v)) for k, v in wins.items()}
    fst = arms["frames"].frames_get()
    for m in arms.values():
        m.close()
    # the decode kernel alone
    dev_bgr = torch.as_tensor(bgr.reshape(-1), device="cuda:0")
    out = torch.empty(3, H, W, dtype=torch.float32, device="cuda:0")
    launch = lambda: capi.check(capi.lib.glic_decode_bgr8(H, W, C.c_void_p(dev_bgr.data_ptr()), C.c_void_p(out.data_ptr()), None),
                                "decode_bgr8")
    for _ in range(20):
        launch()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(args.decode_launches):
        launch()
    e1.record()
    torch.cuda.synchronize()
    dec_us = 1000.0 * e0.elapsed_time(e1) / args.decode_launches
    moved = 3 * W * H + 12 * W * H                                           # bytes the decode reads and writes
    res = {"config": args.config, "P": P, "W": W, "H": H, "iterations_per_window": 8 * reps, "windows": args.windows,
           "ms_per_iter_float": round(med["float"], 4), "ms_per_iter_frames": round(med["frames"], 4),
           "delta_ms": round(med["frames"] - med["float"], 4), "spread_ms": {k: round(v, 4) for k, v in spread.items()},
           "window_ms": {k: [round(x, 4) for x in v] for k, v in wins.items()},
           "decode_us": round(dec_us, 2), "decode_GBps": round(moved / (dec_us * 1e-6) / 1e9, 1),
           "h2d_image_bytes_per_iter": {"float": 12 * W * H, "frames": 0},
           "device_bytes_per_frame": fst.image_bytes / max(1, fst.frames), "frames_stored": fst.frames,
           "same_image": same_image, "card": card()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
