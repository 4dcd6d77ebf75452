"""Cost of mapper checkpoints (glic_mapper_save_checkpoint / glic_mapper_load_checkpoint).

Two cases at 1920x1080:
  1. a cfg2-sized map (500 k rows, SH degree 3) with 100 add_frame keyframes (8-bit images in the frame store);
  2. 2 M rows with 100 add_keyframe keyframes whose float images are pinned host memory.
For each: the median of --reps saves and of --reps loads into a freshly created mapper, each timed by the host clock around the
call (both end in a device synchronise), the file's bytes and the achieved GB/s.  The load follows a save of the same file, so it
reads from the page cache when the file fits there.  The disk's own rate is measured too: --reps writes of a buffer of the same
size with os.write and fsync.  The checkpoint files are written to --out and removed at the end.

    python scripts/checkpoint_bench.py --out DIR [--reps 3] [--cases 1,2]

Prints one JSON line with the medians, every call and the card name and power limit.  Needs a GPU."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

W, H, FX, FY = 1920, 1080, 1000.0, 1000.0
KEYFRAMES = 100


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power, clock = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def payload_bytes(P, keyframe_bytes):
    """the documented bulk sizes: 712 B per degree-3 row and each keyframe's image (the rest is fixed fields)"""
    return 712 * P + KEYFRAMES * keyframe_bytes


def build(case, np, torch):
    from gaussian_lic_b200 import mapper, synthetic as syn
    P = 500_000 if case == 1 else 2_000_000
    m = mapper.Mapper(W, H, FX, FY, W / 2.0, H / 2.0, sh_degree=3, capacity=P)
    g = syn.make_gaussians(P, W, H, FX, FY, sh_degree=3, seed=7)
    keep = []
    rng = np.random.default_rng(case)
    poses = [syn.orbit_pose(i % 8, radius=2.0) for i in range(KEYFRAMES)]
    if case == 1:
        m.enable_frames(1, 0, 0)
        m.initialize(g)
        bgr = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        for i, (R, t) in enumerate(poses):
            q = _quat(np, R)
            bgr[i % H] ^= 0x5A                                  # every frame differs
            m.add_frame(q, t, bgr, np.zeros((0, 3), np.float32), np.zeros((0, 3), np.uint8))
        return m, P, 3 * W * H, keep
    m.initialize(g)
    imgs = torch.empty((KEYFRAMES, 3, H, W), dtype=torch.float32).pin_memory()
    imgs.uniform_()
    keep.append(imgs)
    for i, (R, t) in enumerate(poses):
        m.add_keyframe(R, t, imgs[i])
    return m, P, 12 * W * H, keep


def _quat(np, R):
    """(x, y, z, w) of a rotation matrix (add_frame's odometry order)"""
    R = np.asarray(R, np.float64)
    w = np.sqrt(max(0.0, 1.0 + R[0, 0] + R[1, 1] + R[2, 2])) / 2
    x = np.copysign(np.sqrt(max(0.0, 1.0 + R[0, 0] - R[1, 1] - R[2, 2])) / 2, R[2, 1] - R[1, 2])
    y = np.copysign(np.sqrt(max(0.0, 1.0 - R[0, 0] + R[1, 1] - R[2, 2])) / 2, R[0, 2] - R[2, 0])
    z = np.copysign(np.sqrt(max(0.0, 1.0 - R[0, 0] - R[1, 1] + R[2, 2])) / 2, R[1, 0] - R[0, 1])
    return np.array([x, y, z, w])


def disk_write(path, nbytes, reps, np):
    buf = np.full(64 << 20, 0xA5, np.uint8)
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fd = os.open(path, os.O_WRONLY | os.O_CREAT | os.O_TRUNC, 0o644)
        left = nbytes
        while left > 0:
            left -= os.write(fd, memoryview(buf)[:min(left, buf.nbytes)])
        os.fsync(fd)
        os.close(fd)
        times.append(time.perf_counter() - t0)
        os.remove(path)
    return times


def run_case(case, args, np, torch):
    from gaussian_lic_b200 import capi, mapper
    m, P, kf_bytes, keep = build(case, np, torch)
    m.synchronize()
    path = os.path.join(args.out, "case%d.ckpt" % case)
    saves, loads = [], []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        m.save_checkpoint(path)
        torch.cuda.synchronize()
        saves.append(time.perf_counter() - t0)
    size = os.path.getsize(path)
    st = m.stats()
    m.close()
    m._keep.clear()                                      # the caller's images are released before the loads
    keep.clear()
    for _ in range(args.reps):
        r = mapper.Mapper.__new__(mapper.Mapper)
        r._create(mapper.checkpoint_config(path))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        capi.check(capi.lib.glic_mapper_load_checkpoint(r._h, path.encode()), "mapper_load_checkpoint")
        torch.cuda.synchronize()
        loads.append(time.perf_counter() - t0)
        assert r.stats().num_gaussians == st.num_gaussians
        r.close()
    disk = disk_write(os.path.join(args.out, "disk.bin"), size, args.reps, np)
    os.remove(path)
    gb = size / 1e9
    return {"case": case, "rows": P, "keyframes": KEYFRAMES, "keyframe_kind": "bgr8 add_frame" if case == 1 else "f32 pinned add_keyframe",
            "file_bytes": size, "documented_payload_bytes": payload_bytes(P, kf_bytes), "save_s": median(saves), "load_s": median(loads),
            "save_GBps": gb / median(saves), "load_GBps": gb / median(loads), "disk_write_fsync_GBps": gb / median(disk),
            "saves": saves, "loads": loads, "disk_writes": disk}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", required=True, help="directory for the checkpoint files (removed at the end)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cases", default="1,2")
    args = ap.parse_args()
    import numpy as np
    import torch
    assert torch.cuda.is_available(), "checkpoint_bench needs a GPU"
    os.makedirs(args.out, exist_ok=True)
    out = {"card": card(), "cases": [run_case(int(c), args, np, torch) for c in args.cases.split(",")]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
