"""Cost of glic_mapper_correct_poses (include/glic_b200.h "Pose corrections").

Maps of 500 k and 2 M rows at SH degree 3, anchored in contiguous blocks to 100 training keyframes (as extend() leaves them),
in two cases: every keyframe corrected (every row moves) and one keyframe corrected (1 % of the rows move).  Each call moves the
listed keyframes alternately to a pose and back, so the map stays where it was between windows.  Reported per case:
  - the call's host-clock time (it drains the pipeline first and synchronises at the end), median over `--calls` calls;
  - the row kernel's device time from torch.profiler (CUDA activity of correct_rows_kernel), median over `--calls` calls, taken
    in a run of its own (a child process of this script) so that the profiler does not disturb the host timing;
  - the bytes of the traffic model, 4 B of anchor per row plus 416 B per moved row (rotation 16, mean 12 and SH rest 180 B,
    each read and written), and that rate's share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s).

    python scripts/pose_correction_bench.py [--calls 20] [--rows 500000,2000000]

Prints one JSON line with the results and the card name and power limit.  Needs a GPU; writes nothing."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

HBM_BYTES_PER_S = 3.35e12
KEYFRAMES = 100


def _rot(axis, angle):
    import numpy as np
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * K @ K


def setup_case(P, n_corrected):
    """a mapper of P rows anchored to KEYFRAMES keyframes, and call(i): correct the first n_corrected keyframes, to the moved
    poses for even i and back for odd i"""
    import numpy as np
    from gaussian_lic_b200 import mapper as gmapper
    W, H, f = 64, 48, 50.0
    rng = np.random.default_rng(0)
    g = dict(means=rng.uniform(-5, 5, (P, 3)).astype(np.float32), dc=rng.normal(size=(P, 3)).astype(np.float32),
             sh=rng.normal(scale=0.1, size=(P, 15, 3)).astype(np.float32), opacity_logits=rng.normal(size=P).astype(np.float32),
             log_scales=np.full((P, 3), -3.0, np.float32), rots=rng.normal(size=(P, 4)).astype(np.float32))
    m = gmapper.Mapper(W, H, f, f, W / 2.0, H / 2.0, sh_degree=3, capacity=P)
    m.initialize(g)
    img = np.zeros((3, H, W), np.float32)
    poses = []
    for k in range(KEYFRAMES):
        R, t = _rot([0.1, 1.0, 0.05 * k], 0.01 * k).astype(np.float32), np.array([0.1 * k, 0.0, 0.0], np.float32)
        m.add_keyframe(R, t, img)
        poses.append((R, t))
    m.set_anchors((np.arange(P, dtype=np.int64) * KEYFRAMES // P).astype(np.int32))
    dR, dt = _rot([0.3, -0.2, 1.0], 0.05), np.array([0.02, -0.01, 0.03])
    moved_poses = [((dR @ R).astype(np.float32), (dR @ t + dt).astype(np.float32)) for R, t in poses]
    listed = list(range(n_corrected))

    def call(i):
        target = moved_poses if i % 2 == 0 else poses
        return m.correct_poses([(True, k, *target[k]) for k in listed])
    return m, call


def kernel_times(P, n_corrected, calls):
    """the profiler run: device ms of every correct_rows_kernel launch of `calls` calls after two warm-up calls"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    m, call = setup_case(P, n_corrected)
    call(0)
    call(1)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(calls):
            call(i)
        torch.cuda.synchronize()
    kern = [e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
            for e in prof.events() if "correct_rows_kernel" in e.name]
    m.close()
    return kern


def run_case(P, n_corrected, calls):
    m, call = setup_case(P, n_corrected)
    moved = call(0)                                  # warm-up (and the module load)
    call(1)
    host = []
    for i in range(calls):
        t0 = time.perf_counter()
        call(i)
        host.append((time.perf_counter() - t0) * 1e3)
    m.close()
    child = subprocess.run([sys.executable, os.path.abspath(__file__), "--kernel-case", "%d,%d" % (P, n_corrected), "--calls", str(calls)],
                           capture_output=True, text=True, check=True)
    kern = json.loads(child.stdout.strip().splitlines()[-1])
    bytes_model = 4 * P + 416 * moved
    k_ms = statistics.median(kern) if kern else float("nan")
    return dict(rows=P, corrected_keyframes=n_corrected, moved_rows=moved, host_ms=statistics.median(host), host_ms_all=host,
                kernel_ms=k_ms, kernel_samples=len(kern), model_bytes=bytes_model, kernel_gb_per_s=bytes_model / (k_ms * 1e-3) / 1e9,
                data_sheet_share=bytes_model / (k_ms * 1e-3) / HBM_BYTES_PER_S)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--rows", default="500000,2000000")
    ap.add_argument("--kernel-case", default=None, help=argparse.SUPPRESS)      # "P,n": the profiler run of one case
    args = ap.parse_args()
    if args.kernel_case:
        P, n = (int(x) for x in args.kernel_case.split(","))
        print(json.dumps(kernel_times(P, n, args.calls)))
        return
    import torch
    from pose_bench import card
    assert torch.cuda.is_available(), "pose_correction_bench.py needs a GPU"
    out = {"card": card(), "cases": []}
    for P in [int(x) for x in args.rows.split(",")]:
        for n in (KEYFRAMES, 1):
            out["cases"].append(run_case(P, n, args.calls))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
