"""Cost of per-keyframe valid-pixel masks (glic_l1_ssim_loss_masked, glic_mapper_set_keyframe_mask).

1. The L1 + D-SSIM loss forward + backward at 1920x1080, masked (a random mask with 40 % of the pixels left out) against
   unmasked, with CUDA events over `--launches` calls per window and the two forms alternating window by window.
2. The cfg2 native iteration (exposure_bench.py's rig: eight pinned keyframes, one view per iteration) with every keyframe
   masked against none; two mappers on the same scene, their timed windows alternating.

    python scripts/mask_bench.py [--launches 200] [--steps 50] [--windows 9] [--config cfg2]

Prints one JSON line with the medians, every window and the card name and power limit.  Needs a GPU; writes nothing."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def loss_windows(args, torch, np):
    from gaussian_lic_b200 import capi
    W, H = 1920, 1080
    rng = np.random.default_rng(0)
    dev = "cuda:0"
    img = torch.as_tensor(rng.uniform(0, 1, (3, H, W)).astype(np.float32)).to(dev)
    gt = torch.as_tensor(rng.uniform(0, 1, (3, H, W)).astype(np.float32)).to(dev)
    valid = torch.as_tensor((rng.uniform(0, 1, (H, W)) < 0.6).astype(np.uint8)).to(dev)
    wpr = capi.lib.glic_mask_words_per_row(W)
    words = torch.empty(H * wpr, dtype=torch.int32, device=dev)
    cnt = torch.empty(1, dtype=torch.int32, device=dev)
    capi.check(capi.lib.glic_pack_mask(H, W, capi.ptr(valid), capi.ptr(words), capi.ptr(cnt), None), "pack_mask")
    torch.cuda.synchronize()
    count = int(cnt.item())
    nb = capi.lib.glic_loss_masked_scratch_bytes(H, W)
    scratch = torch.empty(nb, dtype=torch.uint8, device=dev)
    L = torch.empty(1, device=dev)
    d = torch.empty_like(img)

    def call(masked):
        capi.check(capi.lib.glic_l1_ssim_loss_masked(H, W, 0.2, capi.ptr(img), capi.ptr(gt), None, capi.ptr(words) if masked else None,
                                                     wpr, 0, count, 0, capi.ptr(L), capi.ptr(d), None, capi.ptr(scratch), nb, None),
                   "l1_ssim_loss_masked")

    for masked in (False, True):
        for _ in range(20):
            call(masked)
    wins = {"unmasked": [], "masked": []}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.windows):
        for name in ("unmasked", "masked"):
            torch.cuda.synchronize()
            ev0.record()
            for _ in range(args.launches):
                call(name == "masked")
            ev1.record()
            ev1.synchronize()
            wins[name].append(ev0.elapsed_time(ev1) * 1000.0 / args.launches)
    return wins


def iteration_windows(args, torch, np):
    from gaussian_lic_b200 import mapper as gmapper, synthetic as syn
    P, W, H, fx, fy, cx, cy, deg, _ = syn.CONFIGS[args.config]
    g, _ = syn.make_scene(args.config)
    poses = [syn.orbit_pose(v, radius=0.25) for v in range(8)]
    gt_host = torch.as_tensor(syn.make_gt_image(W, H)).pin_memory()
    rng = np.random.default_rng(1)
    arms = {}
    for name in ("none", "masked"):
        m = gmapper.Mapper(W, H, fx, fy, cx, cy, sh_degree=deg, capacity=P)
        m.initialize(g)
        for k, (R_wc, t_wc) in enumerate(poses):
            m.add_keyframe(R_wc, t_wc, gt_host)
            if name == "masked":
                m.set_mask(True, k, rng.uniform(0, 1, (H, W)) < 0.7)
        m.optimize(list(range(8)) * 2)
        arms[name] = m
    batch = list(range(8))
    reps = (args.steps + 7) // 8
    wins = {"none": [], "masked": []}
    for _ in range(args.windows):
        for name in ("none", "masked"):
            torch.cuda.synchronize()
            st = arms[name].optimize(batch * reps)
            wins[name].append(st.ms_optimize / (8 * reps))
    for m in arms.values():
        m.close()
    return wins, dict(P=P, W=W, H=H, iterations_per_window=8 * reps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="cfg2")
    ap.add_argument("--launches", type=int, default=200, help="loss calls per timed window")
    ap.add_argument("--steps", type=int, default=50, help="iterations per timed window")
    ap.add_argument("--windows", type=int, default=9, help="timed windows per arm (alternating)")
    args = ap.parse_args()
    import numpy as np
    import torch
    from exposure_bench import card
    assert torch.cuda.is_available(), "mask_bench.py needs a GPU"
    lw = loss_windows(args, torch, np)
    iw, shape = iteration_windows(args, torch, np)
    med = lambda v: round(float(np.median(v)), 4)
    out = {"loss_1920x1080_us": {k: med(v) for k, v in lw.items()}, "loss_window_us": {k: [round(x, 2) for x in v] for k, v in lw.items()},
           "config": args.config, **shape, "iter_ms": {k: med(v) for k, v in iw.items()},
           "iter_window_ms": {k: [round(x, 4) for x in v] for k, v in iw.items()}, "card": card()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
