"""Every output of a short bit-reproducible training run of the native mapper, for comparing two builds (or two launch modes) bit
for bit: cfg2 (500 k Gaussians, 1920x1080, SH degree 3), set_deterministic(True), optimiser on, densification off, ITERS
iterations of K views each over eight keyframes whose image is resident in device memory and eight whose image is in pinned
host memory (both load paths), one optimize() call per iteration.  Writes an .npz with the parameters and both Adam moments
after the run, each iteration's loss, visible count and regrow count, and the rendered image, PSNR and SSIM of keyframes 0 and 8.
Usage: python scripts/step_parity.py OUT.npz [--views-per-rank K] [--iters N]"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gaussian_lic_b200 import mapper as gmapper, synthetic as syn  # noqa: E402


def run(k, iters, config="cfg2"):
    P, W, H, fx, fy, cx, cy, deg, zmax = syn.CONFIGS[config]
    g, _ = syn.make_scene(config)
    gt_host = torch.as_tensor(syn.make_gt_image(W, H)).pin_memory()
    gt_dev = gt_host.to("cuda:0")
    mp = gmapper.Mapper(W, H, fx, fy, cx, cy, sh_degree=deg, capacity=P, views_per_rank=k)
    try:
        mp.initialize(g)
        poses = [syn.orbit_pose(v, radius=0.25) for v in range(8)]
        for R_wc, t_wc in poses:
            mp.add_keyframe(R_wc, t_wc, gt_dev)       # keyframes 0..7: image in device memory
        for R_wc, t_wc in poses:
            mp.add_keyframe(R_wc, t_wc, gt_host)      # keyframes 8..15: image in pinned host memory
        mp.set_deterministic(True)
        mp.set_optimizer(True)
        out = {"loss": [], "mean_visible": [], "overflow_regrows": []}
        for it in range(iters):
            batch = [(it + j) % 8 + 8 * ((it + j) % 2) for j in range(k)]
            mp.optimize(batch)
            st = mp.stats()
            out["loss"].append(st.last_loss)
            out["mean_visible"].append(st.mean_visible)
            out["overflow_regrows"].append(st.overflow_regrows)
        out = {kk: np.asarray(v) for kk, v in out.items()}
        for kk, v in mp.download(moments=True).items():
            out["param_" + kk] = v
        for idx in (0, 8):
            out["render_%d" % idx] = mp.render(idx)
            out["eval_%d" % idx] = np.asarray(mp.evaluate(idx), np.float64)
        return out
    finally:
        mp.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--views-per-rank", type=int, default=1)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    out = run(a.views_per_rank, a.iters)
    np.savez(a.out, **out)
    print("wrote %d arrays to %s; last loss %.9g" % (len(out), a.out, float(out["loss"][-1])))


if __name__ == "__main__":
    main()
