#!/usr/bin/env python
"""LPIPS pins from the reference's own TorchScript module (src/lpips/lpips_alex.pt, which build() copies to oracle/_ref/ and
converts there into the flat weight file oracle/_ref/lpips_alex.bin; the weights themselves are not committed):

  python tests/golden/make_lpips_golden.py pins [OUT]   -> tests/golden/lpips_pins.npz  (needs a GPU; float64 values)

The pins are the module itself on cuda:0, run in float64 (its parameters and the two images cast to float64), over the seeded
image pairs of PAIRS.  Only the scalars are stored: the images are regenerated from their seeds by make_pair(), which
tests/test_gpu_lpips.py imports.

Why float64 rather than float32 with TF32 off.  The trace recorded every convolution as aten::_convolution with allow_tf32 baked
in as True, so torch.backends.cudnn.allow_tf32 = False changes nothing: as shipped, the module runs its convolutions in TF32.
Rewriting that argument to False (reference_module(allow_tf32=False)) still left the float32 module 2e-5 to 3.5e-4 away from a
float64 CPU restatement on an H100 (torch 2.11), and not even 0 for identical images (up to 1.6e-6), so no float32 run of it
can serve as a 2e-5 yardstick.  In float64 the same module and graph give the network's value itself."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
PT = os.path.join(ROOT, "oracle", "_ref", "lpips_alex.pt")
WEIGHTS = os.path.join(ROOT, "oracle", "_ref", "lpips_alex.bin")
PINS = os.path.join(HERE, "lpips_pins.npz")

SIZES = [(640, 512), (1920, 1080), (31, 31), (333, 197)]           # (W, H)
KINDS = ["identical", "light", "heavy", "unrelated"]
PAIRS = [(W, H, 1000 * i + j, kind) for i, (W, H) in enumerate(SIZES) for j, kind in enumerate(KINDS)]


def _base_image(W, H, rng):
    """smooth colour waves plus a fine texture, in [0,1]"""
    y, x = np.mgrid[0:H, 0:W].astype(np.float64) / max(W, H)
    img = np.empty((3, H, W))
    for c in range(3):
        f = rng.uniform(1.0, 12.0, size=(4, 2))
        ph = rng.uniform(0.0, 2 * np.pi, size=4)
        a = rng.uniform(0.05, 0.2, size=4)
        img[c] = 0.5 + sum(a[i] * np.sin(2 * np.pi * (f[i, 0] * x + f[i, 1] * y) + ph[i]) for i in range(4))
    img += 0.03 * rng.standard_normal(img.shape)
    return np.clip(img, 0.0, 1.0)


def make_pair(W, H, seed, kind):
    """(x, y): two [3,H,W] float32 images in [0,1]; y is x itself, x lightly (0.02) or heavily (0.25) noised, or unrelated"""
    rng = np.random.default_rng(seed)
    x = _base_image(W, H, rng)
    if kind == "identical":
        y = x.copy()
    elif kind == "light":
        y = np.clip(x + 0.02 * rng.standard_normal(x.shape), 0.0, 1.0)
    elif kind == "heavy":
        y = np.clip(x + 0.25 * rng.standard_normal(x.shape), 0.0, 1.0)
    elif kind == "unrelated":
        y = _base_image(W, H, rng)
    else:
        raise ValueError(kind)
    return x.astype(np.float32), y.astype(np.float32)


LAYERS = [(64, 3, 11, 4, 2, True), (192, 64, 5, 1, 2, True), (384, 192, 3, 1, 1, False), (256, 384, 3, 1, 1, False),
          (256, 256, 3, 1, 1, False)]                              # Cout, Cin, k, stride, pad, max pool after the tap


def synthetic_payload(seed):
    """a weight payload of the file's layout with seeded random AlexNet-shaped weights (He-scaled, positive lin weights) and
    the reference's mean / std: exercises every layer of glic_lpips without the reference's weights"""
    rng = np.random.default_rng(seed)
    parts = [np.array([-0.030, -0.088, -0.188, 0.458, 0.448, 0.450])]
    for co, ci, k, _, _, _ in LAYERS:
        parts.append(rng.standard_normal(co * ci * k * k) * np.sqrt(2.0 / (ci * k * k)))
        parts.append(0.05 * rng.standard_normal(co))
    for co, _, _, _, _, _ in LAYERS:
        parts.append(rng.uniform(0.0, 0.2, co))
    return np.concatenate(parts).astype(np.float32)


def lpips64(payload, x, y, device="cuda:0"):
    """the network restated with torch.nn.functional in float64 from a flat payload (x, y: [3,H,W] arrays)"""
    import torch
    import torch.nn.functional as F
    p = torch.from_numpy(np.asarray(payload, np.float64)).to(device)
    mean, std = p[0:3].view(1, 3, 1, 1), p[3:6].view(1, 3, 1, 1)
    off, convs = 6, []
    for co, ci, k, s, pad, pool in LAYERS:
        w = p[off:off + co * ci * k * k].view(co, ci, k, k)
        off += co * ci * k * k
        convs.append((w, p[off:off + co], s, pad, pool))
        off += co
    lins = []
    for co, _, _, _, _, _ in LAYERS:
        lins.append(p[off:off + co].view(1, co, 1, 1))
        off += co

    def taps(img):
        t = (torch.from_numpy(np.asarray(img, np.float64)).to(device)[None].clamp(0, 1) - mean) / std
        out = []
        for w, b, s, pad, pool in convs:
            t = F.relu(F.conv2d(t, w, b, stride=s, padding=pad))
            out.append(t / (torch.sqrt((t * t).sum(1, keepdim=True)) + 1e-10))
            if pool:
                t = F.max_pool2d(t, 3, 2)
        return out

    return float(sum(((a - b) ** 2 * l).sum(1).mean() for a, b, l in zip(taps(x), taps(y), lins)))


def reference_module(pt=PT, allow_tf32=False):
    """the TorchScript module on cuda:0: TF32 off (allow_tf32 = False: both backend switches off and the traced convolutions'
    allow_tf32 argument set to False), or exactly as traced (None: its convolutions run in TF32)"""
    import torch
    m = torch.jit.load(pt, map_location="cuda:0").eval()
    if allow_tf32 is None:
        return m
    torch.backends.cudnn.allow_tf32 = allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = allow_tf32
    for _, sub in m.named_modules():
        try:
            g = sub.graph
        except RuntimeError:
            continue
        for node in g.findAllNodes("aten::_convolution"):
            c = g.insertConstant(bool(allow_tf32))
            c.node().moveBefore(node)
            node.replaceInput(12, c)          # _convolution(..., benchmark, deterministic, cudnn_enabled, allow_tf32)
    return m


def reference_module64(pt=PT):
    """the TorchScript module on cuda:0 with its parameters in float64 (its mean / std buffers are cast back to float32 by the
    graph itself, which promotes to float64 against a float64 image)"""
    import torch
    return torch.jit.load(pt, map_location="cuda:0").eval().double()


def reference_lpips(module, x, y, dtype=None):
    import torch
    with torch.no_grad():
        tx = torch.from_numpy(x).cuda()[None].clamp(0, 1)
        ty = torch.from_numpy(y).cuda()[None].clamp(0, 1)
        if dtype is not None:
            tx, ty = tx.to(dtype), ty.to(dtype)
        return float(module(tx, ty).item())


def main(argv):
    sys.path.insert(0, ROOT)
    what = argv[1] if len(argv) > 1 else ""
    if what == "pins":
        import torch
        out = argv[2] if len(argv) > 2 else PINS
        m = reference_module64()
        vals = np.array([reference_lpips(m, *make_pair(W, H, seed, kind), dtype=torch.float64) for W, H, seed, kind in PAIRS],
                        np.float64)
        np.savez(out, W=np.array([p[0] for p in PAIRS]), H=np.array([p[1] for p in PAIRS]), seed=np.array([p[2] for p in PAIRS]),
                 kind=np.array([p[3] for p in PAIRS]), lpips=vals, device=np.array(torch.cuda.get_device_name(0)),
                 torch_version=np.array(torch.__version__))
        for p, v in zip(PAIRS, vals):
            print(p, "%.8f" % v)
        print("wrote", out)
    else:
        sys.exit(__doc__)


if __name__ == "__main__":
    main(sys.argv)
