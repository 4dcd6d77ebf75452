#!/usr/bin/env python
"""The reference's LPIPS weights for the LPIPS tests and scripts/lpips_bench.py: copies its TorchScript module
(src/lpips/lpips_alex.pt) into oracle/_ref/ and converts it there into the flat weight file glic_lpips reads
(oracle/_ref/lpips_alex.bin, gaussian_lic_b200.lpips_weights; torch on the CPU).  TEST INFRASTRUCTURE ONLY; nothing is compiled.
The ~9.9 MB of weights are derived at build time rather than committed."""
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("GLIC_REFERENCE_ROOT", "/root/reference")
OUT = os.path.join(ROOT, "oracle", "_ref")
PT = os.path.join(OUT, "lpips_alex.pt")
BIN = os.path.join(OUT, "lpips_alex.bin")


def build():
    src = os.path.join(REF, "src", "lpips", "lpips_alex.pt")
    if os.path.isfile(src):
        os.makedirs(OUT, exist_ok=True)
        shutil.copyfile(src, PT)
    if not os.path.isfile(PT):
        return None
    if not os.path.isfile(BIN) or os.path.getmtime(BIN) < os.path.getmtime(PT):
        if ROOT not in sys.path:
            sys.path.insert(0, ROOT)
        from gaussian_lic_b200 import lpips_weights
        tmp = BIN + ".tmp"
        lpips_weights.convert(PT, tmp)
        os.replace(tmp, BIN)
    return BIN


if __name__ == "__main__":
    print("oracle/_ref:", build())
    sys.exit(0)
