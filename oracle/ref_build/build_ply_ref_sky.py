#!/usr/bin/env python
"""Build oracle/_ref/ply_ref_sky: the reference's own tinyply (header-only, compiled from /root/reference/src where it lies)
driven like GaussianModel::saveMap on a model with a skybox, with saveMap's exact row counts.  TEST INFRASTRUCTURE ONLY; g++ only,
no GPU, no torch."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("GLIC_REFERENCE_ROOT", "/root/reference")
OUT = os.path.join(ROOT, "oracle", "_ref")


def build():
    exe = os.path.join(OUT, "ply_ref_sky")
    if not os.path.isfile(os.path.join(REF, "src", "tinyply.h")):
        return exe if os.path.isfile(exe) else None
    os.makedirs(OUT, exist_ok=True)
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-w", "-I", os.path.join(REF, "src"),
                           os.path.join(HERE, "ply_ref_sky.cpp"), "-o", exe])
    return exe


if __name__ == "__main__":
    print("oracle/_ref:", build())
    sys.exit(0)
