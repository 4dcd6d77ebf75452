"""Every kernel of ssim.cu that existed before the masked loss and evaluation forms were added compiles to the same instructions
as then (tests/golden/loss_kernels_sass.json): ssim.cu is compiled here for sm_90a with the library's own flags and each
kernel's SASS is hashed, so the unmasked loss, its exposure and fixed-order forms and the evaluation kernels are provably
untouched by the masked forms beside them.  Needs no GPU; skipped when nvcc is missing or is not the release the hashes were
taken with (another compiler emits other instructions)."""
import hashlib
import importlib.util
import json
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "loss_kernels_sass.json")


def _build_module():
    # build.py itself, without importing the package (which needs the built library)
    spec = importlib.util.spec_from_file_location("glic_build_sass", os.path.join(ROOT, "gaussian_lic_b200", "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    return b


def _kernels(obj, cuobjdump):
    out = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    fs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            # the anonymous namespace's tag is derived from the file, not from the code
            cur = re.sub(r"_GLOBAL__N__[0-9a-f]+_\d+_ssim_cu_[0-9a-f]+", "_GLOBAL__N_", m.group(1))
            fs[cur] = []
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4}\*/\s+(.*?);", line)
        if cur and m:
            fs[cur].append(re.sub(r"\s+", " ", m.group(1)))
    return {name: (len(ins), hashlib.sha256("\n".join(ins).encode()).hexdigest()) for name, ins in fs.items()}


def test_unmasked_loss_and_eval_kernels_keep_their_sass(tmp_path):
    build = _build_module()
    want = json.load(open(GOLDEN))
    if not os.path.isfile(build.NVCC):
        pytest.skip("nvcc not found")
    version = subprocess.run([build.NVCC, "--version"], capture_output=True, text=True).stdout
    if want["nvcc"] not in version:
        pytest.skip("the hashes were taken with nvcc %s" % want["nvcc"])
    obj = str(tmp_path / "ssim.o")
    subprocess.run([build.NVCC] + build.NVCC_FLAGS + ["-c", os.path.join(build.CSRC, "ssim.cu"), "-o", obj], check=True,
                   capture_output=True)
    got = _kernels(obj, os.path.join(os.path.dirname(build.NVCC), "cuobjdump"))
    assert len(want["kernels"]) >= 19
    for name, w in want["kernels"].items():
        assert name in got, name
        assert got[name] == (w["instructions"], w["sha256"]), name
    # the masked forms are kernels of their own next to them
    assert any("masked" in n for n in got)
