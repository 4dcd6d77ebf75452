"""The training and inference forms of render_forward_kernel compile to the same instructions as before the scoring form was
added next to them (tests/golden/render_forward_sass.json): render.cu is compiled here for sm_90a with the library's own flags
and the two forms' SASS is hashed.  Needs no GPU; skipped when nvcc is missing or is not the release the hashes were taken
with (another compiler emits other instructions)."""
import hashlib
import json
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "render_forward_sass.json")


def _forms(obj, cuobjdump):
    out = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    fs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            fs[cur] = []
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4}\*/\s+(.*?);", line)
        if cur and m:
            fs[cur].append(re.sub(r"\s+", " ", m.group(1)))
    res = {}
    for name, ins in fs.items():
        m = re.match(r"_ZN4glic21render_forward_kernelILi([012])EE", name)
        if m:
            res[("train", "infer", "score")[int(m.group(1))]] = (len(ins), hashlib.sha256("\n".join(ins).encode()).hexdigest())
    return res


def test_training_and_inference_forms_keep_their_sass(tmp_path):
    from gaussian_lic_b200 import build
    want = json.load(open(GOLDEN))
    if not os.path.isfile(build.NVCC):
        pytest.skip("nvcc not found")
    version = subprocess.run([build.NVCC, "--version"], capture_output=True, text=True).stdout
    if want["nvcc"] not in version:
        pytest.skip("the hashes were taken with nvcc %s" % want["nvcc"])
    obj = str(tmp_path / "render.o")
    subprocess.run([build.NVCC] + build.NVCC_FLAGS + ["-c", os.path.join(build.CSRC, "render.cu"), "-o", obj], check=True,
                   capture_output=True)
    got = _forms(obj, os.path.join(os.path.dirname(build.NVCC), "cuobjdump"))
    assert set(got) == {"train", "infer", "score"}
    for form in ("train", "infer"):
        assert got[form] == (want[form]["instructions"], want[form]["sha256"]), form
