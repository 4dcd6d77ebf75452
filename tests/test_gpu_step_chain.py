"""The mapper's step launches its kernels as a chain of programmatic dependent launches: each kernel may start while the one
before it still runs, and waits for it before touching anything it produced.  A wait in the wrong place would let a kernel read
a buffer before its producer wrote it; with every launch serialised by CUDA_LAUNCH_BLOCKING=1 no kernel can overlap another.  The
same deterministic cfg2 training run (scripts/step_parity.py) in both modes must give the same bits: parameters, Adam moments,
losses, visible counts, regrows and the rendered images."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(tmp_path, k, blocking):
    out = tmp_path / ("k%d_%s.npz" % (k, "blocking" if blocking else "chained"))
    env = dict(os.environ)
    env.pop("CUDA_LAUNCH_BLOCKING", None)
    if blocking:
        env["CUDA_LAUNCH_BLOCKING"] = "1"
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.join(ROOT, "scripts", "step_parity.py"), str(out),
                                                                           "--views-per-rank", str(k)]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.returncode, r.stdout[-2000:], r.stderr[-4000:])
    return dict(np.load(out))


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 2])
def test_chained_step_matches_serialised_launches(tmp_path, k):
    a = _run(tmp_path, k, blocking=True)
    b = _run(tmp_path, k, blocking=False)
    assert sorted(a) == sorted(b)
    for key in sorted(a):
        assert a[key].shape == b[key].shape, key
        assert a[key].tobytes() == b[key].tobytes(), key
