"""GPU extend() (csrc/extend.cu) against the CPU oracle's restatement of gaussian.cpp:499-638: selection (per-pixel nearest
point, reference tie rule, in-image / positive depth / alpha < 0.99 filter) and initial parameters."""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.mark.parametrize("n,W,H,seed", [(5000, 160, 120, 0), (200_000, 640, 480, 1)])
def test_extend_matches_oracle(oracle32, n, W, H, seed):
    from gaussian_lic_b200 import capi
    lib = capi.lib
    rng = np.random.default_rng(seed)
    fx = fy = 0.6 * W
    cx, cy = W / 2.0, H / 2.0
    pts = np.c_[rng.uniform(-6, 6, n), rng.uniform(-4, 4, n), rng.uniform(-1, 12, n)].astype(np.float32)
    cols = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    rsp = rng.uniform(-0.5, 12, n).astype(np.float32)
    ang = 0.1
    R = np.array([[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]], np.float32)
    t = np.array([0.2, -0.1, 0.3], np.float32)
    T = rng.uniform(0, 0.02, (H, W)).astype(np.float32)
    T[rng.uniform(size=(H, W)) < 0.7] = 1.0
    if n <= 5000:                                            # the O(n^2) oracle
        want = oracle32.extend_select(pts, rsp, R, t, fx, fy, cx, cy, W, H, T)
    else:                                                    # dictionary restatement in float32, same operation order
        pc = (pts[:, 0:1] * R[:, 0] + pts[:, 1:2] * R[:, 1]) + pts[:, 2:3] * R[:, 2] + t
        px = np.floor((pc[:, 0] * np.float32(fx)) / pc[:, 2] + np.float32(cx))
        py = np.floor((pc[:, 1] * np.float32(fy)) / pc[:, 2] + np.float32(cy))
        best = {}
        for i in range(n):
            if not (0 <= px[i] < W and 0 <= py[i] < H):
                continue
            k = (int(px[i]), int(py[i]))
            if k not in best or pc[i, 2] < best[k][1]:
                best[k] = (i, pc[i, 2])
        want = np.array(sorted(i for (x, y), (i, _) in best.items() if rsp[i] > 0 and np.float32(1) - T[y, x] < np.float32(0.99)), np.int32)
    d = lambda a: torch.as_tensor(a).cuda()
    dp, dc_, dr, dT = d(pts), d(cols), d(rsp), d(T)
    ws = torch.empty(lib.glic_extend_bytes(n, W, H), dtype=torch.uint8, device="cuda")
    keep = torch.empty(n, dtype=torch.int32, device="cuda")
    f32 = dict(dtype=torch.float32, device="cuda")
    xyz, fdc, ls, rot, op = torch.empty(n, 3, **f32), torch.empty(n, 3, **f32), torch.empty(n, 3, **f32), torch.empty(n, 4, **f32), torch.empty(n, **f32)
    cnt = C.c_int(0)
    capi.check(lib.glic_extend(n, capi.ptr(dp), capi.ptr(dc_), capi.ptr(dr), R.ctypes.data_as(C.POINTER(C.c_float)),
                               t.ctypes.data_as(C.POINTER(C.c_float)), fx, fy, cx, cy, W, H, capi.ptr(dT), 0.8, capi.ptr(ws),
                               ws.numel(), capi.ptr(keep), capi.ptr(xyz), capi.ptr(fdc), capi.ptr(ls), capi.ptr(rot), capi.ptr(op),
                               C.byref(cnt), None), "extend")
    m = cnt.value
    got = keep[:m].cpu().numpy()
    assert m == len(want) and np.array_equal(got, want)
    init = oracle32.extend_init(want, pts, cols, rsp, 0.8, fx, fy)
    np.testing.assert_array_equal(xyz[:m].cpu().numpy(), init["xyz"])
    np.testing.assert_array_equal(fdc[:m].cpu().numpy(), init["f_dc"])
    np.testing.assert_allclose(ls[:m].cpu().numpy(), init["log_scale"], rtol=2e-6, atol=2e-7)
    np.testing.assert_array_equal(rot[:m].cpu().numpy(), init["rot"])
    np.testing.assert_allclose(op[:m].cpu().numpy(), init["opacity_logit"], rtol=2e-7)
