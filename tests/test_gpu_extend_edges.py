"""glic_extend (csrc/extend.cu) at the selection edges random scenes never reach, compared bit for bit with the exact NumPy
restatement (tests/extend_oracle.py): pixel borders, depth ties, negative and non-finite projections, the filters at their
thresholds, one pixel under a million points, a point on every pixel of a 1920 x 1080 frame, the single-CTA scan across
its 1024-point chunks, degenerate frame shapes and the error contract.

The reference computes the same selection with torch tensor ops on the device (gaussian.cpp:499-631), so torch itself is
the reference's arithmetic here:
  * camera coordinates: torch.matmul(points, R_cw^T) + t with TF32 off is not one fixed operation order on an H100 (the
    uncontracted order extend_pixel uses for n <= 16, an fma chain for n >= 17).  Torch's camera coordinates must be within
    rounding (8 ulps of the sum of the terms' magnitudes) of the kernel's, every point that changes pixel under them has a
    border between its two pixel coordinates, and every changed win on an unmoved point is a depth tie within that
    rounding or is decided by a point that changed pixel.  The counts are printed per case, with how many of the moved
    points lie within 4 ulps of a border and how many changed wins are within 4 ulps of their winner's depth;
  * floor().to(int32) saturates +-inf and maps NaN to 0 (see extend_pixel);
  * the initial rows are torch's ops, bit for bit.
"""
import ctypes as C

import numpy as np
import pytest

import extend_oracle as eo

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

F32 = np.float32
SS = 0.8                                          # scaling_scale
SENTINEL = np.array([0x7FBADBAD], np.uint32).view(F32)[0]   # a NaN payload no kernel writes
C0 = 0.28209479177387814
ULPS = 4
ROUND_ULPS = 8


@pytest.fixture(autouse=True)
def _ieee_matmul():
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False        # the reference's default
    yield
    torch.backends.cuda.matmul.allow_tf32 = old


def _lib():
    from gaussian_lic_b200 import capi
    return capi


def _fptr(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _run(pts, cols, rsp, R, t, fx, fy, cx, cy, W, H, T, ws_bytes=None, rot_shift=0, null=None, count_init=-5):
    """glic_extend on sentinel-filled outputs -> (status, count, keep [n], rows dict of [n, .] numpy arrays)"""
    capi = _lib()
    n = pts.shape[0]
    dev = "cuda"
    d = lambda a: torch.as_tensor(np.ascontiguousarray(a, F32)).to(dev)
    dp, dc, dr, dT = d(pts.reshape(-1, 3)), d(cols.reshape(-1, 3)), d(rsp.reshape(-1)), d(T.reshape(-1))
    need = capi.lib.glic_extend_bytes(n, W, H)
    ws = torch.zeros(max(need if ws_bytes is None else ws_bytes, 1), dtype=torch.uint8, device=dev)
    keep = torch.full((max(n, 1),), -7, dtype=torch.int32, device=dev)
    outs = {k: torch.from_numpy(np.full(max(n, 1) * w + 4, SENTINEL, F32)).to(dev)
            for k, w in (("xyz", 3), ("f_dc", 3), ("log_scale", 3), ("rot", 4), ("opacity", 1))}
    ptrs = dict(points=capi.ptr(dp), colors=capi.ptr(dc), depth=capi.ptr(dr), T=capi.ptr(dT))
    if null:
        ptrs[null] = None
    rot_ptr = C.c_void_p(outs["rot"].data_ptr() + rot_shift)
    cnt = C.c_int(count_init)
    Rh, th = np.ascontiguousarray(R, F32).reshape(9), np.ascontiguousarray(t, F32).reshape(3)
    st = capi.lib.glic_extend(n, ptrs["points"], ptrs["colors"], ptrs["depth"], _fptr(Rh), _fptr(th), float(fx), float(fy),
                              float(cx), float(cy), W, H, ptrs["T"], SS, capi.ptr(ws), ws.numel() if ws_bytes is None else ws_bytes,
                              capi.ptr(keep), capi.ptr(outs["xyz"]), capi.ptr(outs["f_dc"]), capi.ptr(outs["log_scale"]), rot_ptr,
                              capi.ptr(outs["opacity"]), C.byref(cnt), None)
    torch.cuda.synchronize()
    rows = {k: v.cpu().numpy() for k, v in outs.items()}
    return st, cnt.value, keep.cpu().numpy()[:n], rows


def _bits(a):
    return np.ascontiguousarray(a, F32).view(np.uint32)


def torch_init(keep, pts, cols, rsp, fx, fy, ss=SS):
    """The reference's initial rows (gaussian.cpp:613-626) with torch on the device"""
    k = torch.as_tensor(np.asarray(keep, np.int64)).cuda()
    c = torch.as_tensor(np.ascontiguousarray(cols, F32)).cuda().index_select(0, k)
    d = torch.as_tensor(np.ascontiguousarray(rsp, F32)).cuda().index_select(0, k)
    focal = float(F32((F32(fx) + F32(fy)) / 2.0))
    f_dc = (c - 0.5) / C0
    ls = torch.log(ss * d / focal).unsqueeze(1).repeat(1, 3)
    x = 0.1 * torch.ones(k.numel(), 1, dtype=torch.float32, device="cuda")
    op = torch.log(x / (1 - x)).reshape(-1)
    return dict(f_dc=f_dc.cpu().numpy(), log_scale=ls.cpu().numpy(), opacity=op.cpu().numpy())


def check(pts, cols, rsp, R, t, fx, fy, cx, cy, W, H, T, what=""):
    """glic_extend against the restatement: count, survivors, every init row bit for bit, untouched rows past count"""
    sel = eo.select(pts, rsp, R, t, fx, fy, cx, cy, W, H, T)
    st, m, keep, rows = _run(pts, cols, rsp, R, t, fx, fy, cx, cy, W, H, T)
    assert st == 0, what
    want = sel["keep"]
    assert m == want.size, (what, m, want.size)
    assert np.array_equal(keep[:m], want), what
    assert np.all(keep[m:] == -7), what
    n = pts.shape[0]
    ref = torch_init(want, pts, cols, rsp, fx, fy)
    assert np.array_equal(_bits(rows["xyz"][:3 * m]), _bits(pts[want].reshape(-1))), what
    assert np.array_equal(_bits(rows["rot"][:4 * m]), _bits(np.tile([1, 0, 0, 0], m))), what
    for k, w in (("f_dc", 3), ("log_scale", 3), ("opacity", 1)):
        assert np.array_equal(_bits(rows[k][:w * m]), _bits(ref[k].reshape(-1))), (what, k)
    for k, w in (("xyz", 3), ("f_dc", 3), ("log_scale", 3), ("rot", 4), ("opacity", 1)):
        assert np.all(_bits(rows[k][w * m:]) == _bits(SENTINEL)), (what, k)
    if m:                                             # float64 yardstick only
        g = rows["log_scale"][:3 * m:3].astype(np.float64)
        e = np.abs(g - np.log(SS * rsp[want].astype(np.float64) / ((float(fx) + float(fy)) / 2))).max()
        print("%s: n=%d kept=%d, log-scale vs float64 max |err| %.2e" % (what, n, m, e))
    return sel


# ---- step 3: torch's device arithmetic -----------------------------------------------------------------------------------------
def torch_coords(pts, R, t, fx, fy, cx, cy):
    """the reference's expressions on the device: camera coordinates, float pixel coordinates, floor().to(int32)"""
    p = torch.as_tensor(np.ascontiguousarray(pts, F32)).cuda()
    Rt = torch.as_tensor(np.ascontiguousarray(R, F32)).cuda()
    tt = torch.as_tensor(np.ascontiguousarray(t, F32)).cuda()
    pc = torch.matmul(p, Rt.t()) + tt.view(1, 3)
    z = pc[:, 2]
    x = (pc[:, 0] * float(fx)) / z + float(cx)
    y = (pc[:, 1] * float(fy)) / z + float(cy)
    ix, iy = x.floor().to(torch.int32), y.floor().to(torch.int32)
    return pc.cpu().numpy(), x.cpu().numpy(), y.cpu().numpy(), ix.cpu().numpy(), iy.cpu().numpy()


def _same(a, b):
    """bit for bit, any NaN matching any NaN"""
    a, b = np.ascontiguousarray(a, F32), np.ascontiguousarray(b, F32)
    return bool(np.all((_bits(a) == _bits(b)) | (np.isnan(a) & np.isnan(b))))


def _ordered(a):
    b = np.ascontiguousarray(a, F32).view(np.int32).astype(np.int64)
    return np.where(b < 0, -(b & 0x7FFFFFFF), b)


def _ulps(a, b):
    return np.abs(_ordered(a) - _ordered(b))


def _near_border(v):
    with np.errstate(invalid="ignore"):
        r = np.round(v).astype(F32)
        return np.isfinite(v) & (_ulps(v, r) <= ULPS)


def compare_torch(pts, rsp, R, t, fx, fy, cx, cy, W, H, T, sel, what):
    """Torch's coordinates against the restatement's, and the selection they imply against the kernel's -> disagreements"""
    pc, x, y, ix, iy = torch_coords(pts, R, t, fx, fy, cx, cy)
    sel_t = eo.select(pts, rsp, R, t, fx, fy, cx, cy, W, H, T, cam=pc)
    assert _same(sel_t["xf"], x) and _same(sel_t["yf"], y), what
    fin = np.isfinite(x) & (np.abs(x) < 2 ** 31)                    # floor().to(int32) is floor where it fits
    assert np.array_equal(ix[fin], np.floor(x[fin]).astype(np.int64)), what
    diff_cam = int((_bits(pc) != _bits(sel["cam"])).any(1).sum())
    # the two operation orders differ by rounding alone: each of them is within 4 u S of the exact R p + t, S the sum of
    # the terms' magnitudes (u = 2^-24), so they are within 8 ulps of S of each other
    p, Rf, tf = np.asarray(pts, F32).reshape(-1, 3), np.asarray(R, F32), np.asarray(t, F32)
    with np.errstate(all="ignore"):
        S = np.abs(p.astype(np.float64)[:, None, :] * Rf[None]).sum(2) + np.abs(tf)[None]
        bound = ROUND_ULPS * np.spacing(S.astype(F32)).astype(np.float64)
        dc = np.abs(pc.astype(np.float64) - sel["cam"].astype(np.float64))
    ok = (dc <= bound) | (np.isnan(pc) & np.isnan(sel["cam"])) | (pc == sel["cam"])
    assert ok.all(), (what, np.flatnonzero(~ok.all(1))[:10])
    moved = (sel["in_image"] != sel_t["in_image"]) | (sel["px"] != sel_t["px"]) | (sel["py"] != sel_t["py"])
    won = sel["winner"] != sel_t["winner"]
    # a point on another pixel has an integer between its two pixel coordinates; it is counted as near a border when
    # torch's coordinate is within ULPS ulps of it (cancellation in R p + t, amplified by f / z, can move it farther)
    between = np.zeros(len(p), bool)
    with np.errstate(invalid="ignore"):
        for a_, b_ in ((sel["xf"], x), (sel["yf"], y)):
            between |= np.floor(a_) != np.floor(b_)
    assert np.all(between[moved] | ~np.isfinite(x[moved]) | ~np.isfinite(y[moved])), what
    border = _near_border(x) | _near_border(y)
    # a changed win on a point that kept its pixel: its depth and its pixel winner's are within their rounding bounds, or a
    # point that crossed a border into or out of that pixel decided it
    key = np.where(sel["in_image"], sel["py"] * W + sel["px"], -1)
    key_t = np.where(sel_t["in_image"], sel_t["py"] * W + sel_t["px"], -1)
    wk = np.full(W * H, -1, np.int64)
    wk[key[sel["winner"]]] = np.flatnonzero(sel["winner"])
    wt = np.full(W * H, -1, np.int64)
    wt[key_t[sel_t["winner"]]] = np.flatnonzero(sel_t["winner"])
    cand = np.flatnonzero(won & ~moved)
    kk = key[cand]
    tie = np.zeros(cand.size, bool)
    tie4 = np.zeros(cand.size, bool)
    bz = bound[:, 2]
    for w in (wk[kk], wt[kk]):
        tie |= np.abs(pc[cand, 2].astype(np.float64) - pc[w, 2]) <= bz[cand] + bz[w]
        tie4 |= (_ulps(pc[cand, 2], pc[w, 2]) <= ULPS) | (_ulps(sel["cam"][cand, 2], sel["cam"][w, 2]) <= ULPS)
    touched = np.isin(kk, np.r_[key[moved], key_t[moved]])
    bad = cand[~(tie | touched)]
    assert bad.size == 0, (what, bad[:10])
    keep_diff = np.setxor1d(sel["keep"], sel_t["keep"]).size
    print("%s: n=%d camera coords differing from torch's: %d; pixel moved: %d (%d within %d ulps of a border); win changed "
          "on a kept pixel: %d (%d depth ties within %d ulps, %d decided by a moved point); survivors differing: %d"
          % (what, pts.shape[0], diff_cam, int(moved.sum()), int((moved & border).sum()), ULPS, cand.size, int(tie4.sum()), ULPS,
             int((touched & ~tie).sum()), keep_diff))
    return sel_t, diff_cam


# ---- scenes --------------------------------------------------------------------------------------------------------------------
def _rot(rng):
    q = rng.normal(size=4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _scene(n, W, H, seed, behind=0.1):
    """LiDAR-like points in front of (and some behind) a rotated, translated camera with an off-centre principal point"""
    rng = np.random.default_rng(seed)
    fx, fy = F32(0.6 * W + 0.37), F32(0.61 * W - 0.21)
    cx, cy = F32(W * 0.47 + 0.31), F32(H * 0.53 - 0.17)
    z = rng.uniform(0.5, 40, n)
    z[rng.uniform(size=n) < behind] *= -0.3
    u, v = rng.uniform(-0.1 * W, 1.1 * W, n), rng.uniform(-0.1 * H, 1.1 * H, n)
    cam = np.c_[(u - cx) * z / fx, (v - cy) * z / fy, z]
    R = _rot(rng)
    t = rng.uniform(-5, 5, 3)
    pts = ((cam - t) @ R).astype(F32)                              # R^T (cam - t), rows
    cols = rng.uniform(0, 1, (n, 3)).astype(F32)
    rsp = np.abs(z).astype(F32) * F32(1.01)
    rsp[rng.uniform(size=n) < 0.03] = -1.0
    T = rng.uniform(0, 0.03, (H, W)).astype(F32)
    T[rng.uniform(size=(H, W)) < 0.6] = 1.0
    return pts, cols, rsp, R.astype(F32), t.astype(F32), fx, fy, cx, cy, T


@pytest.mark.parametrize("n", [1, 16, 17, 1023, 1024, 1025, 200_000, (1 << 20) + 1])
def test_random_scenes_and_torch_arithmetic(n):
    W, H = 640, 480
    pts, cols, rsp, R, t, fx, fy, cx, cy, T = _scene(n, W, H, n % 1000 + 3)
    sel = check(pts, cols, rsp, R, t, fx, fy, cx, cy, W, H, T, "random n=%d" % n)
    if n >= 1024:
        assert (sel["cam"][sel["keep"], 2] < 0).any()            # behind-camera points are inserted (reference behaviour)
    compare_torch(pts, rsp, R, t, fx, fy, cx, cy, W, H, T, sel, "random n=%d" % n)


def _rz_rx(a, b):
    ca, sa, cb, sb = np.cos(a), np.sin(a), np.cos(b), np.sin(b)
    Rz = np.array([[cb, -sb, 0], [sb, cb, 0], [0, 0, 1]])
    Rx = np.array([[1, 0, 0], [0, ca, -sa], [0, sa, ca]])
    Ry = np.array([[ca, 0, sa], [0, 1, 0], [-sa, 0, ca]])
    return (Rz @ Rx).astype(F32), (Rz @ Ry).astype(F32)


def _from_ordered(k):
    """the float32 whose _ordered value is k"""
    k = int(k)
    b = k if k >= 0 else (-k) | 0x80000000
    return np.array([b & 0xFFFFFFFF], np.uint32).view(F32)[0]


def _land(axis, target, base, R, t, fx, fy, cx, cy):
    """(point_hi, point_lo): base with world coordinate `axis` set to the smallest float32 whose pixel coordinate on `axis`
    is >= target, and to the largest one below it, found by bisection over the float32 values in order.  The rotations used
    leave the camera depth independent of that coordinate (R[2, axis] = 0) and increase the camera coordinate with it
    (R[axis, axis] > 0), so the pixel coordinate is monotone in it."""
    assert R[2, axis] == 0 and R[axis, axis] > 0

    def coord(v):
        p = base.copy()
        p[axis] = v
        xf, yf = eo.pixel_coords(eo.camera_coords(p, R, t), fx, fy, cx, cy)
        return (xf if axis == 0 else yf)[0]
    lo, hi = (int(_ordered(F32(v))[0]) for v in (base[axis] - 1e3, base[axis] + 1e3))
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if coord(_from_ordered(mid)) >= target:
            hi = mid
        else:
            lo = mid
    a, b = base.copy(), base.copy()
    a[axis], b[axis] = _from_ordered(hi), _from_ordered(lo)
    assert coord(a[axis]) >= target > coord(b[axis])
    return a, b


def test_pixel_borders():
    """Projections exactly on k, on the reachable values on either side of k, at 0, W and H, with an off-centre principal
    point and rotations whose rows mix all three coordinates; plus (identity pose, principal point 0) one ulp below 0, W
    and H, a -0.0 coordinate, and exactly W and H."""
    W, H = 640, 480
    fx, fy, cx, cy = F32(383.7), F32(384.9), F32(317.23), F32(243.61)
    Rx, Ry = _rz_rx(0.3, 0.2)
    t = np.array([0.31, -0.17, 0.42], F32)
    rng = np.random.default_rng(4)
    pts = []
    landed = []
    for axis, R, lim in ((0, Rx, W), (1, Ry, H)):
        for k in (0, 1, 317, 318, 243, 244, lim - 1, lim):
            for _ in range(2):
                for attempt in range(40):
                    z = rng.uniform(1, 30)
                    base = np.linalg.solve(R.astype(np.float64), np.array([0.1 * z, -0.05 * z, z]) - t).astype(F32)
                    hi, lo = _land(axis, F32(k), base, R, t, fx, fy, cx, cy)
                    xf, yf = eo.pixel_coords(eo.camera_coords(hi, R, t), fx, fy, cx, cy)
                    if (xf if axis == 0 else yf)[0] == k:
                        break
                else:
                    pytest.fail("no float32 point projects exactly onto %d" % k)
                pts.append((hi, R))
                pts.append((lo, R))
    # one scene per rotation
    for R in (Rx, Ry):
        P = np.array([p for p, r in pts if r is R], F32)
        n = P.shape[0]
        xf, yf = eo.pixel_coords(eo.camera_coords(P, R, t), fx, fy, cx, cy)
        landed.append(int(np.sum(np.isin(np.r_[xf, yf], np.arange(0, W + 1, dtype=F32)))))
        print("borders: %d of %d coordinates exactly on an integer" % (landed[-1], 2 * n))
        cols = rng.uniform(0, 1, (n, 3)).astype(F32)
        rsp = np.ones(n, F32)
        T = np.ones((H, W), F32)
        sel = check(P, cols, rsp, R, t, fx, fy, cx, cy, W, H, T, "borders")
        compare_torch(P, rsp, R, t, fx, fy, cx, cy, W, H, T, sel, "borders")
    assert min(landed) >= 16                                    # the construction put points exactly on integer borders
    # exact float32 neighbours of 0 and W: identity pose, principal point 0, power-of-two focal and depth
    tiny = np.nextafter(F32(0), F32(1))
    W2, H2 = 8, 6
    P = np.array([[1, 1, 2], [1, 1, 2], [0, 1, 2], [-tiny, 1, 4], [np.nextafter(F32(W2), F32(0)), 1, 4], [W2, 1, 4],
                  [-1.5, -1, -2], [1.5, 1, 2], [1, H2, 4], [1, np.nextafter(F32(H2), F32(0)), 4], [-0.0, 3, 4]], F32)
    sel = check(P, np.full((len(P), 3), 0.25, F32), np.ones(len(P), F32), np.eye(3, dtype=F32), np.zeros(3, F32), 4.0, 4.0, 0.0,
                0.0, W2, H2, np.ones((H2, W2), F32), "borders at 0 / W")
    assert sel["in_image"].tolist() == [True, True, True, False, True, False, True, True, False, True, True]
    assert sel["keep"].tolist() == [0, 2, 4, 6, 9, 10]


def test_depth_ties_and_negative_depths():
    """Several points with bit-identical camera depth on one pixel, in both index orders; behind-camera points winning their
    pixels and inserted when depth_rsp > 0."""
    rng = np.random.default_rng(8)
    W, H = 320, 240
    fx, fy, cx, cy = F32(251.3), F32(249.7), F32(161.4), F32(118.9)
    R, t = _rot(rng).astype(F32), np.array([0.5, -0.25, 1.5], F32)
    groups = []
    for g in range(60):
        z = rng.uniform(1.0, 20.0) * (-1 if g % 4 == 0 else 1)
        cam = np.array([rng.uniform(-0.3, 0.3) * z, rng.uniform(-0.3, 0.3) * z, z])
        base = ((cam - t) @ R.astype(np.float64)).astype(F32)
        # neighbours one ulp away in any coordinate: many share the pixel and the depth bits
        steps = rng.integers(-1, 2, (400, 3))
        cand = np.unique(np.nextafter(base, (base + steps).astype(F32)), axis=0)
        s = eo.select(cand, np.ones(len(cand), F32), R, t, fx, fy, cx, cy, W, H, np.ones((H, W), F32))
        zb = _bits(s["cam"][:, 2])
        key = s["py"] * W + s["px"]
        _, inv, cnt = np.unique(np.c_[key, zb], axis=0, return_inverse=True, return_counts=True)
        best = np.flatnonzero(cnt.reshape(-1)[inv.reshape(-1)] >= 3)
        if best.size and s["in_image"][best[0]]:
            members = best[(key[best] == key[best[0]]) & (zb[best] == zb[best[0]])][:5]
            groups.append(cand[members])
    assert len(groups) >= 30
    P = np.concatenate(groups)
    P = P[rng.permutation(len(P))]
    for order in (P, P[::-1].copy()):
        n = len(order)
        cols = rng.uniform(0, 1, (n, 3)).astype(F32)
        rsp = np.full(n, 2.0, F32)
        T = np.ones((H, W), F32)
        sel = check(order, cols, rsp, R, t, fx, fy, cx, cy, W, H, T, "ties")
        zc = sel["cam"][:, 2]
        key = sel["py"] * W + sel["px"]
        for i in sel["keep"]:                                  # the winner is the smallest index of its tied group
            same = np.flatnonzero((key == key[i]) & (zc == zc[i]))
            assert i == same.min() and same.size >= 2
        assert (zc[sel["keep"]] < 0).any() and (zc[sel["keep"]] > 0).any()
        compare_torch(order, rsp, R, t, fx, fy, cx, cy, W, H, T, sel, "ties")


def test_filters_at_their_thresholds():
    """depth_rsp 0.0 / -0.0 / smallest subnormal, and 1 - T exactly 0.99f and one ulp either side, T = 1 and T = 0, on the
    pixels of winners"""
    W, H = 256, 192
    pts, cols, rsp, R, t, fx, fy, cx, cy, T = _scene(30000, W, H, 12, behind=0.0)
    base = eo.select(pts, np.ones(len(pts), F32), R, t, fx, fy, cx, cy, W, H, np.ones((H, W), F32))
    win = np.flatnonzero(base["winner"])
    tiny = np.nextafter(F32(0), F32(1))
    a = np.array([np.nextafter(F32(0.99), F32(0)), F32(0.99), np.nextafter(F32(0.99), F32(1))], F32)
    T_thr = F32(1) - a
    assert np.array_equal(F32(1) - T_thr, a)
    rsp = np.ones(len(pts), F32)
    rsp[win[0::8]] = 0.0
    rsp[win[1::8]] = -0.0
    rsp[win[2::8]] = tiny
    T = np.ones((H, W), F32)
    for j, Tv in enumerate([T_thr[0], T_thr[1], T_thr[2], F32(0), F32(1)]):
        w = win[3 + j::8]
        T[base["py"][w], base["px"][w]] = Tv
    sel = check(pts, cols, rsp, R, t, fx, fy, cx, cy, W, H, T, "thresholds")
    k = set(sel["keep"].tolist())
    assert not k & set(win[0::8]) and not k & set(win[1::8]) and set(win[2::8]) <= k
    assert set(win[3::8]) <= k and set(win[7::8]) <= k                         # alpha one ulp below 0.99f, T = 1
    assert not k & (set(win[4::8]) | set(win[5::8]) | set(win[6::8]))          # alpha 0.99f, one ulp above, 1
    compare_torch(pts, rsp, R, t, fx, fy, cx, cy, W, H, T, sel, "thresholds")


def test_non_finite_projections():
    """z = +-0, z = +-inf and NaN coordinates: the kernel rejects every non-finite projection; a real point behind a NaN one
    keeps its pixel.  Torch's floor().to(int32) on the same coordinates: +-inf saturate (outside), NaN becomes 0."""
    W, H = 64, 48
    fx, fy, cx, cy = 50.0, 50.0, 32.5, 24.5
    R, t = np.eye(3, dtype=F32), np.zeros(3, F32)
    big = F32(3e38)
    nan = np.nan
    P = np.array([[1, 1, 0], [0, 0, 0], [-1, -1, -0.0], [0, 0, -0.0],           # z = 0: +-inf or NaN
                  [nan, 0, 1], [0, nan, 1], [0, 0, nan], [nan, nan, nan],        # NaN coordinates
                  [-0.64, -0.48, 1.0],                                           # a real point on pixel (0, 0)
                  [0.0, 0.0, 2.0]], F32)                                         # a real point on the principal point
    T = np.ones((H, W), F32)
    rsp = np.ones(len(P), F32)
    sel = check(P, np.full((len(P), 3), 0.5, F32), rsp, R, t, fx, fy, cx, cy, W, H, T, "non-finite")
    assert sel["in_image"][:8].sum() == 0 and sel["keep"].tolist() == [8, 9]
    _, x, y, ix, iy = torch_coords(P, R, t, fx, fy, cx, cy)
    nan_rows = [1, 3, 4, 5, 6, 7]                                 # 0/0 and NaN inputs (NaN * 0 spreads through the matmul)
    assert np.all(np.isnan(x[nan_rows])) and np.all(ix[nan_rows] == 0)                # NaN -> 0: column 0 in torch
    assert ix[0] == np.iinfo(np.int32).max and ix[2] == np.iinfo(np.int32).min           # +-inf saturate
    assert iy[0] == np.iinfo(np.int32).max and iy[2] == np.iinfo(np.int32).min
    # z = +-inf (R scales z by 2 so that 1.7e38 overflows): x / +-inf = +-0 puts the points on the principal point with an
    # infinite depth, where -inf wins
    Q = np.array([[0.0, 0.0, big], [0.0, 0.0, -big], [0.0, 0.0, 2.0], [0.0, 0.0, big]], F32)
    Rq = np.diag([1.0, 1.0, 2.0]).astype(F32)
    rq = np.ones(len(Q), F32)
    sel = check(Q, np.full((len(Q), 3), 0.5, F32), rq, Rq, t, fx, fy, cx, cy, W, H, T, "infinite depth")
    z = sel["cam"][:, 2]
    assert np.isposinf(z[0]) and np.isneginf(z[1]) and z[2] == 4 and sel["in_image"].all()
    assert sel["keep"].tolist() == [1]
    compare_torch(Q, rq, Rq, t, fx, fy, cx, cy, W, H, T, sel, "infinite depth")


def test_one_pixel_under_a_million_points():
    n = 1_000_000
    W, H = 64, 48
    rng = np.random.default_rng(3)
    R, t = np.eye(3, dtype=F32), np.zeros(3, F32)
    fx, fy, cx, cy = F32(40.0), F32(40.0), F32(20.5), F32(30.5)
    z = rng.uniform(1.0, 50.0, n).astype(F32)
    z[[600_001, 777_777, 999_998]] = F32(0.5)                     # planted minimum, tied three times
    z[[5, 123_456]] = F32(0.5000001)
    P = np.c_[np.zeros(n), np.zeros(n), z].astype(F32)             # all on pixel (20, 30)
    cols = rng.uniform(0, 1, (n, 3)).astype(F32)
    sel = check(P, cols, np.ones(n, F32), R, t, fx, fy, cx, cy, W, H, np.ones((H, W), F32), "one pixel")
    assert sel["keep"].tolist() == [600_001]
    P[600_001, 2] = F32(0.75)
    sel = check(P, cols, np.ones(n, F32), R, t, fx, fy, cx, cy, W, H, np.ones((H, W), F32), "one pixel, tie")
    assert sel["keep"].tolist() == [777_777]


def _grid_scene(W, H, n, seed):
    """n points on n distinct pixels of a W x H frame (pixel centres), under a general rotation"""
    rng = np.random.default_rng(seed)
    fx, fy = F32(0.7 * W + 0.3), F32(0.7 * W - 0.4)
    cx, cy = F32(W / 2 - 0.37), F32(H / 2 + 0.21)
    pix = rng.permutation(W * H)[:n] if n < W * H else np.arange(W * H)
    u, v = (pix % W) + 0.5, (pix // W) + 0.5
    z = rng.uniform(1, 30, n)
    cam = np.c_[(u - cx) * z / fx, (v - cy) * z / fy, z]
    R = _rot(rng)
    t = rng.uniform(-3, 3, 3)
    return ((cam - t) @ R).astype(F32), rng.uniform(0, 1, (n, 3)).astype(F32), R.astype(F32), t.astype(F32), fx, fy, cx, cy


def test_one_point_per_pixel_of_a_full_hd_frame():
    W, H = 1920, 1080
    P, cols, R, t, fx, fy, cx, cy = _grid_scene(W, H, W * H, 5)
    sel = check(P, cols, np.ones(len(P), F32), R, t, fx, fy, cx, cy, W, H, np.ones((H, W), F32), "1920x1080")
    assert sel["keep"].size == W * H                               # every pixel exactly once


@pytest.mark.parametrize("n", [1, 1023, 1024, 1025, (1 << 20) + 1, (1 << 22) + 3])
def test_scan_across_chunks(n):
    """Distinct pixels, so every flag is the filter's alone: about half kept, with the last point of every 1024-point chunk
    and the last point kept, so a carry that loses a chunk's last flag or a 31-bit position field that overflows shows."""
    W, H = (2560, 1700) if n > 1 << 20 else (1280, 1024) if n > 4096 else (64, 48)
    P, cols, R, t, fx, fy, cx, cy = _grid_scene(W, H, n, n % 977)
    rng = np.random.default_rng(n)
    rsp = np.where(rng.uniform(size=n) < 0.5, 1.0, -1.0).astype(F32)
    rsp[1023::1024] = 1.0
    rsp[-1] = 1.0
    sel = check(P, cols, rsp, R, t, fx, fy, cx, cy, W, H, np.ones((H, W), F32), "scan n=%d" % n)
    assert sel["winner"].all() and sel["keep"].size == int((rsp > 0).sum())


@pytest.mark.parametrize("W,H", [(1, 1), (1, 777), (777, 1)])
def test_degenerate_frames(W, H):
    n = 5000
    rng = np.random.default_rng(W * 7 + H)
    R, t = _rot(rng).astype(F32), rng.uniform(-1, 1, 3).astype(F32)
    fx, fy, cx, cy = F32(3.1 * max(W, H)), F32(2.9 * max(W, H)), F32(W / 2 + 0.13), F32(H / 2 - 0.07)
    z = rng.uniform(-2, 20, n)
    cam = np.c_[rng.normal(0, 0.6 * W / fx, n) * z, rng.normal(0, 0.6 * H / fy, n) * z, z]
    P = ((cam - t) @ R.astype(np.float64)).astype(F32)
    T = np.where(rng.uniform(size=(H, W)) < 0.7, 1.0, 0.005).astype(F32)
    T[0, 0] = 1.0
    rsp = rng.uniform(-0.2, 5, n).astype(F32)
    sel = check(P, rng.uniform(0, 1, (n, 3)).astype(F32), rsp, R, t, fx, fy, cx, cy, W, H, T, "%dx%d" % (W, H))
    assert sel["in_image"].sum() > 50
    compare_torch(P, rsp, R, t, fx, fy, cx, cy, W, H, T, sel, "%dx%d" % (W, H))


def test_contract():
    capi = _lib()
    W, H = 32, 24
    pts, cols, rsp, R, t, fx, fy, cx, cy, T = _scene(500, W, H, 21)
    # n = 0 and a frame where every point is rejected: count 0, nothing written
    st, m, keep, rows = _run(pts[:0], cols[:0], rsp[:0], R, t, fx, fy, cx, cy, W, H, T)
    assert st == 0 and m == 0
    st, m, keep, rows = _run(pts, cols, -np.abs(rsp) - 1, R, t, fx, fy, cx, cy, W, H, T)
    assert st == 0 and m == 0 and np.all(keep == -7)
    assert all(np.all(_bits(v) == _bits(SENTINEL)) for v in rows.values())
    # errors: count_host 0, no output row written
    need = capi.lib.glic_extend_bytes(len(pts), W, H)
    ERR_INVALID_ARGUMENT, ERR_WORKSPACE = -1, -2                  # include/glic_b200.h
    for kw, code in ((dict(ws_bytes=need - 1), ERR_WORKSPACE),
                     (dict(rot_shift=4), ERR_INVALID_ARGUMENT), (dict(rot_shift=8), ERR_INVALID_ARGUMENT),
                     (dict(null="points"), ERR_INVALID_ARGUMENT), (dict(null="colors"), ERR_INVALID_ARGUMENT),
                     (dict(null="depth"), ERR_INVALID_ARGUMENT), (dict(null="T"), ERR_INVALID_ARGUMENT)):
        st, m, keep, rows = _run(pts, cols, rsp, R, t, fx, fy, cx, cy, W, H, T, **kw)
        assert st == code and m == 0, (kw, st, m)
        assert np.all(keep == -7) and all(np.all(_bits(v) == _bits(SENTINEL)) for v in rows.values()), kw
    # the same call with room succeeds
    check(pts, cols, rsp, R, t, fx, fy, cx, cy, W, H, T, "contract")


# ---- step 5: the mapper's extend on its own final_T plane -----------------------------------------------------------------------
MW, MH, MF = 320, 208, 250.0


def _pose(m, k, pose, refined):
    """keyframe k's current pose and the camera block extend() reads: the device block when poses are refined"""
    if refined:
        return m.pose(k, camera=True)
    from gaussian_lic_b200 import mapper
    R_wc, t_wc = (np.asarray(a, F32) for a in pose)
    c = m.cfg
    return R_wc, t_wc, mapper.camera_block(MW, MH, c.fx, c.fy, c.cx, c.cy, R_wc, t_wc)


def _mapper_extend_check(m, k, pose, refined, pts, cols, dep, P0):
    """the rows the mapper appended against the restatement on render_camera's final_T at keyframe k's current camera"""
    R_wc, t_wc, cam = _pose(m, k, pose, refined)
    view = cam["view"].reshape(4, 4).T                             # column-major [R_cw | t_cw]
    R_cw, t_cw = view[:3, :3].astype(F32), view[:3, 3].astype(F32)
    T = m.render_camera(R_wc, t_wc, outputs=("final_T",))["final_T"] if P0 else np.ones((MH, MW), F32)
    inserted = m.extend(pts, cols, dep)
    c = m.cfg
    sel = eo.select(pts, dep, R_cw, t_cw, c.fx, c.fy, c.cx, c.cy, MW, MH, T)
    assert inserted == sel["keep"].size
    new = {kk: v[P0:] for kk, v in m.download().items()}
    want = sel["keep"]
    ref = torch_init(want, pts, cols, dep, c.fx, c.fy, c.scaling_scale)
    assert np.array_equal(_bits(new["means"]), _bits(pts[want]))
    assert np.array_equal(_bits(new["dc"].reshape(-1, 3)), _bits(ref["f_dc"]))
    assert np.array_equal(_bits(new["log_scales"]), _bits(ref["log_scale"]))
    assert np.array_equal(_bits(new["opacity_logits"].reshape(-1)), _bits(ref["opacity"]))
    assert np.all(new["rots"] == np.array([1, 0, 0, 0], F32)) and np.all(new["sh"] == 0)
    w = sel["winner"] & (dep > 0)
    alpha = F32(1) - T[sel["py"][w], sel["px"][w]]
    near = int((_ulps(alpha, F32(0.99)) <= 8).sum())
    opaque = int((alpha >= F32(0.99)).sum())
    closest = int(_ulps(alpha, F32(0.99)).min()) if alpha.size else -1
    print("mapper extend: kept %d of %d; winners dropped by alpha >= 0.99f: %d, with alpha within 8 ulps of 0.99f: %d "
          "(closest: %d ulps)" % (inserted, len(pts), opaque, near, closest))
    return opaque


def _scan(R_wc, t_wc, n, seed):
    rng = np.random.default_rng(seed)
    z = rng.uniform(0.5, 15.0, n)
    cam = np.stack([z * rng.uniform(-0.8, 0.8, n), z * rng.uniform(-0.6, 0.6, n), z], 1)
    pts = (cam @ np.asarray(R_wc, np.float64).T + np.asarray(t_wc, np.float64)).astype(F32)
    dep = np.where(rng.uniform(size=n) < 0.05, -1.0, z).astype(F32)
    return pts, rng.uniform(0, 1, (n, 3)).astype(F32), dep


@pytest.mark.parametrize("case", ["empty", "trained", "pose"])
def test_mapper_extend_exact(case):
    from gaussian_lic_b200 import mapper, synthetic as syn
    from helpers import small_scene
    poses = [syn.orbit_pose(v, radius=2.0) for v in (0, 1)]
    gts = [syn.make_gt_image(MW, MH, seed=3 + i) for i in range(2)]
    m = mapper.Mapper(MW, MH, MF, MF, MW / 2.0 + 3.25, MH / 2.0 - 1.5, sh_degree=3, max_iters=12, scaling_scale=1.0)
    try:
        P0 = 0
        if case != "empty":
            g, _ = small_scene(3000, MW, MH, 5, 3, log_scale_mean=-2.0)
            m.initialize(g)
            P0 = 3000
            if case == "pose":
                m.enable_pose_refinement(1e-3, 1e-3)
            m.add_keyframe(*poses[0], gts[0])
            m.optimize([0, 0, 0])
        m.add_keyframe(*poses[1], gts[1])
        if case == "pose":
            m.optimize([1, 1, 0, 1])
            R_wc, t_wc = m.pose(1)
            assert not np.array_equal(R_wc, np.asarray(poses[1][0], F32))      # the keyframe's pose has moved
        k = 0 if case == "empty" else 1                           # the newest training keyframe, at poses[1]
        refined = case == "pose"
        R_wc, t_wc, _ = _pose(m, k, poses[1], refined)
        pts, cols, dep = _scan(R_wc, t_wc, 60_000, 9)
        opaque = _mapper_extend_check(m, k, poses[1], refined, pts, cols, dep, P0)
        assert (opaque > 0) == (case != "empty")                  # on a trained map the 0.99 threshold drops winners
        if case != "empty":
            # a second scan on the grown map: the plane now includes the rows just appended
            P1 = m.stats().num_gaussians
            pts, cols, dep = _scan(R_wc, t_wc, 30_000, 10)
            _mapper_extend_check(m, k, poses[1], refined, pts, cols, dep, P1)
    finally:
        m.close()
