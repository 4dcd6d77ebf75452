"""The CPU restatement of initialize() (initialize_oracle.py; gaussian.cpp:212-304), CPU only: the sky generator's uniforms,
the LiDAR rows against an independent numpy float64 restatement of gaussian.cpp:223-240, and the sky's geometry."""
import numpy as np
import pytest

import initialize_oracle as io

# config/fastlivo.yaml:3-4 and :28
FX, FY = 431.795259219, 431.550090267
SKY_RADIUS = 1000
C0 = 0.28209479177387814                                   # gaussian.h:46


def test_sky_uniforms_grid_stability_and_seeds():
    n = 50000
    a = io.sky_uniforms(n, 7)
    assert a.shape == (n, 2) and a.dtype == np.float32
    assert np.all(a >= 0.0) and np.all(a < 1.0)
    k = a.astype(np.float64) * 2.0 ** 24                                  # on torch.rand's 2^-24 grid
    assert np.array_equal(k, np.floor(k))
    assert np.array_equal(a, io.sky_uniforms(n, 7))                       # stable for a seed
    assert np.array_equal(a[:100], io.sky_uniforms(100, 7))               # row i does not depend on n (counter-based)
    # the first row of seed 0 is SplitMix64's first output from state 0, 0xE220A8397B1DCDAF (Vigna's reference code)
    first = 0xE220A8397B1DCDAF
    assert io.sky_uniforms(1, 0)[0].tolist() == [(first >> 40) * 2.0 ** -24, ((first >> 16) & 0xFFFFFF) * 2.0 ** -24]
    b = io.sky_uniforms(n, 8)
    assert np.mean(a != b) > 0.99                                         # another seed, another sky
    # roughly uniform: means near 1/2, every tenth of [0, 1) populated near 1/10
    assert np.all(np.abs(a.mean(0) - 0.5) < 0.01)
    for c in range(2):
        h = np.histogram(a[:, c], bins=10, range=(0.0, 1.0))[0] / n
        assert np.all(np.abs(h - 0.1) < 0.01), h


@pytest.mark.parametrize("scaling_scale", [1.0, 2.0])
def test_lidar_rows_match_float64_restatement(scaling_scale):
    """gaussian.cpp:223-240 in numpy float64: every 8-bit value of every channel, depths 0.1 m .. 200 m."""
    v = np.arange(256)
    rng = np.random.default_rng(3)
    rgb = np.stack([v, rng.permutation(v), rng.permutation(v)], 1)
    rgb = np.concatenate([rgb, rng.integers(0, 256, (4000, 3))])
    n = rgb.shape[0]
    colors = rgb / 255.0                                                  # the Dataset's pointcolor_: doubles
    depth = np.concatenate([np.geomspace(0.1, 200.0, n - 2), [0.1, 200.0]]).astype(np.float32)
    pts = rng.normal(size=(n, 3)).astype(np.float32) * 30
    focal = (FX + FY) / 2
    o = io.lidar_init(pts, colors, depth, scaling_scale, focal)
    assert np.array_equal(o["xyz"], pts)
    want_dc = ((colors - 0.5) / C0).astype(np.float32)
    assert np.array_equal(o["f_dc"].view(np.uint32), want_dc.view(np.uint32))
    want_ls = np.log(scaling_scale * depth.astype(np.float64) / focal).astype(np.float32)   # numpy's log, not glibc's
    assert np.array_equal(o["log_scale"].view(np.uint32), np.repeat(want_ls[:, None], 3, 1).view(np.uint32))
    assert np.array_equal(o["rot"], np.tile(np.array([1, 0, 0, 0], np.float32), (n, 1)))
    assert np.all(o["opacity_logit"] == np.float32(np.log(np.float32(0.1) / (np.float32(1.0) - np.float32(0.1)))))
    # the double path matters: the float path of extend()'s kernel gives another f_dc on 157 of the 256 8-bit values
    via_float = ((v.astype(np.float32) / np.float32(255.0) - np.float32(0.5)) / np.float32(C0)).astype(np.float32)
    assert np.sum(via_float != ((v / 255.0 - 0.5) / C0).astype(np.float32)) == 157


def test_opacity_logits_are_correctly_rounded():
    """log(o / (1 - o)) with the ratio in float32 and the log correctly rounded: 0.1 -> -2.1972246, 0.7 -> 0.84729785"""
    for o in (0.1, 0.7):
        q = np.float32(o) / (np.float32(1.0) - np.float32(o))
        e = np.log(np.float64(q))
        got = io.logit32(o)
        below, above = np.nextafter(got, np.float32(-np.inf)), np.nextafter(got, np.float32(np.inf))
        assert abs(float(got) - e) <= min(abs(float(below) - e), abs(float(above) - e))
    assert io.logit32(0.7) == np.float32(0.84729785) and io.logit32(0.1) == np.float32(-2.1972246)


@pytest.mark.parametrize("seed", [0, 123])
def test_sky_rows_geometry(seed):
    n = 1500                                                              # the restatement's knn is O(n^2)
    o = io.sky_init(n, SKY_RADIUS, seed)
    xyz = o["xyz"].astype(np.float64)
    r = np.linalg.norm(xyz, axis=1)
    np.testing.assert_allclose(r, 10.0 * SKY_RADIUS, rtol=1e-6)
    assert np.all(xyz[:, 2] > -4000.0) and np.all(xyz[:, 2] <= 10000.0)  # phi = acos(1 - 1.4 u2), u2 in [0, 1)
    assert np.array_equal(o["f_dc"], np.tile(np.array([0.7, 0.8, 0.95], np.float32), (n, 1)))
    assert np.array_equal(o["rot"], np.tile(np.array([1, 0, 0, 0], np.float32), (n, 1)))
    assert np.all(o["opacity_logit"] == io.logit32(0.7))
    # every sky point's scale is a fraction of the cap's mean spacing: area 2 pi (10 R)^2 (1 + 0.4) shared by n points
    spacing = np.sqrt(2 * np.pi * (10.0 * SKY_RADIUS) ** 2 * 1.4 / n)
    s = np.exp(o["log_scale"][:, 0].astype(np.float64))
    assert np.all(s > 0.01 * spacing) and np.all(s < 3.0 * spacing) and 0.5 < np.median(s) / spacing < 1.5
    assert np.array_equal(o["uv"], io.sky_uniforms(n, seed))
